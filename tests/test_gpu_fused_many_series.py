"""The fused kernel (csrc/fused.cu) over batches large enough that every CTA of its persistent grid runs several series back to
back: the stage buffer and the mbarrier phase parities carry over from one series to the next, and the per-series setup is
rewritten in shared memory.  The batches interleave series the kernel hands back to the pipeline (stale markers, windows
wider than the resident rows, more than FU_MAX_EVENTS drops in one fill, corrupt streams) and series it never takes (several
blocks, jittered timestamps) with good ones, stream columns with const / delta-const ones, and vary the first sample and the
scrape interval per series.  The fused path must match the pipeline (vmb_ctx_set_fused(0)) bit for bit, values and
samplesScanned, with and without an incremental `sum` aggregate."""
import numpy as np
import pytest

import blockgen
from conftest import SEED0
from test_baseline_configs import f64bits

T0 = 1_700_000_000_000
pytestmark = pytest.mark.gpu

KINDS = ["counter", "const", "counter_resets", "delta_const", "gauge", "counter_smooth", "counter_big"]


SCRAPES = [15000, 10000, 30000, 7000, 60000, 15000, 1000]


def _grid():
    """the fused kernel's grid for rate() on this device (vmb_fused_grid)"""
    from victoriametrics_b200 import _lib
    g = int(_lib.lib().vmb_fused_grid())
    assert 132 <= g <= 132 * 5, g
    return g


def _ts(rng, rows):
    """regular timestamps with a per-series first sample and scrape interval, so that the per-series setup (window edges,
    rate() divisors, query grid relative to the first row) differs from one series to the next"""
    dt = SCRAPES[int(rng.integers(0, len(SCRAPES)))]
    return (T0 + int(rng.integers(-900000, 900000)) + dt * np.arange(rows)).astype(np.int64)


def _series(rng, s, rows, hand_back, scale):
    """one series (a list of blocks) of kind s % len(KINDS); every few series one of the shapes the kernel hands back"""
    kind = KINDS[s % len(KINDS)]
    ts = _ts(rng, rows)
    v = blockgen.gen_values(rng, kind, rows)
    c = s % 13
    if hand_back and c == 3:  # a staleness marker: removeCounterResets / dropStaleNaNs hand the series back
        v = blockgen.gen_values(rng, "counter", rows)
        v[int(rng.integers(1, rows))] = (1 << 63) - 2
    elif hand_back and c == 6:  # 50 ms scrape: a 5 m window holds 6000 rows, more than the ring's 4096
        rows = 6000
        ts = (T0 + 50 * np.arange(rows)).astype(np.int64)
        v = blockgen.gen_values(rng, "counter", rows)
    elif hand_back and c == 9 and rows > 400:  # a reset every 4 rows: more than 32 value drops inside one 4 KB fill
        v = blockgen.gen_values(rng, "counter", rows)
        for r in range(100, 400, 4):
            v[r:] -= v[r] - 1
    return [blockgen.OBlock(ts, v, scale, 64, s)]


def _batch(rng, nseries, hand_back=True, not_taken=True, rows=(150, 2600), scale=-2):
    blocks = []
    for s in range(nseries):
        n = int(rng.integers(rows[0], rows[1]))
        if not_taken and s % 11 == 4:  # jittered timestamps: never taken by the kernel
            ts = blockgen.gen_timestamps(rng, "jitter", n, T0 + int(rng.integers(-900000, 900000)))
            blocks.append(blockgen.OBlock(ts, blockgen.gen_values(rng, "counter", n), scale, 64, s))
            continue
        blocks += _series(rng, s, n, hand_back, scale)
        if not_taken and s % 11 == 8:  # a second, later block: a multi-block series
            t2 = blockgen.gen_timestamps(rng, "regular", 300, int(blocks[-1].ts[-1]) + 15000)
            blocks.append(blockgen.OBlock(t2, blockgen.gen_values(rng, "counter", 300), scale, 64, s))
    return blocks


def _rollup(vm, ctx, B, func, nseries, start, end, step, window, fused):
    import torch
    P = 1 + (end - start) // step
    out = torch.full((nseries, P), -7.0, dtype=torch.float64, device="cuda")
    ctx.set_fused(fused)
    try:
        _, scanned = vm.promql.eval_rollup_func(func, B, start, end, step, window, out_dev_ptr=out.data_ptr())
    finally:
        ctx.set_fused(True)
    torch.cuda.synchronize()
    return out.cpu().numpy(), scanned


def _check_rollup(vm, blocks, func, nseries, start, end, step, window):
    ctx = vm.default_context()
    descs, payload = blockgen.to_blockset(blocks)
    B = vm.storage.Blocks(descs, payload, ctx)
    try:
        a, sa = _rollup(vm, ctx, B, func, nseries, start, end, step, window, True)
        b, sb = _rollup(vm, ctx, B, func, nseries, start, end, step, window, False)
    finally:
        B.close()
    assert sa == sb, (func, nseries, sa, sb)
    bad = np.argwhere(f64bits(a) != f64bits(b))
    assert bad.size == 0, (func, nseries, bad[:5])


@pytest.mark.parametrize("func", ["rate", "increase", "avg_over_time", "max_over_time"])
def test_fused_many_series_per_cta(func):
    """4000 series, about six per CTA: every CTA runs several series, next to hand-backs and series it never takes"""
    import victoriametrics_b200 as vm
    rng = np.random.default_rng(SEED0 + 6060)
    n = 4000
    blocks = _batch(rng, n)
    _check_rollup(vm, blocks, func, n, T0 + 300000, T0 + 15000 * 2700, 15000, 300000)


@pytest.mark.parametrize("edge", [-1, 0, 1, "2g+1"])
def test_fused_series_list_around_the_grid_size(edge):
    """the kernel's series list just below, at and above the grid: CTAs with zero, one and two series"""
    import victoriametrics_b200 as vm
    vm.default_context()
    g = _grid()
    nlist = 2 * g + 1 if edge == "2g+1" else g + edge
    rng = np.random.default_rng(SEED0 + 7070 + nlist)
    blocks = _batch(rng, nlist, not_taken=False, rows=(150, 1200))
    _check_rollup(vm, blocks, "rate", nlist, T0 + 300000, T0 + 15000 * 1300, 15000, 300000)


def test_fused_many_series_next_to_corrupt_streams():
    """corrupt plain streams among many good series: the call fails (VMB_ERR_BLOCK_FAILED) on both paths and every other row
    is the same"""
    import torch
    import victoriametrics_b200 as vm
    from victoriametrics_b200 import VmbError
    rng = np.random.default_rng(SEED0 + 8080)
    vm.default_context()
    n = 3 * _grid()
    blocks = _batch(rng, n, not_taken=False, rows=(300, 1500))
    for i, b in enumerate(blocks):
        if b.vmt == 5 and i % 3 == 0:  # plain nearest-delta2 varints: corrupt them directly
            v = b.vdata.copy()
            v[-1] |= 0x80
            b.vdata = v
    ctx = vm.default_context()
    descs, payload = blockgen.to_blockset(blocks)
    B = vm.storage.Blocks(descs, payload, ctx)
    start, end, step, window = T0 + 300000, T0 + 15000 * 1500, 15000, 300000
    P = 1 + (end - start) // step
    res = []
    try:
        for fused in (True, False):
            out = torch.full((n, P), -7.0, dtype=torch.float64, device="cuda")
            ctx.set_fused(fused)
            try:
                with pytest.raises(VmbError) as ei:
                    vm.promql.eval_rollup_func("rate", B, start, end, step, window, out_dev_ptr=out.data_ptr())
            finally:
                ctx.set_fused(True)
            assert ei.value.code == -53
            torch.cuda.synchronize()
            res.append(out.cpu().numpy())
    finally:
        B.close()
    assert np.array_equal(f64bits(res[0]), f64bits(res[1]))


def test_fused_many_series_with_sum_sink():
    """sum(increase(m[5m])) by (g), folded inside the fused kernel: integer samples at scale 0 make every partial sum exact,
    so the fold order does not matter and the result is compared bit for bit, with samplesScanned"""
    import torch
    import victoriametrics_b200 as vm
    rng = np.random.default_rng(SEED0 + 9090)
    n, G = 4000, 37
    blocks = _batch(rng, n, scale=0, rows=(150, 1800))
    groups = ((np.arange(n) * 7) % G).astype(np.uint32)
    start, end, step, window = T0 + 300000, T0 + 15000 * 1900, 15000, 300000
    rc = vm.promql.get_rollup_configs("increase", start, end, step, window)
    ctx = vm.default_context()
    descs, payload = blockgen.to_blockset(blocks)
    B = vm.storage.Blocks(descs, payload, ctx)

    class Buf:
        def __init__(self, nbytes):
            self.t = torch.empty(nbytes // 8, dtype=torch.float64, device="cuda")
            self.ptr = self.t.data_ptr()
    res = {}
    try:
        for fused in (True, False):
            ctx.set_fused(fused)
            try:
                ia = vm.promql.IncrementalAggr("sum", G, rc.points, Buf)
                sc = ia.update_blocks(B, rc, groups)
                res[fused] = (ia.finalize(ctx), sc)
            finally:
                ctx.set_fused(True)
    finally:
        B.close()
    assert res[True][1] == res[False][1]
    assert np.array_equal(f64bits(res[True][0]), f64bits(res[False][0]))
