"""The fused decode+rollup kernel (csrc/fused.cu) against (a) the kernel-per-stage pipeline, bit for bit, and (b) the oracle.

vmb_eval_rollup_device sends every series that qualifies (one block, MarshalTypeDeltaConst timestamps at precisionBits 64)
through the fused kernel and everything else -- including what the kernel hands back at run time -- through the un-fused
pipeline; vmb_ctx_set_fused(0) forces the pipeline for every series.  Both must produce the same bits and the same
samplesScanned (rollup.go:688), whatever the mix of series."""
import ctypes as C

import numpy as np
import pytest

import blockgen
from conftest import SEED0
from rollup_names import RF
from test_baseline_configs import _oracle_rollup_matrix, f64bits

T0 = 1_700_000_000_000
pytestmark = pytest.mark.gpu


def _eval(vm, ctx, B, func, start, end, step, window, nseries, lookback=0, args=None, tr=None, fused=True):
    import torch
    P = 1 + (end - start) // step
    out = torch.full((nseries, P), -7.0, dtype=torch.float64, device="cuda")
    ctx.set_fused(fused)
    kw = {}
    if tr is not None:
        kw = dict(tr_min=tr[0], tr_max=tr[1])
    try:
        _, scanned = vm.promql.eval_rollup_func(func, B, start, end, step, window, lookback, args=args, out_dev_ptr=out.data_ptr(), **kw)
    finally:
        ctx.set_fused(True)
    torch.cuda.synchronize()
    return out.cpu().numpy(), scanned


def _both(vm, blocks, func, start, end, step, window, lookback=0, args=None, tr=None):
    ctx = vm.default_context()
    descs, payload = blockgen.to_blockset(blocks)
    B = vm.storage.Blocks(descs, payload, ctx)
    n = len({b.series_idx for b in blocks})
    a, sa = _eval(vm, ctx, B, func, start, end, step, window, n, lookback, args, tr, fused=True)
    b, sb = _eval(vm, ctx, B, func, start, end, step, window, n, lookback, args, tr, fused=False)
    B.close()
    return a, sa, b, sb


VALUE_FUNCS = ["rate", "increase", "delta", "avg_over_time", "min_over_time", "max_over_time", "sum_over_time", "count_over_time",
               "quantile_over_time", "default_rollup", "last_over_time", "first_over_time", "stddev_over_time", "changes",
               "resets", "increase_pure", "idelta", "median_over_time", "distinct_over_time", "rate_over_sum", "geomean_over_time"]
TS_FUNCS = ["irate", "deriv", "lag", "lifetime", "scrape_interval", "integrate", "tmin_over_time", "tmax_over_time",
            "tfirst_over_time", "tlast_over_time", "tlast_change_over_time", "timestamp", "zscore_over_time", "duration_over_time",
            "predict_linear", "rollup_high", "rollup_open", "ideriv"]


@pytest.mark.parametrize("func", VALUE_FUNCS + TS_FUNCS)
def test_fused_equals_pipeline_and_oracle_per_function(oracle, func):
    import victoriametrics_b200 as vm
    rng = np.random.default_rng(SEED0 + 4242 + len(func))
    kinds = ["counter", "counter_resets", "counter_smooth", "gauge", "gauge_small", "const", "delta_const", "counter_big", "gauge_wide"]
    rows = [8192, 8191, 4097, 513, 100, 33, 2, 3000]
    blocks = [blockgen.OBlock(blockgen.gen_timestamps(rng, "regular", rows[i % len(rows)], T0), blockgen.gen_values(rng, k, rows[i % len(rows)]),
                              -2, 64, i) for i, k in enumerate(kinds * 3)]
    start, end, step, window = T0 + 300000, T0 + 15000 * 8200, 15000, 300000
    P = 1 + (end - start) // step
    args = None
    if func in ("quantile_over_time",):
        args = np.full(P, 0.9)
    if func in ("duration_over_time",):
        args = np.full(P, 20.0)
    if func in ("predict_linear",):
        args = np.full(P, 60.0)
    a, sa, b, sb = _both(vm, blocks, func, start, end, step, window, args=args)
    assert sa == sb
    assert np.array_equal(f64bits(a), f64bits(b)), np.argwhere(f64bits(a) != f64bits(b))[:5]
    exp = _oracle_rollup_matrix(oracle, blocks, func, start, end, step, window, arg=args)
    assert np.array_equal(np.isnan(a), np.isnan(exp))
    assert np.allclose(a, exp, rtol=1e-12, atol=0, equal_nan=True)


GRIDS = [  # (start offset, step, window, lookback)
    (300000, 15000, 300000, 0),
    (300000, 15000, 300000, 600000),
    (1, 15000, 300000, 0),           # grid not aligned with the samples
    (7777, 7001, 33333, 0),          # step and window unrelated to the scrape interval
    (60000, 60000, 3600000, 0),      # increase(m[1h]) step 60 s: 240 rows per window
    (300000, 15000, 0, 0),           # window derived from the step / scrape interval
    (300000, 30000, 15000, 0),       # windows shorter than the step
    (-500000, 15000, 300000, 0),     # the grid starts before the series
    (300000, 5000, 1000, 0),         # windows shorter than the scrape interval
    (300000, 15000, 90000000, 0),    # a window larger than the resident rows: handed to the pipeline
    (300000, 15000, 300000, 1000),   # staleness interval around the scrape interval
    (300000, 15000, 10000, 5000),    # lookback below the scrape interval (removeCounterResets leaves rows raw)
]


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("func", ["rate", "increase", "avg_over_time", "lag", "default_rollup"])
def test_fused_query_grids(oracle, func, grid):
    import victoriametrics_b200 as vm
    rng = np.random.default_rng(SEED0 + 777)
    kinds = ["counter", "counter_resets", "gauge", "counter_smooth"]
    blocks = [blockgen.OBlock(blockgen.gen_timestamps(rng, "regular", 8192, T0), blockgen.gen_values(rng, k, 8192), -2, 64, i)
              for i, k in enumerate(kinds * 2)]
    so, step, window, lookback = grid
    start = T0 + so
    end = T0 + 15000 * 8300
    a, sa, b, sb = _both(vm, blocks, func, start, end, step, window, lookback)
    assert sa == sb
    assert np.array_equal(f64bits(a), f64bits(b)), (grid, np.argwhere(f64bits(a) != f64bits(b))[:5])
    exp = _oracle_rollup_matrix(oracle, blocks, func, start, end, step, window, lookback)
    assert np.allclose(a, exp, rtol=1e-12, atol=0, equal_nan=True), grid


def test_fused_mixed_batch_with_series_the_kernel_does_not_take(oracle):
    """jittered timestamp columns, a multi-block series, staleness markers, a time range that trims rows, one-row blocks: all of
    them in one batch next to series the fused kernel takes"""
    import victoriametrics_b200 as vm
    rng = np.random.default_rng(SEED0 + 99)
    blocks = []
    s = 0
    for k in range(40):
        kind = ["counter", "gauge", "counter_resets"][k % 3]
        tk = "jitter" if k % 5 == 1 else "regular"
        rows = [8192, 1, 2, 777][k % 4] if k % 7 == 3 else 4096
        v = blockgen.gen_values(rng, kind, rows)
        if k % 11 == 5 and rows > 10:
            v = v.copy()
            v[rng.integers(1, rows, 3)] = (1 << 63) - 2  # staleness markers (decimal.go:406)
        blocks.append(blockgen.OBlock(blockgen.gen_timestamps(rng, tk, rows, T0), v, -2, 64, s))
        s += 1
        if k % 13 == 6:  # a series of two time-disjoint blocks
            t2 = blockgen.gen_timestamps(rng, "regular", 2048, T0 + 15000 * 5000)
            blocks.append(blockgen.OBlock(t2, blockgen.gen_values(rng, "counter", 2048), -2, 64, s - 1))
    start, end, step, window = T0 + 300000, T0 + 15000 * 7000, 15000, 300000
    for func in ("rate", "avg_over_time", "default_rollup"):
        for tr in (None, (T0 + 15000 * 100 + 1, T0 + 15000 * 3000)):
            a, sa, b, sb = _both(vm, blocks, func, start, end, step, window, tr=tr)
            assert sa == sb, (func, tr)
            assert np.array_equal(f64bits(a), f64bits(b)), (func, tr)


def test_fused_corrupt_streams_fail_like_the_pipeline(oracle):
    """a corrupted values stream makes the series fail (VMB_ERR_BLOCK_FAILED) with or without the fused kernel, and does not
    disturb its neighbours"""
    import torch
    import victoriametrics_b200 as vm
    from victoriametrics_b200 import VmbError
    rng = np.random.default_rng(SEED0 + 5)
    blocks = [blockgen.OBlock(blockgen.gen_timestamps(rng, "regular", 4096, T0), blockgen.gen_values(rng, "counter_big", 4096), -2, 64, i)
              for i in range(12)]
    assert all(b.vmt == 5 for b in blocks)  # plain varint streams: corrupt them directly
    mutations = {2: "truncate", 5: "tail", 7: "long", 9: "contbit"}
    for i, m in mutations.items():
        v = blocks[i].vdata.copy()
        if m == "truncate":
            v = v[:len(v) // 2]
        elif m == "tail":
            v = np.concatenate([v, np.array([1, 2, 3], dtype=np.uint8)])
        elif m == "long":
            v[100:112] = 0x80
        else:
            v[-1] |= 0x80
        blocks[i].vdata = v
    descs, payload = blockgen.to_blockset(blocks)
    ctx = vm.default_context()
    B = vm.storage.Blocks(descs, payload, ctx)
    start, end, step, window = T0 + 300000, T0 + 15000 * 4095, 15000, 300000
    P = 1 + (end - start) // step
    res = []
    for fused in (True, False):
        out = torch.zeros((12, P), dtype=torch.float64, device="cuda")
        ctx.set_fused(fused)
        with pytest.raises(VmbError) as ei:
            vm.promql.eval_rollup_func("rate", B, start, end, step, window, out_dev_ptr=out.data_ptr())
        ctx.set_fused(True)
        assert ei.value.code == -53
        torch.cuda.synchronize()
        res.append(out.cpu().numpy())
    assert np.array_equal(f64bits(res[0]), f64bits(res[1]))
    good = [i for i in range(12) if i not in mutations]
    exp = _oracle_rollup_matrix(oracle, [blocks[i] for i in good], "rate", start, end, step, window)
    assert np.allclose(res[0][good], exp, rtol=1e-12, atol=0, equal_nan=True)
    # the same through the incremental aggregate (vmb_eval_rollup_aggr_device): the corrupt series are alone in group 0, the
    # aggregate of the other groups is the oracle's fold of the good series
    from rollup_names import AGGR
    G = 4
    groups = np.array([0 if i in mutations else 1 + i % (G - 1) for i in range(12)], dtype=np.uint32)
    rc = vm.promql.get_rollup_configs("rate", start, end, step, window)

    class Buf:
        def __init__(self, nbytes):
            self.t = torch.empty(nbytes // 8, dtype=torch.float64, device="cuda")
            self.ptr = self.t.data_ptr()
    e_v, e_c = np.zeros((G, P)), np.zeros((G, P))
    for k, i in enumerate(good):
        row = np.ascontiguousarray(exp[k])
        oracle.lib().vmo_aggr_update(AGGR["sum"], e_v[groups[i]].ctypes.data_as(oracle.f64p), e_c[groups[i]].ctypes.data_as(oracle.f64p),
                                     row.ctypes.data_as(oracle.f64p), P)
    for g in range(G):
        oracle.lib().vmo_aggr_finalize(AGGR["sum"], e_v[g].ctypes.data_as(oracle.f64p), e_c[g].ctypes.data_as(oracle.f64p), P)
    for fused in (True, False):
        ia = vm.promql.IncrementalAggr("sum", G, P, Buf)
        ctx.set_fused(fused)
        with pytest.raises(VmbError) as ei:
            ia.update_blocks(B, rc, groups)
        ctx.set_fused(True)
        assert ei.value.code == -53, fused
        got = ia.finalize(ctx)
        assert np.allclose(got[1:], e_v[1:], rtol=1e-12, atol=0, equal_nan=True), fused


@pytest.mark.parametrize("entry", ["aggr_device_fused", "aggr_device_unfused", "aggr_host", "rollup_aggr_partial", "topk_candidates"])
def test_group_id_out_of_range_is_rejected(entry):
    """a group id >= ngroups is an invalid argument (-50) for every entry point that groups series"""
    import torch
    import victoriametrics_b200 as vm
    from victoriametrics_b200 import VmbError
    rng = np.random.default_rng(SEED0 + 50)
    S, G = 8, 3
    blocks = [blockgen.OBlock(blockgen.gen_timestamps(rng, "regular", 1024, T0), blockgen.gen_values(rng, "counter", 1024), -2, 64, i)
              for i in range(S)]
    groups = (np.arange(S) % G).astype(np.uint32)
    groups[5] = G
    start, end, step, window = T0 + 300000, T0 + 15000 * 1000, 15000, 300000
    rc = vm.promql.get_rollup_configs("rate", start, end, step, window)
    descs, payload = blockgen.to_blockset(blocks)
    ctx = vm.default_context()

    class Buf:
        def __init__(self, nbytes):
            self.t = torch.empty(max(nbytes // 8, 1), dtype=torch.float64, device="cuda")
            self.ptr = self.t.data_ptr()
    B = vm.storage.Blocks(descs, payload, ctx)
    try:
        with pytest.raises(VmbError) as ei:
            if entry.startswith("aggr_device"):
                ctx.set_fused(entry == "aggr_device_fused")
                try:
                    vm.promql.IncrementalAggr("sum", G, rc.points, Buf).update_blocks(B, rc, groups)
                finally:
                    ctx.set_fused(True)
            elif entry == "aggr_host":
                vm.promql.eval_rollup_aggr_host("sum", "rate", descs, payload, groups, G, start, end, step, window, ctx=ctx)
            elif entry == "rollup_aggr_partial":
                series, _ = vm.storage.decode_blocks(B)
                try:
                    vm.promql.IncrementalAggr("sum", G, rc.points, Buf).update(series, rc, groups)
                finally:
                    series.close()
            else:
                vals = torch.zeros((S, rc.points), dtype=torch.float64, device="cuda")
                vm.promql.topk(2, vals.data_ptr(), S, rc.points, Buf, group_ids=groups, ngroups=G, ctx=ctx)
        assert ei.value.code == -50
    finally:
        B.close()


def test_fused_unaligned_plain_streams_and_all_varint_widths(oracle):
    """plain (not zstd) varint streams start at arbitrary byte offsets of the payload arena; values of every varint width from
    1 to 10 bytes, widths changing inside a block"""
    import victoriametrics_b200 as vm
    rng = np.random.default_rng(SEED0 + 31337)
    blocks = []
    for i in range(48):
        rows = int(rng.integers(2, 8193))
        width = rng.integers(0, 63, rows)
        inc = (rng.integers(0, 1 << 62, rows) >> (62 - width)).astype(np.int64) * rng.choice([-1, 1], rows)
        if i % 3 == 0:
            inc = np.abs(inc)
        v = np.cumsum(inc.astype(np.int64))  # wraps like Go
        blocks.append(blockgen.OBlock(blockgen.gen_timestamps(rng, "regular", rows, T0), v, int(rng.choice([-2, 0, 3])), 64, i))
    start, end, step, window = T0 + 300000, T0 + 15000 * 8200, 15000, 300000
    for func in ("increase", "max_over_time", "delta"):
        a, sa, b, sb = _both(vm, blocks, func, start, end, step, window)
        assert sa == sb
        assert np.array_equal(f64bits(a), f64bits(b)), func
        exp = _oracle_rollup_matrix(oracle, blocks, func, start, end, step, window)
        assert np.allclose(a, exp, rtol=1e-12, atol=0, equal_nan=True), func


@pytest.mark.parametrize("aggr", ["sum", "avg", "count", "min", "max", "sum2", "group", "geomean", "any"])
def test_fused_incremental_aggregate(oracle, aggr):
    """aggr(rollup(m[d])) by (g) with the fold inside the fused kernel (vmb_eval_rollup_aggr_device): every finished series is folded
    into {values, counts}[G x P] from the kernel; series the kernel hands back (jittered timestamps, staleness markers, several
    blocks) are folded by the pipeline into the same state.  geomean / any have no atomic fold: they take the pipeline."""
    import torch
    import victoriametrics_b200 as vm
    from rollup_names import AGGR
    rng = np.random.default_rng(SEED0 + 2024)
    blocks, s = [], 0
    for k in range(60):
        kind = ["counter", "gauge", "counter_resets", "gauge_small"][k % 4]
        tk = "jitter" if k % 6 == 1 else "regular"
        v = blockgen.gen_values(rng, kind, 3000)
        if k % 10 == 7:
            v = v.copy()
            v[rng.integers(1, 3000, 2)] = (1 << 63) - 2
        blocks.append(blockgen.OBlock(blockgen.gen_timestamps(rng, tk, 3000, T0), v, -2, 64, s))
        s += 1
    S, G = s, 7
    groups = (np.arange(S) * 5 % G).astype(np.uint32)
    start, end, step, window = T0 + 300000, T0 + 15000 * 2990, 15000, 300000
    func = "rate" if aggr not in ("min", "max") else "avg_over_time"
    rc = vm.promql.get_rollup_configs(func, start, end, step, window)
    descs, payload = blockgen.to_blockset(blocks)
    ctx = vm.default_context()
    B = vm.storage.Blocks(descs, payload, ctx)

    class Buf:
        def __init__(self, nbytes):
            self.t = torch.empty(nbytes // 8, dtype=torch.float64, device="cuda")
            self.ptr = self.t.data_ptr()
    res = {}
    for fused in (True, False):
        ctx.set_fused(fused)
        try:
            ia = vm.promql.IncrementalAggr(aggr, G, rc.points, Buf)
            sc = ia.update_blocks(B, rc, groups)
            res[fused] = (ia.finalize(ctx), sc)
        finally:
            ctx.set_fused(True)
    assert res[True][1] == res[False][1]
    rolled = _oracle_rollup_matrix(oracle, blocks, func, start, end, step, window)
    e_v, e_c = np.zeros((G, rc.points)), np.zeros((G, rc.points))
    for s_ in range(S):
        row = np.ascontiguousarray(rolled[s_])
        g = int(groups[s_])
        oracle.lib().vmo_aggr_update(AGGR[aggr], e_v[g].ctypes.data_as(oracle.f64p), e_c[g].ctypes.data_as(oracle.f64p),
                                     row.ctypes.data_as(oracle.f64p), rc.points)
    for g in range(G):
        oracle.lib().vmo_aggr_finalize(AGGR[aggr], e_v[g].ctypes.data_as(oracle.f64p), e_c[g].ctypes.data_as(oracle.f64p), rc.points)
    for fused in (True, False):
        got = res[fused][0]
        assert np.array_equal(np.isnan(got), np.isnan(e_v)), (aggr, fused)
        assert np.allclose(got, e_v, rtol=1e-12, atol=0, equal_nan=True), (aggr, fused)
    if aggr in ("min", "max", "count", "group"):  # order independent
        assert np.array_equal(f64bits(res[True][0]), f64bits(res[False][0]))
