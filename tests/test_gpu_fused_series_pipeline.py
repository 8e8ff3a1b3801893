"""The fused kernel's one-series-ahead hand-over (csrc/fused.cu, k_fused_rollup and k_fused_series_records).

k_fused_series_records writes one record per listed series right before the fused launch; a CTA of k_fused_rollup fetches
the record of its next series, and issues that series' first fill into the idle stage buffer, while the current series
finishes.  These tests make a CTA's consecutive series differ in every way the hand-over has to carry: stream, constant and
delta-const columns; series the kernel hands back at their first, a middle or their last fill; one-fill series; lists just
below, at and above the grid; a frame without a content size, whose record must see the size the serial zstd decoder set on
the device; a corrupt frame, whose record must see the status of the decode that ran just before; and the `sum` sink.  A
context with one fused CTA per SM and a one-shot schedule puts many series on every CTA; past its first two a CTA claims
its series from a counter.  Every result is compared with
the un-fused pipeline (vmb_ctx_set_fused(0)) bit for bit, samplesScanned and error codes included."""
import base64
import hashlib
import json
import os

import numpy as np
import pytest

import blockgen
import oracle_lib as O
from conftest import SEED0
from test_baseline_configs import f64bits

T0 = 1_700_000_000_000
STEP = 15000
pytestmark = pytest.mark.gpu
SMS = 132  # VMB_SMS: with VMB_FUSED_CTAS_PER_SM=1 the fused grid is one CTA per SM


@pytest.fixture
def ctx1(monkeypatch):
    """a context whose fused grid is one CTA per SM, one-shot: CTA g runs series g and g + SMS, then claims later entries in
    list order, so every CTA runs several series back to back"""
    import victoriametrics_b200 as vm
    monkeypatch.setenv("VMB_FUSED_CTAS_PER_SM", "1")
    monkeypatch.setenv("VMB_FUSED_CHUNKS", "1")
    c = vm.Context(0)
    monkeypatch.delenv("VMB_FUSED_CTAS_PER_SM")
    monkeypatch.delenv("VMB_FUSED_CHUNKS")
    yield c
    c.close()


def _rows_both(ctx, descs, payload, nseries, func="rate", start=None, end=None, step=STEP, window=300000):
    """(rows, samplesScanned, error code) of the fused path and of the pipeline over the same uploaded blocks"""
    import torch
    import victoriametrics_b200 as vm
    from victoriametrics_b200 import VmbError
    start = T0 + 300000 if start is None else start
    end = T0 + STEP * 6000 if end is None else end
    P = 1 + (end - start) // step
    B = vm.storage.Blocks(descs, payload, ctx)
    res = []
    try:
        for fused in (True, False):
            out = torch.full((nseries, P), -7.0, dtype=torch.float64, device="cuda")
            ctx.set_fused(fused)
            code, scanned = 0, None
            try:
                _, scanned = vm.promql.eval_rollup_func(func, B, start, end, step, window, out_dev_ptr=out.data_ptr())
            except VmbError as e:
                code = e.code
            finally:
                ctx.set_fused(True)
            torch.cuda.synchronize()
            res.append((out.cpu().numpy(), scanned, code))
    finally:
        B.close()
    return res


def _assert_same(res):
    (a, sa, ca), (b, sb, cb) = res
    assert ca == cb, (ca, cb)
    assert sa == sb, (sa, sb)
    bad = np.argwhere(f64bits(a) != f64bits(b))
    assert bad.size == 0, bad[:5]


def _stale_at(rng, rows, r):
    v = blockgen.gen_values(rng, "counter", rows)
    v[r] = (1 << 63) - 2  # a staleness marker: rate() hands the series back at the fill that holds row r
    return v


def _series(rng, shape, s):
    """one block of the given shape; 6000-row `counter` columns are ~12 KB of 2-byte varints, three 4 KB fills"""
    ts = (T0 + STEP * np.arange(6000)).astype(np.int64)
    if shape == "stream":
        return blockgen.OBlock(ts, blockgen.gen_values(rng, "counter", 6000), -2, 64, s)
    if shape == "plain":  # plain nearest-delta2 varints, no zstd
        return blockgen.OBlock(ts, blockgen.gen_values(rng, "counter_big", 6000), -2, 64, s)
    if shape == "resets":
        return blockgen.OBlock(ts, blockgen.gen_values(rng, "counter_resets", 6000), -2, 64, s)
    if shape == "one_fill":  # 1200 rows: one fill
        return blockgen.OBlock(ts[:1200], blockgen.gen_values(rng, "counter", 1200), -2, 64, s)
    if shape in ("const", "delta_const"):
        return blockgen.OBlock(ts, blockgen.gen_values(rng, shape, 6000), -2, 64, s)
    if shape == "bail_first":
        return blockgen.OBlock(ts, _stale_at(rng, 6000, 100), -2, 64, s)
    if shape == "bail_middle":
        return blockgen.OBlock(ts, _stale_at(rng, 6000, 3000), -2, 64, s)
    if shape == "bail_last":
        return blockgen.OBlock(ts, _stale_at(rng, 6000, 5990), -2, 64, s)
    raise KeyError(shape)


def _cta_batch(rng, shapes, nseries):
    """shapes cycle along the list and shift every SMS entries, so that whichever series a CTA runs back to back, their
    shapes differ"""
    return [_series(rng, shapes[(s // SMS + s % len(shapes)) % len(shapes)], s) for s in range(nseries)]


def test_consecutive_series_alternate_column_kinds(ctx1):
    """stream, constant, delta-const, plain and one-fill series one after the other on every CTA"""
    rng = np.random.default_rng(SEED0 + 9301)
    blocks = _cta_batch(rng, ["stream", "const", "stream", "delta_const", "one_fill", "plain", "const", "one_fill"], 6 * SMS + 5)
    descs, payload = blockgen.to_blockset(blocks)
    _assert_same(_rows_both(ctx1, descs, payload, len(blocks)))


def test_bails_at_first_middle_and_last_fill(ctx1):
    """series handed back at their first, a middle and their last fill, directly before and after normal series"""
    rng = np.random.default_rng(SEED0 + 9302)
    shapes = ["stream", "bail_first", "stream", "bail_middle", "one_fill", "bail_last", "bail_first", "const", "bail_last",
              "resets"]
    blocks = _cta_batch(rng, shapes, 5 * SMS + 7)
    descs, payload = blockgen.to_blockset(blocks)
    res = _rows_both(ctx1, descs, payload, len(blocks))
    _assert_same(res)


@pytest.mark.parametrize("edge", [-1, 0, 1])
def test_list_around_the_grid(ctx1, edge):
    """SMS - 1, SMS and SMS + 1 series: CTAs with no series, one series, and the one CTA with a successor"""
    rng = np.random.default_rng(SEED0 + 9303 + edge)
    blocks = [_series(rng, ["stream", "one_fill", "delta_const", "plain"][s % 4], s) for s in range(SMS + edge)]
    descs, payload = blockgen.to_blockset(blocks)
    _assert_same(_rows_both(ctx1, descs, payload, len(blocks)))


def _fixture_frames(names):
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "zstd_shapes.json")) as f:
        cases = {e["name"]: e for e in json.load(f)}
    out = []
    for n in names:
        e = cases[n]
        frame = base64.b64decode(e["frame"])
        assert hashlib.sha256(frame).hexdigest() == e["frame_sha256"], n
        out.append((e["mt"], e["rows"], e["first"], np.frombuffer(frame, np.uint8)))
    return out


def _mixed_blockset(rng, frames, nseries, every):
    """counter series, and every `every`-th series a values column from the zstd fixture (timestamps delta-const)"""
    import victoriametrics_b200 as vm
    bs = vm.storage.BlockSet()
    tdelta = O.marshal_varint64s([STEP])
    for s in range(nseries):
        if s % every == every // 2:
            mt, n, first, frame = frames[(s // every) % len(frames)]
            bs.add_marshaled(dict(first_value=first, min_ts=T0, max_ts=T0 + STEP * (n - 1), ts_size=tdelta.size,
                                  val_size=frame.size, rows=n, series_idx=s, scale=-2, ts_mt=2, val_mt=mt, precision_bits=64),
                             tdelta, frame)
        else:
            b = _series(rng, ["stream", "one_fill"][s % 2], s)
            bs.add_marshaled(b.header(), b.tdata, b.vdata)
    return bs.finish()


def test_frames_without_content_size(ctx1):
    """frames without Frame_Content_Size take the serial decoder, which sets their content size on the device: the records
    written after it must see that size"""
    rng = np.random.default_rng(SEED0 + 9304)
    frames = _fixture_frames(["seq_no_fcs", "seq_rle_literals_no_fcs"])
    n = 3 * SMS + 11
    descs, payload = _mixed_blockset(rng, frames, n, 5)
    res = _rows_both(ctx1, descs, payload, n, func="max_over_time", start=T0, end=T0 + STEP * 6000, step=60000)
    assert res[0][2] == 0
    _assert_same(res)


def test_corrupt_frame(ctx1):
    """a frame the zstd stage fails: the record of its series sees that status, the call fails on both paths with the same
    code and every other row is the same"""
    rng = np.random.default_rng(SEED0 + 9305)
    frames = _fixture_frames(["err_no_fcs_truncated", "seq_no_fcs"])
    n = 2 * SMS + 3
    descs, payload = _mixed_blockset(rng, frames, n, 7)
    res = _rows_both(ctx1, descs, payload, n)
    assert res[0][2] == -53  # VMB_ERR_BLOCK_FAILED
    _assert_same(res)


def test_sum_sink_by_groups(ctx1):
    """sum(rate) by (g) folded inside the fused kernel, scale-0 integer samples, bit for bit with samplesScanned"""
    import torch
    import victoriametrics_b200 as vm
    rng = np.random.default_rng(SEED0 + 9306)
    shapes = ["stream", "const", "bail_middle", "one_fill", "delta_const", "bail_first"]
    blocks = _cta_batch(rng, shapes, 3 * SMS + 2)
    for b in blocks:
        b.scale = 0
    n, G = len(blocks), 5
    groups = ((np.arange(n) * 3) % G).astype(np.uint32)
    start, end, step, window = T0 + 300000, T0 + STEP * 6000, STEP, 300000
    rc = vm.promql.get_rollup_configs("increase", start, end, step, window)
    descs, payload = blockgen.to_blockset(blocks)
    B = vm.storage.Blocks(descs, payload, ctx1)

    class Buf:
        def __init__(self, nbytes):
            self.t = torch.empty(nbytes // 8, dtype=torch.float64, device="cuda")
            self.ptr = self.t.data_ptr()
    res = {}
    try:
        for fused in (True, False):
            ctx1.set_fused(fused)
            try:
                ia = vm.promql.IncrementalAggr("sum", G, rc.points, Buf)
                sc = ia.update_blocks(B, rc, groups)
                res[fused] = (ia.finalize(ctx1), sc)
            finally:
                ctx1.set_fused(True)
    finally:
        B.close()
    assert res[True][1] == res[False][1]
    assert np.array_equal(f64bits(res[True][0]), f64bits(res[False][0]))
