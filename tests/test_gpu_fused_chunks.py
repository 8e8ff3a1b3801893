"""The chunked fused schedule (eval_fused in csrc/api.cu) against the one-shot one, bit for bit.

vmb_eval_rollup_device cuts the fused series into VMB_FUSED_CHUNKS chunks and runs the zstd stage of chunk k + 1 on a second
stream beside the fused kernel of chunk k; VMB_FUSED_CHUNKS=1 decodes every column first and launches the fused kernel once.
Both must write the same bits, the same samplesScanned and the same error code, whatever lies at the chunk edges (the sum sink,
whose atomic fold order is not fixed in either schedule, to 1e-12)."""
import numpy as np
import pytest

import blockgen
from conftest import SEED0
from test_baseline_configs import f64bits

T0 = 1_700_000_000_000
pytestmark = pytest.mark.gpu
CHUNKS = 4


def _contexts(monkeypatch):
    import victoriametrics_b200 as vm
    ctxs = {}
    for c in (CHUNKS, 1):
        monkeypatch.setenv("VMB_FUSED_CHUNKS", str(c))
        ctxs[c] = vm.Context(0)
    monkeypatch.delenv("VMB_FUSED_CHUNKS")
    return ctxs


def _rollup(blocks, monkeypatch, func="rate", rows=None):
    """(output, samplesScanned, error code) of both schedules over the same uploaded blocks"""
    import torch
    import victoriametrics_b200 as vm
    from victoriametrics_b200 import VmbError
    rows = rows or blocks[0].rows
    nseries = len({b.series_idx for b in blocks})
    start, end, step, window = T0 + 60000, T0 + 15000 * (rows - 1), 15000, 120000
    P = 1 + (end - start) // step
    descs, payload = blockgen.to_blockset(blocks)
    ctxs = _contexts(monkeypatch)
    B = vm.storage.Blocks(descs, payload, ctxs[CHUNKS])
    res, launches = {}, {}
    for c, ctx in ctxs.items():
        B.ctx = ctx
        out = torch.full((nseries, P), -7.0, dtype=torch.float64, device="cuda")
        code, scanned = 0, None
        n0 = ctx.launch_count
        try:
            _, scanned = vm.promql.eval_rollup_func(func, B, start, end, step, window, out_dev_ptr=out.data_ptr())
        except VmbError as e:
            code = e.code
        launches[c] = ctx.launch_count - n0
        torch.cuda.synchronize()
        res[c] = (out.cpu().numpy(), scanned, code)
    # the chunked schedule ran: a fused launch and a zstd stage per chunk
    assert launches[CHUNKS] > launches[1], launches
    B.ctx = ctxs[CHUNKS]
    B.close()
    for ctx in ctxs.values():
        ctx.close()
    return res


def _assert_same(res):
    a, b = res[CHUNKS], res[1]
    assert a[2] == b[2]
    assert a[1] == b[1]
    assert np.array_equal(f64bits(a[0]), f64bits(b[0])), np.argwhere(f64bits(a[0]) != f64bits(b[0]))[:5]


def _block(rng, kind, rows, s, ts_kind="regular", scale=-2):
    return blockgen.OBlock(blockgen.gen_timestamps(rng, ts_kind, rows, T0), blockgen.gen_values(rng, kind, rows), scale, 64, s)


def _zstd(b):
    return b.vmt in (1, 4)  # MarshalTypeZSTDNearestDelta2 / MarshalTypeZSTDNearestDelta


def _literals_section(frame):
    """[begin, end) of the Huffman-compressed literals section of a one-block zstd frame without a checksum (the shape the
    library decodes with k_huf_decode), or None for any other shape (RFC 8878 3.1.1, 3.1.1.3.1)"""
    frame = bytes(frame)
    fhd = frame[4]
    fcs_flag, single, checksum, did = fhd >> 6, (fhd >> 5) & 1, (fhd >> 2) & 1, fhd & 3
    pos = 5 + (0 if single else 1) + (0, 1, 2, 4)[did] + ((1 if single else 0), 2, 4, 8)[fcs_flag]
    bh = frame[pos] | (frame[pos + 1] << 8) | (frame[pos + 2] << 16)
    blk = pos + 3
    if checksum or not (bh & 1) or ((bh >> 1) & 3) != 2 or blk + (bh >> 3) != len(frame):
        return None
    b0 = frame[blk]
    if b0 & 3 != 2:
        return None
    sf = (b0 >> 2) & 3
    v = int.from_bytes(frame[blk:blk + 5], "little")
    hdr, csize = (3, (v >> 14) & 0x3ff) if sf < 2 else ((4, (v >> 18) & 0x3fff) if sf == 2 else (5, (v >> 22) & 0x3ffff))
    return blk + hdr, blk + hdr + csize


@pytest.mark.parametrize("edge", ["one", "grid-1", "grid", "grid+1"])
def test_chunk_edges(monkeypatch, edge):
    """chunks of 1, grid - 1, grid and grid + 1 series (grid = the fused kernel's persistent grid when chunked)"""
    import victoriametrics_b200 as vm
    grid = vm._lib.lib().vmb_fused_grid_chunked()
    assert 132 <= grid < vm._lib.lib().vmb_fused_grid()
    per = {"one": 1, "grid-1": grid - 1, "grid": grid, "grid+1": grid + 1}[edge]
    rng = np.random.default_rng(SEED0 + 7100 + per)
    blocks = [_block(rng, "gauge", 1000, s) for s in range(CHUNKS * per)]
    assert any(_zstd(b) for b in blocks)
    _assert_same(_rollup(blocks, monkeypatch))


def test_chunk_of_bailing_series_only(monkeypatch):
    """every series of chunk 2 holds staleness markers: the kernel hands all of them back"""
    rng = np.random.default_rng(SEED0 + 7200)
    per, blocks = 40, []
    for s in range(CHUNKS * per):
        b = _block(rng, "counter", 2000, s)
        if s // per == 2:
            v = b.vals.copy()
            v[rng.integers(1, 2000, 3)] = (1 << 63) - 2
            b = blockgen.OBlock(b.ts, v, -2, 64, s)
        blocks.append(b)
    assert any(_zstd(b) for b in blocks)
    _assert_same(_rollup(blocks, monkeypatch))


def test_corrupt_frame_in_last_chunk(monkeypatch):
    """a damaged zstd frame of a series in the last chunk: the error code still reaches the un-fused path"""
    rng = np.random.default_rng(SEED0 + 7300)
    blocks = [_block(rng, "counter", 2000, s) for s in range(CHUNKS * 30)]
    victim = next(i for i in range(len(blocks) - 1, -1, -1) if _zstd(blocks[i]))
    assert victim >= len(blocks) * (CHUNKS - 1) // CHUNKS
    v = blocks[victim].vdata.copy()
    lo, hi = len(v) // 3, len(v) // 3 + 24
    # still a Huffman frame of a fused series after the damage: only literal bytes change, the headers the upload reads do not
    lit = _literals_section(v)
    assert blocks[victim].tmt == 2 and lit is not None and lit[0] + 8 <= lo and hi <= lit[1], (lit, lo, hi)
    v[lo:hi] = 0xFF
    blocks[victim].vdata = v
    res = _rollup(blocks, monkeypatch)
    assert res[1][2] == -53  # VMB_ERR_BLOCK_FAILED
    _assert_same(res)


def test_unfused_series_in_every_chunk(monkeypatch):
    """jittered (zstd nearest-delta2 timestamps) and two-block series between the fused ones, all along the batch"""
    rng = np.random.default_rng(SEED0 + 7400)
    blocks, s = [], 0
    for k in range(CHUNKS * 25):
        if k % 5 == 1:
            blocks.append(_block(rng, "gauge", 1500, s, ts_kind="jitter"))
        elif k % 7 == 3:
            ts = blockgen.gen_timestamps(rng, "regular", 1500, T0)
            vals = blockgen.gen_values(rng, "counter", 1500)
            blocks.append(blockgen.OBlock(ts[:700], vals[:700], -2, 64, s))
            blocks.append(blockgen.OBlock(ts[700:], vals[700:], -2, 64, s))
        else:
            blocks.append(_block(rng, "counter_resets", 1500, s))
        s += 1
    assert any(_zstd(b) for b in blocks)
    _assert_same(_rollup(blocks, monkeypatch, rows=1500))


def test_sum_sink_at_scale_zero(monkeypatch):
    """sum(rate) by (g) with the fold inside the fused kernel, scale-0 blocks"""
    import torch
    import victoriametrics_b200 as vm
    rng = np.random.default_rng(SEED0 + 7500)
    S, G, rows = CHUNKS * 50, 5, 1200
    blocks = [_block(rng, "counter", rows, s, scale=0) for s in range(S)]
    assert any(_zstd(b) for b in blocks)
    groups = (np.arange(S) * 3 % G).astype(np.uint32)
    start, end, step, window = T0 + 60000, T0 + 15000 * (rows - 1), 15000, 120000
    rc = vm.promql.get_rollup_configs("rate", start, end, step, window)
    descs, payload = blockgen.to_blockset(blocks)
    ctxs = _contexts(monkeypatch)
    B = vm.storage.Blocks(descs, payload, ctxs[CHUNKS])

    class Buf:
        def __init__(self, nbytes):
            self.t = torch.empty(nbytes // 8, dtype=torch.float64, device="cuda")
            self.ptr = self.t.data_ptr()
    res = {}
    for c, ctx in ctxs.items():
        B.ctx = ctx
        ia = vm.promql.IncrementalAggr("sum", G, rc.points, Buf)
        sc = ia.update_blocks(B, rc, groups)
        res[c] = (ia.finalize(ctx), sc)
    B.ctx = ctxs[CHUNKS]
    B.close()
    assert res[CHUNKS][1] == res[1][1]
    # the kernel folds finished series with atomic adds, in whatever order its CTAs finish: equal up to that order
    a, b = res[CHUNKS][0], res[1][0]
    assert np.array_equal(np.isnan(a), np.isnan(b))
    assert np.allclose(a, b, rtol=1e-12, atol=0, equal_nan=True)
    for ctx in ctxs.values():
        ctx.close()
