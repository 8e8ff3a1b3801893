"""The GPU zstd decoders on every frame shape the reference's writers produce, through every entry point that decodes zstd.

Expected values never come from a zstd decoder under test: a case carries its raw varint stream (the input the frame was
made from, checked against libzstd when it was made), and the oracle unmarshals that stream as MarshalType 5 / 6.  A case
is an error exactly where libzstd fails or the varint decode of rows - 1 values does not consume the content.

Cases come from tests/golden/zstd_shapes.json (always) and from a live sweep through the reference's libzstd
(oracle/_ref): levels -7..22, windows, block sizes, raw literals, checksums, strategies, no Frame_Content_Size, the pure-Go
writer's headers, dictated repeat-offset sequences.  Frames without Frame_Content_Size take the serial decoder."""
import base64
import hashlib
import json
import os

import numpy as np
import pytest

from conftest import SEED0
import blockgen
import oracle_lib as O
import partgen
import zstd_shapes as Z

HERE = os.path.dirname(os.path.abspath(__file__))
T0 = 1_700_000_000_000
STEP_MS = 15_000
SCALE = -2


def _fixture():
    out = []
    with open(os.path.join(HERE, "golden", "zstd_shapes.json")) as f:
        for e in json.load(f):
            raw, frame = base64.b64decode(e["raw"]), base64.b64decode(e["frame"])
            assert hashlib.sha256(raw).hexdigest() == e["raw_sha256"], e["name"]
            assert hashlib.sha256(frame).hexdigest() == e["frame_sha256"], e["name"]
            out.append(Z.case(e["name"], e["mt"], e["rows"], e["first"], np.frombuffer(raw, np.uint8),
                              np.frombuffer(frame, np.uint8), e["zstd_ok"]))
    return out


def _ref():
    return O.lib().vmo_zstd_ref_available()


def _factory():
    """the frame factory of oracle/_ref (an oracle/_ref built by an older recipe has libzstd's one-shot calls only)"""
    return O.lib().vmo_zstd_ref_factory_available()


def _cases(source):
    if source == "fixture":
        return _fixture()
    if not _factory():
        pytest.skip("oracle/_ref (the reference's libzstd with the frame factory) was not built")
    return Z.live_corpus(SEED0 + 7100)


def _expected(c):
    """(ok, int64 values) of the column: libzstd must decode the frame and rows - 1 varints must fill the content"""
    if not c["zstd_ok"]:
        return False, None
    rc, vals = O.unmarshal_int64_array(c["raw"], 5 if c["mt"] == 1 else 6, c["first"], c["rows"])
    return rc == 0, (vals.copy() if rc == 0 else None)


def _same(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and bool(np.all((a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))))


# ---------------------------------------------------------------------------------------------------------- CPU checks
@pytest.mark.parametrize("source", ["fixture", "live"])
def test_corpus_holds_every_shape(source):
    cases = _cases(source)
    seen = set()
    for c in cases:
        if c["zstd_ok"]:
            seen |= Z.shapes(c["frame"])
    want = {"prepared_with_sequences", "prepared_literals_only", "prepared_1_stream", "prepared_4_stream", "serial",
            "lit_raw_with_sequences", "lit_rle_with_sequences", "multi_block", "checksum", "no_fcs", "window_descriptor",
            "fcs2", "raw_block", "lit_treeless", "repeat_mode"}
    assert want <= seen, sorted(want - seen)
    # the pure-Go writer's two small-frame header layouts: no FCS below 256 bytes, a 2-byte FCS with a window up to 1024
    pg = [Z.parse_frame(c["frame"]) for c in cases if c["name"].startswith("pure_go_")]
    assert any(f["fcs"] is None and f["window_descriptor"] == 0 for f in pg)
    assert any(f["fcs_size"] == 2 and not f["single"] and f["window_descriptor"] == 0 for f in pg)
    names = {c["name"] for c in cases}
    assert {"err_no_fcs_truncated", "err_no_fcs_over_10_bytes_per_row", "err_block_over_window"} <= names
    assert {"seq_one_block", "seq_checksum", "seq_no_fcs", "seq_two_blocks"} <= names
    if source == "live":
        levels = {int(n.split("_")[0][5:]) for n in names if n.startswith("level")}
        assert levels == set(range(-7, 23))
        assert {c["rows"] for c in cases} >= {13, 8192}


@pytest.mark.parametrize("source", ["fixture", "live"])
def test_oracle_unmarshal_matches_reference(source):
    """the oracle's MarshalType 1 / 4 decode (its own zstd decoder) agrees with libzstd + the varint check on every case"""
    for c in _cases(source):
        ok, vals = _expected(c)
        rc, got = O.unmarshal_int64_array(c["frame"], c["mt"], c["first"], c["rows"])
        assert (rc == 0) == ok, (c["name"], rc)
        if ok:
            assert np.array_equal(got, vals), c["name"]


def test_fixture_frames_still_match_reference_libzstd():
    if not _ref():
        pytest.skip("oracle/_ref (the reference's libzstd) was not built")
    for c in _fixture():
        n, out = O.zstd_ref_decompress_rc(c["frame"], 1 << 20)
        assert (n >= 0) == c["zstd_ok"], c["name"]
        if n >= 0:
            assert np.array_equal(out, c["raw"]), c["name"]


# ---------------------------------------------------------------------------------------------------------- GPU
def _column_cases(cases):
    return [c for c in cases if c["rows"] is not None and 2 <= c["rows"] <= 8192]


@pytest.mark.gpu
@pytest.mark.parametrize("source", ["fixture", "live"])
def test_unmarshal_int64(source):
    import victoriametrics_b200 as vm
    for c in _column_cases(_cases(source)):
        ok, vals = _expected(c)
        try:
            got = vm.encoding.unmarshal_values(c["frame"], c["mt"], c["first"], c["rows"])
            err = None
        except vm.VmbError as e:
            got, err = None, e
        assert (err is None) == ok, (c["name"], err)
        if ok:
            assert np.array_equal(got, vals), c["name"]


def _blockset(cases, column):
    """one block per case: the case's frame as the values column (timestamps MarshalTypeDeltaConst) or as the timestamps
    column (values MarshalTypeConst)"""
    import victoriametrics_b200 as vm
    bs = vm.storage.BlockSet()
    tdelta = O.marshal_varint64s([STEP_MS])
    for i, c in enumerate(cases):
        n = c["rows"]
        if column == "values":
            bs.add_marshaled(dict(first_value=c["first"], min_ts=T0, max_ts=T0 + STEP_MS * (n - 1), ts_size=tdelta.size,
                                  val_size=c["frame"].size, rows=n, series_idx=i, scale=SCALE, ts_mt=2, val_mt=c["mt"],
                                  precision_bits=64), tdelta, c["frame"])
        else:
            ok, vals = _expected(c)
            bs.add_marshaled(dict(first_value=7, min_ts=c["first"], max_ts=int(vals.max()) if ok else c["first"],
                                  ts_size=c["frame"].size, val_size=0, rows=n, series_idx=i, scale=0, ts_mt=c["mt"], val_mt=3,
                                  precision_bits=64), c["frame"], np.zeros(0, np.uint8))
    return bs.finish()


@pytest.mark.gpu
@pytest.mark.parametrize("column", ["values", "timestamps"])
@pytest.mark.parametrize("source", ["fixture", "live"])
def test_decode_blocks_unfused(source, column):
    import victoriametrics_b200 as vm
    cases = _column_cases(_cases(source))
    descs, payload = _blockset(cases, column)
    ctx = vm.default_context()
    ctx.set_fused(False)
    try:
        B = vm.storage.Blocks(descs, payload, ctx)
        ser, status = vm.storage.decode_blocks(B, raise_on_block_error=False)
        got = ser.to_lists()
        ser.close()
        B.close()
    finally:
        ctx.set_fused(True)
    for i, c in enumerate(cases):
        ok, vals = _expected(c)
        assert (status[i] == 0) == ok, (c["name"], int(status[i]))
        if not ok:
            continue
        ts, v = got[i]
        if column == "values":
            assert np.array_equal(ts, T0 + STEP_MS * np.arange(c["rows"], dtype=np.int64)), c["name"]
            assert _same(v, O.decimal_to_float(vals, SCALE)), c["name"]
        else:
            assert np.array_equal(ts, vals), c["name"]
            assert _same(v, np.full(c["rows"], 7.0)), c["name"]


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("source", ["fixture", "live"])
def test_rollup_device(source, fused):
    """decode + max_over_time on device-resident blocks: with the fused kernel on, frames without Frame_Content_Size sit in
    the same batch as prepared frames of ordinary series and reach the fused kernel through the serial decoder"""
    import victoriametrics_b200 as vm
    from rollup_names import RF
    # (the "special" value kind holds staleness markers, which the query path drops before the rollup: its columns are
    # pinned bit for bit by the decode tests above)
    cases = [c for c in _column_cases(_cases(source)) if _expected(c)[0] and "special" not in c["name"]]
    # ordinary series beside them: libzstd's default frames of the same streams
    cases = cases + [dict(c, frame=O.zstd_ref_compress(c["raw"], 1), name=c["name"] + "/default") for c in cases] if _ref() else cases
    descs, payload = _blockset(cases, "values")
    ctx = vm.default_context()
    ctx.set_fused(fused)
    start, end, step, window = T0, T0 + STEP_MS * 8191, 60_000, 300_000
    try:
        B = vm.storage.Blocks(descs, payload, ctx)
        got, _ = vm.promql.eval_rollup_func("max_over_time", B, start, end, step, window)
        B.close()
    finally:
        ctx.set_fused(True)
    rc = vm.promql.get_rollup_configs("max_over_time", start, end, step, window)
    for i, c in enumerate(cases):
        _, vals = _expected(c)
        ts = T0 + STEP_MS * np.arange(c["rows"], dtype=np.int64)
        exp, _ = O.rollup_do(RF["max_over_time"], O.decimal_to_float(vals, SCALE), ts, start, end, step, window,
                             may_adjust_window=rc.MayAdjustWindow, samples_scanned_per_call=rc.samplesScannedPerCall)
        assert _same(got[i], exp), c["name"]


def _batch(frames):
    """vmb_zstd_decompress_bound + vmb_zstd_decompress_batch -> (rc, per-frame status, per-frame bytes)"""
    import ctypes as C
    import victoriametrics_b200 as vm
    from victoriametrics_b200 import _lib
    n = len(frames)
    offs = np.zeros(n + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([f.size for f in frames])
    arena = np.concatenate(frames)
    bound = C.c_uint64(0)
    _lib.check(_lib.lib().vmb_zstd_decompress_bound(arena.ctypes.data_as(_lib.u8p), offs.ctypes.data_as(_lib.u64p), n,
                                                    C.byref(bound)))
    dst = np.zeros(max(bound.value, 1), dtype=np.uint8)
    doffs, dlens, st = np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.int32)
    rc = _lib.lib().vmb_zstd_decompress_batch(vm.default_context().h, arena.ctypes.data_as(_lib.u8p),
                                              offs.ctypes.data_as(_lib.u64p), n, dst.ctypes.data_as(_lib.u8p), dst.size,
                                              doffs.ctypes.data_as(_lib.u64p), dlens.ctypes.data_as(_lib.u32p),
                                              st.ctypes.data_as(_lib.i32p))
    return rc, st, [dst[int(o):int(o) + int(l)] for o, l in zip(doffs, dlens)], bound.value


@pytest.mark.gpu
@pytest.mark.parametrize("source", ["fixture", "live"])
def test_zstd_decompress_batch(source):
    cases = _cases(source)
    if source == "live":
        # long matches up to the block maximum, overlapping their own output (no row limit on this entry point)
        rng = np.random.default_rng(SEED0 + 7101)
        seqs = [(3, 7, 131000), (0, 0, 0), (1, 2, 120000), (0, 5, 0)]  # two blocks of nearly 128 KiB
        src = Z.run_sequences([seqs[0], seqs[2]], np.arange(0, 200), rng, tail=5)
        for name, p in (("long_matches", {}), ("long_matches_no_fcs", dict(contentSizeFlag=0, windowLog=17))):
            cases.append(Z.case(name, 4, None, 0, src, O.zstd_ref_compress_sequences(src, seqs, **p)))
    rc, st, got, bound = _batch([c["frame"] for c in cases])
    assert (rc == 0) == all(c["zstd_ok"] for c in cases)
    assert bound >= sum(c["raw"].size for c in cases if c["zstd_ok"])
    for c, s, g in zip(cases, st, got):
        assert (s == 0) == c["zstd_ok"], (c["name"], int(s))
        if c["zstd_ok"]:
            assert np.array_equal(g, c["raw"]), c["name"]


@pytest.mark.gpu
def test_pure_go_part_collect_decode_rollup(oracle):
    """a part as the reference's builds without cgo write it: metaindex.bin, the index blocks and the short columns have no
    Frame_Content_Size -> collect_blocks -> decode -> rollup, against the oracle on what was written"""
    import victoriametrics_b200 as vm
    from rollup_names import RF
    if not _factory():
        pytest.skip("oracle/_ref (the reference's libzstd with the frame factory) was not built")
    rng = np.random.default_rng(SEED0 + 7102)
    series = []
    for s in range(3):
        rows = (40, 200, 3000)[s]  # a plain column, a zstd column of < 256 varint bytes, a long one
        ts = blockgen.gen_timestamps(rng, "regular", rows, t0=T0)
        blocks = [blockgen.OBlock(ts, blockgen.gen_values(rng, ("gauge", "counter_smooth", "gauge_small")[s], rows), SCALE, 64, s)]
        series.append((partgen.pack_tsid(10, 1, s, 5000 + s), blocks))
    files = partgen.write_part(series, level=int(rng.choice([1, 3])), pure_go=True)
    assert Z.parse_frame(files["metaindex_bin"])["fcs"] is None            # 1 row of 56 B
    assert Z.parse_frame(files["index_bin"])["fcs"] is None                # 3 block headers of 81 B
    cols = [b.vdata for _, bl in series for b in bl if b.vmt in (1, 4)]
    assert any(Z.parse_frame(v)["fcs"] is None for v in cols), "a short column without Frame_Content_Size"
    part = vm.storage.Part(files["metaindex_bin"], files["index_bin"], files["timestamps_bin"], files["values_bin"])
    descs, payload, tsids = part.collect_blocks()
    assert len(descs) == 3 and [t.tobytes() for t in tsids] == [s[0] for s in series]
    B = vm.storage.Blocks(descs, payload)
    ser, status = vm.storage.decode_blocks(B)
    got = ser.to_lists()
    ser.close()
    assert not status.any()
    start, end, step, window = T0 + 60_000, T0 + 3_000_000, 30_000, 300_000
    out, _ = vm.promql.eval_rollup_func("avg_over_time", B, start, end, step, window)
    B.close()
    for i, (_, blocks) in enumerate(series):
        rc, ets, ev, _ = blocks[0].oracle_unmarshal()
        assert rc == 0
        assert np.array_equal(got[i][0], ets) and _same(got[i][1], ev), i
        want, _ = oracle.rollup_do(RF["avg_over_time"], ev.copy(), ets.copy(), start, end, step, window)
        assert np.allclose(out[i], want, rtol=1e-12, atol=0, equal_nan=True), i
