"""vmb_merge_parts / storage.merge_parts on the GPU against the restatement of mergeBlockStreams (tests/part_merge_ref.py) with the
library's host writer: the four files byte for byte and the stats."""
import ctypes as C
import threading
import zlib

import numpy as np
import pytest

import oracle_lib as O
import part_merge_ref as R
import partgen
from blockgen import OBlock, gen_values
from victoriametrics_b200 import _lib, storage

pytestmark = pytest.mark.gpu
T0 = 1_700_000_000_000


def tsid(mid, mg=7):
    return partgen.pack_tsid(mg, 1, 2, mid)


def make_parts(rng, nparts, nseries, rows, step=15_000, kinds=("gauge", "counter"), scales=(0,), pbs=(64,), overlap=False,
               same_ts=False, max_rows=R.MAX_ROWS_PER_BLOCK):
    """nparts parts of nseries series; part p holds rows [p*rows, (p+1)*rows) of each series (or the same range with overlap)"""
    parts = []
    for p in range(nparts):
        series = []
        for s in range(nseries):
            start = 0 if overlap else p * rows
            ts = T0 + (np.arange(start, start + rows, dtype=np.int64) * step)
            if not same_ts:
                ts = ts + int(rng.integers(0, 3))
            vals = gen_values(rng, str(rng.choice(kinds)), rows)
            sc, pb = int(rng.choice(scales)), int(rng.choice(pbs))
            series.append((tsid(s + 1), [OBlock(t, v, sc, pb) for t, v in R.split_rows(ts, vals, max_rows)]))
        parts.append(R.part_from_series(series))
    return parts


def run_both(parts, deadline=R.INT64_MIN, deleted=(), dedup=0, **writer):
    ref = R.merge_parts([b for _, b in parts], deadline, deleted, dedup, **writer)
    ctx = _lib.default_context()
    ctx.set_dedup_interval(dedup)
    try:
        got, st = storage.merge_parts([storage.Part(p["metaindex_bin"], p["index_bin"], p["timestamps_bin"], p["values_bin"])
                                       for p, _ in parts], deadline, deleted)
    finally:
        ctx.set_dedup_interval(0)
    return ref, got, st


def assert_same(ref, got, st):
    assert st == ref["stats"]
    assert got.timestamps_bin.tobytes() == ref["timestamps_bin"]
    assert got.values_bin.tobytes() == ref["values_bin"]
    assert got.index_bin.tobytes() == ref["index_bin"]
    if ref["metaindex_bin"] is not None:
        assert got.metaindex_bin.tobytes() == ref["metaindex_bin"]
    # every frame is accepted by the reference's libzstd
    mi = O.zstd_ref_decompress(got.metaindex_bin, len(ref["metaindex_raw"]) + 16)
    assert mi.tobytes() == ref["metaindex_raw"]


CASES = {
    "fresh_reblocked": dict(nparts=4, nseries=5, rows=1024),
    "full_disjoint": dict(nparts=3, nseries=4, rows=8192),
    "replicas": dict(nparts=3, nseries=3, rows=3000, overlap=True, same_ts=True),
    "scales_pbs": dict(nparts=3, nseries=6, rows=700, overlap=True, scales=(-2, 0, 3), pbs=(64, 20, 8)),
    "big_blocks": dict(nparts=2, nseries=2, rows=16384, overlap=True, max_rows=16384),
    "one_part": dict(nparts=1, nseries=3, rows=500),
    "sixteen_parts": dict(nparts=16, nseries=2, rows=300),
    "many_index_blocks": dict(nparts=2, nseries=1700, rows=3, same_ts=True, kinds=("const",)),  # 1700 blocks: 3 index blocks
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_merge_matches_restatement(name):
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    parts = make_parts(rng, **CASES[name])
    assert_same(*run_both(parts))


@pytest.mark.parametrize("dedup", [15_000, 60_000])
def test_replicas_dedup(dedup):
    rng = np.random.default_rng(dedup)
    parts = make_parts(rng, 3, 3, 2000, overlap=True, same_ts=True)
    assert_same(*run_both(parts, dedup=dedup))


@pytest.mark.parametrize("where", ["inside", "min", "max", "max_plus_1"])
def test_retention_deadline(where):
    rng = np.random.default_rng(5)
    parts = make_parts(rng, 3, 3, 1000, overlap=True)
    h = parts[0][1][0][1]
    d = dict(inside=(h["min_ts"] + h["max_ts"]) // 2, min=h["min_ts"], max=h["max_ts"], max_plus_1=h["max_ts"] + 1)[where]
    assert_same(*run_both(parts, deadline=d))


@pytest.mark.parametrize("which", ["first", "middle", "last", "all"])
def test_deleted_metric_ids(which):
    rng = np.random.default_rng(6)
    parts = make_parts(rng, 2, 5, 400)
    ids = dict(first=[1], middle=[3], last=[5], all=[1, 2, 3, 4, 5])[which]
    ref, got, st = run_both(parts, deleted=ids)
    assert_same(ref, got, st)
    if which == "all":
        assert st["blocks_count"] == 0 and st["min_ts"] == R.INT64_MAX and st["max_ts"] == R.INT64_MIN
        assert got.index_bin.size == 0 and O.zstd_ref_decompress(got.metaindex_bin, 16).size == 0


def test_merged_part_decodes_through_the_query_path():
    rng = np.random.default_rng(9)
    parts = make_parts(rng, 3, 4, 1500, overlap=True)
    ref, got, st = run_both(parts)
    descs, payload, ids = got.collect_blocks()
    assert len(descs) == st["blocks_count"] and int(descs["rows"].sum()) == st["rows_count"]
    assert_round_trip(got, ref)


def test_unsorted_deleted_ids_rejected():
    rng = np.random.default_rng(1)
    (p, _), = make_parts(rng, 1, 2, 10)
    files = (_lib.PartFiles * 1)()
    arrs = [np.frombuffer(p[k], dtype=np.uint8) for k in ("metaindex_bin", "index_bin", "timestamps_bin", "values_bin")]
    for name, a in zip(("metaindex", "index", "timestamps", "values"), arrs):
        setattr(files[0], name, a.ctypes.data_as(_lib.u8p))
        setattr(files[0], name + "_len", a.size)
    dm = np.array([5, 3], dtype=np.uint64)
    h = C.c_void_p()
    st = _lib.MergeStats()
    rc = _lib.lib().vmb_merge_parts(_lib.default_context().h, files, 1, R.INT64_MIN, dm.ctypes.data_as(_lib.u64p), 2, C.byref(h),
                                    C.byref(st))
    assert rc == -50 and not h.value


def test_offsets_outside_a_file_rejected():
    rng = np.random.default_rng(2)
    (p, _), = make_parts(rng, 1, 2, 10)
    bad = storage.Part(p["metaindex_bin"], p["index_bin"], p["timestamps_bin"][:-1], p["values_bin"])
    with pytest.raises(_lib.VmbError) as e:
        storage.merge_parts([bad])
    assert e.value.code == -1


def test_corrupt_payload_merged_vs_pass_through():
    rng = np.random.default_rng(3)
    # merged: two overlapping parts of small blocks; pass-through: full disjoint blocks
    for overlap, rows in ((True, 300), (False, 8192)):
        parts = make_parts(rng, 2, 1, rows, overlap=overlap, kinds=("gauge",))
        p0 = parts[0][0]
        vb = bytearray(p0["values_bin"])
        vb[0] ^= 0xFF
        vb[1:9] = b"\xff" * 8
        p0["values_bin"] = bytes(vb)
        P = [storage.Part(p["metaindex_bin"], p["index_bin"], p["timestamps_bin"], p["values_bin"]) for p, _ in parts]
        if overlap:
            with pytest.raises(_lib.VmbError):
                storage.merge_parts(P)
        else:
            got, _ = storage.merge_parts(P)
            assert got.values_bin.tobytes()[:len(vb)] == bytes(vb)


def test_repeatable_and_concurrent():
    rng = np.random.default_rng(4)
    parts = make_parts(rng, 3, 20, 900, overlap=True)
    P = [storage.Part(p["metaindex_bin"], p["index_bin"], p["timestamps_bin"], p["values_bin"]) for p, _ in parts]
    a, _ = storage.merge_parts(P)
    out = [None, None]

    def work(i):
        import torch
        ctx = _lib.Context()
        s = torch.cuda.Stream()
        ctx.set_stream(s.cuda_stream)
        out[i] = storage.merge_parts(P, ctx=ctx)[0]

    ts = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    for o in out:
        for k in ("metaindex_bin", "index_bin", "timestamps_bin", "values_bin"):
            assert getattr(o, k).tobytes() == getattr(a, k).tobytes()


def family(mt):  # the column kinds of encoding.go:20-43; 5 / 6 are 1 / 4 stored without zstd
    return {5: 1, 6: 4}.get(mt, mt)


def assert_round_trip(got, ref):
    """the GPU part through the query path (collect_blocks + decode_blocks(values_as_int64), one series per block) gives, block by
    block, what the reference side decodes from it (libzstd + the oracle), and the restatement's rows where precisionBits is 64
    (a lossy block's rows change when they are written)"""
    oracle = R.read_part(got.metaindex_bin, got.index_bin, got.timestamps_bin, got.values_bin, len(ref["metaindex_raw"]) + 16)
    descs, payload, _ = got.collect_blocks()
    descs = descs.copy()
    descs["series_idx"] = np.arange(len(descs), dtype=np.uint32)
    series, status = storage.decode_blocks(storage.Blocks(descs, payload), values_as_int64=True)
    assert (status == 0).all()
    rows = series.to_lists(values_dtype=np.int64)
    assert len(rows) == len(ref["blocks"]) == len(oracle)
    for (ts, vs), (_, h, rts, rvs), (_, _, ots, ovs) in zip(rows, ref["blocks"], oracle):
        assert ts.tolist() == ots and vs.tolist() == ovs
        if h["precision_bits"] == 64:
            assert ots == list(rts) and ovs == list(rvs)


REF_CASES = ["fresh_reblocked", "replicas", "scales_pbs", "full_disjoint", "many_index_blocks"]


@pytest.mark.parametrize("name", REF_CASES)
def test_against_reference_libzstd(name):
    """the restatement written by the reference (oracle marshalInt64Array + libzstd) and the GPU part decode, through libzstd alone,
    to the same TSIDs, block boundaries, rows, scales, precisionBits and MarshalType families; every frame of the GPU part is
    libzstd's to read; the query path reads the restatement's rows back"""
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    parts = make_parts(rng, **CASES[name])
    ref_host, got, st = run_both(parts)
    assert_same(ref_host, got, st)
    ref = R.merge_parts([b for _, b in parts], marshal=R.oracle_marshal, frame=R.oracle_frame)
    assert ref["stats"] == st
    a = R.read_part(got.metaindex_bin, got.index_bin, got.timestamps_bin, got.values_bin, len(ref["metaindex_raw"]) + 16)
    b = R.read_part(ref["metaindex_bin"], ref["index_bin"], ref["timestamps_bin"], ref["values_bin"], len(ref["metaindex_raw"]) + 16)
    assert len(a) == len(b)
    for (ta, ha, tsa, va), (tb, hb, tsb, vb) in zip(a, b):
        assert ta == tb and ha["rows"] == hb["rows"] and ha["scale"] == hb["scale"] and ha["precision_bits"] == hb["precision_bits"]
        assert family(ha["ts_mt"]) == family(hb["ts_mt"]) and family(ha["val_mt"]) == family(hb["val_mt"])
        assert tsa == tsb and va == vb
    assert_round_trip(got, ref_host)


def test_calibrate_scale_overflow_on_device():
    """part 0's mantissas cannot take three more digits: CalibrateScale moves the exponent up and divides part 1's values"""
    rng = np.random.default_rng(11)
    n = 600
    ts = T0 + np.arange(n, dtype=np.int64) * 10_000
    big = (R.INT64_MAX // 10 - rng.integers(0, 10 ** 6, n)).astype(np.int64)
    small = rng.integers(-10 ** 9, 10 ** 9, n).astype(np.int64)
    parts = [R.part_from_series([(tsid(1), [OBlock(ts, big, 3)])]), R.part_from_series([(tsid(1), [OBlock(ts + 5_000, small, 0)])])]
    ref, got, st = run_both(parts)
    assert_same(ref, got, st)
    assert [h["scale"] for _, h, _, _ in ref["blocks"]] == [2]
    assert_round_trip(got, ref)


def test_rule5_column_streams_over_128k():
    """16384-row blocks whose values stream lands in (128 KiB, 262143] and compresses.  The writer's frame for such a stream is
    one libzstd rejects, and the stream uncompressed is a payload blockHeader.validate rejects (block_header.go:251): the merge
    fails with VMB_ERR_CAP and writes no part.  The same blocks passed through keep their libzstd frames."""
    from victoriametrics_b200 import encoding
    rng = np.random.default_rng(12)
    n = 16384
    series = []
    for s_ in range(2):
        ts = T0 + np.arange(n, dtype=np.int64) * 1000
        # a few values, never the same twice in a row: every delta takes 9 or 10 varint bytes, and they repeat
        idx = np.cumsum(rng.integers(1, 4, n)) % 4
        vals = np.array([(1 << 62) - 1, -(1 << 62), (1 << 61) + 3, -((1 << 61) + 5)], dtype=np.int64)[idx]
        series.append((tsid(s_ + 1), [OBlock(ts, vals, 0)]))
        data, mt, _ = encoding.marshal_values(vals)
        rc, stream = O.zstd_decompress(data)
        assert mt in (1, 4) and rc == 0 and 128 * 1024 < stream.size <= 262143  # compressible, inside the range
    parts = [R.part_from_series(series)]
    P = [storage.Part(p["metaindex_bin"], p["index_bin"], p["timestamps_bin"], p["values_bin"]) for p, _ in parts]
    ctx = _lib.default_context()
    ctx.set_dedup_interval(1)  # every block re-encoded (no two rows share a millisecond)
    try:
        with pytest.raises(_lib.VmbError) as e:
            storage.merge_parts(P)
        assert e.value.code == -54
    finally:
        ctx.set_dedup_interval(0)
    ref, got, st = run_both(parts)  # dedup off: the blocks pass through as they are
    assert_same(ref, got, st)
    assert_round_trip(got, ref)


def _raw_blocks(frame):
    """the block types of a single-segment zstd frame"""
    fhd = frame[4]
    fcs = {0: 1, 1: 2, 2: 4, 3: 8}[fhd >> 6]
    k, types = 5 + fcs, []
    while True:
        h = frame[k] | frame[k + 1] << 8 | frame[k + 2] << 16
        types.append((h >> 1) & 3)
        k += 3 + (h >> 3 if (h >> 1) & 3 != 1 else 1)
        if h & 1:
            return types, k


@pytest.mark.parametrize("n", [131072, 131073, 200000, 262143, 262144])
def test_rule5_metaindex_frames(n):
    from victoriametrics_b200 import encoding
    rng = np.random.default_rng(n)
    src = rng.integers(0, 6, n).astype(np.uint8)  # compresses well: the writer would pick a Compressed block
    dst = np.zeros(n + 1024, dtype=np.uint8)
    ln = C.c_size_t(0)
    rc = _lib.lib().vmb_merge_metaindex_frame(_lib.default_context().h, src.ctypes.data_as(_lib.u8p), n, dst.ctypes.data_as(_lib.u8p),
                                              dst.size, C.byref(ln))
    assert rc == 0
    frame = dst[:ln.value]
    assert O.zstd_ref_decompress(frame, n + 16).tobytes() == src.tobytes()
    if 128 * 1024 < n <= 262143:
        types, end = _raw_blocks(frame.tobytes())
        assert set(types) == {0} and end == frame.size
    else:
        assert frame.tobytes() == encoding.zstd_compress(src).tobytes()
