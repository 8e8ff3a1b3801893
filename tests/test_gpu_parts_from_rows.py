"""vmb_parts_from_rows / storage.parts_from_rows on the GPU against the restatement of marshalToInmemoryPart (tests/raw_rows_ref.py)
with the library's host writer: every part's four files byte for byte and its stats."""
import ctypes as C
import struct
import threading
import zlib

import numpy as np
import pytest

import oracle_lib as O
import part_merge_ref as M
import partgen
import raw_rows_ref as R
from victoriametrics_b200 import _lib, decimal, storage

pytestmark = pytest.mark.gpu
T0 = 1_700_000_000_000
STALE_NAN = struct.unpack("<d", struct.pack("<Q", 0x7FF0000000000002))[0]  # decimal.StaleNaN


def tsids_of(nseries, mg_mod=97):
    """TSIDs whose order is not the MetricID order: MetricGroupID varies"""
    return np.frombuffer(b"".join(partgen.pack_tsid((s * 7919) % mg_mod + 1, 1, 2, s + 1) for s in range(nseries)),
                         dtype=np.uint8).reshape(nseries, 24)


def values_of(rng, kind, n):
    if kind == "int":
        return rng.integers(-10 ** 6, 10 ** 6, n).astype(np.float64)
    if kind == "dec":  # decimals at several scales
        p = 10.0 ** rng.integers(0, 6, n)
        return np.round(rng.normal(0, 1000, n) * p) / p
    return rng.normal(0, 1, n) * 100  # NormFloat64 * 100


def make_set(rng, nseries, nticks, order="scrape", kind="norm", step=15_000, pbs=(64,)):
    """nseries series x nticks scrapes, rows in `order`: scrape (tick-major, as ingestion sees them), sorted, reversed, shuffled"""
    ids = tsids_of(nseries)
    jitter = rng.integers(0, 1000, nseries)
    sidx = np.tile(np.arange(nseries), nticks)
    tick = np.repeat(np.arange(nticks), nseries)
    ts = T0 + tick.astype(np.int64) * step + jitter[sidx]
    vals = values_of(rng, kind, sidx.size)
    pb = np.asarray(pbs, dtype=np.uint8)[rng.integers(0, len(pbs), nseries)][sidx]
    perm = np.arange(sidx.size)
    if order in ("sorted", "reversed"):
        perm = np.array(R.sort_order(ids[sidx], ts))
        if order == "reversed":
            perm = perm[::-1]
    elif order == "shuffled":
        perm = rng.permutation(sidx.size)
    return ids[sidx][perm], ts[perm], vals[perm], pb[perm]


def run_both(sets, dedup=0, ctx=None):
    ref = [R.marshal_to_inmemory_part(*s, dedup_interval=dedup) for s in sets]
    ctx = ctx or _lib.default_context()
    ctx.set_dedup_interval(dedup)
    try:
        got = storage.parts_from_rows(sets, ctx=ctx)
    finally:
        ctx.set_dedup_interval(0)
    return ref, got


def assert_same(ref, got):
    assert len(ref) == len(got)
    for r, (p, st) in zip(ref, got):
        assert st == r["stats"]
        assert p.timestamps_bin.tobytes() == r["timestamps_bin"]
        assert p.values_bin.tobytes() == r["values_bin"]
        assert p.index_bin.tobytes() == r["index_bin"]
        if r["metaindex_bin"] is not None:
            assert p.metaindex_bin.tobytes() == r["metaindex_bin"]
        assert O.zstd_ref_decompress(p.metaindex_bin, len(r["metaindex_raw"]) + 16).tobytes() == r["metaindex_raw"]


def assert_round_trip(ref, got, sets):
    """each part through the query path (collect_blocks + decode_blocks, one series per block) gives the restatement's rows where
    precisionBits is 64; the values are AppendDecimalToFloat(AppendFloatToDecimal(v)) of the block's sorted rows"""
    for r, (p, st), s in zip(ref, got, sets):
        if not st["blocks_count"]:
            continue
        descs, payload, _ = p.collect_blocks()
        descs = descs.copy()
        descs["series_idx"] = np.arange(len(descs), dtype=np.uint32)
        series, status = storage.decode_blocks(storage.Blocks(descs, payload), values_as_int64=True)
        assert (status == 0).all()
        rows = series.to_lists(values_dtype=np.int64)
        assert len(rows) == len(r["blocks"])
        for (ts, vs), (_, h, rts, rvs, _, _), d in zip(rows, r["blocks"], descs):
            assert int(d["scale"]) == h["scale"]
            if h["precision_bits"] == 64:
                assert ts.tolist() == rts and vs.tolist() == rvs
                f = decimal.append_decimal_to_float(vs, h["scale"])
                exp = decimal.append_decimal_to_float(np.array(rvs, dtype=np.int64), h["scale"])
                assert f.tobytes() == exp.tobytes()
    # without dedup, the blocks hold the sorted rows, each value AppendDecimalToFloat(AppendFloatToDecimal(block))
    for r, s in zip(ref, sets):
        order = R.sort_order(s[0], s[1])
        pos = 0
        for _, h, rts, rvs, _, _ in r["blocks"]:
            if len(rvs) != h["rows"] or h["precision_bits"] != 64:
                return
            rows = order[pos:pos + len(rvs)]
            pos += len(rvs)
            assert rts == [int(s[1][i]) for i in rows]
            m, e = decimal.append_float_to_decimal(np.asarray(s[2], dtype=np.float64)[rows])
            assert decimal.append_decimal_to_float(np.array(rvs, dtype=np.int64), h["scale"]).tobytes() == \
                decimal.append_decimal_to_float(m, e).tobytes()


@pytest.mark.parametrize("order", ["sorted", "reversed", "shuffled", "scrape"])
@pytest.mark.parametrize("kind", ["int", "dec", "norm"])
def test_orders_and_values(order, kind):
    rng = np.random.default_rng(zlib.crc32((order + kind).encode()))
    sets = [make_set(rng, 60, 50, order, kind), make_set(rng, 7, 300, order, kind)]
    ref, got = run_both(sets)
    assert_same(ref, got)
    assert_round_trip(ref, got, sets)


def test_specials_and_extreme_timestamps():
    rng = np.random.default_rng(1)
    ids, ts, vals, pb = make_set(rng, 5, 40, "shuffled")
    vals[::7] = np.nan
    vals[1::11] = np.inf
    vals[2::13] = -np.inf
    vals[3::5] = STALE_NAN
    vals[4::9] = -0.0
    ts[::17] = R.INT64_MIN + rng.integers(0, 3, ts[::17].size)
    ts[1::19] = R.INT64_MAX - rng.integers(0, 3, ts[1::19].size)
    ts[2::23] = -rng.integers(1, 10 ** 12, ts[2::23].size)
    sets = [(ids, ts, vals, pb)]
    ref, got = run_both(sets)
    assert_same(ref, got)
    assert_round_trip(ref, got, sets)


@pytest.mark.parametrize("per_row", [False, True])
def test_lossy_precision_bits(per_row):
    rng = np.random.default_rng(2)
    ids, ts, vals, pb = make_set(rng, 30, 120, "shuffled", "norm", pbs=(1, 2, 7, 20, 64))
    if per_row:  # a block takes the PrecisionBits of its first row
        pb = rng.integers(1, 65, pb.size).astype(np.uint8)
    ref, got = run_both([(ids, ts, vals, pb)])
    assert_same(ref, got)


@pytest.mark.parametrize("order", ["sorted", "shuffled"])
def test_duplicate_rows_keep_input_order(order):
    rng = np.random.default_rng(3)
    ids, ts, vals, pb = make_set(rng, 10, 30, "sorted", "int")
    ids, ts, pb = np.repeat(ids, 3, axis=0), np.repeat(ts, 3), np.repeat(pb, 3)
    vals = rng.integers(0, 1000, ts.size).astype(np.float64)  # equal (TSID, ts), different values
    if order == "shuffled":
        p = rng.permutation(ts.size)
        ids, ts, vals, pb = ids[p], ts[p], vals[p], pb[p]
    ref, got = run_both([(ids, ts, vals, pb)])
    assert_same(ref, got)


@pytest.mark.parametrize("dedup", [15_000, 60_000])
def test_dedup(dedup):
    rng = np.random.default_rng(dedup)
    ids, ts, vals, pb = make_set(rng, 20, 200, "shuffled", "dec", step=5_000)
    ref, got = run_both([(ids, ts, vals, pb), make_set(rng, 3, 500, "scrape", step=20_000)], dedup=dedup)
    assert_same(ref, got)
    assert got[0][1]["rows_count"] < ts.size and got[0][1]["rows_merged"] == ts.size


@pytest.mark.parametrize("n", [1, 2, 8192, 8193, 16385])
def test_one_series_sizes(n):
    rng = np.random.default_rng(n)
    sets = [make_set(rng, 1, n, "shuffled")]
    ref, got = run_both(sets)
    assert_same(ref, got)
    assert got[0][1]["blocks_count"] == (n + 8191) // 8192
    assert_round_trip(ref, got, sets)


def test_same_metric_id_different_tsids():
    """rows of one MetricID under two MetricGroupIDs and JobIDs share blocks; a TSID between them in the sort order splits them"""
    rng = np.random.default_rng(4)
    t = [partgen.pack_tsid(1, 1, 2, 5), partgen.pack_tsid(1, 9, 2, 5), partgen.pack_tsid(2, 1, 2, 7), partgen.pack_tsid(3, 1, 2, 5)]
    ids = np.frombuffer(b"".join(t), dtype=np.uint8).reshape(4, 24)
    s = rng.integers(0, 4, 3000)
    ts = T0 + rng.integers(0, 10 ** 7, s.size)
    sets = [(ids[s], ts, rng.normal(0, 1, s.size), np.full(s.size, 64, np.uint8))]
    ref, got = run_both(sets)
    assert_same(ref, got)
    assert [b[0] for b in ref[0]["blocks"]] == [t[0], t[2], t[3]]


def test_empty_set_among_others():
    rng = np.random.default_rng(5)
    empty = (np.zeros((0, 24), np.uint8), np.zeros(0, np.int64), np.zeros(0), np.zeros(0, np.uint8))
    sets = [empty, make_set(rng, 4, 10), empty, make_set(rng, 3, 5), empty]
    ref, got = run_both(sets)
    assert_same(ref, got)
    for i in (0, 2, 4):
        p, st = got[i]
        assert st == dict(rows_count=0, blocks_count=0, min_ts=R.INT64_MAX, max_ts=R.INT64_MIN, rows_merged=0, rows_deleted=0)
        assert p.index_bin.size == p.timestamps_bin.size == p.values_bin.size == 0


def test_flush_sixteen_shards():
    """flushRowssToInmemoryParts: 16 shards of maxRawRowsPerShard rows each, in scrape order, in one call"""
    rng = np.random.default_rng(6)
    sets = [make_set(rng, 202, 866, "scrape") for _ in range(16)]
    sets = [tuple(a[:174762] for a in s) for s in sets]
    ref, got = run_both(sets)
    assert_same(ref, got)


def test_one_set_of_4m_rows():
    rng = np.random.default_rng(7)
    sets = [make_set(rng, 2048, 2048, "scrape", "dec")]
    ref, got = run_both(sets)
    assert_same(ref, got)


def test_flush_then_merge():
    """merge_parts(parts_from_rows(sets)) equals the restated merge of the restated parts: the whole flushRowssToInmemoryParts"""
    rng = np.random.default_rng(8)
    sets = [make_set(rng, 12, 400, "shuffled", kind) for kind in ("int", "dec", "norm")]
    ref, got = run_both(sets)
    assert_same(ref, got)
    mref = M.merge_parts([R.merge_input(r) for r in ref])
    mgot, mst = storage.merge_parts([p for p, _ in got])
    assert mst == mref["stats"]
    for k in ("metaindex_bin", "index_bin", "timestamps_bin", "values_bin"):
        if mref[k] is not None:
            assert getattr(mgot, k).tobytes() == mref[k], k


def test_repeatable_and_concurrent():
    rng = np.random.default_rng(9)
    sets = [make_set(rng, 50, 200, "shuffled") for _ in range(3)]
    a = storage.parts_from_rows(sets)
    out = [None, None]

    def work(i):
        import torch
        ctx = _lib.Context()
        s = torch.cuda.Stream()
        ctx.set_stream(s.cuda_stream)
        out[i] = storage.parts_from_rows(sets, ctx=ctx)

    th = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    [t.start() for t in th]
    [t.join() for t in th]
    for o in out:
        assert len(o) == len(a)
        for (p, st), (q, sq) in zip(o, a):
            assert st == sq
            for k in ("metaindex_bin", "index_bin", "timestamps_bin", "values_bin"):
                assert getattr(p, k).tobytes() == getattr(q, k).tobytes()


def _raw(sets):
    keep = []
    rows = (_lib.RawRows * len(sets))()
    for r, (t, ts, v, pb) in zip(rows, sets):
        t, ts, v, pb = (np.ascontiguousarray(x) for x in (t, ts, v, pb))
        keep += [t, ts, v, pb]
        r.tsids, r.timestamps = t.ctypes.data_as(_lib.u8p), ts.ctypes.data_as(_lib.i64p)
        r.values, r.precision_bits, r.n = v.ctypes.data_as(_lib.f64p), pb.ctypes.data_as(_lib.u8p), ts.size
    return rows, keep


def test_error_contract():
    rng = np.random.default_rng(10)
    good = make_set(rng, 3, 4)
    ctx = _lib.default_context().h
    L = _lib.lib()
    for bad_pb in (0, 65):
        pb = good[3].copy()
        pb[5] = bad_pb
        rows, keep = _raw([good, (good[0], good[1], good[2], pb)])
        hs = (C.c_void_p * 2)(1, 1)  # not NULL before the call
        st = (_lib.MergeStats * 2)()
        assert L.vmb_parts_from_rows(ctx, rows, 2, hs, st) == -50
        assert not hs[0] and not hs[1]
    rows, keep = _raw([good])
    hs = (C.c_void_p * 1)(1)
    st = (_lib.MergeStats * 1)()
    assert L.vmb_parts_from_rows(None, rows, 1, hs, st) == -50
    assert L.vmb_parts_from_rows(ctx, None, 1, hs, st) == -50
    assert L.vmb_parts_from_rows(ctx, rows, 1, None, st) == -50
    assert L.vmb_parts_from_rows(ctx, rows, 1, hs, None) == -50
    for field in ("tsids", "timestamps", "values", "precision_bits"):
        rows, keep = _raw([good])
        setattr(rows[0], field, None)
        hs[0] = 1
        assert L.vmb_parts_from_rows(ctx, rows, 1, hs, st) == -50 and not hs[0]
    rows, keep = _raw([good])
    rows[0].n = 1 << 32  # raw_row.go:85; rejected before any row is read
    hs[0] = 1
    assert L.vmb_parts_from_rows(ctx, rows, 1, hs, st) == -50 and not hs[0]
