"""The restatement of marshalToInmemoryPart (tests/raw_rows_ref.py) against the reference's own tests: the literal rows of
part_search_test.go, the shapes of inmemory_part_test.go, and the cut rule's corner cases.  CPU only: every part is read back through
libzstd and the oracle (part_merge_ref.read_part)."""
import numpy as np

import partgen
import raw_rows_ref as R

PB = 4  # defaultPrecisionBits inmemory_part_test.go:8


def rows_of(tsids, ts, vals, pb=PB):
    ids = np.frombuffer(b"".join(tsids), dtype=np.uint8).reshape(-1, 24)
    return ids, np.asarray(ts, dtype=np.int64), np.asarray(vals, dtype=np.float64), np.full(len(ts), pb, dtype=np.uint8)


def read_back(part):
    """[(tsid, ts, float values)] of every block, through libzstd and the oracle"""
    out = []
    for t, h, ts, vs in R.read_part(part["metaindex_bin"], part["index_bin"], part["timestamps_bin"], part["values_bin"],
                                    len(part["metaindex_raw"]) + 16):
        out.append((t, ts, [v * 10.0 ** h["scale"] for v in vs]))
    return out


def tsid(mid, mg=0, job=0, inst=0):
    return partgen.pack_tsid(mg, job, inst, mid)


def test_part_search_one_row():  # part_search_test.go:14
    p = R.marshal_to_inmemory_part(*rows_of([tsid(1234)], [100], [345]))
    assert read_back(p) == [(tsid(1234), [100], [345.0])]
    assert p["stats"] == dict(rows_count=1, blocks_count=1, min_ts=100, max_ts=100, rows_merged=1, rows_deleted=0)


def test_part_search_two_rows_one_tsid():  # part_search_test.go:315
    p = R.marshal_to_inmemory_part(*rows_of([tsid(1234)] * 2, [100, 200], [345, 456]))
    assert read_back(p) == [(tsid(1234), [100, 200], [345.0, 456.0])]


def test_part_search_two_rows_two_tsids():  # part_search_test.go:644
    p = R.marshal_to_inmemory_part(*rows_of([tsid(1234), tsid(2345)], [100, 200], [345, 456]))
    assert read_back(p) == [(tsid(1234), [100], [345.0]), (tsid(2345), [200], [456.0])]
    # the same rows given in the other order are sorted first
    q = R.marshal_to_inmemory_part(*rows_of([tsid(2345), tsid(1234)], [200, 100], [456, 345]))
    assert q["index_bin"] == p["index_bin"] and q["values_bin"] == p["values_bin"]


def check_header(p, ts, rows, blocks):  # testInmemoryPartInitFromRows inmemory_part_test.go:52
    st = p["stats"]
    assert (st["rows_count"], st["blocks_count"], st["min_ts"], st["max_ts"]) == (rows, blocks, int(np.min(ts)), int(np.max(ts)))
    assert st["rows_merged"] == rows


def test_inmemory_part_init_from_rows_shapes():  # inmemory_part_test.go:10, a seeded numpy RNG for math/rand
    p = R.marshal_to_inmemory_part(*rows_of([tsid(234)], [123], [456.789]))
    check_header(p, [123], 1, 1)
    rng = np.random.default_rng(1)
    n = 10_000
    ts = (rng.standard_normal(n) * 1e7).astype(np.int64)
    p = R.marshal_to_inmemory_part(*rows_of([tsid(7, 1, 2, 3)] * n, ts, rng.standard_normal(n) * 100))
    check_header(p, ts, n, 2)
    got = read_back(p)
    assert [len(b[1]) for b in got] == [8192, n - 8192]
    assert p["blocks"][0][2] + p["blocks"][1][2] == sorted(ts.tolist())  # the rows written; precisionBits 4 changes them on disk
    ts = (rng.standard_normal(n) * 1e7).astype(np.int64)
    ids = [tsid(i, 1, 2, 3) for i in range(n)]
    pbs = (np.arange(n) % 64 + 1).astype(np.uint8)
    ids_a, ts_a, vals_a, _ = rows_of(ids, ts, rng.standard_normal(n) * 100)
    p = R.marshal_to_inmemory_part(ids_a, ts_a, vals_a, pbs)
    check_header(p, ts, n, n)
    assert [b[1]["precision_bits"] for b in p["blocks"]] == pbs.tolist()


def test_cut_same_metric_id_other_tsids():
    a, b, c = tsid(5, 1, 1), tsid(5, 1, 2), tsid(5, 2, 1)
    p = R.marshal_to_inmemory_part(*rows_of([c, b, a, b], [4, 3, 2, 1], [1, 2, 3, 4], 64))
    assert [(t, ts) for t, ts, _ in read_back(p)] == [(a, [2, 1, 3, 4])]  # one block, the TSID of its first row
    # a row of another MetricID sorted between them splits the MetricID into blocks that are not adjacent
    d = tsid(6, 1, 3)
    p = R.marshal_to_inmemory_part(*rows_of([c, d, b, a], [4, 9, 3, 2], [1, 5, 2, 3], 64))
    assert [(t, ts) for t, ts, _ in read_back(p)] == [(a, [2, 3]), (d, [9]), (c, [4])]


def test_cut_at_max_rows_per_block():
    for n, sizes in ((8192, [8192]), (8193, [8192, 1]), (16385, [8192, 8192, 1])):
        ts = np.arange(n, dtype=np.int64) * 1000
        p = R.marshal_to_inmemory_part(*rows_of([tsid(1)] * n, ts, np.arange(n) % 17, 64))
        assert [b[1]["rows"] for b in p["blocks"]] == sizes
        assert sum((b[1] for b in read_back(p)), []) == ts.tolist()


def test_sorted_input_with_equal_keys_keeps_its_order():
    t = [tsid(1)] * 4 + [tsid(2)] * 2
    ts = [10, 10, 10, 20, 5, 5]
    vals = [3, 1, 2, 7, 9, 8]
    order = R.sort_order(rows_of(t, ts, vals)[0], ts)
    assert order == list(range(6))  # already sorted: the input order
    p = R.marshal_to_inmemory_part(*rows_of(t, ts, vals, 64))
    assert [v for _, _, v in read_back(p)] == [[3.0, 1.0, 2.0, 7.0], [9.0, 8.0]]
    # reversed, rows with equal keys keep their relative input order (the library's stable sort)
    assert R.sort_order(rows_of(t[::-1], ts[::-1], vals)[0], ts[::-1]) == [3, 4, 5, 2, 0, 1]
