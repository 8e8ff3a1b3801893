"""The merge restatement (tests/part_merge_ref.py) on its own: Go's heap ties, the dedup vectors of dedup_test.go, and the part
shapes of merge_test.go.  Needs no GPU: the restatement's writer is the library's host writer."""
import numpy as np
import pytest

import part_merge_ref as R
import partgen
from blockgen import OBlock

T0 = 1_700_000_000_000


def tsid(mid, mg=1):
    return partgen.pack_tsid(mg, 0, 0, mid)


def test_heap_ties_follow_go_container_heap():
    # four parts, every block with the same (MetricID, MinTimestamp): the order is container/heap's, not a stable sort
    h = dict(min_ts=0)
    parts = [[(tsid(1), h)] * 2 for _ in range(4)]
    order = R.merged_order(parts)
    assert len(order) == 8
    # hand-traced: Init keeps [0,1,2,3]; every Fix(0) with equal keys keeps the top; Pop swaps the last reader to the top
    assert order == [(0, 0), (0, 1), (3, 0), (3, 1), (2, 0), (2, 1), (1, 0), (1, 1)]


def test_heap_orders_by_tsid_then_min_timestamp():
    parts = [[(tsid(2), dict(min_ts=5)), (tsid(3), dict(min_ts=0))], [(tsid(1), dict(min_ts=9)), (tsid(2), dict(min_ts=1))],
             [(tsid(2), dict(min_ts=5))]]
    order = R.merged_order(parts)
    got = [(R.metric_id(parts[p][i][0]), parts[p][i][1]["min_ts"]) for p, i in order]
    assert got == [(1, 9), (2, 1), (2, 5), (2, 5), (3, 0)]


@pytest.mark.parametrize("ts,vals,interval,want_ts,want_vals", [
    # the shapes of dedup_test.go:97, traced by hand through dedup.go:94
    ([1000, 1001, 1002, 1003], [1, 2, 3, 4], 0, [1000, 1001, 1002, 1003], [1, 2, 3, 4]),
    ([1000, 1001, 1002, 1003, 1004], [1, 2, 3, 4, 5], 10, [1000, 1004], [1, 5]),
    ([1000, 1000, 1000], [3, 1, 2], 10, [1000], [3]),
    ([1000, 1000, 1001], [R.STALE_NAN, 7, 1], 10, [1000, 1001], [7, 1]),
    ([1000, 1000], [R.STALE_NAN, 7], 1, [1000], [7]),
    ([1000, 1000], [7, R.STALE_NAN], 1, [1000], [7]),
    ([1000, 1000], [R.STALE_NAN, R.STALE_NAN], 1, [1000], [R.STALE_NAN]),
    ([0, 10, 11, 20, 21, 35], [1, 2, 3, 4, 5, 6], 10, [0, 10, 20, 21, 35], [1, 2, 4, 5, 6]),
])
def test_dedup_vectors(ts, vals, interval, want_ts, want_vals):
    assert R.deduplicate_samples_during_merge(ts, vals, interval) == (want_ts, want_vals)


def test_calibrate_scale_overflow_path():
    a = [R.INT64_MAX // 10, 5]
    b = [123456, -123456]
    e = R.calibrate_scale(a, 3, b, 0)
    # a can go up by one digit only: the common exponent is 2 and b is divided by 100 (truncated toward zero)
    assert e == 2 and a == [R.INT64_MAX // 10 * 10, 50] and b == [1234, -1234]


@pytest.mark.parametrize("interval,ts,want_ts,want_vals", [
    # dedup_test.go:178 TestDeduplicateSamplesDuringMerge (values = row index)
    (1, [123], [123], [0]),
    (1, [123, 456], [123, 456], [0, 1]),
    (1, [0, 0, 0, 1, 1, 2, 3, 3, 3, 4], [0, 1, 2, 3, 4], [2, 4, 5, 8, 9]),
    (100, [0, 100, 100, 101, 150, 180, 200, 300, 1000], [0, 100, 200, 300, 1000], [0, 2, 6, 7, 8]),
    (10_000, [10e3, 13e3, 21e3, 22e3, 30e3, 33e3, 39e3, 45e3], [10e3, 13e3, 30e3, 39e3, 45e3], [0, 1, 4, 6, 7]),
    # dedup_test.go:293 TestDeduplicateSamplesDuringMerge_KeepsFirstAndLast (values = row index)
    (1000, [0, 200, 400, 800, 1000, 1300, 1500, 2100, 2400, 2500, 2500], [0, 1000, 1500, 2500], [0, 4, 6, 10]),
    (1000, [0, 100, 200, 300, 700, 1000, 1600, 1700, 1800, 2300, 2400, 2500], [0, 1000, 1800, 2500], [0, 5, 8, 11]),
    (1000, [1000], [1000], [0]),
])
def test_dedup_reference_vectors(interval, ts, want_ts, want_vals):
    ts = [int(t) for t in ts]
    got = R.deduplicate_samples_during_merge(ts, list(range(len(ts))), interval)
    assert got == ([int(t) for t in want_ts], want_vals)
    assert R.deduplicate_samples_during_merge(*got, interval) == got  # a second pass changes nothing


def _stream(series_rows, pb):
    """one blockStreamReader: {metric_id: (ts, vals)} -> restatement input, blocks cut like inmemoryPart.InitFromRows"""
    series = []
    for mid in sorted(series_rows):
        ts, vals = series_rows[mid]
        o = np.argsort(ts, kind="stable")
        ts, vals = np.asarray(ts, dtype=np.int64)[o], np.asarray(vals, dtype=np.int64)[o]
        series.append((tsid(mid), [OBlock(t, v, 0, pb) for t, v in R.split_rows(ts, vals)]))
    return R.part_from_series(series)[1]


def _check(streams, blocks, rows, min_ts, max_ts, pb):
    out = R.merge_parts(streams, marshal=R.oracle_marshal, frame=R.oracle_frame)
    st = out["stats"]
    assert (st["blocks_count"], st["rows_count"], st["min_ts"], st["max_ts"]) == (blocks, rows, min_ts, max_ts)
    assert st["rows_merged"] == rows and st["rows_deleted"] == 0
    # the written part decodes through libzstd and the oracle to the rows the restatement wrote
    got = R.read_part(out["metaindex_bin"], out["index_bin"], out["timestamps_bin"], out["values_bin"], len(out["metaindex_raw"]) + 16)
    assert [(t, h["rows"]) for t, h, _, _ in got] == [(t, h["rows"]) for t, h, _, _ in out["blocks"]]
    if pb == 64:
        assert [(ts, vs) for _, _, ts, vs in got] == [(ts, vs) for _, _, ts, vs in out["blocks"]]


def test_merge_test_go_one_stream_one_row():
    _check([_stream({1: ([123], [5])}, 64)], 1, 1, 123, 123, 64)


def test_merge_test_go_two_streams_big_overlapping_blocks():
    rng = np.random.default_rng(1)
    n1, n2 = R.MAX_ROWS_PER_BLOCK + 234, R.MAX_ROWS_PER_BLOCK + 2344
    s1 = {1: (np.arange(n1) * 2894, (rng.standard_normal(n1) * 100).astype(np.int64))}
    s2 = {1: (np.arange(n2) * 2494, (rng.standard_normal(n2) * 100).astype(np.int64))}
    _check([_stream(s1, 5), _stream(s2, 5)], 3, n1 + n2, 0, max((n1 - 1) * 2894, (n2 - 1) * 2494), 5)


def test_merge_test_go_two_streams_big_sequential_blocks():
    rng = np.random.default_rng(2)
    n1, n2 = R.MAX_ROWS_PER_BLOCK + 234, R.MAX_ROWS_PER_BLOCK - 233
    t1 = np.arange(n1) * 2894
    s1 = {1: (t1, (rng.standard_normal(n1) * 100).astype(np.int64))}
    s2 = {1: (t1[-1] + np.arange(n2) * 2494, (rng.standard_normal(n2) * 100).astype(np.int64))}
    _check([_stream(s1, 5), _stream(s2, 5)], 3, n1 + n2, 0, int(t1[-1] + (n2 - 1) * 2494), 5)


def test_merge_test_go_many_streams_many_blocks_many_rows():
    rng = np.random.default_rng(3)
    streams, total, mn, mx = [], 0, R.INT64_MAX, R.INT64_MIN
    for _ in range(20):
        n = int(rng.integers(113, 500))
        ts = rng.integers(0, 10 ** 9, n)
        vals = rng.integers(-1000, 1000, n)
        rows = {}
        for j in range(n):
            rows.setdefault(j % 113 + 1, ([], []))
            rows[j % 113 + 1][0].append(int(ts[j]))
            rows[j % 113 + 1][1].append(int(vals[j]))
        streams.append(_stream(rows, 64))
        total, mn, mx = total + n, min(mn, int(ts.min())), max(mx, int(ts.max()))
    _check(streams, 113, total, mn, mx, 64)


def test_merge_test_go_one_stream_many_blocks():
    # TestMergeBlockStreamsOneStreamManyBlocksManyRows: one stream, many series of a few rows each
    rng = np.random.default_rng(4)
    rows = {m: (sorted(rng.integers(0, 10 ** 6, 7).tolist()), rng.integers(0, 100, 7).tolist()) for m in range(1, 120)}
    mn = min(r[0][0] for r in rows.values())
    mx = max(r[0][-1] for r in rows.values())
    _check([_stream(rows, 64)], 119, 119 * 7, mn, mx, 64)
