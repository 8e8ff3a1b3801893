"""CPU checks of tests/vm_histogram_ref.py, the restatement vmb_aggr_histogram and vmb_rollup_histogram are held to: Go's log
constants, the bucket rule on the exec_test.go vectors and at every power of ten, the `vmrange` label table, and
histogram_over_time over the oracle's windows."""
import math
import random
import struct

import numpy as np
import pytest

import vm_histogram_ref as H
from vmrange_ref import go_parse_float

NAN, INF = float("nan"), float("inf")


def test_log_constants_match_their_encodings():
    for name, (v, enc) in H.CONSTS.items():
        assert H.bits(v) == enc, name
    # 1/Ln10 is the quotient of Go's Ln10 literal rounded once; its neighbours are farther from it
    q = 1 / H.LN10
    assert H.bits(H.INV_LN10) == 0x3FDBCB7B1526E50E
    for nb in (H.from_bits(0x3FDBCB7B1526E50D), H.from_bits(0x3FDBCB7B1526E50F)):
        assert abs(H.Fraction(nb) - q) > abs(H.Fraction(H.INV_LN10) - q)
    assert H.bits(H.HALF_SQRT2) == 0x3FE6A09E667F3BCD


def test_go_log_is_a_faithful_log():
    rng = random.Random(1)
    for _ in range(20000):
        x = 10 ** rng.uniform(-300, 300)
        y = H.go_log(x)
        assert abs(y - math.log(x)) <= 2 * math.ulp(math.log(x)), x
    assert H.go_log(1.0) == 0.0 and H.go_log(0.0) == -INF and H.go_log(INF) == INF
    assert math.isnan(H.go_log(-1.0)) and math.isnan(H.go_log(NAN))
    assert H.go_log(5e-324) == pytest.approx(math.log(5e-324), rel=1e-15)


def test_label_table():
    labels = H.LABELS
    assert len(labels) == H.NB == 488
    assert labels[0] == "0...1.000e-09" and labels[-1] == "1.000e+18...+Inf"
    assert len(set(labels[1:-1])) == 486
    bounds = [lab.split("...") for lab in labels]
    for a, b in zip(bounds, bounds[1:]):
        assert a[1] == b[0]  # each bucket's end is the next bucket's start
    for a, b in bounds:
        if b != "+Inf":
            assert go_parse_float(a) < go_parse_float(b)
    # the labels do not depend on the last bits of Go's math.Pow(10, 1/18)
    m = 10 ** (1 / 18)
    for d in range(-8, 9):
        assert H.vmrange_labels(H.from_bits(H.bits(m) + d)) == labels, d
    for s in ("1.136e+02...1.292e+02", "8.799e-01...1.000e+00", "1.000e+00...1.136e+00", "1.136e+00...1.292e+00"):
        assert s in labels


def test_product_table_is_the_restated_one():
    from victoriametrics_b200 import promql
    t = promql.vmrange_table()
    assert t["labels"] == H.LABELS
    for b in range(H.NB):
        s, e = H.LABELS[b].split("...")
        assert t["strings"][t["start_ids"][b]] == s and t["strings"][t["end_ids"][b]] == e
        assert H.bits(t["starts"][b]) == H.bits(go_parse_float(s)) and H.bits(t["ends"][b]) == H.bits(go_parse_float(e))
    assert len(t["strings"]) == 489 and len(set(t["strings"])) == 489


def test_exec_test_buckets():
    assert H.LABELS[H.bucket(123.0)] == "1.136e+02...1.292e+02"
    assert H.LABELS[H.bucket(1.0)] == "8.799e-01...1.000e+00"
    assert H.LABELS[H.bucket(1.1)] == "1.000e+00...1.136e+00"
    assert H.LABELS[H.bucket(1.15)] == "1.136e+00...1.292e+00"


def test_powers_of_ten_end_their_bucket():
    for n in range(-8, 18):
        b = H.bucket(float("1e%d" % n))
        assert H.LABELS[b].endswith("...1.000e%+03d" % n), n
        assert H.LABELS[H.bucket(float("1e%d" % n) * 1.0000001)].startswith("1.000e%+03d..." % n), n
    assert H.bucket(1e-9) == 1  # bucketIdx == 0: the first decimal bucket, idx-- needs idx > 0
    assert H.bucket(1e-9 * 0.9999999) == 0
    assert H.bucket(1e18) == 487 and H.bucket(1e18 * 0.9999999) == 486  # bucketIdx == 486: the upper bucket


def test_specials():
    for v in (0.0, -0.0, 5e-324, 2.2250738585072009e-308, 2.2250738585072014e-308, 1e-10):
        assert H.bucket(v) == 0, v
    assert H.bucket(INF) == 487 and H.bucket(1e300) == 487
    for v in (NAN, -1.0, -5e-324, -INF, struct.unpack("<d", struct.pack("<Q", 0x7FF0000000000002))[0]):
        assert H.bucket(v) is None, v


def test_libm_log10_is_not_enough():
    """the reason for the restatement: near the edges libm's log10 puts doubles in other buckets"""
    diff = 0
    for k in range(0, 487, 7):
        e = 10 ** (k / 18 - 9)
        for d in range(-64, 65):
            x = H.from_bits(H.bits(e) + d)
            diff += H.bucket(x) != H.bucket(x, math.log10)
    assert diff > 0


def _plus_sort(left, right):
    """`left + right` on series labelled only by `le` (matching label sets), then sort() by value (stable)"""
    r = dict(right)
    rows = [(le, np.asarray(v) + r[le]) for le, v in left if le in r]
    return sorted(rows, key=lambda x: x[1][-1])


def test_exec_test_histogram_scalar():
    """exec_test.go:5573 sort(histogram(123) + (le 1.000e+02, 1.136e+02, 1.292e+02: 0; +Inf: 1))"""
    rows = H.histogram_le(np.full((1, 6), 123.0), [0], 1)
    got = _plus_sort([(le, v) for _, le, v in rows],
                     [("1.000e+02", 0.0), ("1.136e+02", 0.0), ("1.292e+02", 0.0), ("+Inf", 1.0)])
    assert [(le, v.tolist()) for le, v in got] == [("1.136e+02", [0.0] * 6), ("1.292e+02", [1.0] * 6), ("+Inf", [2.0] * 6)]


def test_exec_test_histogram_vector():
    """exec_test.go:5618 sort(histogram((1, 1.1, 1.15)) + (le 8.799e-01, 1.000e+00, 1.292e+00: 0; +Inf: 1))"""
    vals = np.array([np.full(6, 1.0), np.full(6, 1.1), np.full(6, 1.15)])
    rows = H.histogram_le(vals, [0, 0, 0], 1)
    got = _plus_sort([(le, v) for _, le, v in rows],
                     [("8.799e-01", 0.0), ("1.000e+00", 0.0), ("1.292e+00", 0.0), ("+Inf", 1.0)])
    assert [(le, v.tolist()) for le, v in got] == [("8.799e-01", [0.0] * 6), ("1.000e+00", [1.0] * 6), ("1.292e+00", [3.0] * 6),
                                                   ("+Inf", [4.0] * 6)]


def test_histogram_rows_zero_filled_and_groups():
    vals = np.array([[1.0, NAN, 2.0], [-1.0, NAN, NAN], [1.0, 1.0, 0.0], [NAN, -3.0, NAN]])
    mat, groups, buckets = H.histogram_rows(vals, [0, 0, 0, 1], 2)
    assert groups == [0, 0, 0]  # group 1 holds only NaN and negatives: no rows
    assert buckets == sorted(buckets) and buckets[0] == 0
    assert mat.tolist() == [[0, 0, 1], [2, 1, 0], [0, 0, 1]]


def test_histogram_over_time_restated():
    t = np.arange(0, 100_000, 10_000, dtype=np.int64)
    v = np.array([1.0, 1.0, NAN, -2.0, 1.1, 0.0, 1e30, 1.0, 5.0, 5.0])
    m, scanned = H.histogram_over_time(v, t, 20_000, 90_000, 20_000, 30_000)
    P = 4
    b1, b11, b5 = H.bucket(1.0), H.bucket(1.1), H.bucket(5.0)
    assert sorted(m) == sorted({0, b1, b11, b5, 487})
    for b, row in m.items():
        assert row.shape == (P,)
        assert not (row == 0).any()  # NaN where a window holds none of the bucket
    # windows (t - 30s, t] at t = 20, 40, 60, 80 s: rows {0, 1, 2}, {2, 3, 4}, {4, 5, 6}, {6, 7, 8}
    assert np.array_equal(m[b1], [2, NAN, NAN, 1], equal_nan=True)
    assert np.array_equal(m[b11], [NAN, 1, 1, NAN], equal_nan=True)
    assert np.array_equal(m[487], [NAN, NAN, 1, 1], equal_nan=True)
    assert scanned >= len(v)


def test_numpy_restatement_is_the_scalar_one():
    rng = np.random.default_rng(3)
    v = np.concatenate([10 ** rng.uniform(-12, 21, 20000), [0.0, -0.0, 5e-324, INF, -INF, NAN, -1.0, 1e-9, 1e18, 1.0, 123.0]])
    edges = [H.from_bits(H.bits(10 ** (k / 18 - 9)) + d) for k in range(487) for d in (-2, -1, 0, 1, 2)]
    v = np.concatenate([v, edges])
    want = [-1 if b is None else b for b in map(H.bucket, v.tolist())]
    assert H.bucket_np(v).tolist() == want
    vals = rng.lognormal(0, 1, (40, 9))
    vals[rng.random(vals.shape) < 0.2] = NAN
    gids = rng.integers(0, 3, 40)
    mat, groups, buckets = H.histogram_counts(vals, gids, 3)
    m2, g2, b2 = H.histogram_rows(vals, gids, 3)
    assert groups == g2 and buckets == b2 and np.array_equal(mat, m2)
