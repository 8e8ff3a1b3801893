"""tests/aggr_matrix_ref.py (the reference of vmb_aggr_matrix) on the query vectors of the reference's own
app/vmselect/promql/exec_test.go: the label_set(...) series at 1000 ... 2000 s, step 200 s, and the expected values as written
there.  Where the Go query ends in round(..., 0.001), the result is rounded the same way."""
import numpy as np
import pytest

from aggr_matrix_ref import aggr_matrix_ref

NAN = float("nan")
T = np.arange(1000, 2001, 200, dtype=np.float64)  # time() of exec_test.go: start 1000e3, end 2000e3, step 200e3 ms
FOUR = [T / 100 + 10, T / 200 + 5, T / 110 - 10, T / 90 - 5]  # the share() / zscore() series, k = v1 .. v4


def go_round(v, nearest, p10):
    """transform.go round(q, nearest): p10 = math.Pow10(-e) with (_, e) = decimal.FromFloat(nearest)"""
    with np.errstate(all="ignore"):
        x = v + 0.5 * np.copysign(nearest, v)
        x = x - np.fmod(x, nearest)
        return np.trunc(x * p10) / p10


def r3(v):
    return go_round(np.asarray(v, dtype=np.float64), 0.001, 1e3)


def check(got, want):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape
    assert np.array_equal(np.isnan(got), np.isnan(want)), (got, want)
    assert np.array_equal(got[~np.isnan(got)], want[~np.isnan(want)]), (got, want)


def ten_or_time(second):
    """label_set(10, ...) or label_set(<second>, ...): two series"""
    return np.array([np.full(6, 10.0), second])


@pytest.mark.parametrize("name, rows, want", [
    ("sum", [T / 100], [10, 12, 14, 16, 18, 20]),                                # :5687 sum(time)
    ("geomean", [T / 100], [10, 12, 14, 16, 18, 20]),                            # :5698 geomean(time)
    ("sum2", [T / 100], [100, 144, 196, 256, 324, 400]),                         # :5721 sum2(time)
    ("sum", ten_or_time(T / 100), [20, 22, 24, 26, 28, 30]),                     # :5754 sum(multi-vector)
    ("sum2", ten_or_time(T / 100), [200, 244, 296, 356, 424, 500]),              # :5776
    ("avg", ten_or_time(T / 100), [10, 11, 12, 13, 14, 15]),                     # :5798
    ("stddev", ten_or_time(T / 100), [0, 1, 2, 3, 4, 5]),                        # :5809
    ("count", [np.where(T < 1500, T, NAN), np.where(T < 1800, T, NAN)], [2, 2, 2, 1, NAN, NAN]),  # :5820
    ("min", ten_or_time(T / 100 / 1.5), [6.666666666666667, 8, 9.333333333333334, 10, 10, 10]),      # :5905
    ("max", ten_or_time(T / 100 / 1.5), [10, 10, 10, 10.666666666666666, 12, 13.333333333333334]),   # :5916
    ("group", [np.full(6, 5.0), np.full(6, 6.0), np.full(6, 7.0)], [1, 1, 1, 1, 1, 1]),             # :6552 group() by (test)
])
def test_one_group(name, rows, want):
    out, groups = aggr_matrix_ref(name, np.array(rows, dtype=np.float64))
    check(out[0], want)
    assert groups.tolist() == [0]


def test_geomean_multi_vector():
    """:5765 round(geomean(...), 0.1)"""
    out, _ = aggr_matrix_ref("geomean", ten_or_time(T / 100))
    check(go_round(out[0], 0.1, 10.0), [10, 11, 11.8, 12.6, 13.4, 14.1])


def test_sum_by_known_tag_and_limit():
    """:5831 sum(...) by (foo): {foo="bar"} = 10 and {} = time()/100; :5851 ... limit 1 keeps the group of the first series;
    :5866 by (foo, baz, foo) puts both in one group; :5887 by (__name__) keeps two"""
    vals = ten_or_time(T / 100)
    out, groups = aggr_matrix_ref("sum", vals, [0, 1], 2)
    check(out[0], [10] * 6)
    check(out[1], [10, 12, 14, 16, 18, 20])
    assert groups.tolist() == [0, 1]
    out, groups = aggr_matrix_ref("sum", vals, [0, 1], 2, limit=1)
    assert groups.tolist() == [0]
    check(out[0], [10] * 6)
    out, groups = aggr_matrix_ref("sum", vals, [0, 0], 1)
    check(out[0], [20, 22, 24, 26, 28, 30])
    out, groups = aggr_matrix_ref("sum", vals, [1, 0], 2)
    check(out[1], [10] * 6)
    check(out[0], [10, 12, 14, 16, 18, 20])
    assert groups.tolist() == [1, 0]


def test_share():
    """:5436 sort_by_label(round(share(...), 0.001), "k")"""
    out, mask = aggr_matrix_ref("share", np.array(FOUR))
    assert mask.tolist() == [True] * 4
    check(r3(out[0]), [0.554, 0.521, 0.487, 0.462, 0.442, 0.426])
    check(r3(out[1]), [0.277, 0.26, 0.243, 0.231, 0.221, 0.213])
    check(r3(out[2]), [NAN, 0.022, 0.055, 0.081, 0.1, 0.116])
    check(r3(out[3]), [0.169, 0.197, 0.214, 0.227, 0.237, 0.245])


def test_sum_of_share():
    """:5483 round(sum(share(...)), 0.001) = 1 and :5499 round(sum(share(...) by (k)), 0.001) = 2"""
    sh, _ = aggr_matrix_ref("share", np.array(FOUR))
    s, _ = aggr_matrix_ref("sum", sh)
    check(r3(s[0]), [1] * 6)
    sh, _ = aggr_matrix_ref("share", np.array(FOUR), [0, 1, 0, 1], 2)  # k = v1, v2, v1, v2
    s, _ = aggr_matrix_ref("sum", sh)
    check(r3(s[0]), [2] * 6)


def test_zscore():
    """:5515 sort_by_label(round(zscore(...), 0.001), "k")"""
    out, _ = aggr_matrix_ref("zscore", np.array(FOUR))
    check(r3(out[0]), [1.482, 1.511, 1.535, 1.552, 1.564, 1.57])
    check(r3(out[1]), [0.159, 0.058, -0.042, -0.141, -0.237, -0.329])
    check(r3(out[2]), [-1.285, -1.275, -1.261, -1.242, -1.219, -1.193])
    check(r3(out[3]), [-0.356, -0.294, -0.232, -0.17, -0.108, -0.048])


def test_fast_paths_and_empty_rows():
    """aggrPrepareSeries drops all-NaN rows first, so a group of one value row and an empty row takes the `len(tss) == 1` path"""
    row = np.array([-0.0, 3.0, NAN, np.inf])
    vals = np.array([np.full(4, NAN), row])
    out, groups = aggr_matrix_ref("sum", vals)
    assert groups.tolist() == [0] and np.signbit(out[0, 0])  # the row itself keeps -0.0
    out, _ = aggr_matrix_ref("sum2", vals)
    assert not np.signbit(out[0, 0])  # 0 + (-0.0)(-0.0) = +0.0
    out, _ = aggr_matrix_ref("stdvar", vals)
    check(out[0], [0, 0, NAN, 0])
    out, _ = aggr_matrix_ref("stdvar", np.array([row, row]))
    check(out[0], [0, 0, NAN, NAN])  # the general path: inf - inf
    out, groups = aggr_matrix_ref("count", np.full((2, 4), NAN))
    assert groups.tolist() == [] and np.isnan(out).all()
