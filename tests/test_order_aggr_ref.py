"""tests/order_aggr_ref.py (the reference of vmb_aggr_order) on the query vectors of the reference's own
app/vmselect/promql/exec_test.go: the label_set(...) series at 1000 ... 2000 s, step 200 s, and the expected values as written
there."""
import math

import numpy as np
import pytest

from order_aggr_ref import aggr_order_ref, mad, mode_no_nans, quantile_sorted

NAN, INF = float("nan"), float("inf")
T = np.arange(1000, 2001, 200, dtype=np.float64)  # time() of exec_test.go: start 1000e3, end 2000e3, step 200e3 ms
TEN_OR_T150 = np.array([np.full(6, 10.0), T / 150])  # label_set(10, "foo", "bar") or label_set(time()/150, "baz", "sss")
MAD3 = np.array([T, T * 1.5, T * 0.9])  # alias(time(), "metric1"), alias(time()*1.5, "metric2"), label_set(time()*0.9, ...)


def check(got, want):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape
    assert np.array_equal(np.isnan(got), np.isnan(want)), (got, want)
    assert np.array_equal(got[~np.isnan(got)], want[~np.isnan(want)]), (got, want)


def test_mode():
    """:5418 mode(alias(3), alias(2), alias(3), alias(4), alias(3), alias(2))"""
    out, groups = aggr_order_ref("mode", np.array([np.full(6, x) for x in (3.0, 2.0, 3.0, 4.0, 3.0, 2.0)]))
    check(out[0], [3] * 6)
    assert groups.tolist() == [0]


def test_distinct():
    """:7046 distinct(union(1+time() > 1100, label_set(time() > 1700, "foo", "bar")))"""
    a = np.where(1 + T > 1100, 1 + T, NAN)
    b = np.where(T > 1700, T, NAN)
    out, _ = aggr_order_ref("distinct", np.array([a, b]))
    check(out[0], [NAN, 1, 1, 1, 2, 2])


def test_quantiles():
    """:7218 quantiles("phi", 0.2, 0.5, ...): one output series per phi"""
    out, _ = aggr_order_ref("quantiles", TEN_OR_T150, phis=[0.2, 0.5])
    check(out[0, 0], [7.333333333333334, 8.4, 9.466666666666669, 10.133333333333333, 10.4, 10.666666666666668])
    check(out[1, 0], [8.333333333333334, 9, 9.666666666666668, 10.333333333333332, 11, 11.666666666666668])


@pytest.mark.parametrize("phi, rows, want", [
    (-2, TEN_OR_T150, [-INF] * 6),                                                                       # :7184 quantile(-2)
    (0.2, TEN_OR_T150, [7.333333333333334, 8.4, 9.466666666666669, 10.133333333333333, 10.4, 10.666666666666668]),  # :7196
    (0.5, TEN_OR_T150, [8.333333333333334, 9, 9.666666666666668, 10.333333333333332, 11, 11.666666666666668]),     # :7207 and
    (0.5, np.array([np.full(6, 10.0), T / 150, T / 200]), [6.666666666666667, 8, 9.333333333333334, 10, 10, 10]),  # median()
    (3, TEN_OR_T150, [INF] * 6),                                                                         # :7264 quantile(3)
    (NAN, TEN_OR_T150, [NAN] * 6),                                                                       # quantile(NaN)
])
def test_quantile_one_phi(phi, rows, want):
    """:7184-7275 quantile(phi, ...) and median(...) as quantiles with one phi"""
    out, _ = aggr_order_ref("quantiles", rows, phis=[phi])
    check(out[0, 0], want)


def test_mad():
    """:7282 mad(time(), time()*1.5, time()*0.9)"""
    out, _ = aggr_order_ref("mad", MAD3)
    check(out[0], [100, 120, 140, 160, 180, 200])


def test_outliers_iqr():
    """:7297 outliers_iqr(time(), time()*1.5, time()*10, time()*1.2, time()*0.1): m3 and m5"""
    _, sel = aggr_order_ref("outliers_iqr", np.array([T, T * 1.5, T * 10, T * 1.2, T * 0.1]))
    assert sel.tolist() == [False, False, True, False, True]


@pytest.mark.parametrize("tol, want", [(1, [False, True, False]), (5, [False, False, False])])
def test_outliers_mad(tol, want):
    """:7321 outliers_mad(1, ...) returns metric2; :7337 outliers_mad(5, ...) returns nothing"""
    _, sel = aggr_order_ref("outliers_mad", MAD3, tolerance=tol)
    assert sel.tolist() == want


def test_cell_rules():
    """the rules the kernels reproduce: Inf * 0 in the interpolation, NaN deviations dropped, runs over -0.0 / +0.0"""
    assert math.isnan(quantile_sorted(0.5, [1.0, 2.0, INF]))  # 2 * 1 + Inf * 0
    assert quantile_sorted(0.25, [1.0, 2.0, 3.0, INF]) == 1.75
    med, m = mad([INF, INF, 1.0, 2.0])  # median 2 / 2 + Inf / 2 = Inf, deviations NaN NaN Inf Inf: the NaNs are dropped
    assert med == INF and m == INF
    med, m = mad([1.0, 2.0, INF])  # NaN median: every deviation is NaN
    assert math.isnan(med) and math.isnan(m)
    assert mode_no_nans([0.0, -0.0, 1.0, 1.0]) == 0.0  # one run of two zeros, the first of the longest runs
    assert mode_no_nans([5.0, 1.0, 5.0, 1.0]) == 1.0
    out, _ = aggr_order_ref("distinct", np.array([[0.0], [-0.0], [NAN]]))
    assert out[0, 0] == 1.0


def test_groups_limit_and_empty_rows():
    vals = np.array([np.full(3, NAN), [1.0, 2, 3], [4.0, 5, 6], [7.0, NAN, 9]])
    out, groups = aggr_order_ref("mode", vals, [0, 2, 1, 2], 4)
    assert groups.tolist() == [2, 1] and np.isnan(out[0]).all() and np.isnan(out[3]).all()
    check(out[2], [1, 2, 3])
    _, groups = aggr_order_ref("mode", vals, [0, 2, 1, 2], 4, limit=1)
    assert groups.tolist() == [2]
    _, sel = aggr_order_ref("outliers_iqr", np.array([[1.0], [2.0], [3.0], [100.0]]), [0, 0, 0, 0], limit=1)
    assert sel.tolist() == [False, False, False, True]
