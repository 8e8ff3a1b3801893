"""tests/rank_aggr_ref.py (the reference of vmb_aggr_rank) on the query vectors of the reference's own
app/vmselect/promql/exec_test.go: topk_min(1) ... bottomk_last(1), the three topk_max(k, ..., "remaining_sum") cases (:6622-6850)
and outliersk(0 / 1 / 3) (:7347-7400), with the expected values as written there.  time() is 1000 ... 2000 in steps of 200."""
import numpy as np
import pytest

from rank_aggr_ref import NAMES, int_k, rank_aggr_ref

T = np.arange(1000, 2001, 200, dtype=np.float64)
TEN = [10.0] * 6
T150 = [6.666666666666667, 8, 9.333333333333334, 10.666666666666666, 12, 13.333333333333334]


def result(name, k, vals, remaining=False):
    """the returned series as lists of values, in output order"""
    r = rank_aggr_ref(name, k, np.array(vals), remaining=remaining)
    return [(r["remaining"][-x - 1] if x < 0 else r["masked"][x]).tolist() for x in r["out"]]


@pytest.mark.parametrize("name,div,want", [
    ("topk_min", 150, TEN), ("bottomk_min", 150, T150), ("topk_max", 150, T150), ("bottomk_max", 150, TEN),
    ("topk_avg", 150, T150), ("bottomk_avg", 150, T150), ("topk_median", 150, T150), ("topk_last", 150, T150),
    ("bottomk_median", 15, TEN), ("bottomk_last", 15, TEN)])
def test_range_topk_vectors(name, div, want):
    assert result(name, 1, [np.full(6, 10.0), T / div]) == [want]


def test_remaining_sum_vectors():
    vals = [np.full(6, 10.0), T / 150]
    assert result("topk_max", 1, vals, remaining=True) == [TEN, T150]  # the remaining-sum row comes first, then the survivor
    assert result("topk_max", 2, vals, remaining=True) == [T150, TEN]  # nothing remains: no remaining-sum row
    assert result("topk_max", 3, vals, remaining=True) == [T150, TEN]


def test_outliersk_vectors():
    assert result("outliersk", 0, [np.full(6, 1300.0), T]) == []
    assert result("outliersk", 1, [np.full(6, 2000.0), T]) == [T.tolist()]  # equal scores: the later row is the better one
    assert result("outliersk", 3, [np.full(6, 1300.0), T]) == [T.tolist(), [1300.0] * 6]


def test_int_k():
    nan, inf = float("nan"), float("inf")
    assert [int_k(k, 7) for k in (nan, -1, -0.5, 0, 0.9, 1, 2.99, 7, 8, 1e300, inf, -inf)] == [0, 0, 0, 0, 0, 1, 2, 7, 7, 7, 7, 0]


def test_stable_ties_and_nan_scores():
    """equal scores keep ascending row order from worst to best, so the later row wins; NaN scores are the worst both ways"""
    inf = float("inf")
    vals = np.array([[1.0, 1.0], [1.0, 1.0], [-0.0, 0.0], [0.0, -0.0], [inf, -inf], [-inf, inf]])
    r = rank_aggr_ref("topk_avg", 6, vals)
    assert r["out"].tolist() == [1, 0, 3, 2, 5, 4] and np.isnan(r["scores"][4:]).all()
    assert rank_aggr_ref("bottomk_avg", 6, vals)["out"].tolist() == [3, 2, 1, 0, 5, 4]
    assert rank_aggr_ref("topk_avg", 2, vals)["out"].tolist() == [1, 0]
    assert sorted(NAMES) == sorted(set(NAMES)) and len(NAMES) == 11
