"""tests/range_transform_ref.py (the reference of vmb_transform_range and of smooth_exponential) on the query vectors of the
reference's own app/vmselect/promql/exec_test.go: time() at 1000 ... 2000 s, step 200 s, and the expected values as written
there (`round(..., 0.01)` where the query rounds); plus the rules the tests on the GPU lean on."""
import math

import numpy as np
import pytest

from range_transform_ref import mean, range_row, range_transform_ref, smooth_exponential_ref, stdvar

NAN, INF = float("nan"), float("inf")
STEP = 200_000
T = np.arange(1000, 2001, 200, dtype=np.float64)  # time(): start 1000e3, end 2000e3, step 200e3 ms


def time_where(lo=None, hi=None, hi_incl=False):
    """time() > lo < hi (or <= hi)"""
    keep = np.ones(6, dtype=bool)
    if lo is not None:
        keep &= T > lo
    if hi is not None:
        keep &= (T <= hi) if hi_incl else (T < hi)
    return np.where(keep, T, NAN)


def run(name, row, arg=None):
    out, kept = range_transform_ref(name, np.array([row]), arg, STEP, start=1_000_000)
    return out[0], kept[0]


def check(got, want, nearest=None):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (got, want)
    g, w = got[~np.isnan(got)], want[~np.isnan(want)]
    if nearest is None:
        assert np.array_equal(g, w), (got, want)
    else:  # round(q, nearest)
        assert np.all(np.abs(g - w) <= nearest / 2 + 1e-9 * np.abs(w)), (got, want)


@pytest.mark.parametrize("name, arg, row, want, nearest", [
    ("range_trim_outliers", 0.5, T, [NAN, NAN, 1400, 1600, NAN, NAN], None),                      # :7401
    ("range_trim_outliers", 0.5, time_where(1200), [NAN, NAN, NAN, 1600, 1800, NAN], None),       # :7413
    ("range_trim_spikes", 0.2, T, [NAN, 1200, 1400, 1600, 1800, NAN], None),                      # :7425
    ("range_trim_spikes", 0.2, time_where(1200, 1800, True), [NAN, NAN, NAN, 1600, NAN, NAN], None),  # :7437
    ("range_trim_zscore", 0.9, T, [NAN, 1200, 1400, 1600, 1800, NAN], None),                      # :7449
    ("range_trim_zscore", 0.9, time_where(1200, 1800, True), [NAN, NAN, NAN, 1600, NAN, NAN], None),  # :7461
    ("range_zscore", None, T, [-1.5, -0.9, -0.3, 0.3, 0.9, 1.5], 0.1),                           # :7473
    ("range_zscore", None, time_where(1200, 1800), [NAN, NAN, -1, 1, NAN, NAN], 0.1),             # :7485
    ("range_quantile", 0.5, T, [1500] * 6, None),                                                 # :7497
    ("range_quantile", 0.5, time_where(1200, 2000), [1600] * 6, None),                            # :7509
    ("range_stddev", None, T, [341.57] * 6, 0.01),                                                # :7521 (round)
    ("range_stddev", None, time_where(1200, 1800), [100] * 6, 0.01),                              # :7533
    ("range_stdvar", None, T, [116666.67] * 6, 0.01),                                             # :7545
    ("range_stdvar", None, time_where(1200, 1800), [10000] * 6, 0.01),                            # :7557
    ("range_mad", None, T, [300] * 6, None),                                                      # :8150
    ("range_mad", None, time_where(1200, 1800), [100] * 6, None),                                 # :8162
    ("range_linear_regression", None, T, [1000, 1200, 1400, 1600, 1800, 2000], None),             # :8238
    ("range_linear_regression", None, -T, [-1000, -1200, -1400, -1600, -1800, -2000], None),      # :8250
    ("range_linear_regression", None, time_where(1200, 1800), [1000, 1200, 1400, 1600, 1800, 2000], None),  # :8262
    ("range_linear_regression", None, 100 / T, [0.095, 0.085, 0.075, 0.066, 0.056, 0.046], 0.001),  # :8274 "regress"
])
def test_exec_test_vectors(name, arg, row, want, nearest):
    got, kept = run(name, row, arg)
    assert kept
    check(got, want, nearest)


def test_normalize_two_series():
    """:8094 range_normalize(time(), alias(-time(), "negative")) and :8112 with gaps"""
    out, kept = range_transform_ref("range_normalize", np.array([T, -T]))
    assert kept.all()
    check(out[0], [0, 0.2, 0.4, 0.6, 0.8, 1])
    check(out[1], [1, 0.8, 0.6, 0.4, 0.2, 0])
    out, kept = range_transform_ref("range_normalize", np.array([time_where(1200, 1800), -time_where(1200, 2000)]))
    check(out[0], [NAN, NAN, 0, 1, NAN, NAN])
    check(out[1], [NAN, NAN, 1, 0.5, 0, NAN])


@pytest.mark.parametrize("sf, want", [
    (1, [1000, 1200, 1400, 1600, 1800, 2000]),      # :8003
    (0, [1000] * 6),                                # :8014
    (0.5, [1000, 1100, 1250, 1425, 1612.5, 1806.25]),  # :8025
])
def test_smooth_exponential(sf, want):
    check(smooth_exponential_ref(np.array([T]), sf)[0], want)


def test_rules_the_gpu_tests_lean_on():
    # stdvar: the one-point fast path counts NaNs; no value at all is NaN
    assert stdvar([NAN]) == 0.0 and math.isnan(stdvar([NAN, NAN]))
    # mean() is a plain sum over n, not Welford's running mean: they differ in the last bits
    vals = [0.346, 0.822, 0.33, -1.303, 0.905]
    w = 0.0
    for i, v in enumerate(vals):
        w += (v - w) / (i + 1)
    assert mean(vals) != w
    assert math.isnan(mean([NAN]))
    # normalize drops a row without a value and a row with an infinite range, keeps a one-value row (0/0)
    assert not range_row("range_normalize", np.array([NAN, NAN]))[1]
    assert not range_row("range_normalize", np.array([1.0, INF]))[1]
    out, kept = range_row("range_normalize", np.array([NAN, 3.0]))
    assert kept and np.isnan(out).all()
    # quantile: a NaN result at the last value makes setLastValues fall back to the value before it
    out, _ = range_row("range_quantile", np.array([1.0, 2.0, 3.0]), NAN)
    check(out, [2, 2, 2])
    out, _ = range_row("range_quantile", np.array([NAN, 5.0, NAN]), NAN)
    assert np.isnan(out).all()
    check(range_row("range_quantile", np.array([1.0, 2.0, 3.0]), -1)[0], [-INF] * 3)
    # trim_spikes halves phi: phi >= 2 trims every value; NaN phi trims nothing
    assert np.isnan(range_row("range_trim_spikes", np.array([1.0, 2.0, 3.0]), 2.5)[0]).all()
    check(range_row("range_trim_spikes", np.array([1.0, 2.0, 3.0]), NAN)[0], [1, 2, 3])
    # linear regression: a NaN makes the row non-constant; a one-point row is constant
    out, _ = range_row("range_linear_regression", np.array([5.0, NAN, 5.0]), timestamps=[0, 1000, 2000])
    check(out, [5, 5, 5])
    check(range_row("range_linear_regression", np.array([NAN]), timestamps=[7])[0], [NAN])
    # smooth_exponential: leading Infs are cut unless nothing but Infs follows; sf by absolute index, NaN sf = 1
    check(smooth_exponential_ref(np.array([[NAN, INF, -INF]]), 0.5)[0], [NAN, INF, INF])
    check(smooth_exponential_ref(np.array([[NAN, INF, 2.0, 4.0, INF]]), [0, 0, 0, NAN, 0])[0], [NAN, INF, 2, 4, 4])


def test_range_func_ids_follow_the_header():
    from victoriametrics_b200 import promql
    from test_enum_tables import HDR, _enum
    pub = _enum(HDR, "vmb_range_func")
    assert {"range_" + n[len("VMB_RS_"):].lower(): v for n, v in pub} == promql.RANGE_FUNCS
