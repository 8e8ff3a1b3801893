"""tests/datetime_ref.py (the reference of vmb_transform's date-time and bitmap functions) on the query vectors of the reference's
own app/vmselect/promql/exec_test.go: time() at 1000 ... 2000 s, step 200 s, with the expected values as written there; then the
restatement of Go's calendar against Python's datetime / calendar over years 1..9999, Go's uint32 leap test on negative years,
and a hand-derived table of Go's amd64 float -> uint64 conversion."""
import calendar
import datetime
import math

import numpy as np
import pytest

import datetime_ref as R

NAN, INF = float("nan"), float("inf")
EPOCH = datetime.datetime(1970, 1, 1)


def same(got, want):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    return np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(got[~np.isnan(got)], want[~np.isnan(want)])


@pytest.mark.parametrize("name, row, want", R.EXEC_TEST_DATETIME)
def test_exec_test_datetime_vectors(name, row, want):
    assert same([R.time_field(name, v) for v in row], want)
    assert same(R.np_time_field(name, row), want)


@pytest.mark.parametrize("name, v, w, want", R.EXEC_TEST_BITMAP)
def test_exec_test_bitmap_vectors(name, v, w, want):
    v = np.broadcast_to(np.asarray(v, dtype=np.float64), (6,))
    w = np.broadcast_to(np.asarray(w, dtype=np.float64), (6,))
    assert same([R.bitmap(name, a, b) for a, b in zip(v, w)], want)
    assert same(R.np_bitmap(name, v[None, :], w)[0], want)


def _python_fields(s):
    """the fields by Python's datetime / calendar (years 1..9999)"""
    t = EPOCH + datetime.timedelta(seconds=int(s))
    return {"hour": t.hour, "minute": t.minute, "day_of_month": t.day, "day_of_week": t.isoweekday() % 7,
            "day_of_year": t.timetuple().tm_yday, "days_in_month": calendar.monthrange(t.year, t.month)[1], "month": t.month,
            "year": t.year}


def _unix(y, m, d, sec=0):
    return int((datetime.datetime(y, m, d) - EPOCH).total_seconds()) + sec


def _check_against_python(secs):
    secs = np.asarray(secs, dtype=np.int64)
    want = [_python_fields(s) for s in secs]
    for name in R.DATETIME_FUNCS:
        got = R.np_time_field(name, secs.astype(np.float64))
        assert np.array_equal(got, [w[name] for w in want]), name
    for s, w in zip(secs[::97], want[::97]):
        assert R.go_time_fields(int(s)) == w, s


def test_every_month_boundary_of_years_1_to_9999():
    first = _unix(1, 1, 1)
    secs = [_unix(y, m, 1) + k for y in range(1, 10000) for m in range(1, 13) for k in (-1, 0, 1)]
    _check_against_python([s for s in secs if s >= first])


def test_century_leap_days():
    secs = [_unix(y, m, d) + k for y in (1600, 1700, 1900, 2000, 2100) for m, d in ((2, 28), (3, 1)) for k in (-1, 0, 1, 86399)]
    _check_against_python(secs)
    assert R.time_field("days_in_month", float(_unix(1900, 2, 10))) == 28.0
    assert R.time_field("days_in_month", float(_unix(2000, 2, 10))) == 29.0
    assert R.time_field("day_of_year", float(_unix(2000, 12, 31))) == 366.0
    assert R.time_field("day_of_year", float(_unix(2100, 12, 31))) == 365.0


def test_seeded_seconds_of_years_1_to_9999():
    rng = np.random.default_rng(20261018)
    _check_against_python(rng.integers(_unix(1, 1, 1), _unix(9999, 12, 31, 86399), 100_000))


def _is_leap_year_go(y):  # transform.go:2874 isLeapYear(uint32(t.Year())), literally
    y = y % (1 << 32)
    if y % 4 != 0:
        return False
    if y % 100 != 0:
        return True
    return y % 400 == 0


@pytest.mark.parametrize("year, want", [(-1, 28), (-4, 29), (-100, 29), (-400, 29)])
def test_negative_year_leap_quirk(year, want):
    k = 1 if year > -400 else 2  # the same day 400 * k years later is in datetime's range; 400 years are 146097 days
    s = _unix(year + 400 * k, 2, 10) - k * 146097 * 86400
    f = R.go_time_fields(s)
    assert (f["year"], f["month"], f["day_of_month"]) == (year, 2, 10)
    assert f["days_in_month"] == want == (29 if _is_leap_year_go(year) else 28)
    # the calendar itself is proleptic Gregorian: years -1 and -100 have no February 29
    g = R.go_time_fields(s + 19 * 86400)
    assert (g["month"], g["day_of_month"]) == ((3, 1) if year in (-1, -100) else (2, 29))


def test_truncation_toward_zero_and_pre_1970():
    assert R.time_field("hour", -0.5) == 0.0 and R.time_field("year", -0.5) == 1970.0
    assert R.time_field("hour", -1.0) == 23.0 and R.time_field("year", -1.0) == 1969.0
    assert R.time_field("day_of_week", -1.0) == 3.0  # 1969-12-31 was a Wednesday
    assert R.time_field("minute", -59.9) == 59.0


def test_int64_conversion_table():
    assert R.go_int64(2.0 ** 63) == R.go_int64(INF) == R.go_int64(-INF) == R.go_int64(1e300) == -2 ** 63
    assert R.go_int64(-2.0 ** 63) == -2 ** 63 and R.go_int64(np.nextafter(2.0 ** 63, 0)) == 2 ** 63 - 1024
    assert R.go_int64(-0.9) == 0 and R.go_int64(-1.9) == -1 and R.go_int64(5e-324) == 0


U63, M64 = 1 << 63, (1 << 64) - 1


@pytest.mark.parametrize("v, want", [
    (-1.5, M64), (-1.0, M64), (-0.5, 0), (-0.0, 0), (0.5, 0), (1.5, 1), (-2.0, M64 - 1),
    (2.0 ** 53, 1 << 53), (2.0 ** 53 + 2, (1 << 53) + 2), (float(2 ** 63 - 1024), 2 ** 63 - 1024),
    (2.0 ** 63, U63), (float(2 ** 64 - 2048), 2 ** 64 - 2048), (2.0 ** 64, U63), (1e300, U63), (INF, U63),
    (-INF, U63), (-2.0 ** 63, U63), (-2.0 ** 63 - 2048, U63), (-2.0 ** 62, 3 << 62),
])
def test_uint64_conversion_table(v, want):
    assert R.go_uint64(v) == want
    assert int(R.np_uint64(np.array([v]))[0]) == want


def test_bitmap_rounds_half_to_even():
    assert R.bitmap("bitmap_or", 2.0 ** 53, 1.0) == 2.0 ** 53               # 2^53 + 1: a tie, to the even 2^53
    assert R.bitmap("bitmap_or", 2.0 ** 53 + 2, 1.0) == 2.0 ** 53 + 4       # 2^53 + 3: a tie, to the even 2^53 + 4
    assert R.bitmap("bitmap_xor", 2.0 ** 63, 1024.0) == 2.0 ** 63           # 2^63 + 1024: a tie, to the even 2^63
    assert R.bitmap("bitmap_xor", 2.0 ** 63, 3072.0) == 2.0 ** 63 + 4096    # 2^63 + 3072: a tie, to the even 2^63 + 4096
    assert R.bitmap("bitmap_and", -1.0, 12345.0) == 12345.0
    v = np.array([[2.0 ** 53, 2.0 ** 53 + 2, 2.0 ** 63, 2.0 ** 63]])
    w = np.array([1.0, 1.0, 1024.0, 3072.0])
    assert np.array_equal(R.np_bitmap("bitmap_xor", v, w), [[2.0 ** 53, 2.0 ** 53 + 4, 2.0 ** 63, 2.0 ** 63 + 4096]])
    assert math.isnan(R.bitmap("bitmap_and", 1.0, NAN))
    assert np.isnan(R.np_bitmap("bitmap_or", np.array([[1.0]]), NAN)).all()


def test_numpy_form_matches_the_scalar_form_everywhere():
    rng = np.random.default_rng(7)
    v = np.concatenate([
        rng.uniform(-2.0 ** 63, 2.0 ** 63, 3000),                                   # all of int64, the wrap region's edge included
        -float(R.UNIX_TO_ABSOLUTE) + rng.uniform(-2e10, 2e10, 2000),                # around the wrap
        [-2.0 ** 63, np.nextafter(-2.0 ** 63, 0), np.nextafter(2.0 ** 63, 0), INF, -INF, 1e300, -1e300, 5e-324, -0.0, NAN],
        rng.uniform(-1e12, 1e12, 2000).round(3),
    ])
    for name in R.DATETIME_FUNCS:
        assert same(R.np_time_field(name, v), [R.time_field(name, x) for x in v]), name
    w = rng.permutation(v)
    for name in R.BITMAP_FUNCS:
        assert same(R.np_bitmap(name, v[None, :], w)[0], [R.bitmap(name, a, b) for a, b in zip(v, w)]), name


def test_wrap_region():
    # below -unixToAbsolute the sum wraps to the far end of uint64: -2^63 (every +-Inf and |v| >= 2^63) lands in year ~2.9e11
    f = R.go_time_fields(-2 ** 63)
    assert f["year"] > 2.9e11 and f == R.go_time_fields(R.go_int64(INF))
    assert R.go_time_fields(-R.UNIX_TO_ABSOLUTE)["year"] == -R.ABSOLUTE_YEARS  # the absolute zero instant, March 1
    assert (R.go_time_fields(-R.UNIX_TO_ABSOLUTE)["month"], R.go_time_fields(-R.UNIX_TO_ABSOLUTE)["day_of_month"]) == (3, 1)
    assert R.go_time_fields(-R.UNIX_TO_ABSOLUTE - 1)["year"] > 2.9e11
