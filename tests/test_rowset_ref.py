"""tests/rowset_ref.py against the reference's own app/vmselect/promql/exec_test.go vectors (sort, sort_desc, two_timeseries,
the `or` cases, drop_empty_series, limit_offset, union), with the expected values as written there, and direct cases of the sort
comparator.  CPU only."""
import numpy as np

from rowset_ref import (NAN, drop_empty_series_ref, is_stable_sort, limit_offset_ref, nonempty, set_or_ref, sort_less, sort_rows_ref,
                        union_ref)

T = np.arange(1000, 2001, 200, dtype=np.float64)  # time() at the exec_test.go timestamps
INF = float("inf")


def rows(out, L, R):
    return [(L if s == "l" else R)[i].tolist() for s, i in out]


def same(got, want):
    assert len(got) == len(want), (got, want)
    for g, w in zip(got, want):
        assert np.array_equal(np.array(g), np.array(w), equal_nan=True), (got, want)


def or_(left, ll, right, rl, **kw):
    L, R, out = set_or_ref(np.array(left, dtype=np.float64), ll, np.array(right, dtype=np.float64), rl, **kw)
    return rows(out, L, R), [(ll if s == "l" else rl)[i] for s, i in out]


def sorted_rows(vals, desc=False):
    vals = np.asarray(vals, dtype=np.float64)
    order = sort_rows_ref(vals, desc)
    assert is_stable_sort(vals, order, desc)
    return [vals[i].tolist() for i in order]


# ------------------------------------------------------------------------------------------------ exec_test.go vectors
def test_sort_and_sort_desc():
    # :2691 sort(2 or label_set(1, "xx", "foo")), :2711 sort_desc(1 or label_set(2, "xx", "foo"))
    got, labels = or_([[2.0] * 6], [{}], [[1.0] * 6], [{"xx": "foo"}])
    assert labels == [{}, {"xx": "foo"}]
    same(sorted_rows(got), [[1] * 6, [2] * 6])
    got, _ = or_([[1.0] * 6], [{}], [[2.0] * 6], [{"xx": "foo"}])
    same(sorted_rows(got, desc=True), [[2] * 6, [1] * 6])
    # :2623 two_timeseries: sort_desc(time() or label_set(2, "xx", "foo"))
    got, labels = or_([T], [{}], [[2.0] * 6], [{"xx": "foo"}])
    same(sorted_rows(got, desc=True), [T, [2] * 6])


def test_series_or_series():  # :3075
    got, labels = or_([T, T + 1], [{"x": "foo"}, {"x": "bar"}], [T + 2, T + 3], [{"x": "foo"}, {"x": "baz"}])
    same(got, [T + 1, T, T + 3])
    assert labels == [{"x": "bar"}, {"x": "foo"}, {"x": "baz"}]


def test_scalar_or_scalar():  # :3120 time() > 1400 or 123
    got, _ = or_([np.where(T > 1400, T, NAN)], [{}], [[123.0] * 6], [{}])
    same(got, [[123, 123, 123, 1600, 1800, 2000]])


def test_nan_or_on_series():  # :9570 the left side is empty: it does not clear the right side
    got, labels = or_([[NAN] * 6], [{"a": "a", "b": "b1"}], [[2.0] * 6], [{"a": "a", "b": "b2"}], on=("a",))
    same(got, [[2] * 6])
    assert labels == [{"a": "a", "b": "b2"}]


def test_series_with_nans_or_scalar():  # :9590
    got, _ = or_([np.where(T >= 1600, T, NAN)], [{"a": "a", "b": "b1"}], [[1.0] * 6], [{}])
    same(got, [[NAN, NAN, NAN, 1600, 1800, 2000], [1] * 6])


def test_series_or_on_scalar():  # :9614 ... or on() vector(0)
    got, _ = or_([np.where(T > 1200, T, NAN)], [{"a": "a", "b": "b1"}], [[0.0] * 6], [{}], on=())
    same(got, [[NAN, NAN, 1400, 1600, 1800, 2000], [0, 0, NAN, NAN, NAN, NAN]])


def test_series_or_on_series():  # :9639
    got, labels = or_([np.where(T <= 1200, T, NAN)], [{"a": "a", "b": "b1"}], [np.where(T > 1200, T, NAN)],
                      [{"a": "a", "b": "b2"}], on=("a",))
    same(got, [[1000, 1200, NAN, NAN, NAN, NAN], [NAN, NAN, 1400, 1600, 1800, 2000]])
    assert labels == [{"a": "a", "b": "b1"}, {"a": "a", "b": "b2"}]


def test_drop_empty_series():  # :2073 / :2090
    vals = np.array([np.where(T > 2000, T, NAN), np.where(T + 500 > 2000, T + 500, NAN)])  # foo, bar
    kept = drop_empty_series_ref(vals)
    assert kept == [1]
    got = np.where(np.isnan(vals[kept]), 123.0, vals[kept])  # default 123
    same(sorted_rows(got), [[123, 123, 123, 2100, 2300, 2500]])
    got = np.where(np.isnan(vals), 123.0, vals)
    same(sorted_rows(got), [[123] * 6, [123, 123, 123, 2100, 2300, 2500]])


def test_limit_offset():  # :2547-2600
    by_label = np.array([T * 2, T * 3, T * 1])  # sort_by_label(..., "foo"): a, x, y
    assert [by_label[i].tolist() for i in limit_offset_ref(1, 1, by_label)] == [(T * 3).tolist()]
    assert limit_offset_ref(1, 10, by_label) == []
    desc = np.array([T * 3, T * 2, T * 1])  # sort_by_label_desc(... < 3000, "foo"): 3, 2, 1; foo=3 holds no value below 3000
    desc = np.where(desc < 3000, desc, NAN)
    assert [desc[i].tolist() for i in limit_offset_ref(1, 1, desc)] == [(T * 1).tolist()]


def test_union():  # :3206 sort_desc(union(x{foo="bar"} > 1400, y{foo="baz"} < 1700) default 123)
    x, y = np.where(T > 1400, T, NAN), np.where(T < 1700, T, NAN)
    out = union_ref([[{"__name__": "x", "foo": "bar"}], [{"__name__": "y", "foo": "baz"}]])
    assert out == [(0, 0), (1, 0)]
    vals = np.where(np.isnan([x, y]), 123.0, [x, y])
    same(sorted_rows(vals, desc=True), [[123, 123, 123, 1600, 1800, 2000], [1000, 1200, 1400, 1600, 123, 123]])
    assert union_ref([[{}], [{}]]) == [(0, 0), (1, 0)]  # all scalars: every one of them
    assert union_ref([[{"a": "1"}, {"a": "2"}], [{"a": "2"}, {"a": "3"}]]) == [(0, 0), (0, 1), (1, 1)]


# ------------------------------------------------------------------------------------------------ the comparator
def test_nan_first_in_both_directions():
    a, b = [NAN, 5.0], [1.0, 5.0]
    assert sort_less([NAN], [1.0], False) and sort_less([NAN], [1.0], True)
    assert not sort_less([1.0], [NAN], False) and not sort_less([1.0], [NAN], True)
    assert sort_less(a, b, False) and sort_less(a, b, True)  # equal at the last point, decided by the NaN at point 0
    vals = np.array([[1.0], [NAN], [-INF], [INF], [NAN]])
    assert sort_rows_ref(vals) == [1, 4, 2, 0, 3]
    assert sort_rows_ref(vals, desc=True) == [1, 4, 3, 0, 2]


def test_signed_zeros_tie_and_stability():
    vals = np.array([[1.0, 0.0], [2.0, -0.0], [0.0, 0.0], [1.0, -0.0]])
    assert not sort_less([0.0], [-0.0], False) and not sort_less([-0.0], [0.0], True)
    assert sort_rows_ref(vals) == [2, 0, 3, 1]  # rows 0 and 3 are equal: ascending row order
    assert sort_rows_ref(vals, desc=True) == [1, 0, 3, 2]
    eq = np.tile([[3.0, NAN, 1.0]], (20, 1))  # more than 12 equal rows
    assert sort_rows_ref(eq) == list(range(20)) and sort_rows_ref(eq, desc=True) == list(range(20))


def test_is_stable_sort_agrees_with_the_comparator():
    rng = np.random.default_rng(5)
    for S, P in ((0, 3), (1, 0), (13, 0), (13, 1), (40, 4), (200, 6)):
        vals = rng.integers(0, 3, (S, P)).astype(np.float64)
        vals[rng.random((S, P)) < 0.2] = NAN
        vals[rng.random((S, P)) < 0.1] = -0.0
        for desc in (False, True):
            order = sort_rows_ref(vals, desc)
            assert is_stable_sort(vals, order, desc)
            if S > 2:
                swapped = list(order)
                swapped[0], swapped[-1] = swapped[-1], swapped[0]
                assert not is_stable_sort(vals, swapped, desc) or sort_rows_ref(vals[swapped], desc) == list(range(S))


def test_nonempty():
    assert nonempty(np.array([[NAN, NAN], [NAN, 0.0]])).tolist() == [False, True]
    assert nonempty(np.zeros((2, 0))).tolist() == [False, False]
