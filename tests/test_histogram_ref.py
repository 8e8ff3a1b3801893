"""tests/histogram_ref.py (the reference of vmb_histogram) on the histogram query vectors of the reference's own
app/vmselect/promql/exec_test.go:4009-4835: every series on the time() grid 1000 ... 2000 s, step 200 s, the expected values as
written there, with the query's outer sort() / round() restated here; plus the rules the tests on the GPU lean on.

The histogram_avg / stddev / stdvar vectors of exec_test.go:4105-4170 read histogram_over_time(rand(0)[200s:5s]): Go's seeded
generator and `vmrange` buckets, neither of which this restatement has.  Those three are pinned on hand-worked buckets instead."""
import numpy as np
import pytest

from histogram_ref import SKIP, fraction_cells, go_insertion_sort, histogram_ref, last_non_inf, merge_same_le, quantile_cells

NAN, INF = float("nan"), float("inf")
T = np.arange(1000, 2001, 200, dtype=np.float64)  # time()


def parse_le(s):
    """strconv.ParseFloat of the `le` label; None for a value that does not parse"""
    try:
        return float(s)
    except ValueError:
        return None


def series(*items):
    """label_set(v, k1, v1, ...) `or` ... -> [(values, labels)]"""
    out = []
    for v, *kv in items:
        vals = T.copy() if isinstance(v, str) and v == "time" else np.full(6, float(v))
        out.append((vals, dict(zip(kv[::2], kv[1::2]))))
    return out


def inputs(ss):
    """groupLeTimeseries over the series' labels -> (bucket matrix, group ids, les, ngroups) as vmb_histogram takes them"""
    keys, gids, les = {}, [], []
    for _, labels in ss:
        le = parse_le(labels["le"]) if "le" in labels else None
        if le is None:
            gids.append(SKIP)
            les.append(0.0)
            continue
        key = tuple(sorted((k, v) for k, v in labels.items() if k != "le"))
        gids.append(keys.setdefault(key, len(keys)))
        les.append(le)
    return np.array([v for v, _ in ss]), np.array(gids, dtype=np.uint32), np.array(les), len(keys)


def run(name, ss, *args, bounds=False):
    """histogram_ref on the series, then removeEmptySeries -> the result rows (quantiles: phi-major)"""
    out, lo, up, nonempty = histogram_ref(name, *inputs(ss), *args, bounds=bounds)
    rows = list(np.asarray(out).reshape(-1, 6)) + ([*lo, *up] if bounds else [])
    assert len(rows) == len(nonempty)
    return [r for r, ne in zip(rows, nonempty) if ne]


def sort_rows(rows):
    """sort() of constant series: by the last value"""
    return sorted(rows, key=lambda r: r[-1])


def check(rows, want, nearest=None):
    """the result rows equal `want` (one entry per row: a number or 6 values); with `nearest`, want is round(row, nearest)"""
    assert len(rows) == len(want), (rows, want)
    for got, w in zip(rows, want):
        w = np.broadcast_to(np.asarray(w, dtype=np.float64), (6,))
        if nearest is None:
            assert np.array_equal(got, w), (got, w)
        else:
            assert np.all(np.abs(got - w) <= nearest / 2), (got, w)


NOLE = ("foo", "bar")
TWO = series((100, "le", "200"), (0, "le", "55"))
THREE = series((100, "le", "100"), (40, "le", "50"), (0, "le", "10"))
VALID = series((90, "foo", "bar", "le", "10"), (100, "foo", "bar", "le", "30"), (300, "foo", "bar", "le", "+Inf"),
               (200, "tag", "xx", "le", "10"), (300, "tag", "xx", "le", "30"))
NORMAL = series((0, "foo", "bar", "le", "10"), (100, "foo", "bar", "le", "30"), (300, "foo", "bar", "le", "+Inf"))


EXEC_VECTORS = [
    # :4009-4068 no group, or a group with no value: no result
    ("histogram_quantile", series(("time",)), (0.6,), []),
    ("histogram_share", series(("time",)), (123,), []),
    ("histogram_fraction", series(("time",)), (123, 456), []),
    ("histogram_quantile", series((100, *NOLE)), (0.6,), []),
    ("histogram_share", series((100, *NOLE)), (123,), []),
    ("histogram_fraction", series((100, *NOLE)), (123, 456), []),
    ("histogram_quantile", series((100, "le", "foobar")), (0.6,), []),
    ("histogram_share", series((100, "le", "foobar")), (50,), []),
    ("histogram_fraction", series((100, "le", "foobar")), (50, 60), []),
    ("histogram_quantile", series((100, "le", "+Inf")), (0.6,), []),
    ("histogram_quantile", series((100, "le", "+Inf"), (0, "le", "42")), (0.6,), [42]),       # :4069
    ("histogram_quantile", series((100, "le", "200")), (0.6,), [120]),                      # :4083
    ("histogram_share", series((100, "le", "200")), (80,), [0.4]),                          # :4171
    ("histogram_share", series((100, "le", "200")), (200,), [1]),
    ("histogram_share", series((100, "le", "200")), (300,), [1]),
    ("histogram_fraction", series((100, "le", "200")), (0, 100), [0.5]),                    # :4204
    ("histogram_fraction", series((100, "le", "200")), (200, 300), [0]),
    ("histogram_quantile", TWO, (1,), [200]),                                               # :4284
    ("histogram_share", TWO, (200,), [1]),
    ("histogram_quantile", TWO, (0,), [55]),
    ("histogram_share", TWO, (0,), [0]),
    ("histogram_share", TWO, (55,), [0]),
    ("histogram_fraction", THREE, (0, 100), [1]),                                           # :4354
    ("histogram_fraction", THREE, (0, 10), [0]),
    ("histogram_share", TWO, (105,), [0.3448275862068966]),                                 # :4384
    ("histogram_share", TWO, (55,), [0]),
    ("histogram_fraction", TWO, (55, 105), [0.3448275862068966]),
    ("histogram_quantile", series((100, "le", "200")), (0,), [0]),                          # :4426
    ("histogram_quantile", series((100, "le", "200")), (T / 2 / 1e3,), [[100, 120, 140, 160, 180, 200]]),  # :4437
    ("histogram_share", series((100, "le", "200")), (T / 8,), [[0.625, 0.75, 0.875, 1, 1, 1]]),
    ("histogram_fraction", series((100, "le", "200")), (25, T / 8), [[0.5, 0.625, 0.75, 0.875, 0.875, 0.875]]),
    ("histogram_quantile", NORMAL, (0.2,), [22]),                                           # :4619
    ("histogram_quantiles", NORMAL, (0.2, 0.3), [22, 28]),                                  # :4638
    ("histogram_share", NORMAL, (35,), [0.3333333333333333]),                               # :4678
    ("histogram_fraction", NORMAL, (22, 35), [0.1333333333333333]),
    ("histogram_quantile", series((90, *NOLE, "le", "10"), (-100, *NOLE, "le", "30"), (300, *NOLE, "le", "+Inf")), (0.6,), [30]),
    ("histogram_quantile", series((0, *NOLE, "le", "10"), (0, *NOLE, "le", "30"), (0, *NOLE, "le", "+Inf")), (0.6,), []),  # :4816
    ("histogram_quantile", series((NAN, *NOLE, "le", "10"), (NAN, *NOLE, "le", "30"), (NAN, *NOLE, "le", "+Inf")), (0.6,), []),
]


@pytest.mark.parametrize("name, ss, args, want", EXEC_VECTORS)
def test_exec_test_vectors(name, ss, args, want):
    check(run(name, ss, *args), want)


@pytest.mark.parametrize("name, args, want", [
    ("histogram_quantile", (0.6,), [9, 30]),             # :4491 sort(...)
    ("histogram_share", (25,), [0.325, 0.9166666666666666]),
    ("histogram_fraction", (0, 25), [0.325, 0.9166666666666666]),
])
def test_two_groups_sorted(name, args, want):
    check(sort_rows(run(name, VALID, *args)), want)


def test_bounds_label():
    """:4226, :4255, :4716, :4766: sort() of the value and its lower / upper series"""
    check(sort_rows(run("histogram_quantile", series((100, "le", "200")), 0.6, bounds=True)), [0, 120, 200])
    check(sort_rows(run("histogram_share", series((100, "le", "200")), 120, bounds=True)), [0, 0.6, 1])
    check(sort_rows(run("histogram_quantile", NORMAL, 0.2, bounds=True)), [10, 22, 30])
    check(sort_rows(run("histogram_share", NORMAL, 22, bounds=True)), [0, 0.2, 0.3333333333333333])


def test_rounded_vectors():
    """:4470 duplicate le ("5" and "5.0" merge), round(..., 0.1); :4600 a NaN bucket, round(..., 0.01)"""
    dup = series((90, *NOLE, "le", "5"), (100, *NOLE, "le", "5.0"), (200, *NOLE, "le", "6.0"), (300, *NOLE, "le", "+Inf"))
    check(run("histogram_quantile", dup, 0.6), [4.7], 0.1)
    nan = series((90, *NOLE, "le", "10"), (NAN, *NOLE, "le", "30"), (300, *NOLE, "le", "+Inf"))
    check(run("histogram_quantile", nan, 0.6), [30], 0.01)


def test_moments_on_hand_worked_buckets():
    """le 1: 2, le 2: 5, le 4: 6, +Inf: 6 in shuffled rows: weights 2, 3, 1 at midpoints 0.5, 1.5, 3 -> avg 17/12, stdvar
    65/24 - (17/12)^2 = 101/144"""
    ss = series((6, "le", "+Inf"), (5, "le", "2"), (2, "le", "1"), (6, "le", "4"))
    avg, sv = 17 / 12, 101 / 144
    for name, want in (("histogram_avg", avg), ("histogram_stdvar", sv), ("histogram_stddev", sv ** 0.5)):
        (got,) = run(name, ss)
        assert np.allclose(got, want, rtol=4e-16, atol=0), (name, got, want)
    # weights that add up to 0: NaN; one bucket of weight: stdvar 0
    assert run("histogram_avg", series((3, "le", "1"), (3, "le", "2"), (-3, "le", "3"), (-3, "le", "4"), (0, "le", "5"))) == []
    (got,) = run("histogram_stdvar", series((1, "le", "0.1"), (1, "le", "0.2")))
    assert (got == 0).all()


def test_rules_the_gpu_tests_lean_on():
    # the insertion sort is stable and a NaN blocks moves across it
    assert go_insertion_sort([3.0, 1.0, 2.0, 1.0]) == [1, 3, 2, 0]
    assert go_insertion_sort([3.0, NAN, 1.0, 2.0]) == [0, 1, 2, 3]
    assert go_insertion_sort([NAN, 5.0, 1.0]) == [0, 2, 1]
    assert go_insertion_sort([0.0, -0.0]) == [0, 1]
    # mergeSameLE: NaN never merges; -0.0 and +0.0 merge and keep the first le
    les, vals = merge_same_le([NAN, NAN, 1.0, 1.0, 1.0], [np.array([k]) for k in (1.0, 2.0, 3.0, 4.0, 5.0)])
    assert len(les) == 3 and [v[0] for v in vals] == [1.0, 2.0, 12.0]
    les, _ = merge_same_le([-0.0, 0.0, 1.0], [np.zeros(1)] * 3)
    assert les == [-0.0, 1.0] and np.signbit(les[0])
    assert np.isnan(last_non_inf([INF, -INF])) and last_non_inf([1.0, INF]) == 1.0
    # quantile: vLast == 0 comes before the phi checks; phi < 0 -> (-Inf, -Inf, first bucket); phi > 1 -> (+Inf, vLast, +Inf)
    les, b = [1.0, 2.0], [np.array([0.0, 2.0, 2.0]), np.array([0.0, 4.0, 4.0])]
    q, lo, up = quantile_cells(np.array([-1.0, -1.0, 2.0]), les, b)
    assert np.isnan([q[0], lo[0], up[0]]).all()
    assert (q[1], lo[1], up[1]) == (-INF, -INF, 2.0) and (q[2], lo[2], up[2]) == (INF, 4.0, INF)
    # fraction = share(upper) - share(lower), the share loop after its < 0 and +Inf checks
    assert fraction_cells(np.array([-1.0, 0.5, NAN]), np.array([INF, INF, 1.0]), les, b).tolist()[:2] == [1.0, 0.75]


def test_histogram_func_ids_follow_the_header():
    from victoriametrics_b200 import promql
    from test_enum_tables import HDR, _enum
    pub = {"histogram_" + n[len("VMB_HF_"):].lower(): v for n, v in _enum(HDR, "vmb_hist_func")}
    assert dict(pub, histogram_quantiles=pub["histogram_quantile"]) == promql.HISTOGRAM_FUNCS
