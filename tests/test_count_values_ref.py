"""CPU checks of tests/count_values_ref.py and promql.go_format_float.

The count_values_over_time case of exec_test.go:6066 reads rand(0), whose sequence is Go's math/rand: it cannot be reproduced
without Go, so it is not restated here; the GPU tests feed the same query shape, round(x, 0.4)[200s:5s], with a seeded x."""
import math
import struct

import numpy as np
import pytest

import count_values_ref as R
from victoriametrics_b200.promql import go_format_float

NAN = float("nan")
TS = np.arange(1000, 2001, 200, dtype=np.float64)  # exec_test.go: start 1000 s, end 2000 s, step 200 s


def _as_set(res, group_labels=None):
    out = set()
    for g, rows in res.items():
        for v, c in rows:
            out.add(((group_labels or {}).get(g, ()), go_format_float(v, "f"), tuple(np.where(np.isnan(c), -1, c).tolist())))
    return out


def _expect(*rows):
    return {(grp, lab, tuple(-1 if x != x else x for x in vals)) for grp, lab, vals in rows}


def test_count_values():  # exec_test.go:9078
    res = R.count_values([np.full(6, 10.0), TS / 100], [0, 0], 1)
    one = lambda i: [NAN] * i + [1] + [NAN] * (5 - i)
    assert _as_set(res) == _expect(((), "10", [2, 1, 1, 1, 1, 1]), ((), "12", one(1)), ((), "14", one(2)), ((), "16", one(3)),
                                   ((), "18", one(4)), ((), "20", one(5)))


def test_count_values_big_numbers():  # exec_test.go:9047
    res = R.count_values([np.full(6, 772424014.0), np.full(6, 772424230.0)], [0, 0], 1)
    assert _as_set(res) == _expect(((), "772424014", [1] * 6), ((), "772424230", [1] * 6))


def test_count_values_by_xxx():  # exec_test.go:9150: by (xxx) loses xxx, one group
    res = R.count_values([np.full(6, 10.0), np.floor(TS / 600)], [0, 0], 1)
    assert _as_set(res) == _expect(((), "1", [1, NAN, NAN, NAN, NAN, NAN]), ((), "2", [NAN, 1, 1, 1, NAN, NAN]),
                                   ((), "3", [NAN, NAN, NAN, NAN, 1, 1]), ((), "10", [1] * 6))


def test_count_values_without_baz():  # exec_test.go:9202
    res = R.count_values([np.floor(TS / 600)], [0], 1)
    foo = (("foo", "bar"),)
    assert _as_set(res, {0: foo}) == _expect((foo, "1", [1, NAN, NAN, NAN, NAN, NAN]), (foo, "2", [NAN, 1, 1, 1, NAN, NAN]),
                                             (foo, "3", [NAN, NAN, NAN, NAN, 1, 1]))


def test_count_values_zero_first_seen():
    res = R.count_values([[NAN, -0.0, 0.0], [0.0, 0.0, 1.0]], [0, 0], 1)
    (v0, c0), (v1, c1) = res[0]
    assert math.copysign(1, v0) < 0 and go_format_float(v0, "f") == "-0" and c0.tolist() == [1, 2, 1]


def test_count_values_over_time_windows():
    # 10 s samples, window 30 s at step 60 s: the rows between windows make no key
    ts = np.arange(0, 600_000, 10_000, dtype=np.int64)
    v = np.arange(ts.size, dtype=np.float64)
    m, scanned = R.count_values_over_time(v, ts, 60_000, 540_000, 60_000, 30_000)
    assert sorted(m, key=float) == [go_format_float(x, "g") for x in range(4, 55) if x % 6 in (4, 5, 0)]
    assert scanned == ts.size + 3 * 9


def _bits(x):
    return struct.pack("<d", x)


@pytest.mark.parametrize("v, f, g", [
    (1e-5, "0.00001", "1e-05"), (1.5e-5, "0.000015", "1.5e-05"), (1e-4, "0.0001", "0.0001"), (1e-7, "0.0000001", "1e-07"),
    (1e5, "100000", "100000"), (123456.0, "123456", "123456"), (1e6, "1000000", "1e+06"), (1234567.0, "1234567", "1.234567e+06"),
    (1e21, "1000000000000000000000", "1e+21"), (772424014.0, "772424014", "7.72424014e+08"), (0.1, "0.1", "0.1"),
    (-2.5, "-2.5", "-2.5"), (-1e-7, "-0.0000001", "-1e-07"), (10.0, "10", "10"), (0.4, "0.4", "0.4"), (0.8, "0.8", "0.8"),
    (1.2, "1.2", "1.2"), (5e-324, "0." + "0" * 323 + "5", "5e-324"), (2.2250738585072014e-308, None, "2.2250738585072014e-308"),
    (1.7976931348623157e308, "17976931348623157" + "0" * 292, "1.7976931348623157e+308"), (0.0, "0", "0"), (-0.0, "-0", "-0"),
    (NAN, "NaN", "NaN"), (float("inf"), "+Inf", "+Inf"), (float("-inf"), "-Inf", "-Inf"), (100.0, "100", "100"),
    (1e100, "1" + "0" * 100, "1e+100"), (123.456, "123.456", "123.456"), (0.000123, "0.000123", "0.000123"),
])
def test_go_format_float(v, f, g):
    if f is not None:
        assert go_format_float(v, "f") == f
    assert go_format_float(v, "g") == g
    if v == v and not math.isinf(v):  # both parse back to the same bits
        assert _bits(float(go_format_float(v, "g"))) == _bits(v)
