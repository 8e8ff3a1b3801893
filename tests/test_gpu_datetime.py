"""vmb_transform's date-time functions (hour ... year) and bitmap functions (bitmap_and / or / xor) on device matrices, bit for
bit and NaN payload for NaN payload against tests/datetime_ref.py: the exec_test.go vectors, the edges of Go's conversions and
calendar (years 0 and below, beyond 9999, the wrap below Go's absolute zero year, +-Inf), and seeded matrices."""
import ctypes as C

import numpy as np
import pytest

import datetime_ref as R
from conftest import SEED0

pytestmark = pytest.mark.gpu
NAN, INF = float("nan"), float("inf")
BELOW_2_63 = float(np.nextafter(2.0 ** 63, 0))


def _run(name, m, w=None, ctx=None):
    import torch
    import victoriametrics_b200 as vm
    d = torch.from_numpy(np.ascontiguousarray(m, dtype=np.float64)).cuda()
    args = () if w is None else (w,)
    vm.promql.transform(name, d.data_ptr(), m.shape[0], m.shape[1], *args, ctx=ctx)
    torch.cuda.synchronize()
    return d.cpu().numpy()


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, dtype=np.float64).view(np.uint64), np.asarray(b, dtype=np.float64).view(np.uint64))


def _check(name, m, w=None):
    got, want = _run(name, m, w), R.np_ref(name, m, w)
    if not _bits_equal(got, want):
        bad = np.argwhere(got.view(np.uint64) != want.view(np.uint64))[:5]
        raise AssertionError((name, [(m[tuple(i)], got[tuple(i)], want[tuple(i)]) for i in bad]))


@pytest.mark.parametrize("name, row, want", R.EXEC_TEST_DATETIME)
def test_exec_test_datetime_vectors(name, row, want):
    got = _run(name, np.asarray(row, dtype=np.float64)[None, :])[0]
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(got[~np.isnan(got)], np.asarray(want)[~np.isnan(want)])
    _check(name, np.asarray(row, dtype=np.float64)[None, :])


@pytest.mark.parametrize("name, v, w, want", R.EXEC_TEST_BITMAP)
def test_exec_test_bitmap_vectors(name, v, w, want):
    m = np.broadcast_to(np.asarray(v, dtype=np.float64), (1, 6)).copy()
    got = _run(name, m, w)[0]
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(got[~np.isnan(got)], np.asarray(want)[~np.isnan(want)])
    _check(name, m, w)


def test_hour_compared_and_raised_on_the_device():
    """(hour(time()*1e4) == 4)^1  exec_test.go:9559: the transform, then two binary operators on a one-row scalar each"""
    import torch
    import victoriametrics_b200 as vm
    d = torch.from_numpy(R.T[None, :] * 1e4).cuda()
    four, one = torch.full((1, 6), 4.0, dtype=torch.float64).cuda(), torch.ones((1, 6), dtype=torch.float64).cuda()
    vm.promql.transform("hour", d.data_ptr(), 1, 6)
    vm.promql.binary_op("==", d.data_ptr(), four.data_ptr(), 1, 6, d.data_ptr())
    vm.promql.binary_op("^", d.data_ptr(), one.data_ptr(), 1, 6, d.data_ptr())
    torch.cuda.synchronize()
    got = d.cpu().numpy()[0]
    assert np.array_equal(np.isnan(got), [1, 1, 1, 0, 1, 1]) and got[3] == 4.0


def _edge_values():
    year0 = -62167219200  # 0000-01-01T00:00:00Z
    wrap = -float(R.UNIX_TO_ABSOLUTE)  # a double: 2^63 - 7922867 * 1024
    v = [0.0, -0.0, -0.5, -0.9999, -1.0, -1.5, -59.9, 0.5, 5e-324, -5e-324, 2.2e-308, -2.2e-308, 1e-300, -1e-300,
         -1.0, -86399.0, -86400.0, -86401.0, -1e9, -2208988800.0, -12219292800.0,            # pre-1970, 1900, the Gregorian reform
         year0 + 0.0, year0 - 1.0, year0 + 1.0, year0 - 86400 * 366.0, -62198755200.0, -65335910400.0,  # years 0, -1, -100
         -1e12, -1e15, -1e17, -9e18, -9.2e18,                                                # years far below 0
         253402300800.0, 253402300799.0, 1e12, 1e13, 1e15, 1e17, 9e18, 9.2e18,                 # years 10000 and beyond
         2.0 ** 53, -2.0 ** 53, 2.0 ** 53 + 2, 2.0 ** 62, -2.0 ** 62, BELOW_2_63, -BELOW_2_63, -2.0 ** 63, 2.0 ** 63,
         float(np.nextafter(-2.0 ** 63, 0)), -2.0 ** 63 + 4096, -2.0 ** 63 + 2.0 ** 33,         # the wrap region
         wrap, float(np.nextafter(wrap, 0)), float(np.nextafter(wrap, -INF)), wrap - 86400.0, wrap + 86400.0,
         INF, -INF, 1e300, -1e300, NAN, -NAN, 1700000000.123, 1700006399.999, 951782400.0, 951868799.0, 4107542400.0]
    return np.array(v, dtype=np.float64)


@pytest.mark.parametrize("name", R.DATETIME_FUNCS)
def test_datetime_edges(name):
    v = _edge_values()
    _check(name, v[None, :])
    _check(name, np.tile(v, (3, 1)))  # several rows: the point index wraps inside the grid-stride loop


def test_datetime_edges_follow_the_scalar_restatement():
    v = _edge_values()
    for name in R.DATETIME_FUNCS:
        got = _run(name, v[None, :])[0]
        want = np.array([R.time_field(name, x) for x in v])
        assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(got[~np.isnan(got)], want[~np.isnan(want)]), name
    assert _run("hour", np.array([[-0.5]]))[0, 0] == 0.0
    assert _run("year", np.array([[-2.0 ** 63, INF, -INF]]))[0].tolist() == [R.time_field("year", -2.0 ** 63)] * 3


@pytest.mark.parametrize("name", R.DATETIME_FUNCS)
def test_day_boundaries(name):
    """day boundaries -1 / 0 / +1 s and noon, over +-2^31 days (+-5.9 million years) around 1970"""
    rng = np.random.default_rng(SEED0 + 11)
    n = rng.integers(-(1 << 31), 1 << 31, 4000)
    s = (n * 86400)[:, None] + np.array([-1, 0, 1, 43200])[None, :]
    _check(name, s.reshape(40, -1).astype(np.float64))


def _bitmap_inputs(rng, rows, points):
    pool = np.array([-1.5, -1.0, -0.5, -0.0, 0.0, 0.5, 1.5, 3.999, -2.0 ** 62, -2.0 ** 63, 2.0 ** 53, 2.0 ** 53 + 2, 2.0 ** 60 + 2048,
                     BELOW_2_63, 2.0 ** 63, 2.0 ** 63 + 2048, 1.5 * 2.0 ** 63, float(2 ** 64 - 2048), 2.0 ** 64, 1e300, INF, -INF,
                     NAN, 0xB3, 0x11, 65535.0, 4294967295.0])
    m = np.where(rng.random((rows, points)) < 0.5, rng.choice(pool, (rows, points)),
                 np.trunc(rng.uniform(-2.0 ** 64, 2.0 ** 64, (rows, points)) / rng.choice([1.0, 1e3, 1e9], (rows, points))))
    w = np.where(rng.random(points) < 0.5, rng.choice(pool, points), rng.uniform(-1e19, 2e19, points))
    return m, w


@pytest.mark.parametrize("name", R.BITMAP_FUNCS)
def test_bitmap_edges_and_a_per_point_argument(name):
    rng = np.random.default_rng(SEED0 + 3)
    m, w = _bitmap_inputs(rng, 37, 301)
    assert np.isnan(w).any()
    _check(name, m, w)
    _check(name, m, 0x11)
    _check(name, m, -1.0)


def test_bitmap_rounds_half_to_even():
    m = np.array([[2.0 ** 53, 2.0 ** 53 + 2, 2.0 ** 63, 2.0 ** 63, 2.0 ** 62, float(2 ** 64 - 4096)]])
    w = np.array([1.0, 1.0, 1024.0, 3072.0, 512.0, 1024.0])
    got = _run("bitmap_xor", m, w)[0]
    assert got.tolist() == [2.0 ** 53, 2.0 ** 53 + 4, 2.0 ** 63, 2.0 ** 63 + 4096, 2.0 ** 62, float(2 ** 64 - 4096)]
    _check("bitmap_xor", m, w)
    _check("bitmap_or", m, w)


def _realistic(rng, rows, points):
    m = np.round(rng.uniform(1.5e9, 2e9, (rows, points)), 3)
    m[rng.random(m.shape) < 0.05] = NAN
    return m


def _full_range(rng, rows, points):
    return rng.integers(-(1 << 63), (1 << 63) - 1, (rows, points), dtype=np.int64, endpoint=True).astype(np.float64)


@pytest.mark.parametrize("name", R.DATETIME_FUNCS + R.BITMAP_FUNCS)
def test_seeded_matrices(name):
    rng = np.random.default_rng(SEED0 + 5)
    for m in (_realistic(rng, 257, 1000), _full_range(rng, 129, 1000), rng.uniform(-6e13, 6e13, (64, 999)).round(1)):
        if name in R.BITMAP_FUNCS:
            w = rng.uniform(0, 2.0 ** 40, m.shape[1]).round()
            w[rng.random(w.size) < 0.05] = NAN
            _check(name, m, w)
        else:
            _check(name, m)


def test_large_matrix(name="year"):
    """100 000 x 2048 (1.6 GB): realistic timestamps, +-1.9 million years and all of int64, in rows"""
    import torch
    import victoriametrics_b200 as vm
    rng = np.random.default_rng(SEED0 + 9)
    S, P = 100_000, 2048
    m = np.empty((S, P))
    m[: S // 2] = _realistic(rng, S // 2, P)
    m[S // 2: 3 * S // 4] = rng.uniform(-6e13, 6e13, (S // 4, P))
    m[3 * S // 4:] = _full_range(rng, S - 3 * S // 4, P)
    d = torch.from_numpy(m).cuda()
    vm.promql.transform(name, d.data_ptr(), S, P)
    torch.cuda.synchronize()
    got = d.cpu().numpy()
    del d
    for r0 in range(0, S, 10_000):
        assert _bits_equal(got[r0:r0 + 10_000], R.np_time_field(name, m[r0:r0 + 10_000])), (name, r0)


def test_error_paths():
    import torch
    import victoriametrics_b200 as vm
    lib, ctx = vm._lib.lib(), vm.default_context()
    m = np.arange(12, dtype=np.float64).reshape(3, 4) * 1e8
    d = torch.from_numpy(m).cuda()
    for op in (27, 31, 47, 63, 75, 100, -1):  # an id in each gap, one past the end, a negative one
        assert lib.vmb_transform(ctx.h, op, C.c_void_p(d.data_ptr()), 3, 4, None, None) == -50, op
    for name in R.BITMAP_FUNCS:
        assert lib.vmb_transform(ctx.h, vm.promql.TRANSFORM_FUNCS[name], C.c_void_p(d.data_ptr()), 3, 4, None, None) == -50
    torch.cuda.synchronize()
    assert np.array_equal(d.cpu().numpy(), m)
    assert lib.vmb_transform(ctx.h, vm.promql.TRANSFORM_FUNCS["hour"], C.c_void_p(d.data_ptr()), 0, 4, None, None) == 0


def test_on_a_callers_stream():
    import torch
    import victoriametrics_b200 as vm
    rng = np.random.default_rng(SEED0 + 13)
    m = _realistic(rng, 300, 500)
    w = rng.uniform(0, 1e6, 500).round()
    stream = torch.cuda.Stream()
    ctx = vm.Context(0, stream=stream.cuda_stream)
    try:
        with torch.cuda.stream(stream):
            a = torch.from_numpy(m).cuda()
            b = torch.from_numpy(m).cuda()
            vm.promql.transform("day_of_week", a.data_ptr(), 300, 500, ctx=ctx)
            vm.promql.transform("bitmap_or", b.data_ptr(), 300, 500, w, ctx=ctx)
        stream.synchronize()
        assert _bits_equal(a.cpu().numpy(), R.np_time_field("day_of_week", m))
        assert _bits_equal(b.cpu().numpy(), R.np_bitmap("bitmap_or", m, w))
    finally:
        ctx.close()
