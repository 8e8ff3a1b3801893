"""vmb_transform_range / promql.transform_range and vmb_transform's smooth_exponential bit for bit against
tests/range_transform_ref.py: every function at every sort tier of P (a shared-memory sort, chunks merged in 1 .. 4 passes),
more rows than one grid pass, two row batches, one row longer than the key budget, a matrix past 2^31 elements; all-NaN rows,
single values, leading / trailing NaNs, +-Inf, +-0.0, subnormals, +-DBL_MAX, constant rows; the argument edges; normalize's
kept rows; guard bands, determinism and every error path.  The rule is assert_same_bits (-0.0 != +0.0), except the sign of a
zero range_quantile result where a tied rank holds both zeros (the reference's sort is not stable there)."""
import ctypes as C
import zlib

import numpy as np
import pytest

from conftest import SEED0
from range_transform_ref import FUNCS, ONE_ARG, range_transform_ref, smooth_exponential_ref
from test_gpu_rollup_exact import assert_same_bits

pytestmark = pytest.mark.gpu
NAN, INF = float("nan"), float("inf")
DMAX, SUB = np.finfo(np.float64).max, 5e-324
SENTINEL = -7.25
GUARD = 33
STEP = 15_000
BUDGET = 1 << 27  # OA_BUDGET: keys of one row batch
DEFAULT_ARG = {"range_trim_zscore": 1.0, "range_quantile": 0.9, "range_trim_outliers": 2.0, "range_trim_spikes": 0.1}


def seed(name, k=0):
    return np.random.default_rng(SEED0 + zlib.crc32(("range_transform/%s/%d" % (name, k)).encode()))


@pytest.fixture(scope="module")
def vm():
    import victoriametrics_b200 as v
    return v


def call(vm, name, dev_ptr, S, P, arg=None):
    if name == "smooth_exponential":
        return vm.promql.transform(name, dev_ptr, S, P, arg)
    args = (arg,) if name in ONE_ARG else ()
    return vm.promql.transform_range(name, dev_ptr, S, P, *args, step=STEP)


def run(vm, name, vals, arg=None):
    """-> (matrix after the call, what the call returned); checks the guard bands around the matrix"""
    import torch
    vals = np.ascontiguousarray(vals, dtype=np.float64)
    S, P = vals.shape
    n = S * P
    buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.float64, device="cuda")
    buf[GUARD:GUARD + n] = torch.from_numpy(vals.reshape(-1)).cuda()
    ret = call(vm, name, buf.data_ptr() + 8 * GUARD, S, P, arg)
    torch.cuda.synchronize()
    b = buf.cpu().numpy()
    assert (b[:GUARD] == SENTINEL).all() and (b[GUARD + n:] == SENTINEL).all(), "guard band overwritten"
    return b[GUARD:GUARD + n].reshape(S, P), ret


def ref(name, vals, arg=None):
    if name == "smooth_exponential":
        return smooth_exponential_ref(vals, arg), None
    return range_transform_ref(name, vals, arg, STEP)


def same(got, want, what, name):
    assert_same_bits(got, want, what, "quantile_over_time" if name == "range_quantile" else None)


def check(vm, name, vals, arg=None, what=""):
    if arg is None:
        arg = DEFAULT_ARG.get(name, 0.3)
    got, ret = run(vm, name, vals, arg)
    want, kept = ref(name, vals, arg)
    same(got, want, "%s(%r) %s" % (name, arg, what), name)
    if name == "range_normalize":
        assert np.array_equal(ret, kept), (what, ret, kept)
    return got


def matrix(rng, S, P, ties=False):
    """gauge-like rows over many scales or small integers (ties, constant runs); NaN cells, +-Inf, +-0.0, subnormals, +-DBL_MAX;
    all-NaN rows, one-value rows, leading / trailing NaNs, constant rows"""
    if ties:
        m = rng.integers(-3, 4, (S, P)).astype(np.float64)
    else:
        m = 1000 + np.cumsum(rng.normal(size=(S, P)), axis=1) * 10.0 ** rng.integers(-3, 4, (S, 1))
    m[rng.random((S, P)) < 0.05] = NAN
    sel = rng.random((S, P)) < 0.01
    m[sel] = rng.choice(np.array([INF, -INF, 0.0, -0.0, SUB, -SUB, DMAX, -DMAX]), int(sel.sum()))
    for r in range(S):
        k = r % 8
        if k == 0:
            m[r] = NAN
        elif k == 1:
            m[r] = NAN
            m[r, rng.integers(P)] = rng.normal()
        elif k == 2:
            m[r, :rng.integers(P + 1)] = NAN
        elif k == 3:
            m[r, rng.integers(P + 1):] = NAN
        elif k == 4:
            m[r] = 7.5
    return m


TIER_P = [1, 2, 31, 32, 33, 4096, 4097, 8172, 40_000]


@pytest.mark.parametrize("P", TIER_P)
def test_every_function_every_tier(vm, P):
    rng = seed("tiers", P)
    S = max(9, min(100, 120_000 // P))
    for ties in (False, True):
        vals = matrix(rng, S, P, ties)
        for name in FUNCS + ["smooth_exponential"]:
            check(vm, name, vals, what="P=%d ties=%d" % (P, ties))


def test_exec_test_vectors(vm):
    T = np.arange(1000, 2001, 200, dtype=np.float64)
    got = check(vm, "range_trim_spikes", np.array([T]), 0.2)
    assert np.isnan(got[0, [0, 5]]).all() and got[0, 1:5].tolist() == [1200, 1400, 1600, 1800]
    assert check(vm, "range_quantile", np.array([T]), 0.5)[0].tolist() == [1500] * 6
    assert check(vm, "range_mad", np.array([T]))[0].tolist() == [300] * 6
    assert check(vm, "smooth_exponential", np.array([T]), 0.5)[0].tolist() == [1000, 1100, 1250, 1425, 1612.5, 1806.25]
    got = check(vm, "range_normalize", np.array([T, -T]))
    assert got[0].tolist() == [0, 0.2, 0.4, 0.6, 0.8, 1]


def test_many_rows_more_than_one_grid_pass(vm):
    """300 000 rows: more than one pass of the row-walk grid (132 x 16 CTAs x 128 rows) and of the element grids; compared on a
    sample of rows"""
    rng = seed("rows")
    for P in (1, 3):
        vals = matrix(rng, 300_000, P)
        rows = np.r_[0:300, rng.choice(300_000, 700, replace=False), 299_700:300_000]
        for name in FUNCS + ["smooth_exponential"]:
            arg = DEFAULT_ARG.get(name, 0.3)
            got, ret = run(vm, name, vals, arg)
            want, kept = ref(name, vals[rows], arg)
            same(got[rows], want, "%s P=%d rows" % (name, P), name)
            if name == "range_normalize":
                assert np.array_equal(ret[rows], kept)


def test_value_edges(vm):
    """mean overflow to Inf, Inf - Inf, a zero stddev, +-0.0 ranks, subnormals, one value, constant rows"""
    rows = [
        [DMAX, DMAX, DMAX, 1.0],            # the mean overflows
        [DMAX, -DMAX, DMAX, -DMAX],
        [INF, 1.0, 2.0, 3.0],
        [INF, -INF, 1.0, NAN],
        [INF, INF, INF, INF],               # normalize: Inf - Inf is NaN, not Inf: kept
        [-0.0, 0.0, -0.0, 0.0],
        [0.0, -0.0, NAN, -0.0],
        [SUB, -SUB, SUB, 0.0],
        [5.0, 5.0, 5.0, 5.0],               # constant: zscore 0/0, the regression's const path
        [5.0, 5.0, NAN, 5.0],               # a NaN: not constant
        [NAN, NAN, NAN, 3.0],               # one value: stdvar 0 (not NaN) only for P == 1
        [NAN, NAN, NAN, NAN],
        [1.0, NAN, NAN, NAN],
        [1e300, -1e300, 1e-300, 7.0],
    ]
    vals = np.array(rows)
    for name in FUNCS + ["smooth_exponential"]:
        check(vm, name, vals, what="edges")
        check(vm, name, vals[:, ::-1].copy(), what="edges reversed")
        check(vm, name, vals[:, :1].copy(), what="edges P=1")


def test_argument_edges(vm):
    rng = seed("args")
    vals = np.concatenate([matrix(rng, 40, 37), matrix(rng, 40, 37, ties=True)])
    for phi in (-0.5, 0.0, 0.25, 0.5, 1.0, 1.5, NAN, -INF, INF):
        check(vm, "range_quantile", vals, phi, "phi")
    for phi in (-1.0, 0.0, 0.1, 0.5, 1.0, 1.9, 2.0, 2.5, NAN):
        check(vm, "range_trim_spikes", vals, phi, "phi")
    for z in (0.0, 0.5, -0.5, 1.0, -3.0, NAN, INF):
        check(vm, "range_trim_zscore", vals, z, "z")
    for k in (NAN, 0.0, -1.0, 0.5, 3.0, INF):
        check(vm, "range_trim_outliers", vals, k, "k")
    # a per-point argument: only the first point's value counts (getScalar(...)[0])
    arr = np.r_[0.5, np.full(36, NAN)]
    got, _ = run(vm, "range_quantile", vals, arr)
    same(got, ref("range_quantile", vals, 0.5)[0], "per-point phi", "range_quantile")


def test_smooth_exponential(vm):
    """factors NaN / negative / > 1 / per point; rows that start with Infs, Infs across tile edges, nothing but Infs behind the
    leading NaNs (the walk starts at the first Inf)"""
    rng = seed("smooth")
    P = 100
    vals = matrix(rng, 64, P)
    vals[8, :40] = INF
    vals[9, :3] = NAN
    vals[9, 3:50] = -INF
    vals[10, :] = INF
    vals[11, :5] = NAN
    vals[11, 5:] = rng.choice(np.array([INF, -INF]), P - 5)
    vals[12, :70] = NAN
    vals[12, 70:] = rng.choice(np.array([INF, -INF]), P - 70)
    vals[13, :2] = [INF, NAN]
    vals[14, 40] = INF
    for sf in (0.0, 1.0, 0.3, NAN, -1.0, 2.0, rng.choice(np.array([NAN, -0.5, 0.0, 0.2, 0.7, 1.0, 1.5]), P)):
        check(vm, "smooth_exponential", vals, sf, "sf")


def test_normalize_kept_rows(vm):
    rng = seed("normalize")
    vals = matrix(rng, 200, 45)
    vals[5] = NAN
    vals[6, 3] = INF
    vals[7, 3], vals[7, 9] = -INF, INF
    vals[8] = INF
    vals[9] = NAN
    vals[9, 20] = 4.0
    got = check(vm, "range_normalize", vals)
    _, kept = run(vm, "range_normalize", vals)
    assert not kept[5] and not kept[6] and not kept[7] and kept[8] and kept[9]
    assert np.isnan(got[9]).all()
    assert np.array_equal(got[~kept], vals[~kept], equal_nan=True)  # dropped rows are untouched


def _dev(S, P, seed_k, ints=True):
    import torch
    gen = torch.Generator("cuda").manual_seed(SEED0 + seed_k)
    dv = (torch.randint(-20, 21, (S, P), dtype=torch.float64, device="cuda", generator=gen) if ints else
          torch.randn(S, P, dtype=torch.float64, device="cuda", generator=gen))
    dv[torch.rand(S, P, device="cuda", generator=gen) < 0.05] = NAN
    return dv


def test_two_row_batches(vm):
    """more keys than one batch holds (2^27): a full batch and a shorter last one; rows on both sides of the boundary"""
    S, P = 20_000, 8172
    B = BUDGET // P
    assert B < S
    rows = np.r_[0:3, B - 3:B + 3, S - 3:S]
    for name in FUNCS:
        dv = _dev(S, P, 11, ints=name != "range_linear_regression")
        host = dv[rows].cpu().numpy()
        arg = DEFAULT_ARG.get(name)
        call(vm, name, dv.data_ptr(), S, P, arg)
        want, _ = ref(name, host, arg)
        same(dv[rows].cpu().numpy(), want, "%s batches" % name, name)
        del dv


def test_one_row_longer_than_the_budget(vm):
    """one row of 2^27 + 5000 keys: the budget widens to that row; 15 merge passes"""
    S, P = 1, BUDGET + 5000
    for name in ("range_quantile", "range_mad"):
        dv = _dev(S, P, 12)
        host = dv.cpu().numpy()
        call(vm, name, dv.data_ptr(), S, P, 0.3)
        want, _ = ref(name, host, 0.3)
        same(dv.cpu().numpy(), want, "%s long row" % name, name)
        del dv


def test_past_2_pow_31_elements(vm):
    """S * P just above 2^31 values (17 GB): every index product must be 64-bit; rows at both ends compared"""
    import torch
    S, P = 65_537, 32_768
    assert S * P > 2 ** 31
    rows = np.r_[0:2, S // 2:S // 2 + 1, S - 2:S]  # the last row lies wholly past element 2^31
    for name in ("range_stddev", "range_zscore", "range_linear_regression", "range_quantile", "range_trim_spikes"):
        dv = _dev(S, P, 13, ints=False)
        host = dv[rows].cpu().numpy()
        arg = DEFAULT_ARG.get(name)
        call(vm, name, dv.data_ptr(), S, P, arg)
        want, _ = ref(name, host, arg)
        same(dv[rows].cpu().numpy(), want, "%s 2^31" % name, name)
        del dv
        torch.cuda.empty_cache()


def test_same_call_twice_same_bits(vm):
    rng = seed("twice")
    vals = matrix(rng, 300, 5000)
    for name in ("range_quantile", "range_mad", "range_zscore", "range_linear_regression", "smooth_exponential"):
        a, _ = run(vm, name, vals, DEFAULT_ARG.get(name, 0.3))
        b, _ = run(vm, name, vals, DEFAULT_ARG.get(name, 0.3))
        assert a.tobytes() == b.tobytes(), name


def test_errors_leave_the_matrix_untouched(vm):
    import torch
    from victoriametrics_b200 import _lib
    lib, ctx = _lib.lib(), _lib.default_context()
    S, P = 8, 5
    dv = torch.full((S * P,), SENTINEL, dtype=torch.float64, device="cuda")
    kept = np.full(S, 7, dtype=np.uint8)

    def rs(func, nrows=S, points=P, args=None, nargs=None, k=True, ptr=None):
        a = np.ascontiguousarray(args, dtype=np.float64) if args is not None else None
        na = (0 if a is None else a.size) if nargs is None else nargs
        return lib.vmb_transform_range(ctx.h, func, C.c_void_p(dv.data_ptr() if ptr is None else ptr), nrows, points,
                                       a.ctypes.data_as(_lib.f64p) if a is not None else None, na,
                                       kept.ctypes.data_as(_lib.u8p) if k else None)
    one = [0.5]
    assert rs(10) == -50 and rs(-1) == -50                                     # unknown function
    assert rs(0, args=one) == -50 and rs(7, args=one) == -50                  # stddev, mad take no argument
    assert rs(6) == -50 and rs(8) == -50 and rs(9) == -50 and rs(3) == -50    # quantile, trim_* need one
    assert rs(6, args=[0.5, 0.5]) == -50
    assert rs(6, nargs=1) == -50                                              # nargs without args
    assert rs(4, k=False) == -50                                              # normalize needs row_kept
    for step in (0.0, -15000.0, 1.5, NAN, INF, 1e19):
        assert rs(5, args=[step]) == -50, step
    assert rs(5) == -50
    assert rs(0, nrows=2 ** 31) == -50 and rs(0, points=2 ** 31) == -50
    assert rs(0, ptr=0) == -50
    sf = np.full(P, 0.5)
    assert lib.vmb_transform(ctx.h, vm.promql.TRANSFORM_FUNCS["smooth_exponential"], C.c_void_p(dv.data_ptr()), S, P, None, None) == -50
    assert (dv.cpu().numpy() == SENTINEL).all() and (kept == 7).all()
    assert rs(0, nrows=0) == 0 and rs(6, points=0, args=one) == 0 and (dv.cpu().numpy() == SENTINEL).all()
    assert rs(4) == 0 and (kept == 1).all()
    assert lib.vmb_transform(ctx.h, vm.promql.TRANSFORM_FUNCS["smooth_exponential"], C.c_void_p(dv.data_ptr()), S, P,
                             sf.ctypes.data_as(_lib.f64p), None) == 0
