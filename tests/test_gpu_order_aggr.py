"""vmb_aggr_order / promql.aggr_order bit for bit against tests/order_aggr_ref.py: the exec_test.go vectors, randomised
differentials over every function and group layout, group sizes at every edge of the sort's tiers (a thread or a warp per cell,
one shared-memory sort, chunks and merge passes), shapes of several point batches and one past 2^31 elements, the value edges
(ties, -0.0 / +0.0, +-Inf, NaN medians, subnormals, +-DBL_MAX), every phi edge, tolerances, `limit`, guard bands, determinism and
every error path.  The rule is assert_same_bits (-0.0 != +0.0), except the sign of a zero quantiles / mode result where a tied rank
holds both zeros (EXCEPTIONS["quantile"] of test_gpu_matrix_exact: the reference's sort is not stable there)."""
import ctypes as C
import zlib

import numpy as np
import pytest

from conftest import SEED0
from order_aggr_ref import FUNCS, ROW_FUNCS, aggr_order_ref
from test_enum_tables import HDR, _enum
from test_gpu_matrix_exact import EXCEPTIONS
from test_gpu_rollup_exact import assert_same_bits

pytestmark = pytest.mark.gpu
NAN, INF = float("nan"), float("inf")
DMAX, SUB = np.finfo(np.float64).max, 5e-324
SENTINEL = -7.25
GUARD = 33
C_SORT = 4096  # OA_C: keys of one shared-memory sort
PHIS = [NAN, -2, 0, 0.2, 0.25, 0.5, 0.75, 1, 3]
T = np.arange(1000, 2001, 200, dtype=np.float64)


def seed(name, k=0):
    return np.random.default_rng(SEED0 + zlib.crc32(("order_aggr/%s/%d" % (name, k)).encode()))


@pytest.fixture(scope="module")
def vm():
    import victoriametrics_b200 as v
    return v


def run(vm, name, vals, groups=None, G=1, phis=(0.5,), tol=1.0, limit=0, dv=None):
    """-> (output matrix or None, what aggr_order returned); checks the guard bands around the output"""
    import torch
    if dv is None:
        vals = np.ascontiguousarray(vals, dtype=np.float64)
        dv = torch.from_numpy(vals).cuda()
    S, P = dv.shape
    if name in ROW_FUNCS:
        return None, vm.promql.aggr_order(name, dv.data_ptr(), S, P, None, groups, G, tolerance=tol, limit=limit)
    K = np.asarray(phis).size if name == "quantiles" else 1
    n = K * G * P
    buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.float64, device="cuda")
    ret = vm.promql.aggr_order(name, dv.data_ptr(), S, P, buf.data_ptr() + 8 * GUARD, groups, G, phis=phis, limit=limit)
    torch.cuda.synchronize()
    b = buf.cpu().numpy()
    assert (b[:GUARD] == SENTINEL).all() and (b[GUARD + n:] == SENTINEL).all(), "guard band overwritten"
    out = b[GUARD:GUARD + n]
    return (out.reshape(K, G, P) if name == "quantiles" else out.reshape(G, P)), ret


def same(got, want, what, name):
    assert EXCEPTIONS["quantile"][0] == "zero sign"
    assert_same_bits(got, want, what, "quantile_over_time" if name in ("quantiles", "mode") else None)


def check(vm, name, vals, groups=None, G=1, phis=(0.5,), tol=1.0, limit=0, what=""):
    got, ret = run(vm, name, vals, groups, G, phis, tol, limit)
    want, wret = aggr_order_ref(name, vals, groups, G, phis, tol, limit)
    if name not in ROW_FUNCS:
        same(got, want, "%s %s" % (name, what), name)
    assert np.array_equal(np.asarray(ret), np.asarray(wret)), (name, what, ret, wret)
    return got if name not in ROW_FUNCS else ret


def check_all(vm, vals, groups=None, G=1, what="", tol=1.0):
    for name in FUNCS:
        check(vm, name, vals, groups, G, phis=PHIS, tol=tol, what=what)


# ------------------------------------------------------------------------------------------------ exec_test.go vectors
def test_exec_test_vectors(vm):
    three = np.array([np.full(6, x) for x in (3.0, 2.0, 3.0, 4.0, 3.0, 2.0)])
    assert check(vm, "mode", three)[0].tolist() == [3] * 6
    got = check(vm, "distinct", np.array([np.where(1 + T > 1100, 1 + T, NAN), np.where(T > 1700, T, NAN)]))[0]
    assert np.isnan(got[0]) and got[1:].tolist() == [1, 1, 1, 2, 2]
    ten = np.array([np.full(6, 10.0), T / 150])
    got = check(vm, "quantiles", ten, phis=[0.2, 0.5])
    assert got[0, 0].tolist() == [7.333333333333334, 8.4, 9.466666666666669, 10.133333333333333, 10.4, 10.666666666666668]
    assert got[1, 0].tolist() == [8.333333333333334, 9, 9.666666666666668, 10.333333333333332, 11, 11.666666666666668]
    assert check(vm, "quantiles", ten, phis=[-2])[0, 0].tolist() == [-INF] * 6
    assert check(vm, "quantiles", ten, phis=[3])[0, 0].tolist() == [INF] * 6
    got = check(vm, "quantiles", np.array([np.full(6, 10.0), T / 150, T / 200]))
    assert got[0, 0].tolist() == [6.666666666666667, 8, 9.333333333333334, 10, 10, 10]
    mad3 = np.array([T, T * 1.5, T * 0.9])
    assert check(vm, "mad", mad3)[0].tolist() == [100, 120, 140, 160, 180, 200]
    assert check(vm, "outliers_iqr", np.array([T, T * 1.5, T * 10, T * 1.2, T * 0.1])).tolist() == [0, 0, 1, 0, 1]
    assert check(vm, "outliers_mad", mad3, tol=1).tolist() == [0, 1, 0]
    assert check(vm, "outliers_mad", mad3, tol=5).tolist() == [0, 0, 0]


# ------------------------------------------------------------------------------------------------ randomised differentials
def matrix(rng, S, P, ties=False):
    """normals over many scales, or small integers (heavy ties); -0.0 / +0.0, +-Inf, subnormals, +-DBL_MAX, NaN cells and rows"""
    if ties:
        m = rng.integers(-3, 4, (S, P)).astype(np.float64)
    else:
        m = rng.normal(size=(S, P)) * 10.0 ** rng.integers(-3, 4, (S, P))
    m[rng.random((S, P)) < 0.1] = NAN
    sel = rng.random((S, P)) < 0.04
    m[sel] = rng.choice(np.array([INF, -INF, 0.0, -0.0, SUB, -SUB, DMAX, -DMAX]), int(sel.sum()))
    m[rng.random(S) < 0.08] = NAN  # all-NaN rows
    return m


def layout(rng, kind, S):
    if kind == "one":
        return np.zeros(S, dtype=np.uint32), 1
    if kind == "few":
        return rng.integers(0, 5, S).astype(np.uint32), 6  # group 5 has no rows
    if kind == "singletons":
        return rng.permutation(S).astype(np.uint32), S
    sizes = [S // 2, S // 4, 1, 1, 2, 3]  # skewed
    sizes.append(S - sum(sizes))
    g = np.repeat(np.arange(len(sizes)), sizes).astype(np.uint32)
    rng.shuffle(g)
    return g, len(sizes)


@pytest.mark.parametrize("P", [1, 7, 32, 1000])
@pytest.mark.parametrize("kind", ["one", "few", "singletons", "skewed"])
def test_random_differential(vm, kind, P):
    S = 61 if P == 1000 else 301
    for ties in (False, True):
        rng = seed("%s/%d/%d" % (kind, P, ties))
        vals = matrix(rng, S, P, ties)
        groups, G = layout(rng, kind, S)
        tol = rng.choice(np.array([NAN, 0.0, -1.0, INF, 0.5, 1.0, 3.0]), P)
        check_all(vm, vals, groups, G, what="%s P=%d ties=%d" % (kind, P, ties), tol=tol)


def test_tier_edges(vm):
    """one group of each size at the edges of the finish (thread / warp per cell) and of the sort (one shared-memory sort, chunks
    merged in 1 or 2 passes); small integers, so that runs cross the chunk and merge-tile boundaries"""
    sizes = [1, 2, 3, 31, 32, 33, C_SORT - 1, C_SORT, C_SORT + 1, 2 * C_SORT + 1]
    rng = seed("tiers")
    g = np.repeat(np.arange(len(sizes)), sizes).astype(np.uint32)
    rng.shuffle(g)
    for ties in (True, False):
        vals = matrix(rng, len(g), 3, ties)
        check_all(vm, vals, g, len(sizes), what="tiers ties=%d" % ties, tol=np.array([1.0, 0.0, 2.0]))


def test_one_group_of_100k_rows(vm):
    """one segment of 100 000 keys per point: 25 sorted chunks, 5 merge passes, a warp per cell"""
    rng = seed("100k")
    vals = matrix(rng, 100_000, 2, ties=True)
    vals[:, 1] = rng.normal(size=100_000)
    check_all(vm, vals, what="100k")


def test_value_edges(vm):
    """+-Inf medians and their NaN deviations, a NaN median from Inf * 0, all-NaN cells, +-0.0 runs, DBL_MAX deviations"""
    P = 8
    cols = [
        [1.0, 2.0, INF],                 # median 2 + Inf * 0 = NaN: mad NaN
        [1.0, 2.0, INF, INF],            # median Inf: deviations NaN, NaN, Inf, Inf
        [-INF, -INF, -INF, 5.0],         # median -Inf
        [0.0, -0.0, -0.0, 0.0],          # one run of zeros
        [-0.0, 1.0, 1.0, -0.0, 0.0],
        [DMAX, -DMAX, DMAX, 0.0],        # deviations overflow to Inf
        [NAN, NAN, NAN, NAN],            # an all-NaN cell
        [SUB, -SUB, 0.0, SUB],
    ]
    n = max(len(c) for c in cols)
    vals = np.full((n, P), NAN)
    for p, c in enumerate(cols):
        vals[:len(c), p] = c
    check_all(vm, vals, what="edges", tol=np.array([1.0, 0.0, INF, NAN, -1.0, 1.0, 1.0, 0.5]))
    check_all(vm, vals[::-1].copy(), what="edges reversed")
    check_all(vm, np.full((5, 4), NAN), np.array([0, 1, 0, 1, 0]), 3, what="all-NaN groups")


def test_point_batches(vm):
    """more keys than one batch holds (2^27): two batches of different widths; compared on column strips at both ends and across
    the boundary"""
    import torch
    rng = seed("batches")
    S, P, G = 70_000, 2_000, 8
    B = (1 << 27) // S
    assert B < P
    dv = torch.randint(-20, 21, (S, P), dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(SEED0 + 5))
    dv[torch.rand(S, P, device="cuda", generator=torch.Generator("cuda").manual_seed(SEED0 + 6)) < 0.05] = NAN
    groups = rng.integers(0, G, S).astype(np.uint32)
    strips = np.r_[0:3, B - 3:B + 3, P - 3:P]
    host = dv[:, strips].cpu().numpy()
    for name in FUNCS:
        got, ret = run(vm, name, None, groups, G, phis=[0.1, 0.5, 0.99], tol=2.0, dv=dv)
        want, wret = aggr_order_ref(name, host, groups, G, [0.1, 0.5, 0.99], 2.0)
        if name in ROW_FUNCS:  # the strip cannot see points outside it: a row it selects must be selected overall
            assert not (wret & ~ret).any(), name
            continue
        same(got[..., strips], want, "%s batches" % name, name)
        assert np.array_equal(ret, wret)


def test_past_2_pow_31_elements(vm):
    """S * P just above 2^31 values (17 GB): every index product must be 64-bit; compared on column strips"""
    import torch
    S, P, G = 65_537, 32_768, 3
    assert S * P > 2 ** 31
    gen = torch.Generator("cuda").manual_seed(SEED0 + 7)
    dv = torch.randint(0, 50, (S, P), dtype=torch.float64, device="cuda", generator=gen)
    groups = (np.arange(S) % G).astype(np.uint32)
    strips = np.r_[0:2, P // 2 - 1:P // 2 + 2, P - 2:P]  # the last row lies wholly past element 2^31
    host = dv[:, strips].cpu().numpy()
    for name in ("quantiles", "distinct"):
        got, _ = run(vm, name, None, groups, G, phis=[0.25, 0.5], dv=dv)
        want, _ = aggr_order_ref(name, host, groups, G, [0.25, 0.5])
        same(got[..., strips], want, "%s 2^31" % name, name)
    del dv
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ arguments, limit, determinism
def test_phis_and_tolerances(vm):
    rng = seed("phis")
    vals = matrix(rng, 50, 9, ties=True)
    groups, G = layout(rng, "few", 50)
    got = check(vm, "quantiles", vals, groups, G, phis=PHIS)
    assert got.shape == (len(PHIS), G, 9)
    check(vm, "quantiles", vals, groups, G, phis=0.3)
    for tol in (NAN, 0.0, -1.0, INF, 1.5, rng.choice(np.array([NAN, 0.0, -2.0, INF, 1.0]), 9)):
        check(vm, "outliers_mad", vals, groups, G, tol=tol)


def test_limit_and_group_existence(vm):
    rng = seed("limit")
    S, P = 40, 9
    vals = matrix(rng, S, P)
    groups = rng.integers(0, 8, S).astype(np.uint32)
    vals[groups == 3] = NAN  # group 3 has rows, all empty: not in the output
    vals[:4] = NAN
    for name in FUNCS:
        for limit in (0, 1, 2, 5, 100):
            check(vm, name, vals, groups, 9, phis=[0.5, 0.9], limit=limit, what="limit %d" % limit)
    _, ret = run(vm, "mode", vals, groups, 9)
    assert 3 not in ret.tolist() and 8 not in ret.tolist()


def test_no_rows(vm):
    for P in (1, 40):
        got, ret = run(vm, "quantiles", np.zeros((0, P)), np.zeros(0, dtype=np.uint32), 3, phis=[0.5, 0.9])
        assert np.isnan(got).all() and len(ret) == 0
        got, _ = run(vm, "mad", np.zeros((0, P)), np.zeros(0, dtype=np.uint32), 2)
        assert np.isnan(got).all()


def test_same_call_twice_same_bits(vm):
    rng = seed("twice")
    vals = matrix(rng, 9000, 5)
    groups, G = layout(rng, "skewed", 9000)
    for name in ("quantiles", "mode", "mad"):
        a, _ = run(vm, name, vals, groups, G, phis=PHIS)
        b, _ = run(vm, name, vals, groups, G, phis=PHIS)
        assert a.tobytes() == b.tobytes(), name


def test_quantiles_match_aggr_quantile(vm):
    """quantiles with one phi == vmb_aggr_quantile, on groups within its 2048-series cap"""
    import torch
    rng = seed("aggr_quantile")
    S, P, G = 3000, 17, 3
    vals = matrix(rng, S, P)
    groups = rng.integers(0, G, S).astype(np.uint32)
    dv = torch.from_numpy(vals).cuda()
    for phi in (0.0, 0.3, 0.5, 0.99, 1.0):
        got, _ = run(vm, "quantiles", None, groups, G, phis=[phi], dv=dv)
        old = torch.full((G * P,), SENTINEL, dtype=torch.float64, device="cuda")
        vm.promql.aggr_quantile(phi, dv.data_ptr(), S, P, old.data_ptr(), groups, G)
        assert_same_bits(got[0], old.cpu().numpy().reshape(G, P), "phi %g" % phi, "quantile_over_time")


# ------------------------------------------------------------------------------------------------ errors
def test_errors_leave_the_outputs_untouched(vm):
    import torch
    from victoriametrics_b200 import _lib
    lib, ctx = _lib.lib(), _lib.default_context()
    S, P = 8, 5
    dv = torch.ones(S * P, dtype=torch.float64, device="cuda")
    out = torch.full((2 * S * P,), SENTINEL, dtype=torch.float64, device="cuda")
    ne = np.full(S, 7, dtype=np.uint8)
    sel = np.full(S, 7, dtype=np.uint8)
    phis = np.array([0.5, 0.9])
    tol = np.ones(P)

    def call(func, nseries=S, points=P, groups=np.zeros(S, dtype=np.uint32), G=1, args=None, nargs=None, o=True, n=True, s=True):
        g = np.ascontiguousarray(groups, dtype=np.uint32)
        a = args.ctypes.data_as(_lib.f64p) if args is not None else None
        na = (0 if args is None else args.size) if nargs is None else nargs
        return lib.vmb_aggr_order(ctx.h, func, C.c_void_p(dv.data_ptr()), nseries, points, g.ctypes.data_as(_lib.u32p), G, a, na,
                                  C.c_void_p(out.data_ptr() if o else 0), ne.ctypes.data_as(_lib.u8p) if n else None,
                                  sel.ctypes.data_as(_lib.u8p) if s else None)
    assert call(6) == -50 and call(-1) == -50
    assert call(2, G=0) == -50
    assert call(2, groups=np.array([0, 0, 0, 1, 0, 0, 0, 0]), G=1) == -50
    assert call(2, nseries=2 ** 31) == -50 and call(2, points=2 ** 31) == -50
    assert call(0) == -50 and call(0, args=phis, nargs=0) == -50  # quantiles needs a phi
    assert call(1, args=phis) == -50 and call(2, args=phis) == -50 and call(3, args=phis) == -50 and call(4, args=phis) == -50
    assert call(5) == -50 and call(5, args=np.ones(P - 1)) == -50  # outliers_mad: one tolerance per point
    assert call(0, args=None, nargs=2) == -50  # nargs without args
    assert call(2, o=False) == -50 and call(2, n=False) == -50 and call(4, s=False) == -50
    assert (out.cpu().numpy() == SENTINEL).all() and (ne == 7).all() and (sel == 7).all()
    assert call(0, args=phis) == 0 and (out.cpu().numpy()[:2 * P] == 1).all() and (ne == 1).all()
    assert call(5, args=tol, o=False) == 0 and (sel == 0).all()


def test_enum_follows_the_header(vm):
    pub = _enum(HDR, "vmb_order_aggr")
    assert {n[len("VMB_OA_"):].lower(): v for n, v in pub} == vm.promql.ORDER_AGGR_FUNCS
