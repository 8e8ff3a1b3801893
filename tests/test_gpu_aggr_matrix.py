"""vmb_aggr_matrix / promql.aggr_matrix bit for bit against tests/aggr_matrix_ref.py: the exec_test.go vectors, randomised
differentials over every function, group layout and both kernel mappings (P < 32: a lane per cell; P >= 32: a warp per strip of
32 points), the `len(tss) == 1` fast paths, row flags and `limit`, shapes past one pass of the grid, guard bands around the output
and every error path.  The rule is assert_same_bits (-0.0 != +0.0); geomean over two or more values is the one exception
(EXCEPTIONS["geomean"] of test_gpu_matrix_exact: CUDA's pow and the reference's round differently)."""
import ctypes as C
import zlib

import numpy as np
import pytest

from aggr_matrix_ref import GROUP_FUNCS, ROW_FUNCS, aggr_matrix_ref
from conftest import SEED0
from test_enum_tables import HDR, _enum
from test_gpu_matrix_exact import EXCEPTIONS
from test_gpu_rollup_exact import assert_same_bits

pytestmark = pytest.mark.gpu
NAN, INF = float("nan"), float("inf")
FUNCS = GROUP_FUNCS + ROW_FUNCS
SENTINEL = -7.25
GUARD = 33
T = np.arange(1000, 2001, 200, dtype=np.float64)


def seed(name, k=0):
    return np.random.default_rng(SEED0 + zlib.crc32(("aggr_matrix/%s/%d" % (name, k)).encode()))


@pytest.fixture(scope="module")
def vm():
    import victoriametrics_b200 as v
    return v


def same(got, want, what, name):
    # geomean's exception is the rollup table's geomean_over_time entry, which EXCEPTIONS["geomean"] also names
    assert EXCEPTIONS["geomean"][0] == "rel"
    assert_same_bits(got, want, what, "geomean_over_time" if name == "geomean" else None)


def run(vm, name, vals, groups=None, G=1, limit=0, inplace=False):
    """-> (output matrix, what aggr_matrix returned); checks that the guard bands around the output kept their sentinels"""
    import torch
    vals = np.ascontiguousarray(vals, dtype=np.float64)
    S, P = vals.shape
    rows = S if name in ROW_FUNCS else G
    dv = torch.from_numpy(vals.copy()).cuda()
    buf = torch.full((rows * P + 2 * GUARD,), SENTINEL, dtype=torch.float64, device="cuda")
    out_ptr = dv.data_ptr() if inplace else buf.data_ptr() + 8 * GUARD
    ret = vm.promql.aggr_matrix(name, dv.data_ptr(), S, P, out_ptr, groups, G, limit=limit)
    torch.cuda.synchronize()
    b = buf.cpu().numpy()
    if inplace:
        assert (b == SENTINEL).all()
        return dv.cpu().numpy(), ret
    assert (b[:GUARD] == SENTINEL).all() and (b[GUARD + rows * P:] == SENTINEL).all(), "guard band overwritten"
    return b[GUARD:GUARD + rows * P].reshape(rows, P), ret


def check(vm, name, vals, groups=None, G=1, limit=0, what="", inplace=False):
    got, ret = run(vm, name, vals, groups, G, limit, inplace)
    want, wret = aggr_matrix_ref(name, vals, groups, G, limit)
    same(got, want, "%s %s" % (name, what), name)
    assert np.array_equal(np.asarray(ret), np.asarray(wret)), (name, what, ret, wret)
    return got


# ------------------------------------------------------------------------------------------------ exec_test.go vectors
def test_exec_test_vectors(vm):
    ten = np.full(6, 10.0)
    assert check(vm, "sum", [T / 100])[0].tolist() == [10, 12, 14, 16, 18, 20]
    assert check(vm, "geomean", [T / 100])[0].tolist() == [10, 12, 14, 16, 18, 20]
    assert check(vm, "sum2", [T / 100])[0].tolist() == [100, 144, 196, 256, 324, 400]
    assert check(vm, "sum", [ten, T / 100])[0].tolist() == [20, 22, 24, 26, 28, 30]
    assert check(vm, "sum2", [ten, T / 100])[0].tolist() == [200, 244, 296, 356, 424, 500]
    assert check(vm, "avg", [ten, T / 100])[0].tolist() == [10, 11, 12, 13, 14, 15]
    assert check(vm, "stddev", [ten, T / 100])[0].tolist() == [0, 1, 2, 3, 4, 5]
    got = check(vm, "count", [np.where(T < 1500, T, NAN), np.where(T < 1800, T, NAN)])[0]
    assert got[:4].tolist() == [2, 2, 2, 1] and np.isnan(got[4:]).all()
    assert check(vm, "min", [ten, T / 100 / 1.5])[0].tolist() == [6.666666666666667, 8, 9.333333333333334, 10, 10, 10]
    assert check(vm, "max", [ten, T / 100 / 1.5])[0].tolist() == [10, 10, 10, 10.666666666666666, 12, 13.333333333333334]
    assert check(vm, "group", [np.full(6, 5.0), np.full(6, 6.0), np.full(6, 7.0)])[0].tolist() == [1] * 6
    check(vm, "geomean", [ten, T / 100])
    out = check(vm, "sum", [ten, T / 100], np.array([0, 1]), 2)
    assert out[0].tolist() == [10] * 6 and out[1].tolist() == [10, 12, 14, 16, 18, 20]
    _, groups = run(vm, "sum", np.array([ten, T / 100]), np.array([0, 1]), 2, limit=1)
    assert groups.tolist() == [0]
    four = np.array([T / 100 + 10, T / 200 + 5, T / 110 - 10, T / 90 - 5])
    for name in ROW_FUNCS:
        check(vm, name, four)
        check(vm, name, four, np.array([0, 1, 0, 1]), 2)


# ------------------------------------------------------------------------------------------------ randomised differentials
def matrix(rng, S, P):
    m = rng.normal(size=(S, P)) * 10.0 ** rng.integers(-3, 4, (S, P))
    m[rng.random((S, P)) < 0.1] = NAN
    sel = rng.random((S, P)) < 0.01
    m[sel] = rng.choice(np.array([INF, -INF, 0.0, -0.0]), int(sel.sum()))
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


@pytest.mark.parametrize("P", [1, 7, 32, 8172])
@pytest.mark.parametrize("kind", ["one", "few", "singletons", "skewed"])
def test_random_differential(vm, kind, P):
    S = 97 if P == 8172 else 301
    for k, name in enumerate(FUNCS):
        rng = seed("%s/%d/%s" % (kind, P, name))
        vals = matrix(rng, S, P)
        groups, G = layout(rng, kind, S)
        check(vm, name, vals, groups, G, what="%s P=%d" % (kind, P))


@pytest.mark.parametrize("name", FUNCS)
def test_past_one_grid_pass(vm, name):
    """P = 40: 2 strips x 4000 singleton groups = 8000 warp items, more than the strip kernel's grid (4 x the resident warps), so
    warps take many items and cross strips; P = 7 with 40000 groups: more cells than the lane-per-cell grid holds"""
    rng = seed("grid/" + name)
    for S, P in ((4000, 40), (40000, 7)):
        vals = matrix(rng, S, P)
        groups, G = layout(rng, "singletons", S)
        check(vm, name, vals, groups, G, what="S=%d P=%d" % (S, P))
    vals = matrix(rng, 3000, 40)
    groups = rng.integers(0, 1500, 3000).astype(np.uint32)
    check(vm, name, vals, groups, 1500, what="pairs")


@pytest.mark.parametrize("name", ROW_FUNCS)
def test_share_zscore_in_place(vm, name):
    rng = seed("inplace/" + name)
    for P in (3, 100):
        vals = matrix(rng, 50, P)
        groups, G = layout(rng, "few", 50)
        check(vm, name, vals, groups, G, what="in place P=%d" % P, inplace=True)


# ------------------------------------------------------------------------------------------------ fast-path edges
@pytest.mark.parametrize("P", [3, 40])
def test_fast_path_edges(vm, P):
    z = np.zeros(P)
    empty = np.full(P, NAN)
    negz = np.full(P, -0.0)
    negz[1] = NAN
    for name in ("sum", "avg"):  # the row itself keeps -0.0, with or without empty rows beside it
        for rows in ([negz], [empty, negz, empty]):
            got = check(vm, name, rows)
            assert np.signbit(got[0, 0])
    got = check(vm, "sum2", [negz])  # no fast path: 0 + (-0.0)(-0.0) = +0.0
    assert not np.signbit(got[0, 0])
    inf = z.copy()
    inf[0], inf[1], inf[2] = INF, -INF, NAN
    for name in ("stdvar", "stddev"):
        got = check(vm, name, [empty, inf])  # fast path: 0 where non-NaN, also for +-Inf
        assert got[0, :2].tolist() == [0.0, 0.0] and np.isnan(got[0, 2])
        got = check(vm, name, [inf, inf])  # general path: inf - inf
        assert np.isnan(got[0, :3]).all()
    g3 = np.full(P, 3.0)
    g3[0] = 2.9999999999999996
    for rows in ([g3], [g3, empty], [np.where(np.arange(P) % 2, NAN, g3), np.where(np.arange(P) % 2, g3, NAN)]):
        got, _ = run(vm, "geomean", np.array(rows))
        want, _ = aggr_matrix_ref("geomean", np.array(rows))
        assert_same_bits(got, want, "geomean count == 1 is exact")  # no tolerance
    for name, first, second in (("min", -0.0, 0.0), ("min", 0.0, -0.0), ("max", -0.0, 0.0), ("max", 0.0, -0.0)):
        got = check(vm, name, [np.full(P, first), np.full(P, second)])
        assert np.signbit(got[0, 0]) == np.signbit(first)  # the first of equal zeros
    neg = np.array([np.full(P, -1.0), np.full(P, -2.0)])
    got = check(vm, "share", neg)  # no non-negative value: all NaN
    assert np.isnan(got).all()
    zs = np.array([np.full(P, 0.0), np.full(P, -0.0), np.full(P, -3.0)])
    got = check(vm, "share", zs)  # sum 0: 0 / 0 = NaN, and -0.0 is not < 0
    assert np.isnan(got).all()
    got = check(vm, "zscore", [np.full(P, 5.0)])  # a singleton: (v - v) / 0
    assert np.isnan(got).all()


def test_limit_and_group_existence(vm):
    rng = seed("limit")
    S, P = 40, 9
    vals = matrix(rng, S, P)
    groups = rng.integers(0, 8, S).astype(np.uint32)
    vals[groups == 3] = NAN  # group 3 has rows, all empty: not in the output
    vals[:4] = NAN
    for name in ("sum", "count", "share", "zscore"):
        for limit in (0, 1, 2, 5, 100):
            got, ret = run(vm, name, vals, groups, 9, limit=limit)
            want, wret = aggr_matrix_ref(name, vals, groups, 9, limit)
            same(got, want, "%s limit %d" % (name, limit), name)
            assert np.array_equal(ret, wret)
    _, ret = run(vm, "sum", vals, groups, 9)
    nonempty = ~np.isnan(vals).all(axis=1)
    first = [int(g) for i, g in enumerate(groups) if nonempty[i] and g not in groups[:i][nonempty[:i]]]
    assert ret.tolist() == first and 3 not in first and 8 not in first


def test_no_rows(vm):
    for P in (1, 40):
        got, ret = run(vm, "sum", np.zeros((0, P)), np.zeros(0, dtype=np.uint32), 3)
        assert np.isnan(got).all() and len(ret) == 0


# ------------------------------------------------------------------------------------------------ errors
def test_errors_leave_the_output_untouched(vm):
    import torch
    from victoriametrics_b200 import _lib
    lib, ctx = _lib.lib(), _lib.default_context()
    S, P = 8, 5
    dv = torch.ones(S * P, dtype=torch.float64, device="cuda")
    out = torch.full((S * P,), SENTINEL, dtype=torch.float64, device="cuda")
    flags = np.zeros(S, dtype=np.uint8)

    def call(func, nseries=S, points=P, groups=np.zeros(S, dtype=np.uint32), G=1):
        g = np.ascontiguousarray(groups, dtype=np.uint32)
        return lib.vmb_aggr_matrix(ctx.h, func, C.c_void_p(dv.data_ptr()), nseries, points, g.ctypes.data_as(_lib.u32p), G,
                                   C.c_void_p(out.data_ptr()), flags.ctypes.data_as(_lib.u8p))
    assert call(12) == -50 and call(-1) == -50
    assert call(0, G=0) == -50
    assert call(0, groups=np.array([0, 0, 0, 1, 0, 0, 0, 0]), G=1) == -50
    assert call(0, nseries=2 ** 31) == -50 and call(0, points=2 ** 31) == -50
    assert (out.cpu().numpy() == SENTINEL).all()
    assert call(0) == 0 and (out.cpu().numpy()[:P] == S).all()


def test_enum_follows_the_header(vm):
    pub = _enum(HDR, "vmb_matrix_aggr")
    assert {n[len("VMB_MA_"):].lower(): v for n, v in pub} == vm.promql.MATRIX_AGGR_FUNCS
