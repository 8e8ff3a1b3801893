"""vmb_aggr_rank / promql.aggr_rank bit for bit against tests/rank_aggr_ref.py: the exec_test.go vectors, randomised differentials
over all eleven functions and group layouts, ties and NaN scores in groups on both sides of 12 rows, every kind of k, the
remaining-sum rows, shapes at the edges of the walk and of the row sort, the rows that must stay as they were, every error path,
and the call on a caller's stream and from two host threads.  The rule is assert_same_bits (-0.0 != +0.0) for the matrix, the
remaining sums and the scores, except the sign of a zero topk_median / bottomk_median score where a tied rank holds both -0.0 and
+0.0 (EXCEPTIONS["quantile"] of test_gpu_matrix_exact: the reference's sort is not stable there); the order of the rows does not
depend on that sign."""
import ctypes as C
import threading
import zlib

import numpy as np
import pytest

from conftest import SEED0
from rank_aggr_ref import NAMES, rank_aggr_ref
from test_enum_tables import HDR, _enum
from test_gpu_matrix_exact import EXCEPTIONS
from test_gpu_rollup_exact import assert_same_bits

pytestmark = pytest.mark.gpu
NAN, INF = float("nan"), float("inf")
SENTINEL = -7.25
GUARD = 33
T = np.arange(1000, 2001, 200, dtype=np.float64)


def seed(name, k=0):
    return np.random.default_rng(SEED0 + zlib.crc32(("rank_aggr/%s/%d" % (name, k)).encode()))


@pytest.fixture(scope="module")
def vm():
    import victoriametrics_b200 as v
    return v


def run(vm, name, ks, vals, groups=None, G=1, remaining=False, limit=0, ctx=None):
    """-> dict like rank_aggr_ref's (masked, remaining, out, scores); checks the guard bands around the remaining-sum rows"""
    import torch
    dv = torch.from_numpy(np.ascontiguousarray(vals, dtype=np.float64)).cuda()
    S, P = dv.shape
    buf = torch.full((G * P + 2 * GUARD,), SENTINEL, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()  # the context may run on another stream than torch's
    out, scores = vm.promql.aggr_rank(name, ks, dv.data_ptr(), S, P, groups, G, buf.data_ptr() + 8 * GUARD if remaining else None,
                                      limit, ctx=ctx)
    torch.cuda.synchronize()
    b = buf.cpu().numpy()
    assert (b[:GUARD] == SENTINEL).all() and (b[GUARD + G * P:] == SENTINEL).all(), "guard band overwritten"
    if not remaining:
        assert (b == SENTINEL).all()
    return dict(masked=dv.cpu().numpy(), remaining=b[GUARD:GUARD + G * P].reshape(G, P) if remaining else None, out=out, scores=scores)


def same(got, want, name, what):
    assert EXCEPTIONS["quantile"][0] == "zero sign"
    assert_same_bits(got["scores"], want["scores"], "%s scores %s" % (name, what), "quantile_over_time" if "median" in name else None)
    assert np.array_equal(got["out"], want["out"]), (name, what, got["out"][:20], want["out"][:20])
    assert_same_bits(got["masked"], want["masked"], "%s matrix %s" % (name, what))
    if want["remaining"] is not None:
        assert_same_bits(got["remaining"], want["remaining"], "%s remaining sum %s" % (name, what))


def check(vm, name, ks, vals, groups=None, G=1, remaining=False, limit=0, what=""):
    remaining = remaining and name != "outliersk"
    got = run(vm, name, ks, vals, groups, G, remaining, limit)
    want = rank_aggr_ref(name, ks, vals, groups, G, remaining, limit)
    same(got, want, name, what)
    return [(got["remaining"][-x - 1] if x < 0 else got["masked"][x]).tolist() for x in got["out"]]


def check_all(vm, ks, vals, groups=None, G=1, what="", names=NAMES):
    for name in names:
        for remaining in (False, True):
            check(vm, name, ks, vals, groups, G, remaining, what=what)


# ------------------------------------------------------------------------------------------------ exec_test.go vectors
def test_exec_test_vectors(vm):
    ten, t150 = [10.0] * 6, (T / 150).tolist()
    two = np.array([np.full(6, 10.0), T / 150])
    for name, want in (("topk_min", ten), ("bottomk_min", t150), ("topk_max", t150), ("bottomk_max", ten), ("topk_avg", t150),
                       ("bottomk_avg", t150), ("topk_median", t150), ("topk_last", t150)):
        assert check(vm, name, 1, two) == [want], name
    for name in ("bottomk_median", "bottomk_last"):
        assert check(vm, name, 1, np.array([np.full(6, 10.0), T / 15])) == [ten], name
    assert check(vm, "topk_max", 1, two, remaining=True) == [ten, t150]
    assert check(vm, "topk_max", 2, two, remaining=True) == [t150, ten]
    assert check(vm, "topk_max", 3, two, remaining=True) == [t150, ten]
    assert check(vm, "outliersk", 0, np.array([np.full(6, 1300.0), T])) == []
    assert check(vm, "outliersk", 1, np.array([np.full(6, 2000.0), T])) == [T.tolist()]
    assert check(vm, "outliersk", 3, np.array([np.full(6, 1300.0), T])) == [T.tolist(), [1300.0] * 6]


# ------------------------------------------------------------------------------------------------ randomised differentials
def matrix(rng, S, P, ties=False):
    """normals over many scales (distinct scores), or small integers (tied scores); -0.0 / +0.0, +-Inf, NaN cells, NaN rows"""
    if ties:
        m = rng.integers(-2, 3, (S, P)).astype(np.float64)
    else:
        m = rng.normal(size=(S, P)) * 10.0 ** rng.integers(-3, 4, (S, P))
    m[rng.random((S, P)) < 0.1] = NAN
    sel = rng.random((S, P)) < 0.03
    m[sel] = rng.choice(np.array([INF, -INF, 0.0, -0.0]), int(sel.sum()))
    m[rng.random(S) < 0.08] = NAN  # rows without a value
    return m


def some_ks(rng, P):
    return rng.choice(np.array([0.0, 1.0, 2.0, 2.9, 3.0, 5.0, -1.0, NAN, 7.5, 1000.0, INF, 1e300]), P)


@pytest.mark.parametrize("P", [1, 7, 33, 100])
@pytest.mark.parametrize("kind", ["one", "eight", "singletons"])
def test_random_differential(vm, kind, P):
    S = 200
    for ties in (False, True):
        rng = seed("%s/%d/%d" % (kind, P, ties))
        vals = matrix(rng, S, P, ties)
        if kind == "one":
            groups, G = None, 1
        elif kind == "eight":
            groups, G = rng.integers(0, 8, S).astype(np.uint32), 9  # group 8 has no rows
        else:
            groups, G = rng.permutation(S).astype(np.uint32), S
        check_all(vm, 3, vals, groups, G, what="%s P=%d ties=%d k=3" % (kind, P, ties))
        check_all(vm, some_ks(rng, P), vals, groups, G, what="%s P=%d ties=%d" % (kind, P, ties))


def test_1024_groups(vm):
    rng = seed("1024")
    S, P, G = 5000, 40, 1024
    vals = matrix(rng, S, P)
    groups = rng.integers(0, G, S).astype(np.uint32)
    check_all(vm, some_ks(rng, P), vals, groups, G, what="1024 groups", names=["topk_avg", "bottomk_median", "topk_last", "outliersk"])


def test_ties_and_nan_scores(vm):
    """equal scores, -0.0 against +0.0 and several NaN scores (avg of +Inf and -Inf; outliersk of a row with a NaN), in groups of
    up to 12 rows and above: the stable order over ascending rows decides"""
    rng = seed("ties")
    for n in (2, 5, 12, 13, 40, 300):
        P = 6
        vals = rng.integers(0, 2, (n, P)).astype(np.float64)
        vals[::5] = 0.0
        vals[1::5] = -0.0
        vals[2::7, 0], vals[2::7, 1] = INF, -INF  # avg and median NaN, min -Inf, max +Inf
        vals[3::7, 2] = NAN
        groups = (np.arange(n) % 2).astype(np.uint32) if n > 12 else None
        for k in (1, 3, n):
            check_all(vm, k, vals, groups, 2 if n > 12 else 1, what="ties n=%d k=%d" % (n, k))


def test_groups_above_12_rows_distinct_scores(vm):
    rng = seed("distinct")
    S, P = 900, 50
    vals = rng.normal(size=(S, P)).cumsum(axis=1)
    groups = rng.integers(0, 3, S).astype(np.uint32)
    check_all(vm, 5, vals, groups, 3, what="distinct")


def test_every_kind_of_k(vm):
    rng = seed("ks")
    S, P = 30, 12
    vals = matrix(rng, S, P)
    groups = rng.integers(0, 2, S).astype(np.uint32)
    for ks in (2, 0, -3, NAN, 2.99, 1000, INF, -INF, 1e300,
               np.array([0, 1, 2, 3, NAN, -1, 0.5, 1.5, INF, 1e300, 30, 31], dtype=np.float64)):
        check_all(vm, ks, vals, groups, 2, what="ks %r" % (ks,))


def test_candidate_left_empty_by_the_mask(vm):
    """row 1 is the best by max but holds its only value where k is 0; row 0 survives at the other points"""
    vals = np.array([[1.0, 2.0, 3.0, NAN], [NAN, NAN, NAN, 9.0], [0.5, 0.5, 0.5, 0.5]])
    ks = np.array([2.0, 2.0, 2.0, 0.0])
    got = run(vm, "topk_max", ks, vals, remaining=True)
    want = rank_aggr_ref("topk_max", ks, vals, remaining=True)
    same(got, want, "topk_max", "emptied candidate")
    assert got["out"].tolist() == [-1, 0] and got["masked"][1, 3] == 9.0
    assert got["remaining"][0].tolist() == [0.5, 0.5, 0.5, 9.5]


def test_remaining_sum_nan_at_some_and_at_all_points(vm):
    vals = np.array([[1.0, 2.0, 3.0], [4.0, NAN, 6.0], [NAN, NAN, 9.0], [-0.0, NAN, NAN]])
    groups = np.array([0, 0, 0, 1], dtype=np.uint32)
    got = run(vm, "topk_last", np.array([1.0, 1.0, 3.0]), vals, groups, 3, remaining=True)
    same(got, rank_aggr_ref("topk_last", np.array([1.0, 1.0, 3.0]), vals, groups, 3, True), "topk_last", "remaining NaN")
    rem = got["remaining"]
    assert rem[0, 0] == 5.0 and rem[0, 1] == 2.0 and np.isnan(rem[0, 2])  # NaN at one point
    assert np.isnan(rem[1:]).all() and got["out"].tolist() == [-1, 2, 1, 0, 3]  # group 1: nothing remains; group 2: no rows
    got = run(vm, "bottomk_min", 0, vals, groups, 3, remaining=True)       # k = 0: everything remains; 0 + -0.0 is +0.0
    same(got, rank_aggr_ref("bottomk_min", 0, vals, groups, 3, True), "bottomk_min", "k = 0")
    assert got["out"].tolist() == [-1, -2] and not np.signbit(got["remaining"][1, 0])


def test_rows_that_do_not_survive_keep_their_bits(vm):
    """k = 2 of 400 rows per group: the other rows, the empty ones included, are the bytes they were (NaN payloads too)"""
    rng = seed("untouched")
    S, P = 1200, 70
    vals = matrix(rng, S, P)
    vals.view(np.uint64)[np.isnan(vals)] = 0x7FF8_0000_0000_BEEF  # a payload the library never writes
    groups = (np.arange(S) % 3).astype(np.uint32)
    for name in ("topk_avg", "bottomk_median", "outliersk"):
        got = run(vm, name, 2, vals, groups, 3)
        rows = got["out"][got["out"] >= 0]
        assert len(rows) == 6
        others = np.setdiff1d(np.arange(S), rows)
        assert got["masked"][others].tobytes() == vals[others].tobytes(), name


def test_limit(vm):
    rng = seed("limit")
    S, P = 60, 9
    vals = matrix(rng, S, P)
    groups = rng.integers(0, 6, S).astype(np.uint32)
    vals[groups == 2] = NAN  # group 2 has rows, none with a value
    for limit in (0, 1, 3, 100):
        for name in ("topk_min", "outliersk"):
            got = run(vm, name, 2, vals, groups, 7, remaining=name != "outliersk", limit=limit)
            want = rank_aggr_ref(name, 2, vals, groups, 7, name != "outliersk", limit)
            assert np.array_equal(got["out"], want["out"]), (name, limit)


# ------------------------------------------------------------------------------------------------ shapes
def test_rows_past_the_grid_of_the_walk(vm):
    """more rows than one sweep of the score walk covers (132 SMs x 16 CTAs x 128 rows): the grid-stride loop runs twice"""
    rng = seed("grid")
    S, P = 132 * 16 * 128 + 77, 3
    vals = rng.normal(size=(S, P))
    vals[rng.random((S, P)) < 0.2] = NAN
    groups = (np.arange(S) % 2).astype(np.uint32)
    for name in ("topk_avg", "bottomk_last", "topk_min", "outliersk"):
        check(vm, name, np.array([4.0, 2.0, 7.0]), vals, groups, 2, remaining=True, what="grid")


def test_two_row_batches_of_the_median(vm):
    """more keys than one batch of the row sort holds (2^27): a full batch and a shorter last one; scores checked on rows on both
    sides of the boundary, and the output against a stable ranking of the scores the call returned"""
    import torch
    S, P = 20_000, 8172
    B = (1 << 27) // P
    assert B < S
    gen = torch.Generator("cuda").manual_seed(SEED0 + 21)
    dv = torch.randint(-50, 51, (S, P), dtype=torch.float64, device="cuda", generator=gen)
    dv[torch.rand(S, P, device="cuda", generator=gen) < 0.05] = NAN
    rows = np.r_[0:3, B - 3:B + 3, S - 3:S]
    host = dv[rows].cpu().numpy()
    out, scores = vm.promql.aggr_rank("topk_median", 4, dv.data_ptr(), S, P)
    want = rank_aggr_ref("topk_median", 4, host)["scores"]
    assert_same_bits(scores[rows], want, "median batches", "quantile_over_time")
    order = np.lexsort((scores, ~np.isnan(scores)))[::-1]  # worst to best, stable; then best first
    assert out.tolist() == order[:4].tolist()
    keep = [i for i, r in enumerate(rows.tolist()) if r not in out.tolist()]
    assert dv[rows[keep]].cpu().numpy().tobytes() == host[keep].tobytes()
    del dv
    torch.cuda.empty_cache()


def test_no_rows_and_no_points(vm):
    out, scores = vm.promql.aggr_rank("topk_avg", 1, 0, 0, 5, np.zeros(0, dtype=np.uint32), 3)
    assert len(out) == 0 and len(scores) == 0
    import torch
    dv = torch.zeros(4, dtype=torch.float64, device="cuda")
    out, _ = vm.promql.aggr_rank("topk_avg", 1, dv.data_ptr(), 4, 0, np.zeros(4, dtype=np.uint32), 1)
    assert len(out) == 0


# ------------------------------------------------------------------------------------------------ errors
def test_errors_leave_everything_untouched(vm):
    import torch
    from victoriametrics_b200 import _lib
    lib, ctx = _lib.lib(), _lib.default_context()
    S, P, G = 8, 5, 2
    dv = torch.arange(S * P, dtype=torch.float64, device="cuda")
    before = dv.cpu().numpy().copy()
    rem = torch.full((G * P,), SENTINEL, dtype=torch.float64, device="cuda")
    rne, ne = np.full(G, 7, dtype=np.uint8), np.full(S, 7, dtype=np.uint8)
    rows, counts, scores = np.full(S, 7, dtype=np.uint32), np.full(G, 7, dtype=np.uint32), np.full(S, SENTINEL)
    ks = np.ones(P)
    u8, u32 = (lambda a: a.ctypes.data_as(_lib.u8p)), (lambda a: a.ctypes.data_as(_lib.u32p))

    def call(func, reverse=0, nseries=S, points=P, groups=np.zeros(S, dtype=np.uint32), ngroups=G, k=True, r=True, rn=True, n=True,
             o=True, c=True):
        g = np.ascontiguousarray(groups, dtype=np.uint32)
        return lib.vmb_aggr_rank(ctx.h, func, reverse, C.c_void_p(dv.data_ptr()), nseries, points, u32(g), ngroups,
                                 ks.ctypes.data_as(_lib.f64p) if k else None, C.c_void_p(rem.data_ptr() if r else 0),
                                 u8(rne) if rn else None, u8(ne) if n else None, u32(rows) if o else None,
                                 u32(counts) if c else None, scores.ctypes.data_as(_lib.f64p))
    assert call(6) == -50 and call(-1) == -50
    assert call(0, ngroups=0) == -50
    assert call(0, groups=np.array([0, 0, 0, 2, 0, 0, 0, 0])) == -50
    assert call(0, nseries=2 ** 31) == -50 and call(0, points=2 ** 31) == -50
    assert call(0, k=False) == -50 and call(0, rn=False) == -50 and call(0, n=False) == -50
    assert call(0, o=False) == -50 and call(0, c=False) == -50
    assert call(5, reverse=1, r=False) == -50 and call(5) == -50  # outliersk: neither bottomk nor a remaining sum
    assert dv.cpu().numpy().tobytes() == before.tobytes() and (rem.cpu().numpy() == SENTINEL).all()
    assert (rne == 7).all() and (ne == 7).all() and (rows == 7).all() and (counts == 7).all() and (scores == SENTINEL).all()
    assert call(5, r=False) == 0 and call(0) == 0 and (ne == 1).all() and counts.tolist() == [1, 0] and rne.tolist() == [1, 0]


def test_enum_follows_the_header(vm):
    pub = _enum(HDR, "vmb_rank_func")
    assert {n[len("VMB_RK_"):].lower(): v for n, v in pub} == vm.promql.RANK_FUNCS


# ------------------------------------------------------------------------------------------------ streams and threads
def _catalogue(vm, ctx, vals, groups, G, ks):
    res = {}
    for name in ("topk_avg", "bottomk_median", "topk_max", "outliersk"):
        got = run(vm, name, ks, vals, groups, G, remaining=name != "outliersk", ctx=ctx)
        res[name] = b"".join(np.ascontiguousarray(got[f]).tobytes() for f in ("masked", "out", "scores")) + \
            (got["remaining"].tobytes() if got["remaining"] is not None else b"")
    return res


def test_caller_stream_and_two_threads_equal_the_serial_run(vm):
    """the entry point on a context bound to a caller's non-blocking stream, and from two host threads with a context each, started
    together: the same bytes as the default context's serial run"""
    import torch
    rng = seed("threads")
    S, P, G = 6000, 300, 5
    vals = matrix(rng, S, P)
    groups = rng.integers(0, G, S).astype(np.uint32)
    ks = some_ks(rng, P)
    serial = _catalogue(vm, None, vals, groups, G, ks)
    stream = torch.cuda.Stream()
    ctx = vm.Context(0, stream=stream.cuda_stream)
    try:
        assert _catalogue(vm, ctx, vals, groups, G, ks) == serial
    finally:
        ctx.close()
    barrier = threading.Barrier(2)
    results, errors = [None, None], []

    def worker(i):
        c = None
        try:
            s = torch.cuda.Stream()
            c = vm.Context(0, stream=s.cuda_stream)
            barrier.wait(timeout=120)
            results[i] = _catalogue(vm, c, vals, groups, G, ks)
        except BaseException as e:  # noqa: BLE001 -- reported below
            errors.append("thread %d: %r" % (i, e))
            barrier.abort()
        finally:
            if c is not None:
                c.close()
    ts = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    assert not any(t.is_alive() for t in ts) and not errors, errors
    assert results[0] == serial and results[1] == serial
