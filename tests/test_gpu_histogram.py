"""vmb_histogram / promql.histogram bit for bit against tests/histogram_ref.py: the exec_test.go vectors; randomised groups of 1, 2, 12,
13, 40 and 300 bucket rows (shuffled rows, duplicate / +-Inf / NaN / 0 / negative le, monotone and broken counts, NaN cells, all-NaN
and all-zero groups, rows without a group) for every function at every argument edge, with the bounds outputs; histogram_quantiles
against single-phi calls; P = 1, P < 32, P not a multiple of 32, more cells than one grid pass, a bucket matrix past 2^31 elements;
guard bands, the input untouched, determinism and every error path; and the headline query
histogram_quantile(0.99, sum(rate(...)) by (le, job)) composed on the device from reference-encoded blocks."""
import ctypes as C
import zlib

import numpy as np
import pytest

import blockgen
from conftest import SEED0
from histogram_ref import SKIP, histogram_ref
from aggr_matrix_ref import aggr_matrix_ref
from test_gpu_rollup_exact import assert_same_bits, block_rows, oracle_rows
from test_histogram_ref import EXEC_VECTORS, VALID, inputs

pytestmark = pytest.mark.gpu
NAN, INF = float("nan"), float("inf")
SENTINEL = -7.25
GUARD = 33
T0, DT = 1_700_000_000_000, 15_000
CELLS_PER_PASS = 132 * 32 * 256  # k_histogram: VMB_SMS x 32 CTAs of 256 threads
MOMENTS = ["histogram_avg", "histogram_stddev", "histogram_stdvar"]


def seed(name, k=0):
    return np.random.default_rng(SEED0 + zlib.crc32(("histogram/%s/%d" % (name, k)).encode()))


@pytest.fixture(scope="module")
def vm():
    import victoriametrics_b200 as v
    return v


def guarded(n, fill=SENTINEL):
    import torch
    return torch.full((n + 2 * GUARD,), fill, dtype=torch.float64, device="cuda")


def unguard(buf, n, what):
    b = buf.cpu().numpy()
    assert (b[:GUARD] == SENTINEL).all() and (b[GUARD + n:] == SENTINEL).all(), "%s: guard band overwritten" % what
    return b[GUARD:GUARD + n]


def nphi_of(name, args):
    return len(args) if name == "histogram_quantiles" else 1


def run(vm, name, m, gids, les, G, *args, bounds=False):
    """-> (out, lower, upper, nonempty) from the device, every output inside guard bands, the input checked byte for byte"""
    import torch
    m = np.ascontiguousarray(m, dtype=np.float64)
    S, P = m.shape
    inp = guarded(S * P)
    inp[GUARD:GUARD + S * P] = torch.from_numpy(m.reshape(-1)).cuda()
    no = nphi_of(name, args) * G * P
    out, lo, up = guarded(no), guarded(G * P), guarded(G * P)
    kw = dict(lower_dev_ptr=lo.data_ptr() + 8 * GUARD, upper_dev_ptr=up.data_ptr() + 8 * GUARD) if bounds else {}
    ne = vm.promql.histogram(name, inp.data_ptr() + 8 * GUARD, S, P, gids, les, G, out.data_ptr() + 8 * GUARD, *args, **kw)
    torch.cuda.synchronize()
    assert unguard(inp, S * P, "input").tobytes() == m.tobytes(), "the bucket matrix was modified"
    got = unguard(out, no, "out").reshape((-1, G, P) if name == "histogram_quantiles" else (G, P))
    glo, gup = unguard(lo, G * P, "lower"), unguard(up, G * P, "upper")
    if not bounds:
        assert (glo == SENTINEL).all() and (gup == SENTINEL).all()
        return got, None, None, ne
    return got, glo.reshape(G, P), gup.reshape(G, P), ne


def check(vm, name, m, gids, les, G, *args, bounds=False, what=""):
    got = run(vm, name, m, gids, les, G, *args, bounds=bounds)
    want = histogram_ref(name, m, gids, les, G, *args, bounds=bounds)
    what = "%s %s" % (name, what)
    assert_same_bits(got[0], want[0], what)
    if bounds:
        assert_same_bits(got[1], want[1], what + " lower")
        assert_same_bits(got[2], want[2], what + " upper")
    assert np.array_equal(got[3], want[3]), (what, got[3], want[3])
    return got


def test_exec_test_vectors(vm):
    for name, ss, args, _ in EXEC_VECTORS:
        m, g, le, G = inputs(ss)
        if G:
            check(vm, name, m, g, le, G, *args, what=str(args))
    m, g, le, G = inputs(VALID)
    for name, args in (("histogram_quantile", (0.6,)), ("histogram_share", (25,)), ("histogram_fraction", (0, 25))):
        check(vm, name, m, g, le, G, *args, bounds=name != "histogram_fraction", what="two groups")
    got = run(vm, "histogram_quantile", m, g, le, G, 0.6)[0]
    assert sorted(got[:, 0].tolist()) == [9, 30]


LE_POOL = np.array([-INF, -2.5, -1.0, -0.0, 0.0, 0.1, 0.25, 0.5, 1.0, 1.0, 2.5, 5.0, 10.0, 10.0, 60.0, INF, INF, NAN])


def buckets(rng, sizes, P, nskip=0):
    """groups of the given sizes -> (matrix, group ids, les, G).  Per group one of: monotone counts in le order, broken (noisy)
    counts, NaN cells, all NaN, all zero, small integer counts with ties, negative counts; rows shuffled across all groups, plus
    nskip rows without a group"""
    rows, gids, les = [], [], []
    for g, n in enumerate(sizes):
        le = rng.choice(LE_POOL, n) if n <= 16 else np.r_[rng.choice(LE_POOL, n // 4), rng.integers(-5, 200, n - n // 4) / 4.0]
        order = np.argsort(np.nan_to_num(le, nan=np.inf), kind="stable")
        kind = g % 7
        inc = rng.exponential(50.0, (n, P)) * rng.choice([1e-3, 1.0, 1e6], (n, 1))
        if kind == 5:
            inc = rng.integers(0, 3, (n, P)).astype(np.float64)
        cnt = np.empty((n, P))
        cnt[order] = np.cumsum(inc[order], axis=0)
        if kind == 1:
            cnt += rng.normal(0, 80.0, (n, P))
        elif kind == 2:
            cnt[rng.random((n, P)) < 0.2] = NAN
        elif kind == 3:
            cnt[:] = NAN
        elif kind == 4:
            cnt[:] = 0.0
        elif kind == 6:
            cnt -= cnt.mean()
        rows.append(cnt)
        gids += [g] * n
        les.append(le)
    m, gids, les = np.concatenate(rows), np.array(gids, dtype=np.uint32), np.concatenate(les)
    m = np.concatenate([m, rng.normal(size=(nskip, P))])
    gids = np.r_[gids, np.full(nskip, SKIP, dtype=np.uint32)]
    les = np.r_[les, rng.choice(LE_POOL, nskip)]
    perm = rng.permutation(len(gids))
    return np.ascontiguousarray(m[perm]), gids[perm], les[perm], len(sizes)


def edge_args(rng, m, les, P):
    """per-point arguments at every edge: phi NaN, < 0, 0, 1, > 1 and inside; share le NaN, < 0, +Inf, exactly on a bucket bound;
    fraction bounds from the same pool"""
    phis = np.r_[NAN, -0.5, 0.0, 1.0, 1.5, 0.5, 0.99, 0.01, rng.random(max(P - 8, 0))][:P]
    finite = les[np.isfinite(les)]
    pool = np.r_[NAN, -1.0, -0.0, 0.0, INF, -INF, finite, rng.uniform(-1, 70, 8)]
    share = rng.choice(pool, P)
    share[:min(P, 6)] = [NAN, -1.0, INF, 0.0, finite[0] if finite.size else 1.0, 30.0][:min(P, 6)]
    lower, upper = rng.choice(pool, P), rng.choice(pool, P)
    return phis, share, lower, upper


GROUP_SIZES = [1, 2, 12, 13, 40, 300]


@pytest.mark.parametrize("P", [1, 7, 45, 64])
def test_random_groups_every_function(vm, P):
    rng = seed("random", P)
    sizes = GROUP_SIZES * 2 + [3] * 9
    m, g, le, G = buckets(rng, sizes, P, nskip=11)
    phis, share, lower, upper = edge_args(rng, m, le, P)
    check(vm, "histogram_quantile", m, g, le, G, phis, bounds=True, what="P=%d" % P)
    check(vm, "histogram_quantile", m, g, le, G, phis, what="P=%d no bounds" % P)
    check(vm, "histogram_quantiles", m, g, le, G, phis, 0.5, np.roll(phis, 3), what="P=%d" % P)
    check(vm, "histogram_share", m, g, le, G, share, bounds=True, what="P=%d" % P)
    check(vm, "histogram_fraction", m, g, le, G, lower, upper, what="P=%d" % P)
    for name in MOMENTS:
        check(vm, name, m, g, le, G, what="P=%d" % P)


def test_scalar_edges_one_group(vm):
    """one group of buckets le 1, 2, 5, +Inf with each scalar edge as a constant argument"""
    m = np.array([[10.0, 0, 3], [30.0, 0, 3], [60.0, 0, 3], [80.0, 0, 3]])
    g, le = np.zeros(4, dtype=np.uint32), np.array([1.0, 2.0, 5.0, INF])
    for phi in (NAN, -0.5, 0.0, 0.125, 0.375, 0.75, 1.0, 1.5, -INF, INF):
        check(vm, "histogram_quantile", m, g, le, 1, phi, bounds=True, what="phi=%r" % phi)
    for x in (NAN, -1.0, -0.0, 0.0, 1.0, 1.5, 2.0, 5.0, 7.0, INF, -INF):
        check(vm, "histogram_share", m, g, le, 1, x, bounds=True, what="le=%r" % x)
        for y in (NAN, 0.5, 2.0, 6.0, INF):
            check(vm, "histogram_fraction", m, g, le, 1, x, y, what="(%r, %r)" % (x, y))


@pytest.mark.parametrize("nphi", [1, 3, 8])
def test_quantiles_equal_single_phi_calls(vm, nphi):
    rng = seed("quantiles", nphi)
    P = 45
    m, g, le, G = buckets(rng, GROUP_SIZES + [5] * 6, P, nskip=4)
    phis = [edge_args(rng, m, le, P)[0] if k % 2 == 0 else rng.random(P) for k in range(nphi)]
    many = check(vm, "histogram_quantiles", m, g, le, G, *phis, what="%d phis" % nphi)
    for k, phi in enumerate(phis):
        one = run(vm, "histogram_quantile", m, g, le, G, phi)
        assert many[0][k].tobytes() == one[0].tobytes(), k
        assert np.array_equal(many[3][k * G:(k + 1) * G], one[3]), k


def test_more_cells_than_one_grid_pass(vm):
    rng = seed("grid")
    P = 2000
    G = CELLS_PER_PASS // P + 60
    m, g, le, G = buckets(rng, [3] * G, P)
    assert G * P > CELLS_PER_PASS
    phis, share, _, _ = edge_args(rng, m, le, P)
    check(vm, "histogram_quantile", m, g, le, G, phis, bounds=True, what="grid")
    check(vm, "histogram_share", m, g, le, G, share, what="grid")
    check(vm, "histogram_stdvar", m, g, le, G, what="grid")


def test_past_2_pow_31_elements(vm):
    """a bucket matrix of 2^31 + 4096 values (16 GiB): groups at the start and past element 2^31; every other row has no group"""
    import torch
    P = 64
    S = (1 << 31) // P + 64
    rng = seed("2^31")
    small, gs, ls, G = buckets(rng, [4, 5, 6, 3], P)
    rows = np.r_[0:9, S - 9:S]  # the last rows lie wholly past element 2^31
    gids = np.full(S, SKIP, dtype=np.uint32)
    les = np.zeros(S)
    gids[rows], les[rows] = gs, ls
    dv = torch.empty((S, P), dtype=torch.float64, device="cuda")
    dv[torch.from_numpy(rows).cuda()] = torch.from_numpy(small).cuda()
    phis = edge_args(rng, small, ls, P)[0]
    for name, args in (("histogram_quantile", (phis,)), ("histogram_avg", ())):
        out = torch.full((G, P), SENTINEL, dtype=torch.float64, device="cuda")
        ne = vm.promql.histogram(name, dv.data_ptr(), S, P, gids, les, G, out.data_ptr(), *args)
        want = histogram_ref(name, small, gs, ls, G, *args)
        assert_same_bits(out.cpu().numpy(), want[0], "%s past 2^31" % name)
        assert np.array_equal(ne, want[3])
    del dv
    torch.cuda.empty_cache()


def test_same_call_twice_same_bits(vm):
    rng = seed("twice")
    m, g, le, G = buckets(rng, GROUP_SIZES * 3, 300)
    phis, share, lower, upper = edge_args(rng, m, le, 300)
    for name, args in (("histogram_quantile", (phis,)), ("histogram_share", (share,)), ("histogram_fraction", (lower, upper)),
                       ("histogram_stddev", ())):
        a, b = run(vm, name, m, g, le, G, *args), run(vm, name, m, g, le, G, *args)
        assert a[0].tobytes() == b[0].tobytes() and np.array_equal(a[3], b[3]), name


def test_groups_without_rows_are_nan(vm):
    m = np.array([[1.0, 2.0], [3.0, 4.0]])
    for g in ([SKIP, SKIP], [2, 2]):
        got = check(vm, "histogram_quantile", m, np.array(g, dtype=np.uint32), np.array([1.0, 2.0]), 3, 0.5, bounds=True)
        assert np.isnan(got[0][:2]).all() and not got[3][:2].any()


def test_errors_leave_the_outputs_untouched(vm):
    import torch
    from victoriametrics_b200 import _lib
    lib, ctx = _lib.lib(), _lib.default_context()
    S, P, G = 6, 5, 2
    dv = torch.arange(S * P, dtype=torch.float64, device="cuda")
    out, lo, up = (torch.full((4 * G * P,), SENTINEL, dtype=torch.float64, device="cuda") for _ in range(3))
    flags = np.full(4 * G + 2 * G, 7, dtype=np.uint8)
    gids = np.array([0, 0, 1, 1, SKIP, 1], dtype=np.uint32)
    les = np.array([1.0, 2.0, 1.0, 2.0, NAN, INF])

    def hg(func, nargs=0, args=True, nrows=S, points=P, ngroups=G, bounds=False, lower=None, upper=None, g=gids, le=les,
           ptr=None, optr=None, fl=True):
        a = np.full(max(nargs, 1), 0.5)
        lp = lo.data_ptr() if bounds else lower
        upp = up.data_ptr() if bounds else upper
        return lib.vmb_histogram(ctx.h, func, C.c_void_p(dv.data_ptr() if ptr is None else ptr), nrows, points,
                                 g.ctypes.data_as(_lib.u32p) if g is not None else None,
                                 le.ctypes.data_as(_lib.f64p) if le is not None else None, ngroups,
                                 a.ctypes.data_as(_lib.f64p) if args else None, nargs,
                                 C.c_void_p(out.data_ptr() if optr is None else optr), C.c_void_p(lp) if lp else None,
                                 C.c_void_p(upp) if upp else None, flags.ctypes.data_as(_lib.u8p) if fl else None)
    assert hg(6) == -50 and hg(-1) == -50                                          # unknown function
    for func, bad in ((0, (0, P - 1, P + 1, 2 * P - 1)), (1, (0, P - 1, 2 * P)), (2, (P, 2 * P + 1)), (3, (P,)), (4, (1,)), (5, (P,))):
        for n in bad:
            assert hg(func, n) == -50, (func, n)                                   # wrong nargs
    assert hg(2, 2 * P, bounds=True) == -50 and hg(3, bounds=True) == -50          # bounds on a function without them
    assert hg(0, 2 * P, bounds=True) == -50                                        # ... and on histogram_quantiles
    assert hg(0, P, lower=lo.data_ptr()) == -50 and hg(1, P, upper=up.data_ptr()) == -50  # one bound without the other
    assert hg(0, P, args=False) == -50                                             # missing pointers
    assert hg(0, P, ptr=0) == -50 and hg(0, P, optr=0) == -50 and hg(0, P, fl=False) == -50
    assert hg(0, P, g=None) == -50 and hg(0, P, le=None) == -50
    assert hg(3, g=np.array([0, 0, 2, 1, SKIP, 1], dtype=np.uint32)) == -50       # a group id >= ngroups
    assert hg(3, nrows=2 ** 31) == -50 and hg(3, points=2 ** 31) == -50
    for t in (out, lo, up):
        assert (t.cpu().numpy() == SENTINEL).all()
    assert (flags == 7).all()
    assert hg(0, P, nrows=0) == 0 and hg(0, 0, points=0) == 0 and hg(0, P, ngroups=0) == 0  # no-ops
    for t in (out, lo, up):
        assert (t.cpu().numpy() == SENTINEL).all()
    assert (flags == 7).all()
    assert hg(0, P, bounds=True) == 0 and not (out.cpu().numpy()[:G * P] == SENTINEL).any()


# ------------------------------------------------------------------------------------------------ the headline composition
class Buf:
    def __init__(self, nbytes):
        import torch
        self.t = torch.zeros(max(nbytes // 8, 1), dtype=torch.float64, device="cuda")
        self.ptr = self.t.data_ptr()


LES = [0.005, 0.01, 0.025, 0.05, 0.1, 0.25, 0.5, 1.0, 2.5, INF]


def latency_blocks(rng, jobs, instances, rows=400):
    """http_request_duration_seconds_bucket{le, job, instance}: per instance counters whose bucket le_k counts the observations
    up to le_k (cumulative over the bins, then over time), one counter reset in a few series"""
    blocks, le_of, pair_of = [], [], []  # pair = (job, le) index: the `sum by (le, job)` group
    ts = (T0 + DT * np.arange(rows)).astype(np.int64)
    for j in range(jobs):
        for _ in range(instances):
            bins = rng.integers(0, 40, (rows, len(LES))) * (rng.random((1, len(LES))) < 0.9)
            cum = np.cumsum(np.cumsum(bins, axis=1), axis=0).astype(np.int64)
            for k in range(len(LES)):
                v = cum[:, k].copy()
                if rng.random() < 0.1:
                    v[rows // 2:] -= v[rows // 2]
                blocks.append(blockgen.OBlock(ts, v, 0, 64, len(blocks)))
                le_of.append(LES[k])
                pair_of.append(j * len(LES) + k)
    return blocks, np.array(pair_of, dtype=np.uint32)


def test_headline_composition(vm, oracle):
    """histogram_quantile(0.99, sum(rate(http_request_duration_seconds_bucket[5m])) by (le, job)) on the device:
    reference-encoded blocks -> rate() -> vmb_aggr_matrix sum by (le, job) -> vmb_histogram, bit for bit against the oracle's
    rollup, aggr_matrix_ref and histogram_ref; then the same buckets through the incremental aggregate (whose fused fold adds
    atomically) finalized in place -> vmb_histogram, bit for bit against histogram_ref of that matrix and within 1e-12 of the oracle"""
    import torch
    rng = seed("headline")
    J, I = 6, 4
    blocks, pair = latency_blocks(rng, J, I)
    S, GP = len(blocks), J * len(LES)
    hist_gids = (np.arange(GP) // len(LES)).astype(np.uint32)
    hist_les = np.array(LES * J)
    rc = vm.promql.get_rollup_configs("rate", T0 + 300_000, T0 + DT * 399, 30_000, 300_000)
    P = rc.points
    rate_ref = oracle_rows(oracle, rc, block_rows(blocks))[0]
    sums_ref = aggr_matrix_ref("sum", rate_ref, pair, GP)[0]
    want = histogram_ref("histogram_quantile", sums_ref, hist_gids, hist_les, J, 0.99)
    assert np.isfinite(want[0]).any()
    descs, payload = blockgen.to_blockset(blocks)
    ctx = vm.default_context()
    B = vm.storage.Blocks(descs, payload, ctx)
    try:
        rates = torch.empty((S, P), dtype=torch.float64, device="cuda")
        vm.promql.eval_rollup_func("rate", B, rc.Start, rc.End, rc.Step, rc.Window, out_dev_ptr=rates.data_ptr())
        sums = torch.empty((GP, P), dtype=torch.float64, device="cuda")
        vm.promql.aggr_matrix("sum", rates.data_ptr(), S, P, sums.data_ptr(), group_ids=pair, ngroups=GP)
        q = torch.full((J, P), SENTINEL, dtype=torch.float64, device="cuda")
        ne = vm.promql.histogram("histogram_quantile", sums.data_ptr(), GP, P, hist_gids, hist_les, J, q.data_ptr(), 0.99)
        assert_same_bits(q.cpu().numpy(), want[0], "rate -> sum by (le, job) -> histogram_quantile")
        assert np.array_equal(ne, want[3])

        ia = vm.promql.IncrementalAggr("sum", GP, P, Buf)
        ia.update_blocks(B, rc, pair)
        host = ia.finalize(ctx)  # vmb_aggr_finalize in place on ia.values, then a copy
        q2 = torch.full((J, P), SENTINEL, dtype=torch.float64, device="cuda")
        ne2 = vm.promql.histogram("histogram_quantile", ia.values.ptr, GP, P, hist_gids, hist_les, J, q2.data_ptr(), 0.99)
        got2 = q2.cpu().numpy()
        want2 = histogram_ref("histogram_quantile", host, hist_gids, hist_les, J, 0.99)
        assert_same_bits(got2, want2[0], "incremental sum -> histogram_quantile")
        assert np.array_equal(ne2, want2[3])
        assert np.array_equal(np.isnan(got2), np.isnan(want[0]))
        fin = ~np.isnan(got2)
        assert np.allclose(got2[fin], want[0][fin], rtol=1e-12, atol=0)
    finally:
        B.close()
