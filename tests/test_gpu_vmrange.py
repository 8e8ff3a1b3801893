"""vmb_vmrange_to_le / vmb_buckets_limit (promql.prometheus_buckets / promql.buckets_limit) bit for bit against
tests/vmrange_ref.py: the matrix, the row count, the source rows, the kinds and the `le` strings.  The reference's vectors at
P = 1 and P = 6; randomised groups of 1, 2, 12, 13, 40 and 300 shuffled VictoriaMetrics-style ranges (18 per decade, "%.3e",
with 0...1.000e-09 and ...+Inf) with zero rows, NaN cells, duplicate end strings and duplicate end floats, kept `le` rows and
dropped rows; merge chains taken and refused; the VMB_ERR_CAP round trip; buckets_limit at every limit edge, NaN hits, and its
composition with vmb_histogram; guard bands, the input untouched, determinism, more cells than one grid pass, a matrix past 2^31
elements and every error path; and the headline query histogram_quantile(0.99, sum(rate(...)) by (vmrange, job)) composed on
the device from reference-encoded blocks."""
import ctypes as C
import zlib

import numpy as np
import pytest

import blockgen
import vmrange_ref as V
from aggr_matrix_ref import aggr_matrix_ref
from conftest import SEED0
from histogram_ref import SKIP, histogram_ref
from test_gpu_rollup_exact import assert_same_bits, block_rows, oracle_rows
from test_vmrange_ref import LIMIT_USED, OVERLAPPED, OVERLAPPED_END, TRANSFORM_TEST, VALID, labelled, limit_inputs, prom_rows

pytestmark = pytest.mark.gpu
NAN, INF = float("nan"), float("inf")
SENTINEL = -7.25
GUARD = 33
T0, DT = 1_700_000_000_000, 15_000
CELLS_PER_PASS = 132 * 32 * 256  # k_vr_cumsum: VMB_SMS x 32 CTAs of 256 threads


def seed(name, k=0):
    return np.random.default_rng(SEED0 + zlib.crc32(("vmrange/%s/%d" % (name, k)).encode()))


@pytest.fixture(scope="module")
def vm():
    import victoriametrics_b200 as v
    return v


class Guarded:
    """device_alloc for prometheus_buckets: the output inside guard bands"""

    def __init__(self, nbytes):
        import torch
        self.n = nbytes // 8
        self.t = torch.full((self.n + 2 * GUARD,), SENTINEL, dtype=torch.float64, device="cuda")
        self.ptr = self.t.data_ptr() + 8 * GUARD

    def values(self, what="out"):
        b = self.t.cpu().numpy()
        assert (b[:GUARD] == SENTINEL).all() and (b[GUARD + self.n:] == SENTINEL).all(), "%s: guard band overwritten" % what
        return b[GUARD:GUARD + self.n]


def upload(m):
    import torch
    m = np.ascontiguousarray(m, dtype=np.float64)
    inp = Guarded(m.size * 8)
    inp.t[GUARD:GUARD + m.size] = torch.from_numpy(m.reshape(-1)).cuda()
    return inp


def run_pb(vm, m, vmranges, has_le, groups):
    """-> (matrix, n, src, kinds, les) from the device, the output inside guard bands, the input checked byte for byte"""
    m = np.ascontiguousarray(m, dtype=np.float64)
    S, P = m.shape
    inp = upload(m)
    out, n, src, kinds, les = vm.promql.prometheus_buckets(inp.ptr, S, P, vmranges, has_le, groups, Guarded)
    assert inp.values("input").tobytes() == m.tobytes(), "the bucket matrix was modified"
    got = out.values()
    if n * P == 0:
        return np.zeros((n, P)), n, src, kinds, les
    assert got.size == n * P
    return got.reshape(n, P), n, src, kinds, les


def check_pb(vm, m, vmranges, has_le, groups, what=""):
    got = run_pb(vm, m, vmranges, has_le, groups)
    mat, src, kinds, les = V.vmrange_to_le_arrays(m, vmranges, ["1" if h else None for h in has_le], groups)
    assert got[1] == len(src), (what, got[1], len(src))
    assert np.array_equal(got[2], src), (what, got[2], src)
    assert np.array_equal(got[3], kinds), (what, got[3], kinds)
    assert got[4] == les, (what, got[4], les)
    if len(src):
        assert_same_bits(got[0], mat, "prometheus_buckets " + what)
    return got


def rows_of(ss):
    """labelled series -> (matrix, vmranges, has_le, groups)"""
    keys = {}
    groups = [keys.setdefault(tuple(sorted((k, v) for k, v in l.items() if k not in ("vmrange", "le"))), len(keys))
              for _, l in ss]
    return (np.array([v for v, _ in ss]), [l.get("vmrange") for _, l in ss], [bool(l.get("le")) for _, l in ss], groups)


@pytest.mark.parametrize("P", [1, 6])
def test_reference_vectors(vm, P):
    for line, text, _ in TRANSFORM_TEST:
        rows = prom_rows(text)
        m = np.array([[v] * P for _, v in rows])
        check_pb(vm, m, [l.get("vmrange") for l, _ in rows], [bool(l.get("le")) for l, _ in rows], [0] * len(rows),
                 what="transform_test.go:%d" % line)
    missing = labelled((("t", 20), "xyz", "foo", "bar", "le", "0.2"), (("t", 100), "xxx", "foo", "bar", "vmrange", "foobar"),
                       (("t", 100), "xxx", "foo", "bar", "vmrange", "30...foobar"),
                       (("t", 100), "xxx", "foo", "bar", "vmrange", "30...40"),
                       (("t", 80), "yyy", "foo", "bar", "vmrange", "0...900", "le", "54"),
                       (("t", 40), "yyy", "foo", "bar", "vmrange", "900...+Inf", "le", "2343"))
    for name, items in (("missing", missing), ("valid", labelled(*VALID)), ("overlapped", labelled(*OVERLAPPED)),
                        ("overlapped end", labelled(*OVERLAPPED_END))):
        m, vr, le, g = rows_of(items)
        check_pb(vm, m[:, :P], vr, le, g, what=name)
    m, g, les, G = limit_inputs(labelled(*LIMIT_USED))
    for limit in (0, 2, 5):
        check_limit(vm, limit, m[:, :P], g, les, G)


# ------------------------------------------------------------------------------------------------ randomised groups
BOUNDS = ["%.3e" % (10 ** (e + k / 18)) for e in range(-9, 3) for k in range(18)]


def vm_ranges(rng, n):
    """n VictoriaMetrics-style ranges: adjacent bounds of the 18-per-decade grid, 0...1.000e-09, ...+Inf, duplicates of an end
    string and an end float spelled otherwise"""
    out = []
    for _ in range(n):
        u = rng.random()
        if u < 0.05:
            out.append("0...1.000e-09")
        elif u < 0.1:
            out.append("%s...+Inf" % BOUNDS[-1])
        elif u < 0.15 and out:  # a duplicate end string, another start
            end = out[int(rng.integers(len(out)))].split("...")[1]
            out.append("%s...%s" % (BOUNDS[int(rng.integers(len(BOUNDS)))], end))
        elif u < 0.2:  # the same end float, another spelling
            k = int(rng.integers(len(BOUNDS) - 1))
            out.append("%s...%r" % (BOUNDS[k], float(BOUNDS[k + 1])))
        else:
            k = int(rng.integers(len(BOUNDS) - 1))
            out.append("%s...%s" % (BOUNDS[k], BOUNDS[k + 1]))
    return out


def random_rows(rng, sizes, P, nkept=0, ndrop=0):
    """groups of the given sizes, shuffled together with kept `le` rows and dropped rows -> (m, vmranges, has_le, groups)"""
    vr, g = [], []
    for gi, n in enumerate(sizes):
        vr += vm_ranges(rng, n)
        g += [gi] * n
    S = len(vr)
    m = rng.exponential(3.0, (S, P)) * rng.choice([0.0, 1e-3, 1.0, 1e6], (S, 1), p=[0.2, 0.1, 0.6, 0.1])
    m[rng.random((S, P)) < 0.1] = NAN
    m[rng.random((S, P)) < 0.05] *= -1
    m[rng.random(S) < 0.05] = NAN
    has_le = [False] * S
    drops = ["foo...bar", "1.000e+00", "1.000e+00...x", " 1...2", None, ""]
    vr += [None] * nkept + [drops[k % len(drops)] for k in range(ndrop)]
    has_le += [True] * nkept + [False] * ndrop
    g += [int(rng.integers(max(len(sizes), 1)))] * (nkept + ndrop)
    m = np.concatenate([m, rng.normal(size=(nkept + ndrop, P))])
    perm = rng.permutation(len(vr))
    return (np.ascontiguousarray(m[perm]), [vr[i] for i in perm], [has_le[i] for i in perm], [g[i] for i in perm])


GROUP_SIZES = [1, 2, 12, 13, 40, 300]


@pytest.mark.parametrize("P", [1, 7, 64])
def test_random_groups(vm, P):
    rng = seed("random", P)
    m, vr, le, g = random_rows(rng, GROUP_SIZES * 2 + [3] * 5, P, nkept=7, ndrop=9)
    got = check_pb(vm, m, vr, le, g, what="P=%d" % P)
    assert set(got[3].tolist()) == {V.KEPT, V.BUCKET, V.GAP, V.PINF}


@pytest.mark.parametrize("P", [1, 2, 3, 7, 45, 64])
def test_merge_chains(vm, P):
    """groups whose rows share end strings, mostly NaN, so that merges are both taken and refused along each chain"""
    rng = seed("chains", P)
    vr, g, rows = [], [], []
    for gi in range(24):
        n = int(rng.integers(2, 9))
        ends = ["5", "5.0", "7"][: 1 + gi % 3]
        for k in range(n):
            vr.append("%d...%s" % (k % 4, ends[k % len(ends)]))
            g.append(gi)
            r = np.full(P, NAN)
            on = rng.random(P) < (0.9 if k == 0 else 2.5 / max(P, 1))
            r[on] = rng.integers(1, 9, int(on.sum()))
            if not on.any():
                r[int(rng.integers(P))] = 1.0
            rows.append(r)
    vr.append("3...3")  # a...a after a gap at a: merges into itself
    g.append(24)
    rows.append(np.full(P, 2.0))
    check_pb(vm, np.array(rows), vr, [False] * len(vr), g, what="chains P=%d" % P)


def test_cap_round_trip(vm):
    import torch
    from victoriametrics_b200 import _lib
    lib, ctx = _lib.lib(), _lib.default_context()
    m = np.array([[1.0, 2.0], [3.0, 0.0], [0.0, 0.0], [5.0, 5.0]])
    dv = torch.from_numpy(m.reshape(-1)).cuda()
    gids = np.array([0, 0, 0, V.KEEP], dtype=np.uint32)
    starts, ends = np.array([0.0, 1.0, 2.0, 0.0]), np.array([1.0, 2.0, 3.0, 0.0])
    skeys, ekeys = np.array([0, 1, 2, 0], dtype=np.uint32), np.array([1, 2, 3, 0], dtype=np.uint32)
    out = torch.full((16,), SENTINEL, dtype=torch.float64, device="cuda")
    src, le = np.full(8, 77, dtype=np.uint32), np.full(8, 77, dtype=np.uint32)
    kind = np.full(8, 77, dtype=np.uint8)
    u32 = lambda a: a.ctypes.data_as(_lib.u32p)

    def call(cap, optr):
        n = C.c_size_t(cap)
        rc = lib.vmb_vmrange_to_le(ctx.h, C.c_void_p(dv.data_ptr()), 4, 2, u32(gids), starts.ctypes.data_as(_lib.f64p),
                                   ends.ctypes.data_as(_lib.f64p), u32(skeys), u32(ekeys), 1, optr, C.byref(n), u32(src),
                                   kind.ctypes.data_as(_lib.u8p), u32(le))
        return rc, n.value
    assert call(100, None) == (-54, 4)  # kept, 0...1, 1...2, +Inf (2...3 is all zero)
    assert call(3, C.c_void_p(out.data_ptr())) == (-54, 4)
    assert (out.cpu().numpy() == SENTINEL).all() and (src == 77).all() and (kind == 77).all() and (le == 77).all()
    assert call(4, C.c_void_p(out.data_ptr())) == (0, 4)
    assert src[:4].tolist() == [3, 0, 1, 1] and kind[:4].tolist() == [V.KEPT, V.BUCKET, V.BUCKET, V.PINF]
    assert le[:4].tolist() == [0xFFFFFFFF, 1, 2, 0xFFFFFFFF] and (src[4:] == 77).all()
    assert out.cpu().numpy()[:8].tolist() == [5, 5, 1, 2, 4, 2, 4, 2] and (out.cpu().numpy()[8:] == SENTINEL).all()


def test_same_call_twice_same_bits(vm):
    rng = seed("twice")
    m, vr, le, g = random_rows(rng, GROUP_SIZES * 2, 300, nkept=3, ndrop=3)
    a, b = run_pb(vm, m, vr, le, g), run_pb(vm, m, vr, le, g)
    assert a[0].tobytes() == b[0].tobytes() and np.array_equal(a[2], b[2]) and a[4] == b[4]


def test_more_cells_than_one_grid_pass(vm):
    rng = seed("grid")
    P = 2000
    G = CELLS_PER_PASS // P + 60
    m, vr, le, g = random_rows(rng, [3] * G, P)
    check_pb(vm, m, vr, le, g, what="grid")


# ------------------------------------------------------------------------------------------------ buckets_limit
def check_limit(vm, limit, m, g, les, G):
    m = np.ascontiguousarray(m, dtype=np.float64)
    inp = upload(m)
    got = vm.promql.buckets_limit(limit, inp.ptr, m.shape[0], m.shape[1], g, les, G)
    assert inp.values("input").tobytes() == m.tobytes()
    want = V.buckets_limit_ref(limit, m, g, les, G)
    assert got.tolist() == want, (limit, got, want)
    return got


def le_matrix(rng, sizes, P):
    """prometheus_buckets of random groups through the restatement -> (le matrix, group ids, les, G)"""
    m, vr, le, g = random_rows(rng, sizes, P)
    mat, src, kinds, les = V.vmrange_to_le_arrays(m, vr, [None] * len(vr), g)
    gids = np.array([g[s] for s in src], dtype=np.uint32)
    lev = np.array([V.go_parse_float(x) for x in les])
    return mat, gids, lev, len(sizes)


@pytest.mark.parametrize("P", [1, 7, 64])
def test_buckets_limit(vm, P):
    rng = seed("limit", P)
    mat, gids, les, G = le_matrix(rng, GROUP_SIZES + [5, 4, 3], P)
    gids[rng.random(gids.size) < 0.03] = SKIP
    mat[rng.random(mat.shape) < 0.02] = NAN  # NaN hits
    for limit in (0, 1, 2, 3, 5, 10, 1000, -3):
        check_limit(vm, limit, mat, gids, les, G)


def test_buckets_limit_then_histogram(vm):
    """vmb_histogram over the whole matrix with UINT32_MAX for the rows buckets_limit drops == histogram over the kept rows"""
    import torch
    rng = seed("limit-histogram")
    P = 45
    mat, gids, les, G = le_matrix(rng, [40, 13, 300, 12], P)
    kept = check_limit(vm, 10, mat, gids, les, G)
    masked = np.full(gids.size, SKIP, dtype=np.uint32)
    masked[kept] = gids[kept]
    dv = torch.from_numpy(mat.reshape(-1)).cuda()
    q = torch.full((G, P), SENTINEL, dtype=torch.float64, device="cuda")
    ne = vm.promql.histogram("histogram_quantile", dv.data_ptr(), mat.shape[0], P, masked, les, G, q.data_ptr(), 0.99)
    want = histogram_ref("histogram_quantile", mat[kept], gids[kept], les[kept], G, 0.99)
    assert_same_bits(q.cpu().numpy(), want[0], "buckets_limit -> histogram_quantile")
    assert np.array_equal(ne, want[3])


def test_past_2_pow_31_elements(vm):
    """a matrix of 2^31 + 4096 values (16 GiB): groups at the start and past element 2^31; every other row is dropped.  The
    per-row arrays go to the C ABI directly (the Python wrapper would loop over 33 M labels)"""
    import torch
    from victoriametrics_b200 import _lib
    lib, ctx = _lib.lib(), _lib.default_context()
    P = 64
    S = (1 << 31) // P + 64
    rng = seed("2^31")
    small, vr, le, g = random_rows(rng, [6, 5], P, nkept=1)
    k = len(vr)
    rows = np.r_[0:k // 2, S - (k - k // 2):S]
    dv = torch.empty((S, P), dtype=torch.float64, device="cuda")
    dv[torch.from_numpy(rows).cuda()] = torch.from_numpy(small).cuda()
    gids = np.full(S, V.DROP, dtype=np.uint32)
    starts, ends = np.zeros(S), np.zeros(S)
    skeys, ekeys = np.zeros(S, dtype=np.uint32), np.zeros(S, dtype=np.uint32)
    ids = {}
    for i, r in enumerate(rows.tolist()):
        if not vr[i]:
            gids[r] = V.KEEP if le[i] else V.DROP
            continue
        a, _, b = vr[i].partition("...")
        fa, fb = V.go_parse_float(a), V.go_parse_float(b)
        if "..." in vr[i] and fa is not None and fb is not None:
            gids[r], starts[r], ends[r] = g[i], fa, fb
            skeys[r], ekeys[r] = ids.setdefault(a, len(ids)), ids.setdefault(b, len(ids))
    mat, wsrc, wkinds, wles = V.vmrange_to_le_arrays(small, vr, ["1" if h else None for h in le], g)
    n = len(wsrc)
    out = torch.full((n, P), SENTINEL, dtype=torch.float64, device="cuda")
    src, kind, lek = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint8), np.zeros(n, dtype=np.uint32)
    nout = C.c_size_t(n)
    u32 = lambda a: a.ctypes.data_as(_lib.u32p)
    assert lib.vmb_vmrange_to_le(ctx.h, C.c_void_p(dv.data_ptr()), S, P, u32(gids), starts.ctypes.data_as(_lib.f64p),
                                 ends.ctypes.data_as(_lib.f64p), u32(skeys), u32(ekeys), 2, C.c_void_p(out.data_ptr()),
                                 C.byref(nout), u32(src), kind.ctypes.data_as(_lib.u8p), u32(lek)) == 0
    names = {v: k for k, v in ids.items()}
    assert nout.value == n and np.array_equal(src, rows[wsrc]) and np.array_equal(kind, wkinds)
    assert [None if k == V.KEPT else "+Inf" if k == V.PINF else names[x] for k, x in zip(kind, lek)] == wles
    assert_same_bits(out.cpu().numpy(), mat, "past 2^31")
    gl = np.full(S, SKIP, dtype=np.uint32)
    lev = np.zeros(S)
    gl[rows], lev[rows] = np.array(g, dtype=np.uint32), rng.choice([1.0, 2.0, 5.0, INF], len(rows))
    got = vm.promql.buckets_limit(3, dv.data_ptr(), S, P, gl, lev, 2)
    assert got.tolist() == rows[V.buckets_limit_ref(3, small, np.array(g), lev[rows], 2)].tolist()
    del dv, out
    torch.cuda.empty_cache()


def test_errors_leave_the_outputs_untouched(vm):
    import torch
    from victoriametrics_b200 import _lib
    lib, ctx = _lib.lib(), _lib.default_context()
    S, P = 4, 3
    dv = torch.arange(S * P, dtype=torch.float64, device="cuda") + 1
    out = torch.full((8 * P,), SENTINEL, dtype=torch.float64, device="cuda")
    src, le, rows = (np.full(8, 77, dtype=np.uint32) for _ in range(3))
    kind = np.full(8, 77, dtype=np.uint8)
    gids = np.array([0, 0, V.KEEP, V.DROP], dtype=np.uint32)
    f = np.array([0.0, 1.0, 0.0, 0.0])
    keys = np.array([0, 1, 2, 3], dtype=np.uint32)
    u32 = lambda a: a.ctypes.data_as(_lib.u32p) if a is not None else None
    f64 = lambda a: a.ctypes.data_as(_lib.f64p) if a is not None else None

    def vr(c=ctx.h, ptr=None, nrows=S, points=P, g=gids, st=f, en=f, sk=keys, ek=keys, ngroups=1, cap=8, nout=True, s=src,
           k=kind, l=le):
        n = C.c_size_t(cap)
        return lib.vmb_vmrange_to_le(c, C.c_void_p(dv.data_ptr() if ptr is None else ptr), nrows, points, u32(g), f64(st),
                                     f64(en), u32(sk), u32(ek), ngroups, C.c_void_p(out.data_ptr()),
                                     C.byref(n) if nout else None, u32(s), k.ctypes.data_as(_lib.u8p) if k is not None else None,
                                     u32(l))

    def bl(c=ctx.h, ptr=None, nrows=S, points=P, g=np.array([0, 0, 1, SKIP], dtype=np.uint32), les=f, ngroups=2, limit=3,
           r=rows, nout=True):
        n = C.c_size_t(8)
        return lib.vmb_buckets_limit(c, C.c_void_p(dv.data_ptr() if ptr is None else ptr), nrows, points, u32(g), f64(les),
                                     ngroups, limit, u32(r), C.byref(n) if nout else None)
    for call in (vr, bl):
        assert call(c=None) == -50 and call(nout=False) == -50 and call(ptr=0) == -50
        assert call(nrows=2 ** 31) == -50 and call(points=2 ** 31) == -50
    assert vr(g=np.array([0, 1, V.KEEP, V.DROP], dtype=np.uint32)) == -50  # a group id >= ngroups
    for kw in ("g", "st", "en", "sk", "ek", "s", "k", "l"):
        assert vr(**{kw: None}) == -50, kw
    assert bl(g=np.array([0, 0, 2, SKIP], dtype=np.uint32)) == -50 and bl(g=None) == -50 and bl(les=None) == -50
    assert bl(r=None) == -50
    assert (out.cpu().numpy() == SENTINEL).all() and (src == 77).all() and (kind == 77).all() and (le == 77).all()
    assert (rows == 77).all()
    assert vr(nrows=0) == 0 and bl(nrows=0) == 0 and bl(limit=0) == 0  # no-ops
    assert (out.cpu().numpy() == SENTINEL).all() and (rows == 77).all()
    assert vr() == 0 and bl() == 0


# ------------------------------------------------------------------------------------------------ the headline composition
def client_blocks(rng, jobs, instances, rows=400):
    """m_bucket{vmrange, job, instance} as the VictoriaMetrics `metrics` client exports them: one counter per range, and only the
    ranges an instance has observed; a counter reset in a few series"""
    blocks, pair_of, ranges = [], [], {}
    ts = (T0 + DT * np.arange(rows)).astype(np.int64)
    grid = ["0...1.000e-09"] + ["%s...%s" % (BOUNDS[k], BOUNDS[k + 1]) for k in range(100, 160)] + \
           ["%s...+Inf" % BOUNDS[-1]]
    for j in range(jobs):
        for _ in range(instances):
            centre, width = rng.uniform(10, 50), rng.uniform(2, 8)
            idx = np.clip(np.round(rng.normal(centre, width, (rows, 30))).astype(int), 0, len(grid) - 1)
            for k in np.unique(idx):
                v = np.cumsum((idx == k).sum(axis=1)).astype(np.int64)
                if rng.random() < 0.1:
                    v[rows // 2:] -= v[rows // 2]
                blocks.append(blockgen.OBlock(ts, v, 0, 64, len(blocks)))
                pair_of.append(ranges.setdefault((j, grid[k]), len(ranges)))
    return blocks, np.array(pair_of, dtype=np.uint32), ranges


@pytest.mark.parametrize("limit", [None, 10])
def test_headline_composition(vm, oracle, limit):
    """histogram_quantile(0.99, sum(rate(m_bucket[5m])) by (vmrange, job)) [through buckets_limit(10, ...)] on the device:
    reference-encoded blocks -> rate() -> vmb_aggr_matrix sum by (vmrange, job) -> vmb_vmrange_to_le [-> vmb_buckets_limit]
    -> vmb_histogram, every step bit for bit against the oracle's rollup, aggr_matrix_ref, vmrange_ref and histogram_ref"""
    import torch
    rng = seed("headline", limit or 0)
    J, I = 5, 4
    blocks, pair, ranges = client_blocks(rng, J, I)
    S, GP = len(blocks), len(ranges)
    vr = [r for (_, r) in sorted(ranges, key=ranges.get)]
    job = [j for (j, _) in sorted(ranges, key=ranges.get)]
    rc = vm.promql.get_rollup_configs("rate", T0 + 300_000, T0 + DT * 399, 30_000, 300_000)
    P = rc.points
    rate_ref = oracle_rows(oracle, rc, block_rows(blocks))[0]
    sums_ref = aggr_matrix_ref("sum", rate_ref, pair, GP)[0]
    le_ref, src_ref, _, les_ref = V.vmrange_to_le_arrays(sums_ref, vr, [None] * GP, job)
    gid_ref = np.array([job[s] for s in src_ref], dtype=np.uint32)
    lev_ref = np.array([V.go_parse_float(x) for x in les_ref])
    if limit:
        kept = V.buckets_limit_ref(limit, le_ref, gid_ref, lev_ref, J)
        assert len(kept) < len(src_ref)
        want = histogram_ref("histogram_quantile", le_ref[kept], gid_ref[kept], lev_ref[kept], J, 0.99)
    else:
        want = histogram_ref("histogram_quantile", le_ref, gid_ref, lev_ref, J, 0.99)
    assert np.isfinite(want[0]).any()
    descs, payload = blockgen.to_blockset(blocks)
    ctx = vm.default_context()
    B = vm.storage.Blocks(descs, payload, ctx)
    try:
        rates = torch.empty((S, P), dtype=torch.float64, device="cuda")
        vm.promql.eval_rollup_func("rate", B, rc.Start, rc.End, rc.Step, rc.Window, out_dev_ptr=rates.data_ptr())
        assert_same_bits(rates.cpu().numpy(), rate_ref, "rate")
        sums = torch.empty((GP, P), dtype=torch.float64, device="cuda")
        vm.promql.aggr_matrix("sum", rates.data_ptr(), S, P, sums.data_ptr(), group_ids=pair, ngroups=GP)
        assert_same_bits(sums.cpu().numpy(), sums_ref, "sum by (vmrange, job)")

        def alloc(nbytes):
            b = type("B", (), {})()
            b.t = torch.empty(nbytes // 8, dtype=torch.float64, device="cuda")
            b.ptr = b.t.data_ptr()
            return b
        out, n, src, _, les = vm.promql.prometheus_buckets(sums.data_ptr(), GP, P, vr, [False] * GP, job, alloc)
        assert n == len(src_ref) and np.array_equal(src, src_ref) and les == les_ref
        assert_same_bits(out.t.cpu().numpy().reshape(n, P), le_ref, "prometheus_buckets")
        gids = np.array([job[s] for s in src], dtype=np.uint32)
        lev = np.array([vm.promql.go_parse_float(x) for x in les])
        if limit:
            kept = vm.promql.buckets_limit(limit, out.ptr, n, P, gids, lev, J)
            assert kept.tolist() == V.buckets_limit_ref(limit, le_ref, gid_ref, lev_ref, J)
            masked = np.full(n, SKIP, dtype=np.uint32)
            masked[kept] = gids[kept]
            gids = masked
        q = torch.full((J, P), SENTINEL, dtype=torch.float64, device="cuda")
        ne = vm.promql.histogram("histogram_quantile", out.ptr, n, P, gids, lev, J, q.data_ptr(), 0.99)
        assert_same_bits(q.cpu().numpy(), want[0], "-> histogram_quantile")
        assert np.array_equal(ne, want[3])
    finally:
        B.close()
