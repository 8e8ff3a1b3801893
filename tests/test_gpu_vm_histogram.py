"""vmb_aggr_histogram and vmb_rollup_histogram on the GPU, bit for bit against tests/vm_histogram_ref.py: every sample's bucket
(Go's math.Log10 restated), histogram(q) by (...) before and after its vmrangeBucketsToLE, histogram_over_time over the oracle's
windows, and histogram_quantile(0.99, sum(histogram_over_time(m[5m])) by (vmrange)) composed on the device."""
import ctypes as C
import struct
import threading

import numpy as np
import pytest

import count_values_ref as CV
import vm_histogram_ref as H
from aggr_matrix_ref import aggr_matrix_ref
from blockgen import OBlock, gen_timestamps, gen_values, to_blockset
from histogram_ref import histogram_ref
from vmrange_ref import go_parse_float, vmrange_to_le_ref

pytestmark = pytest.mark.gpu
NAN, INF = float("nan"), float("inf")
GO_NAN = 0x7FF8000000000001
STALE = struct.unpack("<d", struct.pack("<Q", CV.STALE_NAN_BITS))[0]


@pytest.fixture(scope="module")
def vm():
    import victoriametrics_b200 as v
    return v


class Buf:
    def __init__(self, nbytes):
        import torch
        self.t = torch.empty(max(nbytes // 8, 1), dtype=torch.float64, device="cuda")
        self.ptr = self.t.data_ptr()


def gpu_vmrange(vm, vals, gids, G, ctx=None):
    import torch
    vals = np.ascontiguousarray(vals, dtype=np.float64)
    S, P = vals.shape
    d = torch.from_numpy(vals).cuda()
    out, n, groups, buckets = vm.promql.aggr_histogram_vmrange(d.data_ptr(), S, P, np.asarray(gids), G, Buf, ctx=ctx)
    return out.t[:n * P].reshape(n, P).cpu().numpy(), groups.tolist(), buckets.tolist()


def check_vmrange(vm, vals, gids, G, what=""):
    got, groups, buckets = gpu_vmrange(vm, vals, gids, G)
    want, wg, wb = H.histogram_counts(vals, gids, G)
    assert groups == wg and buckets == wb, what
    assert got.view(np.uint64).tolist() == want.view(np.uint64).tolist(), what  # 0, not NaN, where none are


def buckets_of(vm, values):
    """every value's bucket through vmb_aggr_histogram: a [N x 1] matrix whose every row is its own group, -1 for none"""
    import torch
    v = np.ascontiguousarray(values, dtype=np.float64)
    N = v.size
    d = torch.from_numpy(v.reshape(N, 1)).cuda()
    out, n, groups, buckets = vm.promql.aggr_histogram_vmrange(d.data_ptr(), N, 1, np.arange(N), N, Buf)
    assert (out.t[:n].cpu().numpy() == 1).all()
    got = np.full(N, -1, dtype=np.int64)
    got[groups] = buckets
    return got


def test_every_edge_within_64_ulp(vm):
    cands = []
    v, m = 1e-9, 10 ** (1 / 18)
    for k in range(H.DECIMAL + 1):  # the 487 bounds as initBucketRanges reaches them, and the powers 10^(k/18 - 9)
        for e in {v, 10 ** (k / 18 - 9)}:
            u = H.bits(e)
            cands += [H.from_bits(u + d) for d in range(-64, 65)]
        v *= m
    cands = np.array(cands)
    want = [-1 if b is None else b for b in map(H.bucket, cands.tolist())]
    assert buckets_of(vm, cands).tolist() == want


def test_specials_and_log_uniform(vm):
    specials = [0.0, -0.0, 5e-324, 2.2250738585072009e-308, 2.2250738585072014e-308, INF, -INF, NAN, STALE, -1.0, -5e-324, 1e-9,
                1e18, 1.0, 123.0, 1.1, 1.15, 1.7976931348623157e308]
    got = buckets_of(vm, specials).tolist()
    assert got == [-1 if b is None else b for b in map(H.bucket, specials)]
    rng = np.random.default_rng(1)
    x = 10 ** rng.uniform(-12, 21, 1_000_000)
    assert np.array_equal(buckets_of(vm, x), H.bucket_np(x))


def mixed(rng, S, P, sigma=3.0):
    """log-normal values with 5 % NaN, 5 % negatives and 2 % zeros (+0.0 and -0.0)"""
    v = rng.lognormal(0.0, sigma, (S, P))
    r = rng.random((S, P))
    v[r < 0.05] = NAN
    v[(r >= 0.05) & (r < 0.10)] *= -1
    v[(r >= 0.10) & (r < 0.11)] = 0.0
    v[(r >= 0.11) & (r < 0.12)] = -0.0
    return v


@pytest.mark.parametrize("G", [1, 8, 1024, "S"])
def test_seeded(vm, G):
    rng = np.random.default_rng(7 if G == "S" else G)
    S, P = (1000, 64) if G == "S" else (4000, 300)
    G = S if G == "S" else G
    check_vmrange(vm, mixed(rng, S, P), rng.integers(0, G, S), G, "G %d" % G)


@pytest.mark.parametrize("G", [1, 8])
def test_latency_collisions(vm, G):
    """log-normal latencies: most of a group's rows share a few buckets at every point"""
    rng = np.random.default_rng(30 + G)
    S, P = 20000, 300
    check_vmrange(vm, rng.lognormal(np.log(0.05), 0.3, (S, P)), rng.integers(0, G, S), G, "latency G %d" % G)


def test_large_matrix(vm):
    """100 000 x 2048 with G = 8, checked chunk by chunk (the counts of disjoint row sets add up)"""
    import torch
    S, P, G = 100_000, 2048, 8
    rng = np.random.default_rng(41)
    gids = rng.integers(0, G, S)
    torch.manual_seed(41)
    d = torch.exp(torch.randn(S, P, dtype=torch.float64, device="cuda") * 2.0)
    u = torch.rand(S, P, device="cuda")
    d[u < 0.05] = NAN
    d[(u >= 0.05) & (u < 0.1)] *= -1
    out, n, groups, buckets = vm.promql.aggr_histogram_vmrange(d.data_ptr(), S, P, gids, G, Buf)
    got = out.t[:n * P].reshape(n, P).cpu().numpy()
    want = np.zeros((G * H.NB, P))
    for r0 in range(0, S, 5000):
        m, wg, wb = H.histogram_counts(d[r0:r0 + 5000].cpu().numpy(), gids[r0:r0 + 5000], G)
        want[np.array(wg) * H.NB + np.array(wb)] += m
    rows = np.flatnonzero(want.any(axis=1))
    assert groups.tolist() == (rows // H.NB).tolist() and buckets.tolist() == (rows % H.NB).tolist()
    assert np.array_equal(got, want[rows])


def test_nan_and_negative_groups(vm):
    vals = np.array([[NAN] * 5, [-1.0, -2.0, NAN, -INF, -5e-324], [1.0, 2.0, NAN, 0.0, INF], [NAN, -3.0, 4.0, NAN, NAN]])
    check_vmrange(vm, vals, [0, 1, 2, 2], 3, "NaN-only and negative-only groups")
    got, groups, _ = gpu_vmrange(vm, vals, [0, 1, 2, 2], 3)
    assert set(groups) == {2}
    got, groups, _ = gpu_vmrange(vm, vals[:2], [0, 0], 1)
    assert got.shape == (0, 5) and groups == []


def test_by_vmrange(vm):
    """histogram(q) by (vmrange) over rows that already carry a vmrange label: the host's groups are those labels"""
    rng = np.random.default_rng(8)
    vals = rng.lognormal(0, 1, (300, 40))
    labels = [H.LABELS[b] for b in rng.integers(100, 110, 300)]
    keys = sorted(set(labels))
    check_vmrange(vm, vals, [keys.index(x) for x in labels], len(keys), "by (vmrange)")


def test_le_output(vm):
    import torch
    rng = np.random.default_rng(9)
    for S, P, G in ((1, 6, 1), (200, 30, 4), (2000, 50, 16)):
        vals = mixed(rng, S, P, 1.5)
        if S == 1:
            vals[:] = 123.0
        gids = rng.integers(0, G, S)
        d = torch.from_numpy(vals).cuda()
        out, n, groups, les = vm.promql.aggr_histogram(d.data_ptr(), S, P, gids, G, Buf)
        got = out.t[:n * P].reshape(n, P).cpu().numpy()
        mat, wg, wb = H.histogram_counts(vals, gids, G)
        want = vmrange_to_le_ref(mat, [H.LABELS[b] for b in wb], [None] * len(wb), wg)
        assert groups.tolist() == [wg[w[0]] for w in want] and les == [w[2] for w in want]
        assert got.view(np.uint64).tolist() == np.array([w[3] for w in want]).reshape(n, P).view(np.uint64).tolist()


def test_cap_round_trip_and_errors(vm):
    import torch
    from victoriametrics_b200 import _lib
    lib, ctx = _lib.lib(), _lib.default_context()
    S, P = 4, 3
    dv = torch.tensor([[1, 2, 3], [1, 1, NAN], [4, -4, 4], [NAN] * 3], dtype=torch.float64, device="cuda")
    out = torch.full((16 * P,), 7.0, dtype=torch.float64, device="cuda")
    gids = np.array([0, 0, 1, 1], dtype=np.uint32)
    grp = np.full(16, 77, dtype=np.uint32)
    bkt = np.full(16, 77, dtype=np.uint32)
    u32 = lambda a: a.ctypes.data_as(_lib.u32p) if a is not None else None

    def hg(c=ctx.h, ptr=dv.data_ptr(), nseries=S, points=P, g=gids, ngroups=2, o=out.data_ptr(), cap=16, nout=True, og=grp, ob=bkt):
        n = C.c_size_t(cap)
        rc = lib.vmb_aggr_histogram(c, C.c_void_p(ptr), nseries, points, u32(g), ngroups, C.c_void_p(o) if o else None,
                                    C.byref(n) if nout else None, u32(og), u32(ob))
        return rc, n.value

    b = [H.bucket(x) for x in (1.0, 2.0, 3.0, 4.0)]
    assert hg(o=None) == (-54, 4)
    assert hg(cap=3) == (-54, 4)
    assert (grp == 77).all() and (bkt == 77).all() and (out.cpu() == 7).all()
    bad_g = gids.copy()
    bad_g[2] = 2
    for kw in (dict(c=None), dict(ngroups=0), dict(g=bad_g), dict(g=None), dict(nout=False), dict(og=None), dict(ob=None),
               dict(ptr=0), dict(nseries=1 << 31), dict(points=1 << 31)):
        assert hg(**kw)[0] == -50, kw
    assert (grp == 77).all() and (bkt == 77).all() and (out.cpu() == 7).all()
    assert hg() == (0, 4)
    assert grp[:4].tolist() == [0, 0, 0, 1] and bkt[:4].tolist() == [b[0], b[1], b[2], b[3]]
    assert out[:4 * P].cpu().tolist() == [2, 1, 0, 0, 1, 0, 0, 0, 1, 1, 0, 1]
    assert (out[4 * P:].cpu() == 7).all()
    assert hg(nseries=0) == (0, 0) and hg(points=0) == (0, 0)
    # vmb_rollup_histogram: the pointer checks, outputs untouched
    t = np.arange(0, 100_000, 10_000, dtype=np.int64)
    series = vm.storage.Series.from_host([t], [np.ones(t.size)])
    cfg = vm.promql.count_values_over_time_config(0, 90_000, 10_000, 30_000)
    ser = np.full(4, 77, dtype=np.uint32)
    for args in ((None, series.h, C.byref(cfg)), (ctx.h, None, C.byref(cfg)), (ctx.h, series.h, None)):
        n = C.c_size_t(4)
        assert lib.vmb_rollup_histogram(*args, C.c_void_p(out.data_ptr()), C.byref(n), u32(ser), u32(bkt), None) == -50
    n = C.c_size_t(4)
    assert lib.vmb_rollup_histogram(ctx.h, series.h, C.byref(cfg), C.c_void_p(out.data_ptr()), C.byref(n), None, u32(bkt), None) == -50
    bad = vm.promql.count_values_over_time_config(0, 90_000, 10_000, 30_000)
    bad.step = 0
    assert lib.vmb_rollup_histogram(ctx.h, series.h, C.byref(bad), C.c_void_p(out.data_ptr()), C.byref(n), u32(ser), u32(bkt),
                                    None) == -50
    assert (ser == 77).all() and (out[4 * P:].cpu() == 7).all()
    series.close()


# ---- histogram_over_time

def check_over_time(vm, series, ts_list, vals_list, start, end, step, window, lookback_delta=0, what=""):
    out, n, ser, vmranges, scanned = vm.promql.histogram_over_time(series, start, end, step, window, lookback_delta, Buf)
    P = 1 + (end - start) // step
    got = out.t[:n * P].reshape(n, P).cpu().numpy()
    want, want_scanned = [], 0
    for s, (t, v) in enumerate(zip(ts_list, vals_list)):
        m, sc = H.histogram_over_time(v, t, start, end, step, window, lookback_delta)
        want_scanned += sc
        want += [(s, b, m[b]) for b in sorted(m)]
    assert scanned == want_scanned, what
    assert ser.tolist() == [w[0] for w in want] and vmranges == [H.LABELS[w[1]] for w in want], what
    w = np.array([x[2] for x in want]).reshape(len(want), P)
    nan = np.isnan(w)
    assert np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan], w[~nan]), what
    assert (got[nan].view(np.uint64) == GO_NAN).all(), what
    return ser.tolist(), vmranges, got


def test_over_time_blocks(vm):
    rng = np.random.default_rng(11)
    blocks, ts_list, vals_list = [], [], []
    for s in range(24):
        n = int(rng.choice([1, 5, 300, 1000, 4097]))
        t = gen_timestamps(rng, str(rng.choice(["regular", "jitter", "irregular"])), n)
        v = gen_values(rng, "special" if s % 3 == 0 else "gauge_small", n)
        b = OBlock(t, v, int(rng.choice([0, -1, -4, 2])), series_idx=s)
        blocks.append(b)
        ts_list.append(t)
        vals_list.append(CV.O.decimal_to_float(v, b.scale))
    descs, payload = to_blockset(blocks)
    t0 = 1_700_000_000_000
    for start, end, step, window, lb in ((t0, t0 + 3_600_000, 15_000, 300_000, 0), (t0 + 60_000, t0 + 7_200_000, 60_000, 20_000, 0),
                                         (t0, t0 + 3_600_000, 30_000, 0, 45_000), (t0, t0 + 100 * 60_000, 60_000, 0, 0)):
        blk = vm.storage.Blocks(descs, payload)
        series, _ = vm.storage.decode_blocks(blk)
        check_over_time(vm, series, ts_list, vals_list, start, end, step, window, lb, "window %d step %d lb %d" % (window, step, lb))
        series.close()
        blk.close()


def test_over_time_multiblock_overlap(vm):
    rng = np.random.default_rng(12)
    t0 = 1_700_000_000_000
    blocks = []
    for s in range(6):
        t = gen_timestamps(rng, "jitter", 2000, t0)
        v = gen_values(rng, "gauge_small", 2000)
        parts = [(0, 1200), (800, 2000)] if s % 2 else [(0, 1000), (1000, 2000)]
        for a, b in parts:
            blocks.append(OBlock(t[a:b], v[a:b], -2, series_idx=s))
    descs, payload = to_blockset(blocks)
    blk = vm.storage.Blocks(descs, payload)
    series, _ = vm.storage.decode_blocks(blk)
    cols = series.to_lists()  # the rows as the library merged the overlapping blocks: the windows are what is checked here
    check_over_time(vm, series, [c[0] for c in cols], [c[1] for c in cols], t0, t0 + 2000 * 15_000, 45_000, 120_000, 0,
                    "multi-block")
    series.close()
    blk.close()


def test_over_time_host_specials_and_stale(vm):
    t = np.arange(0, 200_000, 10_000, dtype=np.int64)
    v = np.array([0.0, -0.0, NAN, STALE, 1.5, -0.0, 0.0, 0.0, NAN, 1.5, 2.0, STALE, -1e-7, 1e21, INF, -INF, 0.0, 1e-9, NAN, 3.0])
    v2 = np.full(t.size, -1.0)  # only negatives: no rows
    v3 = np.full(t.size, NAN)
    series = vm.storage.Series.from_host([t, t, t], [v, v2, v3])
    ser, vmranges, _ = check_over_time(vm, series, [t, t, t], [v, v2, v3], 20_000, 190_000, 20_000, 30_000, 0, "host")
    assert set(ser) == {0} and vmranges[0] == "0...1.000e-09" and vmranges[-1] == "1.000e+18...+Inf"
    series.close()


def test_over_time_subquery(vm):
    import torch
    rng = np.random.default_rng(13)
    start, end, step = 1_000_000, 2_000_000, 200_000
    sq_start, sq_step = start - 200_000, 5_000
    npts = 1 + (end - sq_start) // sq_step
    x = rng.lognormal(0, 2, (3, npts))
    x[1, ::7] = NAN
    x[2, ::5] = -1.0
    dx = torch.from_numpy(x).cuda()
    series = vm.storage.Series.from_matrix(dx.data_ptr(), 3, npts, sq_start, sq_step)
    ts = sq_start + sq_step * np.arange(npts, dtype=np.int64)
    check_over_time(vm, series, [ts[~np.isnan(r)] for r in x], [r[~np.isnan(r)] for r in x], start, end, step, 200_000, 0,
                    "subquery")
    series.close()


def test_quantile_of_summed_histogram_over_time(vm):
    """histogram_quantile(0.99, sum(histogram_over_time(m[5m])) by (vmrange)): vmb_rollup_histogram -> vmb_aggr_matrix SUM ->
    vmb_vmrange_to_le -> vmb_histogram, against the restatements composed the same way"""
    import torch
    rng = np.random.default_rng(17)
    S, n = 40, 600
    t0 = 1_700_000_000_000
    t = t0 + 15_000 * np.arange(n, dtype=np.int64)
    vals = [rng.lognormal(np.log(0.2), 0.5, n) for _ in range(S)]
    start, end, step, window = t0 + 300_000, t[-1], 60_000, 300_000
    P = 1 + (end - start) // step
    series = vm.storage.Series.from_host([t] * S, vals)
    out, nrow, ser, vmranges, _ = vm.promql.histogram_over_time(series, start, end, step, window, 0, Buf)
    keys = sorted(set(vmranges), key=lambda x: go_parse_float(x.split("...")[1]))
    gids = np.array([keys.index(x) for x in vmranges], dtype=np.uint32)
    summed = torch.empty(len(keys) * P, dtype=torch.float64, device="cuda")
    vm.promql.aggr_matrix("sum", out.ptr, nrow, P, summed.data_ptr(), gids, len(keys))
    le_out, nle, _, _, les = vm.promql.prometheus_buckets(summed.data_ptr(), len(keys), P, keys, [False] * len(keys),
                                                          [0] * len(keys), Buf)
    q = torch.empty(P, dtype=torch.float64, device="cuda")
    les_f = np.array([go_parse_float(x) for x in les])
    vm.promql.histogram("histogram_quantile", le_out.ptr, nle, P, np.zeros(nle, dtype=np.uint32), les_f, 1, q.data_ptr(), 0.99)
    # the restatements
    rows, rlabels = [], []
    for s in range(S):
        m, _ = H.histogram_over_time(vals[s], t, start, end, step, window)
        for b in sorted(m):
            rows.append(m[b])
            rlabels.append(H.LABELS[b])
    assert rlabels == vmranges
    rsum, _ = aggr_matrix_ref("sum", np.array(rows), gids, len(keys))
    le_rows = vmrange_to_le_ref(rsum, keys, [None] * len(keys), [0] * len(keys))
    assert [r[2] for r in le_rows] == les
    want = histogram_ref("histogram_quantile", np.array([r[3] for r in le_rows]), [0] * len(le_rows), les_f, 1, 0.99)[0]
    assert q.cpu().numpy().view(np.uint64).tolist() == want[0].view(np.uint64).tolist()
    series.close()


def test_determinism_stream_and_threads(vm):
    import torch
    from victoriametrics_b200 import _lib
    rng = np.random.default_rng(21)
    S, P = 3000, 50
    vals = rng.lognormal(0, 1, (S, P))
    gids = rng.integers(0, 16, S)
    t = np.arange(0, 3000 * 15_000, 15_000, dtype=np.int64)
    hv = [rng.lognormal(0, 1, t.size) for _ in range(40)]

    def run(ctx):
        a = gpu_vmrange(vm, vals, gids, 16, ctx)
        s = vm.storage.Series.from_host([t] * 40, hv, ctx)
        out, n, ser, vr, sc = vm.promql.histogram_over_time(s, 0, t[-1], 60_000, 300_000, 0, Buf, ctx=ctx)
        torch.cuda.synchronize()
        b = (out.t[:n * (1 + t[-1] // 60_000)].cpu().numpy(), ser.tolist(), vr, sc)
        s.close()
        return a, b

    def same(x, y):
        (a1, g1, b1), (o1, s1, v1, c1) = x
        (a2, g2, b2), (o2, s2, v2, c2) = y
        assert a1.view(np.uint64).tolist() == a2.view(np.uint64).tolist() and g1 == g2 and b1 == b2
        assert o1.view(np.uint64).tolist() == o2.view(np.uint64).tolist() and s1 == s2 and v1 == v2 and c1 == c2

    ref = run(_lib.default_context())
    same(ref, run(_lib.default_context()))
    stream = torch.cuda.Stream()
    ctx = _lib.Context(0, stream.cuda_stream)
    with torch.cuda.stream(stream):
        same(ref, run(ctx))
    ctx.close()
    results, errors = [None, None], []

    def worker(i):
        try:
            s = torch.cuda.Stream()
            c = _lib.Context(0, s.cuda_stream)
            with torch.cuda.stream(s):
                results[i] = run(c)
            c.close()
        except Exception as e:  # noqa: BLE001
            errors.append(e)
    ths = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    assert not errors, errors
    for r in results:
        same(ref, r)
