"""vmb_count_values and vmb_rollup_count_values on the GPU, bit for bit (labels included) against tests/count_values_ref.py: the
restatement of aggr.go's count_values loop, and the string-keyed loop of count_values_over_time over the oracle's windows."""
import ctypes as C
import struct
import threading

import numpy as np
import pytest

import count_values_ref as R
from blockgen import OBlock, gen_timestamps, gen_values, to_blockset

pytestmark = pytest.mark.gpu
NAN, INF = float("nan"), float("inf")
GO_NAN = 0x7FF8000000000001
STALE = struct.unpack("<d", struct.pack("<Q", R.STALE_NAN_BITS))[0]


@pytest.fixture(scope="module")
def vm():
    import victoriametrics_b200 as v
    return v


class Buf:
    def __init__(self, nbytes):
        import torch
        self.t = torch.empty(max(nbytes // 8, 1), dtype=torch.float64, device="cuda")
        self.ptr = self.t.data_ptr()


def assert_counts(got, want, what):
    """equal counts, NaN exactly where the reference has none, and those NaNs Go's bits"""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, what
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), what
    assert np.array_equal(got[~nan], want[~nan]), what
    assert (got[nan].view(np.uint64) == GO_NAN).all(), what


def gpu_count_values(vm, vals, gids, G, ctx=None):
    import torch
    vals = np.ascontiguousarray(vals, dtype=np.float64)
    S, P = vals.shape
    d = torch.from_numpy(vals).cuda()
    out, n, groups, tags = vm.promql.count_values("x", d.data_ptr(), S, P, np.asarray(gids, dtype=np.uint32), G, Buf, ctx=ctx)
    return out.t[:n * P].reshape(n, P).cpu().numpy(), groups.tolist(), [t[1] for t in tags]


def check_count_values(vm, vals, gids, G, what=""):
    vals = np.asarray(vals, dtype=np.float64)
    got, groups, labels = gpu_count_values(vm, vals, gids, G)
    ref = R.count_values(vals, gids, G)
    want = [(g, v, c) for g in sorted(ref) for v, c in sorted(ref[g], key=lambda x: x[0])]
    assert groups == [w[0] for w in want], what
    assert labels == [vm.promql.go_format_float(w[1], "f") for w in want], what
    assert_counts(got, np.array([w[2] for w in want]).reshape(len(want), vals.shape[1]), what)
    return got, groups, labels


TS = np.arange(1000, 2001, 200, dtype=np.float64)


def test_exec_test_vectors(vm):
    check_count_values(vm, [np.full(6, 10.0), TS / 100], [0, 0], 1, "count_values")
    check_count_values(vm, [np.full(6, 772424014.0), np.full(6, 772424230.0)], [0, 0], 1, "big numbers")
    _, _, labels = check_count_values(vm, [np.full(6, 10.0), np.floor(TS / 600)], [0, 0], 1, "by (xxx)")
    assert labels == ["1", "2", "3", "10"]
    check_count_values(vm, [np.floor(TS / 600)], [0], 1, "without (baz)")


@pytest.mark.parametrize("card", [16, 4096])
@pytest.mark.parametrize("G", [1, 8, 1024, "S"])
def test_seeded(vm, card, G):
    rng = np.random.default_rng(card * 7 + (0 if G == "S" else G))
    S, P = 2048, 40
    G = S if G == "S" else G
    vals = rng.integers(0, card, (S, P)).astype(np.float64) * 0.25 - 3
    vals[rng.random((S, P)) < 0.1] = NAN
    gids = rng.integers(0, G, S)
    check_count_values(vm, vals, gids, G, "card %d G %d" % (card, G))


def test_nan_rows_groups_zeros_and_infs(vm):
    P = 7
    vals = np.full((6, P), NAN)
    vals[1] = [0.0, -0.0, 1, INF, -INF, NAN, 0.0]      # group 0: +0.0 met first
    vals[2] = [-0.0, -0.0, 0.0, 2, INF, INF, -INF]
    vals[3] = [NAN, -0.0, 0.0, 5, 5, 5, 5]               # group 1: -0.0 met first (row 3, point 1)
    vals[4] = [0.0, NAN, NAN, NAN, NAN, NAN, NAN]        # a later row's +0.0 at an earlier point does not count
    gids = [0, 0, 0, 1, 1, 2]                            # row 0 (all NaN) in group 0, group 2 only NaN
    got, groups, labels = check_count_values(vm, vals, gids, 4)
    assert groups == [0] * 5 + [1] * 2 and labels == ["-Inf", "0", "1", "2", "+Inf", "-0", "5"]


def test_many_point_batches(vm):
    """S x P past the 2^27-key batch: the batch edge falls inside the matrix (numpy counts instead of the dict loop)"""
    import torch
    rng = np.random.default_rng(5)
    S, P = 1 << 17, 1030
    vals = torch.randint(0, 4, (S, P), dtype=torch.int64, device="cuda").double()
    vals[torch.rand(S, P, device="cuda") < 0.05] = NAN
    vals[0, 0] = -0.0
    rows = torch.from_numpy(rng.integers(0, S, 1000)).cuda()
    vals[rows, 1023] = -0.0
    out, n, groups, tags = vm.promql.count_values("x", vals.data_ptr(), S, P, np.zeros(S, dtype=np.uint32), 1, Buf)
    assert n == 4 and groups.tolist() == [0] * 4 and [t[1] for t in tags] == ["-0", "1", "2", "3"]
    got = out.t[:n * P].reshape(n, P)
    for k in range(4):
        want = (vals == k).sum(0).double()
        want[want == 0] = NAN
        assert_counts(got[k].cpu().numpy(), want.cpu().numpy(), "value %d" % k)


def test_cap_round_trip_and_errors(vm):
    import torch
    from victoriametrics_b200 import _lib
    lib, ctx = _lib.lib(), _lib.default_context()
    S, P = 4, 3
    dv = torch.tensor([[1, 2, 3], [1, 1, NAN], [4, 4, 4], [NAN] * 3], dtype=torch.float64, device="cuda")
    out = torch.full((16 * P,), 7.0, dtype=torch.float64, device="cuda")
    gids = np.array([0, 0, 1, 1], dtype=np.uint32)
    grp = np.full(16, 77, dtype=np.uint32)
    val = np.full(16, 77.0)
    u32 = lambda a: a.ctypes.data_as(_lib.u32p) if a is not None else None

    def cv(c=ctx.h, ptr=dv.data_ptr(), nseries=S, points=P, g=gids, ngroups=2, o=out.data_ptr(), cap=16, nout=True, og=grp,
           ov=val):
        n = C.c_size_t(cap)
        rc = lib.vmb_count_values(c, C.c_void_p(ptr), nseries, points, u32(g), ngroups, C.c_void_p(o) if o else None,
                                  C.byref(n) if nout else None, u32(og), ov.ctypes.data_as(_lib.f64p) if ov is not None else None)
        return rc, n.value

    assert cv(o=None) == (-54, 4)
    assert cv(cap=3) == (-54, 4)
    assert (grp == 77).all() and (val == 77).all() and (out.cpu() == 7).all()
    bad_g = gids.copy()
    bad_g[2] = 2
    for kw in (dict(c=None), dict(ngroups=0), dict(g=bad_g), dict(g=None), dict(nout=False), dict(og=None), dict(ov=None),
               dict(ptr=0), dict(nseries=1 << 31), dict(points=1 << 31)):
        assert cv(**kw)[0] == -50, kw
    assert (grp == 77).all() and (val == 77).all() and (out.cpu() == 7).all()
    assert cv() == (0, 4)
    assert grp[:4].tolist() == [0, 0, 0, 1] and val[:4].tolist() == [1, 2, 3, 4]
    assert (out[4 * P:].cpu() == 7).all()


# ---- count_values_over_time

def ref_over_time(vm, ts_list, vals_list, start, end, step, window, lookback_delta=0):
    rows, scanned = [], 0
    for s, (t, v) in enumerate(zip(ts_list, vals_list)):
        m, sc = R.count_values_over_time(v, t, start, end, step, window, lookback_delta)
        scanned += sc
        rows += [(s, k, m[k]) for k in m]
    return rows, scanned


def check_over_time(vm, series, ts_list, vals_list, start, end, step, window, lookback_delta=0, what=""):
    out, n, ser, tags, scanned = vm.promql.count_values_over_time("foo", series, start, end, step, window, lookback_delta, Buf)
    P = 1 + (end - start) // step
    got = out.t[:n * P].reshape(n, P).cpu().numpy()
    rows, want_scanned = ref_over_time(vm, ts_list, vals_list, start, end, step, window, lookback_delta)
    assert scanned == want_scanned, what
    want = {(s, k): c for s, k, c in rows}
    labels = [t[1] for t in tags]
    assert len(set(zip(ser.tolist(), labels))) == n == len(want), what
    assert ser.tolist() == sorted(ser.tolist()), what
    for i, key in enumerate(zip(ser.tolist(), labels)):
        assert_counts(got[i], want[key], "%s %s" % (what, key))
    return ser.tolist(), labels, got


def test_over_time_blocks(vm):
    rng = np.random.default_rng(11)
    blocks, ts_list, vals_list = [], [], []
    for s in range(24):
        n = int(rng.choice([1, 5, 300, 1000, 4097]))
        t = gen_timestamps(rng, str(rng.choice(["regular", "jitter", "irregular"])), n)
        v = gen_values(rng, "special" if s % 3 == 0 else "gauge_small", n)
        b = OBlock(t, v, int(rng.choice([0, -1, 2])), series_idx=s)
        blocks.append(b)
        ts_list.append(t)
        vals_list.append(R.O.decimal_to_float(v, b.scale))
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
    blocks, ts_list, vals_list = [], [], []
    for s in range(6):
        t = gen_timestamps(rng, "jitter", 2000, t0)
        v = gen_values(rng, "gauge_small", 2000)
        parts = [(0, 1200), (800, 2000)] if s % 2 else [(0, 1000), (1000, 2000)]  # overlapping / disjoint blocks
        for a, b in parts:
            blocks.append(OBlock(t[a:b], v[a:b], 0, series_idx=s))
        ts_list.append(t)
        vals_list.append(v.astype(np.float64))
    descs, payload = to_blockset(blocks)
    blk = vm.storage.Blocks(descs, payload)
    series, _ = vm.storage.decode_blocks(blk)
    # the rows as the library merged the overlapping blocks (the merge has tests of its own): the windows are what is checked here
    cols = series.to_lists()
    check_over_time(vm, series, [c[0] for c in cols], [c[1] for c in cols], t0, t0 + 2000 * 15_000, 45_000, 120_000, 0,
                    "multi-block")
    series.close()
    blk.close()


def test_over_time_host_signs_nans_stale(vm):
    t = np.arange(0, 200_000, 10_000, dtype=np.int64)
    v = np.array([0.0, -0.0, NAN, STALE, 1.5, -0.0, 0.0, 0.0, NAN, 1.5, 2.0, STALE, -1e-7, 1e21, INF, -INF, 0.0, -0.0, NAN, 3.0])
    v2 = np.full(t.size, -0.0)
    series = vm.storage.Series.from_host([t, t], [v, v2])
    ser, labels, _ = check_over_time(vm, series, [t, t], [v, v2], 20_000, 190_000, 20_000, 30_000, 0, "host")
    # the last point is 180 s: the 3.0 at 190 s lies in no window and makes no row
    assert labels[:ser.count(0)] == ["-Inf", "-1e-07", "-0", "0", "1.5", "2", "1e+21", "+Inf", "NaN"]
    series.close()


def test_over_time_subquery(vm):
    """the subquery feed: round(x, 0.4)[200s:5s] with a seeded x, the shape of exec_test.go:6066"""
    import torch
    rng = np.random.default_rng(13)
    start, end, step = 1_000_000, 2_000_000, 200_000
    sq_start, sq_step = start - 200_000, 5_000
    npts = 1 + (end - sq_start) // sq_step
    x = np.round(rng.random((3, npts)) / 0.4) * 0.4
    x[1, ::7] = NAN
    dx = torch.from_numpy(x).cuda()
    series = vm.storage.Series.from_matrix(dx.data_ptr(), 3, npts, sq_start, sq_step)
    ts = sq_start + sq_step * np.arange(npts, dtype=np.int64)
    ts_list = [ts[~np.isnan(r)] for r in x]
    vals_list = [r[~np.isnan(r)] for r in x]
    _, labels, _ = check_over_time(vm, series, ts_list, vals_list, start, end, step, 200_000, 0, "subquery")
    assert set(labels) <= {"0", "0.4", "0.8", "1.2000000000000002"}
    series.close()


def test_determinism_stream_and_threads(vm):
    import torch
    from victoriametrics_b200 import _lib
    rng = np.random.default_rng(21)
    S, P = 3000, 50
    vals = rng.integers(0, 300, (S, P)).astype(np.float64)
    gids = rng.integers(0, 16, S)
    t = np.arange(0, 3000 * 15_000, 15_000, dtype=np.int64)
    hv = [rng.integers(0, 9, t.size).astype(np.float64) for _ in range(40)]

    def run(ctx):
        a = gpu_count_values(vm, vals, gids, 16, ctx)
        s = vm.storage.Series.from_host([t] * 40, hv, ctx)
        out, n, ser, tags, sc = vm.promql.count_values_over_time("foo", s, 0, t[-1], 60_000, 300_000, 0, Buf, ctx=ctx)
        torch.cuda.synchronize()
        b = (out.t[:n * (1 + t[-1] // 60_000)].cpu().numpy(), ser.tolist(), tags, sc)
        s.close()
        return a, b

    def same(x, y):
        (a1, g1, l1), (o1, s1, t1, c1) = x
        (a2, g2, l2), (o2, s2, t2, c2) = y
        assert a1.view(np.uint64).tolist() == a2.view(np.uint64).tolist() and g1 == g2 and l1 == l2
        assert o1.view(np.uint64).tolist() == o2.view(np.uint64).tolist() and s1 == s2 and t1 == t2 and c1 == c2

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
