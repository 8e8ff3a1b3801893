"""vmb_sort_rows, vmb_set_or and vmb_rows_nonempty (promql.sort_rows, set_or, rows_nonempty, drop_empty_series, limit_offset,
union) bit for bit against tests/rowset_ref.py: the exec_test.go vectors, seeded sort / sort_desc over sizes and value patterns,
`or` over every key layout with both matrices, both flag arrays and the output rows, every error path, and the calls on a
caller's stream and from two host threads.  Matrices are compared with assert_same_bits (-0.0 != +0.0); the rows of keys the
call must not touch are compared byte for byte."""
import ctypes as C
import threading
import zlib

import numpy as np
import pytest

from conftest import SEED0
from rowset_ref import (NAN, drop_empty_series_ref, is_stable_sort, limit_offset_ref, nonempty, set_or_ref, sort_rows_ref,
                        tagset_key, union_ref)
from test_gpu_rollup_exact import assert_same_bits

pytestmark = pytest.mark.gpu
INF = float("inf")
T = np.arange(1000, 2001, 200, dtype=np.float64)


def seed(name, k=0):
    return np.random.default_rng(SEED0 + zlib.crc32(("rowset/%s/%d" % (name, k)).encode()))


@pytest.fixture(scope="module")
def vm():
    import victoriametrics_b200 as v
    return v


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def sort_gpu(vm, vals, desc, ctx=None, gather=True):
    import torch
    vals = np.asarray(vals, dtype=np.float64)
    S, P = vals.shape
    dv = dev(vals)
    out = torch.full((max(S * P, 1),), -7.25, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    order = vm.promql.sort_rows(dv.data_ptr(), S, P, desc, out.data_ptr() if gather else None, ctx=ctx)
    torch.cuda.synchronize()
    assert dv.cpu().numpy().tobytes() == vals.tobytes(), "the input changed"
    if gather and S * P:
        assert out.cpu().numpy()[:S * P].reshape(S, P).tobytes() == vals[order].tobytes()
    return order


def check_sort(vm, vals, what):
    vals = np.asarray(vals, dtype=np.float64)
    for desc in (False, True):
        order = sort_gpu(vm, vals, desc)
        if vals.shape[0] <= 13:
            assert order.tolist() == sort_rows_ref(vals, desc), (what, desc, order)
        else:
            assert is_stable_sort(vals, order, desc), (what, desc)


def pattern(rng, kind, S, P):
    if kind == "walk":  # decided at the last point
        v = 1000 + np.cumsum(rng.standard_normal((S, P)), axis=1)
        v[rng.random((S, P)) < 0.05] = NAN
    elif kind == "ints":  # ties at the last point
        v = rng.integers(0, 16, (S, P)).astype(np.float64)
    elif kind == "repeated":  # classes of equal rows
        d = max(1, S // 100)
        base = 1000 + np.cumsum(rng.standard_normal((d, P)), axis=1)
        v = base[np.arange(S) % d]
    else:  # NaN over the last 100 points
        v = 1000 + np.cumsum(rng.standard_normal((S, P)), axis=1)
        v[:, max(0, P - 100):] = NAN
    return v


# ------------------------------------------------------------------------------------------------ sort
@pytest.mark.parametrize("kind", ["walk", "ints", "repeated", "nan_tail"])
@pytest.mark.parametrize("S", [0, 1, 2, 12, 13, 1000])
@pytest.mark.parametrize("P", [0, 1, 6, 8172])
def test_sort_seeded(vm, kind, S, P):
    check_sort(vm, pattern(seed(kind, S * 10000 + P), kind, S, P), (kind, S, P))


@pytest.mark.parametrize("kind", ["walk", "ints", "repeated", "nan_tail"])
@pytest.mark.parametrize("P", [0, 1, 6])
def test_sort_100k_rows(vm, kind, P):
    check_sort(vm, pattern(seed(kind, P), kind, 100_000, P), (kind, P))


def test_sort_100k_rows_8172_points(vm):
    """the measured size, small integers: every round of the refinement; checked on the device, pair by pair"""
    import torch
    S, P = 100_000, 8172
    g = torch.Generator(device="cuda").manual_seed(SEED0 + 8172)
    dv = torch.randint(0, 16, (S, P), device="cuda", generator=g).to(torch.float64)
    dv[:, -3:][torch.rand((S, 3), device="cuda", generator=g) < 0.1] = NAN
    for desc in (False, True):
        torch.cuda.synchronize()
        order = vm.promql.sort_rows(dv.data_ptr(), S, P, desc)
        assert np.array_equal(np.sort(order), np.arange(S))
        o = torch.from_numpy(order).cuda()
        for i0 in range(0, S - 1, 2048):
            i = torch.arange(i0, min(S - 1, i0 + 2048), device="cuda")
            a, b = dv[o[i]], dv[o[i + 1]]
            an, bn = torch.isnan(a), torch.isnan(b)
            differ = (an != bn) | (~an & ~bn & (a != b))
            anyd = differ.any(dim=1)
            n = P - 1 - differ.flip(1).to(torch.int8).argmax(dim=1)
            k = torch.arange(len(i), device="cuda")
            av, bv = a[k, n], b[k, n]
            less = torch.where(torch.isnan(av), True, torch.where(torch.isnan(bv), False, bv < av if desc else av < bv))
            assert bool(torch.where(anyd, less, o[i] < o[i + 1]).all()), (desc, i0)


def test_sort_special_values(vm):
    rng = seed("special")
    v = rng.integers(0, 3, (300, 7)).astype(np.float64)
    v[rng.random(v.shape) < 0.2] = NAN
    v[rng.random(v.shape) < 0.1] = INF
    v[rng.random(v.shape) < 0.1] = -INF
    v[rng.random(v.shape) < 0.1] = -0.0
    v[rng.random(v.shape) < 0.1] = 0.0
    v[::17] = NAN  # all-NaN rows
    check_sort(vm, v, "special")
    for S in (5, 12, 13, 40):  # rows that first differ at point 0, and more than 12 equal rows
        w = np.tile([[NAN, 3.0, -0.0, 2.0]], (S, 1))
        w[::3, 0] = np.arange(len(w[::3]))
        w[1::4, 2] = 0.0
        check_sort(vm, w, ("point 0", S))


# ------------------------------------------------------------------------------------------------ or
def or_gpu(vm, left, ll, right, rl, ctx=None, **kw):
    import torch
    L, R = np.array(left, dtype=np.float64), np.array(right, dtype=np.float64)
    P = L.shape[1]
    dl, dr = dev(L if L.size else np.zeros(1)), dev(R if R.size else np.zeros(1))
    out = torch.full((max((len(ll) + len(rl)) * P, 1),), -7.25, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    rows = vm.promql.set_or(dl.data_ptr(), ll, dr.data_ptr(), rl, P, out.data_ptr(), ctx=ctx, **kw)
    torch.cuda.synchronize()
    gl, gr = dl.cpu().numpy()[:L.size].reshape(L.shape), dr.cpu().numpy()[:R.size].reshape(R.shape)
    o = out.cpu().numpy()[:len(rows) * P].reshape(len(rows), P)
    return gl, gr, rows, o


def check_or(vm, left, ll, right, rl, what, **kw):
    L, R = np.array(left, dtype=np.float64), np.array(right, dtype=np.float64)
    gl, gr, rows, o = or_gpu(vm, L, ll, R, rl, **kw)
    wl, wr, wout = set_or_ref(L, ll, R, rl, **kw)
    assert_same_bits(gl, wl, "%s left" % (what,))
    assert_same_bits(gr, wr, "%s right" % (what,))
    assert rows == [(0 if s == "l" else 1, i) for s, i in wout], (what, rows, wout)
    want = np.array([(wl if s == "l" else wr)[i] for s, i in wout]).reshape(len(wout), L.shape[1])
    assert_same_bits(o, want, "%s output" % (what,))
    # the rows of right keys without a left row keep their bits
    lkeys = {tagset_key(lb, kw.get("on"), kw.get("ignoring", ())) for lb in ll}
    for i, lb in enumerate(rl):
        if tagset_key(lb, kw.get("on"), kw.get("ignoring", ())) not in lkeys:
            assert gr[i].tobytes() == R[i].tobytes(), (what, i)
    return [(wl if s == "l" else wr)[i].tolist() for s, i in wout]


def same(got, want):
    assert len(got) == len(want) and all(np.array_equal(np.array(g), np.array(w), equal_nan=True) for g, w in zip(got, want)), \
        (got, want)


def test_exec_test_vectors(vm):
    same(check_or(vm, [T, T + 1], [{"x": "foo"}, {"x": "bar"}], [T + 2, T + 3], [{"x": "foo"}, {"x": "baz"}], "series or series"),
         [T + 1, T, T + 3])
    same(check_or(vm, [np.where(T > 1400, T, NAN)], [{}], [[123.0] * 6], [{}], "scalar or scalar"),
         [[123, 123, 123, 1600, 1800, 2000]])
    same(check_or(vm, [[NAN] * 6], [{"a": "a", "b": "b1"}], [[2.0] * 6], [{"a": "a", "b": "b2"}], "nan or on() series", on=("a",)),
         [[2] * 6])
    same(check_or(vm, [np.where(T >= 1600, T, NAN)], [{"a": "a", "b": "b1"}], [[1.0] * 6], [{}], "series with NaNs or scalar"),
         [[NAN, NAN, NAN, 1600, 1800, 2000], [1] * 6])
    same(check_or(vm, [np.where(T > 1200, T, NAN)], [{"a": "a", "b": "b1"}], [[0.0] * 6], [{}], "series or on() scalar", on=()),
         [[NAN, NAN, 1400, 1600, 1800, 2000], [0, 0, NAN, NAN, NAN, NAN]])
    same(check_or(vm, [np.where(T <= 1200, T, NAN)], [{"a": "a", "b": "b1"}], [np.where(T > 1200, T, NAN)],
                  [{"a": "a", "b": "b2"}], "series or on() series", on=("a",)),
         [[1000, 1200, NAN, NAN, NAN, NAN], [NAN, NAN, 1400, 1600, 1800, 2000]])
    # sort() / sort_desc() / two_timeseries: `or`, then the sort
    for left, right, desc, want in (([2.0] * 6, [1.0] * 6, False, [[1] * 6, [2] * 6]), ([1.0] * 6, [2.0] * 6, True, [[2] * 6, [1] * 6]),
                                    (T, [2.0] * 6, True, [T, [2] * 6])):
        got = np.array(check_or(vm, [left], [{}], [right], [{"xx": "foo"}], "sort"))
        same(got[sort_gpu(vm, got, desc)], want)


def test_exec_test_vectors_of_the_row_filters(vm):
    import torch
    vals = np.array([np.where(T > 2000, T, NAN), np.where(T + 500 > 2000, T + 500, NAN)])
    dv = dev(vals)
    out = torch.empty(12, dtype=torch.float64, device="cuda")
    assert vm.promql.drop_empty_series(dv.data_ptr(), 2, 6, out.data_ptr()).tolist() == drop_empty_series_ref(vals) == [1]
    torch.cuda.synchronize()
    assert out.cpu().numpy()[:6].tobytes() == vals[1].tobytes()
    by_label = np.array([T * 2, T * 3, T * 1])
    desc = np.array([T * 3, T * 2, T * 1])
    desc = np.where(desc < 3000, desc, NAN)
    for lim, off, v in ((1, 1, by_label), (1, 10, by_label), (1, 1, desc), (5, 0, desc), (0, 0, desc)):
        d = dev(v)
        got = vm.promql.limit_offset(lim, off, d.data_ptr(), 3, 6, out.data_ptr())
        assert got.tolist() == limit_offset_ref(lim, off, v), (lim, off)
        torch.cuda.synchronize()
        assert out.cpu().numpy()[:len(got) * 6].tobytes() == v[got].tobytes()
    x, y = dev([np.where(T > 1400, T, NAN)]), dev([np.where(T < 1700, T, NAN), T])
    args = [(x.data_ptr(), [{"__name__": "x", "foo": "bar"}]), (y.data_ptr(), [{"__name__": "y", "foo": "baz"}, {"__name__": "x", "foo": "bar"}])]
    got = vm.promql.union(args, 6, out.data_ptr())
    assert got == union_ref([a[1] for a in args]) == [(0, 0), (1, 0)]
    torch.cuda.synchronize()
    assert out.cpu().numpy()[:12].tobytes() == np.concatenate([x.cpu().numpy()[0], y.cpu().numpy()[0]]).tobytes()
    assert vm.promql.union([(x.data_ptr(), [{}]), (y.data_ptr(), [{}])], 6) == [(0, 0), (1, 0)]


def values(rng, S, P, nan=0.3, empty=0.1):
    v = np.round(rng.standard_normal((S, P)) * 100, 1)
    v[rng.random((S, P)) < nan] = NAN
    v[rng.random(S) < empty] = NAN
    return v


def layout(rng, name, n):
    """(left labels, right labels, kw) of a key layout; `k` is the key label under on(k), `n` the rest of the name"""
    if name == "1:1 equal names":
        return [{"k": str(i)} for i in range(n)], [{"k": str(i)} for i in range(n)], dict(on=("k",))
    if name == "1:1 different names":
        return [{"k": str(i), "s": "l"} for i in range(n)], [{"k": str(i), "s": "r"} for i in range(n)], dict(on=("k",))
    if name == "N:1 scalar":
        return [{"k": str(i)} for i in range(n)], [{}], dict(on=())
    if name == "N:1 unnamed left":
        return [{}] + [{"k": str(i)} for i in range(n - 1)], [{}], dict(on=())
    if name == "scalar or scalar":
        return [{}], [{}], {}
    if name == "N:M duplicate names":
        ll = [{"k": str(rng.integers(0, 4)), "s": "ab"[rng.integers(0, 2)], "__name__": "m"} for _ in range(n)]
        rl = [{"k": str(rng.integers(0, 5)), "s": "abc"[rng.integers(0, 3)], "__name__": "m"} for _ in range(n)]
        return ll, rl, dict(on=("k",))
    # keys on one side only, and keys whose left rows are all empty (rows of key 0 are made empty below)
    ll = [{"k": str(rng.integers(0, 6)), "s": str(rng.integers(0, 3))} for _ in range(n)]
    rl = [{"k": str(rng.integers(3, 9)), "s": str(rng.integers(0, 3))} for _ in range(n)]
    return ll, rl, dict(ignoring=("s",))


LAYOUTS = ["1:1 equal names", "1:1 different names", "N:1 scalar", "N:1 unnamed left", "scalar or scalar", "N:M duplicate names",
           "one-sided and empty keys"]


@pytest.mark.parametrize("name", LAYOUTS)
@pytest.mark.parametrize("n,P", [(1, 1), (7, 6), (40, 50), (300, 33)])
def test_or_layouts(vm, name, n, P):
    rng = seed(name, n * 1000 + P)
    ll, rl, kw = layout(rng, name, n)
    L, R = values(rng, len(ll), P), values(rng, len(rl), P)
    if name == "one-sided and empty keys":
        L[[i for i, lb in enumerate(ll) if lb["k"] in ("3", "4")]] = NAN
    check_or(vm, L, ll, R, rl, (name, n, P), **kw)


def test_or_many_left_rows_under_one_key(vm):
    """q or on() vector(0) with more left rows than one run of k_or_first, and NaN columns that only late rows fill"""
    rng = seed("vector0")
    for S, P in ((5000, 40), (300, 8172)):
        L = np.full((S, P), NAN)
        for p in range(P):
            first = rng.integers(0, S + S // 4)  # no value at the point when first >= S
            if first < S:
                L[first:, p] = rng.standard_normal(S - first)
                L[rng.random(S) < 0.5, p] = NAN
                L[first, p] = 1.0
        R = np.zeros((1, P))
        check_or(vm, L, [{"k": str(i)} for i in range(S)], R, [{}], ("vector(0)", S, P), on=())
        ll = [{"s": "x"}] * 3 + [{"k": str(i)} for i in range(S - 3)]  # a name shared by several rows of the one key
        R2 = values(rng, 3, P, empty=0)
        check_or(vm, L, ll, R2, [{"s": "x"}, {"s": "y"}, {"s": "x"}], ("one key, shared names", S, P), on=())


def test_or_no_rows_and_no_points(vm):
    check_or(vm, np.zeros((0, 4)), [], values(seed("none"), 3, 4), [{"a": "1"}, {"a": "2"}, {}], "no left rows")
    check_or(vm, values(seed("none", 1), 3, 4), [{"a": "1"}, {"a": "2"}, {}], np.zeros((0, 4)), [], "no right rows")
    gl, gr, rows, _ = or_gpu(vm, np.zeros((2, 0)), [{"a": "1"}, {"a": "2"}], np.zeros((1, 0)), [{"a": "1"}])
    assert rows == [] and gl.shape == (2, 0)


def test_rows_nonempty(vm):
    rng = seed("nonempty")
    for S, P in ((0, 5), (3, 0), (1, 1), (100, 33), (2000, 8172)):
        v = np.full((S, P), NAN)
        if S and P:
            v[rng.random(S) < 0.5, rng.integers(0, P)] = 1.0
            v[::7, P - 1] = -0.0
        d = dev(v if v.size else np.zeros(1))
        assert vm.promql.rows_nonempty(d.data_ptr(), S, P).tolist() == nonempty(v).tolist()


# ------------------------------------------------------------------------------------------------ errors
def test_errors_leave_everything_untouched(vm):
    import torch
    from victoriametrics_b200 import _lib
    lib, ctx = _lib.lib(), _lib.default_context()
    u8, u32 = (lambda a: a.ctypes.data_as(_lib.u8p)), (lambda a: a.ctypes.data_as(_lib.u32p))
    dv = torch.arange(12, dtype=torch.float64, device="cuda")
    before = dv.cpu().numpy().tobytes()
    rows = np.full(4, 7, dtype=np.uint32)
    srt = lambda p=dv.data_ptr(), n=4, pts=3, o=True: lib.vmb_sort_rows(ctx.h, C.c_void_p(p), n, pts, 0, u32(rows) if o else None)
    assert srt(o=False) == -50 and srt(p=0) == -50 and srt(n=2 ** 31) == -50 and srt(pts=2 ** 31) == -50
    assert lib.vmb_sort_rows(None, C.c_void_p(dv.data_ptr()), 4, 3, 0, u32(rows)) == -50
    assert (rows == 7).all()
    flags = np.full(4, 7, dtype=np.uint8)
    assert lib.vmb_rows_nonempty(ctx.h, C.c_void_p(dv.data_ptr()), 4, 3, None) == -50
    assert lib.vmb_rows_nonempty(ctx.h, C.c_void_p(0), 4, 3, u8(flags)) == -50
    assert lib.vmb_rows_nonempty(ctx.h, C.c_void_p(dv.data_ptr()), 2 ** 31, 3, u8(flags)) == -50
    assert (flags == 7).all()
    dr = torch.arange(6, dtype=torch.float64, device="cuda") * -1
    rbefore = dr.cpu().numpy().tobytes()
    lne, rne = np.full(4, 7, dtype=np.uint8), np.full(2, 7, dtype=np.uint8)
    keys, names = np.zeros(4, dtype=np.uint32), np.arange(4, dtype=np.uint32)

    def sor(l=dv.data_ptr(), nl=4, lk=keys, ln=names, r=dr.data_ptr(), nr=2, rk=keys[:2], rn=names[:2], nk=1, pts=3, fl=True, fr=True):
        return lib.vmb_set_or(ctx.h, C.c_void_p(l), nl, u32(lk) if lk is not None else None, u32(ln) if ln is not None else None,
                              C.c_void_p(r), nr, u32(rk) if rk is not None else None, u32(rn) if rn is not None else None, nk, pts,
                              u8(lne) if fl else None, u8(rne) if fr else None)
    assert sor(l=0) == -50 and sor(r=0) == -50 and sor(lk=None) == -50 and sor(ln=None) == -50 and sor(rk=None) == -50
    assert sor(rn=None) == -50 and sor(fl=False) == -50 and sor(fr=False) == -50
    assert sor(lk=np.array([0, 0, 1, 0], dtype=np.uint32)) == -50 and sor(rk=np.array([0, 3], dtype=np.uint32)) == -50
    assert sor(nk=0) == -50 and sor(nl=2 ** 31) == -50 and sor(nr=2 ** 31) == -50 and sor(pts=2 ** 31) == -50
    torch.cuda.synchronize()
    assert dv.cpu().numpy().tobytes() == before and dr.cpu().numpy().tobytes() == rbefore
    assert (lne == 7).all() and (rne == 7).all()
    assert sor() == 0 and lne.tolist() == [1, 1, 1, 1] and rne.tolist() == [0, 0]  # no names match: nothing filled, right cleared
    torch.cuda.synchronize()
    assert dv.cpu().numpy().tobytes() == before and np.isnan(dr.cpu().numpy()).all()
    assert srt() == 0 and rows.tolist() == [0, 1, 2, 3]


# ------------------------------------------------------------------------------------------------ streams and threads
def _catalogue(vm, ctx, inputs):
    res = []
    vals, L, ll, R, rl = inputs
    for desc in (False, True):
        res.append(sort_gpu(vm, vals, desc, ctx=ctx).tobytes())
    gl, gr, rows, o = or_gpu(vm, L, ll, R, rl, ctx=ctx, on=("k",))
    res += [gl.tobytes(), gr.tobytes(), repr(rows).encode(), o.tobytes()]
    d = dev(vals)
    res.append(vm.promql.rows_nonempty(d.data_ptr(), *vals.shape, ctx=ctx).tobytes())
    return res


def test_caller_stream_and_two_threads_equal_the_serial_run(vm):
    import torch
    rng = seed("threads")
    vals = pattern(rng, "ints", 20000, 64)
    vals[::5] = NAN
    ll = [{"k": str(rng.integers(0, 50)), "s": "ab"[rng.integers(0, 2)]} for _ in range(3000)]
    rl = [{"k": str(rng.integers(0, 60)), "s": "ab"[rng.integers(0, 2)]} for _ in range(3000)]
    inputs = (vals, values(rng, 3000, 64), ll, values(rng, 3000, 64), rl)
    serial = _catalogue(vm, None, inputs)
    stream = torch.cuda.Stream()
    ctx = vm.Context(0, stream=stream.cuda_stream)
    try:
        assert _catalogue(vm, ctx, inputs) == serial
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
            results[i] = _catalogue(vm, c, inputs)
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
