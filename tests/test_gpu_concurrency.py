"""Contexts on caller streams and concurrent host threads: every entry-point family, bit for bit against the serial run.

The rest of the suite runs the library one way only: the default context, on the legacy default stream, from one host thread,
with pageable host buffers.  That hides three kinds of bug.  The legacy stream synchronises with every blocking stream, so a copy
or launch that misses the ctx's stream still looks right.  A device-to-host copy into pageable memory returns only once it has
landed, so an entry point that returns before its result copy is done still passes.  And state that is built on first use, or
shared between contexts, is only ever built by one thread.

CATALOGUE below is a set of small seeded calls that reaches every entry-point family.  The serial reference is the catalogue on
the default context, run as the other tests run it (their files pin those outputs).  The other runs must equal it bit for bit
(sum: the bound of EXCEPTIONS["fused sum"] in test_gpu_matrix_exact.py):
  - on a caller stream made with cudaStreamNonBlocking: host outputs in vmb_host_alloc memory, read as soon as the call
    returns, and the stream must be drained by then; device inputs written on that stream by a copy that waits behind a spin
    kernel, so that it is still in flight when the library is called, while the legacy default stream is kept busy too;
    device outputs copied on the caller's stream and read after one event recorded there;
  - on K = 4 contexts, one per host thread and stream, started together, each running the catalogue once in its own order; and
    again in a fresh process, so that first-use initialisation (zstd tables, fused grid sizes, the ctx's second stream) happens
    under concurrency.
"""
import ctypes as C
import math
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import blockgen
from conftest import SEED0

T0 = 1_700_000_000_000
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
K = 4                      # concurrent host threads / contexts
PIPE_CHUNK_BLOCKS = 8      # vmb_eval_rollup_host: 30 blocks -> 4 chunks
FUSED_CHUNKS = 4
SPIN = 2_000_000           # cycles of the kernel a device input waits behind (~1 ms)
LEGACY_SPIN = 10 * SPIN    # ... and of the one the legacy default stream is kept busy with meanwhile
SENT_BYTE = 0xA5           # host output buffers are filled with it before a call
SENT = -7.25e-300          # ... and device output matrices with this value
ERR_BLOCK_FAILED, ERR_INVALID_ARG = -53, -50
GO_NAN = np.array([0x7FF8000000000001], dtype=np.uint64).view(np.float64)[0]
AGGR_IDS = {"sum": 0, "min": 1, "max": 2, "count": 4}


def _vm():
    import victoriametrics_b200 as vm
    return vm


def _L():
    from victoriametrics_b200 import _lib
    return _lib.lib()


def _check(rc, allow=()):
    from victoriametrics_b200 import _lib
    return _lib.check(rc, allow)


# ------------------------------------------------------------------------------------------------ inputs (numpy, seeded)
def _fused_blocks(rng, n, rows=1200):
    """one block per series, delta-const timestamps at precisionBits 64: the series the fused kernel takes; zstd literals in
    every chunk (counter), zstd frames with sequences (counter_smooth)"""
    kinds = ["counter", "counter_smooth", "gauge"]
    return [blockgen.OBlock(blockgen.gen_timestamps(rng, "regular", rows, T0), blockgen.gen_values(rng, kinds[s % 3], rows), -2,
                            64, s) for s in range(n)]


def _matrix(rng, rows, points, nan=0.2):
    m = rng.normal(scale=50.0, size=(rows, points))
    m[rng.random(m.shape) < nan] = np.nan
    m[rng.random(m.shape) < 0.03] = -0.0
    return m


_INPUTS = None


def inputs():
    global _INPUTS
    if _INPUTS is not None:
        return _INPUTS
    rng = np.random.default_rng(SEED0 + 9100)
    I = {}
    dec = blockgen.random_blocks(rng, 40, rows_choices=(1, 33, 513, 4096, 8192),
                                 value_kinds=("counter_smooth", "counter", "gauge", "const", "special", "counter_big"))
    assert sum(b.vmt in (1, 4) for b in dec) >= 8, "the decode batch needs zstd frames"
    I["dec_blocks"] = dec
    I["dec"] = blockgen.to_blockset(dec)
    fb = _fused_blocks(rng, 48)
    I["fused_blocks"] = fb
    I["fused"] = blockgen.to_blockset(fb)
    I["fused_groups"] = (np.arange(len(fb)) * 7 % 5).astype(np.uint32)
    I["fused_cfg"] = ("rate", T0 + 60_000, T0 + 15_000 * 1199, 60_000, 120_000)
    hb = blockgen.random_blocks(rng, 30, rows_choices=(33, 513, 2000), ts_kinds=("regular", "jitter"))
    I["host"] = blockgen.to_blockset(hb)
    I["host_nseries"] = len(hb)
    I["host_cfg"] = ("max_over_time", T0 + 30_000, T0 + 15_000 * 1999, 45_000, 90_000)
    S, P = 70, 53
    I["m"] = _matrix(rng, S, P)
    I["m2"] = _matrix(rng, S, P)
    I["groups"] = rng.integers(0, 6, S).astype(np.uint32)
    I["groups"][:6] = np.arange(6)
    # points where every row of a group is NaN on the right-hand side of the set operator: there `and` drops the left value,
    # so the result tells the group's first value (NaN) from one that was never written
    I["m2"][np.ix_(I["groups"] == 0, np.arange(0, P, 4))] = np.nan
    I["m2"][np.ix_(I["groups"] == 3, np.arange(1, P, 5))] = np.nan
    I["perm"] = rng.permutation(S).astype(np.uint32)
    I["phis"] = np.linspace(-0.1, 1.1, P)
    I["ks"] = np.where(np.arange(P) % 5 == 0, np.nan, (np.arange(P) % 4).astype(np.float64))
    I["a_rows"] = np.where(rng.random(S) < 0.1, -1, rng.integers(0, S, S)).astype(np.int64)
    I["b_rows"] = np.where(rng.random(S) < 0.1, -1, rng.integers(0, S, S)).astype(np.int64)
    I["clamp"] = (np.full(P, -20.0), np.full(P, 30.0))
    # subquery feed: an inner result on the grid T0 .. T0 + 15 s * (Psq - 1)
    I["sq"] = _matrix(rng, 40, 200, nan=0.3)
    # `le` histograms: G groups of B buckets, cumulative counts
    G, B = 5, 6
    les = np.array([0.1, 0.5, 1.0, 5.0, 10.0, np.inf])
    h = np.cumsum(rng.integers(0, 20, (G, B, P)), axis=1).astype(np.float64)
    h[rng.random(h.shape) < 0.05] = np.nan
    I["hist"] = h.reshape(G * B, P)
    I["hist_groups"] = np.repeat(np.arange(G), B).astype(np.uint32)
    I["hist_les"] = np.tile(les, G)
    I["hist_G"] = G
    # vmrange buckets: G groups of 5 buckets with a gap, and one row kept as it is
    edges = ["0", "0.5", "1", "2.5", "5", "10", "25"]
    keys, gids, starts, ends, skeys, ekeys = {}, [], [], [], [], []
    for g in range(4):
        for b in (0, 1, 2, 4, 5):  # 2.5...5 missing: a gap row
            gids.append(g)
            starts.append(float(edges[b]))
            ends.append(float(edges[b + 1]))
            skeys.append(keys.setdefault(edges[b], len(keys)))
            ekeys.append(keys.setdefault(edges[b + 1], len(keys)))
    gids.append(0xFFFFFFFE)
    starts.append(0.0)
    ends.append(0.0)
    skeys.append(0)
    ekeys.append(0)
    n = len(gids)
    I["vr"] = np.where(rng.random((n, P)) < 0.2, 0.0, rng.integers(0, 9, (n, P)).astype(np.float64))
    I["vr_args"] = [np.array(gids, dtype=np.uint32), np.array(starts), np.array(ends), np.array(skeys, dtype=np.uint32),
                    np.array(ekeys, dtype=np.uint32)]
    # write path
    I["cols_i64"] = np.stack([blockgen.gen_values(rng, k, 1000) for k in ("counter", "gauge", "const", "counter_smooth",
                                                                           "gauge_wide", "delta_const")])
    I["cols_f64"] = np.round(rng.normal(100, 30, (5, 700)), 3)
    I["cols_f64"][1, ::7] = np.nan
    I["cols_f64"][2] = rng.normal(0, 1e200, 700)
    zb = [b for b in dec if b.vmt in (1, 4)]
    I["frames"] = zb[:6]
    I["unmarshal"] = max(zb, key=lambda b: b.rows)
    I["decimals"] = blockgen.gen_values(rng, "special", 3000)
    # outliers_iqr: 120 k series x 160 points (19.2 M keys, 154 MB) -- one point batch, so vmb_aggr_order's last internal
    # synchronisation (oa_replan) comes before the gather, the sort of every group (about 20 k rows: merge passes) and the
    # selection, milliseconds of device work queued after it
    I["big"] = _matrix(rng, 120_000, 160)
    I["big_groups"] = rng.integers(0, 6, 120_000).astype(np.uint32)
    _INPUTS = I
    return I


# ------------------------------------------------------------------------------------------------ where a run happens
class Env:
    """One way of calling the library.  serial: the default context on the legacy stream, pageable host buffers, device inputs
    copied before the call returns control (as every other test does).  Otherwise: ctx on a non-blocking caller stream, host
    outputs (and host inputs) in pinned memory, device inputs still being written on the caller stream when the library is
    called.  Every tensor and host buffer a call reads stays referenced until finish() has waited for the caller's stream."""

    def __init__(self, ctx, stream=None, device=0):
        import torch
        self.torch = torch
        self.ctx, self.stream, self.device = ctx, stream, device
        self.serial = stream is None
        self.dev = torch.device("cuda", device)
        self.keep = []
        self._pinned = []
        self.late = []

    # -- host buffers
    def _host_buf(self, shape, dtype):
        dtype = np.dtype(dtype)
        n = int(np.prod(shape)) * dtype.itemsize
        if self.serial:
            return np.empty(shape, dtype)
        p = _L().vmb_host_alloc(max(n, 1))
        assert p, "vmb_host_alloc(%d) failed" % n
        self._pinned.append(p)
        raw = np.frombuffer((C.c_uint8 * max(n, 1)).from_address(p), dtype=np.uint8)[:n]
        return raw.view(dtype).reshape(shape)

    def host_out(self, shape, dtype):
        a = self._host_buf(shape, dtype)
        a.view(np.uint8)[...] = SENT_BYTE
        return a

    def host_in(self, arr):
        arr = np.ascontiguousarray(arr)
        a = self._host_buf(arr.shape, arr.dtype)
        a[...] = arr
        self.keep.append(a)
        return a

    # -- device buffers
    def dev_in(self, a):
        torch = self.torch
        src = torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64))
        if self.serial:
            t = src.to(self.dev)
            self.keep.append(t)
            return t
        with torch.cuda.device(self.device):
            with torch.cuda.stream(torch.cuda.default_stream(self.device)):
                torch.cuda._sleep(LEGACY_SPIN)
            with torch.cuda.stream(self.stream):
                src = src.pin_memory()
                t = torch.full(src.shape, SENT, dtype=torch.float64, device=self.dev)
                torch.cuda._sleep(SPIN)
                t.copy_(src, non_blocking=True)
        self.keep += [src, t]
        return t

    def dev_out(self, *shape):
        torch = self.torch
        if self.serial:
            t = torch.full(shape, SENT, dtype=torch.float64, device=self.dev)
        else:
            with torch.cuda.device(self.device), torch.cuda.stream(self.stream):
                t = torch.full(shape, SENT, dtype=torch.float64, device=self.dev)
        self.keep.append(t)
        return t

    def snap(self, a):
        """a host output as it is when the call that wrote it returns.  Such a call must have drained the ctx's stream: on a
        caller stream nothing else could be running there."""
        if not self.serial and not self.stream.query():
            self.late.append(a.shape)
        return np.array(a, copy=True)

    def finish(self, outs):
        """-> {name: np.ndarray or int}.  Serial: device outputs copied after a device-wide synchronisation.  On a caller stream:
        device outputs copied on that stream into pinned memory, then one event recorded there and waited for -- nothing else,
        so that library work left on any other stream (the legacy one included) is not waited for."""
        torch = self.torch
        if self.serial:
            torch.cuda.synchronize(self.device)
            return {k: v.cpu().numpy() if isinstance(v, torch.Tensor) else v for k, v in outs.items()}
        res = {}
        with torch.cuda.device(self.device), torch.cuda.stream(self.stream):
            for k, v in outs.items():
                if isinstance(v, torch.Tensor):
                    h = torch.empty(v.shape, dtype=v.dtype, pin_memory=True)
                    h.copy_(v, non_blocking=True)
                    v = h
                res[k] = v
            ev = torch.cuda.Event()
            ev.record(self.stream)
        ev.synchronize()
        late, self.late = self.late, []
        assert not late, "host outputs of shapes %s returned before the ctx's stream was done" % late
        return {k: v.numpy().copy() if isinstance(v, torch.Tensor) else v for k, v in res.items()}

    def close(self):
        self.keep = []
        for p in self._pinned:
            _L().vmb_host_free(p)
        self._pinned = []


def _u32(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint32))


def _f64(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _i64(a):
    return a.ctypes.data_as(C.POINTER(C.c_int64))


def _u8(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint8))


def _p(t):
    return C.c_void_p(t.data_ptr())


def _upload(env, descs, payload):
    pay = env.host_in(payload)
    h = C.c_void_p()
    _check(_L().vmb_blocks_upload(env.ctx.h, descs, len(descs), _u8(pay), pay.size, C.byref(h)))
    env.keep.append(descs)
    return h


# ------------------------------------------------------------------------------------------------ the catalogue
def e_decode(env, I):
    """vmb_decode_blocks + vmb_series_layout + vmb_series_download (random blocks, zstd frames with sequences)"""
    L = _L()
    descs, payload = I["dec"]
    b = _upload(env, descs, payload)
    try:
        status = env.host_out(len(descs), np.int32)
        s = C.c_void_p()
        rc = L.vmb_decode_blocks(env.ctx.h, b, INT64_MIN, INT64_MAX, 0, status.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(s))
        _check(rc)
        out = {"status": env.snap(status)}
        try:
            n, rows = L.vmb_series_count(s), L.vmb_series_rows(s)
            starts, counts = env.host_out(n, np.uint64), env.host_out(n, np.uint32)
            _check(L.vmb_series_layout(env.ctx.h, s, starts.ctypes.data_as(C.POINTER(C.c_uint64)), _u32(counts)))
            starts, counts = env.snap(starts), env.snap(counts)
            ts, vals = env.host_out(rows, np.int64), env.host_out(rows, np.float64)
            _check(L.vmb_series_download(env.ctx.h, s, _i64(ts), _f64(vals)))
            ts, vals = env.snap(ts), env.snap(vals)
        finally:
            L.vmb_series_free(s)
    finally:
        L.vmb_blocks_free(b)
    # rows outside a series' live range are scratch; keep the live ones
    sel = np.concatenate([np.arange(a, a + c) for a, c in zip(starts.tolist(), counts.tolist())] or [np.zeros(0, np.int64)])
    out.update(counts=counts, ts=ts[sel.astype(np.int64)], vals=vals[sel.astype(np.int64)])
    return out


def _rc(vm, spec):
    func, start, end, step, window = spec
    return vm.promql.get_rollup_configs(func, start, end, step, window)


def e_fused(env, I):
    """vmb_eval_rollup_device, fused (chunked: the zstd stage of chunk k + 1 on the ctx's second stream) and un-fused"""
    vm, L = _vm(), _L()
    descs, payload = I["fused"]
    b = _upload(env, descs, payload)
    rc = _rc(vm, I["fused_cfg"])
    cfg = rc._cfg()
    out = {}
    try:
        for name, fused in (("fused", True), ("unfused", False)):
            d = env.dev_out(len(descs), rc.points)
            sc = C.c_uint64(0)
            env.ctx.set_fused(fused)
            try:
                _check(L.vmb_eval_rollup_device(env.ctx.h, b, INT64_MIN, INT64_MAX, C.byref(cfg), _p(d), C.byref(sc)))
            finally:
                env.ctx.set_fused(True)
            out[name], out[name + " scanned"] = d, sc.value
    finally:
        L.vmb_blocks_free(b)
    return out


def e_aggr_device(env, I):
    """vmb_eval_rollup_aggr_device (the fold inside the fused kernel) + vmb_aggr_finalize into a host buffer"""
    vm, L = _vm(), _L()
    descs, payload = I["fused"]
    b = _upload(env, descs, payload)
    rc = _rc(vm, I["fused_cfg"])
    cfg = rc._cfg()
    G = int(I["fused_groups"].max()) + 1
    groups = env.host_in(I["fused_groups"])
    out = {}
    try:
        for aggr, aid in AGGR_IDS.items():
            dv, dcnt = env.dev_out(G, rc.points), env.dev_out(G, rc.points)
            sc = C.c_uint64(0)
            _check(L.vmb_eval_rollup_aggr_device(env.ctx.h, b, INT64_MIN, INT64_MAX, C.byref(cfg), aid, _u32(groups), G, _p(dv),
                                                 _p(dcnt), C.byref(sc)))
            h = env.host_out((G, rc.points), np.float64)
            _check(L.vmb_aggr_finalize(env.ctx.h, aid, _p(dv), _p(dcnt), G * rc.points, _f64(h)))
            out["aggr " + aggr], out["aggr %s scanned" % aggr] = env.snap(h), sc.value
    finally:
        L.vmb_blocks_free(b)
    return out


def e_rollup_host(env, I):
    """vmb_eval_rollup_host: the chunked host pipeline (H2D stream, ctx stream, D2H stream), several chunks"""
    vm, L = _vm(), _L()
    descs, payload = I["host"]
    rc = _rc(vm, I["host_cfg"])
    cfg = rc._cfg()
    pay = env.host_in(payload)
    o = env.host_out((I["host_nseries"], rc.points), np.float64)
    st = env.host_out(len(descs), np.int32)
    sc = C.c_uint64(0)
    _check(L.vmb_eval_rollup_host(env.ctx.h, descs, len(descs), _u8(pay), pay.size, INT64_MIN, INT64_MAX, C.byref(cfg), _f64(o),
                                  st.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(sc)))
    return {"out": env.snap(o), "status": env.snap(st), "scanned": sc.value}


def e_subquery(env, I):
    """vmb_series_from_matrix (removeNanValues) + vmb_rollup of the outer function"""
    vm, L = _vm(), _L()
    m = I["sq"]
    dm = env.dev_in(m)
    s = C.c_void_p()
    _check(L.vmb_series_from_matrix(env.ctx.h, _p(dm), m.shape[0], m.shape[1], T0, 15_000, C.byref(s)))
    try:
        rc = vm.promql.get_rollup_configs("avg_over_time", T0 + 60_000, T0 + 15_000 * 199, 30_000, 90_000)
        rc.dropStaleNaNs = False
        cfg = rc._cfg()
        d = env.dev_out(m.shape[0], rc.points)
        sc = C.c_uint64(0)
        _check(L.vmb_rollup(env.ctx.h, s, C.byref(cfg), _p(d), 1, C.byref(sc)))
    finally:
        L.vmb_series_free(s)
    return {"out": d, "scanned": sc.value}


def e_binary(env, I):
    """vmb_binary_op with row lists, the set operator `and` (vmb_group_first_value + `if`) and vmb_matrix_merge_rows"""
    vm, L = _vm(), _L()
    m, m2 = I["m"], I["m2"]
    S, P = m.shape
    G = int(I["groups"].max()) + 1
    left, right = env.dev_in(m), env.dev_in(m2)
    perm = env.host_in(I["perm"])
    d = env.dev_out(S, P)
    _check(L.vmb_binary_op(env.ctx.h, vm.promql.BINARY_OPS["+"], 0, _p(left), _u32(perm), _p(right), None, S, P, _p(d)))
    # every call below reads inputs still being written on the caller's stream
    ar, br = env.host_in(I["a_rows"]), env.host_in(I["b_rows"])
    left, right = env.dev_in(m), env.dev_in(m2)
    dm = env.dev_out(S, 2 * P)
    _check(L.vmb_matrix_merge_rows(env.ctx.h, _p(left), _i64(ar), P, _p(right), _i64(br), P, S, _p(dm)))
    groups = env.host_in(I["groups"])
    right = env.dev_in(m2)
    tmp, dset = env.dev_out(G, P), env.dev_out(S, P)
    _check(L.vmb_group_first_value(env.ctx.h, _p(right), S, P, _u32(groups), G, _p(tmp)))
    left = env.dev_in(m)
    _check(L.vmb_binary_op(env.ctx.h, vm.promql.BINARY_OPS["if"], 0, _p(left), None, _p(tmp), _u32(groups), S, P, _p(dset)))
    return {"plus": d, "first": tmp, "and": dset, "merge": dm}


def e_aggr_matrix(env, I):
    """vmb_aggr_matrix (sum, stddev by groups), vmb_aggr_quantile, vmb_aggr_order (quantiles, outliers_iqr)"""
    vm, L = _vm(), _L()
    m = I["m"]
    S, P = m.shape
    G = int(I["groups"].max()) + 1
    groups = env.host_in(I["groups"])
    out = {}
    for name in ("sum", "stddev"):
        dm = env.dev_in(m)  # every call reads an input still being written on the caller's stream
        d, fl = env.dev_out(G, P), env.host_out(S, np.uint8)
        _check(L.vmb_aggr_matrix(env.ctx.h, vm.promql.MATRIX_AGGR_FUNCS[name], _p(dm), S, P, _u32(groups), G, _p(d), _u8(fl)))
        out[name], out[name + " flags"] = d, env.snap(fl)
    phis = env.host_in(I["phis"])
    dm = env.dev_in(m)
    dq = env.dev_out(G, P)
    _check(L.vmb_aggr_quantile(env.ctx.h, _p(dm), S, P, _u32(groups), G, _f64(phis), _p(dq)))
    out["quantile"] = dq
    qphis = env.host_in(np.array([0.25, 0.9]))
    dm = env.dev_in(m)
    dqs = env.dev_out(2, G, P)
    ne, sel = env.host_out(S, np.uint8), env.host_out(S, np.uint8)
    _check(L.vmb_aggr_order(env.ctx.h, vm.promql.ORDER_AGGR_FUNCS["quantiles"], _p(dm), S, P, _u32(groups), G, _f64(qphis), 2,
                            _p(dqs), _u8(ne), _u8(sel)))
    out["quantiles"], out["quantiles nonempty"] = dqs, env.snap(ne)
    # outliers over the large matrix: a call that returned before its final synchronisation would leave its sort running
    big = I["big"]
    Sb, Pb = big.shape
    gb = env.host_in(I["big_groups"])
    ne, sel = env.host_out(Sb, np.uint8), env.host_out(Sb, np.uint8)
    dm = env.dev_in(big)
    _check(L.vmb_aggr_order(env.ctx.h, vm.promql.ORDER_AGGR_FUNCS["outliers_iqr"], _p(dm), Sb, Pb, _u32(gb), G, None, 0, None,
                            _u8(ne), _u8(sel)))
    out["outliers nonempty"], out["outliers selected"] = env.snap(ne), env.snap(sel)
    return out


def e_transform(env, I):
    """vmb_transform (clamp, running_sum) and vmb_transform_range (range_normalize, range_quantile), in place"""
    vm, L = _vm(), _L()
    m = I["m"]
    S, P = m.shape
    d = env.dev_in(m)
    lo, hi = env.host_in(I["clamp"][0]), env.host_in(I["clamp"][1])
    _check(L.vmb_transform(env.ctx.h, vm.promql.TRANSFORM_FUNCS["clamp"], _p(d), S, P, _f64(lo), _f64(hi)))
    _check(L.vmb_transform(env.ctx.h, vm.promql.TRANSFORM_FUNCS["running_sum"], _p(d), S, P, None, None))
    r = env.dev_in(I["m2"])
    kept = env.host_out(S, np.uint8)
    _check(L.vmb_transform_range(env.ctx.h, vm.promql.RANGE_FUNCS["range_normalize"], _p(r), S, P, None, 0, _u8(kept)))
    out = {"elem": d, "normalize": r, "normalize kept": env.snap(kept)}
    q = env.dev_in(I["m"])
    phi = env.host_in(np.array([0.3]))
    _check(L.vmb_transform_range(env.ctx.h, vm.promql.RANGE_FUNCS["range_quantile"], _p(q), S, P, _f64(phi), 1, None))
    out["range_quantile"] = q
    return out


def e_histogram(env, I):
    """vmb_histogram (histogram_quantile with its bounds series), vmb_vmrange_to_le (count, then write), vmb_buckets_limit"""
    vm, L = _vm(), _L()
    h = I["hist"]
    n, P = h.shape
    G = I["hist_G"]
    dh = env.dev_in(h)
    groups, les = env.host_in(I["hist_groups"]), env.host_in(I["hist_les"])
    phis = env.host_in(I["phis"])
    d, lo, hi = env.dev_out(G, P), env.dev_out(G, P), env.dev_out(G, P)
    fl = env.host_out(3 * G, np.uint8)
    _check(L.vmb_histogram(env.ctx.h, vm.promql.HISTOGRAM_FUNCS["histogram_quantile"], _p(dh), n, P, _u32(groups), _f64(les), G,
                           _f64(phis), P, _p(d), _p(lo), _p(hi), _u8(fl)))
    out = {"quantile": d, "lower": lo, "upper": hi, "flags": env.snap(fl)}
    rows = env.host_out(n, np.uint32)
    dh = env.dev_in(h)
    nout = C.c_size_t(n)
    _check(L.vmb_buckets_limit(env.ctx.h, _p(dh), n, P, _u32(groups), _f64(les), G, 4, _u32(rows), C.byref(nout)))
    out["limit rows"] = env.snap(rows)[:nout.value]
    vr = I["vr"]
    dv = env.dev_in(vr)
    gids, starts, ends, skeys, ekeys = [env.host_in(a) for a in I["vr_args"]]
    ng = 4
    cnt = C.c_size_t(0)
    one_u32, one_u8 = env.host_out(1, np.uint32), env.host_out(1, np.uint8)
    rc = L.vmb_vmrange_to_le(env.ctx.h, _p(dv), vr.shape[0], P, _u32(gids), _f64(starts), _f64(ends), _u32(skeys), _u32(ekeys),
                             ng, None, C.byref(cnt), _u32(one_u32), _u8(one_u8), _u32(one_u32))
    _check(rc, allow=(-54,))
    k = cnt.value
    dout = env.dev_out(k, P)
    src, kind, le = env.host_out(k, np.uint32), env.host_out(k, np.uint8), env.host_out(k, np.uint32)
    _check(L.vmb_vmrange_to_le(env.ctx.h, _p(dv), vr.shape[0], P, _u32(gids), _f64(starts), _f64(ends), _u32(skeys), _u32(ekeys),
                               ng, _p(dout), C.byref(cnt), _u32(src), _u8(kind), _u32(le)))
    out.update({"vmrange": dout, "vmrange n": cnt.value, "vmrange src": env.snap(src), "vmrange kind": env.snap(kind),
                "vmrange le": env.snap(le)})
    return out


def e_topk(env, I):
    """topk: vmb_topk_candidates -> vmb_topk_merge (one part) -> vmb_topk_apply, in place, row flags to a host buffer"""
    L = _L()
    m = I["m"]
    S, P = m.shape
    G, kmax = int(I["groups"].max()) + 1, 3
    d = env.dev_in(m)
    groups = env.host_in(I["groups"])
    sizes = env.host_in(np.bincount(I["groups"], minlength=G).astype(np.uint32))
    ks = env.host_in(I["ks"])
    cand, cand2 = env.dev_out(G * P * kmax * 2), env.dev_out(G * P * kmax * 2)
    _check(L.vmb_topk_candidates(env.ctx.h, _p(d), S, P, _u32(groups), G, kmax, 0, 0, _p(cand)))
    _check(L.vmb_topk_merge(env.ctx.h, _p(cand), 1, G * P, kmax, 0, _p(cand2)))
    fl = env.host_out(S, np.uint8)
    _check(L.vmb_topk_apply(env.ctx.h, _p(d), S, P, _u32(groups), G, _u32(sizes), _p(cand2), kmax, _f64(ks), 0, 0, _u8(fl)))
    return {"vals": d, "flags": env.snap(fl), "cand": cand2}


def e_codec(env, I):
    """the write path and the per-call drop-ins: vmb_marshal_columns_gpu, vmb_float_to_decimal_columns,
    vmb_zstd_decompress_batch, vmb_unmarshal_int64, vmb_decimal_to_float"""
    L = _L()
    out = {}
    v = env.host_in(I["cols_i64"])
    nc, rows = v.shape
    cap = nc * rows * 10 + 4096
    dst, offs = env.host_out(cap, np.uint8), env.host_out(nc + 1, np.uint64)
    mts, firsts = env.host_out(nc, np.uint8), env.host_out(nc, np.int64)
    _check(L.vmb_marshal_columns_gpu(env.ctx.h, _u8(dst), cap, offs.ctypes.data_as(C.POINTER(C.c_uint64)), _u8(mts), _i64(firsts),
                                     _i64(v), nc, rows, 64, 2))
    offs = env.snap(offs)
    out.update({"marshal": env.snap(dst)[:int(offs[-1])], "marshal offs": offs, "marshal mts": env.snap(mts),
                "marshal firsts": env.snap(firsts)})
    f = env.host_in(I["cols_f64"])
    nc, rows = f.shape
    dd, sc = env.host_out((nc, rows), np.int64), env.host_out(nc, np.int16)
    _check(L.vmb_float_to_decimal_columns(env.ctx.h, _i64(dd), sc.ctypes.data_as(C.POINTER(C.c_int16)), _f64(f), nc, rows))
    out["to_decimal"], out["to_decimal scales"] = env.snap(dd), env.snap(sc)
    frames = I["frames"]
    fo = np.zeros(len(frames) + 1, dtype=np.uint64)
    fo[1:] = np.cumsum([b.vdata.size for b in frames])
    fr = env.host_in(np.concatenate([b.vdata for b in frames]))
    fo = env.host_in(fo)
    bound = C.c_uint64(0)
    _check(L.vmb_zstd_decompress_bound(_u8(fr), fo.ctypes.data_as(C.POINTER(C.c_uint64)), len(frames), C.byref(bound)))
    zd = env.host_out(max(bound.value, 1), np.uint8)
    zo, zl, zs = env.host_out(len(frames), np.uint64), env.host_out(len(frames), np.uint32), env.host_out(len(frames), np.int32)
    _check(L.vmb_zstd_decompress_batch(env.ctx.h, _u8(fr), fo.ctypes.data_as(C.POINTER(C.c_uint64)), len(frames), _u8(zd),
                                       zd.size, zo.ctypes.data_as(C.POINTER(C.c_uint64)), _u32(zl),
                                       zs.ctypes.data_as(C.POINTER(C.c_int32))))
    zd, zo, zl = env.snap(zd), env.snap(zo), env.snap(zl)
    out["zstd"] = np.concatenate([zd[int(o):int(o) + int(n)] for o, n in zip(zo, zl)])
    out["zstd lens"], out["zstd status"] = zl, env.snap(zs)
    b = I["unmarshal"]
    src = env.host_in(b.vdata)
    ud = env.host_out(b.rows, np.int64)
    _check(L.vmb_unmarshal_int64(env.ctx.h, _i64(ud), b.rows, _u8(src), src.size, b.vmt, b.first_value))
    out["unmarshal"] = env.snap(ud)
    va = env.host_in(I["decimals"])
    fd = env.host_out(va.size, np.float64)
    _check(L.vmb_decimal_to_float(env.ctx.h, _f64(fd), _i64(va), va.size, -3))
    out["to_float"] = env.snap(fd)
    return out


CATALOGUE = {"decode": e_decode, "fused": e_fused, "aggr_device": e_aggr_device, "rollup_host": e_rollup_host,
             "subquery": e_subquery, "binary": e_binary, "aggr_matrix": e_aggr_matrix, "transform": e_transform,
             "histogram": e_histogram, "topk": e_topk, "codec": e_codec}


def run_entry(env, name):
    return env.finish(CATALOGUE[name](env, inputs()))


def run_catalogue(env, order=None):
    res = {}
    for name in order or list(CATALOGUE):
        res[name] = run_entry(env, name)
    env.close()
    return res


# ------------------------------------------------------------------------------------------------ comparison
def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8) if a.dtype.kind in "fiub" else a


def differing(have, want):
    """indices of the elements whose bits differ"""
    return np.argwhere((_bits(have) != _bits(want)).reshape(want.shape + (-1,)).any(axis=-1))


def sum_within_bound(got, rows, groups):
    """EXCEPTIONS["fused sum"] of test_gpu_matrix_exact: the fused fold adds in the order its CTAs finish; every cell is within
    the error bound of recursive summation of the exact sum of its rows"""
    u = 2.0 ** -53
    bad = []
    for g in range(got.shape[0]):
        for p in range(got.shape[1]):
            col = rows[groups == g, p]
            col = col[~np.isnan(col)]
            if not len(col):
                if not np.isnan(got[g, p]):
                    bad.append((g, p, got[g, p], "nan"))
                continue
            n, A, exact = len(col), float(np.sum(np.abs(col))), math.fsum(col)
            if not abs(got[g, p] - exact) <= (n - 1) * u * A * (1 + 4 * n * u):
                bad.append((g, p, got[g, p], exact))
    return bad


def mismatches(got, ref, what, rows=None):
    """-> list of text lines, empty when every output equals the reference (sum: within the bound around `rows`, the serial
    run's rollup of the same blocks)"""
    out = []
    for entry, r in ref.items():
        g = got.get(entry)
        if g is None:
            out.append("%s %s: missing" % (what, entry))
            continue
        for k, want in r.items():
            have = g[k]
            if k == "aggr sum":
                bad = sum_within_bound(have, rows, inputs()["fused_groups"])
                if bad:
                    out.append("%s %s/%s: %d cells outside the bound, e.g. %s" % (what, entry, k, len(bad), bad[:3]))
                continue
            if isinstance(want, np.ndarray):
                same = want.shape == have.shape and want.dtype == have.dtype and np.array_equal(_bits(want), _bits(have))
            else:
                same = want == have
            if not same:
                detail = ""
                if isinstance(want, np.ndarray) and want.shape == have.shape and want.dtype == have.dtype:
                    diff = differing(have, want)
                    detail = "%d elements differ, first at %s: %r, want %r" % (len(diff), diff[0].tolist(),
                                                                               have[tuple(diff[0])], want[tuple(diff[0])])
                out.append("%s %s/%s differs: %s" % (what, entry, k, detail or (have, want)))
    return out


# ------------------------------------------------------------------------------------------------ environments
class _EnvVars:
    """VMB_FUSED_CHUNKS (read by vmb_ctx_create) and VMB_PIPE_CHUNK_BLOCKS (read by every vmb_eval_rollup_host call)"""

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in ("VMB_FUSED_CHUNKS", "VMB_PIPE_CHUNK_BLOCKS")}
        os.environ["VMB_FUSED_CHUNKS"] = str(FUSED_CHUNKS)
        os.environ["VMB_PIPE_CHUNK_BLOCKS"] = str(PIPE_CHUNK_BLOCKS)
        return self

    def __exit__(self, *a):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def serial_reference():
    vm = _vm()
    with _EnvVars():
        return run_catalogue(Env(vm.default_context()))


def stream_env(device=0):
    import torch
    vm = _vm()
    with torch.cuda.device(device):
        stream = torch.cuda.Stream(device=device)  # cudaStreamNonBlocking
    ctx = vm.Context(device, stream=stream.cuda_stream)
    return Env(ctx, stream, device)


def run_threads(k=K):
    """k contexts, one per thread and non-blocking stream, started together, each running the catalogue once in its own order
    -> ([results], [errors])"""
    import torch
    torch.cuda.init()
    names = list(CATALOGUE)
    barrier = threading.Barrier(k)
    results, errors = [None] * k, []

    def worker(i):
        env = None
        try:
            env = stream_env()
            barrier.wait(timeout=120)
            shift = i * len(names) // k
            results[i] = run_catalogue(env, names[shift:] + names[:shift])
        except BaseException as e:  # noqa: BLE001 -- reported by the caller
            errors.append("thread %d: %r" % (i, e))
            barrier.abort()
        finally:
            if env is not None:
                env.ctx.close()
    with _EnvVars():
        inputs()
        ts = [threading.Thread(target=worker, args=(i,)) for i in range(k)]
        for t in ts:
            t.start()
        for t in ts:
            t.join(timeout=600)
        assert not any(t.is_alive() for t in ts), "a worker thread did not finish"
    return results, errors


# ------------------------------------------------------------------------------------------------ tests
@pytest.fixture(scope="module")
def serial():
    return serial_reference()


@pytest.mark.gpu
def test_serial_reference_sane(serial):
    """the reference itself reached the paths it stands for: decode and zstd statuses clean, the pipeline wrote every row,
    the fused sum is within its bound"""
    assert (serial["decode"]["status"] == 0).all()
    assert (serial["codec"]["zstd status"] == 0).all()
    assert not (serial["rollup_host"]["out"].view(np.uint8) == SENT_BYTE).all(axis=-1).any()
    assert not sum_within_bound(serial["aggr_device"]["aggr sum"], serial["fused"]["fused"], inputs()["fused_groups"])
    assert np.array_equal(_bits(serial["fused"]["fused"]), _bits(serial["fused"]["unfused"]))


@pytest.mark.gpu
def test_fused_entry_runs_the_chunked_schedule():
    """the fused entry's batch has Huffman-literal frames past its first chunk, so a ctx made with VMB_FUSED_CHUNKS=4 runs
    the chunked schedule (zstd stage of the later chunks on the ctx's second stream, joined by events): more launches than
    a ctx made with VMB_FUSED_CHUNKS=1, and the same bits"""
    import torch
    vm = _vm()
    descs, payload = inputs()["fused"]
    rc = _rc(vm, inputs()["fused_cfg"])
    res = {}
    for chunks in (FUSED_CHUNKS, 1):
        old = os.environ.get("VMB_FUSED_CHUNKS")
        os.environ["VMB_FUSED_CHUNKS"] = str(chunks)
        try:
            ctx = vm.Context(0)
        finally:
            if old is None:
                os.environ.pop("VMB_FUSED_CHUNKS")
            else:
                os.environ["VMB_FUSED_CHUNKS"] = old
        try:
            B = vm.storage.Blocks(descs, payload, ctx)
            out = torch.full((len(descs), rc.points), SENT, dtype=torch.float64, device="cuda")
            n0 = ctx.launch_count
            _, sc = vm.promql.eval_rollup_func("rate", B, 0, 0, 0, rc=rc, out_dev_ptr=out.data_ptr())
            ctx.synchronize()
            res[chunks] = (ctx.launch_count - n0, out.cpu().numpy(), sc)
            B.close()
        finally:
            ctx.close()
    assert res[FUSED_CHUNKS][0] > res[1][0], "the fused entry ran one chunk: %s" % {c: r[0] for c, r in res.items()}
    assert np.array_equal(_bits(res[FUSED_CHUNKS][1]), _bits(res[1][1])) and res[FUSED_CHUNKS][2] == res[1][2]


@pytest.mark.gpu
@pytest.mark.parametrize("entry", list(CATALOGUE))
def test_caller_stream_pinned_buffers(serial, entry):
    """one ctx on a cudaStreamNonBlocking stream; host outputs pinned and read when the call returns; device inputs still in
    flight on that stream when the library is called; the only wait is an event on the caller's stream"""
    with _EnvVars():
        env = stream_env()
        try:
            got = {entry: run_entry(env, entry)}
            env.close()
        finally:
            env.ctx.close()
    bad = mismatches(got, {entry: serial[entry]}, "caller stream", serial["fused"]["fused"])
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
def test_concurrent_contexts(serial):
    """K contexts on K threads and streams, the catalogue once each in a rotated order"""
    results, errors = run_threads()
    assert not errors, errors
    bad = []
    for i, r in enumerate(results):
        bad += mismatches(r, serial, "thread %d" % i, serial["fused"]["fused"])
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
def test_concurrent_contexts_first_use():
    """the same in a fresh process, where the threads are the first to use the library: the zstd tables, the fused grid sizes
    and every ctx's second stream are made while the others run; the serial reference follows in that process"""
    env = dict(os.environ)
    args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "first-use"]
    p = subprocess.run(args, env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, (p.stdout[-4000:], p.stderr[-4000:])
    assert "first-use OK" in p.stdout, p.stdout[-4000:]


def _first_values(m, groups, G):
    """vmb_group_first_value's reference: per group and point the first non-NaN value in row order, math.NaN() if none"""
    want = np.full((G, m.shape[1]), GO_NAN)
    for g in range(G):
        sub = m[groups == g]
        has = ~np.isnan(sub)
        first = np.argmax(has, axis=0)
        cols = np.flatnonzero(has.any(axis=0))
        want[g, cols] = sub[first[cols], cols]
    return want


@pytest.mark.gpu
def test_scratch_growth_behind_async_call():
    """vmb_group_first_value returns with its kernel running and reading the ctx's group scratch: 2 groups x 64 points over
    60 k rows that are NaN but for the last row of each group, so every thread walks its whole group (milliseconds).  While
    it runs, topk over 200 k series and 5000 groups grows that scratch (cudaFree + cudaMalloc).  The first result must be the
    one computed from its own input."""
    import torch
    L = _L()
    rng = np.random.default_rng(SEED0 + 9200)
    S, P, G = 60_000, 64, 2
    groups = (np.arange(S) % G).astype(np.uint32)
    m = np.full((S, P), np.nan)
    m[S - G:] = rng.normal(scale=50.0, size=(G, P))
    m[S - G:, ::9] = np.nan  # points where a whole group is NaN
    want = _first_values(m, groups, G)
    env = stream_env()
    try:
        d = env.dev_in(m)
        hg = env.host_in(groups)
        out = env.dev_out(G, P)
        S2, G2 = 200_000, 5000
        big = env.dev_out(S2, 2)
        with torch.cuda.stream(env.stream):
            big.normal_()
        g2 = env.host_in((np.arange(S2) % G2).astype(np.uint32))
        cand = env.dev_out(G2 * 2 * 2 * 2)
        env.finish({})
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(env.stream)
        _check(L.vmb_group_first_value(env.ctx.h, _p(d), S, P, _u32(hg), G, _p(out)))
        e1.record(env.stream)
        pending = not env.stream.query()
        # no synchronisation: the group scratch grows far beyond the first call's CSR while its kernel runs
        _check(L.vmb_topk_candidates(env.ctx.h, _p(big), S2, 2, _u32(g2), G2, 2, 0, 0, _p(cand)))
        got = env.finish({"out": out})["out"]
        env.close()
    finally:
        env.ctx.close()
    ms = e0.elapsed_time(e1)
    assert pending and ms > 1.0, ("vmb_group_first_value's kernel was not running when the scratch grew", pending, ms)
    assert np.array_equal(_bits(got), _bits(want)), differing(got, want)[:5]


@pytest.mark.gpu
def test_destroy_one_ctx_while_another_runs(serial):
    """ctx B runs the fused rollup; then ctx A queues a binary operator behind a ~50 ms spin on its stream
    (vmb_binary_op without row lists returns at once), and B is destroyed while that is still pending.  A's result is the
    element-wise sum of its inputs and B's that of the serial run."""
    import torch
    I, L = inputs(), _L()
    rng = np.random.default_rng(SEED0 + 9300)
    x, y = rng.normal(scale=1e3, size=(500, 300)), rng.normal(scale=1e-3, size=(500, 300))
    x[:, ::7] = -0.0
    with _EnvVars():
        a, b = stream_env(), stream_env()
        try:
            try:
                got_b = run_entry(b, "fused")
                b.close()
                left, right = a.dev_in(x), a.dev_in(y)
                dst = a.dev_out(*x.shape)
                with torch.cuda.stream(a.stream):
                    torch.cuda._sleep(50 * SPIN)
                _check(L.vmb_binary_op(a.ctx.h, _vm().promql.BINARY_OPS["+"], 0, _p(left), None, _p(right), None, x.shape[0],
                                       x.shape[1], _p(dst)))
                pending = not a.stream.query()
            finally:
                b.ctx.close()
            got = a.finish({"sum": dst})
            a.close()
        finally:
            a.ctx.close()
    assert pending, "ctx A's work had finished before ctx B was destroyed"
    assert np.array_equal(_bits(got["sum"]), _bits(x + y)), differing(got["sum"], x + y)[:5]
    bad = mismatches({"fused": got_b}, {"fused": serial["fused"]}, "ctx B")
    assert not bad, "\n".join(bad)


def _thread_errors(calls):
    """calls[i]() -> its rc; every thread calls, waits for the others, then reads vmb_last_error -> [(rc, text)]"""
    k = len(calls)
    barrier = threading.Barrier(k)
    res = [None] * k

    def worker(i):
        rc = calls[i]()
        barrier.wait(timeout=60)  # every thread has set its error text before any reads one
        res[i] = (rc, _L().vmb_last_error().decode())
    ts = [threading.Thread(target=worker, args=(i,)) for i in range(k)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=120)
    return res


def test_last_error_is_per_thread():
    """host-only entry points (no device needed): each thread reads the error text of its own failed call"""
    from victoriametrics_b200 import _lib
    L = _L()
    bufs = [np.zeros(81 * 2 + 1 + i, dtype=np.uint8) for i in range(K)]
    outs = [(_lib.BlockDesc * 2)() for _ in range(K)]

    def call(i):
        return lambda: L.vmb_index_block_unmarshal(outs[i], None, 2, _u8(bufs[i]), bufs[i].size)
    res = _thread_errors([call(i) for i in range(K)])
    for i, (rc, text) in enumerate(res):
        assert rc == -1, (i, rc, text)  # VMB_ERR_SHORT_SRC
        assert text == "invalid number of block headers found: %d bytes; want 2 block headers" % bufs[i].size, (i, text)


@pytest.mark.gpu
def test_last_error_per_thread_and_ctx(serial):
    """threads on their own contexts fail argument checks made before any launch (a group id >= ngroups, topk k > kmax), each
    reads its own text; meanwhile one ctx decodes a corrupt block (VMB_ERR_BLOCK_FAILED) beside one running catalogue entries,
    whose results stay those of the serial run"""
    import torch
    torch.cuda.init()
    L = _L()
    envs = [stream_env() for _ in range(K)]
    try:
        S, P = 50, 7
        m = envs[0].dev_in(np.zeros((S, P)))
        outs = [e.dev_out(4, P) for e in envs]

        def bad_group(i):
            g = np.zeros(S, dtype=np.uint32)
            g[10 + i] = 4 + i  # >= ngroups = 4
            hg = envs[i].host_in(g)
            return lambda: L.vmb_group_first_value(envs[i].ctx.h, _p(m), S, P, _u32(hg), 4, _p(outs[i]))

        def bad_k(i):
            g = envs[i].host_in(np.zeros(S, dtype=np.uint32))
            sz = envs[i].host_in(np.array([S], dtype=np.uint32))
            ks = envs[i].host_in(np.full(P, 5.0 + i))
            return lambda: L.vmb_topk_apply(envs[i].ctx.h, _p(m), S, P, _u32(g), 1, _u32(sz), _p(outs[i]), 2, _f64(ks), 0, 0,
                                            _u8(envs[i].host_out(S, np.uint8)))
        envs[0].finish({})
        res = _thread_errors([bad_group(i) if i % 2 == 0 else bad_k(i) for i in range(K)])
        for i, (rc, text) in enumerate(res):
            assert rc == ERR_INVALID_ARG, (i, rc, text)
            want = ("group id %d of series %d out of range (4 groups)" % (4 + i, 10 + i) if i % 2 == 0 else
                    "topk: k = %g at point 0 keeps %d series of a group, but the candidate lists hold kmax = 2" % (5 + i, 5 + i))
            assert text == want, (i, text)
    finally:
        for e in envs:
            e.close()
            e.ctx.close()
    # a corrupt block on one ctx beside the catalogue on another
    dec = inputs()["dec_blocks"]
    victim = next(i for i, b in enumerate(dec) if b.vmt in (1, 4))
    blocks = list(dec)
    bad = blockgen.OBlock(dec[victim].ts, dec[victim].vals, dec[victim].scale, 64, victim)
    bad.vdata = bad.vdata.copy()
    bad.vdata[:4] = 0  # no zstd magic number: the frame is rejected, the block fails
    blocks[victim] = bad
    descs, payload = blockgen.to_blockset(blocks)
    barrier = threading.Barrier(2)
    out, errs = {}, []

    def corrupt():
        env = stream_env()
        try:
            h = _upload(env, descs, payload)
            barrier.wait(timeout=60)
            for _ in range(3):
                st = env.host_out(len(descs), np.int32)
                s = C.c_void_p()
                rc = L.vmb_decode_blocks(env.ctx.h, h, INT64_MIN, INT64_MAX, 0, st.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(s))
                out.setdefault("rc", []).append(rc)
                out.setdefault("status", []).append(env.snap(st))
                L.vmb_series_free(s)
            L.vmb_blocks_free(h)
            env.finish({})
            env.close()
        except BaseException as e:  # noqa: BLE001
            errs.append(repr(e))
            barrier.abort()
        finally:
            env.ctx.close()

    def clean():
        env = stream_env()
        try:
            barrier.wait(timeout=60)
            out["clean"] = {n: run_entry(env, n) for n in ("decode", "fused", "histogram")}
            env.close()
        except BaseException as e:  # noqa: BLE001
            errs.append(repr(e))
            barrier.abort()
        finally:
            env.ctx.close()
    with _EnvVars():  # set before the threads start: vmb_ctx_create reads the environment
        ts = [threading.Thread(target=f) for f in (corrupt, clean)]
        for t in ts:
            t.start()
        for t in ts:
            t.join(timeout=300)
    assert not errs, errs
    assert out["rc"] == [ERR_BLOCK_FAILED] * 3, out["rc"]
    for st in out["status"]:
        assert st[victim] != 0 and (np.delete(st, victim) == 0).all(), st
    bad = mismatches(out["clean"], {n: serial[n] for n in out["clean"]}, "beside a corrupt block")
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
def test_two_devices_in_one_process(serial):
    """one ctx per H100, concurrently, over the fused, zstd-sequence and histogram entries: the single-device results"""
    import torch
    if torch.cuda.device_count() < 2 or any(torch.cuda.get_device_capability(d) != (9, 0) for d in (0, 1)):
        pytest.skip("needs two H100s")
    names = ("fused", "decode", "histogram")
    res, errs = [None, None], []
    barrier = threading.Barrier(2)

    def worker(dev):
        env = None
        try:
            with torch.cuda.device(dev):
                env = stream_env(dev)
                barrier.wait(timeout=60)
                res[dev] = {n: run_entry(env, n) for n in names}
                env.close()
        except BaseException as e:  # noqa: BLE001
            errs.append("device %d: %r" % (dev, e))
            barrier.abort()
        finally:
            if env is not None:
                env.ctx.close()
    with _EnvVars():
        ts = [threading.Thread(target=worker, args=(d,)) for d in (0, 1)]
        for t in ts:
            t.start()
        for t in ts:
            t.join(timeout=300)
    assert not errs, errs
    bad = []
    for dev in (0, 1):
        bad += mismatches(res[dev], {n: serial[n] for n in names}, "device %d" % dev)
    assert not bad, "\n".join(bad)


def _first_use_main():
    """test_concurrent_contexts_first_use, in its own process: threads first, then the serial reference"""
    results, errors = run_threads()
    if errors:
        print("errors:", errors)
        return 1
    ref = serial_reference()
    bad = []
    for i, r in enumerate(results):
        bad += mismatches(r, ref, "thread %d" % i, ref["fused"]["fused"])
    if bad:
        print("\n".join(bad))
        return 1
    print("first-use OK: %d threads x %d entries" % (len(results), len(CATALOGUE)))
    return 0


if __name__ == "__main__":
    _here = os.path.dirname(os.path.abspath(__file__))
    sys.path[:0] = [_here, os.path.dirname(_here)]
    if sys.argv[1:] == ["first-use"]:
        sys.exit(_first_use_main())
