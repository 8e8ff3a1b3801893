#!/usr/bin/env python3
"""Write path timing: vmb_marshal_columns_gpu end to end (host int64 columns in, host payload / offsets / types out) beside
vmb_marshal_columns on all host threads, and vmb_zstd_compress_batch alone in input GB/s, on three inputs of 100 000 columns x
8192 rows: bench.py configs[1]'s counters, gauges (round(N(5000, 300))) and jittered timestamps (t0 + 15 s * i + U[-50, 50] ms).

It calls the library through ctypes by path (--lib), so the same script times an older build of the library beside this one:
run it once per library, alternating, in the same session.  vmb_zstd_compress_batch is timed where the library has it.  Every
device result is checked against the host encoder's before it is timed.  Prints the card, its power limit and the host thread
count, then one JSON line."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gen(kind, ncols, rows, seed):
    import bench
    O, L = bench.oracle()
    if kind == "timestamps":
        rng = np.random.default_rng(seed)
        ts = bench.T0 + bench.SCRAPE_MS * np.arange(rows, dtype=np.int64)
        return ts[None, :] + rng.integers(-50, 51, (ncols, rows))
    pool = bench.get_pool(bench.host_threads())
    v = np.empty((ncols, rows), dtype=np.int64)
    assert L.vmo_pool_gen_values(pool, bench.KIND_ID[kind], 0, ncols, rows, seed, v.ctypes.data_as(O.i64p)) == 0
    return v


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(ROOT, "victoriametrics_b200", "libvmb200.so"))
    ap.add_argument("--ncols", type=int, default=100_000)
    ap.add_argument("--rows", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-reps", type=int, default=2)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    nthreads = os.cpu_count() or 1
    L = C.CDLL(a.lib)
    vp, sz, u8p, u64p, i64p = C.c_void_p, C.c_size_t, C.POINTER(C.c_uint8), C.POINTER(C.c_uint64), C.POINTER(C.c_int64)
    L.vmb_ctx_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.vmb_marshal_columns.argtypes = [u8p, sz, u64p, u8p, i64p, i64p, sz, sz, C.c_uint8, C.c_int]
    L.vmb_marshal_columns_gpu.argtypes = [vp, u8p, sz, u64p, u8p, i64p, i64p, sz, sz, C.c_uint8, C.c_int]
    has_batch = hasattr(L, "vmb_zstd_compress_batch")
    if has_batch:
        L.vmb_zstd_compress_batch.argtypes = [vp, u8p, u64p, sz, u8p, sz, u64p]
    ctx = vp()
    assert L.vmb_ctx_create(0, C.byref(ctx)) == 0
    ncols, rows = a.ncols, a.rows
    res = {"lib": a.lib, "gpu": smi, "host_threads": nthreads, "ncols": ncols, "rows": rows, "inputs": {}}
    print("card, power limit, max SM clock: %s; host threads: %d; library %s" % (smi, nthreads, a.lib), flush=True)
    for seed, kind in enumerate(("counter", "gauge", "timestamps")):
        v = gen(kind, ncols, rows, 1000 + seed)
        cap = ncols * (rows * 3 + 64)
        outs = {}
        for name in ("gpu", "host"):
            dst = np.empty(cap, dtype=np.uint8)
            offs = np.zeros(ncols + 1, dtype=np.uint64)
            mts = np.zeros(ncols, dtype=np.uint8)
            firsts = np.zeros(ncols, dtype=np.int64)
            args = (dst.ctypes.data_as(u8p), cap, offs.ctypes.data_as(u64p), mts.ctypes.data_as(u8p), firsts.ctypes.data_as(i64p),
                    v.ctypes.data_as(i64p), ncols, rows, 64, nthreads)
            call = (lambda: L.vmb_marshal_columns_gpu(ctx, *args)) if name == "gpu" else (lambda: L.vmb_marshal_columns(*args))
            assert call() == 0  # warm-up (and the result compared below)
            ts = []
            for _ in range(a.reps if name == "gpu" else a.host_reps):
                t = time.perf_counter()
                assert call() == 0
                ts.append(time.perf_counter() - t)
            outs[name] = (dst[:int(offs[-1])].copy(), offs.copy(), mts.copy(), firsts.copy(), float(np.median(ts)))
        g, h = outs["gpu"], outs["host"]
        assert all(np.array_equal(x, y) for x, y in zip(g[:4], h[:4])), kind
        r = {"marshal_gpu_ms": g[4] * 1e3, "marshal_host_ms": h[4] * 1e3, "payload_bytes": int(g[1][-1]),
             "types": {int(t): int(c) for t, c in zip(*np.unique(g[2], return_counts=True))}}
        if has_batch:
            streams = _streams(L, v, ncols, rows, u8p, u64p, i64p, nthreads)
            src = np.concatenate(streams)
            so = np.zeros(len(streams) + 1, dtype=np.uint64)
            so[1:] = np.cumsum([s.size for s in streams])
            dcap = src.size + len(streams) * 16
            dst = np.empty(dcap, dtype=np.uint8)
            do = np.zeros(len(streams) + 1, dtype=np.uint64)
            bargs = (ctx, src.ctypes.data_as(u8p), so.ctypes.data_as(u64p), len(streams), dst.ctypes.data_as(u8p), dcap,
                     do.ctypes.data_as(u64p))
            assert L.vmb_zstd_compress_batch(*bargs) == 0
            ts = []
            for _ in range(a.reps):
                t = time.perf_counter()
                assert L.vmb_zstd_compress_batch(*bargs) == 0
                ts.append(time.perf_counter() - t)
            r["zstd_batch_ms"] = float(np.median(ts)) * 1e3
            r["zstd_batch_input_gbps"] = src.size / float(np.median(ts)) / 1e9
            r["zstd_batch_frames"] = len(streams)
            r["zstd_batch_input_bytes"] = int(src.size)
        res["inputs"][kind] = r
        print(kind, json.dumps(r), flush=True)
        del v, outs
    print(json.dumps(res))


def _streams(L, v, ncols, rows, u8p, u64p, i64p, nthreads):
    """the varint stream of every column of MarshalType 1 / 4 / 5 / 6 (what the zstd stage compresses): the host encoder's
    payload where it kept the stream (5 / 6), the stream decompressed from its frame where it kept the frame (1 / 4)"""
    import victoriametrics_b200 as vm
    cap = ncols * (rows * 3 + 64)
    dst = np.empty(cap, dtype=np.uint8)
    offs = np.zeros(ncols + 1, dtype=np.uint64)
    mts = np.zeros(ncols, dtype=np.uint8)
    firsts = np.zeros(ncols, dtype=np.int64)
    assert L.vmb_marshal_columns(dst.ctypes.data_as(u8p), cap, offs.ctypes.data_as(u64p), mts.ctypes.data_as(u8p),
                                 firsts.ctypes.data_as(i64p), v.ctypes.data_as(i64p), ncols, rows, 64, nthreads) == 0
    kept = [dst[int(offs[c]):int(offs[c + 1])] for c in range(ncols) if mts[c] in (5, 6) and offs[c + 1] > offs[c]]
    framed = [dst[int(offs[c]):int(offs[c + 1])] for c in range(ncols) if mts[c] in (1, 4)]
    out = list(kept)
    for i in range(0, len(framed), 20000):
        out += vm.encoding.decompress_zstd_batch(framed[i:i + 20000])
    return out


if __name__ == "__main__":
    main()
