#!/usr/bin/env python3
"""Time vmb_aggr_histogram and vmb_rollup_histogram at the sizes of a large dashboard query.
histogram(q) by (...): S = 100 000 series x P = 8172 points (6.5 GB) of uniform values in [0, 1000) and of log-normal "latencies"
(median 50 ms, sigma 0.3: most of a group's rows in a few buckets at every point), 5 % NaN, rows dealt round robin to G = 1, 8
and 1024 groups.  G = S does not fit at this size: every row hits about 19 (latency) or 60 (uniform) buckets over 8172 points, an
output of 124 GB or more.  Yardstick: vmb_aggr_matrix
SUM on the same matrix, one read of it.  The floor is one read of the matrix, 8·S·P bytes at 3.35 TB/s.
histogram_over_time(m[5m]) at step 15 s: the count_values_over_time batch of exp_count_values.py (20 000 reference-encoded gauge
series x 8192 samples at 15 s, 6 distinct values), decoded by vmb_decode_blocks.  Yardstick: vmb_rollup_count_values on the same
batch.
Per case, one JSON line:
  count_ms   host clock around the sizing call (d_out == NULL), which ends in a device synchronise;
  call_ms    the same around the call that writes the matrix; median of --repeats after one warm-up;
  kernels    device time per kernel from torch.profiler in a profiled call of its own;
  floor_share  8·S·P / 3.35 TB/s over the kernel time of the writing call.
The card's name and power limit are read in the same run.
  python scripts/exp_vm_histogram.py [--repeats 3] [--only aggr,rollup] [--out results/exp_vm_histogram.jsonl]
"""
import argparse
import copy
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.dont_write_bytecode = True
from exp_rank_aggr import card_info  # noqa: E402

S, P = 100_000, 8172
HBM = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--only", default="aggr,rollup")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    import victoriametrics_b200 as vm
    from blockgen import OBlock, to_blockset
    assert torch.cuda.is_available(), "this measurement needs the GPU"
    card = card_info()
    print(json.dumps({"card": card, "torch_device": torch.cuda.get_device_name(0)}), flush=True)
    lines = []
    lib, ctx = vm._lib.lib(), vm._lib.default_context()
    u32 = lambda x: x.ctypes.data_as(vm._lib.u32p)

    def profiled(fn):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        kern = {}
        for e in prof.events():
            if e.device_type != torch.autograd.DeviceType.CUDA:
                continue
            k = e.name.split("(")[0].replace("void ", "")
            kern[k] = kern.get(k, 0.0) + e.time_range.elapsed_us() / 1e3
        return {k: round(v, 3) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])}

    def timed(fn):
        times = []
        for i in range(a.repeats + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            if i:
                times.append(round((time.perf_counter() - t0) * 1e3, 2))
        return times

    def emit(rec):
        rec.update(card=card.get("name"), power_limit=card.get("power_limit"))
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    if "aggr" in a.only.split(","):
        gen = torch.Generator(device="cuda").manual_seed(20261018)
        for dist in ("uniform", "latency"):
            if dist == "uniform":
                src = torch.rand((S, P), dtype=torch.float64, device="cuda", generator=gen) * 1000
            else:
                src = torch.exp(torch.randn((S, P), dtype=torch.float64, device="cuda", generator=gen) * 0.3 + np.log(0.05))
            src[torch.rand((S, P), device="cuda", generator=gen) < 0.05] = float("nan")
            for G in (1, 8, 1024):
                gids = (np.arange(S) % G).astype(np.uint32)
                nout = C.c_size_t(0)
                grp, bkt = np.zeros(1, dtype=np.uint32), np.zeros(1, dtype=np.uint32)

                def count():
                    nout.value = 0
                    assert lib.vmb_aggr_histogram(ctx.h, C.c_void_p(src.data_ptr()), S, P, u32(gids), G, None, C.byref(nout),
                                                  u32(grp), u32(bkt)) == -54
                count()
                n = nout.value
                out = torch.empty((max(n, 1), P), dtype=torch.float64, device="cuda")
                g2, b2 = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint32)

                def call():
                    nout.value = n
                    assert lib.vmb_aggr_histogram(ctx.h, C.c_void_p(src.data_ptr()), S, P, u32(gids), G, C.c_void_p(out.data_ptr()),
                                                  C.byref(nout), u32(g2), u32(b2)) == 0
                count_ms, call_ms = timed(count), timed(call)
                kern = profiled(call)
                ok = float(out[:n].sum().item()) == float((~torch.isnan(src)).sum().item())  # every non-NaN value is >= 0
                yard = torch.empty((G, P), dtype=torch.float64, device="cuda")
                flags = np.zeros(S, dtype=np.uint8)

                def total():
                    assert lib.vmb_aggr_matrix(ctx.h, 0, C.c_void_p(src.data_ptr()), S, P, u32(gids), G, C.c_void_p(yard.data_ptr()),
                                               flags.ctypes.data_as(vm._lib.u8p)) == 0
                yard_ms = timed(total)
                ykern = profiled(total)
                kms = sum(kern.values())
                emit({"case": "histogram", "values": dist, "S": S, "P": P, "G": G, "rows_out": n, "out_bytes": n * P * 8,
                      "count_ms": count_ms, "call_ms": call_ms, "kernel_ms": round(kms, 2), "kernels": kern,
                      "floor_ms": round(8 * S * P / HBM * 1e3, 2), "floor_share": round(8 * S * P / HBM * 1e3 / kms, 3),
                      "counts_sum_ok": ok, "yardstick_sum_call_ms": yard_ms, "yardstick_sum_kernel_ms": round(sum(ykern.values()), 2)})
                del out, yard
                torch.cuda.empty_cache()
            del src
            torch.cuda.empty_cache()

    if "rollup" in a.only.split(","):
        rng = np.random.default_rng(20261017)
        NS, rows, dt = 20_000, 8192, 15_000
        t0 = 1_700_000_000_000
        ts = t0 + dt * np.arange(rows, dtype=np.int64)
        base = [OBlock(ts, rng.integers(0, 6, rows).astype(np.int64) * 25, -1) for _ in range(64)]
        blocks = []
        for s in range(NS):
            b = copy.copy(base[s % 64])
            b.series_idx = s
            blocks.append(b)
        descs, payload = to_blockset(blocks)
        blk = vm.storage.Blocks(descs, payload)
        cfg = vm.promql.count_values_over_time_config(t0, t0 + dt * (rows - 1), 15_000, 300_000)
        pts = rows
        for name, fn, outarr in (("histogram_over_time", lib.vmb_rollup_histogram, np.uint32),
                                 ("count_values_over_time", lib.vmb_rollup_count_values, np.float64)):
            series, _ = vm.storage.decode_blocks(blk)
            nout, scanned = C.c_size_t(0), C.c_uint64(0)
            ser, key = np.zeros(1, dtype=np.uint32), np.zeros(1, dtype=outarr)
            ptr = (lambda x: x.ctypes.data_as(vm._lib.u32p)) if outarr is np.uint32 else (lambda x: x.ctypes.data_as(vm._lib.f64p))

            def count():
                nout.value = 0
                assert fn(ctx.h, series.h, C.byref(cfg), None, C.byref(nout), u32(ser), ptr(key), C.byref(scanned)) == -54
            count()
            n = nout.value
            out = torch.empty((n, pts), dtype=torch.float64, device="cuda")
            ser2, key2 = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=outarr)

            def call():
                nout.value = n
                assert fn(ctx.h, series.h, C.byref(cfg), C.c_void_p(out.data_ptr()), C.byref(nout), u32(ser2), ptr(key2),
                          C.byref(scanned)) == 0
            count_ms, call_ms = timed(count), timed(call)
            kern = profiled(call)
            emit({"case": name, "series": NS, "samples": rows, "points": pts, "rows_out": n, "out_bytes": n * pts * 8,
                  "samples_scanned": scanned.value, "count_ms": count_ms, "call_ms": call_ms,
                  "kernel_ms": round(sum(kern.values()), 2), "kernels": kern})
            del out
            series.close()
            torch.cuda.empty_cache()
        blk.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
