#!/usr/bin/env python3
"""Time vmb_aggr_matrix (aggr(q) by (...) on a device matrix) at the sizes of a large dashboard query.

Shapes: S = 100 000 series x P = 8172 points (6.5 GB) with G in {1, 8, 1024, S} groups for sum, avg, max, stddev and share, and
S = 1 000 000 x P = 1 (an instant query) with G in {1, 1024}, for sum.  P = 8172 runs the warp-per-strip kernel, P = 1 the
lane-per-cell one.  The matrix is generated on the device from a seed, about 1 % NaN; row r belongs to group r % G.

Per shape, one JSON line: the call time (host clock around the call, which ends in a device synchronise, after warm-up, over at
least --seconds of repeats), the kernel time (device time of the library's kernels from torch.profiler, in a run of its own), the
bytes the aggregate has to move (8 S P read + 8 G P written; share / zscore read the matrix twice and write 8 S P) and the
achieved rate over the kernel time as a share of 3.35 TB/s (the H100 SXM data sheet).  Parity: a 64-point column strip of the
timed output against tests/aggr_matrix_ref.py.  The card's name and power limit are read in the same run.

  python scripts/exp_aggr_matrix.py [--seconds 1] [--out results/exp_aggr_matrix.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.dont_write_bytecode = True

PEAK = 3.35e12
SHAPES = [(100_000, 8172, g, f) for f in ("sum", "avg", "max", "stddev", "share") for g in (1, 8, 1024, 100_000)]
SHAPES += [(1_000_000, 1, g, "sum") for g in (1, 1024)]


def card_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm_max = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": sm_max}
    except Exception as e:
        return {"error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--out", default="")
    a = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    import victoriametrics_b200 as vm
    from aggr_matrix_ref import aggr_matrix_ref

    assert torch.cuda.is_available(), "this measurement needs the GPU"
    card = card_info()
    print(json.dumps({"card": card, "torch_device": torch.cuda.get_device_name(0)}), flush=True)
    lines = []
    mats = {}
    for S, P, G, name in SHAPES:
        if (S, P) not in mats:
            mats.clear()
            torch.cuda.empty_cache()
            gen = torch.Generator(device="cuda").manual_seed(20261015 + S + P)
            m = torch.randn((S, P), dtype=torch.float64, device="cuda", generator=gen) * 100.0
            m[torch.rand((S, P), device="cuda", generator=gen) < 0.01] = float("nan")
            mats[(S, P)] = m
        m = mats[(S, P)]
        rows_out = name in ("share", "zscore")
        out = torch.empty((S if rows_out else G, P), dtype=torch.float64, device="cuda")
        groups = (np.arange(S) % G).astype(np.uint32)

        def call():
            vm.promql.aggr_matrix(name, m.data_ptr(), S, P, out.data_ptr(), groups, G)

        for _ in range(2):
            call()
        torch.cuda.synchronize()
        n, t0 = 0, time.perf_counter()
        while True:
            call()
            n += 1
            el = time.perf_counter() - t0
            if el >= a.seconds and n >= 3:
                break
        call_ms = el / n * 1e3
        reps = 3
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                call()
            torch.cuda.synchronize()
        kern = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and "k_ma_" in e.name:
                k = e.name.split("<")[0].replace("void ", "")
                kern[k] = kern.get(k, 0.0) + e.time_range.elapsed_us() / 1e3 / reps
        kernel_ms = sum(kern.values())
        nbytes = 8 * S * P * (3 if rows_out else 1) + (0 if rows_out else 8 * G * P)
        # parity on a 64-point strip (all of it at P = 1); with 1 % NaN no row is empty within the strip but not outside it
        p0 = (P // 2) & ~31 if P >= 64 else 0
        w = min(64, P)
        strip = m[:, p0:p0 + w].cpu().numpy()
        want, _ = aggr_matrix_ref(name, strip, groups, G)
        got = out[:, p0:p0 + w].cpu().numpy()
        gb, wb = got.view(np.uint64), want.view(np.uint64)
        nan_ok = np.array_equal(np.isnan(got), np.isnan(want))
        bits_ok = bool(nan_ok and np.array_equal(gb[~np.isnan(want)], wb[~np.isnan(want)]))
        rec = {"func": name, "S": S, "P": P, "G": G, "path": "strips" if P >= 32 else "cells", "call_ms": round(call_ms, 4),
               "calls": n, "kernel_ms": round(kernel_ms, 4), "kernels": {k: round(v, 4) for k, v in kern.items()},
               "bytes": nbytes, "kernel_GBps": round(nbytes / kernel_ms / 1e6, 1) if kernel_ms else None,
               "kernel_pct_of_3.35TBps": round(100 * nbytes / (kernel_ms * 1e-3) / PEAK, 1) if kernel_ms else None,
               "call_GBps": round(nbytes / call_ms / 1e6, 1), "parity_strip_bit_exact": bits_ok,
               "card": card.get("name"), "power_limit": card.get("power_limit")}
        print(json.dumps(rec), flush=True)
        lines.append(rec)
        del out
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")
    return 0 if all(r["parity_strip_bit_exact"] for r in lines) else 1


if __name__ == "__main__":
    sys.exit(main())
