#!/usr/bin/env python3
"""Time vmb_transform's date-time functions (hour ... year) and bitmap functions (bitmap_and / or / xor) at the size of a large
dashboard query: S = 100 000 series x P = 8172 points (6.5 GB), on three seeded inputs:
  realistic   unix seconds uniform in 1.5e9 .. 2e9 with millisecond fractions, 5 % NaN;
  full_range  whole seconds uniform over all of int64 (the wrap region included), no NaN;
  bitmap      32-bit status words, with a per-point second argument of 16-bit masks.
The date-time functions run on the first two, the bitmap functions on the third, and `abs` on all three as the yardstick: the
same one read and one write of 8 bytes per cell.

The functions work in place, so every call gets a fresh device copy of the input first; that copy is outside every timing.
Per (function, input), one JSON line:
  call_ms    host clock around the call, which ends in a device synchronise, after one warm-up call, median of --repeats calls;
  kernel_ms  device time of the transform kernel from torch.profiler, in a profiled call of its own;
  GBps       16 S P bytes over kernel time, and that rate as a share of the H100 SXM data-sheet HBM3 bandwidth, 3.35 TB/s
             (3.9 ms at that rate);
  parity     rows 0, S/2 and S-1 compared bit for bit with tests/datetime_ref.py.
The card's name and power limit are read in the same run.

  python scripts/exp_datetime.py [--repeats 5] [--only hour,year] [--out results/exp_datetime.jsonl]
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

S, P = 100_000, 8172
HBM_BPS = 3.35e12


def card_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm_max = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": sm_max}
    except Exception as e:
        return {"error": repr(e)}


def make_input(kind, gen):
    import torch
    if kind == "realistic":
        m = torch.rand((S, P), dtype=torch.float64, device="cuda", generator=gen) * 5e8 + 1.5e9
        m = torch.round(m * 1e3) / 1e3
        m[torch.rand((S, P), device="cuda", generator=gen) < 0.05] = float("nan")
        return m
    if kind == "full_range":
        return torch.randint(-(1 << 63), (1 << 63) - 1, (S, P), dtype=torch.int64, device="cuda", generator=gen).double()
    return torch.randint(0, 1 << 32, (S, P), dtype=torch.int64, device="cuda", generator=gen).double()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--only", default="")
    ap.add_argument("--out", default="")
    a = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    import datetime_ref as R
    import victoriametrics_b200 as vm

    assert torch.cuda.is_available(), "this measurement needs the GPU"
    card = card_info()
    print(json.dumps({"card": card, "torch_device": torch.cuda.get_device_name(0)}), flush=True)
    only = set(a.only.split(",")) if a.only else None
    gen = torch.Generator(device="cuda").manual_seed(20261018)
    w = np.random.default_rng(20261018).integers(0, 1 << 16, P).astype(np.float64)
    check_rows = [0, S // 2, S - 1]
    plan = [("realistic", ["abs"] + R.DATETIME_FUNCS), ("full_range", ["abs"] + R.DATETIME_FUNCS), ("bitmap", ["abs"] + R.BITMAP_FUNCS)]
    lines = []
    for kind, names in plan:
        src = make_input(kind, gen)
        work = torch.empty_like(src)
        host_rows = src[check_rows].cpu().numpy()
        for name in names:
            if only and name not in only and name != "abs":
                continue
            args = (w,) if name in R.BITMAP_FUNCS else ()

            def call():
                vm.promql.transform(name, work.data_ptr(), S, P, *args)
                torch.cuda.synchronize()

            times = []
            for i in range(a.repeats + 1):
                work.copy_(src)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                call()
                if i:
                    times.append((time.perf_counter() - t0) * 1e3)
            work.copy_(src)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                call()
            kern = {}
            for e in prof.events():
                if e.device_type == torch.autograd.DeviceType.CUDA and "k_transform" in e.name:
                    k = e.name.split("(")[0].replace("void ", "")
                    kern[k] = kern.get(k, 0.0) + e.time_range.elapsed_us() / 1e3
            kernel_ms = sum(kern.values())
            moved = 16 * S * P
            rec = {"func": name, "input": kind, "S": S, "P": P, "call_ms_median": round(float(np.median(times)), 3),
                   "call_ms": [round(t, 3) for t in times], "kernel_ms": round(kernel_ms, 3), "kernels": kern,
                   "GBps": round(moved / kernel_ms / 1e6, 1), "share_of_3.35TBps": round(moved / kernel_ms / 1e-3 / HBM_BPS, 3),
                   "card": card.get("name"), "power_limit": card.get("power_limit")}
            got = work[check_rows].cpu().numpy()
            want = np.abs(host_rows) if name == "abs" else R.np_ref(name, host_rows, w)
            rec["parity_rows"] = bool(np.array_equal(got.view(np.uint64), want.view(np.uint64)))
            print(json.dumps(rec), flush=True)
            lines.append(rec)
        del src, work
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")
    return 0 if all(r["parity_rows"] for r in lines) else 1


if __name__ == "__main__":
    sys.exit(main())
