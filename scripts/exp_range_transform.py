#!/usr/bin/env python3
"""Time vmb_transform_range (the whole-series transforms on a device matrix) and smooth_exponential at the size of a large
dashboard query: S = 100 000 series x P = 8172 points (6.5 GB), gauge-like values (a seeded random walk per row) with 5 % NaN.

The functions work in place, so every call gets a fresh device copy of the input first; that copy is outside every timing.
Per function, one JSON line:
  call_ms    host clock around the call, which ends in a device synchronise, after one warm-up call, median of --repeats calls;
  kernels    device time per kernel from torch.profiler, in a profiled call of its own;
  moment functions (stddev, stdvar, zscore, trim_zscore, normalize, linear_regression) and smooth_exponential: the bytes their
             passes move as computed from the shape -- the reduction reads the matrix (8 S P), the rewrite reads (except stddev /
             stdvar) and writes it (8 S P each) -- over kernel time, and that rate as a share of the H100 SXM data-sheet HBM3
             bandwidth, 3.35 TB/s;
  order functions (quantile, mad, trim_outliers, trim_spikes): the share of kernel time spent in the sort (k_oa_block_sort +
             k_oa_merge);
  parity     three rows compared with tests/range_transform_ref.py (== on values, NaN for NaN).
One more line times vmb_aggr_order quantiles (one phi, one group: 8172 cells of 100 000 keys) on the same matrix: the same key
count through the same sort, as a yardstick.  The card's name and power limit are read in the same run.

  python scripts/exp_range_transform.py [--repeats 5] [--only range_quantile,range_mad] [--out results/exp_range_transform.jsonl]
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

S, P, STEP = 100_000, 8172, 15_000
HBM_BPS = 3.35e12
MOMENTS = ["range_stddev", "range_stdvar", "range_zscore", "range_trim_zscore", "range_normalize", "range_linear_regression"]
ORDER = ["range_quantile", "range_mad", "range_trim_outliers", "range_trim_spikes"]
ARGS = {"range_trim_zscore": 2.0, "range_quantile": 0.9, "range_trim_outliers": 3.0, "range_trim_spikes": 0.1,
        "smooth_exponential": 0.2}


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
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--only", default="")
    ap.add_argument("--out", default="")
    a = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    import victoriametrics_b200 as vm
    from range_transform_ref import range_transform_ref, smooth_exponential_ref

    assert torch.cuda.is_available(), "this measurement needs the GPU"
    card = card_info()
    print(json.dumps({"card": card, "torch_device": torch.cuda.get_device_name(0)}), flush=True)
    gen = torch.Generator(device="cuda").manual_seed(20261016)
    src = 1000 + torch.cumsum(torch.randn((S, P), dtype=torch.float64, device="cuda", generator=gen), dim=1)
    src[torch.rand((S, P), device="cuda", generator=gen) < 0.05] = float("nan")
    work = torch.empty_like(src)
    check_rows = [0, S // 2, S - 1]
    host_rows = src[check_rows].cpu().numpy()
    only = set(a.only.split(",")) if a.only else None
    names = [n for n in MOMENTS + ["smooth_exponential"] + ORDER + ["aggr_order_quantile"] if not only or n in only]
    out = torch.empty((1, 1, P), dtype=torch.float64, device="cuda")
    lines = []
    for name in names:
        arg = ARGS.get(name)

        def call():
            if name == "smooth_exponential":
                vm.promql.transform(name, work.data_ptr(), S, P, arg)
            elif name == "aggr_order_quantile":
                vm.promql.aggr_order("quantiles", work.data_ptr(), S, P, out.data_ptr(), phis=[0.9])
            else:
                vm.promql.transform_range(name, work.data_ptr(), S, P, *(() if arg is None else (arg,)), step=STEP)
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
            if e.device_type == torch.autograd.DeviceType.CUDA and ("k_rs_" in e.name or "k_oa_" in e.name or "k_transform" in e.name):
                k = e.name.split("(")[0].replace("void ", "")
                kern[k] = kern.get(k, 0.0) + e.time_range.elapsed_us() / 1e3
        kernel_ms = sum(kern.values())
        rec = {"func": name, "S": S, "P": P, "arg": arg, "call_ms_median": round(float(np.median(times)), 3),
               "call_ms": [round(t, 3) for t in times], "kernel_ms": round(kernel_ms, 3),
               "kernels": {k: round(v, 3) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])},
               "card": card.get("name"), "power_limit": card.get("power_limit")}
        if name in MOMENTS or name == "smooth_exponential":
            cells = 8 * S * P
            if name == "smooth_exponential":
                moved = 2 * cells  # one read and one write in the row walk
            else:
                moved = cells + (cells if name in ("range_stddev", "range_stdvar") else 2 * cells)
            rec["bytes"] = moved
            rec["GBps"] = round(moved / kernel_ms / 1e6, 1)
            rec["share_of_3.35TBps"] = round(moved / kernel_ms / 1e-3 / HBM_BPS, 3)
        else:
            sort_ms = sum(v for k, v in kern.items() if "k_oa_block_sort" in k or "k_oa_merge" in k)
            rec["sort_ms"] = round(sort_ms, 3)
            rec["sort_share"] = round(sort_ms / kernel_ms, 3)
        if name != "aggr_order_quantile":
            got = work[check_rows].cpu().numpy()
            if name == "smooth_exponential":
                want = smooth_exponential_ref(host_rows, arg)
            else:
                want, _ = range_transform_ref(name, host_rows, arg, STEP)
            rec["parity_rows"] = bool(np.array_equal(np.isnan(got), np.isnan(want)) and
                                      np.array_equal(got[~np.isnan(got)], want[~np.isnan(want)]))
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")
    return 0 if all(r.get("parity_rows", True) for r in lines) else 1


if __name__ == "__main__":
    sys.exit(main())
