#!/usr/bin/env python3
"""Time vmb_aggr_rank (topk_avg ... bottomk_last, outliersk on a device matrix) at the size of a large dashboard query:
S = 100 000 series x P = 8172 points (6.5 GB), gauge-like values (a seeded random walk per row) with 5 % NaN, k = 5, in G = 1, 8
and 1024 groups (rows dealt round robin); and at S = 1 000 000 x P = 1 (an instant query), where the host's ranking dominates.

The call masks the surviving rows in place, so every call gets a fresh device copy of the input first; that copy is outside every
timing.  Per case, one JSON line:
  call_ms    host clock around the call, which ends in a device synchronise, after one warm-up call, median of --repeats calls;
  kernels    device time per kernel from torch.profiler, in a profiled call of its own, and their sums by step: score (k_rk_scores,
             or k_rs_keys + k_rk_median), sort (k_oa_block_sort + k_oa_merge), medians (outliersk: k_oa_gather + k_oa_finish),
             remaining (k_ma_fold_* + k_ma_fixup), mask (k_rk_mask);
  host_ms    call_ms minus the kernel time: the ranking on the host, the copies and the launches;
  score pass of min / max / avg / last: the 8 S P bytes it reads over its kernel time, and that rate as a share of the H100 SXM
             data-sheet HBM3 bandwidth, 3.35 TB/s; the same for the remaining-sum fold, which reads the matrix once more;
  rows_written  the rows the call changed (at most k x G), counted by comparing the matrix with the input;
  parity     the scores of three rows compared with tests/rank_aggr_ref.py (== on values, NaN for NaN; not for outliersk).
The card's name and power limit are read in the same run.

  python scripts/exp_rank_aggr.py [--repeats 5] [--only topk_avg,outliersk] [--out results/exp_rank_aggr.jsonl]
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

S, P, K = 100_000, 8172, 5
HBM_BPS = 3.35e12
# (function, groups, remaining sum)
CASES = [("topk_avg", 1, False), ("topk_avg", 8, False), ("topk_avg", 1024, False), ("topk_avg", 1, True), ("topk_avg", 8, True),
         ("topk_avg", 1024, True), ("topk_min", 8, False), ("bottomk_max", 8, False), ("topk_last", 8, False),
         ("topk_median", 8, False), ("outliersk", 8, False)]
STEPS = {"k_rk_scores": "score", "k_rs_keys": "score", "k_rk_median": "score", "k_oa_block_sort": "sort", "k_oa_merge": "sort",
         "k_oa_gather": "medians", "k_oa_finish": "medians", "k_ma_fold": "remaining", "k_ma_fixup": "remaining", "k_rk_mask": "mask"}


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
    from rank_aggr_ref import scores_of

    assert torch.cuda.is_available(), "this measurement needs the GPU"
    card = card_info()
    print(json.dumps({"card": card, "torch_device": torch.cuda.get_device_name(0)}), flush=True)
    only = set(a.only.split(",")) if a.only else None
    lines = []

    def measure(name, s, p, G, remaining, src, work, host_rows, check_rows):
        groups = (np.arange(s) % G).astype(np.uint32)
        rem = torch.empty((G, p), dtype=torch.float64, device="cuda") if remaining else None
        got = {}

        def call():
            got["out"], got["scores"] = vm.promql.aggr_rank(name, K, work.data_ptr(), s, p, groups, G,
                                                            rem.data_ptr() if remaining else None)
            torch.cuda.synchronize()

        times = []
        for i in range(a.repeats + 1):
            work.copy_(src)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            call()
            if i:
                times.append((time.perf_counter() - t0) * 1e3)
        rows_written = int((work.view(torch.int64) != src.view(torch.int64)).any(dim=1).sum().item())
        work.copy_(src)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
        kern, steps = {}, {}
        for e in prof.events():
            if e.device_type != torch.autograd.DeviceType.CUDA:
                continue
            for prefix, step in STEPS.items():
                if prefix in e.name:
                    k = e.name.split("(")[0].replace("void ", "")
                    ms = e.time_range.elapsed_us() / 1e3
                    kern[k] = kern.get(k, 0.0) + ms
                    steps[step] = steps.get(step, 0.0) + ms
                    break
        kernel_ms = sum(kern.values())
        call_ms = float(np.median(times))
        rec = {"func": name, "S": s, "P": p, "G": G, "k": K, "remaining_sum": remaining, "call_ms_median": round(call_ms, 3),
               "call_ms": [round(t, 3) for t in times], "kernel_ms": round(kernel_ms, 3), "host_ms": round(call_ms - kernel_ms, 3),
               "steps_ms": {k: round(v, 3) for k, v in steps.items()},
               "kernels": {k: round(v, 3) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])},
               "rows_written": rows_written, "rows_out": int((got["out"] >= 0).sum()),
               "card": card.get("name"), "power_limit": card.get("power_limit")}
        cells = 8 * s * p
        if name.split("_")[-1] in ("min", "max", "avg", "last") and steps.get("score"):
            rec["score_GBps"] = round(cells / steps["score"] / 1e6, 1)
            rec["score_share_of_3.35TBps"] = round(cells / steps["score"] / 1e-3 / HBM_BPS, 3)
        if remaining and steps.get("remaining"):
            rec["remaining_GBps"] = round(cells / steps["remaining"] / 1e6, 1)
            rec["remaining_share_of_3.35TBps"] = round(cells / steps["remaining"] / 1e-3 / HBM_BPS, 3)
        if name != "outliersk":
            want = scores_of(name.split("_")[-1], host_rows)
            g = got["scores"][check_rows]
            rec["parity_rows"] = bool(np.array_equal(np.isnan(g), np.isnan(want)) and np.array_equal(g[~np.isnan(g)], want[~np.isnan(want)]))
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    for s, p, cases in ((S, P, CASES), (1_000_000, 1, [("topk_avg", 1, False), ("topk_avg", 1024, True), ("topk_median", 8, False)])):
        gen = torch.Generator(device="cuda").manual_seed(20261016)
        src = 1000 + torch.cumsum(torch.randn((s, p), dtype=torch.float64, device="cuda", generator=gen), dim=1)
        src[torch.rand((s, p), device="cuda", generator=gen) < 0.05] = float("nan")
        work = torch.empty_like(src)
        check_rows = [0, s // 2, s - 1]
        host_rows = src[check_rows].cpu().numpy()
        for name, G, remaining in cases:
            if not only or name in only:
                measure(name, s, p, G, remaining, src, work, host_rows, check_rows)
        del src, work
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")
    return 0 if all(r.get("parity_rows", True) for r in lines) else 1


if __name__ == "__main__":
    sys.exit(main())
