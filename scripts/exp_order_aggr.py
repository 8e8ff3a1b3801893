#!/usr/bin/env python3
"""Time vmb_aggr_order (the order-statistic aggregates by (...) on a device matrix) at the sizes of a large dashboard query.

Shapes: S = 100 000 series x P = 8172 points (6.5 GB) with G in {1, 8, 1024, S} groups for each of the six functions (quantiles
with three phis); S = 1 000 000 x P = 1 (an instant query) with G in {1, 1024}; and quantiles with one phi beside
vmb_aggr_quantile (the rank selection capped at 2048 series per group) at G = 64, 1563 rows per group.  The matrix is small
integers (ties) from a seed, about 1 % NaN; row r belongs to group r % G.

Per shape, one JSON line: the call time (host clock around the call, which ends in a device synchronise, after warm-up, over at
least --seconds of repeats), the device time per kernel from torch.profiler in a run of its own, the bytes the gather, the sort
passes and the finish move as computed from the shapes (below), and parity on a column strip against tests/order_aggr_ref.py.
The card's name and power limit are read in the same run.

Bytes, per pass over the S x P values (8-byte keys): gather 8 S P read + 8 S P written; shared-memory sort 16 S P; each merge pass
16 S P over the keys of the groups longer than 4096 rows; finish 8 S P (a read of every key; quantiles reads 2 keys per phi and
cell); mad / outliers_mad sort twice and write the deviation keys (16 S P) in between; outliers read the matrix once more.

  python scripts/exp_order_aggr.py [--seconds 1] [--only quantiles,mad] [--out results/exp_order_aggr.jsonl]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.dont_write_bytecode = True

FUNCS = ["quantiles", "mad", "mode", "distinct", "outliers_iqr", "outliers_mad"]
PHIS = [0.5, 0.9, 0.99]
OA_C, OA_BUDGET = 4096, 1 << 27
SHAPES = [(100_000, 8172, g, f) for f in FUNCS for g in (1, 8, 1024, 100_000)]
SHAPES += [(1_000_000, 1, g, f) for f in FUNCS for g in (1, 1024)]
SHAPES += [(100_000, 8172, 64, "quantile1"), (100_000, 8172, 64, "aggr_quantile")]


def card_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm_max = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": sm_max}
    except Exception as e:
        return {"error": repr(e)}


def model_bytes(name, S, P, G):
    """bytes moved by the gather, the sort passes and the finish, from the shapes"""
    if name == "aggr_quantile":
        return {}
    n = S // G  # rows per group (r % G: sizes differ by at most one)
    kp = 8 * S * P
    passes = max(0, math.ceil(math.log2(math.ceil((n + 1) / OA_C)))) if n > OA_C else 0
    sort = 16 * S * P * (1 if n > 1 else 0) + 16 * S * P * passes
    two = name in ("mad", "outliers_mad")
    b = {"gather": 2 * kp, "sort": sort * (2 if two else 1), "finish": kp * (2 if two else 1)}
    if two:
        b["deviations"] = 2 * kp
    if name.startswith("outliers"):
        b["select"] = kp
    return b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--only", default="")
    ap.add_argument("--out", default="")
    a = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    import victoriametrics_b200 as vm
    from order_aggr_ref import aggr_order_ref

    assert torch.cuda.is_available(), "this measurement needs the GPU"
    card = card_info()
    print(json.dumps({"card": card, "torch_device": torch.cuda.get_device_name(0)}), flush=True)
    only = set(a.only.split(",")) if a.only else None
    lines, mats = [], {}
    for S, P, G, name in SHAPES:
        if only and name not in only:
            continue
        if (S, P) not in mats:
            mats.clear()
            torch.cuda.empty_cache()
            gen = torch.Generator(device="cuda").manual_seed(20261016 + S + P)
            m = torch.randint(-500, 501, (S, P), dtype=torch.float64, device="cuda", generator=gen)
            m[torch.rand((S, P), device="cuda", generator=gen) < 0.01] = float("nan")
            mats[(S, P)] = m
        m = mats[(S, P)]
        groups = (np.arange(S) % G).astype(np.uint32)
        K = len(PHIS) if name == "quantiles" else 1
        rows_out = name.startswith("outliers")
        out = None if rows_out else torch.empty((K, G, P), dtype=torch.float64, device="cuda")
        res = {}

        def call():
            if name == "aggr_quantile":
                vm.promql.aggr_quantile(0.5, m.data_ptr(), S, P, out.data_ptr(), groups, G)
            elif name == "quantile1":
                vm.promql.aggr_order("quantiles", m.data_ptr(), S, P, out.data_ptr(), groups, G, phis=[0.5])
            else:
                res["r"] = vm.promql.aggr_order(name, m.data_ptr(), S, P, None if rows_out else out.data_ptr(), groups, G,
                                                phis=PHIS, tolerance=3.0)

        call()
        torch.cuda.synchronize()
        n, t0 = 0, time.perf_counter()
        while True:
            call()
            n += 1
            el = time.perf_counter() - t0
            if el >= a.seconds and n >= 2:
                break
        call_ms = el / n * 1e3
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        kern = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and ("k_oa_" in e.name or "k_aggr_quantile" in e.name):
                k = e.name.split("(")[0].replace("void ", "")
                kern[k] = kern.get(k, 0.0) + e.time_range.elapsed_us() / 1e3
        kernel_ms = sum(kern.values())
        # parity on a 4-point strip: the reference restatement loops in Python
        p0, w = (P // 2, min(4, P)) if P > 4 else (0, P)
        strip = m[:, p0:p0 + w].cpu().numpy()
        if rows_out:  # the strip cannot see points outside it: a row it selects must be selected overall
            _, want = aggr_order_ref(name, strip, groups, G, tolerance=3.0)
            parity = bool(not (want & ~res["r"]).any())
        else:
            ref_name = "quantiles" if name in ("quantile1", "aggr_quantile") else name
            phis = PHIS if name == "quantiles" else [0.5]
            want, _ = aggr_order_ref(ref_name, strip, groups, G, phis)
            got = out[..., p0:p0 + w].cpu().numpy().reshape(want.shape)
            nan_ok = np.array_equal(np.isnan(got), np.isnan(want))
            ok = ~np.isnan(want)
            parity = bool(nan_ok and np.array_equal(got[ok], want[ok]))  # == : a zero's sign is the sort's choice
        mb = model_bytes(name, S, P, G)
        total = sum(mb.values())
        rec = {"func": name, "S": S, "P": P, "G": G, "call_ms": round(call_ms, 3), "calls": n, "kernel_ms": round(kernel_ms, 3),
               "kernels": {k: round(v, 3) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])},
               "bytes": mb, "kernel_GBps": round(total / kernel_ms / 1e6, 1) if kernel_ms and total else None,
               "parity_strip": parity, "card": card.get("name"), "power_limit": card.get("power_limit")}
        print(json.dumps(rec), flush=True)
        lines.append(rec)
        del out
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")
    return 0 if all(r["parity_strip"] for r in lines) else 1


if __name__ == "__main__":
    sys.exit(main())
