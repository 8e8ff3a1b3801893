#!/usr/bin/env python3
"""Time vmb_sort_rows, vmb_set_or and vmb_rows_nonempty at the size of a large dashboard query, S = 100 000 rows x P = 8172
points (6.5 GB), and at a dashboard's size, 100 rows x 240 points.  Cases:
  sort / sort_desc  a seeded random walk per row with 5 % NaN (decided at the last point); small integers 0..15 (ties at the last
                    point, refined over several rounds); 1 000 distinct rows repeated 100 times (classes of equal rows, one
                    backward read of them); rows that are NaN over their last 100 points;
  or                100 000 + 100 000 rows keyed 1:1, with equal and with different metric names; q or on() vector(0) over
                    100 000 left rows;
  rows_nonempty     the random walk.
`or` changes both matrices, so every call gets fresh device copies first; those copies are outside every timing.  Per case, one
JSON line:
  call_ms    host clock around the call, which ends in a device synchronise, after one warm-up call, median of --repeats calls;
  kernels    device time per kernel from torch.profiler, in a profiled call of its own;
  host_ms    call_ms minus the kernel time: the host's class bookkeeping, the copies and the launches;
  read_GB / read_share_of_3.35TBps  for the passes that read whole rows (k_sr_split, k_or_*, k_rows_nonempty): the bytes they
             must read at least, over their kernel time, as a share of the H100 SXM data-sheet HBM3 bandwidth, 3.35 TB/s;
  ok         the sort order checked pair by pair against the comparator (tests/rowset_ref.py's rule) on the device.
The card's name and power limit are read in the same run.

  python scripts/exp_rowset.py [--repeats 5] [--out results/exp_rowset.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True

HBM_BPS = 3.35e12
PREFIXES = ("k_sr_", "k_oa_", "k_or_", "k_rows_nonempty")


def card_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm_max = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": sm_max}
    except Exception as e:
        return {"error": repr(e)}


def sorted_ok(torch, dv, order, desc):
    S, P = dv.shape
    o = torch.from_numpy(order).cuda()
    for i0 in range(0, S - 1, 2048):
        i = torch.arange(i0, min(S - 1, i0 + 2048), device="cuda")
        a, b = dv[o[i]], dv[o[i + 1]]
        an, bn = torch.isnan(a), torch.isnan(b)
        differ = (an != bn) | (~an & ~bn & (a != b))
        n = P - 1 - differ.flip(1).to(torch.int8).argmax(dim=1)
        k = torch.arange(len(i), device="cuda")
        av, bv = a[k, n], b[k, n]
        less = torch.where(torch.isnan(av), True, torch.where(torch.isnan(bv), False, bv < av if desc else av < bv))
        if not bool(torch.where(differ.any(dim=1), less, o[i] < o[i + 1]).all()):
            return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    import victoriametrics_b200 as vm

    assert torch.cuda.is_available(), "this measurement needs the GPU"
    card = card_info()
    print(json.dumps({"card": card, "torch_device": torch.cuda.get_device_name(0)}), flush=True)
    lines = []

    def measure(case, S, P, call, reset=None, read_bytes=None, check=None):
        times = []
        for i in range(a.repeats + 1):
            if reset:
                reset()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = call()
            torch.cuda.synchronize()
            if i:
                times.append((time.perf_counter() - t0) * 1e3)
        if reset:
            reset()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        kern = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and any(p in e.name for p in PREFIXES):
                k = e.name.split("(")[0].replace("void ", "")
                kern[k] = kern.get(k, 0.0) + e.time_range.elapsed_us() / 1e3
        kernel_ms = sum(kern.values())
        call_ms = float(np.median(times))
        rec = {"case": case, "S": S, "P": P, "call_ms_median": round(call_ms, 3), "call_ms": [round(t, 3) for t in times],
               "kernel_ms": round(kernel_ms, 3), "host_ms": round(call_ms - kernel_ms, 3),
               "kernels": {k: round(v, 3) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])},
               "card": card.get("name"), "power_limit": card.get("power_limit")}
        if read_bytes:
            pref, nbytes = read_bytes
            ms = sum(v for k, v in kern.items() if any(p in k for p in pref))
            if ms:
                rec["read_GB"] = round(nbytes / 1e9, 2)
                rec["read_share_of_3.35TBps"] = round(nbytes / (ms * 1e-3) / HBM_BPS, 3)
        if check:
            rec["ok"] = bool(check(res))
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    for S, P in ((100_000, 8172), (100, 240)):
        gen = torch.Generator(device="cuda").manual_seed(20261017)
        walk = 1000 + torch.cumsum(torch.randn((S, P), dtype=torch.float64, device="cuda", generator=gen), dim=1)
        walk[torch.rand((S, P), device="cuda", generator=gen) < 0.05] = float("nan")
        ints = torch.randint(0, 16, (S, P), device="cuda", generator=gen).to(torch.float64)
        d = max(1, S // 100)
        rep = walk[:d].clone().repeat(S // d + 1, 1)[:S].contiguous()
        tail = walk.clone()
        tail[:, P - 100:] = float("nan")
        for name, m in (("walk", walk), ("ints", ints), ("repeated", rep), ("nan_tail", tail)):
            for desc in (False, True):
                # one backward read: the first 32 points of every row in a random walk, the rows in the other cases
                nb = 8 * S * (P if name == "repeated" else 132 if name == "nan_tail" else 32)
                measure("%s %s" % ("sort_desc" if desc else "sort", name), S, P,
                        lambda m=m, desc=desc: vm.promql.sort_rows(m.data_ptr(), S, P, desc),
                        read_bytes=(("k_sr_split",), nb), check=lambda o, m=m, desc=desc: sorted_ok(torch, m, o, desc))
            del m
        measure("rows_nonempty walk", S, P, lambda: vm.promql.rows_nonempty(walk.data_ptr(), S, P),
                read_bytes=(("k_rows_nonempty",), 8 * S * 32))
        del ints, rep, tail
        torch.cuda.empty_cache()
        right_src = walk.flip(0).contiguous()
        L, R = torch.empty_like(walk), torch.empty_like(walk)
        for name, rl in (("or 1:1 equal names", [{"k": str(i)} for i in range(S)]),
                         ("or 1:1 different names", [{"k": str(i), "s": "r"} for i in range(S)])):
            ll = [{"k": str(i)} for i in range(S)]

            def reset():
                L.copy_(walk)
                R.copy_(right_src)
            measure(name, S, P, lambda ll=ll, rl=rl: vm.promql.set_or(L.data_ptr(), ll, R.data_ptr(), rl, P, on=("k",)), reset,
                    read_bytes=(("k_or_",), 8 * S * P * 2))
        R1 = torch.zeros((1, P), dtype=torch.float64, device="cuda")
        ll = [{"k": str(i)} for i in range(S)]

        def reset0():
            L.copy_(walk)
            R1.zero_()
        measure("or on() vector(0)", S, P, lambda: vm.promql.set_or(L.data_ptr(), ll, R1.data_ptr(), [{}], P, on=()), reset0,
                read_bytes=(("k_or_", "k_rows_nonempty"), 8 * P * 2))
        del walk, right_src, L, R
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")
    return 0 if all(r.get("ok", True) for r in lines) else 1


if __name__ == "__main__":
    sys.exit(main())
