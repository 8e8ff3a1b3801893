#!/usr/bin/env python3
"""Time vmb_histogram (the histogram functions over `le` buckets on a device matrix) at two sizes:

  large      S = 100 000 bucket rows x P = 8172 points (6.5 GB) in groups of 10, 30 and 100 rows (le = 0.005 * 2^k, the last
             +Inf), counts cumulative over the buckets with 1 % NaN cells, for histogram_quantile(0.99) with and without the
             bounds, histogram_quantiles(0.5, 0.9, 0.99), histogram_share(le), histogram_fraction and histogram_stdvar;
  dashboard  30 buckets x 1, 10 and 100 groups x 240 points, where the host side of the call dominates.

Per case one JSON line:
  call_ms    host clock around the call, which ends in a device synchronise, after one warm-up call, median of --repeats calls;
  kernel_ms  device time of k_histogram from torch.profiler, in a profiled call of its own;
  bytes      the bytes model: quantile reads the bucket matrix at most twice (pass 1 to the end, pass 2 up to the interpolating
             bucket), share / fraction / stdvar once, 8 S P per read; every output matrix writes 8 G P.  bytes_min counts one read,
             bytes_max two (they agree for the one-pass functions); share_of_3.35TBps is bytes_min over kernel time as a share of
             the H100 SXM data-sheet HBM3 bandwidth;
  parity     a few groups compared with tests/histogram_ref.py, bit for bit.
The card's name and power limit are read in the same run.

  python scripts/exp_histogram.py [--repeats 5] [--out results/exp_histogram.jsonl]
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


def cases(gs):
    mid = 0.005 * 2 ** (gs // 2)
    return [("histogram_quantile", (0.99,), False), ("histogram_quantile", (0.99,), True),
            ("histogram_quantiles", (0.5, 0.9, 0.99), False), ("histogram_share", (mid,), False),
            ("histogram_fraction", (mid / 4, mid * 4), False), ("histogram_stdvar", (), False)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    import victoriametrics_b200 as vm
    from histogram_ref import histogram_ref

    assert torch.cuda.is_available(), "this measurement needs the GPU"
    card = card_info()
    print(json.dumps({"card": card, "torch_device": torch.cuda.get_device_name(0)}), flush=True)
    gen = torch.Generator(device="cuda").manual_seed(20261016)
    lines = []

    def measure(kind, name, args, bounds, m, rows, points, gids, les, ngroups, repeats):
        nphi = len(args) if name == "histogram_quantiles" else 1
        out = torch.empty((nphi * ngroups, points), dtype=torch.float64, device="cuda")
        lo = torch.empty((ngroups, points), dtype=torch.float64, device="cuda") if bounds else None
        up = torch.empty((ngroups, points), dtype=torch.float64, device="cuda") if bounds else None
        kw = dict(lower_dev_ptr=lo.data_ptr(), upper_dev_ptr=up.data_ptr()) if bounds else {}

        def call():
            vm.promql.histogram(name, m.data_ptr(), rows, points, gids, les, ngroups, out.data_ptr(), *args, **kw)
            torch.cuda.synchronize()

        times = []
        for i in range(repeats + 1):
            t0 = time.perf_counter()
            call()
            if i:
                times.append((time.perf_counter() - t0) * 1e3)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
        kernel_ms = sum(e.time_range.elapsed_us() / 1e3 for e in prof.events()
                        if e.device_type == torch.autograd.DeviceType.CUDA and "k_histogram" in e.name)
        read = 8 * rows * points
        write = 8 * ngroups * points * (nphi + (2 if bounds else 0))
        two = name in ("histogram_quantile", "histogram_quantiles")
        rec = {"size": kind, "func": name, "args": list(args), "bounds": bounds, "rows": rows, "points": points,
               "groups": ngroups, "group_rows": rows // ngroups, "call_ms_median": round(float(np.median(times)), 3),
               "call_ms": [round(t, 3) for t in times], "kernel_ms": round(kernel_ms, 3), "bytes_min": read + write,
               "bytes_max": (2 if two else 1) * read + write,
               "share_of_3.35TBps": round((read + write) / (kernel_ms * 1e-3) / HBM_BPS, 3) if kernel_ms else None,
               "card": card.get("name"), "power_limit": card.get("power_limit")}
        # parity on the first and last two groups
        gs = rows // ngroups
        sel = [0, 1, ngroups - 2, ngroups - 1] if ngroups >= 4 else list(range(ngroups))
        pick = np.concatenate([np.arange(g * gs, (g + 1) * gs) for g in sel])
        host = m[torch.from_numpy(pick).cuda()].cpu().numpy()
        sub_g = np.repeat(np.arange(len(sel), dtype=np.uint32), gs)
        want = histogram_ref(name, host, sub_g, les[pick], len(sel), *args, bounds=bounds)
        got = out.view(nphi, ngroups, points)[:, sel].cpu().numpy()
        w = np.asarray(want[0]).reshape(nphi, len(sel), points)
        ok = np.array_equal(np.isnan(got), np.isnan(w)) and np.array_equal(got[~np.isnan(got)], w[~np.isnan(w)])
        if bounds:
            for dev, ref in ((lo, want[1]), (up, want[2])):
                g2 = dev[sel].cpu().numpy()
                ok = ok and np.array_equal(np.isnan(g2), np.isnan(ref)) and np.array_equal(g2[~np.isnan(g2)], ref[~np.isnan(ref)])
        rec["parity_groups"] = bool(ok)
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    def bucket_matrix(rows, points, gs):
        inc = torch.rand((rows // gs, gs, points), dtype=torch.float64, device="cuda", generator=gen) * 100
        m = torch.cumsum(inc, dim=1).reshape(rows, points)
        m[torch.rand((rows, points), device="cuda", generator=gen) < 0.01] = float("nan")
        les = np.tile(np.r_[0.005 * 2.0 ** np.arange(gs - 1), np.inf], rows // gs)
        gids = np.repeat(np.arange(rows // gs, dtype=np.uint32), gs)
        return m, gids, les

    for gs in (10, 30, 100):
        rows = S // gs * gs
        m, gids, les = bucket_matrix(rows, P, gs)
        for name, args, bounds in cases(gs):
            measure("large", name, args, bounds, m, rows, P, gids, les, rows // gs, a.repeats)
        del m
        torch.cuda.empty_cache()
    for groups in (1, 10, 100):
        rows = 30 * groups
        m, gids, les = bucket_matrix(rows, 240, 30)
        for name, args, bounds in cases(30):
            measure("dashboard", name, args, bounds, m, rows, 240, gids, les, groups, max(a.repeats, 50))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")
    return 0 if all(r["parity_groups"] for r in lines) else 1


if __name__ == "__main__":
    sys.exit(main())
