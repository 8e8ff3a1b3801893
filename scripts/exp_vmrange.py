#!/usr/bin/env python3
"""Time vmb_vmrange_to_le (prometheus_buckets) and vmb_buckets_limit on a device matrix at two sizes:

  large      S = 100 000 `vmrange` rows x P = 8172 points (6.5 GB) in groups of 30, 100 and 300 adjacent ranges of the
             18-per-decade grid, positive rates with 1 % NaN cells;
  dashboard  50 ranges x 1, 10 and 100 groups x 240 points, where the host side of the call dominates.

Per case one JSON line:
  call_ms      host clock around the C ABI calls, which end in a device synchronise: the count call (d_out == NULL) plus the
               call that fills d_out, host plan included; median of --repeats after one warm-up.  wrapper_ms: the same through
               promql.prometheus_buckets, whose per-row label parsing in Python comes on top;
  kernel_ms    device time per kernel from torch.profiler over one count + fill pair (k_vr_flags runs in both calls);
  bytes model  k_vr_flags reads at most 8 S P (a warp stops at the first 32 points that hold a value > 0, so on these rows
               it reads 256 bytes per row and no bandwidth share is given); k_vr_cumsum reads 8 S P and
               writes 8 S_out P; k_vr_hits reads 8 S P of the le matrix.  share_of_3.35TBps: bytes over kernel time as a share
               of the H100 SXM data-sheet HBM3 bandwidth;
  parity       the first two groups compared with tests/vmrange_ref.py, bit for bit.
The card's name and power limit are read in the same run.

  python scripts/exp_vmrange.py [--repeats 5] [--out results/exp_vmrange.jsonl]
"""
import argparse
import ctypes as C
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
KERNELS = ("k_vr_flags", "k_vr_gather", "k_vr_merge", "k_vr_cumsum", "k_vr_hits")


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
    ap.add_argument("--out", default="")
    a = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    import victoriametrics_b200 as vm
    import vmrange_ref as V
    from victoriametrics_b200 import _lib

    assert torch.cuda.is_available(), "this measurement needs the GPU"
    card = card_info()
    print(json.dumps({"card": card, "torch_device": torch.cuda.get_device_name(0)}), flush=True)
    lib, ctx = _lib.lib(), vm.default_context()
    gen = torch.Generator(device="cuda").manual_seed(20261016)
    bounds = ["%.3e" % (10 ** (e + k / 18)) for e in range(-9, 9) for k in range(18)]
    lines = []
    u32 = lambda x: x.ctypes.data_as(_lib.u32p)
    f64 = lambda x: x.ctypes.data_as(_lib.f64p)

    def kernels(prof):
        t, n = {}, {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                for k in KERNELS:
                    if k in e.name:
                        t[k] = t.get(k, 0.0) + e.time_range.elapsed_us() / 1e3
                        n[k] = n.get(k, 0) + 1
        return {k: {"ms": round(t[k], 3), "launches": n[k]} for k in t}

    def measure(kind, rows, points, gs, repeats):
        ngroups = rows // gs
        m = torch.rand((rows, points), dtype=torch.float64, device="cuda", generator=gen) * 100
        m[torch.rand((rows, points), device="cuda", generator=gen) < 0.01] = float("nan")
        vr = ["%s...%s" % (bounds[k], bounds[k + 1]) for _ in range(ngroups) for k in range(20, 20 + gs)]
        gids = np.repeat(np.arange(ngroups, dtype=np.uint32), gs)
        ids = {}
        starts = np.array([float(v.split("...")[0]) for v in vr])
        ends = np.array([float(v.split("...")[1]) for v in vr])
        skeys = np.array([ids.setdefault(v.split("...")[0], len(ids)) for v in vr], dtype=np.uint32)
        ekeys = np.array([ids.setdefault(v.split("...")[1], len(ids)) for v in vr], dtype=np.uint32)
        cap = rows + 2 * ngroups
        out = torch.empty((cap, points), dtype=torch.float64, device="cuda")
        src, le = np.zeros(cap, dtype=np.uint32), np.zeros(cap, dtype=np.uint32)
        kd = np.zeros(cap, dtype=np.uint8)
        nout = C.c_size_t(0)

        def call():
            for optr in (None, C.c_void_p(out.data_ptr())):
                nout.value = cap if optr else 0
                rc = lib.vmb_vmrange_to_le(ctx.h, C.c_void_p(m.data_ptr()), rows, points, u32(gids), f64(starts), f64(ends),
                                           u32(skeys), u32(ekeys), ngroups, optr, C.byref(nout), u32(src),
                                           kd.ctypes.data_as(_lib.u8p), u32(le))
                assert rc == (0 if optr else -54), rc

        def timed(f, n):
            ts = []
            for i in range(n + 1):
                t0 = time.perf_counter()
                f()
                if i:
                    ts.append((time.perf_counter() - t0) * 1e3)
            return ts
        times = timed(call, repeats)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
        kt = kernels(prof)
        nrows_out = nout.value
        wrap = timed(lambda: vm.promql.prometheus_buckets(m.data_ptr(), rows, points, vr, [False] * rows, gids,
                                                          lambda nb: type("B", (), {"ptr": out.data_ptr()})()),
                     max(1, repeats // 5))
        # buckets_limit(10) on the le matrix
        lgids = gids[src[:nrows_out]]
        names = {v: k for k, v in ids.items()}
        les = np.array([np.inf if k == V.PINF else float(names[x]) for k, x in zip(kd[:nrows_out], le[:nrows_out])])
        kept = np.zeros(nrows_out, dtype=np.uint32)
        lim_n = C.c_size_t(0)

        def limit_call():
            lim_n.value = nrows_out
            assert lib.vmb_buckets_limit(ctx.h, C.c_void_p(out.data_ptr()), nrows_out, points, u32(lgids), f64(les), ngroups,
                                         10, u32(kept), C.byref(lim_n)) == 0
        ltimes = timed(limit_call, repeats)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            limit_call()
        lkt = kernels(prof)
        # parity: the first two groups
        sel = min(2, ngroups) * gs
        host = m[:sel].cpu().numpy()
        mat, wsrc, wkinds, _ = V.vmrange_to_le_arrays(host, vr[:sel], [None] * sel, gids[:sel].tolist())
        got = out[:len(wsrc)].cpu().numpy()
        ok = (np.array_equal(src[:len(wsrc)], wsrc) and np.array_equal(kd[:len(wsrc)], wkinds)
              and got.tobytes() == mat.tobytes())
        wl = V.buckets_limit_ref(10, got, lgids[:len(wsrc)], les[:len(wsrc)], min(2, ngroups))
        ok = ok and kept[:len(wl)].tolist() == wl
        rd, wr = 8 * rows * points, 8 * nrows_out * points
        share = lambda b, k: round(b / (kt[k]["ms"] * 1e-3) / HBM_BPS, 3) if k in kt and kt[k]["ms"] else None
        rec = {"size": kind, "rows": rows, "points": points, "groups": ngroups, "group_rows": gs, "rows_out": nrows_out,
               "call_ms_median": round(float(np.median(times)), 3), "call_ms": [round(t, 3) for t in times],
               "wrapper_ms_median": round(float(np.median(wrap)), 3), "kernels": kt,
               "flags_bytes_max": rd,
               "cumsum_bytes": rd + wr, "cumsum_share_of_3.35TBps": share(rd + wr, "k_vr_cumsum"),
               "limit10_call_ms_median": round(float(np.median(ltimes)), 3), "limit10_kernels": lkt,
               "limit10_kept": lim_n.value, "hits_bytes": wr,
               "hits_share_of_3.35TBps": round(wr / (lkt["k_vr_hits"]["ms"] * 1e-3) / HBM_BPS, 3) if "k_vr_hits" in lkt else None,
               "parity_groups": bool(ok), "card": card.get("name"), "power_limit": card.get("power_limit")}
        print(json.dumps(rec), flush=True)
        lines.append(rec)
        del m, out
        torch.cuda.empty_cache()

    for gs in (30, 100, 300):
        measure("large", S // gs * gs, P, gs, a.repeats)
    for groups in (1, 10, 100):
        measure("dashboard", 50 * groups, 240, 50, max(a.repeats, 50))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")
    return 0 if all(r["parity_groups"] for r in lines) else 1


if __name__ == "__main__":
    sys.exit(main())
