#!/usr/bin/env python3
"""Where a fill of the fused rollup kernel spends its cycles, on the flagship workload (bench.py at its defaults: rate(m[5m])
step 15 s over 100 000 reference-encoded blocks x 8192 samples, blocks resident in HBM), run one-shot (one chunk, 5 CTAs/SM).

Builds the phase-clock variant of libvmb200.so (-DVMB_FUSED_PHASES, fused.cu) into a temporary directory -- the product
library is left alone -- and loads it in place of the product.  Lane 0 of every warp adds the clock64() cycles since its
previous mark to the phase that just ended; the table gives SM cycles per fill and per series of one warp, averaged over all
warps, and each phase's share.  The marks themselves cost cycles and order the instructions around them: the shares are
what to read, the absolute sum is somewhat above the product's.  Prints the card, its power limit and SM clock.

  python scripts/exp_fused_phases.py [--func rate] [--kind counter] [--steps 3] [--so PREBUILT.so] [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.dont_write_bytecode = True

import bench  # noqa: E402  (the same generator and query grid as the benchmark)
from fused_kernels import card_info  # noqa: E402

PHASES = ["series setup, first copy", "terminator scan", "parse", "sum scans", "emit", "counter resets", "points",
          "barrier / copy waits"]
WARPS = 4  # FU_WARPS


def build_variant(tmp):
    so = os.path.join(tmp, "libvmb200.so")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "victoriametrics_b200", "csrc"), "OUT=" + so,
                           "LOG=" + os.path.join(tmp, "ptxas.log"), "NVEXTRA=-DVMB_FUSED_PHASES"])
    return so


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=100_000)
    ap.add_argument("--rows", type=int, default=8192)
    ap.add_argument("--func", default="rate", help="rollup function (quantile_over_time takes phi = 0.99)")
    ap.add_argument("--kind", default="counter", choices=["counter", "gauge"], help="generated values")
    ap.add_argument("--steps", type=int, default=3, help="measured calls")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--so", default="", help="a phase-clock build made before (make ... NVEXTRA=-DVMB_FUSED_PHASES) instead of "
                                             "compiling one")
    ap.add_argument("--json", default="", help="also write the result here")
    a = ap.parse_args()

    tmp = tempfile.mkdtemp(prefix="vmb_phases_")
    so = a.so or build_variant(tmp)
    from victoriametrics_b200 import _lib
    _lib.SO_PATH = os.path.abspath(so)
    L = _lib.lib()
    if not hasattr(L, "vmb_fused_phase_cycles"):
        raise SystemExit("%s is not a phase-clock build (vmb_fused_phase_cycles missing)" % so)
    read = L.vmb_fused_phase_cycles
    read.restype = C.c_int
    read.argtypes = [C.c_void_p, C.c_int]
    layout = read(None, 0)
    slots, ctas = layout // 1000, layout % 1000
    assert slots == len(PHASES) + 2, layout

    import torch
    import victoriametrics_b200 as vm
    from victoriametrics_b200 import promql, storage

    dev = 0
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream()
    os.environ["VMB_FUSED_CHUNKS"] = "1"
    ctx = vm.Context(dev, stream.cuda_stream)
    del os.environ["VMB_FUSED_CHUNKS"]
    start, end, step = bench.query_range(a.rows, 300_000, 15_000)
    points = 1 + (end - start) // step
    descs, payload, _ = bench.gen_blocks(a.blocks, a.rows, seed=1234, kind=a.kind)
    args = np.full(points, 0.99) if a.func == "quantile_over_time" else None
    blocks = storage.Blocks(descs, payload, ctx)
    out = torch.empty((a.blocks, points), dtype=torch.float64, device="cuda")

    def run():
        return promql.eval_rollup_func(a.func, blocks, start, end, step, 300_000, args=args, out_dev_ptr=out.data_ptr())

    for _ in range(a.warmup):
        run()
    torch.cuda.synchronize()
    read(None, 1)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        run()
    e1.record()
    e1.synchronize()
    step_ms = e0.elapsed_time(e1) / a.steps
    buf = np.zeros((ctas, slots), dtype=np.uint64)
    if read(buf.ctypes.data, 1) < 0:
        raise SystemExit("reading the phase clocks failed")
    card = card_info(dev)

    used = buf[:, len(PHASES)] > 0  # CTAs that ran a fill
    fills = float(buf[:, len(PHASES)].sum())
    series = float(buf[:, len(PHASES) + 1].sum())
    cyc = buf[:, :len(PHASES)].astype(np.float64).sum(axis=0) / WARPS  # per warp
    per_cta = buf[used, :len(PHASES)].astype(np.float64).sum(axis=1) / WARPS
    tot = cyc.sum()
    print("card: %s, power limit %s, SM clock %s (max %s)" % (card.get("name"), card.get("power_limit"), card.get("sm_clock"),
                                                              card.get("sm_clock_max")))
    print("workload: %s(m[5m]) step 15 s over %s blocks, %d blocks x %d samples, one-shot; %d calls, %.3f ms per call "
          "(phase-clock build)" % (a.func, a.kind, a.blocks, a.rows, a.steps, step_ms))
    print("fills %d (%.1f per series), series %d, CTAs %d, cycles per CTA min / max %.3g / %.3g" %
          (fills, fills / max(series, 1), series, int(used.sum()), per_cta.min() if len(per_cta) else 0,
           per_cta.max() if len(per_cta) else 0))
    print("%-28s %14s %14s %7s" % ("phase", "cycles/fill", "cycles/series", "share"))
    for name, c in zip(PHASES, cyc):
        print("%-28s %14.1f %14.1f %6.1f%%" % (name, c / max(fills, 1), c / max(series, 1), 100.0 * c / tot if tot else 0.0))
    print("%-28s %14.1f %14.1f" % ("total", tot / max(fills, 1), tot / max(series, 1)))
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": card, "func": a.func, "kind": a.kind, "ms_per_call": step_ms, "fills": fills, "series": series,
                       "cycles_per_fill": dict(zip(PHASES, (cyc / max(fills, 1)).tolist())),
                       "cycles_per_series": dict(zip(PHASES, (cyc / max(series, 1)).tolist()))}, f, indent=1)
    blocks.close()
    ctx.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
