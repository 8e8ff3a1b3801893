#!/usr/bin/env python3
"""Device time per kernel of the flagship workload (bench.py at its defaults: rate(m[5m]) step 15 s over 100 000
reference-encoded blocks x 8192 samples, blocks resident in HBM), from one torch.profiler run with CUDA activities.

Prints the card, its power limit and SM clock, the library's own stage split (vmb_ctx_last_stage_ms, CUDA events) and a
table of ms per step per kernel name.  --json PATH also writes the numbers as JSON.

  python scripts/fused_kernels.py [--blocks 100000] [--rows 8192] [--steps 5] [--warmup 3] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True

import bench  # noqa: E402  (the same generator and query grid as the benchmark)

STAGES = ["zstd", "column_decode", "series_preamble", "rollup", "aggregate", "fused_decode_rollup"]


def card_info(index):
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, power, sm, sm_max = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # the table below does not depend on it
        return {"error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=100_000)
    ap.add_argument("--rows", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=5, help="profiled steps")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default="", help="also write the result here")
    a = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import victoriametrics_b200 as vm
    from victoriametrics_b200 import promql, storage

    dev = 0
    torch.cuda.set_device(dev)
    ctx = vm.Context(dev)
    stream = torch.cuda.current_stream()
    ctx.set_stream(stream.cuda_stream)
    start, end, step = bench.query_range(a.rows, 300_000, 15_000)
    points = 1 + (end - start) // step
    descs, payload, _ = bench.gen_blocks(a.blocks, a.rows, seed=1234)
    blocks = storage.Blocks(descs, payload, ctx)
    out = torch.empty((a.blocks, points), dtype=torch.float64, device="cuda")

    def run():
        return promql.eval_rollup_func("rate", blocks, start, end, step, 300_000, out_dev_ptr=out.data_ptr())

    for _ in range(a.warmup):
        run()
    torch.cuda.synchronize()
    ctx.enable_stage_timing(True)
    run()
    stage_ms = ctx.stage_ms()
    ctx.enable_stage_timing(False)
    torch.cuda.synchronize()

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            run()
        torch.cuda.synchronize()
    card = card_info(dev)

    per = defaultdict(lambda: [0.0, 0])
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = e.name.split("(")[0]
            per[name][0] += e.time_range.elapsed_us() / 1e3
            per[name][1] += 1
    total = sum(v[0] for v in per.values()) / a.steps
    rows = sorted(((k, v[0] / a.steps, v[1] / a.steps) for k, v in per.items()), key=lambda r: -r[1])

    print("card: %s, power limit %s, SM clock %s (max %s)" % (card.get("name"), card.get("power_limit"), card.get("sm_clock"),
                                                              card.get("sm_clock_max")))
    print("workload: rate(m[5m]) step 15 s, %d blocks x %d samples, %d profiled steps" % (a.blocks, a.rows, a.steps))
    print("stage split (library CUDA events, one step): " +
          ", ".join("%s %.3f ms" % (n, ms) for n, ms in zip(STAGES, stage_ms) if ms > 0))
    print("%-48s %10s %8s %7s" % ("kernel / copy", "ms/step", "calls", "share"))
    for k, ms, calls in rows:
        print("%-48s %10.3f %8.1f %6.1f%%" % (k[:48], ms, calls, 100.0 * ms / total if total else 0.0))
    print("%-48s %10.3f" % ("total device time", total))
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": card, "stage_ms": dict(zip(STAGES, stage_ms)), "total_ms_per_step": total,
                       "kernels": [{"name": k, "ms_per_step": ms, "calls_per_step": c} for k, ms, c in rows]}, f, indent=1)
    blocks.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
