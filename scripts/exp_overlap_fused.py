#!/usr/bin/env python3
"""Chunked fused schedule on the flagship workload (bench.py at its defaults: rate(m[5m]) step 15 s over 100 000
reference-encoded blocks x 8192 samples, blocks resident in HBM; --func / --kind for the functions of bench.py's configs2):
the zstd stage of chunk k + 1 on a second stream beside the fused kernel of chunk k.

One context per (chunks C, fused CTAs per SM) shape -- VMB_FUSED_CHUNKS / VMB_FUSED_CTAS_PER_SM are read when a context is
created -- all over the same uploaded blocks.  Prints the card, its power limit and SM clock; the step time of every shape
over alternating rounds (CUDA events around whole calls, min / median / max); and per-kernel device time from one
torch.profiler run per listed shape.  --json PATH also writes the numbers as JSON.

  python scripts/exp_overlap_fused.py [--chunks 1,4,8,16] [--ctas 5,4] [--rounds 5] [--steps 5] [--profile 1x5,8x5]
"""
import argparse
import json
import os
import statistics
import sys
from collections import defaultdict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.dont_write_bytecode = True

import bench  # noqa: E402  (the same generator and query grid as the benchmark)
from fused_kernels import card_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=100_000)
    ap.add_argument("--func", default="rate", help="rollup function (quantile_over_time takes phi = 0.99)")
    ap.add_argument("--kind", default="counter", choices=["counter", "gauge"], help="generated values")
    ap.add_argument("--rows", type=int, default=8192)
    ap.add_argument("--chunks", default="1,4,8,16")
    ap.add_argument("--ctas", default="5,4", help="fused CTAs per SM")
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds over all shapes")
    ap.add_argument("--steps", type=int, default=5, help="timed calls per shape and round")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", default="1x5,8x5", help="shapes CxN profiled with torch.profiler ('' = none)")
    ap.add_argument("--json", default="", help="also write the result here")
    a = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import victoriametrics_b200 as vm
    from victoriametrics_b200 import promql, storage

    dev = 0
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream()
    shapes = [(c, n) for n in (int(x) for x in a.ctas.split(",")) for c in (int(x) for x in a.chunks.split(","))]
    ctxs = {}
    for c, n in shapes:
        os.environ["VMB_FUSED_CHUNKS"] = str(c)
        os.environ["VMB_FUSED_CTAS_PER_SM"] = str(n)
        ctxs[(c, n)] = vm.Context(dev, stream.cuda_stream)
    del os.environ["VMB_FUSED_CHUNKS"], os.environ["VMB_FUSED_CTAS_PER_SM"]
    start, end, step = bench.query_range(a.rows, 300_000, 15_000)
    points = 1 + (end - start) // step
    descs, payload, _ = bench.gen_blocks(a.blocks, a.rows, seed=1234, kind=a.kind)
    args = np.full(points, 0.99) if a.func == "quantile_over_time" else None
    blocks = storage.Blocks(descs, payload, ctxs[shapes[0]])
    out = torch.empty((a.blocks, points), dtype=torch.float64, device="cuda")

    def run(shape):
        blocks.ctx = ctxs[shape]
        return promql.eval_rollup_func(a.func, blocks, start, end, step, 300_000, args=args, out_dev_ptr=out.data_ptr())

    ref = None
    for shape in shapes:  # warm-up, and every shape writes the same bits
        for _ in range(a.warmup):
            run(shape)
        torch.cuda.synchronize()
        got = out.view(torch.int64).clone()
        if ref is None:
            ref = got
        elif not torch.equal(ref, got):
            raise SystemExit("shape C=%d x %d CTAs/SM wrote different bits" % shape)
    del ref, got

    times = defaultdict(list)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.rounds):
        for shape in shapes:
            torch.cuda.synchronize()
            e0.record()
            for _ in range(a.steps):
                run(shape)
            e1.record()
            e1.synchronize()
            times[shape].append(e0.elapsed_time(e1) / a.steps)
    stage = {}
    for shape in shapes:
        ctxs[shape].enable_stage_timing(True)
        run(shape)
        stage[shape] = ctxs[shape].stage_ms()
        ctxs[shape].enable_stage_timing(False)
    torch.cuda.synchronize()

    kernels = {}
    for spec in filter(None, a.profile.split(",")):
        shape = tuple(int(x) for x in spec.split("x"))
        if shape not in ctxs:
            continue
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.steps):
                run(shape)
            torch.cuda.synchronize()
        per = defaultdict(float)
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                per[e.name.split("(")[0]] += e.time_range.elapsed_us() / 1e3 / a.steps
        kernels[shape] = sorted(per.items(), key=lambda kv: -kv[1])

    card = card_info(dev)
    print("card: %s, power limit %s, SM clock %s (max %s)" % (card.get("name"), card.get("power_limit"), card.get("sm_clock"),
                                                              card.get("sm_clock_max")))
    print("workload: %s(m[5m]) step 15 s over %s blocks, %d blocks x %d samples; %d rounds x %d calls per shape, alternating" %
          (a.func, a.kind, a.blocks, a.rows, a.rounds, a.steps))
    print("%-22s %9s %9s %9s %10s %10s" % ("shape", "min ms", "median", "max", "zstd ms", "fused ms"))
    for shape in shapes:
        t = times[shape]
        print("C=%-3d %2d CTAs/SM       %9.3f %9.3f %9.3f %10.3f %10.3f" % (shape[0], shape[1], min(t), statistics.median(t), max(t),
                                                                        stage[shape][0], stage[shape][5]))
    for shape, rows in kernels.items():
        print("kernels, C=%d %d CTAs/SM (device ms per step; overlapping kernels both count):" % shape)
        for name, ms in rows[:12]:
            print("  %-50s %9.3f" % (name[:50], ms))
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": card, "steps": {"%dx%d" % s: times[s] for s in shapes},
                       "stage_ms": {"%dx%d" % s: list(stage[s]) for s in shapes},
                       "kernels": {"%dx%d" % s: rows for s, rows in kernels.items()}}, f, indent=1)
    blocks.ctx = ctxs[shapes[0]]
    blocks.close()
    for ctx in ctxs.values():
        ctx.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
