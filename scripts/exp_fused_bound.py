#!/usr/bin/env python3
"""What bounds the fused rollup kernel (k_fused_rollup) on the flagship workload (bench.py at its defaults: rate(m[5m]) step
15 s over 100 000 reference-encoded counter blocks x 8192 samples, blocks resident in HBM), run one-shot (VMB_FUSED_CHUNKS=1:
the zstd stage of the whole batch, then one fused launch).

Attribution builds of libvmb200.so (-DVMB_FUSED_EXP=<mask>, fused.cu) are compiled into a temporary directory -- the product
library is left alone -- and each takes one suspect off the per-row loops while the rest stays live:
     1 store     no per-point store: the points are XOR-folded per thread, one store per thread and series
     2 conflict  raw deltas in a lane-major int32 array (no bank conflicts on the parse's stores and the emit's loads);
                 16 KB more per CTA, so compare it with the product at the caps where both fit
     4 order     the emit's and the points' shared loads not volatile, the emit's stores without a memory clobber
     8 guards    the emit's full four-row batches without the per-row guards, reset candidates and special-value test
    16 rcr       no counter-reset pass over the rows (the emit still finds the candidates)
    32 prologue  every series after a CTA's first reuses that series' record (copied in shared memory instead of fetched; only
                 the output row is its own), its first fill issued one series ahead: what the record fetch costs.  Its
                 streams are the first series', counter resets included, so the per-CTA work differs from the product's
The outputs of these builds may be wrong; only their kernel time is read.  Mask 0 is the product library of the tree.  Every
library runs in its own process over the same generated blocks, the libraries alternate over --rounds, and each process times
k_fused_rollup (torch.profiler device time, after warm-up) at every grid cap of --caps (CTAs per SM, VMB_FUSED_CTAS_PER_SM; the
occupancy calculator caps a build whose CTA does not fit).  Every build must launch as many kernels per call as the product:
a series a build hands to the un-fused path would add that path's launches.

Prints the card, its power limit and SM clock (read in the same run), kernel ms min / max over the rounds and samples (rows)
per SM cycle at the maximum SM clock.  --func avg_over_time --kind gauge runs the generic instantiation's path instead.

--libs name=path,... alternates more libraries with the builds (a parent's product, say); the result digest (wrapping sums of
the result's bits over rows and over columns) tells whether two libraries computed the same.

  python scripts/exp_fused_bound.py [--variants 0,1,2,4,8,16,32] [--caps 3,4,5] [--rounds 2] [--func rate --kind counter]
                                    [--libs name=path,...] [--prebuilt DIR] [--json out]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile
from collections import defaultdict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.dont_write_bytecode = True

NAMES = {0: "product", 1: "store", 2: "conflict", 4: "order", 8: "guards", 16: "rcr", 32: "prologue"}
SMS = 132


def variant_name(mask):
    if isinstance(mask, str):
        return mask
    return NAMES.get(mask) or "+".join(NAMES[b] for b in sorted(NAMES) if b and mask & b)


def build_variant(mask, tmp):
    d = os.path.join(tmp, "exp%d" % mask)
    os.makedirs(d, exist_ok=True)
    so = os.path.join(d, "libvmb200.so")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "victoriametrics_b200", "csrc"), "OUT=" + so,
                           "LOG=" + os.path.join(d, "ptxas.log"), "NVEXTRA=-DVMB_FUSED_EXP=%d" % mask])
    return so


def worker(a):
    """one library: k_fused_rollup ms per call at every cap -> one JSON line on stdout"""
    from victoriametrics_b200 import _lib
    _lib.SO_PATH = os.path.abspath(a.so)
    _lib.lib()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    import victoriametrics_b200 as vm
    from victoriametrics_b200 import promql, storage

    dev = 0
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream()
    caps = [int(x) for x in a.caps.split(",")]
    ctxs = {}
    os.environ["VMB_FUSED_CHUNKS"] = "1"
    for cap in caps:
        os.environ["VMB_FUSED_CTAS_PER_SM"] = str(cap)
        ctxs[cap] = vm.Context(dev, stream.cuda_stream)
    del os.environ["VMB_FUSED_CHUNKS"], os.environ["VMB_FUSED_CTAS_PER_SM"]
    data = np.load(a.data)
    descs, payload = data["descs"], data["payload"]
    start, end, step = bench.query_range(a.rows, 300_000, 15_000)
    points = 1 + (end - start) // step
    blocks = storage.Blocks(descs, payload, ctxs[caps[0]])
    out = torch.empty((descs.shape[0], points), dtype=torch.float64, device="cuda")

    def run(cap):
        blocks.ctx = ctxs[cap]
        promql.eval_rollup_func(a.func, blocks, start, end, step, 300_000, out_dev_ptr=out.data_ptr())

    res = {"ms": {}, "launches": {}, "digest": {}}
    for cap in caps:
        for _ in range(a.warmup):
            run(cap)
        n0 = ctxs[cap].launch_count
        run(cap)
        res["launches"][str(cap)] = ctxs[cap].launch_count - n0
        # wrapping int64 sums of the result's bits over rows and over columns: equal for builds that compute the same
        bits = out.view(torch.int64)
        res["digest"][str(cap)] = hashlib.sha1(bits.sum(dim=1).cpu().numpy().tobytes() +
                                               bits.sum(dim=0).cpu().numpy().tobytes()).hexdigest()[:12]
    torch.cuda.synchronize()
    for cap in caps:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.steps):
                run(cap)
            torch.cuda.synchronize()
        ms = sum(e.time_range.elapsed_us() for e in prof.events()
                 if e.device_type == torch.autograd.DeviceType.CUDA and "k_fused_rollup" in e.name) / 1e3 / a.steps
        res["ms"][str(cap)] = ms
    from fused_kernels import card_info
    res["card"] = card_info(dev)
    blocks.ctx = ctxs[caps[0]]
    blocks.close()
    for ctx in ctxs.values():
        ctx.close()
    print("RESULT " + json.dumps(res), flush=True)
    return 0


def mhz(s):
    try:
        return float(str(s).split()[0])
    except (ValueError, IndexError):
        return float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=100_000)
    ap.add_argument("--rows", type=int, default=8192)
    ap.add_argument("--func", default="rate")
    ap.add_argument("--kind", default="counter", help="bench.gen_blocks kind of the generated blocks")
    ap.add_argument("--variants", default="0,1,2,4,8,16,32", help="VMB_FUSED_EXP masks (0 = the product library)")
    ap.add_argument("--caps", default="3,4,5", help="k_fused_rollup grid caps, CTAs per SM")
    ap.add_argument("--rounds", type=int, default=2, help="alternating rounds over the libraries")
    ap.add_argument("--steps", type=int, default=5, help="profiled calls per cap")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--prebuilt", default="", help="directory with exp<mask>/libvmb200.so made before instead of compiling")
    ap.add_argument("--libs", default="", help="more libraries to alternate with the builds, name=path,... (e.g. the parent's)")
    ap.add_argument("--json", default="", help="also write the result here")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--so", default="", help=argparse.SUPPRESS)
    ap.add_argument("--data", default="", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a)

    import bench
    masks = [int(x) for x in a.variants.split(",") if x]
    tmp = tempfile.mkdtemp(prefix="vmb_fusedexp_")
    libs = {}
    for kv in filter(None, a.libs.split(",")):
        name, path = kv.split("=", 1)
        libs[name] = os.path.abspath(path)
    for m in masks:
        pre = os.path.join(a.prebuilt, "exp%d" % m, "libvmb200.so") if a.prebuilt else ""
        if m == 0:
            libs[m] = os.path.join(ROOT, "victoriametrics_b200", "libvmb200.so")
        elif pre and os.path.exists(pre):
            libs[m] = pre
        else:
            libs[m] = build_variant(m, tmp)
    descs, payload, _ = bench.gen_blocks(a.blocks, a.rows, seed=1234, kind=a.kind)
    data = os.path.join(tmp, "blocks.npz")
    np.savez(data, descs=descs, payload=payload)
    del payload
    samples = a.blocks * a.rows
    masks = list(libs)

    ms = defaultdict(lambda: defaultdict(list))
    launches, digests, card = {}, {}, {}
    for r in range(a.rounds):
        for m in masks:
            cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--so", libs[m], "--data", data, "--caps", a.caps,
                   "--func", a.func, "--rows", str(a.rows), "--steps", str(a.steps), "--warmup", str(a.warmup)]
            p = subprocess.run(cmd, capture_output=True, text=True)
            line = [x for x in p.stdout.splitlines() if x.startswith("RESULT ")]
            if p.returncode or not line:
                sys.stderr.write(p.stdout[-3000:] + p.stderr[-3000:])
                raise SystemExit("variant %s (%s) failed" % (m, variant_name(m)))
            res = json.loads(line[0][7:])
            for cap, v in res["ms"].items():
                ms[m][int(cap)].append(v)
            launches[m] = res["launches"]
            digests[m] = res["digest"]
            card = res["card"]
            print("round %d %-10s %s" % (r, variant_name(m), " ".join("%s:%.3f" % kv for kv in res["ms"].items())), flush=True)

    clk = mhz(card.get("sm_clock_max")) * 1e6
    caps = [int(x) for x in a.caps.split(",")]
    print("card: %s, power limit %s, SM clock %s (max %s)" % (card.get("name"), card.get("power_limit"), card.get("sm_clock"),
                                                              card.get("sm_clock_max")))
    print("workload: %s over %d %s blocks x %d samples, one-shot zstd stage; k_fused_rollup torch.profiler device ms per call, "
          "min-max over %d alternating rounds x %d calls; samples per SM cycle at the maximum SM clock"
          % (a.func, a.blocks, a.kind, a.rows, a.rounds, a.steps))
    print("%-14s" % "variant" + "".join("%22s" % ("%d CTAs/SM" % c) for c in caps) + "   launches per call, result digest")
    for m in masks:
        cells = []
        for c in caps:
            t = ms[m][c]
            cells.append("%8.3f-%-6.3f %5.2f" % (min(t), max(t), samples / (min(t) * 1e-3 * clk * SMS)))
        label = m if isinstance(m, str) else "%d %s" % (m, variant_name(m))
        print("%-14s" % label + "".join("%22s" % x for x in cells) + "   " +
              " ".join("%s" % launches[m][str(c)] for c in caps) + "  " + " ".join(digests[m][str(c)] for c in caps))
    bad = [variant_name(m) for m in masks if launches[m] != launches[masks[0]]]
    if bad:
        print("WARNING: launches per call differ from %s's (different bails): %s" % (variant_name(masks[0]), ", ".join(bad)))
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": card, "samples": samples, "func": a.func, "kind": a.kind,
                       "launches": {variant_name(m): v for m, v in launches.items()},
                       "digest": {variant_name(m): v for m, v in digests.items()},
                       "ms": {variant_name(m): {str(c): v for c, v in per.items()} for m, per in ms.items()}}, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
