#!/usr/bin/env python3
"""What bounds the Huffman literal decoder (k_huf_decode) on the flagship workload (bench.py at its defaults: rate(m[5m])
step 15 s over 100 000 reference-encoded counter blocks x 8192 samples, blocks resident in HBM), run one-shot
(VMB_FUSED_CHUNKS=1: the zstd stage of the whole batch, then one fused launch).

Attribution builds of libvmb200.so (-DVMB_HUF_EXP=<mask>, zstd.cu) are compiled into a temporary directory -- the product
library is left alone -- and each takes one suspect off the symbol loop while the rest stays live:
    1 store     no STG.128: the 16-byte pieces are XOR-folded per lane, one store per stream
    2 lookup    the symbol is cut from the code bits: no perm / adj shared-memory loads
    4 convert   the code length from integer compares on packed thresholds: no I2F / F2I
    8 input     the ring is refilled from registers: no input LDG in the loop
   16 l1        input loads bypass L1 (ld.global.nc.L1::no_allocate)
   64 carveout  shared-memory carveout just large enough for the grid cap, the rest of the SM's memory is L1
The outputs of store, lookup and input are wrong, and those builds fail every frame so that no later kernel reads them; only
their kernel time is read.  Mask 0 is the
product library of the tree.  Every library runs in its own process over the same generated blocks, the libraries alternate
over --rounds, and each process times k_huf_decode (torch.profiler device time, after warm-up) at every grid cap of --caps
(CTAs per SM, VMB_HUF_CTAS_PER_SM).  The phase-clock build (mask 32) adds lane 0's clock64() cycles per phase: table build,
stream set-up + ring priming, head, body, tail.

Prints the card, its power limit and SM clock (read in the same run), kernel ms min / max over the rounds and symbols per SM
cycle at the maximum SM clock.

  python scripts/exp_huf_bound.py [--variants 0,1,2,4,8,16,64] [--caps 2,4,8,12] [--rounds 2] [--prebuilt DIR] [--json out]
"""
import argparse
import ctypes as C
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

NAMES = {0: "product", 1: "store", 2: "lookup", 4: "convert", 8: "input", 16: "l1", 32: "phases", 64: "carveout"}
PHASES = ["table build (+ wait for the warp)", "set-up + priming", "head", "body", "tail"]
SMS = 132
WRONG = 1 | 2 | 8  # masks whose literals are wrong: zstd.cu fails their frames, so that no later kernel reads them


def variant_name(mask):
    return NAMES.get(mask) or "+".join(NAMES[b] for b in sorted(NAMES) if b and mask & b)


def build_variant(mask, tmp):
    d = os.path.join(tmp, "exp%d" % mask)
    os.makedirs(d, exist_ok=True)
    so = os.path.join(d, "libvmb200.so")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "victoriametrics_b200", "csrc"), "OUT=" + so,
                           "LOG=" + os.path.join(d, "ptxas.log"), "NVEXTRA=-DVMB_HUF_EXP=%d" % mask])
    return so


def literal_symbols(descs, payload):
    """literal bytes of the Huffman-coded frames (one compressed block, compressed literals): what k_huf_decode decodes"""
    total = frames = 0
    for col in ("ts", "val"):
        for off, size in zip(descs[col + "_off"].tolist(), descs[col + "_size"].tolist()):
            b = payload[off:off + min(size, 32)].tobytes()
            if size < 12 or b[:4] != b"\x28\xb5\x2f\xfd":
                continue
            fhd = b[4]
            fcs_flag, single, did = fhd >> 6, (fhd >> 5) & 1, fhd & 3
            pos = 5 + (0 if single else 1) + (0, 1, 2, 4)[did] + ((1 if single else 0) if fcs_flag == 0 else (1 << fcs_flag))
            bh = int.from_bytes(b[pos:pos + 3], "little")
            pos += 3
            if (bh >> 1) & 3 != 2 or b[pos] & 3 != 2:
                continue
            sf = (b[pos] >> 2) & 3
            v = int.from_bytes(b[pos:pos + 5], "little")
            total += (v >> 4) & (0x3ff if sf < 2 else (0x3fff if sf == 2 else 0x3ffff))
            frames += 1
    return total, frames


def worker(a):
    """one library: k_huf_decode ms per call at every cap -> one JSON line on stdout"""
    from victoriametrics_b200 import _lib
    _lib.SO_PATH = os.path.abspath(a.so)
    L = _lib.lib()
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
        os.environ["VMB_HUF_CTAS_PER_SM"] = str(cap)
        ctxs[cap] = vm.Context(dev, stream.cuda_stream)
    del os.environ["VMB_FUSED_CHUNKS"], os.environ["VMB_HUF_CTAS_PER_SM"]
    data = np.load(a.data)
    descs, payload = data["descs"], data["payload"]
    start, end, step = bench.query_range(a.rows, 300_000, 15_000)
    points = 1 + (end - start) // step
    blocks = storage.Blocks(descs, payload, ctxs[caps[0]])
    out = torch.empty((descs.shape[0], points), dtype=torch.float64, device="cuda")

    def run(cap):
        blocks.ctx = ctxs[cap]
        try:
            promql.eval_rollup_func("rate", blocks, start, end, step, 300_000, out_dev_ptr=out.data_ptr())
        except _lib.VmbError as e:  # builds that write wrong literals fail every frame on purpose
            if not (a.mask & WRONG and e.code in (-6, -53)):
                raise

    res = {"ms": {}, "phases": None}
    for cap in caps:
        for _ in range(a.warmup):
            run(cap)
    torch.cuda.synchronize()
    for cap in caps:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.steps):
                run(cap)
            torch.cuda.synchronize()
        ms = sum(e.time_range.elapsed_us() for e in prof.events()
                 if e.device_type == torch.autograd.DeviceType.CUDA and e.name.startswith("k_huf_decode")) / 1e3 / a.steps
        res["ms"][str(cap)] = ms
    if hasattr(L, "vmb_huf_phase_cycles"):
        read = L.vmb_huf_phase_cycles
        read.restype = C.c_int
        read.argtypes = [C.c_void_p, C.c_int]
        slots = read(None, 0)
        assert slots == len(PHASES) + 1, slots
        res["phases"] = {}
        for cap in caps:
            torch.cuda.synchronize()
            read(None, 1)
            run(cap)
            torch.cuda.synchronize()
            buf = np.zeros(slots, dtype=np.uint64)
            if read(buf.ctypes.data, 1) < 0:
                raise SystemExit("reading the phase clocks failed")
            res["phases"][str(cap)] = buf.tolist()
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
    ap.add_argument("--variants", default="0,1,2,4,8,16,64,32", help="VMB_HUF_EXP masks (0 = the product library)")
    ap.add_argument("--caps", default="2,4,8,12", help="k_huf_decode grid caps, CTAs per SM")
    ap.add_argument("--rounds", type=int, default=2, help="alternating rounds over the libraries")
    ap.add_argument("--steps", type=int, default=5, help="profiled calls per cap")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--prebuilt", default="", help="directory with exp<mask>/libvmb200.so made before instead of compiling")
    ap.add_argument("--json", default="", help="also write the result here")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--so", default="", help=argparse.SUPPRESS)
    ap.add_argument("--mask", type=int, default=0, help=argparse.SUPPRESS)
    ap.add_argument("--data", default="", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a)

    import bench
    masks = [int(x) for x in a.variants.split(",")]
    tmp = tempfile.mkdtemp(prefix="vmb_hufexp_")
    libs = {}
    for m in masks:
        pre = os.path.join(a.prebuilt, "exp%d" % m, "libvmb200.so") if a.prebuilt else ""
        if m == 0:
            libs[m] = os.path.join(ROOT, "victoriametrics_b200", "libvmb200.so")
        elif pre and os.path.exists(pre):
            libs[m] = pre
        else:
            libs[m] = build_variant(m, tmp)
    descs, payload, _ = bench.gen_blocks(a.blocks, a.rows, seed=1234, kind="counter")
    syms, frames = literal_symbols(descs, payload)
    data = os.path.join(tmp, "blocks.npz")
    np.savez(data, descs=descs, payload=payload)
    del payload

    ms = defaultdict(lambda: defaultdict(list))
    phases, card = {}, {}
    for r in range(a.rounds):
        for m in masks:
            cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--so", libs[m], "--mask", str(m), "--data", data,
                   "--caps", a.caps,
                   "--rows", str(a.rows), "--steps", str(a.steps), "--warmup", str(a.warmup)]
            p = subprocess.run(cmd, capture_output=True, text=True)
            line = [x for x in p.stdout.splitlines() if x.startswith("RESULT ")]
            if p.returncode or not line:
                sys.stderr.write(p.stdout[-3000:] + p.stderr[-3000:])
                raise SystemExit("variant %d (%s) failed" % (m, variant_name(m)))
            res = json.loads(line[0][7:])
            for cap, v in res["ms"].items():
                ms[m][int(cap)].append(v)
            if res["phases"]:
                phases[m] = res["phases"]
            card = res["card"]
            print("round %d %-10s %s" % (r, variant_name(m), " ".join("%s:%.3f" % kv for kv in res["ms"].items())), flush=True)

    clk = mhz(card.get("sm_clock_max")) * 1e6
    caps = [int(x) for x in a.caps.split(",")]
    print("card: %s, power limit %s, SM clock %s (max %s)" % (card.get("name"), card.get("power_limit"), card.get("sm_clock"),
                                                              card.get("sm_clock_max")))
    print("workload: rate(m[5m]) over %d counter blocks x %d samples, one-shot zstd stage; %d Huffman frames, %.3f G literal "
          "symbols; k_huf_decode torch.profiler device ms per call, min-max over %d alternating rounds x %d calls; "
          "symbols per SM cycle at the maximum SM clock" % (a.blocks, a.rows, frames, syms / 1e9, a.rounds, a.steps))
    print("%-22s" % "variant" + "".join("%22s" % ("%d CTAs/SM" % c) for c in caps))
    for m in masks:
        cells = []
        for c in caps:
            t = ms[m][c]
            cells.append("%8.3f-%-6.3f %5.2f" % (min(t), max(t), syms / (min(t) * 1e-3 * clk * SMS)))
        print("%-22s" % ("%d %s" % (m, variant_name(m))) + "".join("%22s" % x for x in cells))
    for m, per in phases.items():
        for c in caps:
            buf = np.array(per[str(c)], dtype=np.float64)
            tot = buf[:len(PHASES)].sum()
            print("phases (%s build, %d CTAs/SM, lane 0 of every warp, %d symbols): " % (variant_name(m), c, int(buf[-1])) +
                  ", ".join("%s %.1f%%" % (n, 100.0 * x / tot) for n, x in zip(PHASES, buf)) +
                  "; body %.1f cycles per symbol step" % (buf[3] / max(buf[-1], 1)))
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": card, "symbols": syms, "frames": frames,
                       "ms": {variant_name(m): {str(c): v for c, v in per.items()} for m, per in ms.items()},
                       "phases": {variant_name(m): v for m, v in phases.items()}}, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
