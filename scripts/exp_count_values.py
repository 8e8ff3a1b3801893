#!/usr/bin/env python3
"""Time vmb_count_values and vmb_rollup_count_values at the sizes of a large dashboard query.

count_values("x", q) by (...): S = 100 000 series x P = 8172 points (6.5 GB, the matrix of exp_order_aggr.py) holding 16 distinct
small integers per group at G = 1, 8 and 1024, and 4096 distinct at G = 1 and 8 (at G = 1024 that would be 4 M output series, far
past -search.maxSeriesPerAggrFunc), 5 % NaN, rows dealt round robin to the groups.  Yardstick: vmb_aggr_order DISTINCT on the same
matrix, which runs the same gather and sort.

count_values_over_time("x", m[5m]) at step 15 s: 20 000 reference-encoded gauge series x 8192 samples at 15 s with 6 distinct
values (64 distinct blocks, repeated), decoded by vmb_decode_blocks.  Yardstick: vmb_rollup with distinct_over_time on the same
batch.

Per case, one JSON line:
  count_ms   host clock around the sizing call (d_out == NULL), which ends in a device synchronise;
  call_ms    the same around the call that writes the matrix; median of --repeats after one warm-up;
  kernels    device time per kernel from torch.profiler in a profiled pair of calls of its own, and their sums by step;
  out_bytes  the output matrix (rows x P x 8).
The card's name and power limit are read in the same run.

  python scripts/exp_count_values.py [--repeats 3] [--only cv,cvt] [--out results/exp_count_values.jsonl]
"""
import argparse
import copy
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.dont_write_bytecode = True

from exp_rank_aggr import card_info  # noqa: E402

S, P = 100_000, 8172
STEPS = {"k_oa_gather": "gather", "k_oa_block_sort": "sort", "k_oa_merge": "sort", "k_oa_finish": "finish", "k_cv_runs": "runs",
         "k_cv_bucket": "distinct", "k_cv_unique": "distinct", "k_cv_fill": "write", "k_cv_scatter": "write",
         "k_cvt_keys": "window_keys", "k_cvt_ids": "count", "k_cvt_count": "count", "k_series_prepare": "preamble",
         "k_rollup": "rollup"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--only", default="cv,cvt")
    ap.add_argument("--out", default="")
    a = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    import victoriametrics_b200 as vm
    from blockgen import OBlock, to_blockset

    assert torch.cuda.is_available(), "this measurement needs the GPU"
    card = card_info()
    print(json.dumps({"card": card, "torch_device": torch.cuda.get_device_name(0)}), flush=True)
    lines = []

    class Buf:
        def __init__(self, nbytes):
            self.t = torch.empty(max(nbytes // 8, 1), dtype=torch.float64, device="cuda")
            self.ptr = self.t.data_ptr()

    def profiled(fn):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        kern, steps = {}, {}
        for e in prof.events():
            if e.device_type != torch.autograd.DeviceType.CUDA:
                continue
            k = e.name.split("(")[0].replace("void ", "")
            ms = e.time_range.elapsed_us() / 1e3
            kern[k] = kern.get(k, 0.0) + ms
            for prefix, step in STEPS.items():
                if prefix in k:
                    steps[step] = steps.get(step, 0.0) + ms
                    break
        return {k: round(v, 3) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])}, {k: round(v, 3) for k, v in steps.items()}

    def timed(fn):
        times = []
        for i in range(a.repeats + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            if i:
                times.append((time.perf_counter() - t0) * 1e3)
        return times

    def emit(rec):
        rec.update(card=card.get("name"), power_limit=card.get("power_limit"))
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    lib, ctx = vm._lib.lib(), vm._lib.default_context()
    if "cv" in a.only.split(","):
        import ctypes as C
        gen = torch.Generator(device="cuda").manual_seed(20261017)
        for card_n, groups in ((16, (1, 8, 1024)), (4096, (1, 8))):
            src = torch.randint(0, card_n, (S, P), dtype=torch.int64, device="cuda", generator=gen).double()
            src[torch.rand((S, P), device="cuda", generator=gen) < 0.05] = float("nan")
            for G in groups:
                gids = (np.arange(S) % G).astype(np.uint32)
                u32 = gids.ctypes.data_as(vm._lib.u32p)
                nout = C.c_size_t(0)
                grp, val = np.zeros(1, dtype=np.uint32), np.zeros(1)

                def count():
                    nout.value = 0
                    rc = lib.vmb_count_values(ctx.h, C.c_void_p(src.data_ptr()), S, P, u32, G, None, C.byref(nout),
                                              grp.ctypes.data_as(vm._lib.u32p), val.ctypes.data_as(vm._lib.f64p))
                    assert rc == -54, rc
                count()
                n = nout.value
                out = torch.empty((n, P), dtype=torch.float64, device="cuda")
                g2, v2 = np.zeros(n, dtype=np.uint32), np.zeros(n)

                def call():
                    nout.value = n
                    assert lib.vmb_count_values(ctx.h, C.c_void_p(src.data_ptr()), S, P, u32, G, C.c_void_p(out.data_ptr()),
                                                C.byref(nout), g2.ctypes.data_as(vm._lib.u32p), v2.ctypes.data_as(vm._lib.f64p)) == 0
                count_ms, call_ms = timed(count), timed(call)
                kern, steps = profiled(call)
                # a spot check: the number of non-NaN cells equals the non-NaN inputs
                ok = int((~torch.isnan(out)).sum().item()) <= S * P and float(torch.nansum(out).item()) == float((~torch.isnan(src)).sum().item())
                yard = torch.empty((G, P), dtype=torch.float64, device="cuda")
                ne = np.zeros(S, dtype=np.uint8)

                def distinct():
                    assert lib.vmb_aggr_order(ctx.h, 3, C.c_void_p(src.data_ptr()), S, P, u32, G, None, 0, C.c_void_p(yard.data_ptr()),
                                              ne.ctypes.data_as(vm._lib.u8p), None) == 0
                yard_ms = timed(distinct)
                ykern, ysteps = profiled(distinct)
                emit({"case": "count_values", "S": S, "P": P, "G": G, "distinct": card_n, "rows_out": n, "out_bytes": n * P * 8,
                      "count_ms": [round(t, 2) for t in count_ms], "call_ms": [round(t, 2) for t in call_ms],
                      "kernel_ms": round(sum(kern.values()), 2), "steps_ms": steps, "kernels": kern, "counts_sum_ok": ok,
                      "yardstick_distinct_ms": [round(t, 2) for t in yard_ms], "yardstick_kernel_ms": round(sum(ykern.values()), 2),
                      "yardstick_steps_ms": ysteps})
                del out, yard
                torch.cuda.empty_cache()
            del src
            torch.cuda.empty_cache()
    if "cvt" in a.only.split(","):
        rng = np.random.default_rng(20261017)
        NS, rows, dt = 20_000, 8192, 15_000
        t0 = 1_700_000_000_000
        ts = t0 + dt * np.arange(rows, dtype=np.int64)
        base = [OBlock(ts, rng.integers(0, 6, rows).astype(np.int64) * 25, -1) for _ in range(64)]
        blocks = []
        for s in range(NS):
            b = copy.copy(base[s % 64])
            b.series_idx = s
            blocks.append(b)
        descs, payload = to_blockset(blocks)
        blk = vm.storage.Blocks(descs, payload)
        start, end, step, window = t0, t0 + dt * (rows - 1), 15_000, 300_000
        pts = 1 + (end - start) // step
        holder = {}

        def over_time():
            series, _ = vm.storage.decode_blocks(blk)
            out, n, ser, tags, sc = vm.promql.count_values_over_time("x", series, start, end, step, window, 0, Buf)
            torch.cuda.synchronize()
            holder.update(n=n, scanned=sc)
            series.close()
            del out

        def decode_only():
            series, _ = vm.storage.decode_blocks(blk)
            torch.cuda.synchronize()
            series.close()

        dec_ms = timed(decode_only)
        call_ms = timed(over_time)
        kern, steps = profiled(over_time)
        rc = vm.promql.get_rollup_configs("distinct_over_time", start, end, step, window)
        yout = torch.empty((NS, pts), dtype=torch.float64, device="cuda")

        def yard():
            series, _ = vm.storage.decode_blocks(blk)
            rc.do_series(series, yout.data_ptr())
            torch.cuda.synchronize()
            series.close()
        yard_ms = timed(yard)
        ykern, ysteps = profiled(yard)
        emit({"case": "count_values_over_time", "series": NS, "samples": rows, "window_ms": window, "step_ms": step, "P": pts,
              "rows_out": holder["n"], "out_bytes": holder["n"] * pts * 8, "samples_scanned": holder["scanned"],
              "decode_ms": [round(t, 2) for t in dec_ms], "call_with_decode_ms": [round(t, 2) for t in call_ms],
              "kernel_ms": round(sum(kern.values()), 2), "steps_ms": steps, "kernels": kern,
              "yardstick_distinct_over_time_with_decode_ms": [round(t, 2) for t in yard_ms],
              "yardstick_kernel_ms": round(sum(ykern.values()), 2), "yardstick_steps_ms": ysteps})
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")
    return 0 if all(r.get("counts_sum_ok", True) for r in lines) else 1


if __name__ == "__main__":
    sys.exit(main())
