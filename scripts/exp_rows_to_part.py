"""Times vmb_parts_from_rows end to end (host rows in, every part's four files out) and prints one JSON line per workload with
rows/s, the digit passes of the radix sort, the card's name and power limit; then, in a separate profiled run per workload, the
kernel time of each stage from torch.profiler.  Inputs come from a seeded RNG:
  flush:   --sets sets x --rows rows (maxRawRowsPerShard = 8 MiB / sizeof(rawRow)), --series series each, in scrape order
           (tick-major, as ingestion sees them): every set needs the sort;
  sorted:  the same rows already in (TSID, Timestamp) order: the sort is skipped;
  big:     one set of --big-series series x 100 scrapes, scrape order.
Usage: python scripts/exp_rows_to_part.py [--sets 16] [--rows 174762] [--series 20000] [--big-series 100000] [--repeat 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from victoriametrics_b200 import storage  # noqa: E402

T0 = 1_700_000_000_000
STAGES = (("sort", ("k_fl_sorted", "k_fl_ranges", "k_fl_digit_mask", "k_fl_sort_count", "k_fl_sort_scatter", "k_fl_scan")),
          ("cut+gather", ("k_fl_run_", "k_fl_cut", "k_fl_gather")),
          ("decimal", ("k_float_to_decimal",)),
          ("dedup", ("k_fl_dedup",)),
          ("marshal+zstd", ("k_marshal_", "k_zstd_frames", "k_scan_lens", "k_compact")),
          ("writer+copies", ("k_ts_shared", "k_gather", "Memcpy", "Memset")))


def make_set(rng, nseries, rows, sort):
    """rows of nseries series in scrape order: tick after tick, every series once per tick (15 s apart, jittered)"""
    mg = (np.arange(nseries, dtype=np.uint64) * 7919) % 97 + 1
    ids = np.zeros((nseries, 24), dtype=np.uint8)
    ids[:, 0:8] = mg.astype(">u8").view(np.uint8).reshape(-1, 8)
    ids[:, 8:12] = np.frombuffer((1).to_bytes(4, "big"), dtype=np.uint8)
    ids[:, 12:16] = np.frombuffer((2).to_bytes(4, "big"), dtype=np.uint8)
    ids[:, 16:24] = (np.arange(nseries, dtype=np.uint64) + 1).astype(">u8").view(np.uint8).reshape(-1, 8)
    s = np.arange(rows) % nseries
    tick = np.arange(rows) // nseries
    ts = T0 + tick.astype(np.int64) * 15_000 + rng.integers(0, 1000, nseries)[s]
    vals = np.round(rng.normal(0, 1, rows) * 100, 2)
    if sort:
        key = ids[s].view(">u8").reshape(rows, 3)
        o = np.lexsort((ts, key[:, 2], key[:, 1], key[:, 0]))
        s, ts, vals = s[o], ts[o], vals[o]
    return np.ascontiguousarray(ids[s]), ts, vals, np.full(rows, 64, np.uint8)


def digit_passes(sets):
    """the radix sort's passes: the digits of (set, TSID, flipped timestamp) that are not the same in every row of the sets it sorts"""
    key = []
    for i, (ids, ts, _, _) in enumerate(sets):
        flipped = (ts.astype(np.uint64) ^ np.uint64(1 << 63)).astype("<u8").view(np.uint8).reshape(-1, 8)
        setb = np.full(ts.size, i, "<u4").view(np.uint8).reshape(-1, 4)
        key.append(np.concatenate([flipped, ids, setb], axis=1))
    k = np.concatenate(key)
    return int((k != k[:1]).any(axis=0).sum())


def is_sorted(ids, ts):
    k = np.concatenate([ids.view(">u8").reshape(-1, 3), (ts.astype(np.uint64) ^ np.uint64(1 << 63))[:, None]], axis=1)
    a, b = k[:-1], k[1:]
    lt = np.zeros(len(a), bool)
    eq = np.ones(len(a), bool)
    for c in range(4):
        lt |= eq & (a[:, c] < b[:, c])
        eq &= a[:, c] == b[:, c]
    return bool((lt | eq).all())


def profile(sets):
    import torch
    from torch.profiler import ProfilerActivity, profile as prof
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        storage.parts_from_rows(sets)
        torch.cuda.synchronize()
    ms = {name: 0.0 for name, _ in STAGES}
    other = 0.0
    for e in p.key_averages():
        t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 1000.0
        if t <= 0:
            continue
        for name, keys in STAGES:
            if any(k in e.key for k in keys):
                ms[name] += t
                break
        else:
            other += t
    ms["other"] = other
    return {k: round(v, 3) for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sets", type=int, default=16)
    ap.add_argument("--rows", type=int, default=174762)
    ap.add_argument("--series", type=int, default=20000)
    ap.add_argument("--big-series", type=int, default=100000)
    ap.add_argument("--repeat", type=int, default=5)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip()
    rng = np.random.default_rng(1)
    flush = [make_set(rng, a.series, a.rows, False) for _ in range(a.sets)]
    rng = np.random.default_rng(1)
    workloads = (("flush", flush), ("sorted", [make_set(rng, a.series, a.rows, True) for _ in range(a.sets)]),
                 ("big", [make_set(rng, a.big_series, a.big_series * 100, False)]))
    for name, sets in workloads:
        storage.parts_from_rows(sets)  # warm-up
        times = []
        for _ in range(a.repeat):
            t = time.perf_counter()
            out = storage.parts_from_rows(sets)
            times.append(time.perf_counter() - t)
        med = float(np.median(times))
        rows = sum(s[1].size for s in sets)
        unsorted = [s for s in sets if not is_sorted(s[0], s[1])]
        print(json.dumps(dict(workload=name, sets=len(sets), rows_in=rows, blocks_out=sum(st["blocks_count"] for _, st in out),
                              sorted_sets=len(sets) - len(unsorted), digit_passes=digit_passes(unsorted) if unsorted else 0,
                              median_s=med, min_s=min(times), rows_per_s=rows / med, card=card)), flush=True)
        print(json.dumps(dict(workload=name, kernel_ms=profile(sets), card=card)), flush=True)


if __name__ == "__main__":
    main()
