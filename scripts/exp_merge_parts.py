"""Times vmb_merge_parts end to end (host buffers in, the merged part's four files out) on two workloads and prints one JSON line
per workload with rows/s, the card's name and power limit.  Inputs are written by the library itself from a seeded RNG:
  fresh:  --parts parts x --series series of one fresh --rows-row block each (every block is re-encoded);
  full:   the same series as full 8192-row blocks, disjoint in time (every block passes through).
Usage: python scripts/exp_merge_parts.py [--parts 8] [--series 20000] [--rows 1024] [--repeat 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from victoriametrics_b200 import _lib, encoding, storage  # noqa: E402


def write_part(tsids, cols_ts, cols_vals, rows, pb=64):
    """a part of one block per series from [nseries x rows] columns (the library's writer; one index block per 809 headers)"""
    ns = len(tsids)
    ctx = _lib.default_context()
    tdata, toffs, tmts, tfirst = encoding.marshal_columns(cols_ts, pb, ctx=ctx)
    vdata, voffs, vmts, vfirst = encoding.marshal_columns(cols_vals, pb, ctx=ctx)
    d = np.zeros(ns, dtype=storage.DESC_DTYPE)
    d["first_value"], d["min_ts"], d["max_ts"] = vfirst, tfirst, cols_ts[:, -1]
    d["ts_off"], d["val_off"] = toffs[:-1], voffs[:-1]
    d["ts_size"], d["val_size"] = np.diff(toffs), np.diff(voffs)
    d["rows"], d["ts_mt"], d["val_mt"], d["precision_bits"] = rows, tmts, vmts, pb
    index, meta = bytearray(), bytearray()
    for i0 in range(0, ns, 809):
        raw = b"".join(storage.marshal_block_header(d[i], tsids[i]) for i in range(i0, min(ns, i0 + 809)))
        fr = encoding.zstd_compress(np.frombuffer(raw, dtype=np.uint8)).tobytes()
        row = np.zeros(1, dtype=storage.METAINDEX_DTYPE)
        row["tsid"][0] = np.frombuffer(tsids[i0], dtype=np.uint8)
        row["min_ts"], row["max_ts"] = d["min_ts"][i0:i0 + 809].min(), d["max_ts"][i0:i0 + 809].max()
        row["index_block_offset"], row["block_headers_count"], row["index_block_size"] = len(index), min(809, ns - i0), len(fr)
        meta += storage.marshal_metaindex_row(row[0])
        index += fr
    mi = encoding.zstd_compress_batch([bytes(meta)])[0]
    return storage.Part(mi, bytes(index), tdata, vdata)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", type=int, default=8)
    ap.add_argument("--series", type=int, default=20000)
    ap.add_argument("--rows", type=int, default=1024)
    ap.add_argument("--repeat", type=int, default=5)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip()
    rng = np.random.default_rng(1)
    tsids = [(7).to_bytes(8, "big") + bytes(8) + (s + 1).to_bytes(8, "big") for s in range(a.series)]
    for name, rows in (("fresh", a.rows), ("full", 8192)):
        parts = []
        for p in range(a.parts):
            t0 = 1_700_000_000_000 + p * rows * 15_000
            ts = t0 + np.arange(rows, dtype=np.int64)[None, :] * 15_000 + rng.integers(0, 50, (a.series, rows))
            ts.sort(axis=1)
            vals = np.cumsum(rng.integers(0, 100, (a.series, rows)), axis=1)
            parts.append(write_part(tsids, ts, vals, rows))
        storage.merge_parts(parts)  # warm-up
        times = []
        for _ in range(a.repeat):
            t = time.perf_counter()
            _, st = storage.merge_parts(parts)
            times.append(time.perf_counter() - t)
        med = float(np.median(times))
        total = a.parts * a.series * rows
        print(json.dumps(dict(workload=name, parts=a.parts, series=a.series, rows_in=total, blocks_out=st["blocks_count"],
                              median_s=med, rows_per_s=total / med, card=card)), flush=True)


if __name__ == "__main__":
    main()
