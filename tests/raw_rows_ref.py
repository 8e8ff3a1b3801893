"""Restatement of the reference's part flush in plain Python (lib/storage), independent of the product's flush code:

  rawRowsSort          raw_row.go:49-75: rows ordered by TSID.Less (the byte order of the 24-byte marshaled TSID), then Timestamp;
                       stably, so rows with equal (TSID, Timestamp) keep their input order (the library's tie rule)
  marshalToInmemoryPart  raw_row.go:81-136: the cut (a block ends where the MetricID differs from the block's first row's, or at
                       maxRowsPerBlock rows; it takes the TSID and PrecisionBits of its first row), AppendFloatToDecimal per block
                       (the library's host vmb_float_to_decimal), then WriteExternalBlock block_stream_writer.go:138 with
                       deduplicateSamplesDuringMerge and the writer rules of part_merge_ref.py

A row set is (tsids [n x 24] uint8, timestamps int64 [n], values float64 [n], precision_bits uint8 [n])."""
import numpy as np

import partgen
from part_merge_ref import (INT64_MAX, INT64_MIN, MAX_BLOCK_SIZE, MAX_ROWS_PER_BLOCK, deduplicate_samples_during_merge, host_frame,
                            host_marshal, read_part)

__all__ = ["sort_order", "cut_blocks", "marshal_to_inmemory_part", "merge_input", "read_part", "INT64_MIN", "INT64_MAX"]


def float_to_decimal(vals):
    """decimal.AppendFloatToDecimal decimal.go:173 -> (mantissas, scale)"""
    from victoriametrics_b200 import decimal
    m, e = decimal.append_float_to_decimal(np.asarray(vals, dtype=np.float64))
    return [int(x) for x in m], e


def sort_order(tsids, ts):
    """the stable order of the rows by (TSID bytes, Timestamp)"""
    t = np.asarray(tsids, dtype=np.uint8).reshape(-1, 24)
    keys = [(bytes(t[i]), int(ts[i])) for i in range(len(ts))]
    return sorted(range(len(ts)), key=keys.__getitem__)


def cut_blocks(tsids, order):
    """raw_row.go:111-127 over the sorted rows -> [(first, end)] positions in `order`"""
    mid = np.ascontiguousarray(np.asarray(tsids, dtype=np.uint8).reshape(-1, 24)[:, 16:24]).view(">u8").ravel().tolist()  # MetricID
    out = []
    start = 0
    for i in range(1, len(order) + 1):
        if i < len(order) and mid[order[i]] == mid[order[start]] and i - start < MAX_ROWS_PER_BLOCK:
            continue
        out.append((start, i))
        start = i
    return out


def marshal_to_inmemory_part(tsids, ts, vals, pbs, dedup_interval=0, marshal=host_marshal, frame=host_frame):
    """one row set -> dict(metaindex_bin, metaindex_raw, index_bin, timestamps_bin, values_bin, stats, blocks) as
    part_merge_ref.merge_parts returns it; blocks = [(tsid, header, ts, mantissas, tdata, vdata)] in file order, the rows as written
    (after dedup).  metaindex_bin is None where the library writes a frame of Raw blocks (an empty metaindex)."""
    tsids = np.asarray(tsids, dtype=np.uint8).reshape(-1, 24)
    ts = [int(x) for x in np.asarray(ts, dtype=np.int64)]
    vals = np.asarray(vals, dtype=np.float64)
    pbs = [int(x) for x in np.asarray(pbs, dtype=np.uint8)]
    st = dict(rows_count=0, blocks_count=0, min_ts=INT64_MAX, max_ts=INT64_MIN, rows_merged=0, rows_deleted=0)
    W = dict(blocks=[], ts=bytearray(), vals=bytearray(), index=bytearray(), meta=bytearray(), cur=bytearray(), mr=None, prev=b"", prev_off=0)

    def flush_index():  # flushIndexData block_stream_writer.go:182
        if not W["cur"]:
            return
        comp = frame(bytes(W["cur"]))
        mr = W["mr"]
        W["meta"] += partgen.pack_metaindex_row(mr["tsid"], mr["count"], mr["min_ts"], mr["max_ts"], len(W["index"]), len(comp))
        W["index"] += comp
        W["cur"] = bytearray()
        W["mr"] = None

    def write(tsid, bts, bvals, scale, pb):  # Block.Init + WriteExternalBlock
        st["rows_merged"] += len(bts)
        if dedup_interval > 0 and len(bts) >= 2:
            bts, bvals = deduplicate_samples_during_merge(bts, bvals, dedup_interval)
        h = dict(scale=scale, precision_bits=pb, rows=len(bvals), max_ts=bts[-1])
        vd, h["val_mt"], h["first_value"] = marshal(bvals, pb)
        td, h["ts_mt"], h["min_ts"] = marshal(bts, pb)
        h["ts_size"], h["val_size"] = len(td), len(vd)
        share = len(W["prev"]) > 0 and td == W["prev"]
        h["ts_off"] = W["prev_off"] if share else len(W["ts"])
        h["val_off"] = len(W["vals"])
        hd = partgen.pack_header(tsid, h)
        if len(W["cur"]) + len(hd) > MAX_BLOCK_SIZE:
            flush_index()
        W["cur"] += hd
        if W["mr"] is None:
            W["mr"] = dict(tsid=tsid, count=0, min_ts=h["min_ts"], max_ts=h["max_ts"])
        mr = W["mr"]
        mr["count"] += 1
        mr["min_ts"], mr["max_ts"] = min(mr["min_ts"], h["min_ts"]), max(mr["max_ts"], h["max_ts"])
        if not share:
            W["prev"], W["prev_off"] = td, len(W["ts"])
            W["ts"] += td
        W["vals"] += vd
        W["blocks"].append((tsid, h, list(bts), list(bvals), td, vd))
        st["blocks_count"] += 1
        st["rows_count"] += h["rows"]
        st["min_ts"], st["max_ts"] = min(st["min_ts"], h["min_ts"]), max(st["max_ts"], h["max_ts"])

    order = sort_order(tsids, ts)
    for a, b in cut_blocks(tsids, order):
        rows = order[a:b]
        mant, scale = float_to_decimal(vals[rows])
        write(bytes(tsids[rows[0]]), [ts[r] for r in rows], mant, scale, pbs[rows[0]])
    flush_index()
    meta = bytes(W["meta"])
    mi = None if len(meta) == 0 or 128 * 1024 < len(meta) <= 262143 else frame(meta)
    return dict(metaindex_bin=mi, metaindex_raw=meta, index_bin=bytes(W["index"]), timestamps_bin=bytes(W["ts"]),
                values_bin=bytes(W["vals"]), stats=st, blocks=W["blocks"])


def merge_input(part):
    """a restated part as part_merge_ref.merge_parts takes it: [(tsid, header, ts, vals, tdata, vdata)], rows as the reference side
    decodes them from the part's files"""
    if not part["blocks"]:
        return []
    rows = read_part(part["metaindex_bin"], part["index_bin"], part["timestamps_bin"], part["values_bin"], len(part["metaindex_raw"]) + 16)
    return [(t, h, ts, vs, b[4], b[5]) for (t, h, ts, vs), b in zip(rows, part["blocks"])]
