"""Test-only writer of the reference's part layout (lib/storage/block_stream_writer.go:138 WriteExternalBlock, :182
flushIndexData): timestamps.bin / values.bin hold the marshaled columns (identical consecutive timestamp payloads stored
once), index.bin the zstd-compressed runs of 81-byte block headers (a run is flushed before it would exceed maxBlockSize),
metaindex.bin one zstd frame of 56-byte rows.  Compression = the reference's libzstd (oracle/_ref), payloads = the oracle's
MarshalData -- nothing of the product is on this side except the struct layouts the checks compare against.
pure_go=True writes the frames in the header layout of the reference's builds without cgo (klauspost/compress): below
256 bytes they carry no Frame_Content_Size, up to 1024 bytes a Window_Descriptor beside it."""
import struct

import numpy as np

import oracle_lib as O
import zstd_shapes

MAX_BLOCK_SIZE = 64 * 1024  # block.go:18


def zz(v):
    return ((v << 1) ^ (v >> 63)) & 0xFFFFFFFFFFFFFFFF


def pack_tsid(metric_group_id, job_id, instance_id, metric_id):
    return struct.pack(">QIIQ", metric_group_id, job_id, instance_id, metric_id)  # tsid.go:62


def pack_header(tsid, h):
    """blockHeader.Marshal block_header.go:104, written independently of the product and of the oracle"""
    sc = h["scale"]
    return tsid + struct.pack(">QQQQQIIIHBBB", zz(h["min_ts"]), zz(h["max_ts"]), zz(h["first_value"]), h["ts_off"], h["val_off"],
                              h["ts_size"], h["val_size"], h["rows"], ((sc << 1) ^ (sc >> 15)) & 0xFFFF, h["ts_mt"], h["val_mt"],
                              h["precision_bits"])


def pack_metaindex_row(tsid, count, min_ts, max_ts, off, size):
    return tsid + struct.pack(">IQQQI", count, zz(min_ts), zz(max_ts), off, size)  # metaindex_row.go:61


def pure_go_columns(block, level):
    """rewrite the zstd columns (MarshalType 1 / 4) of an OBlock in place as the pure-Go writer frames them"""
    for d, mt in (("tdata", "tmt"), ("vdata", "vmt")):
        if getattr(block, mt) in (1, 4):
            raw = O.zstd_ref_decompress(getattr(block, d), block.rows * 10 + 16)
            setattr(block, d, zstd_shapes.pure_go_frame(raw, compressionLevel=level))


def write_part(series, level=1, max_index_block=MAX_BLOCK_SIZE, pure_go=False):
    """series: list of (tsid bytes, [OBlock, ...]) sorted by tsid, blocks by min timestamp.
    -> dict(metaindex_bin, index_bin, timestamps_bin, values_bin, headers=[(tsid, header dict)], index_blocks=n)
    pure_go: every frame in the pure-Go writer's header layout (the blocks' zstd columns are rewritten in place)"""
    def compress(raw):
        raw = np.frombuffer(bytes(raw), dtype=np.uint8)
        return (zstd_shapes.pure_go_frame(raw, compressionLevel=level) if pure_go else O.zstd_ref_compress(raw, level)).tobytes()

    tsb, vsb, index_bin, metaindex = bytearray(), bytearray(), bytearray(), bytearray()
    headers = []
    cur = bytearray()
    mr = None
    prev_ts, prev_ts_off = None, 0
    n_index_blocks = 0

    def flush():
        nonlocal cur, mr, n_index_blocks
        if not cur:
            return
        comp = compress(cur)
        metaindex.extend(pack_metaindex_row(mr["tsid"], mr["count"], mr["min_ts"], mr["max_ts"], len(index_bin), len(comp)))
        index_bin.extend(comp)
        cur = bytearray()
        mr = None
        n_index_blocks += 1

    for tsid, blocks in series:
        for b in blocks:
            if pure_go:
                pure_go_columns(b, level)
            h = b.header()
            td = b.tdata.tobytes()
            if prev_ts is not None and len(prev_ts) > 0 and td == prev_ts:
                h["ts_off"] = prev_ts_off
            else:
                h["ts_off"] = len(tsb)
                prev_ts, prev_ts_off = td, len(tsb)
                tsb.extend(td)
            h["val_off"] = len(vsb)
            vsb.extend(b.vdata.tobytes())
            hd = pack_header(tsid, h)
            if len(cur) + len(hd) > max_index_block:
                flush()
            cur.extend(hd)
            if mr is None:
                mr = dict(tsid=tsid, count=0, min_ts=h["min_ts"], max_ts=h["max_ts"])
            mr["count"] += 1
            mr["min_ts"] = min(mr["min_ts"], h["min_ts"])
            mr["max_ts"] = max(mr["max_ts"], h["max_ts"])
            headers.append((tsid, h))
    flush()
    mi = compress(metaindex)
    return dict(metaindex_bin=mi, index_bin=bytes(index_bin), timestamps_bin=bytes(tsb), values_bin=bytes(vsb), headers=headers,
                index_blocks=n_index_blocks, metaindex_raw=bytes(metaindex))
