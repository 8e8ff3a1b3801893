"""lib/storage/block.go mirror: blocks of one series, their marshaled form, and the batched device decode.

  Block.marshal_data      == Block.MarshalData      block.go:192   (host write path: encoding.MarshalValues/Timestamps)
  BlockSet                == the (header, timestampsData, valuesData) triples of a query, packed into one payload arena;
                             identical timestamp payloads of consecutive blocks are stored once like
                             block_stream_writer.go:143-163
  Blocks / decode_blocks  == Block.UnmarshalData block.go:250 + AppendRowsWithTimeRangeFilter block.go:324, batched
"""
import ctypes as C

import numpy as np

from . import _lib, encoding
from ._lib import BlockDesc, check, lib

MAX_ROWS_PER_BLOCK = 8192  # block.go:15
INT64_MIN = -(1 << 63)
INT64_MAX = (1 << 63) - 1


class Block:
    """one block: <= 8192 rows of one series; values are decimal mantissas with a shared scale"""

    def __init__(self, timestamps, values, scale=0, precision_bits=64, series_idx=0):
        self.timestamps = np.ascontiguousarray(timestamps, dtype=np.int64)
        self.values = np.ascontiguousarray(values, dtype=np.int64)
        if self.timestamps.size != self.values.size or self.values.size == 0:
            raise ValueError("BUG: the number of values must match the number of timestamps and be > 0")  # block.go:225
        self.scale = int(scale)
        self.precision_bits = int(precision_bits)
        self.series_idx = int(series_idx)

    def marshal_data(self):
        """-> (header fields dict, timestampsData, valuesData)   block.go:192"""
        vdata, vmt, first_value = encoding.marshal_values(self.values, self.precision_bits)
        tdata, tmt, min_ts = encoding.marshal_timestamps(self.timestamps, self.precision_bits)
        hdr = dict(first_value=first_value, min_ts=min_ts, max_ts=int(self.timestamps[-1]), ts_size=tdata.size,
                   val_size=vdata.size, rows=self.values.size, series_idx=self.series_idx, scale=self.scale, ts_mt=tmt,
                   val_mt=vmt, precision_bits=self.precision_bits)
        return hdr, tdata, vdata


class BlockSet:
    """host-side descriptors + payload arena (what vmselect collects for one query, netstorage.go:1121)"""

    def __init__(self):
        self._hdrs = []
        self._chunks = []
        self._size = 0
        self._last_ts = None  # (bytes, offset) of the previous block's timestamps payload

    def add_marshaled(self, hdr, tdata, vdata):
        tb = tdata.tobytes()
        if self._last_ts is not None and self._last_ts[0] == tb:
            ts_off = self._last_ts[1]
        else:
            ts_off = self._size
            self._chunks.append(tdata)
            self._size += tdata.size
            self._last_ts = (tb, ts_off)
        val_off = self._size
        self._chunks.append(vdata)
        self._size += vdata.size
        h = dict(hdr)
        h["ts_off"], h["val_off"] = ts_off, val_off
        self._hdrs.append(h)

    def add(self, block):
        self.add_marshaled(*block.marshal_data())

    def finish(self):
        """-> (ctypes array of BlockDesc, payload np.uint8)"""
        descs = (BlockDesc * len(self._hdrs))()
        for d, h in zip(descs, self._hdrs):
            for k, v in h.items():
                setattr(d, k, v)
        payload = np.concatenate(self._chunks) if self._chunks else np.zeros(0, dtype=np.uint8)
        return descs, np.ascontiguousarray(payload, dtype=np.uint8)


def descs_from_arrays(**cols):
    """vectorised construction of a BlockDesc array from numpy columns (bench-sized inputs)"""
    n = len(cols["rows"])
    a = np.zeros(n, dtype=DESC_DTYPE)
    for k, v in cols.items():
        a[k] = v
    return a


DESC_DTYPE = np.dtype([("first_value", "<i8"), ("min_ts", "<i8"), ("max_ts", "<i8"), ("ts_off", "<u8"), ("val_off", "<u8"),
                       ("ts_size", "<u4"), ("val_size", "<u4"), ("rows", "<u4"), ("series_idx", "<u4"), ("scale", "<i2"),
                       ("ts_mt", "u1"), ("val_mt", "u1"), ("precision_bits", "u1"), ("_pad", "u1", (3,))])
METAINDEX_DTYPE = np.dtype([("tsid", "u1", (24,)), ("min_ts", "<i8"), ("max_ts", "<i8"), ("index_block_offset", "<u8"),
                            ("block_headers_count", "<u4"), ("index_block_size", "<u4")])
assert DESC_DTYPE.itemsize == 64 and METAINDEX_DTYPE.itemsize == 56


def marshal_block_header(desc, tsid=None):
    """blockHeader.Marshal block_header.go:104 -> 81 bytes.  desc: BlockDesc or one record of a DESC_DTYPE array"""
    if not isinstance(desc, BlockDesc):
        desc = BlockDesc.from_buffer_copy(np.asarray(desc).tobytes())
    out = (C.c_uint8 * 81)()
    t = None
    if tsid is not None:
        t = (C.c_uint8 * 24).from_buffer_copy(bytes(tsid))
    check(lib().vmb_block_header_marshal(out, C.byref(desc), t))
    return bytes(out)


def unmarshal_block_headers(data, count):
    """unmarshalBlockHeaders block_header.go:261 on an uncompressed index block -> (DESC_DTYPE array, tsids np.uint8[count, 24])"""
    d = np.ascontiguousarray(np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray)) else data, dtype=np.uint8)
    out = np.zeros(max(count, 1), dtype=DESC_DTYPE)
    tsids = np.zeros((max(count, 1), 24), dtype=np.uint8)
    src = d if d.size else np.zeros(1, dtype=np.uint8)
    check(lib().vmb_index_block_unmarshal(out.ctypes.data_as(C.POINTER(BlockDesc)), tsids.ctypes.data_as(_lib.u8p), count,
                                          src.ctypes.data_as(_lib.u8p), d.size))
    return out[:count], tsids[:count]


def unmarshal_metaindex_rows(data):
    """unmarshalMetaindexRows metaindex_row.go:129 on the decompressed metaindex.bin -> METAINDEX_DTYPE array"""
    d = np.ascontiguousarray(np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray)) else data, dtype=np.uint8)
    cap = d.size // 56 + 1
    out = np.zeros(cap, dtype=METAINDEX_DTYPE)
    n = C.c_size_t(0)
    src = d if d.size else np.zeros(1, dtype=np.uint8)
    check(lib().vmb_metaindex_rows_unmarshal(out.ctypes.data_as(C.POINTER(_lib.MetaindexRow)), cap, C.byref(n),
                                             src.ctypes.data_as(_lib.u8p), d.size))
    return out[:n.value]


def marshal_metaindex_row(row):
    """metaindexRow.Marshal metaindex_row.go:61 -> 56 bytes"""
    r = _lib.MetaindexRow.from_buffer_copy(np.asarray(row).tobytes())
    out = (C.c_uint8 * 56)()
    check(lib().vmb_metaindex_row_marshal(out, C.byref(r)))
    return bytes(out)


class Part:
    """The four data files of one part directory (lib/storage/part.go:34: metaindex.bin, index.bin, timestamps.bin, values.bin)
    as byte strings.  collect_blocks() == what partSearch (part_search.go:160 nextBHS -> :238 readIndexBlock) and
    netstorage hand to the query path, for every block of the part at once: metaindex.bin and all the index blocks are
    decompressed on the GPU in two batched calls, the headers become vmb_block_desc records whose offsets point into one
    payload arena [timestamps.bin | values.bin] -- the layout a storage node would DMA the two files into."""

    def __init__(self, metaindex_bin, index_bin, timestamps_bin, values_bin):
        as_u8 = lambda b: np.frombuffer(b, dtype=np.uint8) if isinstance(b, (bytes, bytearray)) else np.asarray(b, dtype=np.uint8)
        self.metaindex_bin, self.index_bin = as_u8(metaindex_bin), as_u8(index_bin)
        self.timestamps_bin, self.values_bin = as_u8(timestamps_bin), as_u8(values_bin)

    def metaindex_rows(self, ctx=None):
        return unmarshal_metaindex_rows(encoding.decompress_zstd_batch([self.metaindex_bin], ctx)[0])

    def collect_blocks(self, ctx=None, tsids=None, tr_min=INT64_MIN, tr_max=INT64_MAX):
        """-> (DESC_DTYPE array with dense series_idx, payload np.uint8, tsids of the series np.uint8[nseries, 24]).
        tsids (optional, iterable of 24-byte TSIDs) and [tr_min, tr_max] filter blocks like partSearch.Init (part_search.go:64)."""
        rows = self.metaindex_rows(ctx)
        frames = []
        for r in rows:
            o, sz = int(r["index_block_offset"]), int(r["index_block_size"])
            if o + sz > self.index_bin.size:
                raise _lib.VmbError(-1, "index block [%d, %d) outside index.bin (%d bytes)" % (o, o + sz, self.index_bin.size))
            frames.append(self.index_bin[o:o + sz])
        blocks = encoding.decompress_zstd_batch(frames, ctx)
        descs, ids = [], []
        for r, ib in zip(rows, blocks):
            d, t = unmarshal_block_headers(ib, int(r["block_headers_count"]))
            descs.append(d)
            ids.append(t)
        descs = np.concatenate(descs)
        ids = np.concatenate(ids)
        keep = (descs["max_ts"] >= tr_min) & (descs["min_ts"] <= tr_max)
        if tsids is not None:
            want = {bytes(t) for t in tsids}
            keep &= np.fromiter((ids[i].tobytes() in want for i in range(len(ids))), dtype=bool, count=len(ids))
        descs, ids = descs[keep], ids[keep]
        if (descs["ts_off"] + descs["ts_size"] > self.timestamps_bin.size).any() or \
                (descs["val_off"] + descs["val_size"] > self.values_bin.size).any():
            raise _lib.VmbError(-1, "block payload outside timestamps.bin / values.bin")
        descs["val_off"] += np.uint64(self.timestamps_bin.size)
        new_series = np.ones(len(descs), dtype=bool)
        if len(descs) > 1:
            new_series[1:] = (ids[1:] != ids[:-1]).any(axis=1)
        descs["series_idx"] = (np.cumsum(new_series) - 1).astype(np.uint32)
        payload = np.concatenate([self.timestamps_bin, self.values_bin])
        return descs, payload, ids[new_series]


def _take_part(h):
    """the files of a vmb_merged_part handle as a Part (copied out), then the handle freed"""
    try:
        out = _lib.PartFiles()
        check(lib().vmb_merged_part_files(h, C.byref(out)))
        copy = lambda ptr, n: np.ctypeslib.as_array(ptr, (n,)).copy() if n else np.zeros(0, dtype=np.uint8)
        return Part(copy(out.metaindex, out.metaindex_len), copy(out.index, out.index_len), copy(out.timestamps, out.timestamps_len),
                    copy(out.values, out.values_len))
    finally:
        lib().vmb_merged_part_free(h)


def parts_from_rows(sets, ctx=None):
    """rawRowsMarshaler.marshalToInmemoryPart (lib/storage/raw_row.go:81) for every row set of a flush in one call on the GPU.
    sets: [(tsids uint8 [n, 24] or [n * 24], timestamps int64 [n], values float64 [n], precision_bits uint8 [n])] ->
    [(Part, stats dict as merge_parts gives it)], one per set.  Rows with equal (TSID, Timestamp) keep their input order.  The
    context's dedup interval applies (Context.set_dedup_interval)."""
    ctx = ctx or _lib.default_context()
    rows = (_lib.RawRows * max(len(sets), 1))()
    keep = []
    for r, (tsids, ts, vals, pbs) in zip(rows, sets):
        t = np.ascontiguousarray(tsids, dtype=np.uint8).reshape(-1)
        a = np.ascontiguousarray(ts, dtype=np.int64)
        v = np.ascontiguousarray(vals, dtype=np.float64)
        p = np.ascontiguousarray(pbs, dtype=np.uint8)
        if not (t.size == 24 * a.size and a.size == v.size == p.size):
            raise ValueError("a row set needs 24 TSID bytes, a timestamp, a value and precisionBits per row")
        keep += [t, a, v, p]
        r.tsids, r.timestamps = t.ctypes.data_as(_lib.u8p), a.ctypes.data_as(_lib.i64p)
        r.values, r.precision_bits, r.n = v.ctypes.data_as(_lib.f64p), p.ctypes.data_as(_lib.u8p), a.size
    hs = (C.c_void_p * max(len(sets), 1))()
    st = (_lib.MergeStats * max(len(sets), 1))()
    check(lib().vmb_parts_from_rows(ctx.h, rows, len(sets), hs, st))
    out = []
    try:
        for i in range(len(sets)):
            out.append((_take_part(hs[i]), {k: int(getattr(st[i], k)) for k, _ in _lib.MergeStats._fields_}))
            hs[i] = None
    finally:
        for h in hs[:len(sets)]:
            if h:
                lib().vmb_merged_part_free(h)
    return out


def merge_parts(parts, retention_deadline=INT64_MIN, deleted_metric_ids=(), ctx=None):
    """mergeBlockStreams (lib/storage/merge.go:19) of `parts` (a list of Part, in that order) on the GPU -> (Part, stats dict with
    rows_count, blocks_count, min_ts, max_ts of the partHeader and the rows_merged / rows_deleted counters).  The context's dedup
    interval applies (Context.set_dedup_interval).  deleted_metric_ids: any iterable of MetricIDs (sorted here)."""
    ctx = ctx or _lib.default_context()
    files = (_lib.PartFiles * max(len(parts), 1))()
    keep = []
    for f, p in zip(files, parts):
        for name in ("metaindex", "index", "timestamps", "values"):
            a = np.ascontiguousarray(getattr(p, name + "_bin"), dtype=np.uint8)
            keep.append(a)
            setattr(f, name, a.ctypes.data_as(_lib.u8p))
            setattr(f, name + "_len", a.size)
    dm = np.unique(np.asarray(list(deleted_metric_ids), dtype=np.uint64))
    h = C.c_void_p()
    st = _lib.MergeStats()
    check(lib().vmb_merge_parts(ctx.h, files, len(parts), int(retention_deadline), dm.ctypes.data_as(_lib.u64p), dm.size, C.byref(h),
                                C.byref(st)))
    try:
        out = _lib.PartFiles()
        check(lib().vmb_merged_part_files(h, C.byref(out)))
        copy = lambda ptr, n: np.ctypeslib.as_array(ptr, (n,)).copy() if n else np.zeros(0, dtype=np.uint8)
        part = Part(copy(out.metaindex, out.metaindex_len), copy(out.index, out.index_len), copy(out.timestamps, out.timestamps_len),
                    copy(out.values, out.values_len))
    finally:
        lib().vmb_merged_part_free(h)
    stats = {k: int(getattr(st, k)) for k, _ in _lib.MergeStats._fields_}
    return part, stats


class Blocks:
    """compressed blocks resident in HBM (vmb_blocks)"""

    def __init__(self, descs, payload, ctx=None):
        self.ctx = ctx or _lib.default_context()
        payload = np.ascontiguousarray(payload, dtype=np.uint8)
        if isinstance(descs, np.ndarray):
            dptr = descs.ctypes.data_as(C.POINTER(BlockDesc))
            n = descs.shape[0]
        else:
            dptr = descs
            n = len(descs)
        h = C.c_void_p()
        check(lib().vmb_blocks_upload(self.ctx.h, dptr, n, payload.ctypes.data_as(_lib.u8p), payload.size, C.byref(h)))
        self.h = h
        self.count = n

    @classmethod
    def from_block_refs(cls, headers, timestamps_bin, values_bin, ctx=None):
        """the BlockRefs of a query (tmp_blocks_file.go:110: one marshaled 81-byte blockHeader per block, series order) + the part's
        timestamps.bin / values.bin -> device-resident blocks (vmb_blocks_upload_part == BlockRef.MustReadBlock search.go:73 for all)"""
        self = cls.__new__(cls)
        self.ctx = ctx or _lib.default_context()
        hb = np.frombuffer(bytes(headers), dtype=np.uint8) if not isinstance(headers, np.ndarray) else np.ascontiguousarray(headers, dtype=np.uint8)
        if hb.size % 81:
            raise ValueError("headers: %d bytes is not a whole number of 81-byte blockHeaders" % hb.size)
        tb = np.frombuffer(timestamps_bin, dtype=np.uint8) if not isinstance(timestamps_bin, np.ndarray) else timestamps_bin
        vb = np.frombuffer(values_bin, dtype=np.uint8) if not isinstance(values_bin, np.ndarray) else values_bin
        h = C.c_void_p()
        self.h = None
        check(lib().vmb_blocks_upload_part(self.ctx.h, hb.ctypes.data_as(_lib.u8p), hb.size // 81, tb.ctypes.data_as(_lib.u8p), tb.size,
                                           vb.ctypes.data_as(_lib.u8p), vb.size, C.byref(h)))
        self.h = h
        self.count = hb.size // 81
        return self

    @property
    def rows(self):
        return int(lib().vmb_blocks_rows(self.h))

    @property
    def compressed_bytes(self):
        return int(lib().vmb_blocks_compressed_bytes(self.h))

    def close(self):
        if self.h:
            lib().vmb_blocks_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Series:
    """decoded columns resident in HBM (vmb_series)"""

    def __init__(self, h, ctx):
        self.h = h
        self.ctx = ctx

    @classmethod
    def from_host(cls, timestamps_list, values_list, ctx=None):
        """series batch from already decoded columns (the arguments of rollupConfig.Do)"""
        ctx = ctx or _lib.default_context()
        offs = np.zeros(len(values_list) + 1, dtype=np.uint64)
        for i, v in enumerate(values_list):
            offs[i + 1] = offs[i] + len(v)
        ts = np.ascontiguousarray(np.concatenate([np.asarray(t, dtype=np.int64) for t in timestamps_list])
                                  if timestamps_list else np.zeros(0), dtype=np.int64)
        vals = np.ascontiguousarray(np.concatenate([np.asarray(v, dtype=np.float64) for v in values_list])
                                    if values_list else np.zeros(0), dtype=np.float64)
        h = C.c_void_p()
        check(lib().vmb_series_from_host(ctx.h, ts.ctypes.data_as(_lib.i64p), vals.ctypes.data_as(_lib.f64p),
                                         offs.ctypes.data_as(_lib.u64p), len(values_list), C.byref(h)))
        return cls(h, ctx)

    @classmethod
    def from_matrix(cls, dev_ptr, nseries, points, start, step, ctx=None):
        """series batch from a DEVICE matrix [nseries x points] on the grid start + i * step, NaN points removed per row
        (removeNanValues eval.go:1027): the feed of a subquery's outer rollup"""
        ctx = ctx or _lib.default_context()
        h = C.c_void_p()
        check(lib().vmb_series_from_matrix(ctx.h, C.c_void_p(int(dev_ptr)), int(nseries), int(points), int(start), int(step), C.byref(h)))
        return cls(h, ctx)

    @property
    def count(self):
        return int(lib().vmb_series_count(self.h))

    @property
    def rows(self):
        return int(lib().vmb_series_rows(self.h))

    def layout(self):
        n = self.count
        starts = np.zeros(n, dtype=np.uint64)
        counts = np.zeros(n, dtype=np.uint32)
        check(lib().vmb_series_layout(self.ctx.h, self.h, starts.ctypes.data_as(_lib.u64p), counts.ctypes.data_as(_lib.u32p)))
        return starts, counts

    def download(self, values_dtype=np.float64):
        r = self.rows
        ts = np.empty(r, dtype=np.int64)
        vals = np.empty(r, dtype=values_dtype)
        check(lib().vmb_series_download(self.ctx.h, self.h, ts.ctypes.data_as(_lib.i64p),
                                        C.cast(vals.ctypes.data, _lib.f64p)))
        return ts, vals

    def to_lists(self, values_dtype=np.float64):
        """-> [(timestamps, values)] per series, after trimming"""
        ts, vals = self.download(values_dtype)
        starts, counts = self.layout()
        return [(ts[s:s + c], vals[s:s + c]) for s, c in zip(starts.tolist(), counts.tolist())]

    def close(self):
        if self.h:
            lib().vmb_series_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def decode_blocks(blocks, tr_min=INT64_MIN, tr_max=INT64_MAX, values_as_int64=False, raise_on_block_error=True):
    """batched Block.UnmarshalData + AppendRowsWithTimeRangeFilter -> (Series, per-block status np.int32)"""
    status = np.zeros(max(blocks.count, 1), dtype=np.int32)
    h = C.c_void_p()
    rc = lib().vmb_decode_blocks(blocks.ctx.h, blocks.h, tr_min, tr_max, 1 if values_as_int64 else 0,
                                 status.ctypes.data_as(_lib.i32p), C.byref(h))
    status = status[:blocks.count]
    if rc == -53 and not raise_on_block_error:
        return Series(h, blocks.ctx), status
    if rc != 0 and h:
        lib().vmb_series_free(h)
    check(rc)
    return Series(h, blocks.ctx), status
