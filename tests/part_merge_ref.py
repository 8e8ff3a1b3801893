"""Restatement of the reference's part merge in plain Python (lib/storage), independent of the product's merge code:

  blockStreamMerger      block_stream_merger.go:30-176, with Go's container/heap (src/container/heap/heap.go) ported literally
  mergeBlockStreams      merge.go:19-156 (the pending-block chain), mergeBlocks :159, skipSamplesOutsideRetention :199,
                         unmarshalAndCalibrateScale :215, Block.tooBig block.go:142, fixupTimestamps block.go:84
  dedup                  deduplicateSamplesDuringMerge dedup.go:94 (needsDedup :158)
  blockStreamWriter      WriteExternalBlock block_stream_writer.go:138, flushIndexData :182, MustClose :116,
                         metaindexRow.RegisterBlockHeader metaindex_row.go:46, partHeader.Reset part_header.go:42

Input parts are lists of (tsid bytes, header dict, ts int64[], values int64[], tdata bytes, vdata bytes) in part order: the blocks
as a blockStreamReader yields them, already unmarshaled for the cases the chain needs.  `marshal` writes a column and `frame` a
zstd frame; the defaults are the library's host writer, with the merge path's rule for 128 KiB < n <= 262143 byte streams."""
import struct

import numpy as np

import oracle_lib as O
import partgen

MAX_ROWS_PER_BLOCK = 8192  # block.go:15
MAX_BLOCK_SIZE = 8 * MAX_ROWS_PER_BLOCK  # block.go:18
STALE_NAN = (1 << 63) - 2  # decimal.go:406 vStaleNaN
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1


def metric_id(tsid):
    return struct.unpack(">Q", tsid[16:24])[0]


# ---- container/heap
def heap_down(h, less, i0, n):
    i = i0
    while True:
        j1 = 2 * i + 1
        if j1 >= n or j1 < 0:
            break
        j = j1
        j2 = j1 + 1
        if j2 < n and less(h, j2, j1):
            j = j2
        if not less(h, j, i):
            break
        h[i], h[j] = h[j], h[i]
        i = j
    return i > i0


def heap_up(h, less, j):
    while True:
        i = (j - 1) // 2
        if i == j or j == 0 or not less(h, j, i):
            break
        h[i], h[j] = h[j], h[i]
        j = i


def heap_init(h, less):
    n = len(h)
    for i in range(n // 2 - 1, -1, -1):
        heap_down(h, less, i, n)


def heap_fix(h, less, i):
    if not heap_down(h, less, i, len(h)):
        heap_up(h, less, i)


def heap_pop(h, less):
    n = len(h) - 1
    h[0], h[n] = h[n], h[0]
    heap_down(h, less, 0, n)
    return h.pop()


def merged_order(parts):
    """blockStreamMerger: [(part index, block index)] in the order NextBlock yields them"""
    pos = [0] * len(parts)

    def less(h, i, j):  # blockStreamReaderHeap.Less block_stream_merger.go:130
        a, b = parts[h[i]][pos[h[i]]], parts[h[j]][pos[h[j]]]
        if metric_id(a[0]) == metric_id(b[0]):
            return a[1]["min_ts"] < b[1]["min_ts"]
        return a[0] < b[0]

    h = [i for i, p in enumerate(parts) if p]
    out = []
    if not h:
        return out
    heap_init(h, less)
    while True:
        p = h[0]
        out.append((p, pos[p]))
        pos[p] += 1
        if pos[p] < len(parts[p]):
            heap_fix(h, less, 0)
        else:
            heap_pop(h, less)
            if not h:
                return out


# ---- decimal.CalibrateScale decimal.go:13
def _max_up_exponent(v):  # decimal.go:268: the largest k <= 18 with |v| <= MaxInt64 / 10^k
    if v == 0 or _special(v):
        return 1024
    v = abs(v)
    k, lim = 0, INT64_MAX
    for t in range(1, 19):
        lim //= 10
        if v <= lim:
            k = t
        else:
            break
    return k


def _special(v):
    return v > INT64_MAX - 2 or v < INT64_MIN + 1


def _wrap(x):
    return ((x + (1 << 63)) % (1 << 64)) - (1 << 63)


def calibrate_scale(a, ae, b, be):
    if ae == be:
        return ae
    if len(a) == 0:
        return be
    if len(b) == 0:
        return ae
    if ae < be:
        a, b, ae, be = b, a, be, ae
    up, down = ae - be, 0
    for v in a:
        d = up - _max_up_exponent(int(v))
        if d > down:
            down = d
    up -= down
    if up > 0:
        m = 10 ** up if up < 19 else 1
        for i in range(len(a)):
            if not _special(int(a[i])):
                a[i] = _wrap(int(a[i]) * m)
    if down > 0:
        for i in range(len(b)):
            if not _special(int(b[i])):
                x = int(b[i])
                b[i] = 0 if down > 18 else (x // 10 ** down if x >= 0 else -((-x) // 10 ** down))
    return be + down


# ---- dedup.go:94
def needs_dedup(ts, interval):
    if len(ts) < 2 or interval <= 0:
        return False
    nxt = _go_mod_sub(ts[0] + interval - 1, interval)
    for t in ts[1:]:
        if t <= nxt:
            return True
        nxt += interval
        if nxt < t:
            nxt = _go_mod_sub(t + interval - 1, interval)
    return False


def _go_mod_sub(x, m):  # x -= x % m with Go's truncated remainder
    r = abs(x) % m
    return x - (r if x >= 0 else -r)


def deduplicate_samples_during_merge(ts, vals, interval):
    ts, vals = [int(t) for t in ts], [int(v) for v in vals]
    if not needs_dedup(ts, interval):
        return ts, vals

    def pick(j):
        tp, vp = ts[j], vals[j]
        while j > 0 and ts[j - 1] == tp:
            j -= 1
            if vals[j] == STALE_NAN:
                continue
            if vp == STALE_NAN:
                vp = vals[j]
                continue
            if vals[j] > vp:
                vp = vals[j]
        return tp, vp

    nxt = _go_mod_sub(ts[0] + interval - 1, interval)
    ot, ov = [], []
    for i in range(1, len(ts)):
        t = ts[i]
        if t <= nxt:
            continue
        a, b = pick(i - 1)
        ot.append(a)
        ov.append(b)
        nxt += interval
        if nxt < t:
            nxt = _go_mod_sub(t + interval - 1, interval)
    a, b = pick(len(ts) - 1)
    ot.append(a)
    ov.append(b)
    return ot, ov


# ---- the column writer
def host_marshal(vals, pb):
    """encoding.MarshalValues with the library's host writer, a stream of 128 KiB < n <= 262143 bytes left uncompressed"""
    from victoriametrics_b200 import encoding
    data, mt, first = encoding.marshal_values(np.asarray(vals, dtype=np.int64), pb)
    if mt in (1, 4):
        rc, stream = O.zstd_decompress(data)
        assert rc == 0
        if 128 * 1024 < stream.size <= 262143:
            return stream.tobytes(), 5 if mt == 1 else 6, first
    return data.tobytes(), mt, first


def host_frame(raw):
    from victoriametrics_b200 import encoding
    return encoding.zstd_compress(np.frombuffer(raw, dtype=np.uint8)).tobytes()


class _B:
    """storage.Block as the chain sees it: raw (header + payloads) or rows"""

    def __init__(self, tsid, h, ts=None, vals=None, tdata=b"", vdata=b"", raw=True):
        self.tsid, self.h = tsid, dict(h)
        self.ts, self.vals, self.tdata, self.vdata, self.raw = ts, vals, tdata, vdata, raw
        self.next = 0

    def too_big(self):  # block.go:142
        rows_count = self.h["rows"] if self.raw else 0
        n = 0 if self.raw else len(self.vals) - self.next
        vd = len(self.vdata) if self.raw else 0
        return rows_count >= MAX_ROWS_PER_BLOCK or n >= MAX_ROWS_PER_BLOCK or vd >= MAX_BLOCK_SIZE


def merge_parts(parts, retention_deadline=INT64_MIN, deleted=(), dedup_interval=0, marshal=host_marshal, frame=host_frame):
    """parts: [[(tsid, header dict, ts, vals, tdata, vdata)]] -> dict(metaindex_bin, index_bin, timestamps_bin, values_bin,
    metaindex_raw, stats, blocks = [(tsid, header, ts, vals)] of every block written, in order).  metaindex_bin is None where the merge path writes Raw blocks (an empty metaindex or 128 KiB < n <=
    262143)."""
    deleted = set(int(x) for x in deleted)
    st = dict(rows_count=0, blocks_count=0, min_ts=INT64_MAX, max_ts=INT64_MIN, rows_merged=0, rows_deleted=0)
    W = dict(blocks=[], ts=bytearray(), vals=bytearray(), index=bytearray(), meta=bytearray(), cur=bytearray(), mr=None, prev=b"", prev_off=0)

    def flush_index():
        if not W["cur"]:
            return
        comp = frame(bytes(W["cur"]))
        mr = W["mr"]
        W["meta"] += partgen.pack_metaindex_row(mr["tsid"], mr["count"], mr["min_ts"], mr["max_ts"], len(W["index"]), len(comp))
        W["index"] += comp
        W["cur"] = bytearray()
        W["mr"] = None

    def write(b):  # WriteExternalBlock
        st["rows_merged"] += b.h["rows"] if b.raw else len(b.vals) - b.next
        if dedup_interval > 0:
            b.raw = False
            ts, vs = b.ts[b.next:], b.vals[b.next:]
            if len(ts) >= 2:
                ts, vs = deduplicate_samples_during_merge(ts, vs, dedup_interval)
            b.ts, b.vals, b.next = list(ts), list(vs), 0
        h = dict(b.h)
        if b.raw:
            td, vd = b.tdata, b.vdata
            W["blocks"].append((b.tsid, h, [int(x) for x in b.ts], [int(x) for x in b.vals]))
        else:
            ts, vs = [int(x) for x in b.ts[b.next:]], [int(x) for x in b.vals[b.next:]]
            vd, h["val_mt"], h["first_value"] = marshal(vs, h["precision_bits"])
            td, h["ts_mt"], h["min_ts"] = marshal(ts, h["precision_bits"])
            h["max_ts"] = ts[-1]
            h["rows"] = len(vs)
            W["blocks"].append((b.tsid, h, ts, vs))
        h["ts_size"], h["val_size"] = len(td), len(vd)
        share = len(W["prev"]) > 0 and td == W["prev"]
        h["ts_off"] = W["prev_off"] if share else len(W["ts"])
        h["val_off"] = len(W["vals"])
        hd = partgen.pack_header(b.tsid, h)
        if len(W["cur"]) + len(hd) > MAX_BLOCK_SIZE:
            flush_index()
        W["cur"] += hd
        if W["mr"] is None:
            W["mr"] = dict(tsid=b.tsid, count=0, min_ts=h["min_ts"], max_ts=h["max_ts"])
        mr = W["mr"]
        mr["count"] += 1
        mr["min_ts"], mr["max_ts"] = min(mr["min_ts"], h["min_ts"]), max(mr["max_ts"], h["max_ts"])
        if not share:
            W["prev"], W["prev_off"] = td, len(W["ts"])
            W["ts"] += td
        W["vals"] += vd
        st["blocks_count"] += 1
        st["rows_count"] += h["rows"]
        st["min_ts"], st["max_ts"] = min(st["min_ts"], h["min_ts"]), max(st["max_ts"], h["max_ts"])

    def unmarshal(b):
        if b.raw:
            b.raw = False
            b.ts, b.vals, b.next = [int(x) for x in b.ts], [int(x) for x in b.vals], 0

    def fixup(b):
        b.h["min_ts"], b.h["max_ts"] = b.ts[b.next], b.ts[-1]

    pending = None
    for p, i in merged_order(parts):
        tsid, h, ts, vals, tdata, vdata = parts[p][i]
        b = _B(tsid, h, list(ts), list(vals), tdata, vdata)
        if metric_id(tsid) in deleted or h["max_ts"] < retention_deadline:
            st["rows_deleted"] += h["rows"]
            continue
        if pending is None:
            pending = b
            continue
        if metric_id(pending.tsid) != metric_id(tsid):
            write(pending)
            pending = b
            continue
        if pending.too_big() and pending.h["max_ts"] <= h["min_ts"]:
            write(pending)
            pending = b
            continue
        unmarshal(pending)
        unmarshal(b)
        sc = calibrate_scale(pending.vals, pending.h["scale"], b.vals, b.h["scale"])
        pending.h["scale"] = b.h["scale"] = sc
        tmp = _B(tsid, dict(scale=sc, precision_bits=min(pending.h["precision_bits"], h["precision_bits"]), rows=0), [], [], raw=False)
        _merge_blocks(tmp, pending, b, retention_deadline, st)
        if len(tmp.ts) <= MAX_ROWS_PER_BLOCK:
            if tmp.ts:
                fixup(tmp)
                pending = tmp
            else:
                pending = None
            continue
        rest = _B(tsid, dict(tmp.h), tmp.ts[MAX_ROWS_PER_BLOCK:], tmp.vals[MAX_ROWS_PER_BLOCK:], raw=False)
        fixup(rest)
        tmp.ts, tmp.vals = tmp.ts[:MAX_ROWS_PER_BLOCK], tmp.vals[:MAX_ROWS_PER_BLOCK]
        fixup(tmp)
        write(tmp)
        pending = rest
    if pending is not None:
        write(pending)
    flush_index()
    meta = bytes(W["meta"])
    mi = None if len(meta) == 0 or 128 * 1024 < len(meta) <= 262143 else frame(meta)
    return dict(metaindex_bin=mi, metaindex_raw=meta, index_bin=bytes(W["index"]), timestamps_bin=bytes(W["ts"]),
                values_bin=bytes(W["vals"]), stats=st, blocks=W["blocks"])


def _merge_blocks(ob, ib1, ib2, deadline, st):  # merge.go:159
    for b in (ib1, ib2):  # skipSamplesOutsideRetention
        if b.h["min_ts"] >= deadline:
            continue
        n0 = b.next
        while b.next < len(b.ts) and b.ts[b.next] < deadline:
            b.next += 1
        st["rows_deleted"] += b.next - n0

    def app(b):
        ob.ts += b.ts[b.next:]
        ob.vals += b.vals[b.next:]

    if ib1.h["max_ts"] < ib2.h["min_ts"]:
        app(ib1), app(ib2)
        return
    if ib2.h["max_ts"] < ib1.h["min_ts"]:
        app(ib2), app(ib1)
        return
    if ib1.next >= len(ib1.ts):
        app(ib2)
        return
    if ib2.next >= len(ib2.ts):
        app(ib1)
        return
    while True:
        i = ib1.next
        ts2 = ib2.ts[ib2.next]
        while i < len(ib1.ts) and ib1.ts[i] <= ts2:
            i += 1
        ob.ts += ib1.ts[ib1.next:i]
        ob.vals += ib1.vals[ib1.next:i]
        ib1.next = i
        if ib1.next >= len(ib1.ts):
            app(ib2)
            return
        ib1, ib2 = ib2, ib1


# ---- test inputs
def part_from_series(series, pure_go=False):
    """series: [(tsid, [OBlock])] sorted by TSID -> (partgen part dict, restatement input list)"""
    part = partgen.write_part(series, pure_go=pure_go)
    blocks = []
    k = 0
    for tsid, bl in series:
        for b in bl:
            _, h = part["headers"][k]
            k += 1
            rc, ts, _, iv = b.oracle_unmarshal()
            assert rc == 0
            blocks.append((tsid, h, ts, iv, b.tdata.tobytes(), b.vdata.tobytes()))
    return part, blocks


def split_rows(ts, vals, max_rows=MAX_ROWS_PER_BLOCK):
    """inmemoryPart.InitFromRows (inmemory_part.go) cuts one series' sorted rows into blocks of at most maxRowsPerBlock"""
    return [(ts[i:i + max_rows], vals[i:i + max_rows]) for i in range(0, len(ts), max_rows)]


def oracle_marshal(vals, pb):
    """encoding.MarshalValues as the reference writes it (the oracle's marshalInt64Array + the reference's libzstd)"""
    data, mt, first = O.marshal_int64_array(np.asarray(vals, dtype=np.int64), pb)
    return data.tobytes(), mt, first


def oracle_frame(raw):
    return O.zstd_ref_compress(np.frombuffer(raw, dtype=np.uint8), 1).tobytes()


def _unzz(u):
    return (u >> 1) ^ -(u & 1)


def unpack_header(b):
    """blockHeader.Unmarshal block_header.go:122 -> (tsid, header dict)"""
    mn, mx, fv, to, vo, ts_, vs_, rows, sc, tmt, vmt, pb = struct.unpack(">QQQQQIIIHBBB", b[24:81])
    return b[:24], dict(min_ts=_unzz(mn), max_ts=_unzz(mx), first_value=_unzz(fv), ts_off=to, val_off=vo, ts_size=ts_, val_size=vs_,
                        rows=rows, scale=(sc >> 1) ^ -(sc & 1), ts_mt=tmt, val_mt=vmt, precision_bits=pb)


def read_part(metaindex_bin, index_bin, timestamps_bin, values_bin, meta_cap):
    """a part decoded by the reference side alone (libzstd for every frame, the oracle's column decoder):
    [(tsid, header dict, ts, vals)] in file order"""
    u8 = lambda b: np.frombuffer(bytes(b), dtype=np.uint8) if isinstance(b, (bytes, bytearray)) else np.asarray(b, dtype=np.uint8)
    metaindex_bin, index_bin, timestamps_bin, values_bin = map(u8, (metaindex_bin, index_bin, timestamps_bin, values_bin))
    mi = O.zstd_ref_decompress(metaindex_bin, meta_cap).tobytes()
    out = []
    for k in range(len(mi) // 56):
        cnt, _, _, off, size = struct.unpack(">IQQQI", mi[k * 56 + 24:k * 56 + 56])
        ib = O.zstd_ref_decompress(index_bin[off:off + size], cnt * 81).tobytes()
        for j in range(cnt):
            t, h = unpack_header(ib[j * 81:(j + 1) * 81])
            cols = []
            for data, mt, first, o, n in ((timestamps_bin, h["ts_mt"], h["min_ts"], h["ts_off"], h["ts_size"]),
                                          (values_bin, h["val_mt"], h["first_value"], h["val_off"], h["val_size"])):
                src = data[o:o + n]
                if mt in (1, 4):  # every zstd column through libzstd
                    src = O.zstd_ref_decompress(src, h["rows"] * 10 + 16)
                    mt = 5 if mt == 1 else 6
                rc, col = O.unmarshal_int64_array(src, mt, first, h["rows"])
                assert rc == 0, rc
                cols.append([int(x) for x in col])
            if h["precision_bits"] < 64:  # EnsureNonDecreasingSequence encoding.go:258
                ts, run = cols[0], h["min_ts"]
                for i in range(len(ts)):
                    run = max(run, ts[i]) if i else h["min_ts"]
                    ts[i] = min(run, h["max_ts"])
                ts[-1] = h["max_ts"]
            out.append((t, h, cols[0], cols[1]))
    return out
