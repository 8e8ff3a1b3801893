"""ctypes binding of the CPU oracle (oracle/libvmoracle.so).  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module; nothing under victoriametrics_b200/ does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_ORACLE_DIR = os.path.join(_ROOT, "oracle")
_SO = os.path.join(_ORACLE_DIR, "libvmoracle.so")

u8p = C.POINTER(C.c_uint8)
i64p = C.POINTER(C.c_int64)
f64p = C.POINTER(C.c_double)
u64p = C.POINTER(C.c_uint64)


def build():
    subprocess.check_call(["make", "-s", "-C", _ORACLE_DIR])


class BlockHeader(C.Structure):
    _fields_ = [("tsid", C.c_uint8 * 24), ("min_ts", C.c_int64), ("max_ts", C.c_int64), ("first_value", C.c_int64),
                ("ts_off", C.c_uint64), ("val_off", C.c_uint64), ("ts_size", C.c_uint32), ("val_size", C.c_uint32),
                ("rows", C.c_uint32), ("scale", C.c_int16), ("ts_mt", C.c_uint8), ("val_mt", C.c_uint8),
                ("precision_bits", C.c_uint8)]


class RollupCfg(C.Structure):
    _fields_ = [("func_id", C.c_int), ("start", C.c_int64), ("end", C.c_int64), ("step", C.c_int64),
                ("window", C.c_int64), ("lookback_delta", C.c_int64), ("min_staleness_ms", C.c_int64),
                ("may_adjust_window", C.c_int), ("is_default_rollup", C.c_int), ("samples_scanned_per_call", C.c_int),
                ("args", f64p), ("args2", f64p)]


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_SO):
        build()
    L = C.CDLL(_SO)
    sz = C.c_size_t
    sig = {
        "vmo_marshal_varint64s": (C.c_int64, [u8p, sz, i64p, sz]),
        "vmo_unmarshal_varint64s": (C.c_int, [i64p, sz, u8p, sz, C.POINTER(sz)]),
        "vmo_nearest_delta": (None, [C.c_int64, C.c_int64, C.c_uint8, C.c_uint8, i64p, u8p]),
        "vmo_get_trailing_zeros": (C.c_uint8, [C.c_int64, C.c_uint8]),
        "vmo_marshal_nearest_delta": (C.c_int64, [u8p, sz, i64p, sz, C.c_uint8, i64p]),
        "vmo_marshal_nearest_delta2": (C.c_int64, [u8p, sz, i64p, sz, C.c_uint8, i64p]),
        "vmo_unmarshal_nearest_delta": (C.c_int, [i64p, u8p, sz, C.c_int64, sz]),
        "vmo_unmarshal_nearest_delta2": (C.c_int, [i64p, u8p, sz, C.c_int64, sz]),
        "vmo_is_const": (C.c_int, [i64p, sz]),
        "vmo_is_delta_const": (C.c_int, [i64p, sz]),
        "vmo_is_gauge": (C.c_int, [i64p, sz]),
        "vmo_get_compress_level": (C.c_int, [sz]),
        "vmo_ensure_non_decreasing": (None, [i64p, sz, C.c_int64, C.c_int64]),
        "vmo_check_timestamps_bounds": (C.c_int, [i64p, sz, C.c_int64, C.c_int64]),
        "vmo_marshal_int64_array": (C.c_int64, [u8p, sz, i64p, sz, C.c_uint8, C.POINTER(C.c_int), i64p]),
        "vmo_unmarshal_int64_array": (C.c_int, [i64p, u8p, sz, C.c_int, C.c_int64, sz]),
        "vmo_zstd_decompress": (C.c_int64, [u8p, sz, u8p, sz]),
        "vmo_zstd_content_size": (C.c_int64, [u8p, sz]),
        "vmo_zstd_ref_available": (C.c_int, []),
        "vmo_zstd_ref_factory_available": (C.c_int, []),
        "vmo_zstd_ref_compress": (C.c_int64, [u8p, sz, u8p, sz, C.c_int]),
        "vmo_zstd_ref_decompress": (C.c_int64, [u8p, sz, u8p, sz]),
        "vmo_zstd_ref_compress_checksum": (C.c_int64, [u8p, sz, u8p, sz, C.c_int]),
        "vmo_zstd_ref_compress_params": (C.c_int64, [u8p, sz, u8p, sz, C.POINTER(C.c_int), C.c_int]),
        "vmo_zstd_ref_compress_sequences": (C.c_int64, [u8p, sz, u8p, sz, C.POINTER(C.c_uint32), sz,
                                                        C.POINTER(C.c_int), C.c_int]),
        "vmo_zstd_content_bound": (C.c_int64, [u8p, sz]),
        "vmo_pow10": (C.c_double, [C.c_int]),
        "vmo_decimal_to_float": (None, [f64p, i64p, sz, C.c_int16]),
        "vmo_float_to_decimal": (C.c_int16, [i64p, f64p, sz]),
        "vmo_calibrate_scale": (C.c_int16, [i64p, sz, C.c_int16, i64p, sz, C.c_int16]),
        "vmo_from_float": (None, [C.c_double, i64p, C.POINTER(C.c_int16)]),
        "vmo_positive_float_to_decimal": (None, [C.c_double, i64p, C.POINTER(C.c_int16)]),
        "vmo_to_float": (C.c_double, [C.c_int64, C.c_int16]),
        "vmo_block_header_marshal": (None, [u8p, C.POINTER(BlockHeader)]),
        "vmo_block_header_unmarshal": (None, [C.POINTER(BlockHeader), u8p]),
        "vmo_block_unmarshal": (C.c_int64, [i64p, f64p, i64p, C.POINTER(BlockHeader), u8p, u8p, C.c_int64, C.c_int64]),
        "vmo_rollup_do": (C.c_uint64, [C.POINTER(RollupCfg), f64p, f64p, i64p, sz]),
        "vmo_rollup_func_call": (C.c_double, [C.c_int, C.c_double, C.c_int64, f64p, i64p, sz, C.c_double, C.c_double,
                                              C.c_int64, sz, C.c_int64, f64p, f64p]),
        "vmo_rollup_points": (C.c_int64, [C.c_int64, C.c_int64, C.c_int64]),
        "vmo_remove_counter_resets": (None, [f64p, i64p, sz, C.c_int64]),
        "vmo_merge_sort_blocks": (sz, [i64p, f64p, u64p, sz, C.c_int64, i64p, f64p]),
        "vmo_deduplicate_samples": (sz, [i64p, f64p, sz, C.c_int64]),
        "vmo_needs_dedup": (C.c_int, [i64p, sz, C.c_int64]),
        "vmo_delta_values": (None, [f64p, sz]),
        "vmo_deriv_values": (None, [f64p, i64p, sz]),
        "vmo_drop_stale_nans": (sz, [f64p, i64p, sz]),
        "vmo_get_scrape_interval": (C.c_int64, [i64p, sz, C.c_int64]),
        "vmo_get_max_prev_interval": (C.c_int64, [C.c_int64]),
        "vmo_quantile": (C.c_double, [C.c_double, f64p, sz]),
        "vmo_mode_no_nans": (C.c_double, [C.c_double, f64p, sz]),
        "vmo_linear_regression": (C.c_double, [f64p, i64p, sz, C.c_int64, f64p]),
        "vmo_aggr_update": (None, [C.c_int, f64p, f64p, f64p, sz]),
        "vmo_aggr_merge": (None, [C.c_int, f64p, f64p, f64p, f64p, sz]),
        "vmo_aggr_finalize": (None, [C.c_int, f64p, f64p, sz]),
    }
    for name, (res, args) in sig.items():
        try:
            fn = getattr(L, name)
        except AttributeError:
            continue
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L


def _u8(a):
    return a.ctypes.data_as(u8p)


def _i64(a):
    return a.ctypes.data_as(i64p)


def _f64(a):
    return a.ctypes.data_as(f64p)


# ---- convenience wrappers (numpy in / numpy out) -------------------------------------------------

def marshal_varint64s(vs):
    vs = np.ascontiguousarray(vs, dtype=np.int64)
    dst = np.empty(len(vs) * 10 + 16, dtype=np.uint8)
    n = lib().vmo_marshal_varint64s(_u8(dst), dst.size, _i64(vs), len(vs))
    assert n >= 0
    return dst[:n].copy()


def unmarshal_varint64s(src, n):
    src = np.ascontiguousarray(src, dtype=np.uint8)
    dst = np.empty(max(n, 1), dtype=np.int64)
    consumed = C.c_size_t(0)
    rc = lib().vmo_unmarshal_varint64s(_i64(dst), n, _u8(src), len(src), C.byref(consumed))
    return rc, dst[:n], consumed.value


def nearest_delta(nxt, prev, pb, prev_tz=None):
    L = lib()
    if prev_tz is None:
        prev_tz = L.vmo_get_trailing_zeros(prev, pb)
    d = C.c_int64(0)
    tz = C.c_uint8(0)
    L.vmo_nearest_delta(nxt, prev, pb, prev_tz, C.byref(d), C.byref(tz))
    return d.value, tz.value


def marshal_nearest_delta(vals, pb, delta2=False):
    vals = np.ascontiguousarray(vals, dtype=np.int64)
    dst = np.empty(len(vals) * 10 + 16, dtype=np.uint8)
    first = C.c_int64(0)
    fn = lib().vmo_marshal_nearest_delta2 if delta2 else lib().vmo_marshal_nearest_delta
    n = fn(_u8(dst), dst.size, _i64(vals), len(vals), pb, C.byref(first))
    assert n >= 0, n
    return dst[:n].copy(), first.value


def unmarshal_nearest_delta(src, first, n, delta2=False):
    src = np.ascontiguousarray(src, dtype=np.uint8)
    dst = np.empty(n, dtype=np.int64)
    fn = lib().vmo_unmarshal_nearest_delta2 if delta2 else lib().vmo_unmarshal_nearest_delta
    rc = fn(_i64(dst), _u8(src), len(src), first, n)
    return rc, dst


def marshal_int64_array(vals, pb=64):
    """encoding.MarshalValues / MarshalTimestamps -> (bytes, mt, first)"""
    vals = np.ascontiguousarray(vals, dtype=np.int64)
    dst = np.empty(len(vals) * 10 + 1024, dtype=np.uint8)
    mt = C.c_int(0)
    first = C.c_int64(0)
    n = lib().vmo_marshal_int64_array(_u8(dst), dst.size, _i64(vals), len(vals), pb, C.byref(mt), C.byref(first))
    if n < 0:
        raise RuntimeError("vmo_marshal_int64_array rc=%d" % n)
    return dst[:n].copy(), mt.value, first.value


def unmarshal_int64_array(src, mt, first, n):
    src = np.ascontiguousarray(src, dtype=np.uint8)
    dst = np.empty(max(n, 1), dtype=np.int64)
    rc = lib().vmo_unmarshal_int64_array(_i64(dst), _u8(src), len(src), mt, first, n)
    return rc, dst[:n]


def zstd_decompress(src):
    """the oracle's own decoder, into Frame_Content_Size or (without one) the bound of the content from the block headers"""
    src = np.ascontiguousarray(src, dtype=np.uint8)
    cs = lib().vmo_zstd_content_bound(_u8(src), len(src))
    if cs < 0:
        return cs, None
    dst = np.empty(cs + 8, dtype=np.uint8)
    n = lib().vmo_zstd_decompress(_u8(dst), cs, _u8(src), len(src))
    if n < 0:
        return n, None
    return 0, dst[:n].copy()


def zstd_ref_compress(src, level):
    src = np.ascontiguousarray(src, dtype=np.uint8)
    dst = np.empty(len(src) + (len(src) >> 7) + 1024, dtype=np.uint8)
    n = lib().vmo_zstd_ref_compress(_u8(dst), dst.size, _u8(src), len(src), level)
    if n < 0:
        raise RuntimeError("zstd ref compress rc=%d" % n)
    return dst[:n].copy()


def zstd_ref_compress_checksum(src, level):
    """a frame with a Content_Checksum (RFC 8878 3.1.1)"""
    src = np.ascontiguousarray(src, dtype=np.uint8)
    dst = np.empty(len(src) + (len(src) >> 7) + 1024, dtype=np.uint8)
    n = lib().vmo_zstd_ref_compress_checksum(_u8(dst), dst.size, _u8(src), len(src), level)
    if n < 0:
        raise RuntimeError("zstd ref compress (checksum) rc=%d" % n)
    return dst[:n].copy()


# ZSTD_cParameter values of libzstd 1.5.7 (zstd.h; the experimental ones under ZSTD_STATIC_LINKING_ONLY)
ZSTD_C = {"compressionLevel": 100, "windowLog": 101, "hashLog": 102, "chainLog": 103, "searchLog": 104, "minMatch": 105,
          "targetLength": 106, "strategy": 107, "targetCBlockSize": 130, "contentSizeFlag": 200, "checksumFlag": 201,
          "literalCompressionMode": 1002, "maxBlockSize": 1015}
ZSTD_LCM_HUFFMAN, ZSTD_LCM_UNCOMPRESSED = 1, 2  # ZSTD_ParamSwitch_e values of literalCompressionMode


def _kv(params):
    kv = []
    for k, v in (params or {}).items():
        kv += [ZSTD_C[k], int(v)]
    return (C.c_int * max(len(kv), 1))(*kv), len(kv) // 2


def zstd_ref_compress_params(src, **params):
    """ZSTD_compress2 with ZSTD_CCtx_setParameter(name, value) for each keyword (names as in ZSTD_C)"""
    src = np.ascontiguousarray(src, dtype=np.uint8)
    dst = np.empty(len(src) + (len(src) >> 7) + 1024, dtype=np.uint8)
    kv, nkv = _kv(params)
    n = lib().vmo_zstd_ref_compress_params(_u8(dst), dst.size, _u8(src), len(src), kv, nkv)
    if n < 0:
        raise RuntimeError("zstd ref compress %s rc=%d" % (params, n))
    return dst[:n].copy()


def zstd_ref_compress_sequences(src, seqs, **params):
    """ZSTD_compressSequences with explicit block delimiters.  seqs: (offset, literal length, match length) triples over
    src; (0, ll, 0) closes a block with ll trailing literals.  Repeat offsets are resolved by the compressor."""
    src = np.ascontiguousarray(src, dtype=np.uint8)
    s = np.ascontiguousarray(np.asarray(seqs, dtype=np.uint32).reshape(-1, 3))
    dst = np.empty(len(src) + (len(src) >> 7) + 1024, dtype=np.uint8)
    params.setdefault("minMatch", 3)  # (the validation rejects matches shorter than minMatch)
    kv, nkv = _kv(params)
    n = lib().vmo_zstd_ref_compress_sequences(_u8(dst), dst.size, _u8(src), len(src), s.ctypes.data_as(C.POINTER(C.c_uint32)),
                                              len(s), kv, nkv)
    if n < 0:
        raise RuntimeError("zstd ref compress_sequences rc=%d" % n)
    return dst[:n].copy()


def zstd_ref_decompress_rc(src, cap):
    """libzstd's ZSTD_decompressDCtx into cap bytes: (length or a negative rc, bytes or None)"""
    src = np.ascontiguousarray(src, dtype=np.uint8)
    dst = np.empty(cap + 8, dtype=np.uint8)
    n = lib().vmo_zstd_ref_decompress(_u8(dst), cap, _u8(src), len(src))
    return (n, dst[:n].copy()) if n >= 0 else (n, None)


def zstd_ref_decompress(src, cap):
    src = np.ascontiguousarray(src, dtype=np.uint8)
    dst = np.empty(cap + 8, dtype=np.uint8)
    n = lib().vmo_zstd_ref_decompress(_u8(dst), cap, _u8(src), len(src))
    if n < 0:
        raise RuntimeError("zstd ref decompress rc=%d" % n)
    return dst[:n].copy()


def decimal_to_float(va, e):
    va = np.ascontiguousarray(va, dtype=np.int64)
    dst = np.empty(len(va), dtype=np.float64)
    lib().vmo_decimal_to_float(_f64(dst), _i64(va), len(va), e)
    return dst


def float_to_decimal(fa):
    fa = np.ascontiguousarray(fa, dtype=np.float64)
    dst = np.empty(len(fa), dtype=np.int64)
    e = lib().vmo_float_to_decimal(_i64(dst), _f64(fa), len(fa))
    return dst, e


def rollup_do(func_id, values, timestamps, start, end, step, window, lookback_delta=0, may_adjust_window=False,
              is_default_rollup=False, samples_scanned_per_call=0, args=None, args2=None, min_staleness_ms=0):
    values = np.ascontiguousarray(values, dtype=np.float64)
    timestamps = np.ascontiguousarray(timestamps, dtype=np.int64)
    p = 1 + (end - start) // step
    out = np.empty(p, dtype=np.float64)
    cfg = RollupCfg(func_id, start, end, step, window, lookback_delta, min_staleness_ms, int(may_adjust_window),
                    int(is_default_rollup), samples_scanned_per_call, None, None)
    keep = []
    if args is not None:
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(args, dtype=np.float64), (p,)))
        keep.append(a)
        cfg.args = _f64(a)
    if args2 is not None:
        a2 = np.ascontiguousarray(np.broadcast_to(np.asarray(args2, dtype=np.float64), (p,)))
        keep.append(a2)
        cfg.args2 = _f64(a2)
    scanned = lib().vmo_rollup_do(C.byref(cfg), _f64(out), _f64(values), _i64(timestamps), len(values))
    return out, scanned


def merge_sort_blocks(ts_list, val_list, dedup_interval=0):
    """netstorage.go:566 mergeSortBlocks over per-block (timestamps, values) arrays -> (timestamps, values)"""
    offs = np.zeros(len(ts_list) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(t) for t in ts_list])
    n = int(offs[-1])
    ts = np.ascontiguousarray(np.concatenate([np.asarray(t, dtype=np.int64) for t in ts_list]) if n else np.zeros(0, np.int64))
    vals = np.ascontiguousarray(np.concatenate([np.asarray(v, dtype=np.float64) for v in val_list]) if n else np.zeros(0, np.float64))
    ots, ovals = np.zeros(max(n, 1), dtype=np.int64), np.zeros(max(n, 1), dtype=np.float64)
    m = lib().vmo_merge_sort_blocks(ts.ctypes.data_as(i64p), vals.ctypes.data_as(f64p), offs.ctypes.data_as(u64p), len(ts_list),
                                    int(dedup_interval), ots.ctypes.data_as(i64p), ovals.ctypes.data_as(f64p))
    return ots[:m].copy(), ovals[:m].copy()


def deduplicate_samples(ts, vals, interval):
    ts = np.array(ts, dtype=np.int64)
    vals = np.array(vals, dtype=np.float64)
    if len(ts) == 0:
        return ts, vals
    m = lib().vmo_deduplicate_samples(ts.ctypes.data_as(i64p), vals.ctypes.data_as(f64p), len(ts), int(interval))
    return ts[:m].copy(), vals[:m].copy()
