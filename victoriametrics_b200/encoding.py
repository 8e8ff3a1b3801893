"""lib/encoding/encoding.go mirror: (Un)MarshalValues / (Un)MarshalTimestamps."""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import check, lib

# MarshalType encoding.go:20-43
MarshalTypeZSTDNearestDelta2 = 1
MarshalTypeDeltaConst = 2
MarshalTypeConst = 3
MarshalTypeZSTDNearestDelta = 4
MarshalTypeNearestDelta2 = 5
MarshalTypeNearestDelta = 6


def marshal_values(values, precision_bits=64):
    """encoding.MarshalValues encoding.go:103 -> (bytes as np.uint8, MarshalType, firstValue)"""
    a = np.ascontiguousarray(values, dtype=np.int64)
    if a.size == 0:
        raise ValueError("BUG: a must contain at least one item")  # encoding.go:121
    dst = np.empty(a.size * 10 + 1024, dtype=np.uint8)
    n = C.c_size_t(0)
    mt = C.c_int(0)
    first = C.c_int64(0)
    check(lib().vmb_marshal_int64(dst.ctypes.data_as(_lib.u8p), dst.size, C.byref(n), C.byref(mt), C.byref(first),
                                  a.ctypes.data_as(_lib.i64p), a.size, precision_bits))
    return dst[:n.value].copy(), mt.value, first.value


marshal_timestamps = marshal_values  # encoding.go:82: same body


def unmarshal_values(src, mt, first_value, items_count, ctx=None):
    """encoding.UnmarshalValues encoding.go:111 -> np.int64[items_count]; raises VmbError like the Go error return"""
    ctx = ctx or _lib.default_context()
    s = np.ascontiguousarray(src, dtype=np.uint8)
    dst = np.empty(max(items_count, 1), dtype=np.int64)
    check(lib().vmb_unmarshal_int64(ctx.h, dst.ctypes.data_as(_lib.i64p), items_count, s.ctypes.data_as(_lib.u8p), s.size,
                                    int(mt), int(first_value)))
    return dst[:items_count]


unmarshal_timestamps = unmarshal_values  # encoding.go:90


def zstd_compress(src):
    """the library's own zstd writer (valid frames; see include/vmb200.h vmb_marshal_int64)"""
    s = np.ascontiguousarray(src, dtype=np.uint8)
    dst = np.empty(s.size + (s.size >> 6) + 64, dtype=np.uint8)
    n = C.c_size_t(0)
    check(lib().vmb_zstd_compress(dst.ctypes.data_as(_lib.u8p), dst.size, C.byref(n), s.ctypes.data_as(_lib.u8p), s.size))
    return dst[:n.value].copy()


def zstd_compress_batch(sources, ctx=None):
    """encoding.CompressZSTDLevel compress.go:13 for a list of sources at once (GPU) -> list of np.uint8 frames, each equal to
    zstd_compress(source) byte for byte.  Every source needs 1 byte .. 128 MiB."""
    ctx = ctx or _lib.default_context()
    srcs = [np.ascontiguousarray(np.frombuffer(s, dtype=np.uint8) if isinstance(s, (bytes, bytearray)) else s, dtype=np.uint8)
            for s in sources]
    n = len(srcs)
    if n == 0:
        return []
    offs = np.zeros(n + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([s.size for s in srcs])
    arena = np.concatenate(srcs)
    if arena.size == 0:
        arena = np.zeros(1, dtype=np.uint8)
    # the writer never makes a frame larger than the Raw-block frame: header + source + a 3-byte header per 128 KiB
    dst = np.empty(int(offs[-1]) + n * 9 + 3 * sum(-(-s.size // (1 << 17)) for s in srcs), dtype=np.uint8)
    doffs = np.zeros(n + 1, dtype=np.uint64)
    check(lib().vmb_zstd_compress_batch(ctx.h, arena.ctypes.data_as(_lib.u8p), offs.ctypes.data_as(_lib.u64p), n,
                                        dst.ctypes.data_as(_lib.u8p), dst.size, doffs.ctypes.data_as(_lib.u64p)))
    return [dst[int(doffs[i]):int(doffs[i + 1])].copy() for i in range(n)]


def decompress_zstd_batch(frames, ctx=None):
    """encoding.DecompressZSTD compress.go:27 for a list of frames at once (GPU) -> list of np.uint8 arrays.
    Raises VmbError(VMB_ERR_ZSTD) if a frame is corrupt, like the Go error return."""
    ctx = ctx or _lib.default_context()
    frames = [np.ascontiguousarray(np.frombuffer(f, dtype=np.uint8) if isinstance(f, (bytes, bytearray)) else f, dtype=np.uint8)
              for f in frames]
    n = len(frames)
    if n == 0:
        return []
    offs = np.zeros(n + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([f.size for f in frames])
    arena = np.concatenate(frames) if n else np.zeros(0, dtype=np.uint8)
    if arena.size == 0:
        arena = np.zeros(1, dtype=np.uint8)
    bound = C.c_uint64(0)
    check(lib().vmb_zstd_decompress_bound(arena.ctypes.data_as(_lib.u8p), offs.ctypes.data_as(_lib.u64p), n, C.byref(bound)))
    dst = np.empty(max(bound.value, 1), dtype=np.uint8)
    doffs = np.zeros(n, dtype=np.uint64)
    dlens = np.zeros(n, dtype=np.uint32)
    st = np.zeros(n, dtype=np.int32)
    check(lib().vmb_zstd_decompress_batch(ctx.h, arena.ctypes.data_as(_lib.u8p), offs.ctypes.data_as(_lib.u64p), n,
                                          dst.ctypes.data_as(_lib.u8p), dst.size, doffs.ctypes.data_as(_lib.u64p),
                                          dlens.ctypes.data_as(_lib.u32p), st.ctypes.data_as(_lib.i32p)))
    return [dst[int(o):int(o) + int(l)] for o, l in zip(doffs, dlens)]


def marshal_columns(vals2d, precision_bits=64, nthreads=None, ctx=None):
    """batched MarshalValues for equal-length columns: vals2d [ncols x rows] int64
    -> (payload np.uint8, offs np.uint64[ncols+1], mts np.uint8[ncols], firsts np.int64[ncols]).
    ctx given: everything runs on the GPU (vmb_marshal_columns_gpu, csrc/encode.cu) -- type detection, delta coding, varint
    packing, the zstd stage with the 0.9 rule, and the compaction of the payloads; nthreads is then not used.  Without ctx,
    nthreads host threads do the work.  The bytes are the same either way."""
    import os
    a = np.ascontiguousarray(vals2d, dtype=np.int64)
    ncols, rows = a.shape
    nthreads = nthreads or os.cpu_count() or 1
    dst = np.empty(ncols * (rows * 10 + 64), dtype=np.uint8)
    offs = np.zeros(ncols + 1, dtype=np.uint64)
    mts = np.zeros(ncols, dtype=np.uint8)
    firsts = np.zeros(ncols, dtype=np.int64)
    if ctx is not None:
        check(lib().vmb_marshal_columns_gpu(ctx.h, dst.ctypes.data_as(_lib.u8p), dst.size, offs.ctypes.data_as(_lib.u64p),
                                            mts.ctypes.data_as(_lib.u8p), firsts.ctypes.data_as(_lib.i64p),
                                            a.ctypes.data_as(_lib.i64p), ncols, rows, precision_bits, nthreads))
    else:
        check(lib().vmb_marshal_columns(dst.ctypes.data_as(_lib.u8p), dst.size, offs.ctypes.data_as(_lib.u64p),
                                        mts.ctypes.data_as(_lib.u8p), firsts.ctypes.data_as(_lib.i64p),
                                        a.ctypes.data_as(_lib.i64p), ncols, rows, precision_bits, nthreads))
    return dst[:int(offs[-1])].copy(), offs, mts, firsts
