"""ctypes binding of libvmb200.so (include/vmb200.h).  Fails loudly if the CUDA library is missing: there is no CPU path."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, "libvmb200.so")

u8p = C.POINTER(C.c_uint8)
i64p = C.POINTER(C.c_int64)
f64p = C.POINTER(C.c_double)
u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)
i32p = C.POINTER(C.c_int32)


class BlockDesc(C.Structure):
    """vmb_block_desc == lib/storage/block_header.go:19 blockHeader"""
    _fields_ = [("first_value", C.c_int64), ("min_ts", C.c_int64), ("max_ts", C.c_int64), ("ts_off", C.c_uint64),
                ("val_off", C.c_uint64), ("ts_size", C.c_uint32), ("val_size", C.c_uint32), ("rows", C.c_uint32),
                ("series_idx", C.c_uint32), ("scale", C.c_int16), ("ts_mt", C.c_uint8), ("val_mt", C.c_uint8),
                ("precision_bits", C.c_uint8), ("_pad", C.c_uint8 * 3)]


assert C.sizeof(BlockDesc) == 64


class MetaindexRow(C.Structure):
    """vmb_metaindex_row == lib/storage/metaindex_row.go:12 metaindexRow"""
    _fields_ = [("tsid", C.c_uint8 * 24), ("min_ts", C.c_int64), ("max_ts", C.c_int64), ("index_block_offset", C.c_uint64),
                ("block_headers_count", C.c_uint32), ("index_block_size", C.c_uint32)]


assert C.sizeof(MetaindexRow) == 56


class PartFiles(C.Structure):
    """vmb_part_files: the four data files of a part (lib/storage/part.go:34)"""
    _fields_ = [("metaindex", u8p), ("index", u8p), ("timestamps", u8p), ("values", u8p), ("metaindex_len", C.c_uint64),
                ("index_len", C.c_uint64), ("timestamps_len", C.c_uint64), ("values_len", C.c_uint64)]


class MergeStats(C.Structure):
    """vmb_merge_stats: partHeader after the merge + the rowsMerged / rowsDeleted counters"""
    _fields_ = [("rows_count", C.c_uint64), ("blocks_count", C.c_uint64), ("min_ts", C.c_int64), ("max_ts", C.c_int64),
                ("rows_merged", C.c_uint64), ("rows_deleted", C.c_uint64)]


class RawRows(C.Structure):
    """vmb_raw_rows: one row set of a flush (n rawRows of lib/storage/raw_row.go:12 as columns)"""
    _fields_ = [("tsids", u8p), ("timestamps", i64p), ("values", f64p), ("precision_bits", u8p), ("n", C.c_uint64)]


class RollupCfg(C.Structure):
    """vmb_rollup_cfg == rollupConfig (rollup.go:574)"""
    _fields_ = [("func_id", C.c_int32), ("flags", C.c_uint32), ("start", C.c_int64), ("end", C.c_int64),
                ("step", C.c_int64), ("window", C.c_int64), ("lookback_delta", C.c_int64),
                ("min_staleness_ms", C.c_int64), ("samples_scanned_per_call", C.c_int32), ("_pad", C.c_int32),
                ("args", f64p), ("args2", f64p)]


class VmbError(RuntimeError):
    def __init__(self, code, msg=""):
        super().__init__("libvmb200 error %d: %s" % (code, msg))
        self.code = code


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise ImportError("victoriametrics_b200: %s is missing -- build it with `python -c 'import __graft_entry__ as g; "
                          "g.build()'` (nvcc, sm_90a). There is no CPU fallback." % SO_PATH)
    L = C.CDLL(SO_PATH)
    sz = C.c_size_t
    vp = C.c_void_p
    sig = {
        "vmb_ctx_create": (C.c_int, [C.c_int, C.POINTER(vp)]),
        "vmb_ctx_destroy": (None, [vp]),
        "vmb_ctx_set_stream": (C.c_int, [vp, vp]),
        "vmb_ctx_synchronize": (C.c_int, [vp]),
        "vmb_ctx_set_fused": (C.c_int, [vp, C.c_int]),
        "vmb_comm_get_unique_id": (C.c_int, [u8p]),
        "vmb_ctx_comm_init": (C.c_int, [vp, u8p, C.c_int, C.c_int]),
        "vmb_ctx_comm_attach": (C.c_int, [vp, vp, C.c_int, C.c_int]),
        "vmb_ctx_comm_destroy": (C.c_int, [vp]),
        "vmb_ctx_comm_size": (C.c_int, [vp]),
        "vmb_ctx_comm_rank": (C.c_int, [vp]),
        "vmb_aggr_allreduce": (C.c_int, [vp, C.c_int, vp, vp, sz]),
        "vmb_topk_allgather": (C.c_int, [vp, vp, sz, vp]),
        "vmb_eval_rollup_aggr_dist": (C.c_int, [vp, vp, C.c_int64, C.c_int64, C.POINTER(RollupCfg), C.c_int, u32p, C.c_uint32, f64p, u64p]),
        "vmb_last_error": (C.c_char_p, []),
        "vmb_version": (C.c_int, []),
        "vmb_fused_grid": (C.c_int, []),
        "vmb_fused_grid_chunked": (C.c_int, []),
        "vmb_ctx_launch_count": (C.c_uint64, [vp]),
        "vmb_block_desc_from_header": (C.c_int, [C.POINTER(BlockDesc), u8p, u8p]),
        "vmb_block_header_marshal": (C.c_int, [u8p, C.POINTER(BlockDesc), u8p]),
        "vmb_index_block_unmarshal": (C.c_int, [C.POINTER(BlockDesc), u8p, sz, u8p, sz]),
        "vmb_metaindex_rows_unmarshal": (C.c_int, [C.POINTER(MetaindexRow), sz, C.POINTER(sz), u8p, sz]),
        "vmb_metaindex_row_marshal": (C.c_int, [u8p, C.POINTER(MetaindexRow)]),
        "vmb_zstd_decompress_bound": (C.c_int, [u8p, u64p, sz, u64p]),
        "vmb_zstd_decompress_batch": (C.c_int, [vp, u8p, u64p, sz, u8p, sz, u64p, u32p, i32p]),
        "vmb_zstd_compress_batch": (C.c_int, [vp, u8p, u64p, sz, u8p, sz, u64p]),
        "vmb_merge_parts": (C.c_int, [vp, C.POINTER(PartFiles), sz, C.c_int64, u64p, sz, C.POINTER(vp), C.POINTER(MergeStats)]),
        "vmb_parts_from_rows": (C.c_int, [vp, C.POINTER(RawRows), sz, C.POINTER(vp), C.POINTER(MergeStats)]),
        "vmb_merged_part_files": (C.c_int, [vp, C.POINTER(PartFiles)]),
        "vmb_merged_part_free": (None, [vp]),
        "vmb_merge_metaindex_frame": (C.c_int, [vp, u8p, sz, u8p, sz, C.POINTER(sz)]),
        "vmb_calibrate_scale": (C.c_int, [i64p, sz, C.c_int16, i64p, sz, C.c_int16, C.POINTER(C.c_int16)]),
        "vmb_unmarshal_int64": (C.c_int, [vp, i64p, sz, u8p, sz, C.c_int, C.c_int64]),
        "vmb_decimal_to_float": (C.c_int, [vp, f64p, i64p, sz, C.c_int16]),
        "vmb_marshal_int64": (C.c_int, [u8p, sz, C.POINTER(sz), C.POINTER(C.c_int), i64p, i64p, sz, C.c_uint8]),
        "vmb_float_to_decimal": (C.c_int, [i64p, C.POINTER(C.c_int16), f64p, sz]),
        "vmb_float_to_decimal_columns": (C.c_int, [vp, i64p, C.POINTER(C.c_int16), f64p, sz, sz]),
        "vmb_zstd_compress": (C.c_int, [u8p, sz, C.POINTER(sz), u8p, sz]),
        "vmb_marshal_columns": (C.c_int, [u8p, sz, u64p, u8p, i64p, i64p, sz, sz, C.c_uint8, C.c_int]),
        "vmb_marshal_columns_gpu": (C.c_int, [vp, u8p, sz, u64p, u8p, i64p, i64p, sz, sz, C.c_uint8, C.c_int]),
        "vmb_blocks_upload": (C.c_int, [vp, C.POINTER(BlockDesc), sz, u8p, sz, C.POINTER(vp)]),
        "vmb_blocks_upload_part": (C.c_int, [vp, u8p, sz, u8p, sz, u8p, sz, C.POINTER(vp)]),
        "vmb_blocks_free": (None, [vp]),
        "vmb_blocks_count": (sz, [vp]),
        "vmb_blocks_rows": (C.c_uint64, [vp]),
        "vmb_blocks_compressed_bytes": (C.c_uint64, [vp]),
        "vmb_decode_blocks": (C.c_int, [vp, vp, C.c_int64, C.c_int64, C.c_uint32, i32p, C.POINTER(vp)]),
        "vmb_series_from_host": (C.c_int, [vp, i64p, f64p, u64p, sz, C.POINTER(vp)]),
        "vmb_series_from_matrix": (C.c_int, [vp, vp, sz, sz, C.c_int64, C.c_int64, C.POINTER(vp)]),
        "vmb_series_free": (None, [vp]),
        "vmb_series_count": (sz, [vp]),
        "vmb_series_rows": (C.c_uint64, [vp]),
        "vmb_series_layout": (C.c_int, [vp, vp, u64p, u32p]),
        "vmb_series_download": (C.c_int, [vp, vp, i64p, f64p]),
        "vmb_rollup_points": (C.c_int64, [C.POINTER(RollupCfg)]),
        "vmb_rollup": (C.c_int, [vp, vp, C.POINTER(RollupCfg), vp, C.c_int, u64p]),
        "vmb_rollup_aggr_partial": (C.c_int, [vp, vp, C.POINTER(RollupCfg), C.c_int, u32p, C.c_uint32, vp, vp, vp, u64p]),
        "vmb_aggr_merge": (C.c_int, [vp, C.c_int, vp, vp, vp, vp, sz]),
        "vmb_aggr_prepare_allreduce": (C.c_int, [vp, C.c_int, vp, vp, sz]),
        "vmb_aggr_finalize": (C.c_int, [vp, C.c_int, vp, vp, sz, f64p]),
        "vmb_eval_rollup_host": (C.c_int, [vp, C.POINTER(BlockDesc), sz, u8p, sz, C.c_int64, C.c_int64,
                                           C.POINTER(RollupCfg), f64p, i32p, u64p]),
        "vmb_eval_rollup_device": (C.c_int, [vp, vp, C.c_int64, C.c_int64, C.POINTER(RollupCfg), vp, u64p]),
        "vmb_eval_rollup_aggr_host": (C.c_int, [vp, C.POINTER(BlockDesc), C.c_size_t, u8p, C.c_size_t, C.c_int64, C.c_int64,
                                                C.POINTER(RollupCfg), C.c_int, u32p, C.c_uint32, f64p, i32p, u64p]),
        "vmb_eval_rollup_aggr_host_partial": (C.c_int, [vp, C.POINTER(BlockDesc), C.c_size_t, u8p, C.c_size_t, C.c_int64, C.c_int64,
                                                        C.POINTER(RollupCfg), C.c_int, u32p, C.c_uint32, vp, vp, i32p, u64p]),
        "vmb_eval_rollup_aggr_device": (C.c_int, [vp, vp, C.c_int64, C.c_int64, C.POINTER(RollupCfg), C.c_int, u32p, C.c_uint32,
                                                  vp, vp, u64p]),
        "vmb_ctx_set_dedup_interval": (C.c_int, [vp, C.c_int64]),
        "vmb_topk_candidates": (C.c_int, [vp, vp, C.c_size_t, C.c_size_t, u32p, C.c_uint32, C.c_uint32, C.c_int, C.c_uint64, vp]),
        "vmb_topk_merge": (C.c_int, [vp, vp, C.c_uint32, C.c_size_t, C.c_uint32, C.c_int, vp]),
        "vmb_topk_apply": (C.c_int, [vp, vp, C.c_size_t, C.c_size_t, u32p, C.c_uint32, u32p, vp, C.c_uint32, f64p, C.c_int, C.c_uint64, u8p]),
        "vmb_binary_op": (C.c_int, [vp, C.c_int, C.c_int, vp, u32p, vp, u32p, sz, sz, vp]),
        "vmb_matrix_merge_rows": (C.c_int, [vp, vp, i64p, sz, vp, i64p, sz, sz, vp]),
        "vmb_aggr_quantile": (C.c_int, [vp, vp, sz, sz, u32p, C.c_uint32, f64p, vp]),
        "vmb_group_first_value": (C.c_int, [vp, vp, sz, sz, u32p, C.c_uint32, vp]),
        "vmb_aggr_matrix": (C.c_int, [vp, C.c_int, vp, sz, sz, u32p, C.c_uint32, vp, u8p]),
        "vmb_aggr_order": (C.c_int, [vp, C.c_int, vp, sz, sz, u32p, C.c_uint32, f64p, sz, vp, u8p, u8p]),
        "vmb_transform": (C.c_int, [vp, C.c_int, vp, sz, sz, f64p, f64p]),
        "vmb_transform_range": (C.c_int, [vp, C.c_int, vp, sz, sz, f64p, sz, u8p]),
        "vmb_histogram": (C.c_int, [vp, C.c_int, vp, sz, sz, u32p, f64p, C.c_uint32, f64p, sz, vp, vp, vp, u8p]),
        "vmb_vmrange_to_le": (C.c_int, [vp, vp, sz, sz, u32p, f64p, f64p, u32p, u32p, C.c_uint32, vp, C.POINTER(sz), u32p, u8p,
                                        u32p]),
        "vmb_buckets_limit": (C.c_int, [vp, vp, sz, sz, u32p, f64p, C.c_uint32, C.c_int64, u32p, C.POINTER(sz)]),
        "vmb_aggr_rank": (C.c_int, [vp, C.c_int, C.c_int, vp, sz, sz, u32p, C.c_uint32, f64p, vp, u8p, u8p, u32p, u32p, f64p]),
        "vmb_count_values": (C.c_int, [vp, vp, sz, sz, u32p, C.c_uint32, vp, C.POINTER(sz), u32p, f64p]),
        "vmb_rollup_count_values": (C.c_int, [vp, vp, C.POINTER(RollupCfg), vp, C.POINTER(sz), u32p, f64p, u64p]),
        "vmb_aggr_histogram": (C.c_int, [vp, vp, sz, sz, u32p, C.c_uint32, vp, C.POINTER(sz), u32p, u32p]),
        "vmb_rollup_histogram": (C.c_int, [vp, vp, C.POINTER(RollupCfg), vp, C.POINTER(sz), u32p, u32p, u64p]),
        "vmb_rows_nonempty": (C.c_int, [vp, vp, sz, sz, u8p]),
        "vmb_sort_rows": (C.c_int, [vp, vp, sz, sz, C.c_int, u32p]),
        "vmb_set_or": (C.c_int, [vp, vp, sz, u32p, u32p, vp, sz, u32p, u32p, C.c_uint32, sz, u8p, u8p]),
        "vmb_host_alloc": (vp, [sz]),
        "vmb_host_free": (None, [vp]),
        "vmb_ctx_last_stage_ms": (C.c_float, [vp, C.c_int]),
        "vmb_ctx_enable_stage_timing": (C.c_int, [vp, C.c_int]),
    }
    missing = []
    for name, (res, args) in sig.items():
        try:
            fn = getattr(L, name)
        except AttributeError:
            missing.append(name)
            continue
        fn.restype = res
        fn.argtypes = args
    if missing:
        raise ImportError("libvmb200.so lacks symbols declared in include/vmb200.h: %s" % missing)
    _lib = L
    return L


EXPORTED = None  # filled lazily by tests: list of symbol names


def check(rc, allow=()):
    if rc != 0 and rc not in allow:
        raise VmbError(rc, lib().vmb_last_error().decode("utf-8", "replace"))
    return rc


class Context:
    """vmb_ctx: one per process per GPU."""

    def __init__(self, device=0, stream=None):
        h = C.c_void_p()
        check(lib().vmb_ctx_create(device, C.byref(h)))
        self.h = h
        self.device = device
        if stream is not None:
            self.set_stream(stream)

    def set_stream(self, stream):
        check(lib().vmb_ctx_set_stream(self.h, C.c_void_p(int(stream))))

    def set_dedup_interval(self, interval_ms):
        """storage.SetDedupInterval (lib/storage/dedup.go:15): -dedup.minScrapeInterval in ms, 0 = off"""
        check(lib().vmb_ctx_set_dedup_interval(self.h, int(interval_ms)))

    def synchronize(self):
        check(lib().vmb_ctx_synchronize(self.h))

    @property
    def launch_count(self):
        return int(lib().vmb_ctx_launch_count(self.h))

    def set_fused(self, on=True):
        """vmb_ctx_set_fused: fused decode+rollup kernel for the series that qualify (default on)"""
        check(lib().vmb_ctx_set_fused(self.h, int(on)))

    # ---- multi-GPU (csrc/comm.inc): one process per GPU, NCCL inside the library
    @staticmethod
    def comm_unique_id():
        """vmb_comm_get_unique_id (rank 0) -> 128 bytes to hand to every rank"""
        buf = (C.c_uint8 * 128)()
        check(lib().vmb_comm_get_unique_id(buf))
        return bytes(buf)

    def comm_init(self, unique_id, nranks, rank):
        buf = (C.c_uint8 * 128).from_buffer_copy(bytes(unique_id))
        check(lib().vmb_ctx_comm_init(self.h, buf, int(nranks), int(rank)))

    def comm_destroy(self):
        check(lib().vmb_ctx_comm_destroy(self.h))

    @property
    def comm_size(self):
        return int(lib().vmb_ctx_comm_size(self.h))

    def enable_stage_timing(self, on=True):
        check(lib().vmb_ctx_enable_stage_timing(self.h, int(on)))

    def stage_ms(self):
        return [float(lib().vmb_ctx_last_stage_ms(self.h, i)) for i in range(6)]

    def close(self):
        if self.h:
            lib().vmb_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_default_ctx = None


def default_context():
    global _default_ctx
    if _default_ctx is None:
        dev = int(os.environ.get("LOCAL_RANK", "0"))
        _default_ctx = Context(dev)
    return _default_ctx
