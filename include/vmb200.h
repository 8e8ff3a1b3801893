/*
 * vmb200.h -- C ABI of libvmb200: an H100-native (sm_90a) implementation of VictoriaMetrics' data-parallel
 * hot path: the per-series block codec (lib/encoding + lib/decimal) and the range-vector rollup executor
 * (app/vmselect/promql), as scoped by SURVEY.md section 8.
 *
 * The reference has no FFI for this path (it is plain Go calls); each entry point below names the Go function
 * (file:line under the reference checkout) it replaces.  The Go-side cgo binding is shown in INTEGRATION.md.
 *
 * Conventions
 *   - every function returns 0 (VMB_OK) or a negative VMB_ERR_* code; vmb_last_error() gives thread-local text.
 *   - plain pointers and sizes only.  Host buffers are caller-owned and never retained after return.
 *   - device memory is library-owned behind opaque handles (vmb_blocks, vmb_series), or caller-owned raw device
 *     pointers where an argument is documented as "device pointer" (e.g. a torch tensor's data_ptr()).
 *   - there is NO CPU fallback: every compute entry point launches CUDA kernels and fails with
 *     VMB_ERR_CUDA if no sm_90 (H100-class) device is usable.
 *   - all kernels of one vmb_ctx are issued on the ctx's stream (vmb_ctx_set_stream), so the caller can
 *     bracket them with its own CUDA events.
 *   - an entry point with a host output returns with it written and the ctx's stream drained (pinned or pageable).
 *     These return before their kernels finish (wait on the ctx's stream before reading their device outputs):
 *       vmb_group_first_value, vmb_topk_candidates   -- their kernels read the ctx's group scratch (grp)
 *       vmb_topk_merge, vmb_aggr_merge, vmb_aggr_prepare_allreduce, vmb_series_from_matrix -- no ctx scratch
 *       vmb_binary_op without row lists, vmb_transform without per-point arguments         -- no ctx scratch
 *     Growing that scratch in a later call frees it with cudaFree, which waits for the device first.
 */
#ifndef VMB200_H
#define VMB200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VMB_OK 0
/* per-column decode errors: same numbering as the reference error sites they stand for */
#define VMB_ERR_SHORT_SRC (-1)        /* lib/encoding/int.go:183,199,211 */
#define VMB_ERR_VARINT_TOO_BIG (-2)   /* int.go:272 */
#define VMB_ERR_VARINT_TOO_LONG (-3)  /* int.go:277 */
#define VMB_ERR_TAIL (-4)             /* nearest_delta.go:65, encoding.go:238 */
#define VMB_ERR_MARSHAL_TYPE (-5)     /* encoding.go:248 */
#define VMB_ERR_ZSTD (-6)             /* encoding.go:181,193 */
#define VMB_ERR_CONST_TAIL (-7)       /* encoding.go:217 */
#define VMB_ERR_DELTA_CONST (-8)      /* encoding.go:235 */
#define VMB_ERR_TS_BOUNDS (-9)        /* lib/storage/block.go:298 checkTimestampsBounds */
#define VMB_ERR_ROWS (-10)            /* block.go:263 RowsCount must be > 0; block_header.go:233 <= 16384 */
#define VMB_ERR_BLOCK_ORDER (-11)     /* internal consistency check of the series assembly (a hole between time-disjoint blocks) */
/* API-level errors */
#define VMB_ERR_INVALID_ARG (-50)     /* the Go code would logger.Panicf("BUG: ...") */
#define VMB_ERR_CUDA (-51)
#define VMB_ERR_NOMEM (-52)
#define VMB_ERR_BLOCK_FAILED (-53)    /* at least one block failed to decode; see the per-block status array */
#define VMB_ERR_CAP (-54)
#define VMB_ERR_COMM (-55)            /* NCCL could not be loaded, or a collective failed (vmb_last_error has the NCCL text) */

typedef struct vmb_ctx vmb_ctx;
typedef struct vmb_blocks vmb_blocks;  /* compressed blocks resident in HBM (descriptors + payload arena) */
typedef struct vmb_series vmb_series;  /* decoded columns resident in HBM: int64 timestamps + f64 values per series */

/* ---- context ------------------------------------------------------------------------------------------- */
int vmb_ctx_create(int device, vmb_ctx** out);
void vmb_ctx_destroy(vmb_ctx* ctx);
/* stream = a cudaStream_t (0 = legacy default stream). */
int vmb_ctx_set_stream(vmb_ctx* ctx, void* stream);
/* storage.SetDedupInterval lib/storage/dedup.go:15 (-dedup.minScrapeInterval), in ms; 0 (default) = off.  Applied by every
 * block-decoding entry point after the series are assembled (netstorage.go:611 DeduplicateSamples). */
int vmb_ctx_set_dedup_interval(vmb_ctx* ctx, int64_t interval_ms);
/* The one-call device paths (vmb_eval_rollup_device, vmb_eval_rollup_aggr_device) run series that qualify -- one block,
 * MarshalTypeDeltaConst timestamps at precisionBits 64 -- through one fused kernel per batch: decode into shared memory,
 * removeCounterResets and rollupConfig.Do without materialising the decoded columns (the per-series shape of eval.go:1855-1866).
 * Everything else takes the kernel-per-stage pipeline.  enable = 0 forces that pipeline for every series (default: 1; the
 * environment variable VMB_NO_FUSED sets the default to 0).  Results are bit-identical either way. */
int vmb_ctx_set_fused(vmb_ctx* ctx, int enable);
/* CTAs of the fused kernel's (persistent) grid on the current device for rate(): a series list of at most this many series runs
 * one series per CTA.  Never more than 132 x 5. */
int vmb_fused_grid(void);
/* The same for rate() when the call runs its fused series in chunks, the zstd stage of the next chunk beside the fused kernel
 * (at most 132 x 4 CTAs: the rest of the SM is left to the zstd kernels; the other functions keep vmb_fused_grid()). */
int vmb_fused_grid_chunked(void);
int vmb_ctx_synchronize(vmb_ctx* ctx);
const char* vmb_last_error(void);
int vmb_version(void);
/* number of kernel launches issued by this ctx since creation (for bench.py's gpu_launches) */
uint64_t vmb_ctx_launch_count(const vmb_ctx* ctx);

/* ---- block descriptor  ==  lib/storage/block_header.go:19-82 blockHeader (the 81-byte wire form is parsed by
 * vmb_block_desc_from_header) --------------------------------------------------------------------------- */
typedef struct {
    int64_t first_value;     /* FirstValue */
    int64_t min_ts;          /* MinTimestamp (== firstTimestamp passed to UnmarshalTimestamps) */
    int64_t max_ts;          /* MaxTimestamp */
    uint64_t ts_off;         /* byte offset of the timestamps payload inside the payload arena */
    uint64_t val_off;        /* byte offset of the values payload inside the payload arena */
    uint32_t ts_size;        /* TimestampsBlockSize */
    uint32_t val_size;       /* ValuesBlockSize */
    uint32_t rows;           /* RowsCount, 1..16384 */
    uint32_t series_idx;     /* dense series index; the blocks of one series are consecutive, in any order (may overlap) */
    int16_t scale;           /* Scale: value = mantissa * 10^scale */
    uint8_t ts_mt;           /* TimestampsMarshalType 1..6 (lib/encoding/encoding.go:20-43) */
    uint8_t val_mt;          /* ValuesMarshalType */
    uint8_t precision_bits;  /* PrecisionBits 1..64 */
    uint8_t _pad[3];
} vmb_block_desc; /* 64 bytes */

/* blockHeader.Unmarshal block_header.go:122 (81 bytes, big endian); ts_off/val_off are taken from the header
 * (file offsets) -- the caller rebases them onto its payload arena.  series_idx is left 0. */
int vmb_block_desc_from_header(vmb_block_desc* out, const uint8_t header[81], uint8_t tsid_out[24]);

/* blockHeader.Marshal block_header.go:104 (inverse of the above; tsid may be NULL = zeros) */
int vmb_block_header_marshal(uint8_t header[81], const vmb_block_desc* d, const uint8_t tsid[24]);
/* unmarshalBlockHeaders block_header.go:261 (part_search.go:247): an uncompressed index block = `count` 81-byte headers
 * sorted by TSID.  out[count]; tsids ([count * 24], may be NULL) receives the TSIDs.  Errors: wrong length
 * (VMB_ERR_SHORT_SRC / VMB_ERR_ROWS), a header that fails blockHeader.validate (:230), unsorted TSIDs (VMB_ERR_INVALID_ARG). */
int vmb_index_block_unmarshal(vmb_block_desc* out, uint8_t* tsids, size_t count, const uint8_t* data, size_t len);
/* metaindexRow metaindex_row.go:12 (56-byte big-endian wire form :61) */
typedef struct {
    uint8_t tsid[24];
    int64_t min_ts, max_ts;
    uint64_t index_block_offset;
    uint32_t block_headers_count, index_block_size;
} vmb_metaindex_row; /* 56 bytes */
/* unmarshalMetaindexRows metaindex_row.go:129 on the decompressed metaindex.bin (vmb_zstd_decompress_batch below);
 * *n receives the number of rows (also when cap is too small: VMB_ERR_CAP).  Same checks as the Go code: at least one row,
 * BlockHeadersCount > 0, IndexBlockSize <= 2*maxBlockSize, rows sorted by TSID. */
int vmb_metaindex_rows_unmarshal(vmb_metaindex_row* out, size_t cap, size_t* n, const uint8_t* data, size_t len);
int vmb_metaindex_row_marshal(uint8_t out[56], const vmb_metaindex_row* row); /* metaindexRow.Marshal :61 */
/* encoding.DecompressZSTD (lib/encoding/compress.go:27) for n frames at once on the GPU -- index blocks (part_search.go:238)
 * and metaindex.bin (metaindex_row.go:134) go through the same kernels as the block payloads.  frames + offs[n+1] = the
 * compressed frames back to back; every frame must declare its content size (libzstd/gozstd always do; sanity cap 128 MiB).
 * Frame i is written to dst + dst_offs[i] (16-byte aligned), dst_lens[i] bytes; vmb_zstd_decompress_bound gives the dst size.
 * statuses ([n], may be NULL): 0 or VMB_ERR_ZSTD per frame; returns VMB_ERR_ZSTD if any frame failed. */
int vmb_zstd_decompress_bound(const uint8_t* frames, const uint64_t* offs, size_t n, uint64_t* out_bytes);
int vmb_zstd_decompress_batch(vmb_ctx* ctx, const uint8_t* frames, const uint64_t* offs, size_t n, uint8_t* dst,
                              size_t dst_cap, uint64_t* dst_offs, uint32_t* dst_lens, int32_t* statuses);
/* encoding.CompressZSTDLevel (lib/encoding/compress.go:13) for n sources at once on the GPU, host buffers, on the ctx's stream --
 * the frames of a part's index blocks and metaindex (block_stream_writer.go:121,191).  src + offs[n+1] = the sources back to back,
 * each 1 byte .. 128 MiB.  Frame i == vmb_zstd_compress(source i), byte for byte.  Frames are written back to back into dst;
 * dst_offs[n+1] receives their offsets.  dst_cap too small: VMB_ERR_CAP, dst_offs[n] = the bytes needed, dst untouched.
 * VMB_ERR_INVALID_ARG for an empty or oversized source or a NULL pointer.  n == 0: dst_offs[0] = 0.
 * Limit (the writer's, shared with vmb_zstd_compress and the marshal paths): a source of 128 KiB < n <= 262143 bytes that compresses
 * gets ONE Compressed block whose literals regenerate more than Block_Maximum_Size (128 KiB).  The library's decoder accepts that
 * frame; libzstd and klauspost (blockdec.go:345) reject it.  Index blocks (<= 64 KiB, block_stream_writer.go:152) never reach it;
 * a metaindex of more than 128 KiB does, so it must not be compressed with this writer. */
int vmb_zstd_compress_batch(vmb_ctx* ctx, const uint8_t* src, const uint64_t* offs, size_t n, uint8_t* dst, size_t dst_cap,
                            uint64_t* dst_offs);

/* ---- part merges  ==  mergeBlockStreams (lib/storage/merge.go:19) + blockStreamWriter (block_stream_writer.go) ----------------- */
typedef struct {  /* the four data files of a part directory (part.go:34), host buffers */
    const uint8_t *metaindex, *index, *timestamps, *values;
    uint64_t metaindex_len, index_len, timestamps_len, values_len;
} vmb_part_files;
typedef struct {
    uint64_t rows_count, blocks_count; /* partHeader after the merge; min_ts / max_ts = INT64_MAX / INT64_MIN when nothing is left */
    int64_t min_ts, max_ts;
    uint64_t rows_merged, rows_deleted; /* the rowsMerged / rowsDeleted counters of mergeBlockStreams */
} vmb_merge_stats;
typedef struct vmb_merged_part vmb_merged_part;
/* Merges parts[0..nparts) in that order (blockStreamMerger's heap and its ties: block_stream_merger.go) into one part, byte for byte
 * what mergeBlockStreams writes with the library's zstd writer in place of CompressZSTDLevel:
 *   - blocks of deleted_metric_ids (sorted ascending, unique; VMB_ERR_INVALID_ARG otherwise) and blocks with MaxTimestamp <
 *     retention_deadline are dropped, rows before the deadline inside merged blocks too (all counted in rows_deleted);
 *   - blocks of one MetricID are merged by the pending-block chain of merge.go:65-156 (CalibrateScale, PrecisionBits = min,
 *     mergeBlocks, the split at 8192 rows); a block the chain never unmarshals keeps its payload bytes as they are;
 *   - the ctx's dedup interval (vmb_ctx_set_dedup_interval) > 0: deduplicateSamplesDuringMerge (dedup.go:94) on every block;
 *   - identical consecutive timestamps payloads are stored once, index blocks hold at most 809 headers, one metaindex frame.
 * Every frame is accepted by libzstd: a column stream of 128 KiB < n <= 262143 bytes gets no frame of the writer (MarshalType 1 -> 5,
 * 4 -> 6), a metaindex of that size (or an empty one) goes into a frame of Raw blocks.  A re-encoded column whose payload exceeds
 * 128 KiB (such a stream uncompressed; blockHeader.validate block_header.go:248 rejects it) fails the merge with VMB_ERR_CAP.  A part whose metaindex decodes to 0 bytes
 * is an empty part.  Errors: offsets outside a file (VMB_ERR_SHORT_SRC), a header or metaindex row that fails validation, a block
 * the merge must unmarshal that fails to decode (its VMB_ERR_* code); *out is then NULL.  Device memory for the whole merge is
 * needed at once (VMB_ERR_NOMEM otherwise): about 64 bytes per row of every block the merge may unmarshal (the decoded rows and
 * the chain's three regions), plus the payloads and the encoder's scratch. */
int vmb_merge_parts(vmb_ctx* ctx, const vmb_part_files* parts, size_t nparts, int64_t retention_deadline,
                    const uint64_t* deleted_metric_ids, size_t ndeleted, vmb_merged_part** out, vmb_merge_stats* stats);
/* the metaindex frame vmb_merge_parts writes for an n-byte metaindex (exposed for tests): the library's zstd writer, a frame of Raw
 * blocks for n == 0 and 128 KiB < n <= 262143.  *out_len = the frame's length (also with VMB_ERR_CAP when cap is too small). */
int vmb_merge_metaindex_frame(vmb_ctx* ctx, const uint8_t* src, size_t n, uint8_t* dst, size_t cap, size_t* out_len);
/* the merged part's files: pointers into the part's pinned host memory, valid until vmb_merged_part_free */
int vmb_merged_part_files(const vmb_merged_part* p, vmb_part_files* files);
void vmb_merged_part_free(vmb_merged_part* p);

/* ---- part flushes  ==  rawRowsMarshaler.marshalToInmemoryPart (lib/storage/raw_row.go:81) for every row set of a flush ------- */
typedef struct {            /* one rowss[i] of partition.flushRowssToInmemoryParts (partition.go:603): n rawRows (raw_row.go:12) */
    const uint8_t* tsids;   /* [n * 24] marshaled TSIDs (tsid.go:62: MetricGroupID, JobID, InstanceID, MetricID, big endian) */
    const int64_t* timestamps;
    const double* values;
    const uint8_t* precision_bits; /* 1..64 each */
    uint64_t n;
} vmb_raw_rows;
/* Turns each sets[i] into one part, out[i], byte for byte what marshalToInmemoryPart writes with the library's zstd writer in place
 * of CompressZSTDLevel(-5); stats[i] = its partHeader, rows_merged = n, rows_deleted = 0.  All sets go through the device in one
 * pass; the parts go to vmb_merge_parts as they are (the reference's mustMergeInmemoryParts).  Per set:
 *   - the rows are ordered by (TSID, Timestamp) (rawRowsSort.Less raw_row.go:49), the TSID compared as its 24 marshaled bytes.
 *     Tie rule: rows with equal (TSID, Timestamp) keep their input order (a stable sort).  The reference keeps the input order
 *     when the set is already sorted and otherwise leaves such rows in the order of Go's unstable sort.Sort, so the two agree
 *     whenever the input is sorted or no two rows share (TSID, Timestamp);
 *   - a block ends where a row's MetricID differs from the MetricID of the block's first row, or at 8192 rows (raw_row.go:111);
 *     the block takes the TSID and PrecisionBits of its first row.  Rows of one MetricID with different TSIDs can share a block,
 *     and one MetricID can own blocks that are not adjacent;
 *   - per block: AppendFloatToDecimal (one scale), then the ctx's dedup interval > 0: deduplicateSamplesDuringMerge, then the
 *     columns, timestamps payload sharing, index blocks and the metaindex as vmb_merge_parts writes them.
 * An empty set gives an empty part (no blocks, zero rows).  Errors: a NULL pointer or n >= 2^32 (VMB_ERR_INVALID_ARG), a
 * precisionBits outside 1..64 (VMB_ERR_INVALID_ARG, as CheckPrecisionBits encoding.go:68), device memory for the whole call
 * missing (VMB_ERR_NOMEM: about 90 bytes a row plus the encoder's scratch); every out[i] is then NULL.  Free each part with
 * vmb_merged_part_free. */
int vmb_parts_from_rows(vmb_ctx* ctx, const vmb_raw_rows* sets, size_t nsets, vmb_merged_part** out /* [nsets] */,
                        vmb_merge_stats* stats /* [nsets] */);

/* ---- per-call drop-ins (single column; host buffers; run on the GPU) ------------------------------------- */
/* encoding.UnmarshalValues / UnmarshalTimestamps  encoding.go:111 / :90 (unmarshalInt64Array :173) */
int vmb_unmarshal_int64(vmb_ctx* ctx, int64_t* dst, size_t items_count, const uint8_t* src, size_t src_len, int mt,
                        int64_t first_value);
/* decimal.AppendDecimalToFloat  lib/decimal/decimal.go:100 */
int vmb_decimal_to_float(vmb_ctx* ctx, double* dst, const int64_t* va, size_t n, int16_t e);
/* encoding.MarshalValues / MarshalTimestamps  encoding.go:103 / :82 (marshalInt64Array :119).
 * Host-side encoder (the write path stays on the host this round, SURVEY 7 step 6); zstd frames are produced by
 * the library's own Huffman-literals compressor: valid zstd that libzstd/klauspost decode, not byte-identical to
 * libzstd's output (compressed bytes are unpinned by the reference's tests, SURVEY 8c). */
int vmb_marshal_int64(uint8_t* dst, size_t cap, size_t* out_len, int* out_mt, int64_t* out_first, const int64_t* vals,
                      size_t n, uint8_t precision_bits);
/* the library's zstd writer on its own (exposed for tests); see the limit under vmb_zstd_compress_batch */
int vmb_zstd_compress(uint8_t* dst, size_t cap, size_t* out_len, const uint8_t* src, size_t n);
/* Block.MarshalData (block.go:192) for ncols equal-length int64 columns on `nthreads` host threads: payloads are written
 * back to back into dst, offs[ncols+1] receives their offsets, mts/firsts the MarshalType and first value of each. */
int vmb_marshal_columns(uint8_t* dst, size_t cap, uint64_t* offs, uint8_t* mts, int64_t* firsts, const int64_t* vals,
                        size_t ncols, size_t rows, uint8_t precision_bits, int nthreads);
/* The same entirely on the GPU (csrc/encode.cu): isConst / isDeltaConst / isGauge (encoding.go:289-369) as one pass of warp
 * reductions per column, nearest-delta / delta2 (lossless, and the lossy precisionBits < 64 state machine of nearest_delta.go:83),
 * zig-zag varint packing by warp scans; then the zstd stage of streams >= 128 bytes with the library's zstd writer (one CTA per
 * frame), the 0.9 rule (encoding.go:152-167, type 1 -> 5 / 4 -> 6 where the frame is rejected) and the compaction of the payloads
 * in column order.  Byte-identical to vmb_marshal_columns (payload, offsets, types, firsts); VMB_ERR_CAP when cap is too small
 * (offs[ncols] = the bytes needed).  vals: HOST [ncols x rows], rows <= 16384.  nthreads is not read: it only ever chose how many
 * host threads compressed. */
int vmb_marshal_columns_gpu(vmb_ctx* ctx, uint8_t* dst, size_t cap, uint64_t* offs, uint8_t* mts, int64_t* firsts,
                            const int64_t* vals, size_t ncols, size_t rows, uint8_t precision_bits, int nthreads);
/* decimal.AppendFloatToDecimal decimal.go:173 (host-side, write path) */
int vmb_float_to_decimal(int64_t* dst, int16_t* out_scale, const double* src, size_t n);
/* ... for ncols equal-length columns on the GPU (one warp per column: FromFloat per value, min-exponent / overflow reductions,
 * rescale); dst HOST [ncols x rows], scales HOST [ncols], src HOST [ncols x rows].  Same results as the call above per column. */
int vmb_float_to_decimal_columns(vmb_ctx* ctx, int64_t* dst, int16_t* scales, const double* src, size_t ncols, size_t rows);
/* decimal.CalibrateScale decimal.go:13 (host-side; block merge path lib/storage/merge.go): a and b are rescaled in place to
 * the common exponent returned in *out_e. */
int vmb_calibrate_scale(int64_t* a, size_t na, int16_t ae, int64_t* b, size_t nb, int16_t be, int16_t* out_e);

/* ---- batched block decode  ==  Block.UnmarshalData (block.go:250) + AppendRowsWithTimeRangeFilter (:324)
 * for every block of a query at once (replaces netstorage.go:425 packedTimeseries.Unpack fan-out) ------------- */
/* copies descriptors + payload host->device (the one H2D of the path). payload_len bytes are copied. */
int vmb_blocks_upload(vmb_ctx* ctx, const vmb_block_desc* descs, size_t nblocks, const uint8_t* payload,
                      size_t payload_len, vmb_blocks** out);
/* The same from a part on disk: `headers` = nblocks marshaled blockHeaders (81 bytes each) -- what vmselect keeps per block in its
 * tmpBlocksFile (tmp_blocks_file.go:110 WriteBlockRefData, parsed back by BlockRef.Init lib/storage/search.go:38) --, in series
 * order (consecutive headers with the same TSID form one series; netstorage.go groups BlockRefs that way); timestamps_bin /
 * values_bin = the part's two data files (mmap'ed or read), addressed by TimestampsBlockOffset / ValuesBlockOffset like
 * BlockRef.MustReadBlock search.go:73.  Only the referenced byte ranges are copied.  Errors: a header that fails
 * blockHeader.validate, offsets outside the files (VMB_ERR_SHORT_SRC). */
int vmb_blocks_upload_part(vmb_ctx* ctx, const uint8_t* headers, size_t nblocks, const uint8_t* timestamps_bin, size_t ts_len,
                           const uint8_t* values_bin, size_t val_len, vmb_blocks** out);
void vmb_blocks_free(vmb_blocks* b);
size_t vmb_blocks_count(const vmb_blocks* b);
uint64_t vmb_blocks_rows(const vmb_blocks* b);           /* sum of RowsCount */
uint64_t vmb_blocks_compressed_bytes(const vmb_blocks* b); /* sum of ts_size + val_size */

#define VMB_DECODE_VALUES_AS_INT64 1u /* leave values as int64 mantissas (no decimal->float) */
/* decodes all blocks; rows outside [tr_min, tr_max] are trimmed like filterTimestamps (block.go:331).
 * block_status (host, nblocks entries, may be NULL) receives 0 or a VMB_ERR_* per block.
 * Returns VMB_ERR_BLOCK_FAILED if any block failed (the batch is still returned; failed blocks have 0 rows). */
int vmb_decode_blocks(vmb_ctx* ctx, const vmb_blocks* blocks, int64_t tr_min, int64_t tr_max, uint32_t flags,
                      int32_t* block_status, vmb_series** out);

/* builds a device batch from already-decoded host columns (the `values, timestamps` arguments of
 * rollupConfig.Do): series s owns rows [offsets[s], offsets[s+1]) */
int vmb_series_from_host(vmb_ctx* ctx, const int64_t* timestamps, const double* values, const uint64_t* offsets,
                         size_t nseries, vmb_series** out);
/* the feed of evalRollupFuncWithSubquery (eval.go:910): the inner expression's result, a DEVICE matrix [nseries x points] on the grid
 * start, start + step, ..., becomes a batch of series -- removeNanValues (eval.go:1027) drops the NaN points of every row together
 * with their timestamps -- for vmb_rollup with the outer function's config (its preFunc flags apply as usual; dropStaleNaNs does not,
 * there is nothing stale left).  The matrix is not modified and not retained. */
int vmb_series_from_matrix(vmb_ctx* ctx, const double* d_matrix, size_t nseries, size_t points, int64_t start, int64_t step,
                           vmb_series** out);
void vmb_series_free(vmb_series* s);
size_t vmb_series_count(const vmb_series* s);
uint64_t vmb_series_rows(const vmb_series* s); /* allocated rows (before trimming / stale-NaN drop) */
/* per-series current (start,row count) -> host arrays of nseries entries */
int vmb_series_layout(vmb_ctx* ctx, const vmb_series* s, uint64_t* starts, uint32_t* counts);
/* copies the dense decoded columns (vmb_series_rows entries each) device->host; either pointer may be NULL */
int vmb_series_download(vmb_ctx* ctx, const vmb_series* s, int64_t* timestamps, double* values);

/* ---- rollup  ==  rollupConfig.Do (rollup.go:688) for every series at once, preceded by the per-series preamble of
 * eval.go:1855 (dropStaleNaNs eval.go:1985, preFunc = removeCounterResets rollup.go:921) ------------------------- */
enum vmb_rollup_func { /* rollup.go:24-108; names in comments are the MetricsQL names */
    VMB_RF_DEFAULT_ROLLUP = 0, VMB_RF_RATE /* rate, deriv_fast */, VMB_RF_DELTA /* delta, increase */, VMB_RF_AVG,
    VMB_RF_MIN, VMB_RF_MAX, VMB_RF_SUM, VMB_RF_COUNT, VMB_RF_QUANTILE, VMB_RF_FIRST, VMB_RF_LAST, VMB_RF_RANGE,
    VMB_RF_SUM2, VMB_RF_STDDEV, VMB_RF_STDVAR, VMB_RF_IDERIV /* ideriv, irate */, VMB_RF_IDELTA, VMB_RF_DERIV,
    VMB_RF_INCREASE_PURE, VMB_RF_CHANGES, VMB_RF_CHANGES_PROMETHEUS, VMB_RF_RESETS /* resets, decreases_over_time */,
    VMB_RF_INCREASES, VMB_RF_INTEGRATE, VMB_RF_LAG, VMB_RF_LIFETIME, VMB_RF_SCRAPE_INTERVAL, VMB_RF_TMIN, VMB_RF_TMAX,
    VMB_RF_TFIRST, VMB_RF_TLAST /* tlast_over_time, timestamp */, VMB_RF_TLAST_CHANGE, VMB_RF_MODE, VMB_RF_MAD,
    VMB_RF_OUTLIER_IQR, VMB_RF_ZSCORE, VMB_RF_ASCENT, VMB_RF_DESCENT, VMB_RF_DISTINCT, VMB_RF_GEOMEAN,
    VMB_RF_PREDICT_LINEAR, VMB_RF_HOLT_WINTERS, VMB_RF_HOEFFDING_LOWER, VMB_RF_HOEFFDING_UPPER, VMB_RF_DURATION,
    VMB_RF_COUNT_LE, VMB_RF_COUNT_GT, VMB_RF_COUNT_EQ, VMB_RF_COUNT_NE, VMB_RF_SHARE_LE, VMB_RF_SHARE_GT,
    VMB_RF_SHARE_EQ, VMB_RF_SUM_LE, VMB_RF_SUM_GT, VMB_RF_SUM_EQ, VMB_RF_PRESENT, VMB_RF_ABSENT, VMB_RF_STALE_SAMPLES,
    VMB_RF_MEDIAN, VMB_RF_RATE_OVER_SUM, VMB_RF_DELTA_PROMETHEUS /* delta_prometheus, increase_prometheus */,
    VMB_RF_RATE_PROMETHEUS, VMB_RF_OPEN, VMB_RF_CLOSE, VMB_RF_HIGH, VMB_RF_LOW, VMB_RF__COUNT
};

#define VMB_RC_MAY_ADJUST_WINDOW 1u     /* rollupFuncsCanAdjustWindow rollup.go:199 */
#define VMB_RC_IS_DEFAULT_ROLLUP 2u     /* funcName == "default_rollup" rollup.go:408 */
#define VMB_RC_REMOVE_COUNTER_RESETS 4u /* rollupFuncsRemoveCounterResets rollup.go:223: preFunc */
#define VMB_RC_DROP_STALE_NANS 8u       /* eval.go:1985 (not for default_rollup / stale_samples_over_time) */
/* value preFuncs of the multi-output rollups (getRollupConfigs rollup.go:440-476), applied after removeCounterResets,
 * once per batch like it */
#define VMB_RC_PRE_DELTA_VALUES 16u     /* rollup_increase / rollup_delta: deltaValues rollup.go:960 */
#define VMB_RC_PRE_DERIV_VALUES 32u     /* rollup_rate / rollup_deriv: derivValues rollup.go:976 */
#define VMB_RC_PRE_SCRAPE_INTERVAL 64u  /* rollup_scrape_interval: seconds between samples rollup.go:462-474 */
#define VMB_RC_PRE_MASK 112u

typedef struct { /* == rollupConfig rollup.go:574 + what getRollupConfigs (rollup.go:374) derives from the func name */
    int32_t func_id;          /* enum vmb_rollup_func */
    uint32_t flags;           /* VMB_RC_* */
    int64_t start, end, step; /* ms; output grid = start, start+step, ... <= end (eval.go:230 getTimestamps) */
    int64_t window;           /* ms; 0 = not set */
    int64_t lookback_delta;   /* ms; rollupConfig.LookbackDelta */
    int64_t min_staleness_ms; /* -search.minStalenessInterval rollup.go:20 */
    int32_t samples_scanned_per_call; /* rollupFuncsSamplesScannedPerCall rollup.go:238; 0 = len(window) */
    int32_t _pad;
    const double* args;       /* host, P entries or NULL: per-point scalar arg (phi / limit / secs / sf) */
    const double* args2;      /* host, P entries or NULL: second per-point arg (holt_winters tf) */
} vmb_rollup_cfg;

/* number of output points: 1 + (end-start)/step  (eval.go:243) */
int64_t vmb_rollup_points(const vmb_rollup_cfg* cfg);

/* Runs the per-series preamble (in place on the batch: call once per batch) and the rollup.
 * out: [nseries x P] row-major doubles; out_is_device != 0 => out is a device pointer, else host.
 * samples_scanned (host, may be NULL) = sum over series of rollupConfig.Do's second result. */
int vmb_rollup(vmb_ctx* ctx, vmb_series* series, const vmb_rollup_cfg* cfg, double* out, int out_is_device,
               uint64_t* samples_scanned);

/* ---- aggr(rollup(...)) by (...)  ==  evalRollupWithIncrementalAggregate eval.go:1804 + aggr_incremental.go ------ */
enum vmb_aggr_func { VMB_AGGR_SUM = 0, VMB_AGGR_MIN, VMB_AGGR_MAX, VMB_AGGR_AVG, VMB_AGGR_COUNT, VMB_AGGR_SUM2,
                     VMB_AGGR_GEOMEAN, VMB_AGGR_ANY, VMB_AGGR_GROUP };
/* Per-GPU partial state (the per-worker incrementalAggrContext, aggr_incremental.go:184): folds every series of the
 * batch into d_values/d_counts ([ngroups x P] DEVICE pointers, overwritten). group_ids: host, nseries entries, dense
 * ids assigned by the host from the group-by label set (identically on all ranks).  Within a group the series are
 * folded in ascending series order (deterministic).  d_rollup_scratch: device pointer to [nseries x P] doubles or
 * NULL to let the library allocate it. */
int vmb_rollup_aggr_partial(vmb_ctx* ctx, vmb_series* series, const vmb_rollup_cfg* cfg, int aggr_id,
                            const uint32_t* group_ids, uint32_t ngroups, double* d_values, double* d_counts,
                            double* d_rollup_scratch, uint64_t* samples_scanned);
/* mergeAggr* (aggr_incremental.go:218...): dst <- merge(dst, src), all DEVICE pointers, n = ngroups*P.
 * (Multi-GPU runs replace this by one NCCL all-reduce of values and counts for sum/avg/count/sum2, see DESIGN.md.) */
int vmb_aggr_merge(vmb_ctx* ctx, int aggr_id, double* d_dst_values, double* d_dst_counts, const double* d_src_values,
                   const double* d_src_counts, size_t n);
/* makes partial state all-reduce-able with ncclSum (values of empty cells zeroed) or ncclMin/ncclMax (+-Inf) */
int vmb_aggr_prepare_allreduce(vmb_ctx* ctx, int aggr_id, double* d_values, const double* d_counts, size_t n);
/* finalizeAggr* (aggr_incremental.go:189,:368,:400...): in place on DEVICE pointers, then optional copy to out_host */
int vmb_aggr_finalize(vmb_ctx* ctx, int aggr_id, double* d_values, const double* d_counts, size_t n, double* out_host);

/* ---- topk(k, q) / bottomk(k, q)  ==  newAggrFuncTopK aggr.go:646 on a DEVICE matrix d_vals[nseries x P] (e.g. the output
 * of vmb_rollup / vmb_eval_rollup_device): per group and point only the k best values survive, the others become NaN
 * (fillNaNsAtIdx aggr.go:786); rows left without a value are reported so that the host drops them (removeEmptySeries).
 * Exactly k values survive per (group, point); equal values rank by ascending GLOBAL series id (series_id_base + row), one of
 * the outcomes of the reference's unstable sort.Slice, identical on every run and rank.
 *   1. vmb_topk_candidates: d_cand[ngroups x P x kmax] entries of 16 bytes {f64 value, f64 global series id} <- the kmax best
 *      non-NaN values of this process per (group, point), best first, NaN padded; kmax = the largest k of the query, <= 64.
 *      reverse != 0: bottomk.  series_id_base: global id of this process's row 0 (0 on a single GPU).
 *   2. several processes: all-gather the candidate arrays (vmb_topk_allgather: count = cells * kmax * 2 doubles), then
 *      vmb_topk_merge([nparts x cells x kmax] entries, cells = ngroups*P).
 *   3. vmb_topk_apply: ks = one k per point (HOST, getIntK aggr.go:793: NaN / negative -> 0, capped by the group size);
 *      group_sizes = series per group over ALL processes (HOST); row_nonempty = HOST array, 1 byte per series.
 *      Every point must satisfy min(floor(ks[p]), largest group size) <= kmax, the kmax the lists were built with (the entry
 *      that decides a survivor has to be in its list); otherwise VMB_ERR_INVALID_ARG and d_vals is left as it was. */
int vmb_topk_candidates(vmb_ctx* ctx, const double* d_vals, size_t nseries, size_t points, const uint32_t* group_ids,
                        uint32_t ngroups, uint32_t kmax, int reverse, uint64_t series_id_base, double* d_cand);
int vmb_topk_merge(vmb_ctx* ctx, const double* d_parts, uint32_t nparts, size_t cells, uint32_t kmax, int reverse, double* d_cand);
int vmb_topk_apply(vmb_ctx* ctx, double* d_vals, size_t nseries, size_t points, const uint32_t* group_ids, uint32_t ngroups,
                   const uint32_t* group_sizes, const double* d_cand, uint32_t kmax, const double* ks, int reverse,
                   uint64_t series_id_base, unsigned char* row_nonempty);

/* ---- whole path in one call with HOST buffers (what a patched evalRollupNoIncrementalAggregate, eval.go:1845,
 * would call): H2D of descriptors+payload, decode, preamble, rollup, D2H of the [nseries x P] result; processed in
 * chunks so copies overlap the kernels.  out_host: [nseries x P]. */
int vmb_eval_rollup_host(vmb_ctx* ctx, const vmb_block_desc* descs, size_t nblocks, const uint8_t* payload,
                         size_t payload_len, int64_t tr_min, int64_t tr_max, const vmb_rollup_cfg* cfg, double* out_host,
                         int32_t* block_status, uint64_t* samples_scanned);

/* device-resident variant used for kernel-only timing: decode + preamble + rollup, result left in d_out (device) */
int vmb_eval_rollup_device(vmb_ctx* ctx, const vmb_blocks* blocks, int64_t tr_min, int64_t tr_max,
                           const vmb_rollup_cfg* cfg, double* d_out, uint64_t* samples_scanned);

/* aggregate variant of the host path (evalRollupWithIncrementalAggregate eval.go:1804 end to end): the same chunked
 * pipeline as vmb_eval_rollup_host, but every chunk's [series x P] matrix is folded on the GPU into {values, counts}[G x P]
 * and only the finalized [ngroups x P] result (host pointer) travels back.  group_ids: one dense id per series of the batch. */
int vmb_eval_rollup_aggr_host(vmb_ctx* ctx, const vmb_block_desc* descs, size_t nblocks, const uint8_t* payload,
                              size_t payload_len, int64_t tr_min, int64_t tr_max, const vmb_rollup_cfg* cfg, int aggr_id,
                              const uint32_t* group_ids, uint32_t ngroups, double* out_host, int32_t* block_status,
                              uint64_t* samples_scanned);

/* ... without the final step: the partial state of this batch is left in the caller's DEVICE buffers {values, counts}
 * [ngroups x P] (overwritten), for vmb_aggr_merge or vmb_aggr_prepare_allreduce + all-reduce + vmb_aggr_finalize (multi-GPU) */
int vmb_eval_rollup_aggr_host_partial(vmb_ctx* ctx, const vmb_block_desc* descs, size_t nblocks, const uint8_t* payload,
                                      size_t payload_len, int64_t tr_min, int64_t tr_max, const vmb_rollup_cfg* cfg, int aggr_id,
                                      const uint32_t* group_ids, uint32_t ngroups, double* d_values, double* d_counts,
                                      int32_t* block_status, uint64_t* samples_scanned);

/* aggregate variant of the device-resident path: decode + preamble + rollup + vmb_rollup_aggr_partial in one call, decoded
 * columns cached in the library (per-rank step of `aggr(rollup(m[d])) by (...)`, eval.go:1804) */
int vmb_eval_rollup_aggr_device(vmb_ctx* ctx, const vmb_blocks* blocks, int64_t tr_min, int64_t tr_max,
                                const vmb_rollup_cfg* cfg, int aggr_id, const uint32_t* group_ids, uint32_t ngroups,
                                double* d_values, double* d_counts, uint64_t* samples_scanned);

/* ---- post-rollup operations on DEVICE matrices [series x points] (keep a query's intermediate results in HBM across the expression
 * tree) ------------------------------------------------------------------------------------------------------------------ */
enum vmb_binop { /* binary_op.go:15-43; the element functions of vendor/.../metricsql/binaryop/funcs.go */
    VMB_BO_PLUS = 0, VMB_BO_MINUS, VMB_BO_MUL, VMB_BO_DIV, VMB_BO_MOD, VMB_BO_POW, VMB_BO_ATAN2, VMB_BO_EQ, VMB_BO_NEQ, VMB_BO_GT,
    VMB_BO_LT, VMB_BO_GTE, VMB_BO_LTE, VMB_BO_DEFAULT, VMB_BO_IF, VMB_BO_IFNOT
};
/* newBinaryOpFunc binary_op.go:155-203: d_dst[i][j] = op(d_left[left_rows[i]][j], d_right[right_rows[i]][j]) for the npairs series
 * pairs the host matched by tag set (adjustBinaryOpTags :205).  left_rows / right_rows: HOST row indices or NULL = row i; a scalar
 * operand is a one-row matrix with all indices 0.  Comparisons: without is_bool they filter (left or NaN), with it they give 1 / 0
 * (NaN for a NaN left) -- newBinaryOpCmpFunc :132.  d_dst may alias d_left when left_rows is NULL. */
int vmb_binary_op(vmb_ctx* ctx, int op, int is_bool, const double* d_left, const uint32_t* left_rows, const double* d_right,
                  const uint32_t* right_rows, size_t npairs, size_t points, double* d_dst);
/* The set operators on top of it.  Their right-hand side is first reduced per tag-set group (createTimeseriesMapByTagSet binary_op.go:657
 * puts several series under one key): d_out[g][j] = the first non-NaN value among the rows with group_ids[row] == g at point j, in row
 * order, NaN when there is none -- all that addRightNaNsToLeft (:444), addLeftNaNsIfNoRightNaNs (:625) and fillLeftNaNsWithRightValues
 * (:516) read from tssRight.  Then, with right_rows[i] = the group of left row i:
 *   `and` (binaryOpAnd :430) / `if` = vmb_binary_op(VMB_BO_IF),  `unless` (:610) / `ifnot` = VMB_BO_IFNOT,  `default` = VMB_BO_DEFAULT;
 * left rows whose key has no right group are dropped (`and`) or kept as they are (`unless`, `default`) by the host's tag matching, which
 * also owns removeEmptySeries (exec.go:193).  `or` (:483) fills and clears by metric name instead: vmb_set_or. */
int vmb_group_first_value(vmb_ctx* ctx, const double* d_vals, size_t nseries, size_t points, const uint32_t* group_ids, uint32_t ngroups,
                          double* d_out);

/* Transform functions that only look at values (app/vmselect/promql/transform.go), in place on a DEVICE matrix [nrows x points]; labels,
 * sorting and the choice of series stay with the host.  Element functions (newTransformFuncOneArg :180 and friends) are applied to
 * every value, NaN included, like doTransformValues :195; row functions walk each series in point order like the reference (float
 * addition order is part of the result).  arg1 / arg2: HOST arrays of `points` values = getScalar of the scalar arguments:
 *   clamp(q, min, max): arg1 = min, arg2 = max;  clamp_min / clamp_max: arg1;  round(q, nearest): arg1 = nearest, arg2 =
 *   math.Pow10(-e) with (_, e) = decimal.FromFloat(nearest) (transform.go:2341; vmb_float_to_decimal gives e).
 *   smooth_exponential(q, sf): arg1 = sf (getScalar(args[1], 1)).  bitmap_and / or / xor(q, w): arg1 = w.  Others: NULL.
 * smooth_exponential (:1664): leading NaNs, then leading +-Infs are skipped (if nothing but +-Infs follows, nothing is cut); avg
 * starts at the first kept value, which stays as it is; later NaNs stay, a later +-Inf becomes the current avg, any other v
 * becomes avg = avg*(1-sf) + v*sf with sf = arg1 at the point's own index, NaN -> 1, clamped to [0, 1].
 * Date-time functions hour, minute, day_of_month, day_of_week, day_of_year, days_in_month, month, year (newTransformFuncDateTime
 * :333): a NaN stays as it is (:347); any other v becomes the field of time.Unix(int64(v), 0).UTC() as a double: hour = sod / 3600,
 * minute = sod / 60 % 60 with sod the second of the UTC day (floor semantics before 1970), day_of_week 0 = Sunday, day_of_year
 * 1..366, year astronomical (year 0 exists; negative years), days_in_month the reference's table with its leap test on
 * uint32(year) (:2874: February of year -100 has 29 days).  The zero-argument forms are these on time()'s one-row matrix.
 * Bitmap functions bitmap_and / or / xor(q, w) (newTransformBitmap :2724): NaN (math.NaN()) where v or w is NaN, else
 * float64(op(uint64(v), uint64(w))), rounded to nearest even.
 * Two Go-platform assumptions fix what Go leaves to the implementation, both unverified for want of a Go toolchain:
 *   - conversions as on amd64 at the default GOAMD64 level: int64(v) = trunc(v) for -2^63 <= v < 2^63, else -2^63 (+-Inf
 *     included; CVTTSD2SQ); uint64(v) = uint64(int64(v)) for v < 2^63 (-1.5 -> 2^64 - 1, -Inf -> 2^63), else
 *     uint64(int64(v - 2^63)) | 2^63 ([2^63, 2^64) exact, >= 2^64 and +Inf -> 2^63) -- ssagen's float64ToUint64;
 *   - Go 1.26's time arithmetic (the reference's go.mod): abs = uint64(s + 9223372028741760000) seconds since March 1 of year
 *     -292277022400 (absoluteYears), split in uint64.  For s >= -9223372028741760000 that is the proleptic Gregorian calendar
 *     (the verified domain: every int64 second but the lowest 8.1e9); below it, -2^63 included, the sum wraps and the fields
 *     follow Go's wrapped arithmetic (csrc/go_conv.cuh restates it).
 * exp / ln / log2 / log10 / trigonometric / hyperbolic functions are the CUDA math library's (<= 2 ulp from Go's); everything else is
 * bit-exact.  VMB_ERR_INVALID_ARG for ids 27..31, 47..63, >= 75 and for a missing argument array. */
enum vmb_transform_func {
    VMB_TF_ABS = 0, VMB_TF_CEIL, VMB_TF_FLOOR, VMB_TF_SQRT, VMB_TF_EXP, VMB_TF_LN, VMB_TF_LOG2, VMB_TF_LOG10, VMB_TF_SIN, VMB_TF_COS,
    VMB_TF_TAN, VMB_TF_ASIN, VMB_TF_ACOS, VMB_TF_ATAN, VMB_TF_SINH, VMB_TF_COSH, VMB_TF_TANH, VMB_TF_ASINH, VMB_TF_ACOSH, VMB_TF_ATANH,
    VMB_TF_DEG, VMB_TF_RAD, VMB_TF_SGN, VMB_TF_CLAMP, VMB_TF_CLAMP_MIN, VMB_TF_CLAMP_MAX, VMB_TF_ROUND,
    /* row functions: running_* (:1308), range_* = running + setLastValues (:1335, :1650), range_first / range_last (:1620, :1640),
     * keep_last_value / keep_next_value (:1214, :1237), remove_resets = removeCounterResetsMaybeNaNs (:2906) */
    VMB_TF_RUNNING_SUM = 32, VMB_TF_RUNNING_MIN, VMB_TF_RUNNING_MAX, VMB_TF_RUNNING_AVG, VMB_TF_RANGE_SUM, VMB_TF_RANGE_MIN,
    VMB_TF_RANGE_MAX, VMB_TF_RANGE_AVG, VMB_TF_RANGE_FIRST, VMB_TF_RANGE_LAST, VMB_TF_KEEP_LAST_VALUE, VMB_TF_KEEP_NEXT_VALUE,
    VMB_TF_REMOVE_RESETS, VMB_TF_INTERPOLATE /* :1261 */, VMB_TF_SMOOTH_EXPONENTIAL /* :1664 */,
    /* date-time (:1171 hour, :2314 minute, :2318 month, :2785 year, :360-376 the rest) and bitmap (:2710-2744) functions */
    VMB_TF_HOUR = 64, VMB_TF_MINUTE, VMB_TF_DAY_OF_MONTH, VMB_TF_DAY_OF_WEEK, VMB_TF_DAY_OF_YEAR, VMB_TF_DAYS_IN_MONTH, VMB_TF_MONTH,
    VMB_TF_YEAR, VMB_TF_BITMAP_AND, VMB_TF_BITMAP_OR, VMB_TF_BITMAP_XOR
};
int vmb_transform(vmb_ctx* ctx, int func, double* d_matrix, size_t nrows, size_t points, const double* arg1, const double* arg2);
/* The transforms that reduce a whole series and then rewrite it (app/vmselect/promql/transform.go), in place on a DEVICE matrix
 * [nrows x points], row by row.  args: HOST, the getScalar(...)[0] of the function's scalar argument as the host has it; the
 * library applies the reference's own math.Abs(z) and phi /= 2.
 *   STDDEV, STDVAR (:1550, :1566 -> rollup.go:1803,1808)  nargs 0.  Welford over the row, NaNs skipped; a one-point row is 0 (the
 *                 len(values) == 1 fast path counts NaNs), a row without a value NaN.  Every point, NaN ones included, gets it.
 *   ZSCORE (:1408)  nargs 0.  (v - avg) / stddev at every point, avg = mean() (:1425: sum / n over the non-NaN values, 0/0 for
 *                 none), not Welford's running mean.
 *   TRIM_ZSCORE (:1379)  nargs 1, args[0] = z.  NaN where |v - avg| / stddev > |z| (a NaN comparison trims nothing).
 *   NORMALIZE (:1347)  nargs 0.  vMin / vMax over the non-NaN values, d = vMax - vMin; a row where d is +-Inf (one without a value
 *                 included) is dropped by the reference: left as it is with row_kept[row] = 0.  Kept rows (row_kept 1) get
 *                 (v - vMin) / d at every point; such a row can be all NaN.  row_kept: HOST, nrows bytes, required here only.
 *   LINEAR_REGRESSION (:1513 -> rollup.go:1099)  nargs 1, args[0] = step in ms (a positive integer): the points' timestamps are
 *                 start + j*step and only t - t0 = j*step is read.  areConstValues (rollup.go:1137) on the raw row (any NaN makes
 *                 it non-constant unless points == 1), sums over the non-NaN values with dt = float64(j*step)/1e3, the 1e-6 tDiff
 *                 guard; every point gets v + k*float64(j*step)/1e3 in Go's order, without FMA.
 *   QUANTILE (:1582)  nargs 1, args[0] = phi.  quantileSorted (aggr.go:922) of the sorted non-NaN values goes to the last non-NaN
 *                 point, then setLastValues (:1650) fills the row with the last non-NaN value it then holds (a NaN result there
 *                 leaves the one before it, if any); phi < 0, > 1, NaN: -Inf, +Inf, NaN.  A row without a value stays as it is.
 *   MAD (:1534 -> rollup.go:1476)  nargs 0.  The median, then the median of |v - median| with NaNs dropped, at every point.
 *   TRIM_OUTLIERS (:1437)  nargs 1, args[0] = k.  NaN where |v - median| > k * mad.
 *   TRIM_SPIKES (:1465)  nargs 1, args[0] = phi.  phi /= 2; NaN where v > quantileSorted(1 - phi) or v < quantileSorted(phi) of
 *                 the sorted non-NaN values; NaN points stay, and an empty row or a NaN phi trims nothing.
 * Bit-exact except the sign of a zero QUANTILE result where a tied rank holds both -0.0 and +0.0 (the reference's sort is not
 * stable there either).  VMB_ERR_INVALID_ARG for an unknown func, a wrong nargs, a missing args or (NORMALIZE) row_kept, a step
 * that is not a positive integer (or puts (points - 1) * step past int64), or nrows / points > 2^31 - 1; VMB_ERR_NOMEM when the sort's scratch (at most 2 GiB of keys, or
 * two rows of them if one row needs more) cannot be had; the matrix is untouched in both cases.  nrows == 0 or points == 0: no-op. */
enum vmb_range_func { VMB_RS_STDDEV = 0, VMB_RS_STDVAR, VMB_RS_ZSCORE, VMB_RS_TRIM_ZSCORE, VMB_RS_NORMALIZE,
                      VMB_RS_LINEAR_REGRESSION, VMB_RS_QUANTILE, VMB_RS_MAD, VMB_RS_TRIM_OUTLIERS, VMB_RS_TRIM_SPIKES };
int vmb_transform_range(vmb_ctx* ctx, int func, double* d_matrix, size_t nrows, size_t points, const double* args, size_t nargs,
                        unsigned char* row_kept);
/* mergeSeries rollup_result_cache.go:618: d_dst[nrows x (pa + pb)], row i = d_a[a_rows[i]] ++ d_b[b_rows[i]]; a negative index
 * stands for a series missing on that side (NaNs, :677-690).  a_rows / b_rows: HOST, matched by metric name by the caller. */
int vmb_matrix_merge_rows(vmb_ctx* ctx, const double* d_a, const int64_t* a_rows, size_t pa, const double* d_b, const int64_t* b_rows,
                          size_t pb, size_t nrows, double* d_dst);
/* quantile(phi, q) by (...) / median(q) by (...)  aggr.go:1217-1240 newAggrQuantileFunc: d_out[ngroups x P], phis = one phi per
 * point (HOST).  Per (group, point) the NaNs are dropped and aggr.go:870 quantile applies; rank selection, quadratic in the group
 * size: groups of more than 2048 series return VMB_ERR_CAP. */
int vmb_aggr_quantile(vmb_ctx* ctx, const double* d_vals, size_t nseries, size_t points, const uint32_t* group_ids, uint32_t ngroups,
                      const double* phis, double* d_out);
/* aggr(q) by (...) for any argument q (aggrFuncExt aggr.go:110 with aggrFuncSum :185 ... aggrFuncZScore :493): the non-incremental
 * aggregates on a DEVICE matrix d_vals[nseries x P].  Not the ids of vmb_aggr_func: those are the incremental callbacks, whose sum
 * starts from the first value instead of 0 +.  group_ids: HOST, dense ids < ngroups.  Within a group the rows are folded in
 * ascending row order.  Rows without a non-NaN value belong to no group (removeEmptySeries :124), and a group left with one row
 * takes the reference's fast path: sum / avg / min / max / geomean return that row as it is, stddev / stdvar 0 where it has a value.
 *   d_out: [ngroups x P]; rows of groups without a non-empty row are NaN.  SHARE / ZSCORE: [nseries x P] instead, every row
 *   rewritten from its group's statistics; d_out may be d_vals.
 *   row_nonempty: HOST, nseries bytes, 1 where the row holds a non-NaN value (as in vmb_topk_apply); the host derives from it which
 *   groups exist, `limit N` (the first N groups in order of their first non-empty row) and which rows share / zscore return.
 * Bit-exact except geomean over two or more values (pow).  VMB_ERR_INVALID_ARG for an unknown func, ngroups == 0, a group id >=
 * ngroups or nseries / points > 2^31 - 1, with d_out untouched.  nseries == 0: d_out is NaN. */
enum vmb_matrix_aggr { VMB_MA_SUM = 0, VMB_MA_SUM2, VMB_MA_MIN, VMB_MA_MAX, VMB_MA_AVG, VMB_MA_COUNT, VMB_MA_GROUP,
                       VMB_MA_GEOMEAN, VMB_MA_STDDEV, VMB_MA_STDVAR, VMB_MA_SHARE, VMB_MA_ZSCORE };
int vmb_aggr_matrix(vmb_ctx* ctx, int func, const double* d_vals, size_t nseries, size_t points, const uint32_t* group_ids,
                    uint32_t ngroups, double* d_out, unsigned char* row_nonempty);
/* The order-statistic aggregates by (...) for any argument q, on a DEVICE matrix d_vals[nseries x P], with no cap on the group size:
 * quantiles (aggrFuncQuantiles aggr.go:1162), mad (:942), mode (:446), distinct (:423), outliers_iqr (:952), outliers_mad (:1004).
 * Each reads the sorted non-NaN values of every (group, point) cell.  group_ids, row_nonempty and the groups without a non-empty
 * row as in vmb_aggr_matrix; none of the six has a one-row fast path.  args: HOST.
 *   QUANTILES     args = nargs >= 1 phis; d_out [nargs x ngroups x P], phi-major (one [ngroups x P] matrix per phi)
 *   MAD, MODE, DISTINCT  nargs == 0; d_out [ngroups x P]
 *   OUTLIERS_IQR  nargs == 0; OUTLIERS_MAD: args = nargs == P tolerances, one per point.  d_out is not used (may be NULL);
 *                 row_selected: HOST, nseries bytes, 1 for a row with a point outside its cell's bounds.
 * Bit-exact except the sign of a zero quantiles / mode result where a tied rank holds both -0.0 and +0.0 (the reference's sort is
 * not stable there either).  VMB_ERR_INVALID_ARG for an unknown func, ngroups == 0, a group id >= ngroups, a wrong nargs, a missing
 * pointer or nseries / points > 2^31 - 1, with the outputs untouched; VMB_ERR_NOMEM when the scratch (at most 2 GiB of keys, or two
 * point columns of them if one column needs more) cannot be had.  nseries == 0: d_out is NaN. */
enum vmb_order_aggr { VMB_OA_QUANTILES = 0, VMB_OA_MAD, VMB_OA_MODE, VMB_OA_DISTINCT, VMB_OA_OUTLIERS_IQR, VMB_OA_OUTLIERS_MAD };
int vmb_aggr_order(vmb_ctx* ctx, int func, const double* d_vals, size_t nseries, size_t points, const uint32_t* group_ids,
                   uint32_t ngroups, const double* args, size_t nargs, double* d_out, unsigned char* row_nonempty,
                   unsigned char* row_selected);
/* The histogram functions over Prometheus `le` buckets (app/vmselect/promql/transform.go:634-1169) on a DEVICE matrix d_buckets
 * [nrows x P], one bucket series per row; read only, it must not overlap an output.  `vmrange` buckets go through
 * vmb_vmrange_to_le (below) first, as every histogram_* of the reference does (vmrangeBucketsToLE).
 *   group_ids: HOST, one per row, the dense id of the row's label set without `le` (groupLeTimeseries :1097); UINT32_MAX for a row
 *              without an `le` label or whose `le` does not parse (:1102, :1106): it belongs to no group.
 *   les:       HOST, one per row, the parsed `le`.
 *   args:      HOST.  QUANTILE: nargs = nphi x P, a block of P phis (getScalar) per phi: one phi is histogram_quantile, several are
 *              histogram_quantiles with d_out [nphi x ngroups x P], phi-major.  SHARE: nargs = P, one le per point.  FRACTION:
 *              nargs = 2P, the lower le of every point, then the upper.  AVG, STDDEV, STDVAR: nargs = 0.
 *   d_out:     [ngroups x P] (QUANTILE: [nphi x ngroups x P]).
 *   d_lower, d_upper: both or neither, QUANTILE with one phi and SHARE only: the boundsLabel series [ngroups x P] each
 *              (:1064-1086, :705-728).
 *   out_nonempty: HOST, one byte per output row -- the d_out rows, then the d_lower rows, then the d_upper rows --, 1 where the row
 *              holds a non-NaN value (removeEmptySeries exec.go:133).
 * Each group's rows are ordered as Go's sort.Slice(xss, xss[i].le < xss[j].le) orders up to 12 elements: a stable insertion sort,
 * a NaN le left where that loop leaves it; the library uses this order for every group size (for more than 12 rows with equal or
 * NaN le values Go's pdqsort may order them otherwise).  Per (group, point):
 *   QUANTILE, SHARE, FRACTION: mergeSameLE (:1151) sums consecutive equal le into the first in order, fixBrokenBuckets (:1122) turns a
 *     NaN first bucket into 0 and a NaN or smaller later one into the value before it (not for a single bucket), then the loops of
 *     :1010-1056 (vLast == 0 before the phi < 0 / > 1 checks, lastNonInf falling back to NaN), :661-697 and :759-795.
 *   AVG, STDDEV, STDVAR (:876-931): the raw rows in that order, +-Inf le skipped, weights v - vPrev, stdvar < 0 clamped to 0, stddev =
 *     sqrt(stdvar).
 * Bit-identical to the Go loops.  A group without rows is NaN.  The query errors of the reference (histogram_fraction's lower >= upper
 * :749) stay with the host.  VMB_ERR_INVALID_ARG for an unknown func, a wrong nargs, bounds on a function without them, a missing
 * pointer, a group id >= ngroups other than UINT32_MAX, or nrows / points > 2^31 - 1, with the outputs untouched.  nrows == 0,
 * points == 0 or ngroups == 0: no-op. */
enum vmb_hist_func { VMB_HF_QUANTILE = 0, VMB_HF_SHARE, VMB_HF_FRACTION, VMB_HF_AVG, VMB_HF_STDDEV, VMB_HF_STDVAR };
int vmb_histogram(vmb_ctx* ctx, int func, const double* d_buckets, size_t nrows, size_t points, const uint32_t* group_ids,
                  const double* les, uint32_t ngroups, const double* args, size_t nargs, double* d_out, double* d_lower,
                  double* d_upper, unsigned char* out_nonempty);
/* prometheus_buckets: vmrangeBucketsToLE (app/vmselect/promql/transform.go:494-632) on a DEVICE matrix d_buckets [nrows x P] of
 * VictoriaMetrics histogram buckets (`vmrange="<start>...<end>"`); read only, it must not overlap d_out.  Labels stay with the
 * host, which passes numbers and string ids:
 *   group_ids: HOST, one per row: the dense id (< ngroups) of the row's label set without `vmrange` and `le`; VMB_VR_KEEP for a row
 *              without `vmrange` but with a non-empty `le` (kept as it is, :510); UINT32_MAX for a row that is dropped: no
 *              `vmrange` and no `le`, no "..." in it, or a start or end that strconv.ParseFloat rejects (:517-530).
 *   starts, ends: HOST, one per row, the parsed start and end (read for grouped rows only).
 *   start_keys, end_keys: HOST, one per row, ids of the start and end STRINGS: equal strings, equal ids; different strings,
 *              different ids (the reference keys its maps by the strings, so `1e2` and `100` stay apart).
 *   d_out:     [*nout x P]: the kept rows in input order, then the groups in ascending id, each in the reference's output order.
 *   nout:      in: the capacity of d_out in rows; out: the rows needed.  d_out == NULL or too small: VMB_ERR_CAP, nothing else
 *              written (a first call with d_out == NULL sizes d_out exactly).
 *   out_src, out_kind, out_le: HOST, one per output row: the input row it comes from; enum vmb_vr_kind; the string id of its `le`
 *              (start key for a gap row, end key for a bucket row; UINT32_MAX for a kept row, whose own `le` stays, and for a
 *              +Inf row, whose `le` is "+Inf").
 * Per group, sorted by end (the order of hg_sort_rows: Go's sort.Slice for up to 12 rows; for more than 12 rows with equal or NaN
 * ends Go's pdqsort may order them otherwise), the rows are walked with the previous end starting at 0: a row without a value > 0
 * is skipped; a start != the previous end adds a zero gap row with le = start unless that string was seen (it then names the
 * source row, not the gap row); the row takes le = end, and an end string already seen merges the row into the row it names
 * (mergeNonOverlappingTimeseries binary_op.go:367: at most 2 overlapping points, P > 2) instead of being output; a +Inf row
 * follows unless the last end is +Inf.  Then every point runs count += v over the output rows, v > 0 and not NaN.  Bit-identical
 * to the reference.  VMB_ERR_INVALID_ARG for a missing pointer, a group id >= ngroups other than VMB_VR_KEEP / UINT32_MAX, or
 * nrows / points > 2^31 - 1, with the outputs untouched.  nrows == 0: *nout = 0. */
#define VMB_VR_KEEP 0xfffffffeu
enum vmb_vr_kind { VMB_VR_KEPT = 0, VMB_VR_BUCKET, VMB_VR_GAP, VMB_VR_INF };
int vmb_vmrange_to_le(vmb_ctx* ctx, const double* d_buckets, size_t nrows, size_t points, const uint32_t* group_ids,
                      const double* starts, const double* ends, const uint32_t* start_keys, const uint32_t* end_keys,
                      uint32_t ngroups, double* d_out, size_t* nout, uint32_t* out_src, unsigned char* out_kind,
                      uint32_t* out_le);
/* buckets_limit(limit, buckets) (transform.go:386-483) on a DEVICE `le` matrix d_buckets [nrows x P], usually the d_out of
 * vmb_vmrange_to_le in its order.  group_ids / les as in vmb_histogram: the dense id of the row's label set without `le`, UINT32_MAX
 * for a row without a parsable `le` (dropped, :418-427).  limit <= 0: no rows; limit < 3 counts as 3.  A group of at most limit
 * rows is kept in input order; a larger one is sorted by le (hg_sort_rows, as in vmb_histogram), every row gets hits = the sum
 * over the points, in order, of v - v(previous row) (0 before the first), and the adjacent pair with the fewest hits is merged
 * (the lower row dropped, its hits added to the next) until limit rows are left; the first and the last row stay.
 *   out_rows:  HOST, the kept rows, groups in ascending id.  nout: in: the capacity of out_rows; out: the rows kept
 *              (VMB_ERR_CAP when the capacity is too small; nrows always suffices).
 * No matrix is written: vmb_histogram over d_buckets with UINT32_MAX for the rows not kept is histogram_*(buckets_limit(...)).
 * Errors as vmb_vmrange_to_le. */
int vmb_buckets_limit(vmb_ctx* ctx, const double* d_buckets, size_t nrows, size_t points, const uint32_t* group_ids,
                      const double* les, uint32_t ngroups, int64_t limit, uint32_t* out_rows, size_t* nout);
/* The aggregates that rank whole series, on a DEVICE matrix d_vals [nseries x P]: topk_min / topk_max / topk_avg / topk_median /
 * topk_last(k, q [, "remaining_sum"]) by (...) and their bottomk_* twins (reverse != 0) (newAggrFuncRangeTopK aggr.go:677 ->
 * getRangeTopKTimeseries :704), and outliersk(k, q) by (...) (aggrFuncOutliersK :1040; reverse must be 0, d_remaining NULL).
 * group_ids: HOST, dense ids < ngroups.  Rows without a non-NaN value belong to no group (removeEmptySeries :124).  ks: HOST, one k
 * per point (getScalar); kn = getIntK(ks[p], n_g) (:793: NaN and negative are 0, truncation, at most the n_g rows of the group).
 *   score  MIN / MAX (:804, :818): the first value while that is NaN, then the smaller / larger non-NaN ones; AVG (:832): the sum of
 *          the non-NaN values in point order over their number; MEDIAN (:848): quantile(0.5) of the non-NaN values; LAST (:852): the
 *          last non-NaN value; OUTLIERSK (:1053): the sum over the points, in order and without FMA, of (v - median)^2, the median
 *          (:1066) taken per point over the group's rows -- a row with a NaN anywhere scores NaN.
 *   order  every group is ordered as a STABLE sort of its rows, in ascending row order, by lessWithNaNs (:1259; reverse:
 *          greaterWithNaNs :1270; a NaN score is the worst in both).  Both are strict weak orders, so this is what Go's sort.Slice
 *          returns for up to 12 rows (its insertion sort) and one of the outcomes of its unstable pdqsort beyond that; rows with
 *          distinct non-NaN scores are not affected.  -0.0 and +0.0 tie.
 *   mask   at point p every row but the kn best of its group becomes NaN (fillNaNsAtIdx :786).  A survivor is a row that then still
 *          holds a non-NaN value.  ONLY SURVIVORS ARE WRITTEN: every other row of d_vals -- one without a value, one outside the k
 *          best of every point, one that holds no value where it is among them -- keeps the bits it had, and is not in out_rows.
 *   d_remaining: DEVICE [ngroups x P] or NULL (no third argument): per (group, point) 0 + v + v ... over the non-NaN values of the
 *          rows outside the kn best, from the worst on, NaN for none (getRemainingSumTimeseries :751).  remaining_nonempty: HOST,
 *          ngroups bytes, required with d_remaining: 1 where the group's row holds a value.
 *   row_nonempty: HOST, nseries bytes, 1 where the row held a non-NaN value before the call (as in vmb_aggr_matrix: the host derives
 *          from it which groups exist and `limit N`).
 *   out_rows: HOST, capacity nseries: the survivors, groups in ascending id, each from best to worst (the reference's output order
 *          after reverseSeries :743).  out_counts: HOST, ngroups: the survivors of every group.  The host puts a group's
 *          remaining-sum row, where it holds a value, before the group's survivors, applies `limit N` and owns the labels.
 *   scores: HOST, nseries doubles, or NULL: the score of every row (one without a value: NaN).
 * Bit-exact except the sign of a zero MEDIAN score where a tied rank holds both -0.0 and +0.0 (the reference's sort is not stable
 * there either; the order of the rows does not depend on it).  VMB_ERR_INVALID_ARG for an unknown func, ngroups == 0, a group id
 * >= ngroups, a missing pointer, reverse or d_remaining with OUTLIERSK, or nseries / points > 2^31 - 1; VMB_ERR_NOMEM when the
 * scratch (MEDIAN: at most 2 GiB of keys, as vmb_transform_range) cannot be had; d_vals, d_remaining and the host outputs are
 * untouched in both cases.  nseries == 0 or points == 0: out_counts is zeroed, nothing else. */
enum vmb_rank_func { VMB_RK_MIN = 0, VMB_RK_MAX, VMB_RK_AVG, VMB_RK_MEDIAN, VMB_RK_LAST, VMB_RK_OUTLIERSK };
int vmb_aggr_rank(vmb_ctx* ctx, int func, int reverse, double* d_vals, size_t nseries, size_t points, const uint32_t* group_ids,
                  uint32_t ngroups, const double* ks, double* d_remaining, unsigned char* remaining_nonempty,
                  unsigned char* row_nonempty, uint32_t* out_rows, uint32_t* out_counts, double* scores);

/* count_values("label", q) by (...) (the afe closure of aggr.go:594) on a DEVICE matrix d_vals [nseries x P]; read only, it must
 * not overlap d_out.  Labels stay with the host, which gets back the exact double that names every output row and formats it
 * (strconv.FormatFloat(v, 'f', -1, 64)).
 *   group_ids: HOST, dense ids < ngroups, from the grouping after removing `label` from by (...) or adding it to without (...)
 *              (:576-592).  Within a group the rows are visited in ascending row order.
 *   Values:    NaN is skipped; values compare as Go's map[float64] compares them, so -0.0 and +0.0 are ONE key.  The zero row is
 *              named by the first zero in the reference's loop order (the group's rows in order, then the points): out_value is
 *              -0.0 exactly when that zero is -0.0.  Every other key has one bit pattern.
 *   d_out:     [*nout x P]: one row per (group, distinct value), groups ascending, then values ascending (the reference's order is a
 *              Go map's, so any fixed order is as good; this one is the same on every run).  A cell holds the number of the group's
 *              rows with that value at that point, NaN where it is 0.  Groups without a value have no rows.
 *   nout:      in: the capacity of d_out in rows; out: the rows needed.  d_out == NULL or too small: VMB_ERR_CAP, nothing else
 *              written (a first call with d_out == NULL sizes d_out exactly; the host compares the count with
 *              -search.maxSeriesPerAggrFunc, :603 / :639, before it allocates anything).
 *   out_group, out_value: HOST, one per output row: its group; the value that names it.
 * Bit-identical to the reference.  VMB_ERR_INVALID_ARG for ngroups == 0, a group id >= ngroups, a missing pointer, or nseries /
 * points > 2^31 - 1, with the outputs untouched; VMB_ERR_NOMEM when the scratch (the sort's as vmb_aggr_order, and 16 bytes per
 * non-NaN output cell) cannot be had, or for more than 2^32 - 1 non-NaN output cells.  nseries == 0 or points == 0: *nout = 0. */
int vmb_count_values(vmb_ctx* ctx, const double* d_vals, size_t nseries, size_t points, const uint32_t* group_ids, uint32_t ngroups,
                     double* d_out, size_t* nout, uint32_t* out_group, double* out_value);
/* count_values_over_time("label", m[d]) on a series batch: rollupConfig.DoTimeseriesMap (rollup.go:693) with newRollupCountValues
 * (:1490), the timeseriesMap path of eval.go:957 (subqueries) and :1860 (blocks).  The batch may come from vmb_decode_blocks,
 * vmb_series_from_host or vmb_series_from_matrix.  The series preamble runs in place as in vmb_rollup, from cfg->flags
 * (getRollupConfigs sets only VMB_RC_DROP_STALE_NANS for this function); cfg->func_id is not read.  Point p counts the rows
 * [i_p, j_p) of its window, by the rules of rollupConfig.doInternal (window 0, LookbackDelta, maxPrevInterval) that vmb_rollup uses.
 *   Keys:      the 'g' string of the value (strconv.FormatFloat(v, 'g', -1, 64)): every NaN is one key ("NaN"), -0.0 and +0.0 are
 *              two ("-0", "0"), every other key is the exact bits.  A value makes a row only if it lies in some window.
 *   d_out:     [*nout x P]: one row per (series, key), series ascending, then keys in the order of aggr_order.inc's keys (values
 *              ascending, -0.0 before +0.0, NaN last).  A cell holds the count of the key in that point's window, NaN where it is 0.
 *   out_series, out_value: HOST, one per output row: its series; the value that names it (Go's NaN bits for the NaN row).
 *   nout:      as in vmb_count_values.
 *   samples_scanned: HOST, may be NULL: what rollupConfig.Do reports, len(values) plus every window's length, summed over series.
 * Bit-identical to the reference.  Errors as vmb_count_values, plus the vmb_rollup_cfg checks of vmb_rollup (not the func_id). */
int vmb_rollup_count_values(vmb_ctx* ctx, vmb_series* series, const vmb_rollup_cfg* cfg, double* d_out, size_t* nout,
                            uint32_t* out_series, double* out_value, uint64_t* samples_scanned);

/* VictoriaMetrics' log-scale histogram buckets (metrics.Histogram.Update, vendor/github.com/VictoriaMetrics/metrics/histogram.go:88),
 * the buckets of histogram(q) and histogram_over_time(m[d]).
 *   Rule:      NaN and v < 0 are skipped: they count toward no bucket.  Otherwise bucketIdx = (Log10(v) + 9) * 18: < 0 is the
 *              lower bucket (0, -0.0, +-subnormals, everything below about 1e-9), >= 486 the upper bucket (+Inf included), else
 *              idx = (unsigned)bucketIdx, one less when bucketIdx is a whole number > 0 (10^n ends its bucket).
 *   Numbering: 0 the lower bucket "0...1.000e-09"; 1 + idx the decimal bucket idx; 487 the upper bucket "1.000e+18...+Inf".
 *   Labels:    no strings cross the ABI.  The label of decimal bucket idx is start + "..." + end as initBucketRanges (:220) builds
 *              them: v = Pow10(-9), start = %.3e of v; for each bucket v *= Pow(10, 1/18), end = %.3e of v, the next start = end.
 *   Log10:     Go's math.Log10 is Log(x) * (1/Ln10) with Log the fdlibm e_log.c algorithm of math/log.go; the library performs
 *              those IEEE operations in Go's order with explicit rounding, so its bucket is Go's bit for bit.  One assumption is
 *              not verified: that Go's amd64 assembly Log (log_amd64.s) gives the bits of the pure-Go code on every input (its
 *              differing steps are exact, and every subnormal falls in the lower bucket however it is reduced).
 *
 * histogram(q) by (...) (aggrFuncHistogram aggr.go:256) on a DEVICE matrix d_vals [nseries x P] (read only; it must not overlap
 * d_out), up to its final vmrangeBucketsToLE, which is vmb_vmrange_to_le on d_out.
 *   group_ids: HOST, dense ids < ngroups.
 *   d_out:     [*nout x P]: one row per (group, bucket hit at some point), groups ascending, then buckets ascending.  A cell holds
 *              the number of the group's rows in that bucket at that point, and 0 (not NaN) where there is none: the reference
 *              zero-fills a row when it creates it (:272-275).  A group whose rows hold only NaN or negative values has no rows.
 *   nout:      in: the capacity of d_out in rows; out: the rows needed.  d_out == NULL or too small: VMB_ERR_CAP, nothing else
 *              written (a first call with d_out == NULL sizes d_out exactly).
 *   out_group, out_bucket: HOST, one per output row: its group; its bucket number.
 * Bit-identical to the reference (counts are whole numbers, so the order of the additions does not matter).
 * VMB_ERR_INVALID_ARG for ngroups == 0, a group id >= ngroups, a missing pointer, or nseries / points > 2^31 - 1, with the outputs
 * untouched; VMB_ERR_NOMEM when the scratch (8 bytes per row and 128 per group) cannot be had, or for more than 2^32 - 1 output
 * rows.  nseries == 0 or points == 0: *nout = 0. */
int vmb_aggr_histogram(vmb_ctx* ctx, const double* d_vals, size_t nseries, size_t points, const uint32_t* group_ids,
                       uint32_t ngroups, double* d_out, size_t* nout, uint32_t* out_group, uint32_t* out_bucket);
/* histogram_over_time(m[d]) on a series batch: rollupConfig.DoTimeseriesMap (rollup.go:693) with rollupHistogram (:1526), the
 * path of vmb_rollup_count_values with the bucket of a sample as its key: the same batches, the same series preamble from
 * cfg->flags (getRollupConfigs sets only VMB_RC_DROP_STALE_NANS for this function; cfg->func_id is not read) and the same windows.
 *   d_out:     [*nout x P]: one row per (series, bucket that occurs in some point's window), series ascending, then buckets
 *              ascending.  A cell holds the count of the bucket in that point's window, NaN where it is 0 (the rows are copies of
 *              the origin, whose values are NaN).  A skipped sample (NaN, v < 0) makes no row and counts nowhere.
 *   out_series, out_bucket: HOST, one per output row: its series; its bucket number.
 *   nout, samples_scanned: as in vmb_rollup_count_values (skipped samples are scanned).
 * Bit-identical to the reference, under the assumption stated above.  Errors as vmb_rollup_count_values. */
int vmb_rollup_histogram(vmb_ctx* ctx, vmb_series* series, const vmb_rollup_cfg* cfg, double* d_out, size_t* nout,
                         uint32_t* out_series, uint32_t* out_bucket, uint64_t* samples_scanned);

/* removeEmptySeries (exec.go:193) on a DEVICE matrix d_vals [nrows x P], read only: flags (HOST, nrows bytes) = 1 where the row
 * holds a non-NaN value.  The host builds drop_empty_series (transform.go:1939), limit_offset (:2275) and union (:1725) on it and
 * on vmb_matrix_merge_rows.  VMB_ERR_INVALID_ARG for a missing pointer or nrows / points > 2^31 - 1, flags untouched.  points == 0:
 * every flag 0. */
int vmb_rows_nonempty(vmb_ctx* ctx, const double* d_vals, size_t nrows, size_t points, unsigned char* flags);
/* sort(q) / sort_desc(q) (newTransformFuncSort transform.go:2557) on a DEVICE matrix d_vals [nrows x P], read only.
 *   out_rows: HOST, nrows: the rows in output order; vmb_matrix_merge_rows with pb = 0 applies it.
 *   order    row a comes before row b at the highest point n where they differ, walking n = P - 1 down to 0: a row that is NaN where
 *            the other is not comes first in both directions; both NaN, or a == b (so -0.0 == +0.0), moves on to n - 1; otherwise
 *            a < b (desc != 0: b < a) decides.  +-Inf are ordinary values.  Rows equal at every point are equal.
 * This is a strict weak order, and the library returns its STABLE sort: equal rows keep ascending row order.  That is what Go's
 * sort.Slice returns for up to 12 rows (its insertion sort) and one of the outcomes of its unstable pdqsort beyond that; rows that
 * differ at some point are not affected.  VMB_ERR_INVALID_ARG for a missing pointer or nrows / points > 2^31 - 1; VMB_ERR_NOMEM when
 * the scratch (about 53 bytes per row) cannot be had; out_rows untouched in both cases.  nrows == 0: no-op; points == 0: the
 * identity. */
int vmb_sort_rows(vmb_ctx* ctx, const double* d_vals, size_t nrows, size_t points, int desc, uint32_t* out_rows);
/* `or` (binaryOpOr binary_op.go:483 with fillLeftNaNsWithRightValuesOrMerge :542), in place on two DEVICE matrices d_left [nleft x
 * P] and d_right [nright x P] (they must not overlap).  Labels stay with the host, which passes ids:
 *   left_keys, right_keys: HOST, dense ids < nkeys of every row's key (createTimeseriesMapByTagSet :657).
 *   left_names, right_names: HOST, ids of every row's marshalled sorted metric name: equal ids are names that can be merged.  The
 *            scalar fast path (:543) applies when a key's right side is one row with an empty name; its rows merge only if the
 *            key's non-empty left side is one unnamed row.  The host expresses that through the ids: it gives such a right row an id
 *            no left row has, unless the key's non-empty left side is a single unnamed row.
 * Per key and point, in the reference's order: the left rows without a non-NaN value (left_nonempty 0, removeEmptySeries :488,
 * taken before the fill) take no part.  For each other left row in row order, leftIsNaN is read once; then for each right row of
 * the key in row order, a right row with the same name fills a NaN left value with its current value (the last such row wins, and
 * a value an earlier left row has cleared is copied as NaN), and the right value becomes NaN if the left value is not NaN or the
 * names match.  Rows of keys without a non-empty left row, or without a right row, keep their bits.
 *   left_nonempty, right_nonempty: HOST, nleft / nright bytes: 1 where the row holds a non-NaN value, the left rows before the
 *            fill, the right rows after it.  The host keeps the left rows with a value, sorted by metric name, then per right key
 *            all its right rows if no left row has the key (an all-empty left side still has it), otherwise those still
 *            non-empty, sorted by metric name, and gathers the output with vmb_matrix_merge_rows.
 * Bit-identical to the reference (a cleared value is Go's NaN).  VMB_ERR_INVALID_ARG for a missing pointer, a key >= nkeys or
 * nleft / nright / points > 2^31 - 1; VMB_ERR_NOMEM when the scratch cannot be had; the matrices and the flags are untouched in
 * both cases.  points == 0: every flag 0. */
int vmb_set_or(vmb_ctx* ctx, double* d_left, size_t nleft, const uint32_t* left_keys, const uint32_t* left_names, double* d_right,
               size_t nright, const uint32_t* right_keys, const uint32_t* right_names, uint32_t nkeys, size_t points,
               unsigned char* left_nonempty, unsigned char* right_nonempty);

/* ---- multi-GPU: one process per GPU, the ONE exchange step of the path inside the library (SURVEY 8e) ------------------
 * aggr(rollup(m[d])) by (...): every rank folds its shard of the series into {values, counts}[G x P] (the per-worker
 * incrementalAggrContext, aggr_incremental.go:184), the partial states are merged by one ncclAllReduce per array -- the GPU
 * counterpart of the merge loop in finalizeTimeseries (aggr_incremental.go:141-168) -- and finalized on every rank.
 * NCCL is dlopen()ed ("libnccl.so.2", or $VMB_NCCL_LIB): no link-time dependency; in a process that already holds an NCCL it is
 * the same library instance.  Bootstrap: rank 0 calls vmb_comm_get_unique_id and hands the 128 bytes to the other ranks by any
 * means (the Go host: over vmselect's own RPC), then every rank calls vmb_ctx_comm_init; or vmb_ctx_comm_attach with an
 * ncclComm_t the host created itself.  Group ids must be assigned identically on all ranks. */
int vmb_comm_get_unique_id(uint8_t id[128]);                                  /* ncclGetUniqueId */
int vmb_ctx_comm_init(vmb_ctx* ctx, const uint8_t id[128], int nranks, int rank); /* ncclCommInitRank on the ctx's device */
int vmb_ctx_comm_attach(vmb_ctx* ctx, void* nccl_comm, int nranks, int rank);  /* the host's own ncclComm_t (not destroyed by the ctx) */
int vmb_ctx_comm_destroy(vmb_ctx* ctx);
int vmb_ctx_comm_size(const vmb_ctx* ctx);                                     /* 1 without a communicator */
int vmb_ctx_comm_rank(const vmb_ctx* ctx);
/* exchange step on DEVICE partial states, in place, on the ctx stream: identity into empty cells, all-reduce of the values with
 * the aggregate's operator (sum / min / max / prod) and of the counts with sum.  No-op without a communicator. */
int vmb_aggr_allreduce(vmb_ctx* ctx, int aggr_id, double* d_values, double* d_counts, size_t n);
/* topk(): candidate lists of all ranks side by side, d_parts[nranks x count] (input of vmb_topk_merge) -- ncclAllGather */
int vmb_topk_allgather(vmb_ctx* ctx, const double* d_cand, size_t count, double* d_parts);
/* the whole query step on every rank in one call: fold this rank's device-resident blocks, all-reduce, finalize;
 * out_host [ngroups x P] (may be NULL) receives the (identical on all ranks) result */
int vmb_eval_rollup_aggr_dist(vmb_ctx* ctx, const vmb_blocks* blocks, int64_t tr_min, int64_t tr_max, const vmb_rollup_cfg* cfg,
                              int aggr_id, const uint32_t* group_ids, uint32_t ngroups, double* out_host, uint64_t* samples_scanned);

/* pinned host memory helpers (cudaHostAlloc) for callers that want full PCIe speed */
void* vmb_host_alloc(size_t bytes);
void vmb_host_free(void* p);

/* timing hooks: elapsed device time (ms) of the named stage during the last batched call on this ctx;
 * stage: 0 = zstd, 1 = column decode, 2 = series preamble, 3 = rollup, 4 = aggregate, 5 = fused decode+rollup kernel
 * (with the fused kernel on, stage 1 is the whole un-fused sub-batch of the series it did not take, stages 2-3 are 0) */
float vmb_ctx_last_stage_ms(const vmb_ctx* ctx, int stage);
int vmb_ctx_enable_stage_timing(vmb_ctx* ctx, int enable);

#ifdef __cplusplus
}
#endif
#endif /* VMB200_H */
