// libvmb200: C ABI (include/vmb200.h), device memory management and kernel orchestration.
// Single translation unit: the kernel files are included below so that no relocatable device code is needed.
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "decode.cu"
#include "rollup.cu"
#include "fused.cu"
#include "zstd.cu"
#include "marshal.inc"
#include "encode.cu"

// ------------------------------------------------------------------------------------------------ errors
static thread_local char g_err[512];
void vmb_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
extern "C" const char* vmb_last_error(void) { return g_err; }
extern "C" int vmb_version(void) { return 100; }

#define CU(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) {                                                                   \
            vmb_set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
            return VMB_ERR_CUDA;                                                                   \
        }                                                                                          \
    } while (0)

struct DevBuf {  // grow-only device buffer
    void* p = nullptr;
    size_t cap = 0;
    int reserve(size_t bytes) {
        if (bytes <= cap) return 0;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        size_t want = bytes + (bytes >> 3) + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) {
            vmb_set_error("cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
            p = nullptr;
            return VMB_ERR_NOMEM;
        }
        cap = want;
        return 0;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
};

// Stages of vmb_ctx_last_stage_ms, numbered as in vmb200.h.  The un-fused path records ctx->ev[s] where stage s begins and
// ev[ST_FUSED] where the aggregate ends, so stage s spans ev[s] .. ev[s + 1]; eval_fused says which events it records.
enum Stage { ST_ZSTD, ST_DECODE, ST_PREAMBLE, ST_ROLLUP, ST_AGGR, ST_FUSED, ST__COUNT };

#define FUSED_CHUNKS_DEFAULT 4u /* eval_fused: chunks of the fused series list (VMB_FUSED_CHUNKS overrides) */
#define FUSED_CHUNKS_MAX 64u

struct vmb_ctx {
    int device = 0;
    cudaStream_t stream = 0;
    uint64_t launches = 0;
    bool timing = false;
    float stage_ms[ST__COUNT] = {};
    cudaEvent_t ev[ST__COUNT] = {};
    // scratch (reused across calls)
    DevBuf zseq;  // decoded zstd sequences (8 B each) between k_zstd_seq_decode and k_zstd_seq_exec
    DevBuf zscratch, zlit, zstatus, zjobs, zws, args1, args2, rolled, counters, tmp_out, grp, mheap, mnext;
    DevBuf bail, sub_arrays;  // fused path: series handed to the un-fused pipeline, and that sub-batch's arrays
    DevBuf enc_vals, enc_deltas, enc_out, enc_meta;  // vmb_marshal_columns_gpu
    DevBuf aggr_state, grp_ids;  // vmb_eval_rollup_aggr_dist: {values, counts}[G x P]; device copy of the per-series group ids
    // vmb_aggr_order / vmb_transform_range: a batch's keys, its merge buffer, per-cell (per-row) statistics, sort plan
    DevBuf oa_keys, oa_keys2, oa_cell, oa_meta;
    void* comm = nullptr;     // ncclComm_t (comm.inc); nullptr = single GPU
    bool comm_owned = false;
    int comm_ranks = 1, comm_rank = 0;
    bool fused = true;           // vmb_ctx_set_fused: series that qualify go through the fused decode+rollup kernel (fused.cu)
    // fused path: the series are cut into this many chunks; the zstd stage of chunk k + 1 runs on zstream beside the fused
    // kernel of chunk k (1 = zstd of the whole batch, then one fused launch)
    uint32_t fused_chunks = 0;  // 0: eval_fused's own choice (fused_chunks()); VMB_FUSED_CHUNKS sets it
    // CTAs per SM of the fused grid (<= FU_CTAS_PER_SM); 0 = FU_CTAS_PER_SM_OVERLAP when chunked, FU_CTAS_PER_SM otherwise
    uint32_t fused_ctas_per_sm = 0;
    cudaStream_t zstream = nullptr;               // created on first use, non-blocking
    std::vector<cudaEvent_t> zev;                 // zev[k]: the zstd stage of chunk k is done
    int64_t dedup_interval = 0;  // storage.SetDedupInterval (lib/storage/dedup.go:15), ms; 0 = deduplication off
    struct vmb_series* col_cache = nullptr;  // decoded columns of the one-call device paths, sized for the largest batch seen
    void* h_pinned = nullptr;  // small pinned staging area for counters
    void* pipe = nullptr;      // pipeline.inc: streams, events and double-buffered slots of vmb_eval_rollup_host
    void (*pipe_destroy)(void*) = nullptr;
};

struct vmb_blocks {
    vmb_ctx* ctx = nullptr;
    size_t nblocks = 0, nseries = 0;
    uint64_t rows = 0, compressed = 0, scratch_total = 0;
    uint64_t merge_rows = 0;  // rows of the series whose blocks overlap in time: size of the merge area behind the blocks
    uint64_t seq_total = 0;   // zstd sequences over all VMB_ZK_HUF columns (size of the record arena)
    bool needs_lit = false;
    uint32_t n_huf = 0, n_gen = 0, n_bad = 0;
    uint8_t* d_arrays = nullptr;          // the one allocation of the d_ arrays other than the payload (PlanArrays); nullptr in a view
    uint64_t* d_ser_merge_off = nullptr;  // per series: offset into the merge area, UINT64_MAX = none
    vmb_block_desc* d_descs = nullptr;
    uint8_t* d_payload = nullptr;        // = d_payload_alloc + 64
    uint8_t* d_payload_alloc = nullptr;
    ColInfo* d_cols = nullptr;
    uint64_t* d_row_off = nullptr;
    uint32_t* d_huf_list = nullptr;
    uint32_t* d_gen_list = nullptr;
    uint32_t* d_bad_list = nullptr;
    uint32_t* d_ser_first = nullptr;
    uint32_t* d_ser_nblocks = nullptr;
    // fused path (fused.cu): series the fused kernel may take (one block, delta-const timestamps at precisionBits 64, a known
    // values MarshalType), the others, and host copies of what a sub-batch for the un-fused pipeline is built from
    uint32_t* d_fused_list = nullptr;
    std::vector<uint32_t> h_fused, h_unfused, h_ser_first, h_ser_nblocks;
    // d_huf_list holds the columns no fused series reads first, then the values columns of h_fused in that order:
    // h_huf_upto[j] = where the entries of h_fused[j..] begin (size h_fused.size() + 1)
    std::vector<uint32_t> h_huf_upto;
    std::vector<vmb_block_desc> h_descs;
    std::vector<ColInfo> h_cols;
};

struct vmb_series {
    vmb_ctx* ctx = nullptr;
    size_t nseries = 0, nblocks = 0;
    uint64_t rows = 0;
    int64_t* d_ts = nullptr;
    double* d_vals = nullptr;
    SeriesMeta* d_meta = nullptr;
    uint32_t* d_blk_lo = nullptr;
    uint32_t* d_blk_hi = nullptr;
    int32_t* d_blk_status = nullptr;
    bool stale_dropped = false, resets_removed = false;
    uint32_t pre_applied = 0;  // VMB_RC_PRE_* already applied to the values (at most one of them, once)
    bool rolled = false;       // a rollup ran on this batch: its values were processed in place with the flags below
    uint32_t applied_mut = 0;  // VMB_RC_DROP_STALE_NANS | VMB_RC_REMOVE_COUNTER_RESETS of that first call
    int64_t applied_max_stale = 0;  // removeCounterResets' staleness interval of that call (rollup.go:380-387)
    bool values_are_int = false;
};

static inline void count_launch(vmb_ctx* c, int n = 1) { c->launches += (uint64_t)n; }
static inline size_t al16(size_t x) { return (x + 15) & ~(size_t)15; }

// ------------------------------------------------------------------------------------------------ context
extern "C" int vmb_ctx_create(int device, vmb_ctx** out) {
    if (!out) return VMB_ERR_INVALID_ARG;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        vmb_set_error("no CUDA device available (%s): libvmb200 has no CPU fallback", cudaGetErrorString(e));
        return VMB_ERR_CUDA;
    }
    if (device < 0 || device >= ndev) {
        vmb_set_error("device %d out of range (%d devices)", device, ndev);
        return VMB_ERR_INVALID_ARG;
    }
    CU(cudaSetDevice(device));
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {  // sm_90a code runs on compute capability 9.0 only
        vmb_set_error("device %d is sm_%d%d; libvmb200 is built for sm_90a (H100) only", device, prop.major, prop.minor);
        return VMB_ERR_CUDA;
    }
    vmb_ctx* c = new vmb_ctx();
    c->device = device;
    c->fused = getenv("VMB_NO_FUSED") == nullptr;  // A/B switches for profiles
    if (const char* s = getenv("VMB_FUSED_CHUNKS")) {
        const long v = atol(s);
        c->fused_chunks = v < 1 ? 1u : (v > (long)FUSED_CHUNKS_MAX ? FUSED_CHUNKS_MAX : (uint32_t)v);
    }
    if (const char* s = getenv("VMB_FUSED_CTAS_PER_SM")) {
        const long v = atol(s);
        c->fused_ctas_per_sm = v < 1 ? 1u : (v > FU_CTAS_PER_SM ? (uint32_t)FU_CTAS_PER_SM : (uint32_t)v);
    }
    for (cudaEvent_t& e : c->ev) CU(cudaEventCreate(&e));
    CU(cudaHostAlloc(&c->h_pinned, 4096, cudaHostAllocDefault));
    *out = c;
    return VMB_OK;
}
extern "C" void vmb_series_free(vmb_series* s);
extern "C" int vmb_ctx_comm_destroy(vmb_ctx* ctx);
extern "C" void vmb_ctx_destroy(vmb_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    vmb_ctx_comm_destroy(c);
    if (c->col_cache) vmb_series_free(c->col_cache);
    c->col_cache = nullptr;
    DevBuf* bufs[] = {&c->zscratch, &c->zlit, &c->zstatus, &c->zjobs, &c->zws, &c->args1, &c->args2, &c->rolled,
                      &c->counters, &c->tmp_out, &c->grp, &c->mheap, &c->mnext, &c->zseq, &c->bail, &c->sub_arrays, &c->aggr_state, &c->grp_ids, &c->enc_vals, &c->enc_deltas, &c->enc_out, &c->enc_meta,
                      &c->oa_keys, &c->oa_keys2, &c->oa_cell, &c->oa_meta};
    for (DevBuf* b : bufs) b->release();
    for (cudaEvent_t e : c->ev)
        if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : c->zev) cudaEventDestroy(e);
    if (c->zstream) cudaStreamDestroy(c->zstream);
    if (c->h_pinned) cudaFreeHost(c->h_pinned);
    if (c->pipe && c->pipe_destroy) c->pipe_destroy(c->pipe);
    delete c;
}
extern "C" int vmb_ctx_set_stream(vmb_ctx* c, void* stream) {
    if (!c) return VMB_ERR_INVALID_ARG;
    c->stream = (cudaStream_t)stream;
    return VMB_OK;
}
extern "C" int vmb_ctx_set_dedup_interval(vmb_ctx* c, int64_t interval_ms) {
    if (!c || interval_ms < 0) return VMB_ERR_INVALID_ARG;
    c->dedup_interval = interval_ms;
    return VMB_OK;
}
extern "C" int vmb_ctx_set_fused(vmb_ctx* c, int enable) {
    if (!c) return VMB_ERR_INVALID_ARG;
    c->fused = enable != 0;
    return VMB_OK;
}
extern "C" int vmb_ctx_synchronize(vmb_ctx* c) {
    if (!c) return VMB_ERR_INVALID_ARG;
    CU(cudaSetDevice(c->device));
    CU(cudaStreamSynchronize(c->stream));
    return VMB_OK;
}
extern "C" uint64_t vmb_ctx_launch_count(const vmb_ctx* c) { return c ? c->launches : 0; }
extern "C" float vmb_ctx_last_stage_ms(const vmb_ctx* c, int stage) {
    return (c && stage >= 0 && stage < ST__COUNT) ? c->stage_ms[stage] : 0.f;
}
extern "C" int vmb_ctx_enable_stage_timing(vmb_ctx* c, int enable) {
    if (!c) return VMB_ERR_INVALID_ARG;
    c->timing = enable != 0;
    return VMB_OK;
}
extern "C" void* vmb_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) return nullptr;
    return p;
}
extern "C" void vmb_host_free(void* p) {
    if (p) cudaFreeHost(p);
}

// ------------------------------------------------------------------------------------------------ block header
static inline uint64_t be_get(const uint8_t* s, int n) {
    uint64_t v = 0;
    for (int i = 0; i < n; i++) v = (v << 8) | s[i];
    return v;
}
extern "C" int vmb_block_desc_from_header(vmb_block_desc* d, const uint8_t h[81], uint8_t tsid_out[24]) {
    if (!d || !h) return VMB_ERR_INVALID_ARG;
    memset(d, 0, sizeof(*d));
    if (tsid_out) memcpy(tsid_out, h, 24);
    auto unzz = [](uint64_t u) { return (int64_t)(u >> 1) ^ -(int64_t)(u & 1); };  // int.go:79
    d->min_ts = unzz(be_get(h + 24, 8));
    d->max_ts = unzz(be_get(h + 32, 8));
    d->first_value = unzz(be_get(h + 40, 8));
    d->ts_off = be_get(h + 48, 8);
    d->val_off = be_get(h + 56, 8);
    d->ts_size = (uint32_t)be_get(h + 64, 4);
    d->val_size = (uint32_t)be_get(h + 68, 4);
    d->rows = (uint32_t)be_get(h + 72, 4);
    uint16_t u = (uint16_t)be_get(h + 76, 2);
    d->scale = (int16_t)((int16_t)(u >> 1) ^ (int16_t)(-(int16_t)(u & 1)));  // int.go:61
    d->ts_mt = h[78];
    d->val_mt = h[79];
    d->precision_bits = h[80];
    // blockHeader.validate block_header.go:230
    if (d->rows == 0 || d->rows > 16384) return VMB_ERR_ROWS;
    if (d->ts_mt > 6 || d->val_mt > 6) return VMB_ERR_MARSHAL_TYPE;
    if (d->precision_bits < 1 || d->precision_bits > 64) return VMB_ERR_INVALID_ARG;
    if (d->ts_size > 131072 || d->val_size > 131072) return VMB_ERR_INVALID_ARG;
    return VMB_OK;
}

static inline void be_put(uint8_t* d, uint64_t v, int n) {
    for (int i = 0; i < n; i++) d[i] = (uint8_t)(v >> (8 * (n - 1 - i)));
}
// blockHeader.Marshal block_header.go:104
extern "C" int vmb_block_header_marshal(uint8_t h[81], const vmb_block_desc* d, const uint8_t tsid[24]) {
    if (!h || !d) return VMB_ERR_INVALID_ARG;
    if (tsid) memcpy(h, tsid, 24);
    else memset(h, 0, 24);
    auto zz = [](int64_t v) { return (uint64_t)((v << 1) ^ (v >> 63)); };  // int.go:75
    be_put(h + 24, zz(d->min_ts), 8);
    be_put(h + 32, zz(d->max_ts), 8);
    be_put(h + 40, zz(d->first_value), 8);
    be_put(h + 48, d->ts_off, 8);
    be_put(h + 56, d->val_off, 8);
    be_put(h + 64, d->ts_size, 4);
    be_put(h + 68, d->val_size, 4);
    be_put(h + 72, d->rows, 4);
    be_put(h + 76, (uint16_t)((d->scale << 1) ^ (d->scale >> 15)), 2);  // int.go:57
    h[78] = d->ts_mt;
    h[79] = d->val_mt;
    h[80] = d->precision_bits;
    return VMB_OK;
}
// unmarshalBlockHeaders block_header.go:261: `count` headers back to back, sorted by TSID (TSID.Less tsid.go:89 == memcmp of
// the big-endian wire form)
extern "C" int vmb_index_block_unmarshal(vmb_block_desc* out, uint8_t* tsids, size_t count, const uint8_t* data, size_t len) {
    if (!out || !data || count == 0) return VMB_ERR_INVALID_ARG;
    if (len != count * 81) {
        vmb_set_error("invalid number of block headers found: %zu bytes; want %zu block headers", len, count);
        return len % 81 ? VMB_ERR_SHORT_SRC : VMB_ERR_ROWS;
    }
    for (size_t i = 0; i < count; i++) {
        int rc = vmb_block_desc_from_header(&out[i], data + i * 81, tsids ? tsids + i * 24 : nullptr);
        if (rc) {
            vmb_set_error("cannot unmarshal block header %zu: error %d", i, rc);
            return rc;
        }
        if (i && memcmp(data + (i - 1) * 81, data + i * 81, 24) > 0) {
            vmb_set_error("block headers must be sorted by tsid (header %zu)", i);
            return VMB_ERR_INVALID_ARG;
        }
    }
    return VMB_OK;
}
// metaindexRow.Unmarshal + unmarshalMetaindexRows metaindex_row.go:72 / :129 (on the decompressed bytes): 56-byte rows
extern "C" int vmb_metaindex_rows_unmarshal(vmb_metaindex_row* out, size_t cap, size_t* n_out, const uint8_t* data, size_t len) {
    if (!n_out || (len && !data)) return VMB_ERR_INVALID_ARG;
    *n_out = 0;
    if (len == 0) {
        vmb_set_error("expecting non-zero metaindex rows; got zero");
        return VMB_ERR_SHORT_SRC;
    }
    if (len % 56) {
        vmb_set_error("cannot unmarshal metaindexRow #%zu: %zu trailing bytes", len / 56, len % 56);
        return VMB_ERR_SHORT_SRC;
    }
    const size_t n = len / 56;
    *n_out = n;
    if (n > cap || !out) return VMB_ERR_CAP;
    auto unzz = [](uint64_t u) { return (int64_t)(u >> 1) ^ -(int64_t)(u & 1); };
    for (size_t i = 0; i < n; i++) {
        const uint8_t* r = data + i * 56;
        vmb_metaindex_row& m = out[i];
        memcpy(m.tsid, r, 24);
        m.block_headers_count = (uint32_t)be_get(r + 24, 4);
        m.min_ts = unzz(be_get(r + 28, 8));
        m.max_ts = unzz(be_get(r + 36, 8));
        m.index_block_offset = be_get(r + 44, 8);
        m.index_block_size = (uint32_t)be_get(r + 52, 4);
        if (m.block_headers_count == 0) {
            vmb_set_error("metaindexRow #%zu: BlockHeadersCount must be greater than 0", i);
            return VMB_ERR_ROWS;
        }
        if (m.index_block_size > 131072) {
            vmb_set_error("metaindexRow #%zu: too big IndexBlockSize %u", i, m.index_block_size);
            return VMB_ERR_INVALID_ARG;
        }
        if (i && memcmp(r - 56, r, 24) > 0) {
            vmb_set_error("metaindexRow values must be sorted by TSID (row %zu)", i);
            return VMB_ERR_INVALID_ARG;
        }
    }
    return VMB_OK;
}
extern "C" int vmb_metaindex_row_marshal(uint8_t out[56], const vmb_metaindex_row* m) {  // metaindex_row.go:61
    if (!out || !m) return VMB_ERR_INVALID_ARG;
    auto zz = [](int64_t v) { return (uint64_t)((v << 1) ^ (v >> 63)); };
    memcpy(out, m->tsid, 24);
    be_put(out + 24, m->block_headers_count, 4);
    be_put(out + 28, zz(m->min_ts), 8);
    be_put(out + 36, zz(m->max_ts), 8);
    be_put(out + 44, m->index_block_offset, 8);
    be_put(out + 52, m->index_block_size, 4);
    return VMB_OK;
}

// ------------------------------------------------------------------------------------------------ upload
template <class T>
static int dev_alloc(T** p, size_t n) {
    *p = nullptr;
    cudaError_t e = cudaMalloc((void**)p, (n ? n : 1) * sizeof(T));
    if (e != cudaSuccess) {
        vmb_set_error("cudaMalloc(%zu) failed: %s", n * sizeof(T), cudaGetErrorString(e));
        return VMB_ERR_NOMEM;
    }
    return 0;
}

extern "C" void vmb_blocks_free(vmb_blocks* b) {
    if (!b) return;
    if (b->ctx) cudaSetDevice(b->ctx->device);
    cudaFree(b->d_arrays);
    cudaFree(b->d_payload_alloc);
    delete b;
}
extern "C" size_t vmb_blocks_count(const vmb_blocks* b) { return b ? b->nblocks : 0; }
extern "C" uint64_t vmb_blocks_rows(const vmb_blocks* b) { return b ? b->rows : 0; }
extern "C" uint64_t vmb_blocks_compressed_bytes(const vmb_blocks* b) { return b ? b->compressed : 0; }

// host-side analysis shared by upload paths; fills the vectors
struct BlocksPlan {
    std::vector<ColInfo> cols;
    std::vector<uint64_t> row_off;
    std::vector<uint32_t> huf, gen, bad, ser_first, ser_nblocks, fused, unfused, huf_upto;
    std::vector<uint64_t> ser_merge_off;
    uint64_t rows = 0, compressed = 0, scratch_total = 0, merge_rows = 0, seq_total = 0;
    bool needs_lit = false;
    unsigned long long content_bound = 0;  // vmb_zstd_decompress_batch: cap on Frame_Content_Size instead of 10 bytes per row
};
// row layout of the decoded blocks, the series map and the merge area: needs the descriptors only
static void plan_layout(BlocksPlan& pl, const vmb_block_desc* descs, size_t nblocks) {
    pl.row_off.resize(nblocks + 1);
    pl.rows = 0;
    pl.ser_first.clear();
    pl.ser_nblocks.clear();
    for (size_t b = 0; b < nblocks; b++) {
        const vmb_block_desc& d = descs[b];
        pl.row_off[b] = pl.rows;
        pl.rows += d.rows <= 16384 ? d.rows : 0;  // invalid blocks get status VMB_ERR_ROWS in the kernel and occupy no rows
        if (b == 0 || d.series_idx != descs[b - 1].series_idx) {
            pl.ser_first.push_back((uint32_t)b);
            pl.ser_nblocks.push_back(1);
        } else {
            pl.ser_nblocks.back()++;
        }
    }
    pl.row_off[nblocks] = pl.rows;
    // Multi-block series (netstorage.go:566 mergeSortBlocks): lay the decoded blocks of a series out in min-timestamp order,
    // whatever order they arrived in.  When consecutive blocks are strictly disjoint in time the series is then the plain
    // concatenation of its blocks; otherwise (overlap, touching ranges, replicas) it is merged on the GPU into the merge
    // area behind the decoded blocks.
    pl.ser_merge_off.assign(pl.ser_first.size(), UINT64_MAX);
    pl.merge_rows = 0;
    std::vector<uint32_t> order;
    for (size_t s = 0; s < pl.ser_first.size(); s++) {
        const uint32_t fb = pl.ser_first[s], nb = pl.ser_nblocks[s];
        if (nb < 2) continue;
        order.resize(nb);
        for (uint32_t k = 0; k < nb; k++) order[k] = fb + k;
        std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return descs[a].min_ts < descs[b].min_ts; });
        uint64_t r = pl.row_off[fb], total = 0;
        bool overlap = false;
        for (uint32_t k = 0; k < nb; k++) {
            const vmb_block_desc& d = descs[order[k]];
            const uint64_t rows = d.rows <= 16384 ? d.rows : 0;
            pl.row_off[order[k]] = r + total;
            total += rows;
            if (k + 1 < nb && d.max_ts >= descs[order[k + 1]].min_ts) overlap = true;
        }
        if (overlap) {
            pl.ser_merge_off[s] = pl.merge_rows;
            pl.merge_rows += total;
        }
    }
}

static int plan_blocks(BlocksPlan& pl, const vmb_block_desc* descs, size_t nblocks, const uint8_t* payload, size_t payload_len) {
    pl.cols.resize(2 * nblocks);
    uint64_t scratch = 0;
    for (size_t b = 0; b < nblocks; b++) {
        const vmb_block_desc& d = descs[b];
        pl.compressed += (uint64_t)d.ts_size + d.val_size;
        if ((uint64_t)d.ts_off + d.ts_size > payload_len || (uint64_t)d.val_off + d.val_size > payload_len) {
            vmb_set_error("block %zu: payload range outside the arena (len %zu)", b, payload_len);
            return VMB_ERR_INVALID_ARG;
        }
        for (int which = 0; which < 2; which++) {
            ColInfo& ci = pl.cols[2 * b + which];
            memset(&ci, 0, sizeof(ci));
            int mt = which ? d.val_mt : d.ts_mt;
            if (mt != 1 && mt != 4) continue;
            const uint8_t* src = payload + (which ? d.val_off : d.ts_off);
            uint32_t len = which ? d.val_size : d.ts_size;
            uint32_t cs = 0;
            bool needs_lit = false;
            uint32_t nseq = 0;
            ci.kind = zstd_classify_host(src, len, d.rows <= 16384 ? d.rows : 0, &cs, &needs_lit, &nseq, pl.content_bound);
            if (ci.kind == VMB_ZK_HUF && nseq) {
                if (pl.seq_total + nseq > 0xffffffffull) {
                    vmb_set_error("more than 2^32 zstd sequences in one batch: split it");
                    return VMB_ERR_INVALID_ARG;
                }
                ci.nseq = nseq;
                ci.seq_rec_off = (uint32_t)pl.seq_total;
                pl.seq_total += nseq;
            }
            ci.content_size = cs;
            uint32_t col = (uint32_t)(2 * b + which);
            if (ci.kind == VMB_ZK_BAD) {
                pl.bad.push_back(col);
                continue;
            }
            ci.scratch_off = scratch;
            scratch += ((uint64_t)cs + 15) & ~(uint64_t)15;
            if (needs_lit) pl.needs_lit = true;
            if (ci.kind == VMB_ZK_HUF) pl.huf.push_back(col);
            else pl.gen.push_back(col);
        }
    }
    pl.scratch_total = scratch;
    plan_layout(pl, descs, nblocks);
    // series the fused kernel (fused.cu) may take: one block, timestamps MarshalTypeDeltaConst at precisionBits 64, a values
    // column it decodes; what it meets at run time beyond that (corrupt streams, staleness markers, ...) comes back on its bail list
    for (size_t s = 0; s < pl.ser_first.size(); s++) {
        const uint32_t fb = pl.ser_first[s];
        const vmb_block_desc& d = descs[fb];
        const bool ok = pl.ser_nblocks[s] == 1 && d.ts_mt == 2 && d.precision_bits >= 64 && d.rows >= 2 && d.rows <= 16384 &&
                        d.val_mt >= 1 && d.val_mt <= 6 && pl.cols[2 * fb + 1].kind != VMB_ZK_BAD;
        (ok ? pl.fused : pl.unfused).push_back((uint32_t)s);
    }
    // order the Huffman jobs by the fused series that reads them, so that the zstd stage of any run of consecutive fused
    // series is one range of the list (eval_fused's chunks); the order of the jobs changes no output
    std::vector<uint32_t> fpos(2 * nblocks, UINT32_MAX);
    for (size_t j = 0; j < pl.fused.size(); j++) fpos[2 * (size_t)pl.ser_first[pl.fused[j]] + 1] = (uint32_t)j;
    std::stable_sort(pl.huf.begin(), pl.huf.end(), [&](uint32_t a, uint32_t b) {
        return fpos[a] + 1u < fpos[b] + 1u;  // UINT32_MAX (read by no fused series) wraps to 0: first
    });
    pl.huf_upto.assign(pl.fused.size() + 1, (uint32_t)pl.huf.size());
    for (size_t i = pl.huf.size(); i-- > 0;) {
        const uint32_t j = fpos[pl.huf[i]];
        if (j == UINT32_MAX) break;
        pl.huf_upto[j] = (uint32_t)i;
    }
    for (size_t j = pl.fused.size(); j-- > 0;) pl.huf_upto[j] = std::min(pl.huf_upto[j], pl.huf_upto[j + 1]);
    return 0;
}

// The descriptors and the arrays of a BlocksPlan in one buffer (16-byte aligned, in this order), followed by up to three uint32
// arrays of the caller: packed on the host, copied to the device in one transfer and bound to a vmb_blocks there.
struct PlanArrays {
    size_t nblocks, descs, cols, row_off, huf, gen, bad, ser_first, ser_nblocks, ser_merge_off, extra[3], bytes;
    PlanArrays(const BlocksPlan& pl, size_t nb, size_t n_extra0 = 0, size_t n_extra1 = 0, size_t n_extra2 = 0) : nblocks(nb) {
        const size_t ns = pl.ser_first.size();
        size_t o = 0;
        auto take = [&](size_t n) {
            const size_t at = o;
            o = al16(o + n);
            return at;
        };
        descs = take(nb * sizeof(vmb_block_desc));
        cols = take(2 * nb * sizeof(ColInfo));
        row_off = take((nb + 1) * sizeof(uint64_t));
        huf = take(pl.huf.size() * 4);
        gen = take(pl.gen.size() * 4);
        bad = take(pl.bad.size() * 4);
        ser_first = take(ns * 4);
        ser_nblocks = take(ns * 4);
        ser_merge_off = take(ns * 8);
        extra[0] = take(n_extra0 * 4);
        extra[1] = take(n_extra1 * 4);
        extra[2] = take(n_extra2 * 4);
        bytes = o;
    }
    // d == nullptr: the caller writes the descriptors at h + descs itself
    void pack(uint8_t* h, const BlocksPlan& pl, const vmb_block_desc* d) const {
        auto put = [h](size_t at, const auto& v) {
            if (!v.empty()) memcpy(h + at, v.data(), v.size() * sizeof(v[0]));
        };
        if (d && nblocks) memcpy(h + descs, d, nblocks * sizeof(vmb_block_desc));
        put(cols, pl.cols);
        put(row_off, pl.row_off);
        put(huf, pl.huf);
        put(gen, pl.gen);
        put(bad, pl.bad);
        put(ser_first, pl.ser_first);
        put(ser_nblocks, pl.ser_nblocks);
        put(ser_merge_off, pl.ser_merge_off);
    }
    // sizes of `pl` and array pointers into the packed copy at d; the payload is the caller's
    void bind(vmb_blocks* b, uint8_t* d, const BlocksPlan& pl) const {
        b->nblocks = nblocks;
        b->nseries = pl.ser_first.size();
        b->rows = pl.rows;
        b->compressed = pl.compressed;
        b->scratch_total = pl.scratch_total;
        b->merge_rows = pl.merge_rows;
        b->seq_total = pl.seq_total;
        b->needs_lit = pl.needs_lit;
        b->n_huf = (uint32_t)pl.huf.size();
        b->n_gen = (uint32_t)pl.gen.size();
        b->n_bad = (uint32_t)pl.bad.size();
        b->d_descs = (vmb_block_desc*)(d + descs);
        b->d_cols = (ColInfo*)(d + cols);
        b->d_row_off = (uint64_t*)(d + row_off);
        b->d_huf_list = (uint32_t*)(d + huf);
        b->d_gen_list = (uint32_t*)(d + gen);
        b->d_bad_list = (uint32_t*)(d + bad);
        b->d_ser_first = (uint32_t*)(d + ser_first);
        b->d_ser_nblocks = (uint32_t*)(d + ser_nblocks);
        b->d_ser_merge_off = (uint64_t*)(d + ser_merge_off);
    }
    uint32_t* extra_at(uint8_t* base, int i) const { return (uint32_t*)(base + extra[i]); }
};

static int blocks_upload_impl(vmb_ctx* ctx, const vmb_block_desc* descs, size_t nblocks, const uint8_t* payload, size_t payload_len,
                              vmb_blocks** out, unsigned long long content_bound) {
    if (!ctx || !out || (nblocks && !descs) || (payload_len && !payload) || nblocks > 0x7fffffffu / 2) return VMB_ERR_INVALID_ARG;
    CU(cudaSetDevice(ctx->device));
    BlocksPlan pl;
    pl.content_bound = content_bound;
    int rc = plan_blocks(pl, descs, nblocks, payload, payload_len);
    if (rc) return rc;
    const PlanArrays L(pl, nblocks, pl.fused.size());
    std::vector<uint8_t> h(L.bytes);
    L.pack(h.data(), pl, descs);
    if (!pl.fused.empty()) memcpy(L.extra_at(h.data(), 0), pl.fused.data(), pl.fused.size() * 4);
    vmb_blocks* b = new vmb_blocks();
    b->ctx = ctx;
    // 64 bytes of slack on both sides of the payload: the bitstream windows of zstd.cu read up to 11 bytes before a stream's first byte
    rc = dev_alloc(&b->d_arrays, L.bytes);
    if (!rc) rc = dev_alloc(&b->d_payload_alloc, payload_len + 128);
    if (!rc) {
        L.bind(b, b->d_arrays, pl);
        b->d_fused_list = L.extra_at(b->d_arrays, 0);
        b->d_payload = b->d_payload_alloc + 64;
        cudaStream_t st = ctx->stream;
        cudaError_t e = cudaMemcpyAsync(b->d_arrays, h.data(), L.bytes, cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) e = cudaMemsetAsync(b->d_payload_alloc, 0, 64, st);
        if (e == cudaSuccess && payload_len) e = cudaMemcpyAsync(b->d_payload, payload, payload_len, cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) e = cudaMemsetAsync(b->d_payload + payload_len, 0, 64, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);  // `h` goes out of scope
        if (e != cudaSuccess) {
            vmb_set_error("uploading %zu blocks: %s", nblocks, cudaGetErrorString(e));
            rc = VMB_ERR_CUDA;
        }
    }
    if (rc) {
        vmb_blocks_free(b);
        return rc;
    }
    b->h_descs.assign(descs, descs + nblocks);
    b->h_cols = pl.cols;
    b->h_ser_first = pl.ser_first;
    b->h_ser_nblocks = pl.ser_nblocks;
    b->h_fused = pl.fused;
    b->h_unfused = pl.unfused;
    b->h_huf_upto = pl.huf_upto;
    *out = b;
    return VMB_OK;
}
extern "C" int vmb_blocks_upload(vmb_ctx* ctx, const vmb_block_desc* descs, size_t nblocks, const uint8_t* payload,
                                 size_t payload_len, vmb_blocks** out) {
    return blocks_upload_impl(ctx, descs, nblocks, payload, payload_len, out, 0);
}

// The feed of a query from a part on disk: what netstorage keeps per block in its tmpBlocksFile is the marshaled blockHeader
// (tmp_blocks_file.go:110 WriteBlockRefData; BlockRef.Init lib/storage/search.go:38 parses it back) and the block itself is
// read from the part's timestamps.bin / values.bin at the header's offsets (BlockRef.MustReadBlock search.go:73).  Here: all
// BlockRefs of a query at once -- the referenced byte ranges are gathered into one arena and go to the device in one copy.
extern "C" int vmb_blocks_upload_part(vmb_ctx* ctx, const uint8_t* headers, size_t nblocks, const uint8_t* timestamps_bin, size_t ts_len,
                                      const uint8_t* values_bin, size_t val_len, vmb_blocks** out) {
    if (!ctx || !out || (nblocks && !headers) || (ts_len && !timestamps_bin) || (val_len && !values_bin)) return VMB_ERR_INVALID_ARG;
    std::vector<vmb_block_desc> descs(nblocks);
    size_t total = 0;
    uint8_t prev_tsid[24], tsid[24];
    uint32_t series = 0;
    for (size_t i = 0; i < nblocks; i++) {
        vmb_block_desc& d = descs[i];
        int rc = vmb_block_desc_from_header(&d, headers + i * 81, tsid);
        if (rc) return rc;
        if (d.ts_off > ts_len || d.ts_size > ts_len - d.ts_off || d.val_off > val_len || d.val_size > val_len - d.val_off) {
            vmb_set_error("block %zu references bytes outside the part files (timestamps [%llu, +%u) of %zu, values [%llu, +%u) of %zu)", i,
                          (unsigned long long)d.ts_off, d.ts_size, ts_len, (unsigned long long)d.val_off, d.val_size, val_len);
            return VMB_ERR_SHORT_SRC;
        }
        // the blocks of one series are consecutive (netstorage.go:1414 groups the BlockRefs by metric name = by TSID)
        if (i && memcmp(tsid, prev_tsid, 24) != 0) series++;
        memcpy(prev_tsid, tsid, 24);
        d.series_idx = series;
        total += al16((size_t)d.ts_size) + al16((size_t)d.val_size);
    }
    std::vector<uint8_t> arena(total + 16);
    size_t pos = 0;
    for (size_t i = 0; i < nblocks; i++) {
        vmb_block_desc& d = descs[i];
        if (d.ts_size) memcpy(arena.data() + pos, timestamps_bin + d.ts_off, d.ts_size);
        d.ts_off = pos;
        pos += al16((size_t)d.ts_size);
        if (d.val_size) memcpy(arena.data() + pos, values_bin + d.val_off, d.val_size);
        d.val_off = pos;
        pos += al16((size_t)d.val_size);
    }
    return blocks_upload_impl(ctx, descs.data(), nblocks, arena.data(), pos, out, 0);
}

// ------------------------------------------------------------------------------------------------ series batches
extern "C" void vmb_series_free(vmb_series* s) {
    if (!s) return;
    if (s->ctx) cudaSetDevice(s->ctx->device);
    cudaFree(s->d_ts);
    cudaFree(s->d_vals);
    cudaFree(s->d_meta);
    cudaFree(s->d_blk_lo);
    cudaFree(s->d_blk_hi);
    cudaFree(s->d_blk_status);
    delete s;
}
extern "C" size_t vmb_series_count(const vmb_series* s) { return s ? s->nseries : 0; }
extern "C" uint64_t vmb_series_rows(const vmb_series* s) { return s ? s->rows : 0; }

__global__ void k_set_status(int32_t* status, const uint32_t* list, uint32_t n, int32_t v) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) status[list[i]] = v;
}

// the Huffman-literal frames d_huf_list[h0, h1) of `b` on stream st: headers, literals, sequences (Z as run_zstd set it up)
static void zstd_huf_range(vmb_ctx* ctx, const vmb_blocks* b, ZstdParams Z, uint32_t h0, uint32_t h1, cudaStream_t st) {
    if (h0 >= h1) return;
    Z.jobs = (HufJob*)ctx->zjobs.p + h0;
    Z.list = b->d_huf_list + h0;
    Z.count = h1 - h0;
    launch_zstd_prepare(Z, st);
    launch_huf_decode(Z, st);
    count_launch(ctx, 2);
    if (b->needs_lit) {
        launch_zstd_sequences(Z, st);
        count_launch(ctx, 2);
    }
}

// zstd stage: every compressed column of `b` is decompressed into ctx->zscratch (at ColInfo::scratch_off); per-column status
// in ctx->zstatus ([2 * nblocks] int32).  *d_zstatus_out = nullptr when the batch holds no zstd column.  With huf_end < n_huf
// only the Huffman frames d_huf_list[0, huf_end) are decoded here and *Zrest receives what zstd_huf_range needs for the others.
static int run_zstd(vmb_ctx* ctx, const vmb_blocks* b, int32_t** d_zstatus_out, uint32_t huf_end = UINT32_MAX,
                    ZstdParams* Zrest = nullptr) {
    cudaStream_t st = ctx->stream;
    *d_zstatus_out = nullptr;
    if (b->n_huf + b->n_gen + b->n_bad == 0) return VMB_OK;
    int rc;
    if ((rc = ctx->zscratch.reserve(b->scratch_total + 64))) return rc;
    if ((rc = ctx->zstatus.reserve(2 * b->nblocks * sizeof(int32_t)))) return rc;
    int32_t* d_zstatus = (int32_t*)ctx->zstatus.p;
    CU(cudaMemsetAsync(d_zstatus, 0, 2 * b->nblocks * sizeof(int32_t), st));
    if (b->needs_lit && (rc = ctx->zlit.reserve(b->scratch_total + 64))) return rc;
    ZstdParams Z;
    memset(&Z, 0, sizeof(Z));
    Z.descs = b->d_descs;
    Z.cols = b->d_cols;
    Z.payload = b->d_payload;
    Z.scratch = (uint8_t*)ctx->zscratch.p;
    Z.lit = b->needs_lit ? (uint8_t*)ctx->zlit.p : nullptr;
    if (b->seq_total) {
        if ((rc = ctx->zseq.reserve(b->seq_total * 8))) return rc;
        Z.seq_rec = (unsigned long long*)ctx->zseq.p;
    }
    Z.status = d_zstatus;
    if (b->n_bad) {
        k_set_status<<<(b->n_bad + 127) / 128, 128, 0, st>>>(d_zstatus, b->d_bad_list, b->n_bad, VMB_ERR_ZSTD);
        count_launch(ctx);
    }
    const uint32_t ws_threads = VMB_SMS * 2u * 32u;
    if (b->needs_lit || b->n_gen) {
        if ((rc = ctx->zws.reserve((size_t)ws_threads * zstd_serial_ws_bytes()))) return rc;
        Z.ws = ctx->zws.p;
        Z.ws_count = ws_threads;
    }
    if (b->n_huf && (rc = ctx->zjobs.reserve((size_t)b->n_huf * sizeof(HufJob)))) return rc;
    if (Zrest) *Zrest = Z;
    zstd_huf_range(ctx, b, Z, 0, std::min(huf_end, b->n_huf), st);
    if (b->n_gen) {
        Z.list = b->d_gen_list;
        Z.count = b->n_gen;
        launch_zstd_serial(Z, 1, st);
        count_launch(ctx);
    }
    *d_zstatus_out = d_zstatus;
    return VMB_OK;
}

// runs zstd + column decode + series assembly into `s` (whose buffers are already allocated)
// zstd_done: the zstd stage of the upload this (sub-)batch belongs to ran already, its status array is d_zstatus_in, its column
// infos (with the lengths the frames produced) d_zcols_in, and block k of `b` is block d_blk_map[k] of that upload
static int run_decode(vmb_ctx* ctx, const vmb_blocks* b, vmb_series* s, int64_t tr_min, int64_t tr_max, uint32_t flags,
                      unsigned int* d_failed, bool zstd_done = false, int32_t* d_zstatus_in = nullptr,
                      const uint32_t* d_blk_map = nullptr, const ColInfo* d_zcols_in = nullptr) {
    cudaStream_t st = ctx->stream;
    if (ctx->timing && !zstd_done) CU(cudaEventRecord(ctx->ev[ST_ZSTD], st));
    int32_t* d_zstatus = d_zstatus_in;
    if (!zstd_done) {
        int rc = run_zstd(ctx, b, &d_zstatus);
        if (rc) return rc;
    }
    if (ctx->timing && !zstd_done) CU(cudaEventRecord(ctx->ev[ST_DECODE], st));
    DecodeParams D;
    memset(&D, 0, sizeof(D));
    D.descs = b->d_descs;
    D.cols = b->d_cols;
    D.payload = b->d_payload;
    D.scratch = (const uint8_t*)ctx->zscratch.p;
    D.zstd_status = d_zstatus;
    D.zstd_cols = zstd_done ? d_zcols_in : b->d_cols;
    D.blk_map = d_blk_map;
    D.row_off = b->d_row_off;
    D.ts_out = s->d_ts;
    D.val_out = s->d_vals;
    D.blk_lo = s->d_blk_lo;
    D.blk_hi = s->d_blk_hi;
    D.status = s->d_blk_status;
    D.nblocks = (uint32_t)b->nblocks;
    D.flags = flags;
    D.tr_min = tr_min;
    D.tr_max = tr_max;
    launch_decode_columns(D, st);
    count_launch(ctx);
    RollupParams R;
    memset(&R, 0, sizeof(R));
    R.meta = s->d_meta;
    R.nseries = (uint32_t)s->nseries;
    R.ser_first_block = b->d_ser_first;
    R.ser_nblocks = b->d_ser_nblocks;
    R.row_off = b->d_row_off;
    R.blk_lo = s->d_blk_lo;
    R.blk_hi = s->d_blk_hi;
    R.descs = b->d_descs;
    R.blk_status = s->d_blk_status;
    R.failed_blocks = d_failed;
    R.ser_merge_off = b->d_ser_merge_off;
    R.rows_total = b->rows;
    R.ts = s->d_ts;
    R.vals = s->d_vals;
    R.dedup_interval = (flags & VMB_DECODE_VALUES_AS_INT64) ? 0 : ctx->dedup_interval;
    launch_series_assemble(R, st);
    count_launch(ctx);
    if (b->merge_rows) {
        if (flags & VMB_DECODE_VALUES_AS_INT64) {
            vmb_set_error("series with overlapping blocks cannot be assembled from VMB_DECODE_VALUES_AS_INT64 columns");
            return VMB_ERR_INVALID_ARG;
        }
        int rc;
        if ((rc = ctx->mheap.reserve(b->nblocks * sizeof(uint32_t)))) return rc;
        if ((rc = ctx->mnext.reserve(b->nblocks * sizeof(uint32_t)))) return rc;
        R.merge_heap = (uint32_t*)ctx->mheap.p;
        R.merge_next = (uint32_t*)ctx->mnext.p;
        launch_series_merge(R, st);
        count_launch(ctx);
    }
    if (R.dedup_interval > 0) {
        launch_series_dedup(R, st);
        count_launch(ctx);
    }
    if (ctx->timing && !zstd_done) CU(cudaEventRecord(ctx->ev[ST_PREAMBLE], st));
    CU(cudaGetLastError());
    return 0;
}

static int alloc_series_for(vmb_ctx* ctx, const vmb_blocks* b, vmb_series** out) {
    vmb_series* s = new vmb_series();
    s->ctx = ctx;
    s->nseries = b->nseries;
    s->nblocks = b->nblocks;
    s->rows = b->rows + b->merge_rows;  // decoded blocks, then the merge area
    int rc = 0;
    if (!rc) rc = dev_alloc(&s->d_ts, s->rows + 8);
    if (!rc) rc = dev_alloc(&s->d_vals, s->rows + 8);
    if (!rc) rc = dev_alloc(&s->d_meta, b->nseries);
    if (!rc) rc = dev_alloc(&s->d_blk_lo, b->nblocks);
    if (!rc) rc = dev_alloc(&s->d_blk_hi, b->nblocks);
    if (!rc) rc = dev_alloc(&s->d_blk_status, b->nblocks);
    if (rc) {
        vmb_series_free(s);
        return rc;
    }
    *out = s;
    return 0;
}

// stage_ms[stage] = time from ev[from] to ev[to]
static int stage_span(vmb_ctx* ctx, int stage, int from, int to) {
    float ms = 0;
    CU(cudaEventElapsedTime(&ms, ctx->ev[from], ctx->ev[to]));
    ctx->stage_ms[stage] = ms;
    return 0;
}
// the un-fused stages [first, end) of the last call
static void collect_stage_times(vmb_ctx* ctx, int first, int end) {
    if (ctx->timing)
        for (int s = first; s < end; s++) stage_span(ctx, s, s, s + 1);
}

// ------------------------------------------------------------------------------------------------ counters
// ctx->counters holds the counters of one call; the first 16 bytes are copied to the same offsets of ctx->h_pinned, which
// also takes the fused path's bail count
enum : size_t { PIN_FAILED = 0, PIN_SCANNED = 8, PIN_COUNTERS_BYTES = 16, PIN_BAIL = 64 };
struct Counters {
    unsigned int* d_failed;         // series whose blocks failed to decode
    unsigned long long* d_scanned;  // samplesScanned
};
static int counters_zero(vmb_ctx* ctx, cudaStream_t st, Counters* c) {
    int rc;
    if ((rc = ctx->counters.reserve(PIN_COUNTERS_BYTES))) return rc;
    c->d_failed = (unsigned int*)((char*)ctx->counters.p + PIN_FAILED);
    c->d_scanned = (unsigned long long*)((char*)ctx->counters.p + PIN_SCANNED);
    CU(cudaMemsetAsync(ctx->counters.p, 0, PIN_COUNTERS_BYTES, st));
    return 0;
}
// copies the counters back after the work queued on `st` and synchronises it
static int counters_read(vmb_ctx* ctx, cudaStream_t st, uint64_t* samples_scanned) {
    char* h = (char*)ctx->h_pinned;
    CU(cudaMemcpyAsync(h, ctx->counters.p, PIN_COUNTERS_BYTES, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (samples_scanned) *samples_scanned = *(unsigned long long*)(h + PIN_SCANNED);
    const unsigned int failed = *(unsigned int*)(h + PIN_FAILED);
    if (failed) {
        vmb_set_error("%u series hold blocks that failed to decode (see the per-block status)", failed);
        return VMB_ERR_BLOCK_FAILED;
    }
    return 0;
}

// CU() for code that owns a freshly allocated vmb_series `s` (and possibly a scratch device pointer): release before returning
#define CUS(call, extra)                                                                           \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) {                                                                   \
            vmb_set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
            vmb_series_free(s);                                                                    \
            cudaFree(extra);                                                                       \
            return VMB_ERR_CUDA;                                                                   \
        }                                                                                          \
    } while (0)

extern "C" int vmb_decode_blocks(vmb_ctx* ctx, const vmb_blocks* b, int64_t tr_min, int64_t tr_max, uint32_t flags,
                                 int32_t* block_status, vmb_series** out) {
    if (!ctx || !b || !out) return VMB_ERR_INVALID_ARG;
    CU(cudaSetDevice(ctx->device));
    vmb_series* s = nullptr;
    int rc = alloc_series_for(ctx, b, &s);
    if (rc) return rc;
    s->values_are_int = (flags & VMB_DECODE_VALUES_AS_INT64) != 0;
    Counters c;
    rc = counters_zero(ctx, ctx->stream, &c);
    if (!rc) rc = run_decode(ctx, b, s, tr_min, tr_max, flags, c.d_failed);
    if (!rc && block_status && b->nblocks)
        CUS(cudaMemcpyAsync(block_status, s->d_blk_status, b->nblocks * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream), nullptr);
    if (!rc) rc = counters_read(ctx, ctx->stream, nullptr);
    if (rc && rc != VMB_ERR_BLOCK_FAILED) {
        vmb_series_free(s);
        return rc;
    }
    collect_stage_times(ctx, ST_ZSTD, ST_PREAMBLE);
    *out = s;
    return rc;
}

__global__ void k_meta_from_offsets(SeriesMeta* meta, const uint64_t* offsets, uint32_t n) {
    uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    SeriesMeta m;
    m.start = offsets[s];
    m.n = (uint32_t)(offsets[s + 1] - offsets[s]);
    m.flags = VMB_SER_STALE | VMB_SER_DROP;  // host-built batch: staleness markers / value drops unknown => dropStaleNaNs and removeCounterResets scan
    m.max_prev_interval = 0;
    m.window = 0;
    meta[s] = m;
}

extern "C" int vmb_series_from_host(vmb_ctx* ctx, const int64_t* timestamps, const double* values, const uint64_t* offsets,
                                    size_t nseries, vmb_series** out) {
    if (!ctx || !out || !offsets || nseries > 0x7fffffffu) return VMB_ERR_INVALID_ARG;
    CU(cudaSetDevice(ctx->device));
    uint64_t rows = offsets[nseries];
    if (rows && (!timestamps || !values)) return VMB_ERR_INVALID_ARG;
    for (size_t i = 0; i < nseries; i++)
        if (offsets[i + 1] < offsets[i] || offsets[i + 1] - offsets[i] > 0xffffffffull) return VMB_ERR_INVALID_ARG;
    vmb_series* s = new vmb_series();
    s->ctx = ctx;
    s->nseries = nseries;
    s->rows = rows;
    int rc = 0;
    uint64_t* d_off = nullptr;
    if (!rc) rc = dev_alloc(&s->d_ts, rows + 8);
    if (!rc) rc = dev_alloc(&s->d_vals, rows + 8);
    if (!rc) rc = dev_alloc(&s->d_meta, nseries);
    if (!rc) rc = dev_alloc(&d_off, nseries + 1);
    if (rc) {
        vmb_series_free(s);
        cudaFree(d_off);
        return rc;
    }
    cudaStream_t st = ctx->stream;
    if (rows) {
        CUS(cudaMemcpyAsync(s->d_ts, timestamps, rows * 8, cudaMemcpyHostToDevice, st), d_off);
        CUS(cudaMemcpyAsync(s->d_vals, values, rows * 8, cudaMemcpyHostToDevice, st), d_off);
    }
    CUS(cudaMemcpyAsync(d_off, offsets, (nseries + 1) * 8, cudaMemcpyHostToDevice, st), d_off);
    if (nseries) {
        k_meta_from_offsets<<<(unsigned)((nseries + 127) / 128), 128, 0, st>>>(s->d_meta, d_off, (uint32_t)nseries);
        count_launch(ctx);
    }
    CUS(cudaStreamSynchronize(st), d_off);
    cudaFree(d_off);
    *out = s;
    return VMB_OK;
}

// removeNanValues (eval.go:1027) for every row of a DEVICE matrix at once: the feed of evalRollupFuncWithSubquery (eval.go:910), whose
// inner expression was evaluated on the shared grid start, start + step, ...: row s becomes a series of its non-NaN points with
// their grid timestamps (one warp per row, ballot compaction; capacity `points` rows per series)
__global__ void __launch_bounds__(128) k_series_from_matrix(const double* __restrict__ m, uint32_t nseries, uint32_t points, int64_t start,
                                                            int64_t step, int64_t* ts, double* vals, SeriesMeta* meta) {
    const int lane = threadIdx.x & 31;
    const uint32_t wpg = gridDim.x * (blockDim.x >> 5);
    for (uint32_t s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < nseries; s += wpg) {
        const double* row = m + (size_t)s * points;
        const size_t o0 = (size_t)s * points;
        uint32_t o = 0;
        for (uint32_t b = 0; b < points; b += 32) {
            const uint32_t i = b + lane;
            const double x = i < points ? row[i] : 0.0;
            const bool keep = i < points && !isnan(x);
            const uint32_t bal = __ballot_sync(0xffffffffu, keep);
            if (keep) {
                const uint32_t r = o + __popc(bal & ((1u << lane) - 1u));
                vals[o0 + r] = x;
                ts[o0 + r] = start + (int64_t)i * step;
            }
            o += __popc(bal);
        }
        if (lane == 0) {
            SeriesMeta mm;
            mm.start = o0;
            mm.n = o;
            mm.flags = VMB_SER_DROP;  // no staleness markers can be left (they are NaNs); value drops unknown => removeCounterResets scans
            mm.max_prev_interval = 0;
            mm.window = 0;
            meta[s] = mm;
        }
    }
}

extern "C" int vmb_series_from_matrix(vmb_ctx* ctx, const double* d_matrix, size_t nseries, size_t points, int64_t start, int64_t step,
                                      vmb_series** out) {
    if (!ctx || !out || (nseries && points && !d_matrix) || step <= 0 || nseries > 0x7fffffffu || points > 0x7fffffffu)
        return VMB_ERR_INVALID_ARG;
    CU(cudaSetDevice(ctx->device));
    vmb_series* s = new vmb_series();
    s->ctx = ctx;
    s->nseries = nseries;
    s->rows = (uint64_t)nseries * points;
    int rc = 0;
    if (!rc) rc = dev_alloc(&s->d_ts, s->rows + 8);
    if (!rc) rc = dev_alloc(&s->d_vals, s->rows + 8);
    if (!rc) rc = dev_alloc(&s->d_meta, nseries);
    if (rc) {
        vmb_series_free(s);
        return rc;
    }
    if (nseries) {
        uint32_t grid = (uint32_t)((nseries + 3) / 4);
        if (grid > VMB_SMS * 16u) grid = VMB_SMS * 16u;
        k_series_from_matrix<<<grid, 128, 0, ctx->stream>>>(d_matrix, (uint32_t)nseries, (uint32_t)points, start, step, s->d_ts, s->d_vals,
                                                           s->d_meta);
        count_launch(ctx);
    }
    CUS(cudaGetLastError(), nullptr);
    *out = s;
    return VMB_OK;
}

extern "C" int vmb_series_layout(vmb_ctx* ctx, const vmb_series* s, uint64_t* starts, uint32_t* counts) {
    if (!ctx || !s) return VMB_ERR_INVALID_ARG;
    CU(cudaSetDevice(ctx->device));
    std::vector<SeriesMeta> m(s->nseries);
    if (s->nseries) CU(cudaMemcpyAsync(m.data(), s->d_meta, s->nseries * sizeof(SeriesMeta), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    for (size_t i = 0; i < s->nseries; i++) {
        if (starts) starts[i] = m[i].start;
        if (counts) counts[i] = m[i].n;
    }
    return VMB_OK;
}

extern "C" int vmb_series_download(vmb_ctx* ctx, const vmb_series* s, int64_t* timestamps, double* values) {
    if (!ctx || !s) return VMB_ERR_INVALID_ARG;
    CU(cudaSetDevice(ctx->device));
    if (timestamps && s->rows) CU(cudaMemcpyAsync(timestamps, s->d_ts, s->rows * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (values && s->rows) CU(cudaMemcpyAsync(values, s->d_vals, s->rows * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return VMB_OK;
}

// ------------------------------------------------------------------------------------------------ per-call drop-ins
extern "C" int vmb_unmarshal_int64(vmb_ctx* ctx, int64_t* dst, size_t n, const uint8_t* src, size_t src_len, int mt,
                                   int64_t first_value) {
    if (!ctx || (n && !dst) || (src_len && !src)) return VMB_ERR_INVALID_ARG;
    if (n < 1 || n > 16384 || src_len > (1u << 20)) return VMB_ERR_INVALID_ARG;  // Go: Panicf("BUG: itemsCount ...")
    vmb_block_desc d;
    memset(&d, 0, sizeof(d));
    d.first_value = first_value;
    d.ts_mt = 3;  // constant timestamps column: no payload
    d.val_mt = (uint8_t)mt;
    d.val_off = 0;
    d.val_size = (uint32_t)src_len;
    d.rows = (uint32_t)n;
    d.precision_bits = 64;
    d.min_ts = 0;
    d.max_ts = 0;
    if (mt < 1 || mt > 6) return VMB_ERR_MARSHAL_TYPE;  // encoding.go:248
    vmb_blocks* b = nullptr;
    int rc = vmb_blocks_upload(ctx, &d, 1, src, src_len, &b);
    if (rc) return rc;
    vmb_series* s = nullptr;
    int32_t status = 0;
    rc = vmb_decode_blocks(ctx, b, INT64_MIN, INT64_MAX, VMB_DECODE_VALUES_AS_INT64, &status, &s);
    if (rc == VMB_OK || rc == VMB_ERR_BLOCK_FAILED) {
        if (status) rc = status;
        else {
            cudaError_t e = cudaMemcpy(dst, s->d_vals, n * 8, cudaMemcpyDeviceToHost);
            rc = e == cudaSuccess ? VMB_OK : VMB_ERR_CUDA;
        }
    }
    vmb_series_free(s);
    vmb_blocks_free(b);
    return rc;
}

extern "C" int vmb_decimal_to_float(vmb_ctx* ctx, double* dst, const int64_t* va, size_t n, int16_t e) {
    if (!ctx || (n && (!dst || !va))) return VMB_ERR_INVALID_ARG;
    if (!n) return VMB_OK;
    CU(cudaSetDevice(ctx->device));
    int rc;
    if ((rc = ctx->tmp_out.reserve(n * 16))) return rc;
    int64_t* d_in = (int64_t*)ctx->tmp_out.p;
    double* d_out = (double*)ctx->tmp_out.p + n;
    CU(cudaMemcpyAsync(d_in, va, n * 8, cudaMemcpyHostToDevice, ctx->stream));
    launch_decimal_to_float(d_out, d_in, n, e, ctx->stream);
    count_launch(ctx);
    CU(cudaMemcpyAsync(dst, d_out, n * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return VMB_OK;
}

extern "C" int vmb_marshal_int64(uint8_t* dst, size_t cap, size_t* out_len, int* out_mt, int64_t* out_first,
                                 const int64_t* vals, size_t n, uint8_t precision_bits) {
    if (!out_len || !out_mt || !out_first || !vals) return VMB_ERR_INVALID_ARG;
    std::vector<uint8_t> out;
    int rc = vmb_host::marshal_int64_array(out, out_mt, out_first, vals, n, precision_bits);
    if (rc) return rc;
    *out_len = out.size();
    if (out.size() > cap) return VMB_ERR_CAP;
    if (!out.empty()) memcpy(dst, out.data(), out.size());
    return VMB_OK;
}
extern "C" int vmb_float_to_decimal(int64_t* dst, int16_t* out_scale, const double* src, size_t n) {
    if (!out_scale || (n && (!dst || !src))) return VMB_ERR_INVALID_ARG;
    *out_scale = vmb_host::float_to_decimal(dst, src, n);
    return VMB_OK;
}
// exposed for tests: the library's own zstd writer
extern "C" int vmb_zstd_compress(uint8_t* dst, size_t cap, size_t* out_len, const uint8_t* src, size_t n) {
    if (!out_len || !src || n == 0) return VMB_ERR_INVALID_ARG;
    std::vector<uint8_t> out;
    vmb_host::zstd_compress_huf(out, src, n);
    *out_len = out.size();
    if (out.size() > cap) return VMB_ERR_CAP;
    memcpy(dst, out.data(), out.size());
    return VMB_OK;
}

extern "C" int vmb_calibrate_scale(int64_t* a, size_t na, int16_t ae, int64_t* b, size_t nb, int16_t be, int16_t* out_e) {
    if (!out_e || (na && !a) || (nb && !b)) return VMB_ERR_INVALID_ARG;
    *out_e = vmb_host::calibrate_scale(a, na, ae, b, nb, be);
    return VMB_OK;
}

// encoding.DecompressZSTD (compress.go:27) for a batch of frames, on the GPU.  Every frame travels as the values column of a
// pseudo block (MarshalTypeZSTDNearestDelta over the frame's bytes) through the same kernels as the block payloads; only the
// zstd stage runs.  Layout of dst: frame i at dst_offs[i] (16-byte aligned, in frame order), dst_lens[i] bytes.
static const uint32_t kZstdBatchRows = 16384;  // (pseudo blocks: the row count plays no role below)
// metaindex.bin is decompressed by the reference without a size limit (metaindex_row.go:134): the bound is the frame's own
// Frame_Content_Size under a sanity cap
static const unsigned long long kZstdBatchMaxContent = 1ull << 27;
extern "C" int vmb_zstd_decompress_bound(const uint8_t* frames, const uint64_t* offs, size_t n, uint64_t* out_bytes) {
    if (!out_bytes || (n && (!frames || !offs))) return VMB_ERR_INVALID_ARG;
    uint64_t tot = 0;
    for (size_t i = 0; i < n; i++) {
        if (offs[i + 1] < offs[i] || offs[i + 1] - offs[i] > 0xffffffffull) return VMB_ERR_INVALID_ARG;
        uint32_t cs = 0, nseq = 0;
        bool lit = false;
        const uint8_t kind = zstd_classify_host(frames + offs[i], (uint32_t)(offs[i + 1] - offs[i]), kZstdBatchRows, &cs, &lit, &nseq, kZstdBatchMaxContent);
        if (kind != VMB_ZK_BAD) tot += ((uint64_t)cs + 15) & ~(uint64_t)15;
    }
    *out_bytes = tot;
    return VMB_OK;
}
extern "C" int vmb_zstd_decompress_batch(vmb_ctx* ctx, const uint8_t* frames, const uint64_t* offs, size_t n, uint8_t* dst,
                                         size_t dst_cap, uint64_t* dst_offs, uint32_t* dst_lens, int32_t* statuses) {
    if (!ctx || !frames || !offs || !dst_offs || !dst_lens || n == 0 || n > 0x7fffffffull) return VMB_ERR_INVALID_ARG;
    CU(cudaSetDevice(ctx->device));
    std::vector<vmb_block_desc> descs(n);
    for (size_t i = 0; i < n; i++) {
        if (offs[i + 1] < offs[i] || offs[i + 1] - offs[i] > 0xffffffffull) return VMB_ERR_INVALID_ARG;
        vmb_block_desc& d = descs[i];
        memset(&d, 0, sizeof(d));
        d.ts_mt = 3;
        d.val_mt = 4;
        d.val_off = offs[i];
        d.val_size = (uint32_t)(offs[i + 1] - offs[i]);
        d.rows = kZstdBatchRows;
        d.precision_bits = 64;
        d.series_idx = (uint32_t)i;
    }
    vmb_blocks* b = nullptr;
    int rc = blocks_upload_impl(ctx, descs.data(), n, frames, (size_t)offs[n], &b, kZstdBatchMaxContent);
    if (rc) return rc;
    std::vector<ColInfo> cols(2 * n);
    std::vector<int32_t> st(2 * n, 0);
    int32_t* d_zstatus = nullptr;
    cudaError_t e = cudaSuccess;
    rc = run_zstd(ctx, b, &d_zstatus);
    if (rc == VMB_OK) {
        e = cudaMemcpyAsync(cols.data(), b->d_cols, cols.size() * sizeof(ColInfo), cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess && d_zstatus)
            e = cudaMemcpyAsync(st.data(), d_zstatus, st.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess && b->scratch_total) {
            if (b->scratch_total > dst_cap || !dst) rc = VMB_ERR_CAP;
            else e = cudaMemcpyAsync(dst, ctx->zscratch.p, b->scratch_total, cudaMemcpyDeviceToHost, ctx->stream);
        }
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) {
            vmb_set_error("vmb_zstd_decompress_batch: %s", cudaGetErrorString(e));
            rc = VMB_ERR_CUDA;
        }
    }
    vmb_blocks_free(b);
    if (rc) return rc;
    int bad = 0;
    for (size_t i = 0; i < n; i++) {
        const ColInfo& ci = cols[2 * i + 1];
        const int32_t s = st[2 * i + 1];
        dst_offs[i] = ci.scratch_off;
        dst_lens[i] = s ? 0u : ci.content_size;
        if (statuses) statuses[i] = s;
        bad += s != 0;
    }
    if (bad) {
        vmb_set_error("%d of %zu zstd frames failed to decompress", bad, n);
        return VMB_ERR_ZSTD;
    }
    return VMB_OK;
}

// ------------------------------------------------------------------------------------------------ rollup
extern "C" int64_t vmb_rollup_points(const vmb_rollup_cfg* cfg) {
    if (!cfg || cfg->step <= 0 || cfg->start > cfg->end) return -1;
    return 1 + (cfg->end - cfg->start) / cfg->step;
}

static int check_cfg(const vmb_rollup_cfg* cfg, int64_t* points) {
    // rollup.go:703-714: the Go code panics ("BUG: ...") on these
    if (!cfg || cfg->step <= 0 || cfg->start > cfg->end || cfg->window < 0 || cfg->func_id < 0 || cfg->func_id >= VMB_RF__COUNT) {
        vmb_set_error("invalid rollup config (step must be > 0, start <= end, window >= 0, known func_id)");
        return VMB_ERR_INVALID_ARG;
    }
    *points = 1 + (cfg->end - cfg->start) / cfg->step;
    if (*points > 0x7fffffff) return VMB_ERR_INVALID_ARG;
    // functions with a per-point argument (rollup.go: newRollupQuantile, newRollupPredictLinear, ... newRollupHoltWinters)
    if ((cfg->func_id == VMB_RF_QUANTILE || (cfg->func_id >= VMB_RF_PREDICT_LINEAR && cfg->func_id <= VMB_RF_SUM_EQ)) && !cfg->args) {
        vmb_set_error("rollup func %d needs cfg.args (one value per output point)", cfg->func_id);
        return VMB_ERR_INVALID_ARG;
    }
    if (cfg->func_id == VMB_RF_HOLT_WINTERS && (!cfg->args || !cfg->args2)) {
        vmb_set_error("holt_winters needs cfg.args (sf) and cfg.args2 (tf)");
        return VMB_ERR_INVALID_ARG;
    }
    return 0;
}

// series preamble + rollup into d_out (device). d_scanned: device u64 accumulator (already zeroed) or nullptr
// the per-point arguments of a rollup config, uploaded into the ctx: dev = *cfg with DEVICE args / args2
static int upload_cfg_args(vmb_ctx* ctx, const vmb_rollup_cfg* cfg, int64_t points, vmb_rollup_cfg* dev) {
    cudaStream_t st = ctx->stream;
    *dev = *cfg;
    dev->args = nullptr;
    dev->args2 = nullptr;
    int rc;
    if (cfg->args) {
        if ((rc = ctx->args1.reserve((size_t)points * 8))) return rc;
        CU(cudaMemcpyAsync(ctx->args1.p, cfg->args, (size_t)points * 8, cudaMemcpyHostToDevice, st));
        dev->args = (const double*)ctx->args1.p;
    }
    if (cfg->args2) {
        if ((rc = ctx->args2.reserve((size_t)points * 8))) return rc;
        CU(cudaMemcpyAsync(ctx->args2.p, cfg->args2, (size_t)points * 8, cudaMemcpyHostToDevice, st));
        dev->args2 = (const double*)ctx->args2.p;
    }
    return 0;
}

static int run_rollup(vmb_ctx* ctx, vmb_series* s, const vmb_rollup_cfg* cfg, int64_t points, double* d_out,
                      unsigned long long* d_scanned, const uint32_t* d_out_rows = nullptr, bool record_events = true) {
    cudaStream_t st = ctx->stream;
    RollupParams R;
    memset(&R, 0, sizeof(R));
    int rc;
    if ((rc = upload_cfg_args(ctx, cfg, points, &R.cfg))) return rc;
    R.out_rows = d_out_rows;
    R.meta = s->d_meta;
    R.ts = s->d_ts;
    R.vals = s->d_vals;
    R.out = d_out;
    R.scanned = d_scanned;
    R.nseries = (uint32_t)s->nseries;
    R.npoints = (uint32_t)points;
    // data-mutating parts of the preamble run once per batch; a later call must ask for the same mutations (the rows it would
    // read have been processed for the first one: dropStaleNaNs, removeCounterResets with its staleness interval)
    uint32_t flags = cfg->flags;
    {
        const uint32_t mut = flags & (VMB_RC_DROP_STALE_NANS | VMB_RC_REMOVE_COUNTER_RESETS);
        const int64_t max_stale = (flags & VMB_RC_REMOVE_COUNTER_RESETS) && cfg->lookback_delta != 0 ? cfg->lookback_delta + cfg->window : 0;
        if (s->rolled && (mut != s->applied_mut || max_stale != s->applied_max_stale)) {
            vmb_set_error("this batch was already rolled up with other in-place preprocessing (dropStaleNaNs / removeCounterResets / "
                          "staleness interval): decode it again");
            return VMB_ERR_INVALID_ARG;
        }
        s->rolled = true;
        s->applied_mut = mut;
        s->applied_max_stale = max_stale;
    }
    if (s->stale_dropped) flags &= ~VMB_RC_DROP_STALE_NANS;
    if (s->resets_removed) flags &= ~VMB_RC_REMOVE_COUNTER_RESETS;
    {
        const uint32_t pre = flags & VMB_RC_PRE_MASK;
        if (pre & (pre - 1)) {
            vmb_set_error("at most one value preFunc (VMB_RC_PRE_*) per rollup config");
            return VMB_ERR_INVALID_ARG;
        }
        if (s->pre_applied && pre != s->pre_applied) {
            vmb_set_error("this batch already went through another value preFunc: decode it again");
            return VMB_ERR_INVALID_ARG;
        }
        if (s->pre_applied) flags &= ~VMB_RC_PRE_MASK;
        else s->pre_applied = pre;
    }
    R.cfg.flags = flags;
    launch_series_prepare(R, st);
    count_launch(ctx);
    if (flags & VMB_RC_DROP_STALE_NANS) s->stale_dropped = true;
    if (flags & VMB_RC_REMOVE_COUNTER_RESETS) s->resets_removed = true;
    if (ctx->timing && record_events) CU(cudaEventRecord(ctx->ev[ST_ROLLUP], st));
    R.cfg.flags = cfg->flags;
    launch_rollup(R, st);
    count_launch(ctx);
    if (ctx->timing && record_events) CU(cudaEventRecord(ctx->ev[ST_AGGR], st));
    CU(cudaGetLastError());
    return 0;
}

extern "C" int vmb_rollup(vmb_ctx* ctx, vmb_series* s, const vmb_rollup_cfg* cfg, double* out, int out_is_device,
                          uint64_t* samples_scanned) {
    if (!ctx || !s || !out) return VMB_ERR_INVALID_ARG;
    if (s->values_are_int) {
        vmb_set_error("batch was decoded with VMB_DECODE_VALUES_AS_INT64");
        return VMB_ERR_INVALID_ARG;
    }
    int64_t points;
    int rc = check_cfg(cfg, &points);
    if (rc) return rc;
    CU(cudaSetDevice(ctx->device));
    size_t total = (size_t)s->nseries * (size_t)points;
    double* d_out = out;
    if (!out_is_device) {
        if ((rc = ctx->tmp_out.reserve(total * 8))) return rc;
        d_out = (double*)ctx->tmp_out.p;
    }
    Counters c;
    if ((rc = counters_zero(ctx, ctx->stream, &c))) return rc;
    if (ctx->timing) CU(cudaEventRecord(ctx->ev[ST_PREAMBLE], ctx->stream));
    if ((rc = run_rollup(ctx, s, cfg, points, d_out, c.d_scanned))) return rc;
    if (!out_is_device && total) CU(cudaMemcpyAsync(out, d_out, total * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if ((rc = counters_read(ctx, ctx->stream, samples_scanned))) return rc;
    collect_stage_times(ctx, ST_PREAMBLE, ST_AGGR);
    return VMB_OK;
}

// ------------------------------------------------------------------------------------------------ aggregates
// CSR of n series by group into caller memory: start[ngroups + 1], order[n] = the series of group g at start[g] ..
// start[g + 1], ascending (the fold order that keeps sum / avg reproducible bit for bit).  Series i of the batch is series
// sub[i] of group_ids (i itself without sub).
static int group_id_error(uint32_t g, size_t series, uint32_t ngroups) {
    vmb_set_error("group id %u of series %zu out of range (%u groups)", g, series, ngroups);
    return VMB_ERR_INVALID_ARG;
}
static int group_csr(const uint32_t* group_ids, const uint32_t* sub, size_t n, uint32_t ngroups, uint32_t* start, uint32_t* order) {
    memset(start, 0, ((size_t)ngroups + 1) * 4);
    for (size_t i = 0; i < n; i++) {
        const size_t s = sub ? sub[i] : i;
        if (group_ids[s] >= ngroups) return group_id_error(group_ids[s], s, ngroups);
        start[group_ids[s] + 1]++;
    }
    for (uint32_t g = 0; g < ngroups; g++) start[g + 1] += start[g];
    std::vector<uint32_t> cur(start, start + ngroups);
    for (size_t i = 0; i < n; i++) order[cur[group_ids[sub ? sub[i] : i]]++] = (uint32_t)i;
    return 0;
}
// group_csr into ctx->grp (start, order, then `extra` uint32 the caller fills); `h` holds the host copy and must live until the
// stream is synchronised
static int upload_group_csr(vmb_ctx* ctx, std::vector<uint32_t>& h, const uint32_t* group_ids, const uint32_t* sub, size_t n,
                            uint32_t ngroups, size_t extra, uint32_t** d_csr) {
    h.resize((size_t)ngroups + 1 + n);
    int rc = group_csr(group_ids, sub, n, ngroups, h.data(), h.data() + ngroups + 1);
    if (!rc) rc = ctx->grp.reserve((h.size() + extra) * sizeof(uint32_t));
    if (rc) return rc;
    *d_csr = (uint32_t*)ctx->grp.p;
    CU(cudaMemcpyAsync(*d_csr, h.data(), h.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    return 0;
}

// where an incremental aggregate (evalRollupWithIncrementalAggregate eval.go:1804) folds the rolled-up series: {values,
// counts}[G x P] in DEVICE memory, by the caller's per-series group ids (host)
struct AggrTarget {
    int aggr_id;
    const uint32_t* group_ids;
    uint32_t ngroups;
    double* d_values;
    double* d_counts;
};
static void launch_aggr_merge(vmb_ctx* ctx, cudaStream_t st, int aggr_id, double* dv, double* dc, const double* sv, const double* sc,
                              size_t n) {
    k_aggr_merge<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(aggr_id, dv, dc, sv, sc, n);
    count_launch(ctx);
}
// fold the rows `rolled` [series x P] by the group CSR d_csr (upload_group_csr) into t; with d_partial ({values, counts}, 2 x G x P
// scratch) the fold goes there and is merged into t, otherwise it overwrites t
static void aggr_fold(vmb_ctx* ctx, cudaStream_t st, const AggrTarget& t, const double* rolled, const uint32_t* d_csr, int64_t points,
                      double* d_partial) {
    const size_t cells = (size_t)t.ngroups * (size_t)points;
    AggrParams A;
    A.rolled = rolled;
    A.grp_start = d_csr;
    A.grp_series = d_csr + t.ngroups + 1;
    A.values = d_partial ? d_partial : t.d_values;
    A.counts = d_partial ? d_partial + cells : t.d_counts;
    A.ngroups = t.ngroups;
    A.npoints = (uint32_t)points;
    A.aggr = t.aggr_id;
    k_aggr_fold<<<(unsigned)((cells + 127) / 128), 128, 0, st>>>(A);
    count_launch(ctx);
    if (d_partial) launch_aggr_merge(ctx, st, t.aggr_id, t.d_values, t.d_counts, A.values, A.counts, cells);
}

extern "C" int vmb_rollup_aggr_partial(vmb_ctx* ctx, vmb_series* s, const vmb_rollup_cfg* cfg, int aggr_id,
                                       const uint32_t* group_ids, uint32_t ngroups, double* d_values, double* d_counts,
                                       double* d_rollup_scratch, uint64_t* samples_scanned) {
    if (!ctx || !s || !group_ids || !d_values || !d_counts || ngroups == 0 || aggr_id < 0 || aggr_id > VMB_AGGR_GROUP)
        return VMB_ERR_INVALID_ARG;
    int64_t points;
    int rc = check_cfg(cfg, &points);
    if (rc) return rc;
    CU(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    size_t total = (size_t)s->nseries * (size_t)points;
    double* d_rolled = d_rollup_scratch;
    if (!d_rolled) {
        if ((rc = ctx->rolled.reserve(total * 8))) return rc;
        d_rolled = (double*)ctx->rolled.p;
    }
    const AggrTarget t = {aggr_id, group_ids, ngroups, d_values, d_counts};
    std::vector<uint32_t> h_csr;
    uint32_t* d_csr;
    if ((rc = upload_group_csr(ctx, h_csr, group_ids, nullptr, s->nseries, ngroups, 0, &d_csr))) return rc;
    Counters c;
    if ((rc = counters_zero(ctx, st, &c))) return rc;
    if (ctx->timing) CU(cudaEventRecord(ctx->ev[ST_PREAMBLE], st));
    if ((rc = run_rollup(ctx, s, cfg, points, d_rolled, c.d_scanned))) return rc;
    aggr_fold(ctx, st, t, d_rolled, d_csr, points, nullptr);
    if (ctx->timing) CU(cudaEventRecord(ctx->ev[ST_FUSED], st));
    if ((rc = counters_read(ctx, st, samples_scanned))) return rc;  // synchronises: `h_csr` goes out of scope
    collect_stage_times(ctx, ST_PREAMBLE, ST_FUSED);
    return VMB_OK;
}

extern "C" int vmb_aggr_merge(vmb_ctx* ctx, int aggr_id, double* dv, double* dc, const double* sv, const double* sc, size_t n) {
    if (!ctx || !dv || !dc || !sv || !sc) return VMB_ERR_INVALID_ARG;
    CU(cudaSetDevice(ctx->device));
    if (n) launch_aggr_merge(ctx, ctx->stream, aggr_id, dv, dc, sv, sc, n);
    CU(cudaGetLastError());
    return VMB_OK;
}
extern "C" int vmb_aggr_prepare_allreduce(vmb_ctx* ctx, int aggr_id, double* dv, const double* dc, size_t n) {
    if (!ctx || !dv || !dc) return VMB_ERR_INVALID_ARG;
    CU(cudaSetDevice(ctx->device));
    if (n) {
        k_aggr_prepare_allreduce<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(aggr_id, dv, dc, n);
        count_launch(ctx);
    }
    CU(cudaGetLastError());
    return VMB_OK;
}
extern "C" int vmb_aggr_finalize(vmb_ctx* ctx, int aggr_id, double* dv, const double* dc, size_t n, double* out_host) {
    if (!ctx || !dv || !dc) return VMB_ERR_INVALID_ARG;
    CU(cudaSetDevice(ctx->device));
    if (n) {
        k_aggr_finalize<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(aggr_id, dv, dc, n);
        count_launch(ctx);
        if (out_host) CU(cudaMemcpyAsync(out_host, dv, n * 8, cudaMemcpyDeviceToHost, ctx->stream));
    }
    CU(cudaStreamSynchronize(ctx->stream));
    return VMB_OK;
}

// ------------------------------------------------------------------------------------------------ whole path
// *view = the decoded columns of the one-call device paths, sized to `b`, with no preprocessing applied yet.  The columns are
// owned by the ctx and grown to the largest batch seen.
static int column_cache_view(vmb_ctx* ctx, const vmb_blocks* b, vmb_series* view) {
    vmb_series* c = ctx->col_cache;
    if (c && (c->rows < b->rows + b->merge_rows || c->nseries < b->nseries || c->nblocks < b->nblocks)) {
        vmb_series_free(c);
        ctx->col_cache = c = nullptr;
    }
    if (!c) {
        int rc = alloc_series_for(ctx, b, &c);
        if (rc) return rc;
        ctx->col_cache = c;
    }
    *view = *c;
    view->nseries = b->nseries;
    view->nblocks = b->nblocks;
    view->rows = b->rows + b->merge_rows;
    view->stale_dropped = view->resets_removed = view->rolled = false;
    view->pre_applied = 0;
    return 0;
}

// ---- fused path (fused.cu): zstd stage, then ONE kernel per series batch that decodes into shared memory and rolls up; the series
// it hands back (bail list) and the ones it never takes (multi-block series, other timestamp encodings) go through the un-fused
// pipeline as a sub-batch that writes the same output rows.
static const size_t FUSED_SMEM = (sizeof(FusedSmem) + 15) & ~(size_t)15;
// persistent grid of one instantiation: VMB_SMS x the CTAs per SM the occupancy calculator allows, at most FU_CTAS_PER_SM
// (eval_fused's tmp_out holds one row per CTA of that many)
template <typename K>
static uint32_t fused_grid(K kernel) {
    int blocks_per_sm = 0;
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FUSED_SMEM);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, kernel, FU_THREADS, FUSED_SMEM) != cudaSuccess || blocks_per_sm < 1)
        blocks_per_sm = 1;
    if (blocks_per_sm > FU_CTAS_PER_SM) blocks_per_sm = FU_CTAS_PER_SM;
    return VMB_SMS * (uint32_t)blocks_per_sm;
}

extern "C" int vmb_fused_grid(void) {
    static const uint32_t grid = fused_grid(k_fused_rollup<VMB_RF_RATE>);
    return (int)grid;
}
extern "C" int vmb_fused_grid_chunked(void) {
    return (int)std::min<uint32_t>((uint32_t)vmb_fused_grid(), VMB_SMS * FU_CTAS_PER_SM_OVERLAP);
}

// CTAs per SM of the fused grid of a call cut into C chunks: FU_CTAS_PER_SM, or FU_CTAS_PER_SM_OVERLAP for rate() beside the
// zstd stage of the next chunk (VMB_FUSED_CTAS_PER_SM overrides both, for measurements)
// chunks of a fused call: FUSED_CHUNKS_DEFAULT when the zstd stage of chunks 1.. has Huffman frames to hide under the fused
// kernel, else 1 (nothing to overlap: the 5-CTA one-shot schedule)
static uint32_t fused_chunks(const vmb_ctx* ctx, const vmb_blocks* b) {
    const size_t nf = b->h_fused.size();
    uint32_t C = ctx->fused_chunks ? ctx->fused_chunks : FUSED_CHUNKS_DEFAULT;
    if (C > nf) C = (uint32_t)nf;
    if (C <= 1 || b->n_huf == 0) return 1;
    return b->h_huf_upto[nf / C] < b->n_huf ? C : 1u;
}

static uint32_t fused_ctas_per_sm(const vmb_ctx* ctx, uint32_t C, const vmb_rollup_cfg* cfg) {
    if (ctx->fused_ctas_per_sm) return ctx->fused_ctas_per_sm;
    // rate()'s fused kernel costs about as much as the zstd stage: giving up a fused CTA per SM to the Huffman kernel pays.  The
    // heavier functions (avg / max / quantile_over_time: 2-3.5x the zstd stage) lose more on the fused side than the overlap gains
    // and keep 5; their chunks still overlap where fused CTAs leave room (DESIGN.md section 8)
    return C > 1 && cfg->func_id == VMB_RF_RATE ? FU_CTAS_PER_SM_OVERLAP : FU_CTAS_PER_SM;
}

// ctas_per_sm (<= FU_CTAS_PER_SM) caps the grid below what the occupancy calculator allows
static void launch_fused(const FusedParams& P, uint32_t ctas_per_sm, cudaStream_t st) {
    if (!P.nlist) return;
    const size_t smem0 = FUSED_SMEM;
#define FUSED_LAUNCH(KERNEL, SMEM)                                                                                \
    do {                                                                                                          \
        static const uint32_t grid0 = fused_grid(KERNEL);                                                         \
        uint32_t grid = std::min(grid0, VMB_SMS * ctas_per_sm);                                                   \
        if (grid > P.nlist) grid = P.nlist;                                                                       \
        KERNEL<<<grid, FU_THREADS, (SMEM), st>>>(P);                                                              \
    } while (0)
    switch (P.cfg.func_id) {  // the value-only functions of BASELINE.json's configs get their own instantiation
#define FUSED_CASE(F) case F: FUSED_LAUNCH((k_fused_rollup<F>), smem0); break;
        FUSED_CASE(VMB_RF_RATE)
        FUSED_CASE(VMB_RF_DELTA)
        FUSED_CASE(VMB_RF_AVG)
        FUSED_CASE(VMB_RF_MIN)
        FUSED_CASE(VMB_RF_MAX)
        FUSED_CASE(VMB_RF_SUM)
        FUSED_CASE(VMB_RF_COUNT)
        FUSED_CASE(VMB_RF_QUANTILE)
        FUSED_CASE(VMB_RF_DEFAULT_ROLLUP)
        // the next most common dashboard functions: a lean instantiation instead of the all-functions one (which spills)
        FUSED_CASE(VMB_RF_IDERIV)
        FUSED_CASE(VMB_RF_IDELTA)
        FUSED_CASE(VMB_RF_LAST)
        FUSED_CASE(VMB_RF_FIRST)
        FUSED_CASE(VMB_RF_STDDEV)
        FUSED_CASE(VMB_RF_STDVAR)
        FUSED_CASE(VMB_RF_CHANGES)
        FUSED_CASE(VMB_RF_DERIV)
#undef FUSED_CASE
        default: FUSED_LAUNCH((k_fused_rollup<-1>), smem0); break;
    }
#undef FUSED_LAUNCH
}

static bool fused_enabled(const vmb_ctx* ctx, const vmb_blocks* b, const vmb_rollup_cfg* cfg) {
    return ctx->fused && !b->h_fused.empty() && ctx->dedup_interval == 0 && !(cfg->flags & VMB_RC_PRE_MASK);
}

// the un-fused pipeline over the series `sub` (ascending) of an upload whose zstd stage already ran: a sub-batch is built from
// the host copies of the descriptors, decoded into the ctx's column cache and rolled up into the rows sub[i] of d_out
// (dense_rows: series sub[i] writes row i of d_out instead of row sub[i])
static int run_unfused_subset(vmb_ctx* ctx, const vmb_blocks* b, const std::vector<uint32_t>& sub, int32_t* d_zstatus,
                              int64_t tr_min, int64_t tr_max, const vmb_rollup_cfg* cfg, int64_t points, double* d_out,
                              const Counters& c, bool dense_rows) {
    cudaStream_t st = ctx->stream;
    std::vector<vmb_block_desc> descs;
    std::vector<uint32_t> blk_map;
    BlocksPlan pl;
    for (size_t i = 0; i < sub.size(); i++) {
        const uint32_t fb = b->h_ser_first[sub[i]], nb = b->h_ser_nblocks[sub[i]];
        for (uint32_t k = 0; k < nb; k++) {
            vmb_block_desc d = b->h_descs[fb + k];
            d.series_idx = (uint32_t)i;
            descs.push_back(d);
            pl.cols.push_back(b->h_cols[2 * (size_t)(fb + k)]);
            pl.cols.push_back(b->h_cols[2 * (size_t)(fb + k) + 1]);
            blk_map.push_back(fb + k);
        }
    }
    const size_t cn = descs.size(), cs = sub.size();
    plan_layout(pl, descs.data(), cn);
    const PlanArrays L(pl, cn, cn, cs);  // extras: block map, output rows
    std::vector<uint8_t> hs(L.bytes);
    L.pack(hs.data(), pl, descs.data());
    memcpy(L.extra_at(hs.data(), 0), blk_map.data(), cn * 4);
    memcpy(L.extra_at(hs.data(), 1), sub.data(), cs * 4);
    int rc;
    if ((rc = ctx->sub_arrays.reserve(L.bytes + 64))) return rc;
    CU(cudaMemcpyAsync(ctx->sub_arrays.p, hs.data(), L.bytes, cudaMemcpyHostToDevice, st));
    uint8_t* da = (uint8_t*)ctx->sub_arrays.p;
    vmb_blocks bv;
    bv.ctx = ctx;
    L.bind(&bv, da, pl);
    bv.d_payload = b->d_payload;
    vmb_series view;
    if ((rc = column_cache_view(ctx, &bv, &view))) return rc;
    rc = run_decode(ctx, &bv, &view, tr_min, tr_max, 0, c.d_failed, true, d_zstatus, L.extra_at(da, 0), b->d_cols);
    if (!rc) rc = run_rollup(ctx, &view, cfg, points, d_out, c.d_scanned, dense_rows ? nullptr : L.extra_at(da, 1), false);
    cudaError_t e = cudaStreamSynchronize(st);  // `hs` goes out of scope
    if (!rc && e != cudaSuccess) {
        vmb_set_error("un-fused sub-batch: %s", cudaGetErrorString(e));
        rc = VMB_ERR_CUDA;
    }
    return rc;
}

static bool aggr_fusable(int aggr_id) {
    return aggr_id == VMB_AGGR_SUM || aggr_id == VMB_AGGR_AVG || aggr_id == VMB_AGGR_COUNT || aggr_id == VMB_AGGR_GROUP ||
           aggr_id == VMB_AGGR_SUM2 || aggr_id == VMB_AGGR_MIN || aggr_id == VMB_AGGR_MAX;
}
// identity of the fold: 0 for sum-like states, +-Inf for min / max; counts 0
__global__ void k_aggr_init(int aggr, double* dv, double* dc, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    dv[i] = aggr == VMB_AGGR_MIN ? D_INF : (aggr == VMB_AGGR_MAX ? -D_INF : 0.0);
    dc[i] = 0.0;
}

// decode + preamble + rollup of an uploaded block set through the fused kernel, into d_out or, with af, folded into af's state
// (initialised here) instead of written to a [series x P] matrix.  Synchronises the stream once (the bail count has to reach the
// host); the counters are left on the device.  The fused series run in ctx->fused_chunks chunks: the zstd stage of chunk k + 1
// runs on ctx->zstream while chunk k's fused kernel runs on the ctx stream, ordered by events only (nothing waits for the two
// kernels to share an SM).  Events, all on the ctx stream: ev[ST_ZSTD] .. ev[ST_DECODE] the zstd work nothing overlaps (the
// columns of the un-fused series, the generic frames and chunk 0), ev[ST_DECODE] .. ev[ST_PREAMBLE] first fused launch to last
// fused completion, ev[ST_ROLLUP] .. ev[ST_AGGR] the un-fused sub-batch.
static int eval_fused(vmb_ctx* ctx, const vmb_blocks* b, int64_t tr_min, int64_t tr_max, const vmb_rollup_cfg* cfg, int64_t points,
                      double* d_out, const Counters& c, const AggrTarget* af) {
    cudaStream_t st = ctx->stream;
    int rc;
    if (af) {
        if ((rc = ctx->grp_ids.reserve((b->nseries + 1) * sizeof(uint32_t)))) return rc;
        CU(cudaMemcpyAsync(ctx->grp_ids.p, af->group_ids, b->nseries * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
        const size_t cells = (size_t)af->ngroups * (size_t)points;
        k_aggr_init<<<(unsigned)((cells + 255) / 256), 256, 0, st>>>(af->aggr_id, af->d_values, af->d_counts, cells);
        count_launch(ctx);
    }
    const size_t nf = b->h_fused.size();
    // everything that can fail before any work is forked to zstream
    if ((rc = ctx->bail.reserve((nf + 2) * sizeof(uint32_t)))) return rc;
    unsigned int* d_bail_count = (unsigned int*)ctx->bail.p;
    uint32_t* d_bail_list = (uint32_t*)ctx->bail.p + 2;
    FusedParams F;
    memset(&F, 0, sizeof(F));
    if ((rc = upload_cfg_args(ctx, cfg, points, &F.cfg))) return rc;
    F.descs = b->d_descs;
    F.cols = b->d_cols;
    F.payload = b->d_payload;
    F.ser_first_block = b->d_ser_first;
    F.out = d_out;
    if (af) {  // one scratch row per CTA (launch_fused caps the grid at VMB_SMS * FU_CTAS_PER_SM CTAs)
        if ((rc = ctx->tmp_out.reserve((size_t)VMB_SMS * FU_CTAS_PER_SM * (size_t)points * 8))) return rc;
        F.out = (double*)ctx->tmp_out.p;
        F.aggr_values = af->d_values;
        F.aggr_counts = af->d_counts;
        F.group_ids = (const uint32_t*)ctx->grp_ids.p;
        F.aggr_id = af->aggr_id;
    }
    F.scanned = c.d_scanned;
    F.bail_list = d_bail_list;
    F.bail_count = d_bail_count;
    F.npoints = (uint32_t)points;
    F.tr_min = tr_min;
    F.tr_max = tr_max;
    // chunk k = the fused series [nf * k / C, nf * (k + 1) / C); its Huffman frames are d_huf_list[huf_upto[..]] of those bounds
    const uint32_t C = fused_chunks(ctx, b);
    auto chunk_begin = [&](uint32_t k) { return (uint32_t)(nf * k / C); };
    if (C > 1) {
        if (!ctx->zstream) CU(cudaStreamCreateWithFlags(&ctx->zstream, cudaStreamNonBlocking));
        while (ctx->zev.size() < C) {
            cudaEvent_t e;
            CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
            ctx->zev.push_back(e);
        }
    }
    if (ctx->timing) CU(cudaEventRecord(ctx->ev[ST_ZSTD], st));
    int32_t* d_zstatus = nullptr;
    ZstdParams Z = {};
    // on st: everything but the Huffman frames of chunks 1..C-1 (= the whole stage when C == 1)
    if ((rc = run_zstd(ctx, b, &d_zstatus, C > 1 ? b->h_huf_upto[chunk_begin(1)] : UINT32_MAX, &Z))) return rc;
    if (ctx->timing) CU(cudaEventRecord(ctx->ev[ST_DECODE], st));
    // st joins zstream on every way out of here, errors included, so that the next call cannot reuse the zstd buffers under it
    struct Join {
        cudaStream_t st;
        cudaEvent_t done = nullptr;
        ~Join() {
            if (done) cudaStreamWaitEvent(st, done, 0);
        }
    } join{st};
    if (C > 1) {  // the rest on zstream, one chunk after the other, behind what st has queued so far
        CU(cudaEventRecord(ctx->zev[0], st));
        CU(cudaStreamWaitEvent(ctx->zstream, ctx->zev[0], 0));
        for (uint32_t k = 1; k < C; k++) {
            zstd_huf_range(ctx, b, Z, b->h_huf_upto[chunk_begin(k)], b->h_huf_upto[chunk_begin(k + 1)], ctx->zstream);
            cudaError_t e = cudaEventRecord(ctx->zev[k], ctx->zstream);
            if (e == cudaSuccess) join.done = ctx->zev[k];
            CU(e);
        }
    }
    CU(cudaMemsetAsync(d_bail_count, 0, 8, st));
    F.scratch = (const uint8_t*)ctx->zscratch.p;
    F.zstd_status = d_zstatus;
    const uint32_t ctas_per_sm = fused_ctas_per_sm(ctx, C, cfg);
    for (uint32_t k = 0; k < C; k++) {  // chunk k starts when its zstd stage is done (chunk 0's ran on st)
        if (k) CU(cudaStreamWaitEvent(st, ctx->zev[k], 0));
        F.ser_list = b->d_fused_list + chunk_begin(k);
        F.nlist = chunk_begin(k + 1) - chunk_begin(k);
        launch_fused(F, ctas_per_sm, st);
        count_launch(ctx);
    }
    if (ctx->timing) CU(cudaEventRecord(ctx->ev[ST_PREAMBLE], st));
    CU(cudaGetLastError());
    unsigned int* h_bail = (unsigned int*)((char*)ctx->h_pinned + PIN_BAIL);
    CU(cudaMemcpyAsync(h_bail, d_bail_count, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    std::vector<uint32_t> sub(b->h_unfused);
    if (*h_bail) {
        const size_t n0 = sub.size();
        sub.resize(n0 + *h_bail);
        CU(cudaMemcpy(sub.data() + n0, d_bail_list, (size_t)*h_bail * 4, cudaMemcpyDeviceToHost));
        std::sort(sub.begin(), sub.end());
    }
    if (ctx->timing) {
        for (float& ms : ctx->stage_ms) ms = 0.f;
        stage_span(ctx, ST_ZSTD, ST_ZSTD, ST_DECODE);
        stage_span(ctx, ST_FUSED, ST_DECODE, ST_PREAMBLE);
    }
    if (!sub.empty()) {
        if (ctx->timing) CU(cudaEventRecord(ctx->ev[ST_ROLLUP], st));
        if (!af) {
            if ((rc = run_unfused_subset(ctx, b, sub, d_zstatus, tr_min, tr_max, cfg, points, d_out, c, false))) return rc;
        } else {
            // the sub-batch's rows go to a dense scratch matrix, are folded per group and merged in
            const size_t cs = sub.size(), cells = (size_t)af->ngroups * (size_t)points;
            if ((rc = ctx->rolled.reserve((cs * (size_t)points + 2 * cells) * 8 + 64))) return rc;
            double* d_rows = (double*)ctx->rolled.p;
            if ((rc = run_unfused_subset(ctx, b, sub, d_zstatus, tr_min, tr_max, cfg, points, d_rows, c, true))) return rc;
            std::vector<uint32_t> h_csr;
            uint32_t* d_csr;
            if ((rc = upload_group_csr(ctx, h_csr, af->group_ids, sub.data(), cs, af->ngroups, 0, &d_csr))) return rc;
            aggr_fold(ctx, st, *af, d_rows, d_csr, points, d_rows + cs * (size_t)points);
            CU(cudaStreamSynchronize(st));  // `h_csr` goes out of scope
        }
        if (ctx->timing) {
            CU(cudaEventRecord(ctx->ev[ST_AGGR], st));
            CU(cudaStreamSynchronize(st));
            stage_span(ctx, ST_DECODE, ST_ROLLUP, ST_AGGR);  // the un-fused sub-batch as a whole (decode + preamble + rollup)
        }
    }
    return 0;
}

// decode + preamble + rollup of device-resident blocks into the [series x P] matrix d_out or, with aggr, folded into aggr's state:
// through the fused kernel where it applies, else through the kernel-per-stage pipeline over the ctx's column cache
static int eval_device(vmb_ctx* ctx, const vmb_blocks* b, int64_t tr_min, int64_t tr_max, const vmb_rollup_cfg* cfg, int64_t points,
                       double* d_out, const AggrTarget* aggr, uint64_t* samples_scanned) {
    cudaStream_t st = ctx->stream;
    const bool fused = fused_enabled(ctx, b, cfg) && (!aggr || aggr_fusable(aggr->aggr_id));
    int rc;
    std::vector<uint32_t> h_csr;  // lives until counters_read synchronises
    uint32_t* d_csr = nullptr;
    if (aggr && fused) {  // the fused kernel reads the group of every series; group_csr checks only those of the sub-batch
        for (size_t i = 0; i < b->nseries; i++)
            if (aggr->group_ids[i] >= aggr->ngroups) return group_id_error(aggr->group_ids[i], i, aggr->ngroups);
    } else if (aggr) {
        if ((rc = upload_group_csr(ctx, h_csr, aggr->group_ids, nullptr, b->nseries, aggr->ngroups, 0, &d_csr))) return rc;
    }
    Counters c;
    if ((rc = counters_zero(ctx, st, &c))) return rc;
    if (fused) {
        if ((rc = eval_fused(ctx, b, tr_min, tr_max, cfg, points, d_out, c, aggr))) return rc;
        return counters_read(ctx, st, samples_scanned);
    }
    vmb_series view;
    if ((rc = column_cache_view(ctx, b, &view))) return rc;
    if ((rc = run_decode(ctx, b, &view, tr_min, tr_max, 0, c.d_failed))) return rc;
    double* d_rows = d_out;
    if (aggr) {
        if ((rc = ctx->rolled.reserve((size_t)b->nseries * (size_t)points * 8))) return rc;
        d_rows = (double*)ctx->rolled.p;
    }
    if ((rc = run_rollup(ctx, &view, cfg, points, d_rows, c.d_scanned))) return rc;
    if (aggr) {
        aggr_fold(ctx, st, *aggr, d_rows, d_csr, points, nullptr);
        if (ctx->timing) CU(cudaEventRecord(ctx->ev[ST_FUSED], st));
    }
    rc = counters_read(ctx, st, samples_scanned);
    if (rc && rc != VMB_ERR_BLOCK_FAILED) return rc;
    if (aggr) {
        collect_stage_times(ctx, ST_PREAMBLE, ST_FUSED);  // as vmb_rollup_aggr_partial
    } else if (ctx->timing) {
        collect_stage_times(ctx, ST_ZSTD, ST_AGGR);
        ctx->stage_ms[ST_FUSED] = 0.f;
    }
    return rc;
}

extern "C" int vmb_eval_rollup_device(vmb_ctx* ctx, const vmb_blocks* b, int64_t tr_min, int64_t tr_max,
                                      const vmb_rollup_cfg* cfg, double* d_out, uint64_t* samples_scanned) {
    if (!ctx || !b || !d_out) return VMB_ERR_INVALID_ARG;
    int64_t points;
    int rc = check_cfg(cfg, &points);
    if (rc) return rc;
    CU(cudaSetDevice(ctx->device));
    return eval_device(ctx, b, tr_min, tr_max, cfg, points, d_out, nullptr, samples_scanned);
}

// decode + preamble + rollup + per-GPU incremental aggregate of device-resident blocks (evalRollupWithIncrementalAggregate
// eval.go:1804 for one rank)
extern "C" int vmb_eval_rollup_aggr_device(vmb_ctx* ctx, const vmb_blocks* b, int64_t tr_min, int64_t tr_max,
                                           const vmb_rollup_cfg* cfg, int aggr_id, const uint32_t* group_ids, uint32_t ngroups,
                                           double* d_values, double* d_counts, uint64_t* samples_scanned) {
    if (!ctx || !b || !group_ids || !d_values || !d_counts || ngroups == 0 || aggr_id < 0 || aggr_id > VMB_AGGR_GROUP)
        return VMB_ERR_INVALID_ARG;
    int64_t points;
    int rc = check_cfg(cfg, &points);
    if (rc) return rc;
    CU(cudaSetDevice(ctx->device));
    const AggrTarget t = {aggr_id, group_ids, ngroups, d_values, d_counts};
    return eval_device(ctx, b, tr_min, tr_max, cfg, points, nullptr, &t, samples_scanned);
}

#include "pipeline.inc"
#include "topk.inc"
#include "comm.inc"
#include "matrix_ops.inc"
#include "aggr_matrix.inc"
#include "aggr_order.inc"
#include "transform.inc"
#include "range_transform.inc"
#include "histogram.inc"

// ------------------------------------------------------------------------------------------------ batched host encoder
#include <atomic>
#include <thread>
// Block.MarshalData (block.go:192) for many equal-length columns at once on host threads (write path / test+bench input
// generation).  vals: [ncols x rows]; dst receives the payloads back to back, offs[ncols+1] their offsets.
extern "C" int vmb_marshal_columns(uint8_t* dst, size_t cap, uint64_t* offs, uint8_t* mts, int64_t* firsts,
                                   const int64_t* vals, size_t ncols, size_t rows, uint8_t precision_bits, int nthreads) {
    if (!dst || !offs || !mts || !firsts || !vals || rows == 0) return VMB_ERR_INVALID_ARG;
    std::vector<std::vector<uint8_t>> outs(ncols);
    std::atomic<size_t> next{0};
    std::atomic<int> err{0};
    auto worker = [&]() {
        for (;;) {
            size_t c = next.fetch_add(1);
            if (c >= ncols) break;
            int mt = 0;
            int64_t first = 0;
            int rc = vmb_host::marshal_int64_array(outs[c], &mt, &first, vals + c * rows, rows, precision_bits);
            if (rc) err = rc;
            mts[c] = (uint8_t)mt;
            firsts[c] = first;
        }
    };
    if (nthreads <= 1) worker();
    else {
        std::vector<std::thread> th;
        for (int t = 0; t < nthreads; t++) th.emplace_back(worker);
        for (auto& t : th) t.join();
    }
    if (err.load()) return err.load();
    uint64_t o = 0;
    for (size_t c = 0; c < ncols; c++) {
        offs[c] = o;
        if (o + outs[c].size() > cap) return VMB_ERR_CAP;
        if (!outs[c].empty()) memcpy(dst + o, outs[c].data(), outs[c].size());
        o += outs[c].size();
    }
    offs[ncols] = o;
    return VMB_OK;
}

// Block.MarshalData (block.go:192) for many equal-length columns with the int64 work on the GPU (csrc/encode.cu): type detection,
// nearest-delta / delta2 (lossless and lossy precisionBits), zig-zag varint packing; the zstd stage of streams >= 128 bytes and the
// 0.9 rule (encoding.go:152-167) follow on `nthreads` host threads with the library's zstd writer.  Same output layout and the same
// bytes as vmb_marshal_columns.
extern "C" int vmb_marshal_columns_gpu(vmb_ctx* ctx, uint8_t* dst, size_t cap, uint64_t* offs, uint8_t* mts, int64_t* firsts,
                                       const int64_t* vals, size_t ncols, size_t rows, uint8_t precision_bits, int nthreads) {
    if (!ctx || !dst || !offs || !mts || !firsts || !vals || rows == 0 || rows > 16384 || ncols > 0x7fffffffu || precision_bits < 1 ||
        precision_bits > 64)
        return VMB_ERR_INVALID_ARG;
    CU(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    if (ncols == 0) {
        offs[0] = 0;
        return VMB_OK;
    }
    int rc;
    const size_t nvals = ncols * rows;
    if ((rc = ctx->enc_vals.reserve(nvals * 8))) return rc;
    // per column: u32 size | u8 mt (padded to 4) | i64 first | u64 offset
    const size_t o_sizes = 0, o_mts = al16(o_sizes + ncols * 4), o_firsts = al16(o_mts + ncols), o_offs = al16(o_firsts + ncols * 8);
    if ((rc = ctx->enc_meta.reserve(al16(o_offs + ncols * 8) + 64))) return rc;
    const bool may_be_lossy = precision_bits < 64;
    if (may_be_lossy && (rc = ctx->enc_deltas.reserve(nvals * 8))) return rc;
    CU(cudaMemcpyAsync(ctx->enc_vals.p, vals, nvals * 8, cudaMemcpyHostToDevice, st));
    uint8_t* dm = (uint8_t*)ctx->enc_meta.p;
    MarshalParams M;
    memset(&M, 0, sizeof(M));
    M.vals = (const int64_t*)ctx->enc_vals.p;
    M.deltas = may_be_lossy ? (int64_t*)ctx->enc_deltas.p : nullptr;
    M.sizes = (uint32_t*)(dm + o_sizes);
    M.mts = dm + o_mts;
    M.firsts = (int64_t*)(dm + o_firsts);
    M.offs = (const uint64_t*)(dm + o_offs);
    M.ncols = (uint32_t)ncols;
    M.rows = (uint32_t)rows;
    M.pb = precision_bits;
    launch_marshal_plan(M, st);
    count_launch(ctx);
    std::vector<uint32_t> sizes(ncols);
    std::vector<uint8_t> pmts(ncols);
    CU(cudaMemcpyAsync(sizes.data(), M.sizes, ncols * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(pmts.data(), M.mts, ncols, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(firsts, M.firsts, ncols * 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    std::vector<uint64_t> soffs(ncols + 1, 0);
    for (size_t c = 0; c < ncols; c++) soffs[c + 1] = soffs[c] + sizes[c];
    const uint64_t total = soffs[ncols];
    if ((rc = ctx->enc_out.reserve(total + 64))) return rc;
    CU(cudaMemcpyAsync(dm + o_offs, soffs.data(), ncols * 8, cudaMemcpyHostToDevice, st));
    M.out = (uint8_t*)ctx->enc_out.p;
    launch_marshal_pack(M, st);
    count_launch(ctx);
    std::vector<uint8_t> streams(total + 1);
    if (total) CU(cudaMemcpyAsync(streams.data(), M.out, total, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    // ---- zstd stage + the 0.9 rule on host threads
    std::vector<std::vector<uint8_t>> outs(ncols);
    std::atomic<size_t> next{0};
    auto worker = [&]() {
        for (;;) {
            const size_t c = next.fetch_add(1);
            if (c >= ncols) break;
            const uint8_t* bb = streams.data() + soffs[c];
            const size_t blen = sizes[c];
            uint8_t mt = pmts[c];
            if (mt == 1 || mt == 4) {
                const size_t min_compressible = 128;  // encoding.go:15
                if (blen >= min_compressible) vmb_host::zstd_compress_huf(outs[c], bb, blen);
                if (blen < min_compressible || (double)outs[c].size() > 0.9 * (double)blen) {  // encoding.go:156
                    mt = mt == 1 ? 5 : 6;
                    outs[c].assign(bb, bb + blen);
                }
            } else {
                outs[c].assign(bb, bb + blen);
            }
            mts[c] = mt;
        }
    };
    if (nthreads <= 1) worker();
    else {
        std::vector<std::thread> th;
        for (int t = 0; t < nthreads; t++) th.emplace_back(worker);
        for (auto& t : th) t.join();
    }
    uint64_t o = 0;
    for (size_t c = 0; c < ncols; c++) {
        offs[c] = o;
        if (o + outs[c].size() > cap) return VMB_ERR_CAP;
        if (!outs[c].empty()) memcpy(dst + o, outs[c].data(), outs[c].size());
        o += outs[c].size();
    }
    offs[ncols] = o;
    return VMB_OK;
}

// decimal.AppendFloatToDecimal (decimal.go:173) for ncols equal-length float64 columns on the GPU: dst [ncols x rows] mantissas,
// scales[ncols] the common exponent of each column (what Block.Init / the ingest path compute per block before MarshalData)
extern "C" int vmb_float_to_decimal_columns(vmb_ctx* ctx, int64_t* dst, int16_t* scales, const double* src, size_t ncols, size_t rows) {
    if (!ctx || !dst || !scales || !src || rows == 0 || ncols > 0x7fffffffu || rows > 0x7fffffffu) return VMB_ERR_INVALID_ARG;
    if (ncols == 0) return VMB_OK;
    CU(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    const size_t n = ncols * rows;
    int rc;
    if ((rc = ctx->enc_vals.reserve(n * 8))) return rc;
    if ((rc = ctx->enc_deltas.reserve(n * 8))) return rc;
    if ((rc = ctx->enc_meta.reserve(al16(n * 2) + al16(ncols * 2) + 64))) return rc;
    double* d_src = (double*)ctx->enc_vals.p;
    int64_t* d_dst = (int64_t*)ctx->enc_deltas.p;
    int16_t* d_ea = (int16_t*)ctx->enc_meta.p;
    int16_t* d_sc = (int16_t*)((uint8_t*)ctx->enc_meta.p + al16(n * 2));
    CU(cudaMemcpyAsync(d_src, src, n * 8, cudaMemcpyHostToDevice, st));
    uint32_t grid = (uint32_t)((ncols + 3) / 4);
    if (grid > VMB_SMS * 16u) grid = VMB_SMS * 16u;
    k_float_to_decimal<<<grid, 128, 0, st>>>(d_src, d_dst, d_ea, d_sc, (uint32_t)ncols, (uint32_t)rows);
    count_launch(ctx);
    CU(cudaMemcpyAsync(dst, d_dst, n * 8, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(scales, d_sc, ncols * 2, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    return VMB_OK;
}
