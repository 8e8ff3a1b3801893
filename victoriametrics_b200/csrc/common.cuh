// libvmb200 internal declarations shared by the .cu files (product code; never includes anything from oracle/).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/vmb200.h"

#define VMB_WARP 32
#define VMB_FULL 0xffffffffu
#define VMB_SMS 132u  // streaming multiprocessors of an H100 SXM: grid-stride launches cap their grids at a multiple of it

// lib/decimal/decimal.go:403-415
#define VMB_V_INF_POS INT64_MAX
#define VMB_V_INF_NEG INT64_MIN
#define VMB_V_STALE_NAN (INT64_MAX - 1)
#define VMB_V_MAX (INT64_MAX - 2)
#define VMB_V_MIN (INT64_MIN + 1)
#define VMB_STALE_NAN_BITS 0x7ff0000000000002ULL

// per-column zstd classification computed on the host at upload time (api.cu)
enum : uint8_t {
    VMB_ZK_NONE = 0,     // column is not zstd (mt 2,3,5,6)
    VMB_ZK_HUF = 1,      // single compressed block, Huffman literals: handled by the lane-packed Huffman kernel
    VMB_ZK_GENERIC = 2,  // anything else: serial per-thread frame decoder
    VMB_ZK_BAD = 3,      // header does not parse: VMB_ERR_ZSTD
};

struct ColInfo {            // one per column (2 per block: [2*b] timestamps, [2*b+1] values)
    uint64_t scratch_off;   // where the decompressed varint bytes go inside the zstd scratch arena
    uint32_t content_size;  // decompressed size: Frame_Content_Size; without one, the host's bound until the serial
                            // decoder stores the length the frame produced (in the device copy)
    uint8_t kind;           // VMB_ZK_*
    uint8_t _pad[3];
    uint32_t nseq;          // VMB_ZK_HUF: Number_of_Sequences of the block (read by the host plan from the section header)
    uint32_t seq_rec_off;   // where this column's decoded sequence records start in the record arena
    uint32_t _pad2;
};
static_assert(sizeof(ColInfo) == 32, "ColInfo layout");

// job record written by the zstd prepare kernel for the lane-packed Huffman kernel
struct HufJob {
    uint64_t src_off;        // payload offset of the first Huffman stream (after tree description / jump table)
    uint64_t dst_off;        // destination offset (scratch arena, or literal arena when sequences follow)
    uint32_t stream_size[4]; // compressed sizes (stream_size[1..3] == 0 for single-stream)
    uint32_t regen_size;     // regenerated literal bytes
    uint32_t col;            // column index (2*block + which)
    uint32_t seq_off;        // offset of the sequences section relative to the frame start
    uint32_t seq_size;       // bytes in the sequences section (incl. nbSeq header)
    uint8_t nbits[256];      // code length per symbol (0 = unused); 8-byte aligned (offset 48)
    uint8_t table_log;       // Max_Number_of_Bits
    uint8_t nstreams;        // 1 or 4; 0 = job invalid
    uint8_t dst_is_lit;      // 1: dst_off is into the literal arena (sequences will run afterwards)
    uint8_t seq_big;         // set by k_zstd_seq_decode<false>: a sequence table has > 256 states, decoded by the second launch
    uint8_t _pad[4];
};
static_assert(sizeof(HufJob) == 312, "HufJob layout");

// SeriesMeta::flags, bits 0-3; bits 8-23 hold the first row with a value drop (SeriesMeta::first_drop)
enum : uint32_t {
    VMB_SER_STALE = 1u,    // the series may hold Prometheus staleness markers: dropStaleNaNs has something to do
    VMB_SER_DROP = 2u,     // the series may hold a value below its predecessor (or a NaN): removeCounterResets has something to do
    VMB_SER_MERGED = 4u,   // the series is assembled by k_series_merge
    VMB_SER_TS_AP = 8u,    // the timestamps are an arithmetic progression (one block, MarshalTypeDeltaConst timestamps, no
                           // deduplication): the rollup kernel derives them from the row index instead of reading them
};

struct SeriesMeta {
    uint64_t start;          // first row of the series inside the dense columns
    uint32_t n;              // rows (after trimming / stale-NaN drop)
    uint32_t flags;          // VMB_SER_* | first_drop() << 8
    int64_t max_prev_interval;
    int64_t window;          // effective window (rollup.go:747-756)
    // the row removeCounterResets may start from: nothing before the first value drop changes (0: unknown)
    __host__ __device__ __forceinline__ uint32_t first_drop() const { return (flags >> 8) & 0xffffu; }
    __host__ __device__ __forceinline__ void set_first_drop(uint32_t row) { flags = (flags & ~(0xffffu << 8)) | ((row & 0xffffu) << 8); }
};
static_assert(sizeof(SeriesMeta) == 32, "SeriesMeta layout");

// blk_hi, the per-block word k_decode_columns writes beside blk_lo (the first kept row) for k_series_assemble / k_series_merge:
// bits 0-14 end of the kept rows (<= 16384), bits 15-28 first row with a value drop, bit 30 "may change under
// removeCounterResets", bit 31 "holds a staleness marker"
__host__ __device__ __forceinline__ uint32_t blk_hi_pack(uint32_t end, uint32_t first_drop, bool may_change, bool stale) {
    return end | (first_drop << 15) | ((uint32_t)may_change << 30) | ((uint32_t)stale << 31);
}
__host__ __device__ __forceinline__ uint32_t blk_hi_end(uint32_t w) { return w & 0x7fffu; }
__host__ __device__ __forceinline__ uint32_t blk_hi_first_drop(uint32_t w) { return (w >> 15) & 0x3fffu; }
__host__ __device__ __forceinline__ bool blk_hi_may_change(uint32_t w) { return (w >> 30) & 1u; }
__host__ __device__ __forceinline__ bool blk_hi_stale(uint32_t w) { return w >> 31; }

// ---- small device helpers ---------------------------------------------------------------------------------------
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ uint64_t shfl_u64(uint64_t v, int src) {
    uint32_t lo = __shfl_sync(VMB_FULL, (uint32_t)v, src);
    uint32_t hi = __shfl_sync(VMB_FULL, (uint32_t)(v >> 32), src);
    return ((uint64_t)hi << 32) | lo;
}
__device__ __forceinline__ uint64_t shfl_up_u64(uint64_t v, int d) {
    uint32_t lo = __shfl_up_sync(VMB_FULL, (uint32_t)v, d);
    uint32_t hi = __shfl_up_sync(VMB_FULL, (uint32_t)(v >> 32), d);
    return ((uint64_t)hi << 32) | lo;
}
__device__ __forceinline__ double shfl_f64(double v, int src) {
    return __longlong_as_double((long long)shfl_u64((uint64_t)__double_as_longlong(v), src));
}
__device__ __forceinline__ double shfl_up_f64(double v, int d) {
    return __longlong_as_double((long long)shfl_up_u64((uint64_t)__double_as_longlong(v), d));
}

// little-endian u32 at an arbitrary byte address; touches only the two aligned words that contain it.
// The payload / scratch arenas are over-allocated by 64 bytes so the second word is always readable.
__device__ __forceinline__ uint32_t load_u32_unaligned(const uint8_t* p) {
    uintptr_t a = (uintptr_t)p;
    const uint32_t* w = (const uint32_t*)(a & ~(uintptr_t)3);
    uint32_t sh = (uint32_t)(a & 3) * 8;
    uint32_t lo = w[0];
    if (sh == 0) return lo;
    uint32_t hi = w[1];
    return __funnelshift_r(lo, hi, sh);
}

// Go math.Pow10 (stdlib table product), see decimal.cu
__device__ double vmb_pow10(int n);

// error helper for host code
void vmb_set_error(const char* fmt, ...);
