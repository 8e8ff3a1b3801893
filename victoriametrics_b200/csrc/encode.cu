// Write path on the GPU: encoding.MarshalValues / MarshalTimestamps for many equal-length columns at once
// (Block.MarshalData lib/storage/block.go:192 as the merge path calls it, lib/storage/merge.go:227-235).
//
//   lib/encoding/encoding.go:119   marshalInt64Array: type selection
//   lib/encoding/encoding.go:289   isConst, :311 isDeltaConst, :331 isGauge
//   lib/encoding/nearest_delta.go:15, nearest_delta2.go:15   delta / delta-of-delta (+ :83 nearestDelta for precisionBits < 64)
//   lib/encoding/int.go:107        MarshalVarInt64s (zig-zag LEB128)
//
// One warp per column, two kernels:
//   k_marshal_plan:  the three detection scans as ONE pass of warp reductions (every early return of isGauge is an "exists"
//                    condition, the reset count an order-independent sum), the MarshalType, and the byte size of the varint
//                    stream (a warp sum of per-value lengths); for precisionBits < 64 the lossy deltas -- a sequential state
//                    machine (trailingZeros, v) -- are produced by one lane into a scratch column first;
//   k_marshal_pack:  per 32-value chunk the lengths are scanned over the warp and every lane writes its varint at its offset.
// The byte offsets between the two come from an exclusive prefix sum of the sizes (host, ncols entries).  Then the zstd stage of
// encoding.go:152-167 on the device, for the streams of type 1 / 4 of >= 128 bytes:
//   k_zstd_frames:    the library's zstd writer (rules: zstd_writer.cuh, shared with the host writer), one CTA per frame, each
//                     frame into its own slot (also vmb_zstd_compress_batch);
//   k_marshal_select: the 0.9 rule per column (a rejected frame turns 1 -> 5 / 4 -> 6 and keeps the stream);
//   k_scan_lens, k_compact: the payloads' offsets and the payloads back to back in column order.
#pragma once

struct MarshalParams {
    const int64_t* vals;      // [ncols x rows]
    int64_t* deltas;          // scratch [ncols x rows] (precisionBits < 64 only, else nullptr)
    uint8_t* out;             // varint streams, column c at offs[c]
    const uint64_t* offs;     // [ncols] (pack)
    uint32_t* sizes;          // [ncols] (plan)
    uint8_t* mts;             // [ncols]: 3 const, 2 delta-const, 4 gauge -> nearest delta, 1 counter -> nearest delta2
    int64_t* firsts;          // [ncols]
    uint32_t ncols, rows;
    uint32_t pb;              // precisionBits 1..64
    // ragged columns (the merge path): column c holds col_rows[c] values at vals + col_off[c] with precisionBits col_pb[c];
    // nullptr: every column holds `rows` values at c * rows with precisionBits pb
    const uint64_t* col_off;
    const uint32_t* col_rows;
    const uint8_t* col_pb;
};

namespace {

__device__ __forceinline__ uint32_t varint_len(uint64_t u) {  // bytes of the LEB128 form, int.go:107
    const uint32_t bits = u ? 64u - (uint32_t)__clzll((long long)u) : 1u;
    return (bits + 6u) / 7u;
}
__device__ __forceinline__ uint64_t zz64(int64_t v) { return (uint64_t)((v << 1) ^ (v >> 63)); }

__device__ __forceinline__ uint32_t enc_bitlen(uint64_t x) { return x ? 64u - (uint32_t)__clzll((long long)x) : 0u; }
// getTrailingZeros nearest_delta.go:134
__device__ __forceinline__ uint32_t enc_trailing_zeros(int64_t v, uint32_t pb) {
    const uint64_t a = v < 0 ? (uint64_t)0 - (uint64_t)v : (uint64_t)v;
    const uint32_t vb = enc_bitlen(a);
    return vb <= pb ? 0u : vb - pb;
}
// nearestDelta nearest_delta.go:83 (uint8 arithmetic of the trailing-zeros state kept)
__device__ __forceinline__ void enc_nearest_delta(int64_t next, int64_t prev, uint32_t pb, uint32_t ptz, int64_t* dout, uint32_t* tzout) {
    const int64_t d = (int64_t)((uint64_t)next - (uint64_t)prev);
    const uint32_t dec = ptz ? ptz - 1u : 0u;
    if (d == 0) { *dout = 0; *tzout = dec; return; }
    const uint64_t origin = next < 0 ? (uint64_t)0 - (uint64_t)next : (uint64_t)next;
    const uint32_t ob = enc_bitlen(origin);
    if (ob <= pb) { *dout = d; *tzout = dec; return; }
    const uint32_t tz = ob - pb;
    if (tz > ((ptz + 4u) & 0xffu)) { *dout = d; *tzout = (ptz + 2u) & 0xffu; return; }
    if (((tz + 4u) & 0xffu) < ptz) { *dout = d; *tzout = (ptz - 2u) & 0xffu; return; }
    const bool minus = d < 0;
    const uint64_t ad = minus ? (uint64_t)0 - (uint64_t)d : (uint64_t)d;
    const uint64_t mask = tz >= 64u ? 0ull : (~(uint64_t)0 << tz);
    const uint64_t nd = ad & mask;
    *dout = (int64_t)(minus ? (uint64_t)0 - nd : nd);
    *tzout = tz;
}

// the i-th value of the varint stream of a column (i >= 1): lossless forms straight from the column, lossy ones from the scratch
__device__ __forceinline__ int64_t enc_stream_value(const int64_t* a, const int64_t* dl, uint32_t i, bool delta2, bool lossy) {
    if (lossy) return dl[i];
    if (!delta2 || i == 1) return (int64_t)((uint64_t)a[i] - (uint64_t)a[i - 1]);
    return (int64_t)((uint64_t)a[i] - 2ull * (uint64_t)a[i - 1] + (uint64_t)a[i - 2]);  // next - v - d1, nearest_delta2.go:30
}

// where column c lives, how many values it holds and at which precisionBits it is written
__device__ __forceinline__ void enc_col(const MarshalParams& P, uint32_t c, uint64_t* off, uint32_t* n, uint32_t* pb) {
    if (P.col_off) {
        *off = P.col_off[c];
        *n = P.col_rows[c];
        *pb = P.col_pb[c];
    } else {
        *off = (uint64_t)c * P.rows;
        *n = P.rows;
        *pb = P.pb;
    }
}

}  // namespace

__global__ void __launch_bounds__(128) k_marshal_plan(MarshalParams P) {
    const int lane = lane_id();
    const uint32_t wpg = gridDim.x * (blockDim.x >> 5);
    for (uint32_t c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c < P.ncols; c += wpg) {
        uint64_t co;
        uint32_t n, cpb;
        enc_col(P, c, &co, &n, &cpb);
        const int64_t* a = P.vals + co;
        const int64_t a0 = a[0];
        // ---- detection: isConst, isDeltaConst, isGauge in one pass
        const uint64_t d1 = n >= 2 ? (uint64_t)a[1] - (uint64_t)a0 : 0ull;
        bool all_eq = true, dconst = n >= 2, imm = false;
        uint32_t resets = 0;
        for (uint32_t i = 1 + lane; i < n; i += 32) {
            const int64_t v = a[i], pv = a[i - 1];
            all_eq &= v == a0;
            dconst &= ((uint64_t)v - (uint64_t)pv) == d1;
            if (v < pv) {
                if (v < 0 || v > (pv >> 3)) imm = true;  // encoding.go:349-357
                resets++;
            }
        }
        all_eq = __all_sync(VMB_FULL, all_eq);
        dconst = __all_sync(VMB_FULL, dconst);
        imm = __any_sync(VMB_FULL, imm);
#pragma unroll
        for (int o = 16; o; o >>= 1) resets += __shfl_xor_sync(VMB_FULL, resets, o);
        bool gauge = false;
        if (n >= 2) gauge = a0 < 0 || imm || (resets > 2 && resets > (n >> 3));
        uint32_t mt, size = 0;
        if (all_eq) mt = 3;                                     // MarshalTypeConst encoding.go:124
        else if (dconst) {
            mt = 2;                                             // MarshalTypeDeltaConst :130
            size = varint_len(zz64((int64_t)d1));
        } else {
            mt = gauge ? 4u : 1u;
            const bool delta2 = !gauge;
            uint32_t pb = cpb;
            if (gauge && pb < 6) pb += 2;                        // encoding.go:141
            const bool lossy = pb < 64;
            int64_t* dl = lossy ? P.deltas + co : nullptr;
            if (lossy) {
                // the state machine of nearest_delta.go:36-42 / nearest_delta2.go:39-46, sequential by construction
                if (lane == 0) {
                    if (!delta2) {
                        int64_t v = a0;
                        uint32_t tz = enc_trailing_zeros(v, pb);
                        for (uint32_t i = 1; i < n; i++) {
                            int64_t d;
                            enc_nearest_delta(a[i], v, pb, tz, &d, &tz);
                            v = (int64_t)((uint64_t)v + (uint64_t)d);
                            dl[i] = d;
                        }
                    } else {
                        int64_t dd = (int64_t)d1, v = a[1];
                        dl[1] = dd;
                        uint32_t tz = enc_trailing_zeros(v, pb);
                        for (uint32_t i = 2; i < n; i++) {
                            int64_t d2;
                            enc_nearest_delta((int64_t)((uint64_t)a[i] - (uint64_t)v), dd, pb, tz, &d2, &tz);
                            dd = (int64_t)((uint64_t)dd + (uint64_t)d2);
                            v = (int64_t)((uint64_t)v + (uint64_t)dd);
                            dl[i] = d2;
                        }
                    }
                }
                __syncwarp();
            }
            for (uint32_t i = 1 + lane; i < n; i += 32) size += varint_len(zz64(enc_stream_value(a, dl, i, delta2, lossy)));
#pragma unroll
            for (int o = 16; o; o >>= 1) size += __shfl_xor_sync(VMB_FULL, size, o);
        }
        if (lane == 0) {
            P.mts[c] = (uint8_t)mt;
            P.sizes[c] = size;
            P.firsts[c] = a0;
        }
    }
}

__global__ void __launch_bounds__(128) k_marshal_pack(MarshalParams P) {
    const int lane = lane_id();
    const uint32_t wpg = gridDim.x * (blockDim.x >> 5);
    for (uint32_t c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c < P.ncols; c += wpg) {
        const uint32_t mt = P.mts[c];
        if (mt == 3) continue;
        uint64_t co;
        uint32_t n, cpb;
        enc_col(P, c, &co, &n, &cpb);
        const int64_t* a = P.vals + co;
        uint8_t* out = P.out + P.offs[c];
        if (mt == 2) {
            if (lane == 0) {
                uint64_t u = zz64((int64_t)((uint64_t)a[1] - (uint64_t)a[0]));
                uint32_t k = 0;
                while (u >= 0x80) { out[k++] = (uint8_t)(u | 0x80); u >>= 7; }
                out[k] = (uint8_t)u;
            }
            continue;
        }
        const bool delta2 = mt == 1;
        uint32_t pb = cpb;
        if (!delta2 && pb < 6) pb += 2;
        const bool lossy = pb < 64;
        const int64_t* dl = lossy ? P.deltas + co : nullptr;
        uint32_t base = 0;
        for (uint32_t i0 = 1; i0 < n; i0 += 32) {
            const uint32_t i = i0 + lane;
            uint64_t u = 0;
            uint32_t len = 0;
            if (i < n) {
                u = zz64(enc_stream_value(a, dl, i, delta2, lossy));
                len = varint_len(u);
            }
            uint32_t inc = len;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(VMB_FULL, inc, o);
                if (lane >= o) inc += t;
            }
            uint8_t* w = out + base + inc - len;
            for (uint32_t k = 0; k + 1 < len; k++) {
                w[k] = (uint8_t)(u | 0x80);
                u >>= 7;
            }
            if (len) w[len - 1] = (uint8_t)u;
            base += __shfl_sync(VMB_FULL, inc, 31);
        }
    }
}

// ---- decimal.AppendFloatToDecimal (lib/decimal/decimal.go:173-257) for many columns: one warp per column.
// FromFloat per value (:437, the same code as the host encoder: marshal.inc is compiled for both sides), the minimum exponent over
// the non-special values (:203-211), the down-shift that keeps every up-scaled mantissa inside int64 (:213-224), the rescale
// (:231-249); the all-zeros / all-ones fast paths (:177-184) come out of the same reductions.
// Ragged columns (the flush path): column c holds col_rows[c] values at col_off[c] of src, dst and ea; nullptr: every column holds
// `rows` values at c * rows.
__global__ void __launch_bounds__(128) k_float_to_decimal(const double* __restrict__ src, int64_t* __restrict__ dst, int16_t* __restrict__ ea,
                                                          int16_t* __restrict__ scales, uint32_t ncols, uint32_t rows,
                                                          const uint64_t* __restrict__ col_off, const uint32_t* __restrict__ col_rows) {
    const int lane = lane_id();
    const uint32_t wpg = gridDim.x * (blockDim.x >> 5);
    for (uint32_t c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c < ncols; c += wpg) {
        const size_t co = col_off ? col_off[c] : (size_t)c * rows;
        const uint32_t n = col_off ? col_rows[c] : rows;
        const double* f = src + co;
        int64_t* v = dst + co;
        int16_t* e = ea + co;
        bool zeros = true, ones = true;
        int min_exp = 32767;
        for (uint32_t i = lane; i < n; i += 32) {
            const double x = f[i];
            const unsigned long long b = (unsigned long long)__double_as_longlong(x);
            zeros &= b == 0ull;
            ones &= b == 0x3ff0000000000000ull;
            int64_t vi;
            int16_t ei;
            vmb_host::from_float(x, &vi, &ei);
            v[i] = vi;
            e[i] = ei;
            if (ei < min_exp && !vmb_host::special(vi)) min_exp = ei;
        }
        zeros = __all_sync(VMB_FULL, zeros);
        ones = __all_sync(VMB_FULL, ones);
#pragma unroll
        for (int o = 16; o; o >>= 1) min_exp = min(min_exp, __shfl_xor_sync(VMB_FULL, min_exp, o));
        __syncwarp();
        if (zeros || ones) {
            for (uint32_t i = lane; i < n; i += 32) v[i] = ones ? 1 : 0;
            if (lane == 0) scales[c] = 0;
            continue;
        }
        int down = 0;
        for (uint32_t i = lane; i < n; i += 32) {
            const int up = (int16_t)(e[i] - min_exp);
            const int d = (int16_t)(up - vmb_host::max_up_exponent(v[i]));
            down = max(down, d);
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) down = max(down, __shfl_xor_sync(VMB_FULL, down, o));
        const int16_t mexp = (int16_t)(min_exp + down);
        for (uint32_t i = lane; i < n; i += 32) {
            int64_t x = v[i];
            if (vmb_host::special(x)) continue;
            int adj = (int16_t)(e[i] - mexp);
            while (adj > 0) { x = (int64_t)((uint64_t)x * 10u); adj--; }
            while (adj < 0) { x /= 10; adj++; }
            v[i] = x;
        }
        if (lane == 0) scales[c] = mexp;
    }
}

// ---- the library's zstd writer on the device (rules: zstd_writer.cuh): one CTA per frame, frames into 4-byte aligned slots
struct ZstdFrameJobs {
    uint8_t* base;             // sources and slots
    const uint64_t* src_off;   // [n]
    const uint32_t* len;       // [n] source bytes; 0: no frame
    const uint64_t* slot_off;  // [n] 4-byte aligned, room for zw::raw_frame_len(len) rounded up to 4
    uint32_t* frame_len;       // [n] out
    uint32_t n;
};

constexpr int kZwThreads = 256, kZwWarps = kZwThreads / 32, kZwPerThread = 16, kZwTile = kZwThreads * kZwPerThread;

__global__ void __launch_bounds__(kZwThreads, 4) k_zstd_frames(ZstdFrameJobs J) {
    __shared__ uint32_t whist[kZwWarps][256];
    __shared__ uint32_t hist[4][256];
    __shared__ uint32_t cnt[256];
    __shared__ uint32_t cl[256];  // code | len << 16
    __shared__ uint32_t red[kZwWarps];
    __shared__ uint32_t start[zw::kHufMaxBits + 1];
    __shared__ __align__(16) uint8_t tile[kZwTile];
    __shared__ zw::FramePlan P;
    __shared__ zw::HufWork W;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (uint32_t j = blockIdx.x; j < J.n; j += gridDim.x) {
        const uint64_t n = J.len[j];
        if (n == 0) {
            if (tid == 0) J.frame_len[j] = 0;
            continue;
        }
        const uint8_t* src = J.base + J.src_off[j];
        uint8_t* dst = J.base + J.slot_off[j];
        const int nseg = n <= zw::kSingleStreamMax ? 1 : 4;
        // ---- histograms of the segments: per-warp counts, then summed
        for (int k = 0; k < nseg; k++) {
            uint64_t b, e;
            zw::segment(n, nseg, k, &b, &e);
            for (int i = tid; i < kZwWarps * 256; i += kZwThreads) (&whist[0][0])[i] = 0;
            __syncthreads();
            for (uint64_t i = b + tid; i < e; i += kZwThreads) atomicAdd(&whist[wid][src[i]], 1u);
            __syncthreads();
            uint32_t c = 0;
#pragma unroll
            for (int w = 0; w < kZwWarps; w++) c += whist[w][tid];
            hist[k][tid] = c;
            cnt[tid] = (k ? cnt[tid] : 0u) + c;
            __syncthreads();
        }
        if (tid == 0) zw::plan_table(P, n, cnt, W);
        __syncthreads();
        if (P.mode == zw::kHuf) {
            // bits per segment (block reductions), canonical codes one symbol per thread
            const uint32_t ln = P.lens[tid];
            for (int k = 0; k < nseg; k++) {
                uint32_t v = hist[k][tid] * ln;
#pragma unroll
                for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(VMB_FULL, v, o);
                if (lane == 0) red[wid] = v;
                __syncthreads();
                if (tid == 0) {
                    uint32_t t = 0;
                    for (int w = 0; w < kZwWarps; w++) t += red[w];
                    P.seg_bits[k] = t;
                }
                __syncthreads();
            }
            if (tid == 0) {
                zw::code_starts(start, P.lens, P.maxbits);
                zw::plan_layout(P);
            }
            __syncthreads();
            if (P.mode == zw::kHuf && ln) {
                uint32_t rank = 0;
                for (int t = 0; t < tid; t++) rank += P.lens[t] == ln;
                cl[tid] = zw::canonical_code(start, (int)ln, rank, P.maxbits) | (ln << 16);
            }
        }
        // ---- the frame: zeroed words, the head, then the body
        const uint64_t flen = P.frame_len;
        uint32_t* dw = reinterpret_cast<uint32_t*>(dst);
        if (P.mode == zw::kHuf)
            for (uint64_t i = tid; i < (flen + 3) / 4; i += kZwThreads) dw[i] = 0;
        __syncthreads();
        for (int i = tid; i < P.head_len; i += kZwThreads) dst[i] = P.head[i];
        if (tid == 0) J.frame_len[j] = (uint32_t)flen;
        if (P.mode == zw::kRle) {
            if (tid == 0) dst[P.head_len] = src[0];
        } else if (P.mode == zw::kRaw) {
            uint8_t* o = dst + P.head_len;
            for (uint64_t pos = 0; pos < n; pos += zw::kMaxBlock) {
                const uint64_t c = n - pos < zw::kMaxBlock ? n - pos : zw::kMaxBlock;
                if (tid == 0) zw::block_header(o, pos + c == n, 0, (uint32_t)c);
                for (uint64_t i = tid; i < c; i += kZwThreads) o[3 + i] = src[pos + i];
                o += 3 + c;
            }
        } else {
            __syncthreads();  // head bytes before the merges into the words they share
            for (int k = 0; k < nseg; k++) {
                uint64_t b, e;
                zw::segment(n, nseg, k, &b, &e);
                const uint32_t m = (uint32_t)(e - b);
                const uint64_t sbase = (uint64_t)P.stream_off[k] * 8;  // bit 0 of the stream in the frame
                uint64_t carry = 0;
                for (uint32_t r0 = 0; r0 < m; r0 += kZwTile) {
                    // tile in stream order: position r holds the symbol at e - 1 - r
                    const uint32_t tn = m - r0 < (uint32_t)kZwTile ? m - r0 : (uint32_t)kZwTile;
                    const uint64_t hi = e - 1 - r0;  // the symbol at r = r0
                    for (uint32_t i = tid; i < tn; i += kZwThreads) tile[tn - 1 - i] = src[hi - (tn - 1) + i];
                    __syncthreads();
                    uint32_t mine[kZwPerThread];
                    uint32_t bits = 0;
                    const uint32_t q0 = (uint32_t)tid * kZwPerThread;
#pragma unroll
                    for (int q = 0; q < kZwPerThread; q++) {
                        mine[q] = q0 + q < tn ? cl[tile[q0 + q]] : 0u;
                        bits += mine[q] >> 16;
                    }
                    // exclusive scan of the bit counts over the CTA
                    uint32_t inc = bits;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const uint32_t t = __shfl_up_sync(VMB_FULL, inc, o);
                        if (lane >= o) inc += t;
                    }
                    if (lane == 31) red[wid] = inc;
                    __syncthreads();
                    uint32_t before = 0, total = 0;
#pragma unroll
                    for (int w = 0; w < kZwWarps; w++) {
                        before += w < wid ? red[w] : 0u;
                        total += red[w];
                    }
                    if (bits) {
                        const uint64_t p = sbase + carry + before + inc - bits;
                        uint64_t w = p >> 5;
                        int c = (int)(p & 31);
                        const bool shared_first = c != 0;
                        bool first = true;
                        uint64_t acc = 0;
#pragma unroll
                        for (int q = 0; q < kZwPerThread; q++) {
                            acc |= (uint64_t)(mine[q] & 0xffffu) << c;
                            c += (int)(mine[q] >> 16);
                            if (c >= 32) {
                                if (first && shared_first) atomicOr(dw + w, (uint32_t)acc);
                                else dw[w] = (uint32_t)acc;
                                first = false;
                                acc >>= 32;
                                c -= 32;
                                w++;
                            }
                        }
                        if (c) atomicOr(dw + w, (uint32_t)acc);
                    }
                    carry += total;
                    __syncthreads();
                }
                if (tid == 0) {  // the end mark after the last symbol
                    const uint64_t p = sbase + P.seg_bits[k];
                    atomicOr(dw + (p >> 5), 1u << (p & 31));
                }
            }
        }
        __syncthreads();
    }
}

// the 0.9 rule of encoding.go:156 for the columns the writer compressed, and what each column's payload is: the frame, or its
// varint stream (MarshalType 1 -> 5, 4 -> 6 where the frame was rejected or never made)
__global__ void k_marshal_select(const uint32_t* __restrict__ sizes, const uint64_t* __restrict__ soffs, const ZstdFrameJobs J,
                                 uint8_t* __restrict__ mts, uint64_t* __restrict__ copy_src, uint32_t* __restrict__ copy_len, uint32_t ncols) {
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < ncols; c += gridDim.x * blockDim.x) {
        uint32_t mt = mts[c];
        const uint32_t sz = sizes[c], fl = J.len[c] ? J.frame_len[c] : 0u;
        if (mt == 1 || mt == 4) {
            if (fl == 0 || (double)fl > 0.9 * (double)sz) mt = mt == 1 ? 5u : 6u;
        }
        const bool framed = mt == 1 || mt == 4;
        copy_src[c] = framed ? J.slot_off[c] : soffs[c];
        copy_len[c] = framed ? fl : sz;
        mts[c] = (uint8_t)mt;
    }
}

// offs[0..n] = exclusive prefix sum of len[0..n): one CTA
__global__ void __launch_bounds__(1024) k_scan_lens(const uint32_t* __restrict__ len, uint64_t* __restrict__ offs, uint32_t n) {
    __shared__ uint64_t wsum[32];
    __shared__ uint64_t carry;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (uint32_t i0 = 0; i0 < n; i0 += 1024) {
        const uint32_t i = i0 + tid;
        const uint64_t v = i < n ? len[i] : 0ull;
        uint64_t inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t t = shfl_up_u64(inc, o);
            if (lane >= o) inc += t;
        }
        if (lane == 31) wsum[wid] = inc;
        __syncthreads();
        uint64_t before = carry;
        for (int w = 0; w < wid; w++) before += wsum[w];
        if (i < n) offs[i] = before + inc - v;
        __syncthreads();
        if (tid == 1023) carry = before + inc;
        __syncthreads();
    }
    if (tid == 0) offs[n] = carry;
}

// dst + offs[c] <- base + src[c], offs[c+1] - offs[c] bytes: one warp per item.  Source and destination are aligned differently,
// so the destination's aligned 32-bit words are stored whole, each put together from the two aligned source words it straddles
// (an aligned word holding an in-range byte lies inside the allocation); only the unaligned head and tail go byte by byte.
__global__ void __launch_bounds__(256) k_compact(const uint8_t* __restrict__ base, const uint64_t* __restrict__ src,
                                                 const uint64_t* __restrict__ offs, uint8_t* __restrict__ dst, uint32_t n) {
    const int lane = lane_id();
    const uint32_t wpg = gridDim.x * (blockDim.x >> 5);
    for (uint32_t c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c < n; c += wpg) {
        const uint8_t* s = base + src[c];
        uint8_t* d = dst + offs[c];
        const uint64_t len = offs[c + 1] - offs[c];
        const uint64_t head = min(len, (uint64_t)((4u - ((uint32_t)(uintptr_t)d & 3u)) & 3u));
        if ((uint64_t)lane < head) d[lane] = s[lane];
        const uint64_t nw = (len - head) >> 2;
        const uintptr_t sa = (uintptr_t)(s + head);
        const uint32_t* sw = reinterpret_cast<const uint32_t*>(sa & ~(uintptr_t)3);
        const uint32_t sh = (uint32_t)(sa & 3) * 8u;
        uint32_t* dw = reinterpret_cast<uint32_t*>(d + head);
        if (sh == 0)
            for (uint64_t k = lane; k < nw; k += 32) dw[k] = sw[k];
        else
            for (uint64_t k = lane; k < nw; k += 32) dw[k] = __funnelshift_r(sw[k], sw[k + 1], sh);
        const uint64_t done = head + nw * 4;
        if ((uint64_t)lane < len - done) d[done + lane] = s[done + lane];
    }
}

void launch_zstd_frames(const ZstdFrameJobs& J, cudaStream_t st) {
    if (!J.n) return;
    const uint32_t grid = J.n < VMB_SMS * 8u ? J.n : VMB_SMS * 8u;
    k_zstd_frames<<<grid, kZwThreads, 0, st>>>(J);
}
void launch_marshal_select(const uint32_t* sizes, const uint64_t* soffs, const ZstdFrameJobs& J, uint8_t* mts, uint64_t* copy_src,
                           uint32_t* copy_len, uint32_t ncols, cudaStream_t st) {
    uint32_t grid = (ncols + 255) / 256;
    if (grid > VMB_SMS * 8u) grid = VMB_SMS * 8u;
    k_marshal_select<<<grid, 256, 0, st>>>(sizes, soffs, J, mts, copy_src, copy_len, ncols);
}
void launch_scan_lens(const uint32_t* len, uint64_t* offs, uint32_t n, cudaStream_t st) { k_scan_lens<<<1, 1024, 0, st>>>(len, offs, n); }
void launch_compact(const uint8_t* base, const uint64_t* src, const uint64_t* offs, uint8_t* dst, uint32_t n, cudaStream_t st) {
    if (!n) return;
    uint32_t grid = (n + 7) / 8;
    if (grid > VMB_SMS * 16u) grid = VMB_SMS * 16u;
    k_compact<<<grid, 256, 0, st>>>(base, src, offs, dst, n);
}

void launch_marshal_plan(const MarshalParams& P, cudaStream_t st) {
    if (!P.ncols) return;
    uint32_t grid = (P.ncols + 3) / 4;
    if (grid > VMB_SMS * 16u) grid = VMB_SMS * 16u;
    k_marshal_plan<<<grid, 128, 0, st>>>(P);
}
void launch_marshal_pack(const MarshalParams& P, cudaStream_t st) {
    if (!P.ncols) return;
    uint32_t grid = (P.ncols + 3) / 4;
    if (grid > VMB_SMS * 16u) grid = VMB_SMS * 16u;
    k_marshal_pack<<<grid, 128, 0, st>>>(P);
}
