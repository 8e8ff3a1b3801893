// Column decode kernel: varint -> (double) prefix sum -> int64 timestamps / float64 values, one warp per block.
//
// Replaces, for every block of a batch at once:
//   lib/encoding/encoding.go:173   unmarshalInt64Array        (dispatch on MarshalType)
//   lib/encoding/int.go:182-284    UnmarshalVarInt64s         (zig-zag LEB128)
//   lib/encoding/nearest_delta.go:53, nearest_delta2.go:57    (prefix sum / double prefix sum)
//   lib/storage/block.go:250-296   Block.UnmarshalData        (validation, EnsureNonDecreasingSequence)
//   lib/storage/block.go:324-349   AppendRowsWithTimeRangeFilter / filterTimestamps
//   lib/decimal/decimal.go:100     AppendDecimalToFloat
//
// Layout: a warp walks the varint byte stream in 512-byte tiles (decode_stream.cuh): terminators are found byte-major,
// the values are then dealt out value-major, and per-lane partial sums are combined with one warp scan per tile
// ((count, sum, sum-of-prefix-sums) is an associative triple under wrapping int64 arithmetic), so the result is
// bit-identical to the sequential Go loop.
#include "common.cuh"

namespace {

__constant__ double c_pow10tab[32] = {1e00, 1e01, 1e02, 1e03, 1e04, 1e05, 1e06, 1e07, 1e08, 1e09, 1e10,
                                      1e11, 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21,
                                      1e22, 1e23, 1e24, 1e25, 1e26, 1e27, 1e28, 1e29, 1e30, 1e31};
__constant__ double c_pow10postab32[10] = {1e00, 1e32, 1e64, 1e96, 1e128, 1e160, 1e192, 1e224, 1e256, 1e288};
__constant__ double c_pow10negtab32[11] = {1e-00,  1e-32,  1e-64,  1e-96,  1e-128, 1e-160,
                                           1e-192, 1e-224, 1e-256, 1e-288, 1e-320};

}  // namespace

// Go stdlib math.Pow10: pow10postab32[n/32] * pow10tab[n%32] (a PRODUCT of two table doubles, not pow()).
__device__ double vmb_pow10(int n) {
    if (0 <= n && n <= 308) return __dmul_rn(c_pow10postab32[(unsigned)n / 32], c_pow10tab[(unsigned)n % 32]);
    if (-323 <= n && n <= 0) return __ddiv_rn(c_pow10negtab32[(unsigned)(-n) / 32], c_pow10tab[(unsigned)(-n) % 32]);
    if (n > 0) return __longlong_as_double(0x7ff0000000000000LL);
    return 0.0;
}

namespace {

struct Dec {  // decimal.AppendDecimalToFloat decimal.go:100 for one block (scale fixed)
    double e10, rcp;
    int mode;  // 0: e==0, -1: divide, -2: divide through the reciprocal (exact, see below), +1: multiply
    __device__ void init(int16_t e) {
        mode = e == 0 ? 0 : (e < 0 ? -1 : 1);
        e10 = e < 0 ? vmb_pow10(-(int)e) : vmb_pow10((int)e);
        rcp = 0.0;
        // x / 10^k for 1 <= k <= 22 (10^k exact in binary64, quotients of int64-range x stay normal): with r = RN(1/p),
        // q = RN(x*r), rem = x - q*p (exact by FMA), RN(q + rem*r) is the correctly rounded quotient (Markstein's
        // division step), i.e. bit-identical to the IEEE division Go performs, at 3 flops instead of ~30 instructions.
        // Checked at random on the host for every k (440 M operands, 0 mismatches) and on the GPU against the oracle's
        // IEEE division by tests/test_gpu_parity.py::test_decimal_to_float_kats_bit_exact.
        if (e < 0 && e >= -22) {
            mode = -2;
            rcp = __drcp_rn(e10);
        }
    }
    // the arithmetic of conv() alone: for mantissas that are not one of the three special values (the caller checks)
    __device__ __forceinline__ double conv_plain(int64_t v) const {
        double f = __ll2double_rn(v);
        if (mode == -2) {
            double q = __dmul_rn(f, rcp);
            double rem = __fma_rn(-q, e10, f);
            f = __fma_rn(rem, rcp, q);
        } else if (mode < 0) f = __ddiv_rn(f, e10);
        else if (mode > 0) f = __dmul_rn(f, e10);
        return f;
    }
    __device__ __forceinline__ double conv(int64_t v) const {
        double f = __ll2double_rn(v);
        if (mode == -2) {
            double q = __dmul_rn(f, rcp);
            double rem = __fma_rn(-q, e10, f);
            f = __fma_rn(rem, rcp, q);
        } else if (mode < 0) f = __ddiv_rn(f, e10);
        else if (mode > 0) f = __dmul_rn(f, e10);
        // isSpecialValue decimal.go:417: v in {vStaleNaN = 2^63-2, vInfPos = 2^63-1, vInfNeg = -2^63}, three consecutive
        // values in wrapping arithmetic: one unsigned range test instead of three 64-bit comparisons
        if ((uint64_t)v - 0x7FFFFFFFFFFFFFFEull < 3ull) {
            if (v == VMB_V_INF_POS) f = __longlong_as_double(0x7ff0000000000000LL);
            else if (v == VMB_V_INF_NEG) f = __longlong_as_double((long long)0xfff0000000000000ULL);
            else f = __longlong_as_double((long long)VMB_STALE_NAN_BITS);
        }
        return f;
    }
};

// timestamps emitter: stores int64, validates monotonicity (block.go:298) and tracks the time-range trim
struct TsEmit {
    int64_t* out;
    int64_t tr_min, tr_max;
    uint32_t lo, hi1;  // lane-local: min pos with ts >= tr_min ; 1 + max pos with ts <= tr_max
    bool validate, bad_order;
    bool inside;       // every value of the column is known to lie inside [tr_min, tr_max]: nothing to track
    __device__ void init(int64_t* o, int64_t a, int64_t b, bool v) {
        out = o; tr_min = a; tr_max = b; lo = 0xffffffffu; hi1 = 0; validate = v; bad_order = false; inside = false;
    }
    __device__ __forceinline__ void emit(uint32_t pos, int64_t v, int64_t prev) {
        out[pos] = v;
        if (validate && v < prev) bad_order = true;
        if (!inside) {
            if (v >= tr_min && pos < lo) lo = pos;
            if (v <= tr_max && pos + 1 > hi1) hi1 = pos + 1;
        }
    }
    __device__ __forceinline__ void note_decrease() {}
    // a non-decreasing arithmetic progression first..last with n values: inside the range as a whole?
    __device__ __forceinline__ void note_progression(int64_t first, int64_t last, uint32_t n) {
        if (first <= last && first >= tr_min && last <= tr_max) {
            inside = true;
            lo = 0;
            hi1 = n;
        }
    }
};

struct ValEmit {
    void* out;
    Dec dec;
    bool as_int;
    bool saw_stale;  // a Prometheus staleness marker (decimal.go:406 vStaleNaN) was emitted: dropStaleNaNs has work to do
    uint32_t first_drop;  // first row whose mantissa is below its predecessor (lane-local minimum)
    bool saw_drop;   // some mantissa is below its predecessor: the only way removeCounterResets (rollup.go:921) can change
                     // this block (decimal -> float is monotone inside a block: one scale), besides NaNs (saw_stale)
    __device__ void init(void* o, int16_t scale, bool ai) {
        out = o; as_int = ai; saw_stale = false; saw_drop = false; first_drop = 0xffffffffu; dec.init(scale);
    }
    __device__ __forceinline__ void note_decrease() { saw_drop = true; first_drop = 1; }
    __device__ __forceinline__ void note_progression(int64_t, int64_t, uint32_t) {}
    __device__ __forceinline__ void emit(uint32_t pos, int64_t v, int64_t pv) {
        if ((uint64_t)v - 0x7FFFFFFFFFFFFFFEull < 3ull) saw_stale |= (v == VMB_V_STALE_NAN);
        if (v < pv) {
            saw_drop = true;
            first_drop = min(first_drop, pos);
        }
        if (as_int) ((int64_t*)out)[pos] = v;
        else ((double*)out)[pos] = dec.conv(v);
    }
};

__device__ __forceinline__ uint32_t term_mask4(uint32_t w) {
    // the four sign bits moved to bits 0, 8, 16, 24, then gathered by one multiplication: t * (2^21 + 2^14 + 2^7 + 1) puts them at
    // bits 21..24 (every other partial product lands on a bit of its own below 21 or above 24: no carries)
    const uint32_t t = (~w & 0x80808080u) >> 7;
    return ((t * 0x204081u) >> 21) & 0xfu;
}

// UnmarshalVarInt64 int.go:173 (binary.Uvarint + zig-zag) on <= 11 bytes, executed redundantly by every lane
__device__ int read_single_varint(const uint8_t* src, uint32_t len, int64_t* out, uint32_t* used) {
    uint64_t u = 0;
    uint32_t shift = 0;
    for (uint32_t i = 0; i < len; i++) {
        if (i == 10) return VMB_ERR_DELTA_CONST;
        uint32_t b = src[i];
        if (b < 0x80) {
            if (i == 9 && b > 1) return VMB_ERR_DELTA_CONST;
            u |= (uint64_t)b << shift;
            *out = (int64_t)(u >> 1) ^ -(int64_t)(u & 1);
            *used = i + 1;
            return 0;
        }
        u |= (uint64_t)(b & 0x7f) << shift;
        shift += 7;
    }
    return VMB_ERR_DELTA_CONST;
}

}  // namespace
#include "decode_stream.cuh"
namespace {

template <class E>
__device__ int decode_column(const uint8_t* src, uint32_t len, int mt, int64_t first, uint32_t n, E& em, DecodeSmem* sm) {
    const int lane = lane_id();
    switch (mt) {
        case 1:  // MarshalTypeZSTDNearestDelta2 (src already decompressed into the scratch arena)
        case 5:  // MarshalTypeNearestDelta2
            return decode_delta_stream_v2(src, len, n, first, true, em, sm);
        case 4:  // MarshalTypeZSTDNearestDelta
        case 6:  // MarshalTypeNearestDelta
            return decode_delta_stream_v2(src, len, n, first, false, em, sm);
        case 3: {  // MarshalTypeConst encoding.go:215
            if (len > 0) return VMB_ERR_CONST_TAIL;
            for (uint32_t i = lane; i < n; i += 32) em.emit(i, first, first);
            return 0;
        }
        case 2: {  // MarshalTypeDeltaConst encoding.go:231
            int64_t d = 0;
            uint32_t used = 0;
            int rc = read_single_varint(src, len, &d, &used);
            if (rc) return rc;
            if (used < len) return VMB_ERR_TAIL;
            // non-decreasing as a whole?  d >= 0 is not enough: first + i*d wraps like the Go loop (encoding.go:240 v += d), e.g.
            // the two-row column {5216, MinInt64+1} is stored as delta-const with a positive (wrapped) delta
            const int64_t last = (int64_t)((uint64_t)first + (uint64_t)(n - 1) * (uint64_t)d);
            const bool monotone = d >= 0 && (n == 1 || (uint64_t)d <= (uint64_t)0x7fffffffffffffffLL / (n - 1)) && last >= first;
            if (monotone) em.note_progression(first, last, n);
            for (uint32_t i = lane; i < n; i += 32) {
                int64_t v = (int64_t)((uint64_t)first + (uint64_t)i * (uint64_t)d);
                em.emit(i, v, v);
            }
            if (!monotone) em.note_decrease();
            return 0;
        }
        default:
            return VMB_ERR_MARSHAL_TYPE;
    }
}

}  // namespace

struct DecodeParams {
    const vmb_block_desc* descs;
    const ColInfo* cols;
    const uint8_t* payload;
    const uint8_t* scratch;       // zstd output arena
    const int32_t* zstd_status;   // per column (2*nblocks) or nullptr
    const ColInfo* zstd_cols;     // the column infos the zstd stage ran on: their content_size is the length each frame produced
    const uint32_t* blk_map;      // sub-batch of a larger upload: block b is block blk_map[b] of the batch zstd_status belongs to
    const uint64_t* row_off;      // per block: first row in the dense columns
    int64_t* ts_out;
    void* val_out;
    uint32_t* blk_lo;             // per block: kept rows [lo, hi)
    uint32_t* blk_hi;
    int32_t* status;              // per block
    uint32_t nblocks;
    uint32_t flags;
    int64_t tr_min, tr_max;
};

__global__ void __launch_bounds__(128) k_decode_columns(DecodeParams P) {
    __shared__ DecodeSmem s_dec[4];
    DecodeSmem* sm = &s_dec[threadIdx.x >> 5];
    const int lane = lane_id();
    const uint32_t warps_per_grid = gridDim.x * (blockDim.x >> 5);
    for (uint32_t b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); b < P.nblocks; b += warps_per_grid) {
        const vmb_block_desc d = P.descs[b];
        const uint64_t ro = P.row_off[b];
        int rc = 0;
        uint32_t lo = 0, hi = 0;
        const uint32_t zb = P.blk_map ? P.blk_map[b] : b;
        if (d.rows == 0 || d.rows > 16384u) rc = VMB_ERR_ROWS;  // block.go:262, block_header.go:233
        if (!rc && P.zstd_status) {
            int z0 = P.zstd_status[2 * zb], z1 = P.zstd_status[2 * zb + 1];
            if (z0) rc = z0;
            else if (z1) rc = z1;
        }
        if (!rc) {
            // ---- timestamps (encoding.UnmarshalTimestamps encoding.go:90)
            const ColInfo ci = P.cols[2 * b];
            const uint8_t* src = ci.kind == VMB_ZK_NONE ? P.payload + d.ts_off : P.scratch + ci.scratch_off;
            uint32_t len = ci.kind == VMB_ZK_NONE ? d.ts_size : P.zstd_cols[2 * zb].content_size;
            TsEmit te;
            const bool needs_validation = d.precision_bits >= 64 && (d.ts_mt == 5 || d.ts_mt == 6);  // encoding.go:46
            te.init(P.ts_out + ro, P.tr_min, P.tr_max, needs_validation);
            rc = decode_column(src, len, d.ts_mt, d.min_ts, d.rows, te, sm);
            __syncwarp();
            if (!rc && d.precision_bits < 64) {
                // EnsureNonDecreasingSequence encoding.go:258 == a[0]=min; prefix max; clamp to max; a[n-1]=max
                int64_t* a = P.ts_out + ro;
                int64_t run = d.min_ts;
                te.lo = 0xffffffffu;
                te.hi1 = 0;
                for (uint32_t base = 0; base < d.rows; base += 32) {
                    uint32_t i = base + lane;
                    int64_t x = i < d.rows ? a[i] : INT64_MIN;
                    if (i == 0) x = d.min_ts;
#pragma unroll
                    for (int off = 1; off < 32; off <<= 1) {
                        int64_t y = (int64_t)shfl_up_u64((uint64_t)x, off);
                        if (lane >= off && y > x) x = y;
                    }
                    if (run > x) x = run;
                    run = (int64_t)shfl_u64((uint64_t)x, 31);
                    if (i < d.rows) {
                        int64_t o = (i == d.rows - 1) ? d.max_ts : (x < d.max_ts ? x : d.max_ts);
                        a[i] = o;
                        if (o >= P.tr_min && i < te.lo) te.lo = i;
                        if (o <= P.tr_max && i + 1 > te.hi1) te.hi1 = i + 1;
                    }
                }
            } else if (!rc && needs_validation) {
                // checkTimestampsBounds block.go:298: order (tracked while emitting) and last <= MaxTimestamp
                bool bad = __any_sync(VMB_FULL, te.bad_order);
                __syncwarp();
                if (bad || P.ts_out[ro + d.rows - 1] > d.max_ts) rc = VMB_ERR_TS_BOUNDS;
            }
            if (!rc) {
                uint32_t l = te.lo, h = te.hi1;
#pragma unroll
                for (int off = 16; off; off >>= 1) {
                    l = min(l, __shfl_xor_sync(VMB_FULL, l, off));
                    h = max(h, __shfl_xor_sync(VMB_FULL, h, off));
                }
                lo = l == 0xffffffffu ? d.rows : l;  // filterTimestamps block.go:331
                hi = h > lo ? h : lo;
            }
        }
        if (!rc) {
            // ---- values (encoding.UnmarshalValues encoding.go:111 + decimal.AppendDecimalToFloat)
            const ColInfo ci = P.cols[2 * b + 1];
            const uint8_t* src = ci.kind == VMB_ZK_NONE ? P.payload + d.val_off : P.scratch + ci.scratch_off;
            uint32_t len = ci.kind == VMB_ZK_NONE ? d.val_size : P.zstd_cols[2 * zb + 1].content_size;
            ValEmit ve;
            const bool as_int = (P.flags & VMB_DECODE_VALUES_AS_INT64) != 0;
            ve.init(as_int ? (void*)((int64_t*)P.val_out + ro) : (void*)((double*)P.val_out + ro), d.scale, as_int);
            rc = decode_column(src, len, d.val_mt, d.first_value, d.rows, ve, sm);
            const bool may_change = __any_sync(VMB_FULL, ve.saw_stale || ve.saw_drop);
            uint32_t fd = 0;
            if (may_change) {
                fd = ve.first_drop;
#pragma unroll
                for (int off = 16; off; off >>= 1) fd = min(fd, __shfl_xor_sync(VMB_FULL, fd, off));
                fd = fd < 16384u ? fd : 0u;
            }
            hi = blk_hi_pack(hi, fd, may_change, __any_sync(VMB_FULL, ve.saw_stale));
        }
        if (lane == 0) {
            P.status[b] = rc;
            P.blk_lo[b] = rc ? 0u : lo;
            P.blk_hi[b] = rc ? 0u : hi;
        }
    }
}

void launch_decode_columns(const DecodeParams& P, cudaStream_t st) {
    if (P.nblocks == 0) return;
    int warps = 4;
    uint32_t grid = (P.nblocks + warps - 1) / warps;
    uint32_t maxgrid = VMB_SMS * 16u;
    if (grid > maxgrid) grid = maxgrid;
    k_decode_columns<<<grid, warps * 32, 0, st>>>(P);
}

// ---- decimal.AppendDecimalToFloat as a flat elementwise kernel (per-call drop-in vmb_decimal_to_float)
__global__ void k_decimal_to_float(double* __restrict__ dst, const int64_t* __restrict__ va, size_t n, int16_t e) {
    Dec dec;
    dec.init(e);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        dst[i] = dec.conv(va[i]);
}

void launch_decimal_to_float(double* dst, const int64_t* va, size_t n, int16_t e, cudaStream_t st) {
    if (!n) return;
    size_t blocks = (n + 255) / 256;
    if (blocks > VMB_SMS * 32) blocks = VMB_SMS * 32;
    k_decimal_to_float<<<(unsigned)blocks, 256, 0, st>>>(dst, va, n, e);
}
