// Fused series kernel: varint / nearest-delta(2) decode -> decimal->float -> removeCounterResets -> rollupConfig.Do in ONE CTA per
// series, the decoded column living only in shared memory.
//
// Reference shape (one goroutine per series, nothing materialised per batch):
//   app/vmselect/promql/eval.go:1855-1866   the per-series closure of evalRollupNoIncrementalAggregate
//   app/vmselect/netstorage/netstorage.go:425  packedTimeseries.Unpack
//   lib/storage/block.go:250-296            Block.UnmarshalData  (lib/encoding/encoding.go:173 unmarshalInt64Array,
//                                           nearest_delta2.go:57, nearest_delta.go:53, int.go:182-284)
//   lib/decimal/decimal.go:100              AppendDecimalToFloat
//   app/vmselect/promql/rollup.go:921       removeCounterResets
//   app/vmselect/promql/rollup.go:701-823   rollupConfig.doInternal + the rollup functions
//
// What the un-fused pipeline (k_decode_columns -> k_series_assemble -> k_series_prepare -> k_rollup) writes to and re-reads
// from HBM -- 16 bytes per sample of decoded columns -- never leaves the SM here: per series the kernel reads the varint bytes
// once (TMA bulk copies into a double-buffered shared-memory stage, completion on an mbarrier) and writes the result row once.
//
// Scope: series made of ONE block whose timestamps column is MarshalTypeDeltaConst at precisionBits = 64 (rows sit at
// t0 + row * dt: no timestamp is ever materialised), inside the query's time range, without staleness markers when they
// would have to be dropped.  Everything else -- multi-block series, jittered timestamp columns, corrupt input, windows that
// do not fit the resident rows -- is handed to the un-fused pipeline through a device-side bail list; the host runs it for
// exactly those series afterwards (same output rows), so every error code and corner case keeps its one implementation.
//
// Decode inside the CTA (4 warps, one 1 KB tile each per fill):
//   1. every lane takes 2 x 16 bytes of its warp's tile, finds the varint terminators (bytes < 0x80); counts are scanned over
//      the warp and over the CTA, which gives every lane the row of its first value;
//   2. a lane decodes the varints whose terminator lies in each of its 16-byte groups (7-bit groups compacted once, then one
//      shift-and-mask per value; the bytes of a varint that starts in the previous 16 bytes are carried in), zig-zag decodes
//      them, stores them raw at their rows and keeps (count, sum, sum of prefix sums);
//   3. the triples are combined over the lanes and over the warps -- (s2A + s2B + cntB * s1A) is associative under wrapping
//      int64 arithmetic, so the prefix sums are bit-identical to the sequential Go loop; with the counts known from step 1 the
//      combination is two plain sum scans: s1, then t = s2 + cnt * (exclusive prefix of s1);
//   4. every lane replays its values with the scanned prefix, converts mantissa -> float64 (decimal.go:100) and overwrites
//      the raw value in place.
#pragma once
#include <type_traits>

#define FU_THREADS 128
#define FU_WARPS 4
#define FU_CTAS_PER_SM 5                  /* __launch_bounds__ minimum: 5 x ~43 KB of shared memory, 96 registers per thread */
#define FU_CTAS_PER_SM_OVERLAP 4          /* grid beside the zstd stage of the next chunk: leaves 16 k registers, ~50 KB */
#define FU_CAP 4096                       /* rows of one series resident in shared memory */
#define FU_G 2                            /* 16-byte groups per lane and fill: 4 warps x 32 lanes x 32 bytes = one 4 KB fill */
#define FU_TILE (512 * FU_G)
#define FU_FILL (FU_WARPS * FU_TILE)      /* bytes staged per fill */
#define FU_STAGE (16 + FU_FILL + 16)      /* 16 bytes of the previous tile in front, 16 bytes of padding behind */
#define FU_MAX_EVENTS 32                  /* counter resets inside one fill handled by the parallel path */

// Phase-clock build (-DVMB_FUSED_PHASES, scripts/exp_fused_phases.py; never the product): lane 0 of every warp adds the clock64()
// cycles since its previous mark to the phase that just ended, and the CTA's totals land in fu_phase_cyc[blockIdx.x].  Without
// the macro FU_PH() expands to nothing and the kernel compiles to the same SASS.
enum {
    FU_PH_SETUP,   // series setup, the first copy of a series, the tail of a series
    FU_PH_TERM,    // terminator scan and the tile counts
    FU_PH_PARSE,   // varint parse (and generated rows of constant columns)
    FU_PH_SCAN,    // the two sum scans over the warp and over the warps
    FU_PH_EMIT,    // replay of the values and float conversion
    FU_PH_RCR,     // counter-reset work
    FU_PH_POINTS,  // points and the slide of the resident rows
    FU_PH_WAIT,    // barriers, and copies of fills after a series' first
    FU_PH_N,
    FU_PH_FILLS = FU_PH_N,  // counters kept by warp 0: fills, series
    FU_PH_SERIES,
    FU_PH_SLOTS
};
#ifdef VMB_FUSED_PHASES
#define FU_PH_CTAS (VMB_SMS * FU_CTAS_PER_SM)
__device__ unsigned long long fu_phase_cyc[FU_PH_CTAS][FU_PH_SLOTS];
#define FU_PH(k)                                              \
    do {                                                      \
        const long long ph_c = clock64();                     \
        if (lane == 0) S.ph[w][(k)] += (unsigned long long)(ph_c - ph_t); \
        ph_t = ph_c;                                          \
    } while (0)
#define FU_PH_COUNT(k) \
    do {               \
        if (tid == 0) S.ph[0][(k)]++; \
    } while (0)
#else
#define FU_PH(k) ((void)0)
#define FU_PH_COUNT(k) ((void)0)
#endif

struct FusedParams {
    const vmb_block_desc* descs;
    const ColInfo* cols;
    const uint8_t* payload;
    const uint8_t* scratch;          // zstd output arena
    const int32_t* zstd_status;      // per column (2*nblocks) or nullptr
    const uint32_t* ser_list;        // series handled by this launch
    const uint32_t* ser_first_block; // per series
    vmb_rollup_cfg cfg;              // args / args2: DEVICE pointers
    double* out;                     // [nseries x P]
    unsigned long long* scanned;
    uint32_t* bail_list;             // series this kernel could not finish (-> un-fused pipeline)
    unsigned int* bail_count;
    uint32_t nlist;
    uint32_t npoints;
    int64_t tr_min, tr_max;
    // incremental aggregate sink (aggr_incremental.go:98 updateTimeseries): with aggr_values set, `out` is a scratch of one row
    // per CTA ([gridDim.x x P], L2 resident); a series that made it to its end is folded from there into {values, counts}
    // [group x P] of its group (red.global: the cells of a query live in L2) -- a series handed to the un-fused path folds nothing
    double* aggr_values;
    double* aggr_counts;
    const uint32_t* group_ids;       // per series (device)
    int aggr_id;
};

namespace {

// what one thread derives from the block header and the query for a series (everybody else reads it from shared memory)
struct FuSeries {
    const uint8_t* A;        // 16-byte aligned base of the values stream; stream byte i sits at A[shift + i]
    int64_t t_org, dts, window, max_prev, dconst, first_value;
    uint32_t shift, len, n, end_al;
    int32_t start_r, step32, win32, mpi32;  // the query grid relative to the first row, all below 2^30 in magnitude
    int32_t lin_k, iq0, jq0;                // step % dt == 0: the window edges of point q are iq0 + q * lin_k, jq0 + q * lin_k
    double dec_e10, dec_rcp;                // Dec (decimal.go:100) of the block's scale
    double rate_D, rate_R;                  // rate(): divisor of a full window and its reciprocal (rate_dt = the span in ms, -1: none)
    int32_t rate_dt, rate_rows, dec_mode;
    uint32_t s;              // the series (its output row)
    int16_t scale;
    uint8_t bail, is_stream, delta2, do_rcr, stale_matters, lin;
};

struct FusedSmem {
    double val[FU_CAP];
    alignas(16) uint8_t stage[2][FU_STAGE];
    unsigned long long mbar[2];
    unsigned long long w_s1[FU_WARPS], w_s2[FU_WARPS];
    uint32_t w_cnt[FU_WARPS];
    double ev_amt[FU_MAX_EVENTS], ev_cum[FU_MAX_EVENTS];
    uint32_t ev_row[FU_MAX_EVENTS];
    uint32_t nev;
    unsigned long long nd_v, nd_d1;  // nearest-delta(2) state in front of the next fill: last value, last delta
    uint32_t flags;  // bit 0: bail (set while parsing, read behind the barrier that ends the parse)
    uint32_t flags_emit;  // the same for the emit pass: a word of its own, so that a warp already emitting cannot race a warp still reading `flags`
    unsigned long long s_part[FU_WARPS];
    unsigned long long s_thr[FU_THREADS];  // this thread's share of samplesScanned over the series the CTA finished
    unsigned long long s_ser[FU_THREADS];  // the same for the current series (dropped when it is handed to the un-fused path)
    FuSeries ser;  // the current series (read where it is used: it stays valid for the whole series)
#ifdef VMB_FUSED_PHASES
    unsigned long long ph[FU_WARPS][FU_PH_SLOTS];
#endif
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// waits for the phase with the given parity; a copy that never lands (a driver / addressing fault) traps instead of hanging
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) {
            if ((threadIdx.x & 31) == 0) printf("fused: TMA copy did not land (block %u warp %u parity %u)\n", blockIdx.x, threadIdx.x >> 5, parity);
            __trap();
        }
    }
}
// 1-D bulk copy global -> shared through the TMA engine; completion is signalled on the mbarrier (complete_tx)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// Resident rows: absolute row r of the series lives at val[fu_swz(r)] -- a ring over FU_CAP rows (sliding the window moves
// no data) whose low index bits are XOR-swizzled with bits 3..6: the lanes of a warp write / replay runs of ~8 consecutive
// rows each (stride 64 bytes: two banks without the swizzle, a 16-way conflict), and the points read consecutive rows; both
// patterns spread over all banks this way.
#define FU_MASK (FU_CAP - 1)
__device__ __forceinline__ uint32_t fu_swz(uint32_t row) {
    row &= FU_MASK;
    return row ^ ((row >> 3) & 15u);
}
// the same on byte offsets (row * 8): three instructions per access
__device__ __forceinline__ uint32_t fu_swz_b(uint32_t row) {
    const uint32_t o = row << 3;
    return (o ^ ((o >> 3) & 0x78u)) & (uint32_t)(FU_CAP * 8 - 1);
}
__device__ __forceinline__ double fu_ld(const double* s, uint32_t row) {
    return *reinterpret_cast<const double*>(reinterpret_cast<const char*>(s) + fu_swz_b(row));
}
__device__ __forceinline__ double& fu_ref(double* s, uint32_t row) {
    return *reinterpret_cast<double*>(reinterpret_cast<char*>(s) + fu_swz_b(row));
}
// the same through a 32-bit shared-space address of val[] (no generic -> shared window arithmetic per access)
__device__ __forceinline__ double fu_lds(uint32_t val_s, uint32_t row) {
    double v;
    asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(val_s + fu_swz_b(row)));
    return v;
}
__device__ __forceinline__ void fu_sts(uint32_t val_s, uint32_t row, double v) {
    asm volatile("st.shared.f64 [%0], %1;" ::"r"(val_s + fu_swz_b(row)), "d"(v) : "memory");
}
__device__ __forceinline__ long long fu_lds_i64(uint32_t val_s, uint32_t row) {
    long long v;
    asm volatile("ld.shared.b64 %0, [%1];" : "=l"(v) : "r"(val_s + fu_swz_b(row)));
    return v;
}
__device__ __forceinline__ void fu_sts_i64(uint32_t val_s, uint32_t row, long long v) {
    asm volatile("st.shared.b64 [%0], %1;" ::"r"(val_s + fu_swz_b(row)), "l"(v) : "memory");
}
struct FuVals {  // read view for the rollup functions: element i is row r + i
    const double* s;
    uint32_t r;
    __device__ __forceinline__ double operator[](int32_t i) const { return fu_ld(s, r + i); }
    __device__ __forceinline__ FuVals operator+(uint32_t k) const { return FuVals{s, r + k}; }
    __device__ __forceinline__ FuVals& operator++() { r++; return *this; }
    __device__ __forceinline__ FuVals operator++(int) { FuVals o = *this; r++; return o; }
};
struct FuValsRW {  // read/write by absolute row
    double* s;
    __device__ __forceinline__ double& operator[](uint32_t row) const { return fu_ref(s, row); }
};
struct FuTs {  // timestamps of a MarshalTypeDeltaConst column are never stored: element i is t + i * dt
    int64_t t, dt;
    __device__ __forceinline__ int64_t operator[](int64_t i) const { return t + i * dt; }  // (i = -1: the row in front)
    __device__ __forceinline__ FuTs operator+(uint32_t k) const { return FuTs{t + (int64_t)k * dt, dt}; }
    __device__ __forceinline__ FuTs& operator++() { t += dt; return *this; }
    __device__ __forceinline__ FuTs operator++(int) { FuTs o = *this; t += dt; return o; }
};

__device__ __forceinline__ uint32_t fu_term_mask16(const uint4& c) {
    return term_mask4(c.x) | (term_mask4(c.y) << 4) | (term_mask4(c.z) << 8) | (term_mask4(c.w) << 12);
}
// bits k of a 16-byte group at stream position g0 that lie inside [lo, hi)
__device__ __forceinline__ uint32_t fu_valid16(int64_t g0, int64_t lo, int64_t hi) {
    int64_t a = lo - g0, b = hi - g0;
    a = a < 0 ? 0 : (a > 16 ? 16 : a);
    b = b < 0 ? 0 : (b > 16 ? 16 : b);
    if (b <= a) return 0u;
    return ((1u << b) - 1u) & ~((1u << a) - 1u);
}
__device__ __forceinline__ uint32_t compact7(uint32_t w) {
    return (w & 0x7fu) | ((w & 0x7f00u) >> 1) | ((w & 0x7f0000u) >> 2) | ((w & 0x7f000000u) >> 3);
}

// max / min on a double cell by integer atomics (no NaN operands).  Doubles with the sign bit clear order like signed integers
// and sit above every double with it set; those order in reverse as unsigned integers and sit above every other double there:
//   max: sign clear -> signed max, set -> unsigned min;   min: sign clear -> signed min, set -> unsigned max.
// So -0.0 ranks just below +0.0: a cell whose series all give -0.0 keeps -0.0, as the reference's fold does; for a mix of
// the two zeros the result is the one the reference gets when that zero comes first (its order is scheduling dependent too).
__device__ __forceinline__ void fu_atomic_max(double* a, double v) {
    const long long b = __double_as_longlong(v);
    if (b >= 0) atomicMax((long long*)a, b);
    else atomicMin((unsigned long long*)a, (unsigned long long)b);
}
__device__ __forceinline__ void fu_atomic_min(double* a, double v) {
    const long long b = __double_as_longlong(v);
    if (b >= 0) atomicMin((long long*)a, b);
    else atomicMax((unsigned long long*)a, (unsigned long long)b);
}
// updateAggrSum / Min / Max / Avg / Count / Sum2 (aggr_incremental.go:200-458) for one point of one series: NaN is skipped;
// the order in which series reach a cell is scheduling dependent, as in the reference (one incrementalAggrContext per worker)
__device__ __forceinline__ void fu_fold(int aggr, double* values, double* counts, size_t cell, double v) {
    if (isnan(v)) return;
    switch (aggr) {
        case VMB_AGGR_SUM:
        case VMB_AGGR_AVG:
            atomicAdd(values + cell, v);
            atomicAdd(counts + cell, 1.0);
            break;
        case VMB_AGGR_COUNT:
        case VMB_AGGR_GROUP:
            atomicAdd(values + cell, 1.0);
            break;
        case VMB_AGGR_SUM2:
            atomicAdd(values + cell, __dmul_rn(v, v));
            atomicAdd(counts + cell, 1.0);
            break;
        case VMB_AGGR_MIN:
            fu_atomic_min(values + cell, v);
            atomicAdd(counts + cell, 1.0);
            break;
        case VMB_AGGR_MAX:
            fu_atomic_max(values + cell, v);
            atomicAdd(counts + cell, 1.0);
            break;
    }
}

__device__ __forceinline__ int32_t fu_floor_div(int32_t a, int32_t b) {  // b > 0
    int32_t q = a / b;
    return q - ((a % b) < 0 ? 1 : 0);
}

// per-series setup, executed by ONE thread: block header -> what the fill / points loops need; bail = the series goes to the
// un-fused pipeline (anything this kernel does not take, see the head of the file)
__device__ void fu_series_setup(const FusedParams& P, uint32_t s, FuSeries* out) {
    const vmb_rollup_cfg& rc = P.cfg;
    FuSeries o;
    memset(&o, 0, sizeof(o));
    const uint32_t b = P.ser_first_block[s];
    const vmb_block_desc d = P.descs[b];
    const uint32_t n = d.rows;
    bool bail = n < 2u || n > 16384u || d.ts_mt != 2 || d.precision_bits < 64;
    if (!bail && P.zstd_status) bail = P.zstd_status[2 * b] != 0 || P.zstd_status[2 * b + 1] != 0;
    // ---- timestamps: MarshalTypeDeltaConst (encoding.go:231) = first + i * dt
    int64_t dts = 0;
    if (!bail) {
        uint32_t used = 0;
        bail = read_single_varint(P.payload + d.ts_off, d.ts_size, &dts, &used) != 0 || used < d.ts_size;
    }
    const int64_t LIM = (int64_t)1 << 30;
    bail = bail || dts <= 0 || dts >= LIM || (int64_t)(n - 1) * dts >= LIM;
    const int64_t t_org = d.min_ts;
    bail = bail || t_org < P.tr_min || t_org + (int64_t)(n - 1) * dts > P.tr_max;  // rows trimmed by the time range: un-fused path
    int64_t max_prev = 0, window = 0;
    if (!bail) {
        // rows sit at t_org + row * dts (n >= 2): every interval getScrapeInterval looks at is dts
        const PrevWindow pw = prev_interval_window(rc, scrape_interval(rc.step, n - 1 > 20 ? 20 : n - 1, [&](int) { return (double)dts; }));
        max_prev = pw.max_prev;
        window = pw.window;
        const int64_t a0 = rc.start - window - max_prev - t_org, a1 = rc.end - t_org;
        bail = !(a0 > -LIM && a0 < LIM && a1 > -LIM && a1 < LIM && window < LIM && max_prev < LIM && rc.step < LIM);
    }
    // ---- values column
    const int mt = d.val_mt;
    o.is_stream = mt == 1 || mt == 4 || mt == 5 || mt == 6;
    o.delta2 = mt == 1 || mt == 5;
    if (!bail) {
        if (o.is_stream) {
            const ColInfo ci = P.cols[2 * b + 1];
            const uint8_t* src = ci.kind == VMB_ZK_NONE ? P.payload + d.val_off : P.scratch + ci.scratch_off;
            o.len = ci.kind == VMB_ZK_NONE ? d.val_size : ci.content_size;
            o.shift = (uint32_t)((uintptr_t)src & 15u);
            o.A = src - o.shift;
            bail = o.len < n - 1;  // int.go:183
        } else if (mt == 3) {
            bail = d.val_size != 0;
        } else if (mt == 2) {
            uint32_t used = 0;
            bail = read_single_varint(P.payload + d.val_off, d.val_size, &o.dconst, &used) != 0 || used < d.val_size;
            // a wrapping / decreasing progression is a removeCounterResets matter: leave it to the un-fused path
            bail = bail || o.dconst < 0 || (uint64_t)o.dconst > (uint64_t)0x7fffffffffffffffLL / (n - 1) ||
                   (int64_t)((uint64_t)d.first_value + (uint64_t)(n - 1) * (uint64_t)o.dconst) < d.first_value;
        } else {
            bail = true;
        }
    }
    const bool want_rcr = (rc.flags & VMB_RC_REMOVE_COUNTER_RESETS) != 0;
    o.stale_matters = (rc.flags & VMB_RC_DROP_STALE_NANS) != 0 || want_rcr || (rc.flags & VMB_RC_PRE_MASK) != 0;
    bail = bail || (rc.flags & VMB_RC_PRE_MASK) != 0;  // value preFuncs of the multi-output rollups: un-fused path
    // removeCounterResets with a staleness interval below the scrape interval leaves every row raw (rollup.go:937): nothing to do
    const int64_t max_stale = rc.lookback_delta != 0 ? rc.lookback_delta + rc.window : 0;
    o.do_rcr = want_rcr && !(max_stale > 0 && dts > max_stale);
    if (!bail && o.stale_matters && d.first_value == VMB_V_STALE_NAN) bail = true;
    o.t_org = t_org;
    o.dts = dts;
    o.window = window;
    o.max_prev = max_prev;
    o.first_value = d.first_value;
    o.n = n;
    o.end_al = (uint32_t)(((uint64_t)o.shift + o.len + 15u) & ~(uint64_t)15);
    o.scale = d.scale;
    if (!bail) {
        o.start_r = (int32_t)(rc.start - t_org);
        o.step32 = (int32_t)rc.step;
        o.win32 = (int32_t)window;
        o.mpi32 = (int32_t)max_prev;
        const int32_t dt_row = (int32_t)dts;
        if (o.step32 % dt_row == 0) {
            // rows with timestamp <= t_org + x: clamp(floor(x / dt) + 1, 0, n); x advances by a whole number of rows per point
            o.lin = 1;
            o.lin_k = o.step32 / dt_row;
            o.jq0 = fu_floor_div(o.start_r, dt_row) + 1;
            o.iq0 = fu_floor_div(o.start_r - o.win32, dt_row) + 1;
        }
    }
    {
        Dec dec;
        dec.init(d.scale);
        o.dec_e10 = dec.e10;
        o.dec_rcp = dec.rcp;
        o.dec_mode = dec.mode;
    }
    o.rate_dt = -1;
    o.rate_D = o.rate_R = 1.0;
    if (!bail && (rc.func_id == VMB_RF_RATE || rc.func_id == VMB_RF_DELTA)) {  // (delta / increase use rate_rows, rate_dt > 0 only)
        const int32_t dt_row = (int32_t)dts;
        const int32_t rows_w = o.lin ? o.jq0 - o.iq0 : o.win32 / dt_row;
        if (rows_w >= 1 && (int64_t)rows_w * dt_row < ((int64_t)1 << 30)) {
            o.rate_rows = rows_w;
            o.rate_dt = rows_w * dt_row;
            o.rate_D = ms_to_s((int64_t)o.rate_dt);
            o.rate_R = 1.0 / o.rate_D;
            // (Markstein's correction needs a significand of D that is not all ones)
            if (((unsigned long long)__double_as_longlong(o.rate_D) & 0xfffffffffffffull) == 0xfffffffffffffull) o.rate_dt = -1;
        }
    }
    o.s = s;
    o.bail = bail;
    *out = o;
}

// Dec (decimal.go:100) of the series' scale, rebuilt from shared memory where it is used
__device__ __forceinline__ Dec fu_dec(const FuSeries& o) {
    Dec d;
    d.e10 = o.dec_e10;
    d.rcp = o.dec_rcp;
    d.mode = o.dec_mode;
    return d;
}

// stage buffer `bf` <- aligned bytes [fs - 16, fs + FU_FILL) of the stream (clamped to its 16-byte aligned end); one thread
__device__ __forceinline__ void fu_stage_copy(FusedSmem& S, const uint8_t* A, uint32_t end_al, uint32_t fs, uint32_t bf) {
    if (fs < end_al) {
        const uint32_t lo = fs ? fs - 16u : 0u;
        const uint32_t hi = fs + FU_FILL < end_al ? fs + FU_FILL : end_al;
        mbar_expect_tx(&S.mbar[bf], hi - lo);
        bulk_g2s(&S.stage[bf][fs ? 0 : 16], A + lo, hi - lo, &S.mbar[bf]);
    }
}

// one thread: series s -> `ser`, and the first fill of its stream (a column the kernel takes) into the idle stage buffer `bf`
__device__ void fu_series_begin(const FusedParams& P, FusedSmem& S, uint32_t s, FuSeries* ser, uint32_t bf) {
    fu_series_setup(P, s, ser);
    if (!ser->bail && ser->is_stream) fu_stage_copy(S, ser->A, ser->end_al, 0, bf);
}

}  // namespace

template <int F>
__global__ void __launch_bounds__(FU_THREADS, FU_CTAS_PER_SM) k_fused_rollup(FusedParams P) {
    extern __shared__ __align__(16) unsigned char fu_raw[];
    FusedSmem& S = *reinterpret_cast<FusedSmem*>(fu_raw);
    const FuValsRW RV{S.val};  // RV[absolute row]
    uint32_t val_s = smem_u32(S.val);
    asm volatile("" : "+r"(val_s));  // opaque: kept in a register instead of being rebuilt from the CTA's shared window per access
    const vmb_rollup_cfg& rc = P.cfg;
    const uint32_t tid = threadIdx.x, lane = tid & 31u, w = tid >> 5;
    S.s_thr[tid] = 0;
    uint32_t par = 0;             // bit b: mbarrier phase parity of stage buffer b (carried over the series)
    uint32_t buf = 0;             // stage buffer of the next tile; a series starts in the one its predecessor left it at
    if (tid == 0) {
        mbar_init(&S.mbar[0], 1);
        mbar_init(&S.mbar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
#ifdef VMB_FUSED_PHASES
    for (uint32_t k = tid; k < FU_WARPS * FU_PH_SLOTS; k += FU_THREADS) (&S.ph[0][0])[k] = 0;
    long long ph_t = clock64();
#endif
    __syncthreads();

    for (uint32_t li = blockIdx.x; li < P.nlist; li += gridDim.x) {
        __syncthreads();  // the previous series is done with the shared memory
        if (tid == 0) {
            fu_series_begin(P, S, P.ser_list[li], &S.ser, buf);
            S.flags = 0;
            S.flags_emit = 0;
            S.nev = 0;
        }
        __syncthreads();
        const FuSeries& SE = S.ser;
        bool bail = SE.bail != 0;
        const uint32_t n = SE.n;
        // what the fill needs is held in registers; what only the points need is read from SE (stays valid for the whole series)
        // where it is used, so that it is not live through the parse
        const bool is_stream = SE.is_stream != 0;
        const int64_t first_value = SE.first_value;
        const int32_t dt_row = (int32_t)SE.dts;
        const uint32_t nvar = n - 1;

        auto issue_copy = [&](uint32_t fs, uint32_t bf) {
            if (tid == 0) fu_stage_copy(S, SE.A, SE.end_al, fs, bf);
        };
        uint32_t fs = 0;                   // next unconsumed tile (aligned stream offset); stage[buf] holds it
        bool copy_pending = !bail && is_stream;  // the first fill is in flight (fu_series_begin)
        // first row (nearest_delta2.go:75 / nearest_delta.go:64: as[0] = firstValue)
        uint32_t N = 0;                    // varints decoded so far
        uint32_t base = 0, cnt = 0, p = 0;
        uint32_t gen_rows = 0;             // rows produced so far (const / delta-const columns)
        double corr = 0.0, prev_raw = 0.0;
        bool stream_done = !is_stream;
        if (!bail) {
            if (tid == 0) {
                S.val[0] = fu_dec(SE).conv(first_value);  // (fu_swz(0) == 0)
                S.nd_v = (uint64_t)first_value;
                S.nd_d1 = 0;
            }
            cnt = 1;
            gen_rows = 1;
        }
        S.s_ser[tid] = tid == 0 ? n : 0u;  // samplesScanned starts at len(values) rollup.go:766
        __syncthreads();
        if (!bail) prev_raw = S.val[0];
        FU_PH_COUNT(FU_PH_SERIES);
        FU_PH(FU_PH_SETUP);

        uint32_t guard = 0;
        while (!bail && (p < P.npoints || !stream_done)) {
            if (++guard > 200000u) {  // every iteration consumes a tile or emits a point: this cannot be reached (the pipeline takes it)
                bail = true;
                break;
            }
            // ================= fill: decode the next tiles of the stream into rows [cnt, ...)
            uint32_t cnt_old = cnt;
            bool progressed = false;
            if (is_stream && !stream_done) {
                FU_PH(FU_PH_POINTS);
                FU_PH_COUNT(FU_PH_FILLS);
                if (copy_pending) {
                    mbar_wait(&S.mbar[buf], (par >> buf) & 1u);
                    par ^= 1u << buf;
                    copy_pending = false;
                }
                FU_PH(fs ? FU_PH_WAIT : FU_PH_SETUP);
                const uint8_t* st = &S.stage[buf][16];  // aligned stream byte `fs` sits at st[0]
                const uint32_t end_al = SE.end_al;
                const int64_t vlo = (int64_t)SE.shift, vhi = vlo + SE.len;  // valid stream positions in aligned coordinates
                const bool delta2 = SE.delta2 != 0, do_rcr = SE.do_rcr != 0, stale_matters = SE.stale_matters != 0;
                const uint32_t off = w * FU_TILE + lane * (16u * FU_G);
                const int64_t g0 = (int64_t)fs + off;
                uint32_t t_own[FU_G], vm[FU_G], tm[FU_G], pbm[FU_G];
#pragma unroll
                for (int g = 0; g < FU_G; g++) t_own[g] = fu_term_mask16(*reinterpret_cast<const uint4*>(st + off + 16 * g));
                const uint32_t prv_w = *reinterpret_cast<const uint32_t*>(st + off - 4);  // the four bytes in front of the lane's bytes
                const int64_t gw = (int64_t)fs + w * FU_TILE;  // first byte of the warp's tile
                if (gw - 16 >= vlo && gw + FU_TILE <= vhi) {
                    // the tile and the 16 bytes in front of it lie inside the stream (all but the first and last tile of a column)
                    uint32_t t_prev = __shfl_up_sync(VMB_FULL, t_own[FU_G - 1], 1);
                    if (lane == 0) t_prev = fu_term_mask16(*reinterpret_cast<const uint4*>(st + off - 16));
#pragma unroll
                    for (int g = 0; g < FU_G; g++) {
                        vm[g] = 0xffffu;
                        tm[g] = t_own[g];
                        pbm[g] = g ? t_own[g - 1] : t_prev;
                    }
                } else {
                    const uint32_t t_prv = fu_term_mask16(*reinterpret_cast<const uint4*>(st + off - 16));
#pragma unroll
                    for (int g = 0; g < FU_G; g++) {
                        const int64_t gg = g0 + 16 * g;
                        vm[g] = fu_valid16(gg, vlo, vhi);
                        tm[g] = t_own[g] & vm[g];
                        // boundaries of the previous 16 bytes: terminators, and everything in front of the stream start
                        const uint32_t pvm = fu_valid16(gg - 16, vlo, vhi);
                        pbm[g] = (((g ? t_own[g - 1] : t_prv) & pvm) | (gg - 16 < vlo ? ~pvm : 0u)) & 0xffffu;
                    }
                }
                uint32_t cl = 0;
#pragma unroll
                for (int g = 0; g < FU_G; g++) cl += (uint32_t)__popc(tm[g]);
                uint32_t incl = cl;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    uint32_t t = __shfl_up_sync(VMB_FULL, incl, o);
                    if (lane >= (uint32_t)o) incl += t;
                }
                if (lane == 31) S.w_cnt[w] = incl;
                if (tid == 0) S.nev = 0;  // (everybody read the previous fill's events before the barrier that ended it)
                FU_PH(FU_PH_TERM);
                __syncthreads();
                FU_PH(FU_PH_WAIT);
                // whole tiles that fit the resident rows (pass-through once the points are done: rows are only validated)
                const bool discard = p >= P.npoints;
                if (discard) { cnt = 1; cnt_old = 1; }  // rows are not needed any more: decode over the same ring slots
                // lane k < FU_WARPS holds the count of warp k; inclusive scan over those lanes; a tile fits when the rows before it and its own
                // fit the ring; K = the leading tiles that fit
                uint32_t K, tot, rb;
                {
                    const uint32_t t = lane < FU_WARPS ? S.w_cnt[lane] : 0u;
                    uint32_t ic = t;
#pragma unroll
                    for (int o = 1; o < FU_WARPS; o <<= 1) {
                        const uint32_t u = __shfl_up_sync(VMB_FULL, ic, o);
                        if (lane >= (uint32_t)o) ic += u;
                    }
                    const uint32_t fits = __ballot_sync(VMB_FULL, lane < FU_WARPS && cnt + ic <= FU_CAP) & ((1u << FU_WARPS) - 1u);
                    K = (uint32_t)__ffs((int)(~fits & ((2u << FU_WARPS) - 1u))) - 1u;  // number of leading ones
                    tot = K ? __shfl_sync(VMB_FULL, ic, (int)K - 1) : 0u;
                    const uint32_t ex = __shfl_sync(VMB_FULL, ic - t, (int)(w < FU_WARPS ? w : 0));
                    rb = w < K ? ex : 0u;
                }
                if (N + tot > nvar) bail = true;  // more varints than rows: nearest_delta.go:65 "unexpected tail" -> un-fused path
                const uint32_t fs_next = fs + K * FU_TILE;
                const bool done_after = fs_next >= end_al;
                if (!bail && K) {
                    if (!done_after) {
                        issue_copy(fs_next, buf ^ 1u);
                        copy_pending = true;
                    }
                    FU_PH(FU_PH_TERM);
                    // ---- parse: the varints whose terminator lies in this lane's 16 bytes
                    uint64_t s1 = 0, s2 = 0;
                    const uint32_t row0 = base + cnt + rb + incl - cl;  // absolute row of the lane's first value
                    bool bad = false;
                    // per group: carried-in bytes = behind the last boundary of the previous 16 bytes (15 - msb(pbm)); does any varint
                    // that ends in this warp's tile have more than 4 bytes?  Continuation bytes of [previous 16 | own 16] as one mask:
                    // a run of four of them that reaches into the last 4 + 16 bytes (conservative)
                    uint32_t carry[FU_G];
                    bool lng = false;
#pragma unroll
                    for (int g = 0; g < FU_G; g++) {
                        carry[g] = pbm[g] ? (uint32_t)__clz((int)pbm[g]) - 16u : 16u;
                        const uint32_t c32 = ((~pbm[g]) & 0xffffu) | ((~t_own[g] & vm[g]) << 16);
                        const uint32_t run4 = c32 & (c32 >> 1) & (c32 >> 2) & (c32 >> 3);
                        lng |= tm[g] && (((run4 >> 12) != 0u) || carry[g] > 3u);
                        // a run of continuation bytes over a whole 16-byte group inside the stream: a varint of > 16 bytes
                        if (w < K && vm[g] == 0xffffu && tm[g] == 0 && pbm[g] == 0) bad = true;
                    }
                    const bool any_long = __any_sync(VMB_FULL, w < K && lng) != 0;
                    if (w < K && cl) {
                        uint32_t row = row0;
                        // the varints whose terminator lies in one 16-byte group; prev_w = the four bytes in front of the group
                        auto parse16 = [&](const uint4 own, const uint32_t prev_w, uint32_t m, const uint32_t vmg, const uint32_t cr,
                                           const uint32_t boff) {
                            // 7-bit groups of the own 16 bytes as a 112-bit number q3:q2:q1:q0
                            const uint32_t c0 = compact7(own.x), c1 = compact7(own.y), c2 = compact7(own.z), c3 = compact7(own.w);
                            uint32_t q0 = c0 | (c1 << 28), q1 = (c1 >> 4) | (c2 << 24), q2 = (c2 >> 8) | (c3 << 20), q3 = c3 >> 12;
                            auto drop_groups = [&](uint32_t sh) {  // q >>= sh (sh = 7 * bytes <= 112)
                                while (sh >= 32u) {
                                    q0 = q1; q1 = q2; q2 = q3; q3 = 0;
                                    sh -= 32u;
                                }
                                q0 = __funnelshift_r(q0, q1, sh);
                                q1 = __funnelshift_r(q1, q2, sh);
                                q2 = __funnelshift_r(q2, q3, sh);
                                q3 >>= sh;
                            };
                            uint32_t pos = 0;  // byte position of the current varint's first own byte
                            if (!(vmg & 1u)) {  // the stream starts inside this group: skip the bytes in front of it
                                pos = (uint32_t)__ffs((int)vmg) - 1u;
                                m >>= pos;
                                drop_groups(7u * pos);
                            }
                            if (!any_long) {
                                // every varint of the tile has <= 4 bytes (28 bits): one shift-and-mask per value, no branches inside
                                uint32_t cval = 0, cbits = 0;  // value and width of the carried-in bytes (first varint only)
                                if (cr) {
                                    cval = compact7(prev_w) >> (7u * (4u - cr));
                                    cbits = 7u * cr;
                                }
                                while (m) {
                                    const uint32_t L = (uint32_t)__ffs((int)m);  // own bytes of this varint
                                    const uint32_t sh = 7u * L;
                                    const uint32_t u = ((q0 & ~(0xffffffffu << sh)) << cbits) | cval;
                                    const int v32 = (int)((u >> 1) ^ (0u - (u & 1u)));
                                    const long long v = (long long)v32;
                                    fu_sts_i64(val_s, row, v);  // raw zig-zag decoded delta, replaced by the value in step 4
                                    s1 += (uint64_t)v;
                                    s2 += s1;
                                    row++;
                                    m >>= L;
                                    q0 = __funnelshift_r(q0, q1, sh);
                                    q1 = __funnelshift_r(q1, q2, sh);
                                    q2 = __funnelshift_r(q2, q3, sh);
                                    q3 >>= sh;
                                    cval = 0;
                                    cbits = 0;
                                }
                            } else {
                                uint32_t cb = cr;  // carried-in bytes of the first varint
                                while (m) {
                                    const uint32_t L = (uint32_t)__ffs((int)m);  // own bytes of this varint
                                    long long v;
                                    if (7u * (L + cb) <= 28u) {
                                        const uint32_t cval = cb ? compact7(prev_w) >> (7u * (4u - cb)) : 0u;
                                        const uint32_t u = ((q0 & ~(0xffffffffu << (7u * L))) << (7u * cb)) | cval;
                                        v = (long long)(int)((u >> 1) ^ (0u - (u & 1u)));
                                    } else {
                                        // long varint (> 4 bytes): byte loop over the staged bytes, int.go:196-284
                                        const int sb = (int)(boff + pos) - (int)cb;  // first byte, relative to st
                                        const uint32_t vl = L + cb;
                                        uint64_t u = 0;
                                        if (vl > 10) {
                                            bad = true;
                                        } else {
                                            for (uint32_t bb = 0; bb < vl; bb++) {
                                                const uint32_t byte = st[sb + (int)bb];
                                                if (bb == 9) {
                                                    if (byte > 1u) bad = true;
                                                    u |= (uint64_t)1 << 63;
                                                } else {
                                                    u |= (uint64_t)(byte & 0x7fu) << (7 * bb);
                                                }
                                            }
                                        }
                                        v = (long long)(u >> 1) ^ -(long long)(u & 1);
                                    }
                                    fu_sts_i64(val_s, row, v);
                                    s1 += (uint64_t)v;
                                    s2 += s1;
                                    row++;
                                    cb = 0;
                                    pos += L;
                                    m >>= L;
                                    drop_groups(7u * L);
                                }
                            }
                        };
#pragma unroll
                        for (int g = 0; g < FU_G; g++) {
                            if (tm[g])
                                parse16(*reinterpret_cast<const uint4*>(st + off + 16 * g),
                                        g ? *reinterpret_cast<const uint32_t*>(st + off + 16 * g - 4) : prv_w, tm[g], vm[g], carry[g],
                                        off + 16u * g);
                        }
                    }
                    FU_PH(FU_PH_PARSE);
                    // ---- scan (s1, s2) over the warp.  combine(A then B): s2 = s2A + s2B + cntB * s1A, so with E1(l) = the plain
                    // exclusive prefix of s1, the inclusive prefix of s2 is the plain prefix sum of t_l = s2_l + cnt_l * E1(l): two sum
                    // scans (wrapping int64 arithmetic: bit-identical to the sequential Go loop), the counts are known from step 1
                    const uint32_t mycnt = w < K ? cl : 0u;
                    uint64_t is1 = s1;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const uint64_t a = shfl_up_u64(is1, o);
                        if (lane >= (uint32_t)o) is1 += a;
                    }
                    const uint64_t es1_ = is1 - s1;  // lanes in front of this one
                    const uint64_t t2 = s2 + (uint64_t)mycnt * es1_;
                    uint64_t is2 = t2;
                    if (delta2) {
#pragma unroll
                        for (int o = 1; o < 32; o <<= 1) {
                            const uint64_t a = shfl_up_u64(is2, o);
                            if (lane >= (uint32_t)o) is2 += a;
                        }
                    }
                    if (lane == 31) {
                        S.w_s1[w] = is1;
                        S.w_s2[w] = is2;
                    }
                    if (bad) S.flags = 1u;
                    FU_PH(FU_PH_SCAN);
                    __syncthreads();
                    FU_PH(FU_PH_WAIT);
                    if (S.flags & 1u) bail = true;
                    // exclusive prefix over the warps in front, and the totals of the fill: lane k < K holds warp k's triple, one
                    // FU_WARPS-lane scan, warp w picks lane w - 1 (prefix) and everybody lane K - 1 (totals)
                    uint32_t pc, tc;
                    uint64_t ps1, ps2, ts1, ts2;
                    {
                        const bool act = lane < K;
                        const uint32_t c0_ = act ? S.w_cnt[lane] : 0u;
                        const uint64_t a1_0 = act ? S.w_s1[lane] : 0ull, a2_0 = act ? S.w_s2[lane] : 0ull;
                        uint32_t c_ = c0_;
                        uint64_t a1 = a1_0;
#pragma unroll
                        for (int o = 1; o < FU_WARPS; o <<= 1) {
                            const uint32_t bc = __shfl_up_sync(VMB_FULL, c_, o);
                            const uint64_t b1 = shfl_up_u64(a1, o);
                            if (lane >= (uint32_t)o) {
                                a1 += b1;
                                c_ += bc;
                            }
                        }
                        uint64_t a2 = a2_0 + (uint64_t)c0_ * (a1 - a1_0);  // the same two-scan form over the warps
                        if (delta2) {
#pragma unroll
                            for (int o = 1; o < FU_WARPS; o <<= 1) {
                                const uint64_t b2 = shfl_up_u64(a2, o);
                                if (lane >= (uint32_t)o) a2 += b2;
                            }
                        }
                        const int src_p = w ? (int)w - 1 : 0, src_t = (int)K - 1;
                        pc = __shfl_sync(VMB_FULL, c_, src_p);
                        ps1 = shfl_u64(a1, src_p);
                        ps2 = shfl_u64(a2, src_p);
                        if (w == 0) { pc = 0; ps1 = 0; ps2 = 0; }
                        tc = __shfl_sync(VMB_FULL, c_, src_t);
                        ts1 = shfl_u64(a1, src_t);
                        ts2 = shfl_u64(a2, src_t);
                    }
                    FU_PH(FU_PH_SCAN);
                    // ---- emit: replay the lane's values with the scanned prefix, mantissa -> float64 in place
                    const uint32_t ecnt = incl - cl;         // lanes in front, this warp (step 1)
                    const uint64_t es1 = es1_, es2 = is2 - t2;
                    if (!bail && w < K && cl) {
                        // prefix in front of the lane = (warps in front) then (lanes in front)
                        const uint32_t fcnt = pc + ecnt;
                        const uint64_t fs1 = ps1 + es1;
                        const uint64_t fs2 = ps2 + es2 + (uint64_t)ecnt * ps1;
                        const uint64_t V = S.nd_v, D1 = S.nd_d1;
                        uint64_t d1 = D1 + fs1;
                        uint64_t v = delta2 ? (V + fs2 + (uint64_t)fcnt * D1) : (V + fs1);
                        bool saw_stale = false;
                        uint32_t cand = 0;  // bit k: row0 + k holds a smaller value than the row in front (a lane has <= 32 rows)
                        const uint64_t v0 = v;
                        const Dec dec = fu_dec(SE);
                        auto emit_run = [&](auto is_delta2) {
                            constexpr bool D2 = decltype(is_delta2)::value;
                            // four rows per step: their deltas are loaded first, their conversions are independent of each other and
                            // overlap, their stores come last (row by row, every row waited for its load and for the store in front)
                            for (uint32_t k = 0; k < cl; k += 4) {
                                uint64_t x[4], vv[4];
#pragma unroll
                                for (int i = 0; i < 4; i++) x[i] = (uint64_t)fu_lds_i64(val_s, row0 + k + i);  // (past cl: not used)
#pragma unroll
                                for (int i = 0; i < 4; i++) {
                                    const uint64_t pv = v;
                                    if (k + i < cl) {
                                        if (D2) {
                                            d1 += x[i];
                                            v += d1;
                                        } else {
                                            v += x[i];
                                        }
                                        cand |= (uint32_t)((int64_t)v < (int64_t)pv) << (k + i);
                                    }
                                    vv[i] = v;
                                }
                                double f[4];
#pragma unroll
                                for (int i = 0; i < 4; i++) f[i] = dec.conv_plain((int64_t)vv[i]);
#pragma unroll
                                for (int i = 0; i < 4; i++) {
                                    if (k + i < cl) {
                                        if (vv[i] - 0x7FFFFFFFFFFFFFFEull < 3ull) {  // vStaleNaN / vInfPos / vInfNeg (decimal.go:403-417)
                                            f[i] = dec.conv((int64_t)vv[i]);
                                            saw_stale |= ((int64_t)vv[i] == VMB_V_STALE_NAN);
                                        }
                                        fu_sts(val_s, row0 + k + i, f[i]);
                                    }
                                }
                            }
                        };
                        if (delta2) emit_run(std::true_type{});
                        else emit_run(std::false_type{});
                        // candidate counter resets (the conversion is monotone): the exact test is on the floats, rollup.go:928
                        if (do_rcr && cand) {
                            do {
                                const uint32_t k = (uint32_t)__ffs((int)cand) - 1u;
                                cand &= cand - 1u;
                                const double f = fu_lds(val_s, row0 + k), pf = k ? fu_lds(val_s, row0 + k - 1u) : dec.conv((int64_t)v0);
                                const double dd = f - pf;
                                if (dd < 0) {
                                    const double amt = ((-dd * 8) < pf) ? (pf - f) : pf;
                                    const uint32_t e = atomicAdd(&S.nev, 1u);
                                    if (e < FU_MAX_EVENTS) {
                                        S.ev_row[e] = row0 + k;
                                        S.ev_amt[e] = amt;
                                    }
                                }
                            } while (cand);
                        }
                        if (saw_stale && stale_matters) S.flags_emit = 1u;
                    }
                    FU_PH(FU_PH_EMIT);
                    // ---- carries: thread 0 stores them behind the barrier that ends the fill (every lane has read the old ones by then)
                    uint64_t nV = 0, nD1 = 0;
                    if (tid == 0) {
                        nV = S.nd_v;
                        nD1 = S.nd_d1;
                        if (delta2) {
                            nV += ts2 + (uint64_t)tc * nD1;
                            nD1 += ts1;
                        } else {
                            nV += ts1;
                        }
                    }
                    N += tc;
                    cnt += tot;
                    fs = fs_next;
                    buf ^= 1u;
                    progressed = true;
                    if (done_after) {
                        stream_done = true;
                        // nearest_delta.go:59-71: exactly n - 1 varints, the stream ends on a terminator
                        if (N != nvar) bail = true;
                    }
                    __syncthreads();
                    FU_PH(FU_PH_WAIT);
                    if (tid == 0) {
                        S.nd_v = nV;
                        S.nd_d1 = nD1;
                    }
                    if ((S.flags | S.flags_emit) & 1u) bail = true;
                    if (stream_done && !bail) {
                        const uint32_t last_al = (uint32_t)(vhi - 1);  // aligned position of the last stream byte
                        if (SE.A[last_al] >= 0x80) bail = true;
                    }
                }
            } else if (!is_stream && gen_rows < n) {
                // MarshalTypeConst (encoding.go:215) / MarshalTypeDeltaConst (:231) values: rows generated in place
                const uint32_t take = min(n - gen_rows, (uint32_t)FU_CAP - cnt);
                for (uint32_t k = tid; k < take; k += FU_THREADS) {
                    const uint32_t r = gen_rows + k;
                    const int64_t v = (int64_t)((uint64_t)SE.first_value + (uint64_t)r * (uint64_t)SE.dconst);
                    RV[base + cnt + k] = fu_dec(SE).conv(v);
                    if (SE.stale_matters && v == VMB_V_STALE_NAN) S.flags = 1u;
                }
                progressed = take > 0;
                gen_rows += take;
                cnt += take;
                N = gen_rows - 1;
                FU_PH(FU_PH_PARSE);
                __syncthreads();
                FU_PH(FU_PH_WAIT);
                if (S.flags & 1u) bail = true;
            }
            if (bail) break;
            const bool all_rows = is_stream ? stream_done : gen_rows == n;
            if (p >= P.npoints) continue;  // only validating the rest of the stream

            // ================= removeCounterResets over the new rows [cnt_old, cnt)  (rollup.go:921)
            if (SE.do_rcr && cnt > cnt_old) {
                const uint32_t nev = S.nev;
                const double raw_last = RV[base + cnt - 1];
                if (nev > FU_MAX_EVENTS) {
                    bail = true;  // a fill full of resets: un-fused path
                } else if (nev == 0 && corr != 0.0 && isfinite(corr) && fu_ld(S.val, base + cnt_old) + corr >= fu_ld(S.val, base + cnt_old - 1)) {
                    // no value drop inside the fill (nor at its front) and its first corrected row is not below the last output: raw
                    // rows are non-decreasing, x -> RN(x + corr) keeps the order, so the clamp of rollup.go:954 cannot fire: one pass
                    // (four rows per thread and step, their loads issued before the first store)
                    for (uint32_t k = cnt_old + tid; k < cnt; k += 4 * FU_THREADS) {
                        double x[4];
#pragma unroll
                        for (int i = 0; i < 4; i++) x[i] = fu_lds(val_s, base + k + i * FU_THREADS);  // (past cnt: values not used)
#pragma unroll
                        for (int i = 0; i < 4; i++)
                            if (k + i * FU_THREADS < cnt) fu_sts(val_s, base + k + i * FU_THREADS, x[i] + corr);
                    }
                    FU_PH(FU_PH_RCR);
                    __syncthreads();
                    FU_PH(FU_PH_WAIT);
                } else if (nev || corr != 0.0) {
                    if (tid == 0) {
                        // events in row order, corrections accumulated sequentially like the Go loop
                        for (uint32_t a = 1; a < nev; a++) {
                            const uint32_t rr = S.ev_row[a];
                            const double aa = S.ev_amt[a];
                            int bq = (int)a - 1;
                            while (bq >= 0 && S.ev_row[bq] > rr) {
                                S.ev_row[bq + 1] = S.ev_row[bq];
                                S.ev_amt[bq + 1] = S.ev_amt[bq];
                                bq--;
                            }
                            S.ev_row[bq + 1] = rr;
                            S.ev_amt[bq + 1] = aa;
                        }
                        double c = corr;
                        for (uint32_t a = 0; a < nev; a++) {
                            c = c + S.ev_amt[a];
                            S.ev_cum[a] = c;
                        }
                    }
                    FU_PH(FU_PH_RCR);
                    __syncthreads();
                    FU_PH(FU_PH_WAIT);
                    // corrected values are non-decreasing unless float rounding interferes: check that first, without writing
                    const double prev_out = RV[base + cnt_old - 1];
                    bool viol = false;
                    for (uint32_t k = cnt_old + tid; k < cnt; k += FU_THREADS) {
                        const uint32_t ar = base + k;
                        double ck = corr, cp = corr;
                        for (uint32_t a = 0; a < nev; a++) {
                            if (S.ev_row[a] <= ar) ck = S.ev_cum[a];
                            if (S.ev_row[a] + 1u <= ar) cp = S.ev_cum[a];
                        }
                        const double mk = RV[ar] + ck;
                        const double mp = k == cnt_old ? prev_out : RV[ar - 1] + cp;
                        viol |= !(mk >= mp);  // a clamp would fire, or a NaN is involved
                    }
                    FU_PH(FU_PH_RCR);
                    const int any_viol = __syncthreads_or((int)viol);
                    FU_PH(FU_PH_WAIT);
                    if (!any_viol) {
                        for (uint32_t k = cnt_old + tid; k < cnt; k += FU_THREADS) {
                            const uint32_t ar = base + k;
                            double ck = corr;
                            for (uint32_t a = 0; a < nev; a++)
                                if (S.ev_row[a] <= ar) ck = S.ev_cum[a];
                            RV[ar] = RV[ar] + ck;
                        }
                    } else if (w == 0) {
                        // the exact sequential pass (rare): one warp, 32 rows at a time, state carried like k_series_prepare
                        RcrState stt;
                        stt.corr = corr;
                        stt.prev_raw = prev_raw;
                        stt.prev_out = prev_out;
                        stt.prev_ts = 0;
                        for (uint32_t cb = base + cnt_old; cb < base + cnt; cb += 32) {
                            const uint32_t i_ = cb + lane;
                            const double x = i_ < base + cnt ? RV[i_] : 0.0;
                            rcr_chunk(stt, RV, cb, base + cnt, x, 0, 0, (int)lane);
                        }
                    }
                    if (nev) corr = S.ev_cum[nev - 1];
                    FU_PH(FU_PH_RCR);
                    __syncthreads();
                    FU_PH(FU_PH_WAIT);
                }
                prev_raw = raw_last;
            }
            FU_PH(FU_PH_RCR);

            // ================= points whose window lies inside the resident rows
            const int32_t start_r = SE.start_r, step32 = SE.step32, win32 = SE.win32, mpi32 = SE.mpi32;
            const bool lin = SE.lin != 0;
            const int32_t lin_k = SE.lin_k, iq0 = SE.iq0, jq0 = SE.jq0;
            const float inv_row = 1.0f / (float)dt_row;
            uint32_t p_end;
            if (all_rows) p_end = P.npoints;
            else {
                const int64_t tl = (int64_t)(base + cnt - 1) * dt_row - 1 - start_r;  // tEnd < timestamp of the last resident row
                p_end = tl < 0 ? 0u : min(P.npoints, (uint32_t)tl / (uint32_t)step32 + 1u);
            }
            if (p_end <= p) {
                if (!progressed) bail = true;  // the window of point p does not fit FU_CAP rows: un-fused path
                FU_PH(FU_PH_POINTS);
                __syncthreads();
                FU_PH(FU_PH_WAIT);
                continue;
            }
            {
                // rate(): the divisor of a full window, its reciprocal (used only when a point's divisor is exactly this one)
                const int32_t rate_dt = SE.rate_dt, rate_rows = SE.rate_rows;
                const double rate_D = SE.rate_D, rate_R = SE.rate_R;
                // a previous sample right in front of the window always passes `ts > tStart - maxPrevInterval` when maxPrevInterval >= dt
                const bool prev_always = mpi32 >= dt_row;
                const uint32_t spc = (uint32_t)rc.samples_scanned_per_call;
                uint32_t sc32 = 0;
                unsigned long long scanned = 0;
                const FuVals WV{S.val, base};  // WV[k] = resident row base + k
                const bool to_aggr = P.aggr_values != nullptr;
                double* out_row = P.out + (to_aggr ? (size_t)blockIdx.x : (size_t)SE.s) * P.npoints;
                asm volatile("" : "+l"(out_row));  // (kept in registers: the loops below are tight)
                auto put = [&](uint32_t q, double v) { out_row[q] = v; };
                uint32_t sc_interior = spc ? spc : (uint32_t)rate_rows;  // samplesScanned of an interior rate() point
                asm volatile("" : "+r"(sc_interior));
                // a point from its window edges (rate_edges / window_point): every point the interior path below does not take
                auto point = [&](uint32_t q) {
                    const int32_t xj = start_r + (int32_t)q * step32;
                    uint32_t i, j;
                    if (lin) {  // edges advance by a whole number of rows per point: no division
                        const int32_t is_ = iq0 + (int32_t)q * lin_k, js_ = jq0 + (int32_t)q * lin_k;
                        i = (uint32_t)min(max(is_, 0), (int32_t)n);
                        j = (uint32_t)min(max(js_, 0), (int32_t)n);
                    } else {
                        i = seek_ap(xj - win32, dt_row, inv_row, n);
                        j = seek_ap(xj, dt_row, inv_row, n);
                    }
                    i = i < base ? base : (i > base + cnt ? base + cnt : i);
                    j = j < base ? base : (j > base + cnt ? base + cnt : j);
                    if (j < i) j = i;
                    if (F == VMB_RF_RATE) {
                        // rollupDerivFast (rollup.go:1954) with the division through the cached reciprocal
                        sc32 += spc ? spc : j - i;
                        const RateEdges<int32_t> e = rate_edges(WV, RowTs32{base, dt_row}, base, n, cnt, i, j, xj - win32 - mpi32);
                        const double x = e.x;
                        double qv;
                        const uint32_t ex = ((uint32_t)__double2hiint(x) >> 20) & 0x7ffu;
                        if (e.dt == rate_dt && (x == 0.0 || ex - 123u < 1800u)) {
                            // x / D with D = RN(dt / 1e3), R = RN(1 / D): q = RN(x R), rem = x - q D (exact), RN(q + rem R) is the correctly
                            // rounded quotient (Markstein's step; |x| in [2^-900, 2^900], D in [1e-3, 2^30/1e3]: no under/overflow anywhere)
                            const double q0 = __dmul_rn(x, rate_R);
                            const double rem = __fma_rn(-q0, rate_D, x);
                            qv = x == 0.0 ? x : __fma_rn(rem, rate_R, q0);
                        } else {
                            qv = x / ms_to_s((int64_t)e.dt);
                        }
                        put(q, e.result(qv));
                    } else {
                        // the window's views start at row i; its timestamp is formed as t(i - 1) + dt, which keeps k_fused_rollup<-1> at 92
                        // registers (t_org + i * dt costs one more)
                        const int64_t t_im1 = SE.t_org + ((int64_t)i - 1) * SE.dts;
                        put(q, window_point<F>(rc, FuVals{S.val, i}, FuTs{t_im1 + SE.dts, SE.dts}, i, n, i, j, q, SE.window, SE.max_prev, scanned));
                    }
                };
                if ((F == VMB_RF_RATE || F == VMB_RF_DELTA) && lin && rate_dt > 0 && prev_always) {
                    // interior points: the window [i, j) holds rate_rows rows and row i - 1 exists: (v[j-1] - v[i-1]) / D.  Four points
                    // per thread, their eight edge loads issued before any arithmetic (a point off the range reads ring slots whose
                    // values are not used)
                    for (uint32_t q = p + tid; q < p_end; q += 4 * FU_THREADS) {
                        double vp[4], vl[4];
#pragma unroll
                        for (int k = 0; k < 4; k++) {
                            const int32_t is_ = iq0 + (int32_t)(q + k * FU_THREADS) * lin_k;
                            vp[k] = fu_lds(val_s, (uint32_t)is_ - 1u);
                            vl[k] = fu_lds(val_s, (uint32_t)(is_ + rate_rows) - 1u);
                        }
                        uint32_t rest = 0;  // points of the four the interior path does not take
#pragma unroll
                        for (int k = 0; k < 4; k++) {
                            const uint32_t qk = q + k * FU_THREADS;
                            if (qk >= p_end) break;
                            const int32_t is_ = iq0 + (int32_t)qk * lin_k;
                            const double x = vl[k] - vp[k];
                            bool ok = is_ >= 1 && is_ + rate_rows <= (int32_t)n && !isnan(vp[k]);
                            double r = x;  // rollupDelta rollup.go:1859 with a previous value: values[n - 1] - prevValue
                            if (F == VMB_RF_RATE) {
                                const uint32_t ex = ((uint32_t)__double2hiint(x) >> 20) & 0x7ffu;
                                ok = ok && (x == 0.0 || ex - 123u < 1800u);
                                const double q0 = __dmul_rn(x, rate_R);
                                const double rem = __fma_rn(-q0, rate_D, x);
                                r = x == 0.0 ? x : __fma_rn(rem, rate_R, q0);
                            }
                            if (ok) {
                                sc32 += sc_interior;
                                put(qk, r);
                            } else {
                                rest |= 1u << k;
                            }
                        }
                        while (rest) {
                            const int k = __ffs((int)rest) - 1;
                            rest &= rest - 1u;
                            point(q + (uint32_t)k * FU_THREADS);
                        }
                    }
                } else {
#pragma unroll 2
                    for (uint32_t q = p + tid; q < p_end; q += FU_THREADS) point(q);
                }
                S.s_ser[tid] += scanned + sc32;
            }
            p = p_end;
            FU_PH(FU_PH_POINTS);
            __syncthreads();
            FU_PH(FU_PH_WAIT);
            if (p >= P.npoints) continue;
            // ================= slide: keep rows from (first row after tStart(p)) - 1
            {
                uint32_t lo = lin ? (uint32_t)min(max(iq0 + (int32_t)p * lin_k, 0), (int32_t)n)
                                  : seek_ap(start_r + (int32_t)p * step32 - win32, dt_row, inv_row, n);
                lo = lo < base ? base : (lo > base + cnt ? base + cnt : lo);
                uint32_t nb = lo > base ? lo - 1 : base;
                if (nb > base + cnt - 1) nb = base + cnt - 1;
                cnt -= nb - base;  // a ring: sliding the window moves no data
                base = nb;
            }
        }
        // a copy still in flight must land before the buffer is reused by the next series
        if (copy_pending) {
            mbar_wait(&S.mbar[buf], (par >> buf) & 1u);
            par ^= 1u << buf;
        }
        if (bail) {
            if (tid == 0) {
                const unsigned int e = atomicAdd(P.bail_count, 1u);
                P.bail_list[e] = SE.s;
            }
        } else {
            S.s_thr[tid] += S.s_ser[tid];
            if (P.aggr_values) {  // the finished row -> the group's partial state
                __syncthreads();
                const double* row = P.out + (size_t)blockIdx.x * P.npoints;
                const size_t cell0 = (size_t)P.group_ids[SE.s] * P.npoints;
                for (uint32_t q = tid; q < P.npoints; q += FU_THREADS) fu_fold(P.aggr_id, P.aggr_values, P.aggr_counts, cell0 + q, row[q]);
            }
        }
        FU_PH(FU_PH_SETUP);
    }
#ifdef VMB_FUSED_PHASES
    if (lane == 0)
        for (int k = 0; k < FU_PH_SLOTS; k++) atomicAdd(&fu_phase_cyc[blockIdx.x][k], S.ph[w][k]);
#endif
    unsigned long long scanned = S.s_thr[tid];
    // block reduce -> one atomic per CTA
    __syncthreads();
#pragma unroll
    for (int o = 16; o; o >>= 1) scanned += shfl_u64(scanned, (lane_id() ^ o));
    if (lane == 0) S.s_part[w] = scanned;
    __syncthreads();
    if (tid == 0) {
        unsigned long long tot = 0;
        for (int k = 0; k < FU_WARPS; k++) tot += S.s_part[k];
        if (tot) atomicAdd(P.scanned, tot);
    }
}

#ifdef VMB_FUSED_PHASES
// phase-clock build only: copies fu_phase_cyc ([FU_PH_CTAS x FU_PH_SLOTS], cycles summed over the warps of a CTA) to `out`,
// then zeroes it (reset != 0); returns FU_PH_SLOTS * 1000 + FU_PH_CTAS so that the caller can check the layout
extern "C" int vmb_fused_phase_cycles(unsigned long long* out, int reset) {
    if (out && cudaMemcpyFromSymbol(out, fu_phase_cyc, sizeof(fu_phase_cyc)) != cudaSuccess) return -1;
    if (reset) {
        static const unsigned long long zero[FU_PH_CTAS][FU_PH_SLOTS] = {};
        if (cudaMemcpyToSymbol(fu_phase_cyc, zero, sizeof(zero)) != cudaSuccess) return -1;
    }
    return FU_PH_SLOTS * 1000 + FU_PH_CTAS;
}
#endif
