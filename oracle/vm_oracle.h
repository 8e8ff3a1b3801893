/*
 * vm_oracle.h -- C API of the CPU ORACLE (test infrastructure, NOT product code).
 *
 * The oracle is a plain C++17 restatement of the reference's (VictoriaMetrics, Go)
 * block codec and rollup executor.  It exists only so that tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs can check (or time) the
 * reference algorithm on the CPU.  Nothing under victoriametrics_b200/ may include,
 * link or dlopen anything from this directory.
 *
 * Every function cites the reference file:line (relative to /root/reference) it follows.
 *
 * Pinning status: pinned against the reference's own known-answer tests
 * (tests/golden/go_kats.json, extracted from the reference *_test.go files by
 * tests/golden/extract_go_kats.py) and, for zstd, against libzstd 1.5.7 -- the very
 * static library the reference's cgo build links
 * (vendor/github.com/valyala/gozstd/libzstd_linux_amd64.a) -- through oracle/_ref.
 */
#ifndef VM_ORACLE_H
#define VM_ORACLE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* error codes shared by the oracle entry points */
#define VMO_OK 0
#define VMO_ERR_SHORT_SRC (-1)       /* int.go:183 "too small len(src)" / unexpected end of varint */
#define VMO_ERR_VARINT_TOO_BIG (-2)  /* int.go:272 */
#define VMO_ERR_VARINT_TOO_LONG (-3) /* int.go:277 */
#define VMO_ERR_TAIL (-4)            /* nearest_delta.go:65 / encoding.go:238 trailing data */
#define VMO_ERR_MARSHAL_TYPE (-5)    /* encoding.go:248 */
#define VMO_ERR_ZSTD (-6)            /* encoding.go:181 */
#define VMO_ERR_CONST_TAIL (-7)      /* encoding.go:217 */
#define VMO_ERR_DELTA_CONST (-8)     /* encoding.go:235 */
#define VMO_ERR_TS_BOUNDS (-9)       /* block.go:298 */
#define VMO_ERR_NO_ZSTD_REF (-100)   /* oracle/_ref/libzstd_ref.so not built (needs /root/reference) */
#define VMO_ERR_CAP (-101)
#define VMO_ERR_BUG (-102)           /* the Go code would logger.Panicf("BUG: ...") */

/* ---- lib/encoding/int.go ---- */
int64_t vmo_marshal_varint64s(uint8_t* dst, size_t cap, const int64_t* vs, size_t n);
int vmo_unmarshal_varint64s(int64_t* dst, size_t n, const uint8_t* src, size_t src_len, size_t* consumed);
int64_t vmo_marshal_int64_be(uint8_t* dst, int64_t v);   /* MarshalInt64 int.go:69 */
int64_t vmo_unmarshal_int64_be(const uint8_t* src);      /* UnmarshalInt64 int.go:79 */

/* ---- lib/encoding/nearest_delta.go, nearest_delta2.go ---- */
void vmo_nearest_delta(int64_t next, int64_t prev, uint8_t pb, uint8_t prev_tz, int64_t* d, uint8_t* tz);
uint8_t vmo_get_trailing_zeros(int64_t v, uint8_t pb);
int64_t vmo_marshal_nearest_delta(uint8_t* dst, size_t cap, const int64_t* src, size_t n, uint8_t pb, int64_t* first);
int64_t vmo_marshal_nearest_delta2(uint8_t* dst, size_t cap, const int64_t* src, size_t n, uint8_t pb, int64_t* first);
int vmo_unmarshal_nearest_delta(int64_t* dst, const uint8_t* src, size_t src_len, int64_t first, size_t n);
int vmo_unmarshal_nearest_delta2(int64_t* dst, const uint8_t* src, size_t src_len, int64_t first, size_t n);

/* ---- lib/encoding/encoding.go ---- */
int vmo_is_const(const int64_t* a, size_t n);
int vmo_is_delta_const(const int64_t* a, size_t n);
int vmo_is_gauge(const int64_t* a, size_t n);
int vmo_get_compress_level(size_t n);
void vmo_ensure_non_decreasing(int64_t* a, size_t n, int64_t vmin, int64_t vmax);
int vmo_check_timestamps_bounds(const int64_t* ts, size_t n, int64_t tmin, int64_t tmax);
/* marshalInt64Array encoding.go:119.  Returns bytes written or <0. */
int64_t vmo_marshal_int64_array(uint8_t* dst, size_t cap, const int64_t* a, size_t n, uint8_t pb, int* mt, int64_t* first);
/* unmarshalInt64Array encoding.go:173 */
int vmo_unmarshal_int64_array(int64_t* dst, const uint8_t* src, size_t src_len, int mt, int64_t first, size_t n);

/* ---- zstd ---- */
/* own restatement of the zstd frame format (RFC 8878); returns regenerated size or <0 */
int64_t vmo_zstd_decompress(uint8_t* dst, size_t cap, const uint8_t* src, size_t src_len);
int64_t vmo_zstd_content_size(const uint8_t* src, size_t src_len);
/* Frame_Content_Size, or for a frame without one an upper bound of its content from the block headers */
int64_t vmo_zstd_content_bound(const uint8_t* src, size_t src_len);
/* libzstd 1.5.7 (the reference's own) through oracle/_ref/libzstd_ref.so */
int vmo_zstd_ref_available(void);
int64_t vmo_zstd_ref_compress(uint8_t* dst, size_t cap, const uint8_t* src, size_t n, int level);
int64_t vmo_zstd_ref_decompress(uint8_t* dst, size_t cap, const uint8_t* src, size_t n);
int64_t vmo_zstd_ref_compress_checksum(uint8_t* dst, size_t cap, const uint8_t* src, size_t n, int level); /* with Content_Checksum */
/* both functions below are present (an oracle/_ref built by an older recipe lacks them) */
int vmo_zstd_ref_factory_available(void);
/* ZSTD_compress2 after ZSTD_CCtx_setParameter(kv[2i], kv[2i+1]) for i < nkv */
int64_t vmo_zstd_ref_compress_params(uint8_t* dst, size_t cap, const uint8_t* src, size_t n, const int* kv, int nkv);
/* ZSTD_compressSequences with explicit block delimiters: nseq (offset, literal length, match length) triples */
int64_t vmo_zstd_ref_compress_sequences(uint8_t* dst, size_t cap, const uint8_t* src, size_t n, const uint32_t* seq, size_t nseq,
                                        const int* kv, int nkv);

/* ---- lib/decimal/decimal.go ---- */
double vmo_pow10(int n); /* Go math.Pow10 */
void vmo_decimal_to_float(double* dst, const int64_t* va, size_t n, int16_t e);
int16_t vmo_float_to_decimal(int64_t* dst, const double* src, size_t n);
int16_t vmo_calibrate_scale(int64_t* a, size_t na, int16_t ae, int64_t* b, size_t nb, int16_t be);
void vmo_from_float(double f, int64_t* v, int16_t* e);
void vmo_positive_float_to_decimal(double f, int64_t* v, int16_t* e);
double vmo_to_float(int64_t v, int16_t e);

/* ---- lib/storage/block_header.go (81-byte wire form) ---- */
typedef struct {
    uint8_t tsid[24];
    int64_t min_ts, max_ts, first_value;
    uint64_t ts_off, val_off;
    uint32_t ts_size, val_size, rows;
    int16_t scale;
    uint8_t ts_mt, val_mt, precision_bits;
} vmo_block_header;
void vmo_block_header_marshal(uint8_t dst[81], const vmo_block_header* bh);
void vmo_block_header_unmarshal(vmo_block_header* bh, const uint8_t src[81]);

/* ---- app/vmselect/promql/rollup.go ---- */
typedef struct {
    int func_id;            /* VMO_RF_* below */
    int64_t start, end, step, window;
    int64_t lookback_delta;
    int64_t min_staleness_ms; /* -search.minStalenessInterval */
    int may_adjust_window;
    int is_default_rollup;
    int samples_scanned_per_call;
    const double* args;     /* per-point scalar arg (phis / limits / secs / sf); may be NULL */
    const double* args2;    /* second per-point arg (holt_winters tf) */
} vmo_rollup_cfg;

enum {
    VMO_RF_DEFAULT_ROLLUP = 0, VMO_RF_RATE /*deriv_fast*/, VMO_RF_DELTA /*increase*/, VMO_RF_AVG, VMO_RF_MIN, VMO_RF_MAX,
    VMO_RF_SUM, VMO_RF_COUNT, VMO_RF_QUANTILE, VMO_RF_FIRST, VMO_RF_LAST, VMO_RF_RANGE, VMO_RF_SUM2, VMO_RF_STDDEV,
    VMO_RF_STDVAR, VMO_RF_IDERIV /*irate*/, VMO_RF_IDELTA, VMO_RF_DERIV /*deriv slow*/, VMO_RF_INCREASE_PURE,
    VMO_RF_CHANGES, VMO_RF_CHANGES_PROMETHEUS, VMO_RF_RESETS, VMO_RF_INCREASES, VMO_RF_INTEGRATE, VMO_RF_LAG,
    VMO_RF_LIFETIME, VMO_RF_SCRAPE_INTERVAL, VMO_RF_TMIN, VMO_RF_TMAX, VMO_RF_TFIRST, VMO_RF_TLAST,
    VMO_RF_TLAST_CHANGE, VMO_RF_MODE, VMO_RF_MAD, VMO_RF_OUTLIER_IQR, VMO_RF_ZSCORE, VMO_RF_ASCENT, VMO_RF_DESCENT,
    VMO_RF_DISTINCT, VMO_RF_GEOMEAN, VMO_RF_PREDICT_LINEAR, VMO_RF_HOLT_WINTERS, VMO_RF_HOEFFDING_LOWER,
    VMO_RF_HOEFFDING_UPPER, VMO_RF_DURATION, VMO_RF_COUNT_LE, VMO_RF_COUNT_GT, VMO_RF_COUNT_EQ, VMO_RF_COUNT_NE,
    VMO_RF_SHARE_LE, VMO_RF_SHARE_GT, VMO_RF_SHARE_EQ, VMO_RF_SUM_LE, VMO_RF_SUM_GT, VMO_RF_SUM_EQ,
    VMO_RF_PRESENT, VMO_RF_ABSENT, VMO_RF_STALE_SAMPLES, VMO_RF_MEDIAN, VMO_RF_RATE_OVER_SUM,
    VMO_RF_DELTA_PROMETHEUS, VMO_RF_RATE_PROMETHEUS, VMO_RF_OPEN, VMO_RF_CLOSE, VMO_RF_HIGH, VMO_RF_LOW,
    VMO_RF__COUNT
};

/* rollupConfig.Do rollup.go:688; out has P = 1+(end-start)/step entries. returns samplesScanned */
uint64_t vmo_rollup_do(const vmo_rollup_cfg* cfg, double* out, const double* values, const int64_t* timestamps, size_t n);
double vmo_rollup_func_call(int func_id, double prev_value, int64_t prev_ts, const double* values, const int64_t* ts,
                            size_t n, double real_prev, double real_next, int64_t curr_ts, size_t idx, int64_t window,
                            const double* args, const double* args2);
int64_t vmo_rollup_points(int64_t start, int64_t end, int64_t step);
void vmo_remove_counter_resets(double* values, const int64_t* timestamps, size_t n, int64_t max_staleness);
void vmo_delta_values(double* values, size_t n);
void vmo_deriv_values(double* values, const int64_t* timestamps, size_t n);
size_t vmo_drop_stale_nans(double* values, int64_t* timestamps, size_t n);
/* series assembly: netstorage.go:566 mergeSortBlocks (blocks = row ranges [offsets[b], offsets[b+1]) of ts/vals, each sorted),
 * lib/storage/dedup.go:30 DeduplicateSamples (in place, returns the new length), :158 needsDedup */
size_t vmo_merge_sort_blocks(const int64_t* ts, const double* vals, const uint64_t* offsets, size_t nblocks,
                             int64_t dedup_interval, int64_t* out_ts, double* out_vals);
size_t vmo_deduplicate_samples(int64_t* ts, double* vals, size_t n, int64_t interval);
int vmo_needs_dedup(const int64_t* ts, size_t n, int64_t interval);
int64_t vmo_get_scrape_interval(const int64_t* timestamps, size_t n, int64_t default_interval);
int64_t vmo_get_max_prev_interval(int64_t scrape_interval);
double vmo_quantile(double phi, const double* values, size_t n);
double vmo_mode_no_nans(double prev, double* a, size_t n);
double vmo_linear_regression(const double* values, const int64_t* ts, size_t n, int64_t intercept, double* k);

/* ---- app/vmselect/promql/aggr_incremental.go ---- */
enum { VMO_AGGR_SUM = 0, VMO_AGGR_MIN, VMO_AGGR_MAX, VMO_AGGR_AVG, VMO_AGGR_COUNT, VMO_AGGR_SUM2, VMO_AGGR_GEOMEAN,
       VMO_AGGR_ANY, VMO_AGGR_GROUP };
/* updateAggr* : fold one rolled-up series (P points) into (dst_values, dst_counts) */
void vmo_aggr_update(int aggr, double* dst_values, double* dst_counts, const double* values, size_t p);
/* mergeAggr* */
void vmo_aggr_merge(int aggr, double* dst_values, double* dst_counts, const double* src_values, const double* src_counts, size_t p);
/* finalizeAggr* */
void vmo_aggr_finalize(int aggr, double* dst_values, const double* dst_counts, size_t p);

/* ---- whole hot path on one block, as Block.UnmarshalData + AppendRowsWithTimeRangeFilter do ----
 * (lib/storage/block.go:250, :324). returns rows kept (after time-range filter) or <0 */
int64_t vmo_block_unmarshal(int64_t* ts_out, double* val_out, int64_t* ival_scratch, const vmo_block_header* bh,
                            const uint8_t* ts_data, const uint8_t* val_data, int64_t tr_min, int64_t tr_max);

#ifdef __cplusplus
}
#endif
#endif
