// Rollup executor kernels.
//
// Replaces, for every series of a batch at once:
//   app/vmselect/promql/eval.go:1985   dropStaleNaNs
//   app/vmselect/promql/rollup.go:921  removeCounterResets                       (k_series_prepare)
//   app/vmselect/promql/rollup.go:871  getScrapeInterval, :899 getMaxPrevInterval (k_series_prepare)
//   app/vmselect/promql/rollup.go:701  rollupConfig.doInternal                    (k_rollup: one thread per output point)
//   app/vmselect/promql/rollup.go:1030-2445 the rollup functions                 (call_func)
//   app/vmselect/promql/aggr.go:870 quantile, :541 modeNoNaNs
//   app/vmselect/promql/aggr_incremental.go:189-458 update/merge/finalize         (k_aggr_*)
#include "common.cuh"

namespace {

#define D_NAN __longlong_as_double(0x7ff8000000000001LL)  /* Go math.NaN() bit pattern */
#define D_INF __longlong_as_double(0x7ff0000000000000LL)

__device__ __forceinline__ bool is_stale_nan(double f) { return (uint64_t)__double_as_longlong(f) == VMB_STALE_NAN_BITS; }

// ---- order statistics without storage: the k-th smallest (0-based) non-NaN value of T(v[0..n)).
template <class VP, class T>
__device__ double kth_smallest(VP v, uint32_t n, uint32_t k, T tf) {
    for (uint32_t a = 0; a < n; a++) {
        double x = tf(v[a]);
        if (isnan(x)) continue;
        uint32_t less = 0, leq = 0;
        for (uint32_t b = 0; b < n; b++) {
            double y = tf(v[b]);
            less += (y < x);
            leq += (y <= x);
        }
        if (less <= k && k < leq) return x;
    }
    return D_NAN;
}

struct Ident {
    __device__ double operator()(double x) const { return x; }
};
struct AbsDev {
    double c;
    __device__ double operator()(double x) const { return fabs(x - c); }
};

// quantile aggr.go:870 = drop NaNs, sort, quantileSorted aggr.go:922
template <class VP, class T>
__device__ double quantile_tf(double phi, VP v, uint32_t n, T tf) {
    // quantile_over_time(0.99, m[5m]) and friends: if no value is NaN (the rule, after dropStaleNaNs) both order statistics are
    // among the TWO largest values whenever n - 1 - floor(phi (n - 1)) <= 1 -- one pass keeping two maxima and counting
    if (n && phi >= 0 && phi <= 1) {
        const double rank_n = phi * ((double)n - 1);
        const double lower_n = fmax(0.0, floor(rank_n));
        if ((double)(n - 1) - lower_n <= 1.0) {
            uint32_t m2 = 0;
            double u0 = -D_INF, u1 = -D_INF;  // u0 >= u1
            for (uint32_t a = 0; a < n; a++) {
                const double x = tf(v[a]);
                if (isnan(x)) continue;
                m2++;
                if (x > u1) {
                    u1 = x;
                    if (u1 > u0) { const double s = u0; u0 = u1; u1 = s; }
                }
            }
            if (m2 == n) {
                const double upper_n = fmin((double)n - 1, lower_n + 1);
                const double weight_n = rank_n - floor(rank_n);
                const uint32_t dl = n - 1 - (uint32_t)(int)lower_n, du = n - 1 - (uint32_t)(int)upper_n;
                const double vlo_ = dl == 0 ? u0 : u1, vhi_ = du == 0 ? u0 : u1;
                return vlo_ * (1 - weight_n) + vhi_ * weight_n;
            }
        }
    }
    // one pass: the number of non-NaN values and the four largest of them, sorted in registers (phi = 0.9 ... 1 over the usual
    // 20-sample window needs nothing else)
    uint32_t m = 0;
    double t0 = -D_INF, t1 = -D_INF, t2 = -D_INF, t3 = -D_INF;  // t0 >= t1 >= t2 >= t3
    for (uint32_t a = 0; a < n; a++) {
        double x = tf(v[a]);
        if (isnan(x)) continue;
        m++;
        // (a max / min ladder without branches was measured: 7 DSETP + 14 selects per element on this part, 30 % slower)
        if (x > t3) {
            t3 = x;
            if (t3 > t2) { double s = t2; t2 = t3; t3 = s; }
            if (t2 > t1) { double s = t1; t1 = t2; t2 = s; }
            if (t1 > t0) { double s = t0; t0 = t1; t1 = s; }
        }
    }
    if (m == 0 || isnan(phi)) return D_NAN;
    if (phi < 0) return -D_INF;
    if (phi > 1) return D_INF;
    double nn = (double)m;
    double rank = phi * (nn - 1);
    double lower = fmax(0.0, floor(rank));
    double upper = fmin(nn - 1, lower + 1);
    double weight = rank - floor(rank);
    const uint32_t kl = (uint32_t)(int)lower, ku = (uint32_t)(int)upper;
    double vlo, vhi;
    if (m - 1 - kl <= 3) {
        // both order statistics are among the four largest values
        const uint32_t dl = m - 1 - kl, du = m - 1 - ku;  // distance from the maximum
        vlo = dl == 0 ? t0 : (dl == 1 ? t1 : (dl == 2 ? t2 : t3));
        vhi = du == 0 ? t0 : (du == 1 ? t1 : (du == 2 ? t2 : t3));
    } else if (ku <= 3) {
        t0 = t1 = t2 = t3 = D_INF;  // now t0 <= t1 <= t2 <= t3: the four smallest
        for (uint32_t a = 0; a < n; a++) {
            double x = tf(v[a]);
            if (isnan(x)) continue;
            if (x < t3) {
                t3 = x;
                if (t3 < t2) { double s = t2; t2 = t3; t3 = s; }
                if (t2 < t1) { double s = t1; t1 = t2; t2 = s; }
                if (t1 < t0) { double s = t0; t0 = t1; t1 = s; }
            }
        }
        vlo = kl == 0 ? t0 : (kl == 1 ? t1 : (kl == 2 ? t2 : t3));
        vhi = ku == 0 ? t0 : (ku == 1 ? t1 : (ku == 2 ? t2 : t3));
    } else {
        // general case: rank every value once, pick both neighbours of the rank in the same pass
        vlo = vhi = D_NAN;
        for (uint32_t a = 0; a < n; a++) {
            double x = tf(v[a]);
            if (isnan(x)) continue;
            uint32_t less = 0, leq = 0;
            for (uint32_t b = 0; b < n; b++) {
                double y = tf(v[b]);
                less += (y < x);
                leq += (y <= x);
            }
            if (less <= kl && kl < leq) vlo = x;
            if (less <= ku && ku < leq) vhi = x;
        }
    }
    return vlo * (1 - weight) + vhi * weight;
}
template <class VP>
__device__ double quantile(double phi, VP v, uint32_t n) { return quantile_tf(phi, v, n, Ident()); }

// rollupFuncArg rollup.go:523.  VP / TP: how the window's values / timestamps are reached -- plain pointers for columns in global
// or shared memory, small view types (operator[], +, ++) for the fused kernel's swizzled ring of values and its computed
// timestamps (fused.cu)
template <class VP, class TP>
struct WinT {
    double prevValue;
    int64_t prevTimestamp;
    VP values;
    TP timestamps;
    uint32_t n;
    double realPrevValue, realNextValue;
    int64_t currTimestamp;
    uint32_t idx;
    int64_t window;
    const double* args;
    const double* args2;
};

// stdvar rollup.go:1808 in step form: add() takes the values in order, result(n) applies the fast paths on n = len(values),
// NaNs counted.  Shared by the rollup windows and the whole-row range_stddev / range_stdvar / range_zscore (range_transform.inc).
struct Welford {
    double avg = 0, count = 0, q = 0;
    __device__ __forceinline__ void add(double x) {
        if (isnan(x)) return;
        count += 1;
        double avgNew = avg + (x - avg) / count;
        q += (x - avg) * (x - avgNew);
        avg = avgNew;
    }
    __device__ __forceinline__ double result(uint64_t n) const {
        if (n == 0) return D_NAN;
        if (n == 1) return 0;
        if (count == 0) return D_NAN;
        return q / count;
    }
};
template <class VP>
__device__ double stdvar(VP v, uint32_t n) {
    Welford w;
    if (n > 1)
        for (uint32_t i = 0; i < n; i++) w.add(v[i]);
    return w.result(n);
}
template <class W>
__device__ double r_sum(const W& r) {
    if (r.n == 0) return D_NAN;
    double s = 0;
    for (uint32_t i = 0; i < r.n; i++) s += r.values[i];
    return s;
}
template <class W>
__device__ double r_avg(const W& r) { return r.n == 0 ? D_NAN : r_sum(r) / (double)r.n; }
template <class W>
__device__ double r_min(const W& r) {
    if (r.n == 0) return D_NAN;
    double m = r.values[0];
    for (uint32_t i = 0; i < r.n; i++)
        if (r.values[i] < m) m = r.values[i];
    return m;
}
template <class W>
__device__ double r_max(const W& r) {
    if (r.n == 0) return D_NAN;
    double m = r.values[0];
    for (uint32_t i = 0; i < r.n; i++)
        if (r.values[i] > m) m = r.values[i];
    return m;
}
template <class W>
__device__ double r_last(const W& r) { return r.n == 0 ? D_NAN : r.values[r.n - 1]; }
template <class W>
__device__ double r_lag(const W& r) {  // rollup.go:2055
    if (r.n == 0) {
        if (isnan(r.prevValue)) return D_NAN;
        return (double)(r.currTimestamp - r.prevTimestamp) / 1e3;
    }
    return (double)(r.currTimestamp - r.timestamps[r.n - 1]) / 1e3;
}
template <class W>
__device__ double r_scrape_interval(const W& r) {  // rollup.go:2067
    if (isnan(r.prevValue)) {
        if (r.n < 2) return D_NAN;
        return ((double)(r.timestamps[r.n - 1] - r.timestamps[0]) / 1e3) / (double)(r.n - 1);
    }
    if (r.n == 0) return D_NAN;
    return ((double)(r.timestamps[r.n - 1] - r.prevTimestamp) / 1e3) / (double)r.n;
}

// linearRegression rollup.go:1108-1134 (after the empty and constant cases) in step form: add() takes the non-NaN (dt, v) pairs
// in order, fit() gives (v, k).  Shared by the rollup windows and the whole-row range_linear_regression (range_transform.inc).
struct LinRegSums {
    double vSum = 0, tSum = 0, tvSum = 0, ttSum = 0;
    int cnt = 0;
    __device__ __forceinline__ void add(double dt, double v) {
        vSum += v;
        tSum += dt;
        tvSum = __dadd_rn(tvSum, __dmul_rn(dt, v));  // no FMA contraction: Go does not fuse on amd64
        ttSum = __dadd_rn(ttSum, __dmul_rn(dt, dt));
        cnt++;
    }
    __device__ __forceinline__ void fit(double* vout, double* kout) const {
        if (cnt == 0) {
            *vout = D_NAN;
            *kout = D_NAN;
            return;
        }
        double k = 0;
        double tDiff = __dsub_rn(ttSum, __ddiv_rn(__dmul_rn(tSum, tSum), (double)cnt));
        if (fabs(tDiff) >= 1e-6) k = __ddiv_rn(__dsub_rn(tvSum, __ddiv_rn(__dmul_rn(tSum, vSum), (double)cnt)), tDiff);
        *vout = __dsub_rn(__ddiv_rn(vSum, (double)cnt), __ddiv_rn(__dmul_rn(k, tSum), (double)cnt));
        *kout = k;
    }
};

template <class W>
__device__ void linear_regression(const W& r, double* vout, double* kout) {  // rollup.go:1099
    auto values = r.values;
    uint32_t n = r.n;
    if (n == 0) {
        *vout = D_NAN;
        *kout = D_NAN;
        return;
    }
    bool isconst = true;  // areConstValues rollup.go:1136
    for (uint32_t i = 1; i < n; i++)
        if (values[i] != values[i - 1]) {
            isconst = false;
            break;
        }
    if (isconst) {
        *vout = values[0];
        *kout = 0;
        return;
    }
    LinRegSums s;
    for (uint32_t i = 0; i < n; i++) {
        double v = values[i];
        if (isnan(v)) continue;
        s.add((double)(r.timestamps[i] - r.currTimestamp) / 1e3, v);
    }
    s.fit(vout, kout);
}

template <class W>
__device__ double r_delta(const W& r) {  // rollupDelta rollup.go:1859
    auto values = r.values;
    uint32_t n = r.n;
    double prevValue = r.prevValue;
    if (isnan(prevValue)) {
        if (n == 0) return D_NAN;
        if (!isnan(r.realPrevValue)) return values[n - 1] - r.realPrevValue;
        double d = 0;
        if (n > 1) d = values[1] - values[0];
        else if (!isnan(r.realNextValue)) d = r.realNextValue - values[0];
        if (fabs(values[0]) < 10 * (fabs(d) + 1)) prevValue = 0;
        else {
            prevValue = values[0];
            values++;
            n--;
        }
    }
    if (n == 0) return 0;
    return values[n - 1] - prevValue;
}
template <class W>
__device__ double r_deriv_fast(const W& r) {  // rollupDerivFast rollup.go:1954
    double prevValue = r.prevValue;
    int64_t prevTimestamp = r.prevTimestamp;
    if (isnan(prevValue)) {
        if (r.n < 2) return D_NAN;
        prevValue = r.values[0];
        prevTimestamp = r.timestamps[0];
    } else if (r.n == 0) {
        return 0;
    }
    double dv = r.values[r.n - 1] - prevValue;
    double dt = (double)(r.timestamps[r.n - 1] - prevTimestamp) / 1e3;
    return dv / dt;
}
template <class W>
__device__ double r_ideriv(const W& r) {  // rollupIderiv rollup.go:1991
    auto values = r.values;
    auto ts = r.timestamps;
    uint32_t n = r.n;
    if (n < 2) {
        if (n == 0) return D_NAN;
        if (isnan(r.prevValue)) return D_NAN;
        return (values[0] - r.prevValue) / ((double)(ts[0] - r.prevTimestamp) / 1e3);
    }
    double vEnd = values[n - 1];
    int64_t tEnd = ts[n - 1];
    uint32_t tn = n - 1;
    while (tn > 0 && ts[tn - 1] >= tEnd) tn--;
    int64_t tStart;
    double vStart;
    if (tn == 0) {
        if (isnan(r.prevValue)) return 0;
        tStart = r.prevTimestamp;
        vStart = r.prevValue;
    } else {
        tStart = ts[tn - 1];
        vStart = values[tn - 1];
    }
    return (vEnd - vStart) / ((double)(tEnd - tStart) / 1e3);
}
template <class W>
__device__ double r_idelta(const W& r) {  // rollup.go:1915
    if (r.n == 0) return isnan(r.prevValue) ? D_NAN : 0.0;
    double last = r.values[r.n - 1];
    if (r.n == 1) return isnan(r.prevValue) ? last : last - r.prevValue;
    return last - r.values[r.n - 2];
}
template <class W>
__device__ double r_increase_pure(const W& r) {  // rollup.go:1835
    double prevValue = r.prevValue;
    if (isnan(prevValue)) {
        if (r.n == 0) return D_NAN;
        prevValue = 0;
        if (!isnan(r.realPrevValue)) prevValue = r.realPrevValue;
    }
    if (r.n == 0) return 0;
    return r.values[r.n - 1] - prevValue;
}
template <class W>
__device__ double r_changes(const W& r, bool prometheus) {  // rollup.go:2106 / :2080
    auto values = r.values;
    uint32_t n = r.n;
    double prev;
    int cnt = 0;
    if (prometheus) {
        if (n < 1) return D_NAN;
        prev = values[0];
        values++;
        n--;
    } else {
        prev = r.prevValue;
        if (isnan(prev)) {
            if (n == 0) return D_NAN;
            if (!isnan(r.realPrevValue)) prev = r.realPrevValue;
            else {
                cnt++;
                prev = values[0];
                values++;
                n--;
            }
        }
    }
    for (uint32_t i = 0; i < n; i++) {
        double v = values[i];
        if (v != prev) {
            if (fabs(v - prev) < 1e-12 * fabs(v)) continue;
            cnt++;
            prev = v;
        }
    }
    return (double)cnt;
}
template <class W>
__device__ double r_incr_or_resets(const W& r, bool increases) {  // rollup.go:2139 / :2174
    auto values = r.values;
    uint32_t n = r.n;
    if (n == 0) return isnan(r.prevValue) ? D_NAN : 0.0;
    double prev = r.prevValue;
    if (isnan(prev)) {
        prev = values[0];
        values++;
        n--;
    }
    if (n == 0) return 0;
    int cnt = 0;
    for (uint32_t i = 0; i < n; i++) {
        double v = values[i];
        bool hit = increases ? (v > prev) : (v < prev);
        if (hit) {
            if (fabs(v - prev) < 1e-12 * fabs(v)) continue;
            cnt++;
        }
        prev = v;
    }
    return (double)cnt;
}
template <class W>
__device__ double r_integrate(const W& r) {  // rollup.go:2417
    auto values = r.values;
    auto ts = r.timestamps;
    uint32_t n = r.n;
    double prevValue = r.prevValue;
    int64_t prevTimestamp = r.currTimestamp - r.window;
    if (isnan(prevValue)) {
        if (n == 0) return D_NAN;
        prevValue = values[0];
        prevTimestamp = ts[0];
        values++;
        ts++;
        n--;
    }
    double sum = 0;
    for (uint32_t i = 0; i < n; i++) {
        double dt = (double)(ts[i] - prevTimestamp) / 1e3;
        sum = __dadd_rn(sum, __dmul_rn(prevValue, dt));
        prevTimestamp = ts[i];
        prevValue = values[i];
    }
    double dt = (double)(r.currTimestamp - prevTimestamp) / 1e3;
    return __dadd_rn(sum, __dmul_rn(prevValue, dt));
}
template <class W>
__device__ double r_lifetime(const W& r) {  // rollup.go:2040
    if (isnan(r.prevValue)) {
        if (r.n < 2) return D_NAN;
        return (double)(r.timestamps[r.n - 1] - r.timestamps[0]) / 1e3;
    }
    if (r.n == 0) return D_NAN;
    return (double)(r.timestamps[r.n - 1] - r.prevTimestamp) / 1e3;
}
template <class W>
__device__ double r_tminmax(const W& r, bool is_min) {  // rollup.go:1603 / :1623
    if (r.n == 0) return D_NAN;
    double m = r.values[0];
    int64_t t = r.timestamps[0];
    for (uint32_t i = 0; i < r.n; i++) {
        double v = r.values[i];
        if (is_min ? (v <= m) : (v >= m)) {
            m = v;
            t = r.timestamps[i];
        }
    }
    return (double)t / 1e3;
}
template <class W>
__device__ double r_tlast_change(const W& r) {  // rollup.go:1669
    if (r.n == 0) return D_NAN;
    double last = r.values[r.n - 1];
    for (int i = (int)r.n - 2; i >= 0; i--)
        if (r.values[i] != last) return (double)r.timestamps[i + 1] / 1e3;
    if (isnan(r.prevValue) || r.prevValue != last) return (double)r.timestamps[0] / 1e3;
    return D_NAN;
}
// modeNoNaNs aggr.go:541 driven by runs of equal values in ascending order (no sort buffer)
template <class W>
__device__ double r_mode(const W& r) {
    double prevValue = r.prevValue;
    uint32_t n = r.n;
    if (n == 0) return prevValue;
    auto v = r.values;
    long long j = -1, dMax = 0;
    double mode = prevValue;
    // the Go code sorts with sort.Float64s, which orders NaNs first; windows never hold NaNs here (eval.go:1985)
    double cur = -D_INF;
    bool first = true;
    uint32_t consumed = 0;  // sorted index of the current run start
    while (consumed < n) {
        // next distinct value: the smallest value > cur (or >= -inf for the first run)
        double nxt = D_INF;
        bool found = false;
        for (uint32_t a = 0; a < n; a++) {
            double x = v[a];
            if ((first ? (x >= cur) : (x > cur)) && (!found || x < nxt)) {
                nxt = x;
                found = true;
            }
        }
        if (!found) break;  // only NaNs left
        uint32_t c = 0;
        for (uint32_t a = 0; a < n; a++) c += (v[a] == nxt);
        long long i = consumed;
        if (!(prevValue == nxt)) {
            long long d = i - j;
            if (d > dMax || isnan(mode)) {
                dMax = d;
                mode = prevValue;
            }
            j = i;
            prevValue = nxt;
        }
        consumed += c;
        cur = nxt;
        first = false;
    }
    long long d = (long long)n - j;
    if (d > dMax || isnan(mode)) mode = prevValue;
    return mode;
}
template <class W>
__device__ double r_outlier_iqr(const W& r) {  // rollup.go:1427
    if (r.n < 2) return D_NAN;
    double q25 = quantile(0.25, r.values, r.n), q75 = quantile(0.75, r.values, r.n);
    double iqr = 1.5 * (q75 - q25);
    double v = r.values[r.n - 1];
    if (v > q75 + iqr || v < q25 - iqr) return v;
    return D_NAN;
}
template <class W>
__device__ double r_zscore(const W& r) {  // rollup.go:2361
    double si = r_scrape_interval(r), lag = r_lag(r);
    if (isnan(si) || isnan(lag) || lag > si) return D_NAN;
    double d = r_last(r) - r_avg(r);
    if (d == 0) return 0;
    return d / sqrt(stdvar(r.values, r.n));
}
template <class W>
__device__ double r_ascent_descent(const W& r, bool ascent) {  // rollup.go:2315 / :2338
    auto values = r.values;
    uint32_t n = r.n;
    double prev = r.prevValue;
    if (isnan(prev)) {
        if (n == 0) return D_NAN;
        prev = values[0];
        values++;
        n--;
    }
    double s = 0;
    for (uint32_t i = 0; i < n; i++) {
        double v = values[i];
        double d = ascent ? (v - prev) : (prev - v);
        if (d > 0) s += d;
        prev = v;
    }
    return s;
}
template <class W>
__device__ double r_distinct(const W& r) {  // rollup.go:2403 (Go map[float64]: NaN keys never collide)
    if (r.n == 0) return D_NAN;
    uint32_t d = 0;
    for (uint32_t a = 0; a < r.n; a++) {
        double x = r.values[a];
        bool dup = false;
        for (uint32_t b = 0; b < a; b++)
            if (r.values[b] == x) {
                dup = true;
                break;
            }
        d += !dup;
    }
    return (double)d;
}
template <class W>
__device__ double r_holt_winters(const W& r) {  // rollup.go:1030
    auto values = r.values;
    uint32_t n = r.n;
    if (n == 0) return D_NAN;
    double sf = r.args[r.idx];
    if (sf < 0 || sf > 1) return D_NAN;
    double tf = r.args2[r.idx];
    if (tf < 0 || tf > 1) return D_NAN;
    double s0 = r.prevValue;
    if (isnan(s0)) {
        s0 = values[0];
        values++;
        n--;
        if (n == 0) return s0;
    }
    double b0 = values[0] - s0;
    for (uint32_t i = 0; i < n; i++) {
        double v = values[i];
        double s1 = __dadd_rn(__dmul_rn(sf, v), __dmul_rn(1 - sf, s0 + b0));
        double b1 = __dadd_rn(__dmul_rn(tf, s1 - s0), __dmul_rn(1 - tf, b0));
        s0 = s1;
        b0 = b1;
    }
    return s0;
}
template <class W>
__device__ void hoeffding(const W& r, double* bound, double* avg) {  // rollup.go:1353
    if (r.n == 0) {
        *bound = D_NAN;
        *avg = D_NAN;
        return;
    }
    if (r.n == 1) {
        *bound = 0;
        *avg = r.values[0];
        return;
    }
    double vRange = r_max(r) - r_min(r);
    *avg = r_avg(r);
    if (vRange <= 0) {
        *bound = 0;
        return;
    }
    double phi = r.args[r.idx];
    if (phi >= 1) {
        *bound = D_INF;
        return;
    }
    if (phi <= 0) {
        *bound = 0;
        return;
    }
    *bound = vRange * sqrt(log(1 / (1 - phi)) / (2 * (double)r.n));
}
template <class W>
__device__ double r_duration(const W& r) {  // rollup.go:1151
    if (r.n == 0) return D_NAN;
    int64_t tPrev = r.timestamps[0], dSum = 0;
    int64_t dMax = (int64_t)(r.args[r.idx] * 1000);
    for (uint32_t i = 0; i < r.n; i++) {
        int64_t d = r.timestamps[i] - tPrev;
        if (d <= dMax) dSum += d;
        tPrev = r.timestamps[i];
    }
    return (double)dSum / 1000;
}
enum { F_LE, F_GT, F_EQ, F_NE };
template <class W>
__device__ double r_filter(const W& r, int cmp, bool sum, bool share) {  // rollup.go:1321, :1275
    if (r.n == 0) return D_NAN;
    double lim = r.args[r.idx], acc = 0;
    int cnt = 0;
    for (uint32_t i = 0; i < r.n; i++) {
        double v = r.values[i];
        bool hit = cmp == F_LE ? v <= lim : cmp == F_GT ? v > lim : cmp == F_EQ ? v == lim : v != lim;
        if (hit) {
            acc += v;
            cnt++;
        }
    }
    if (sum) return acc;
    if (share) return (double)cnt / (double)r.n;
    return (double)cnt;
}
template <class W>
__device__ uint32_t candlestick_len(const W& r) {  // rollup.go:2228
    uint32_t n = r.n;
    while (n > 0 && r.timestamps[n - 1] >= r.currTimestamp) n--;
    return n;
}
template <class W>
__device__ double candlestick_first(const W& r) {
    return (r.prevTimestamp + r.window >= r.currTimestamp) ? r.prevValue : D_NAN;
}

template <class W>
__device__ double call_func(int f, const W& r) {
    switch (f) {
        case VMB_RF_DEFAULT_ROLLUP:
        case VMB_RF_LAST: return r_last(r);
        case VMB_RF_RATE: return r_deriv_fast(r);
        case VMB_RF_DELTA: return r_delta(r);
        case VMB_RF_AVG: return r_avg(r);
        case VMB_RF_MIN: return r_min(r);
        case VMB_RF_MAX: return r_max(r);
        case VMB_RF_SUM: return r_sum(r);
        case VMB_RF_COUNT: return r.n == 0 ? D_NAN : (double)r.n;
        case VMB_RF_QUANTILE: return quantile(r.args[r.idx], r.values, r.n);
        case VMB_RF_MEDIAN: return quantile(0.5, r.values, r.n);
        case VMB_RF_FIRST: return r.n == 0 ? D_NAN : r.values[0];
        case VMB_RF_RANGE: return r_max(r) - r_min(r);
        case VMB_RF_SUM2: {
            if (r.n == 0) return D_NAN;
            double s = 0;
            for (uint32_t i = 0; i < r.n; i++) s = __dadd_rn(s, __dmul_rn(r.values[i], r.values[i]));
            return s;
        }
        case VMB_RF_STDDEV: return sqrt(stdvar(r.values, r.n));
        case VMB_RF_STDVAR: return stdvar(r.values, r.n);
        case VMB_RF_IDERIV: return r_ideriv(r);
        case VMB_RF_IDELTA: return r_idelta(r);
        case VMB_RF_DERIV: {
            double v, k;
            linear_regression(r, &v, &k);
            return k;
        }
        case VMB_RF_INCREASE_PURE: return r_increase_pure(r);
        case VMB_RF_CHANGES: return r_changes(r, false);
        case VMB_RF_CHANGES_PROMETHEUS: return r_changes(r, true);
        case VMB_RF_RESETS: return r_incr_or_resets(r, false);
        case VMB_RF_INCREASES: return r_incr_or_resets(r, true);
        case VMB_RF_INTEGRATE: return r_integrate(r);
        case VMB_RF_LAG: return r_lag(r);
        case VMB_RF_LIFETIME: return r_lifetime(r);
        case VMB_RF_SCRAPE_INTERVAL: return r_scrape_interval(r);
        case VMB_RF_TMIN: return r_tminmax(r, true);
        case VMB_RF_TMAX: return r_tminmax(r, false);
        case VMB_RF_TFIRST: return r.n == 0 ? D_NAN : (double)r.timestamps[0] / 1e3;
        case VMB_RF_TLAST: return r.n == 0 ? D_NAN : (double)r.timestamps[r.n - 1] / 1e3;
        case VMB_RF_TLAST_CHANGE: return r_tlast_change(r);
        case VMB_RF_MODE: return r_mode(r);
        case VMB_RF_MAD: {  // rollup.go:1469 mad
            double median = quantile(0.5, r.values, r.n);
            return quantile_tf(0.5, r.values, r.n, AbsDev{median});
        }
        case VMB_RF_OUTLIER_IQR: return r_outlier_iqr(r);
        case VMB_RF_ZSCORE: return r_zscore(r);
        case VMB_RF_ASCENT: return r_ascent_descent(r, true);
        case VMB_RF_DESCENT: return r_ascent_descent(r, false);
        case VMB_RF_DISTINCT: return r_distinct(r);
        case VMB_RF_GEOMEAN: {  // rollup.go:1741
            if (r.n == 0) return D_NAN;
            double p = 1.0;
            for (uint32_t i = 0; i < r.n; i++) p *= r.values[i];
            return pow(p, 1 / (double)r.n);
        }
        case VMB_RF_PREDICT_LINEAR: {  // rollup.go:1080
            double v, k;
            linear_regression(r, &v, &k);
            if (isnan(v)) return D_NAN;
            return __dadd_rn(v, __dmul_rn(k, r.args[r.idx]));
        }
        case VMB_RF_HOLT_WINTERS: return r_holt_winters(r);
        case VMB_RF_HOEFFDING_LOWER: {
            double b, a;
            hoeffding(r, &b, &a);
            return a - b;
        }
        case VMB_RF_HOEFFDING_UPPER: {
            double b, a;
            hoeffding(r, &b, &a);
            return a + b;
        }
        case VMB_RF_DURATION: return r_duration(r);
        case VMB_RF_COUNT_LE: return r_filter(r, F_LE, false, false);
        case VMB_RF_COUNT_GT: return r_filter(r, F_GT, false, false);
        case VMB_RF_COUNT_EQ: return r_filter(r, F_EQ, false, false);
        case VMB_RF_COUNT_NE: return r_filter(r, F_NE, false, false);
        case VMB_RF_SHARE_LE: return r_filter(r, F_LE, false, true);
        case VMB_RF_SHARE_GT: return r_filter(r, F_GT, false, true);
        case VMB_RF_SHARE_EQ: return r_filter(r, F_EQ, false, true);
        case VMB_RF_SUM_LE: return r_filter(r, F_LE, true, false);
        case VMB_RF_SUM_GT: return r_filter(r, F_GT, true, false);
        case VMB_RF_SUM_EQ: return r_filter(r, F_EQ, true, false);
        case VMB_RF_PRESENT: return r.n > 0 ? 1.0 : D_NAN;
        case VMB_RF_ABSENT: return r.n == 0 ? 1.0 : D_NAN;
        case VMB_RF_STALE_SAMPLES: {
            if (r.n == 0) return D_NAN;
            int c = 0;
            for (uint32_t i = 0; i < r.n; i++) c += is_stale_nan(r.values[i]);
            return (double)c;
        }
        case VMB_RF_RATE_OVER_SUM: {  // rollup.go:1705
            if (r.n == 0) return D_NAN;
            double sum = 0;
            for (uint32_t i = 0; i < r.n; i++) sum += r.values[i];
            return sum / ((double)r.window / 1e3);
        }
        case VMB_RF_DELTA_PROMETHEUS: return r.n < 2 ? D_NAN : r.values[r.n - 1] - r.values[0];  // rollup.go:1903
        case VMB_RF_RATE_PROMETHEUS: {  // rollup.go:1946
            if (r.n < 2) return D_NAN;
            double delta = r.values[r.n - 1] - r.values[0];
            if (isnan(delta) || r.window == 0) return D_NAN;
            return delta / ((double)r.window / 1e3);
        }
        case VMB_RF_OPEN: {
            double v = candlestick_first(r);
            if (!isnan(v)) return v;
            return candlestick_len(r) == 0 ? D_NAN : r.values[0];
        }
        case VMB_RF_CLOSE: {
            uint32_t n = candlestick_len(r);
            return n == 0 ? candlestick_first(r) : r.values[n - 1];
        }
        case VMB_RF_HIGH:
        case VMB_RF_LOW: {
            uint32_t n = candlestick_len(r);
            auto values = r.values;
            double m = candlestick_first(r);
            if (isnan(m)) {
                if (n == 0) return D_NAN;
                m = values[0];
                values++;
                n--;
            }
            for (uint32_t i = 0; i < n; i++)
                if (f == VMB_RF_HIGH ? values[i] > m : values[i] < m) m = values[i];
            return m;
        }
    }
    return D_NAN;
}

// first index in ts[0..n) with ts > x  (== seekFirstTimestampIdxAfter rollup.go:825 on sorted input)
__device__ __forceinline__ uint32_t upper_bound_ts(const int64_t* __restrict__ ts, uint32_t n, int64_t x) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        uint32_t mid = (lo + hi) >> 1;
        if (ts[mid] <= x) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

}  // namespace

struct RollupParams {
    vmb_rollup_cfg cfg;      // args/args2 replaced by DEVICE pointers (or nullptr)
    SeriesMeta* meta;
    int64_t* ts;
    double* vals;
    double* out;             // [nseries x P]
    const uint32_t* out_rows;  // series s writes row out_rows[s] of `out` (nullptr: row s)
    unsigned long long* scanned;  // device accumulator
    uint32_t nseries;
    uint32_t npoints;
    // series assembly from decoded blocks (nullptr when the batch was built from host columns)
    const uint32_t* ser_first_block;
    const uint32_t* ser_nblocks;
    const uint64_t* row_off;
    const uint32_t* blk_lo;
    const uint32_t* blk_hi;
    const vmb_block_desc* descs;
    int32_t* blk_status;
    unsigned int* failed_blocks;  // device counter: blocks with a non-zero status
    // series whose blocks overlap in time (or touch): merged into [rows_total + ser_merge_off[s], ...) of ts/vals
    const uint64_t* ser_merge_off;  // per series, UINT64_MAX = blocks are disjoint (plain concatenation); may be nullptr
    uint64_t rows_total;            // rows of the decoded blocks = start of the merge area
    uint32_t* merge_heap;           // scratch, one entry per block: the sortBlocksHeap of the series
    uint32_t* merge_next;           // scratch, one entry per block: sortBlock.NextIdx
    int64_t dedup_interval;         // storage.GetDedupInterval(), ms; 0 = off
};

// one thread per series: [start, n) from the kept row ranges of its blocks (netstorage.go:444 unpackTo + the part of
// mergeSortBlocks netstorage.go:566 that needs no data movement: blocks that are disjoint in time were laid out in time order
// by the host plan, so the series is the concatenation of their kept rows).  Series with overlapping blocks get their start
// in the merge area and are filled by k_series_merge.
__global__ void k_series_assemble(RollupParams P) {
    uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= P.nseries) return;
    uint32_t fb = P.ser_first_block[s], nb = P.ser_nblocks[s];
    SeriesMeta m;
    m.start = 0;
    m.n = 0;
    m.flags = 0u;
    m.max_prev_interval = 0;
    m.window = 0;
    bool failed = false;
    for (uint32_t k = 0; k < nb; k++) {  // staleness markers and value drops: known per block from the decode kernel
        if (P.blk_status[fb + k]) failed = true;
        if (blk_hi_stale(P.blk_hi[fb + k])) m.flags |= VMB_SER_STALE;
        if (blk_hi_may_change(P.blk_hi[fb + k])) m.flags |= VMB_SER_DROP;
    }
    const uint64_t moff = P.ser_merge_off ? P.ser_merge_off[s] : ~0ull;
    if (!failed && nb) {
        if (moff != ~0ull) {
            m.start = P.rows_total + moff;
            m.flags |= VMB_SER_MERGED | VMB_SER_DROP;  // (merged rows interleave blocks: always a candidate for removeCounterResets)
        } else {
            uint64_t lo = ~0ull, hi = 0, kept = 0;
            for (uint32_t k = 0; k < nb; k++) {
                const uint32_t a = P.blk_lo[fb + k], b = blk_hi_end(P.blk_hi[fb + k]);
                if (b <= a) continue;  // trimmed away completely
                const uint64_t r = P.row_off[fb + k];
                lo = r + a < lo ? r + a : lo;
                hi = r + b > hi ? r + b : hi;
                kept += b - a;
            }
            // a value drop across a block boundary (time-disjoint blocks, laid out in time order): compare the decoded values
            // on both sides of every boundary.  Many blocks per series: no search, the series is simply a candidate.
            if (nb > 1 && !(m.flags & VMB_SER_DROP)) {
                if (nb > 16) m.flags |= VMB_SER_DROP;
                else {
                    for (uint32_t k = 0; k < nb && !(m.flags & VMB_SER_DROP); k++) {
                        const uint64_t endk = P.row_off[fb + k] + P.descs[fb + k].rows;  // first row of the next block in layout
                        for (uint32_t j = 0; j < nb; j++) {
                            if (j != k && P.row_off[fb + j] == endk && P.descs[fb + j].rows) {
                                const double a = P.vals[endk - 1], b = P.vals[endk];
                                if (!(b - a >= 0)) m.flags |= VMB_SER_DROP;  // drop or NaN
                            }
                        }
                    }
                }
            }
            if (kept) {
                if (hi - lo != kept) {  // a hole inside the series: cannot happen for time-disjoint blocks and one time range
                    for (uint32_t k = 0; k < nb; k++) P.blk_status[fb + k] = VMB_ERR_BLOCK_ORDER;
                    failed = true;
                } else {
                    m.start = lo;
                    m.n = (uint32_t)kept;
                    // (precisionBits < 64 sends the timestamps through EnsureNonDecreasingSequence, which may move the last one)
                    if (nb == 1 && kept >= 2 && P.descs[fb].ts_mt == 2 && P.descs[fb].precision_bits >= 64 && P.dedup_interval <= 0)
                        m.flags |= VMB_SER_TS_AP;
                    if (nb == 1 && P.dedup_interval <= 0 && !(m.flags & VMB_SER_STALE)) {
                        const uint32_t fd = blk_hi_first_drop(P.blk_hi[fb]), a = P.blk_lo[fb];
                        if (fd > a) m.set_first_drop(fd - a);
                    }
                }
            }
        }
    }
    P.meta[s] = m;
    if (failed && P.failed_blocks) atomicAdd(P.failed_blocks, 1u);
}

// ---- mergeSortBlocks netstorage.go:566 for the series whose blocks overlap: one warp per series replays the reference's
// loop -- container/heap over the blocks ordered by their next timestamp (Init / Fix / Pop with Go's exact sift rules, so
// that samples with equal timestamps come out in the reference's order), "copy from the top block everything not after the
// next block's head" -- with the copies, the binary search and equalSamplesPrefix done by the 32 lanes together.
// All lanes run the control flow redundantly on the same values; lane 0 writes the heap, __syncwarp() orders it.
struct MergeHeap {
    volatile uint32_t* h;     // block ids
    volatile uint32_t* next;  // NextIdx per block (row inside the block)
    const int64_t* ts;
    const uint64_t* row_off;
    int lane;
    __device__ __forceinline__ int64_t head(uint32_t b) const { return ts[row_off[b] + next[b]]; }
    __device__ __forceinline__ bool less(uint32_t i, uint32_t j) const { return head(h[i]) < head(h[j]); }
    __device__ __forceinline__ void swap(uint32_t i, uint32_t j) {
        uint32_t a = h[i], b = h[j];
        __syncwarp();
        if (lane == 0) { h[i] = b; h[j] = a; }
        __syncwarp();
    }
    __device__ bool down(uint32_t i0, uint32_t n) {
        uint32_t i = i0;
        for (;;) {
            uint32_t j1 = 2 * i + 1;
            if (j1 >= n) break;
            uint32_t j = j1;
            if (j1 + 1 < n && less(j1 + 1, j1)) j = j1 + 1;
            if (!less(j, i)) break;
            swap(i, j);
            i = j;
        }
        return i > i0;
    }
};

__global__ void __launch_bounds__(128) k_series_merge(RollupParams P) {
    const int lane = lane_id();
    const uint32_t warps_per_grid = gridDim.x * (blockDim.x >> 5);
    for (uint32_t s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < P.nseries; s += warps_per_grid) {
        if (P.ser_merge_off[s] == ~0ull) continue;
        SeriesMeta m = P.meta[s];
        if (!(m.flags & VMB_SER_MERGED)) continue;  // failed series
        const uint32_t fb = P.ser_first_block[s], nb = P.ser_nblocks[s];
        MergeHeap H;
        H.h = P.merge_heap + fb;
        H.next = P.merge_next;
        H.ts = P.ts;
        H.row_off = P.row_off;
        H.lane = lane;
        uint32_t hn = 0;
        for (uint32_t k = 0; k < nb; k++) {  // empty blocks never enter the heap (netstorage.go:568)
            const uint32_t b = fb + k, lo = P.blk_lo[b], hi = blk_hi_end(P.blk_hi[b]);
            if (hi > lo) {
                if (lane == 0) { H.h[hn] = b; H.next[b] = lo; }
                hn++;
            }
        }
        __syncwarp();
        for (uint32_t i = hn / 2; i-- > 0;) H.down(i, hn);  // heap.Init
        uint64_t o = m.start;
        while (hn) {
            const uint32_t top = H.h[0];
            const uint32_t idx = H.next[top], end = blk_hi_end(P.blk_hi[top]);
            const uint64_t trow = P.row_off[top];
            uint32_t adv, ncopy;
            if (hn == 1) {
                adv = ncopy = end - idx;
            } else {
                uint32_t nx = H.h[1];
                if (hn >= 3 && !(H.head(H.h[1]) <= H.head(H.h[2]))) nx = H.h[2];  // getNextBlock netstorage.go:689
                const int64_t ts_next = H.head(nx);
                uint32_t eq = 0;
                if (P.dedup_interval > 0) {  // equalSamplesPrefix netstorage.go:622: timestamps first, then value bits
                    const uint64_t nrow = P.row_off[nx] + H.next[nx];
                    const uint32_t lim = min(end - idx, blk_hi_end(P.blk_hi[nx]) - H.next[nx]);
                    uint32_t nt = 0;
                    for (; nt < lim; nt += 32) {
                        const uint32_t k = nt + lane;
                        const bool same = k < lim && P.ts[trow + idx + k] == P.ts[nrow + k];
                        const uint32_t bad = ~__ballot_sync(VMB_FULL, same);
                        if (bad) { nt += __ffs((int)bad) - 1; break; }
                    }
                    nt = min(nt, lim);
                    for (; eq < nt; eq += 32) {
                        const uint32_t k = eq + lane;
                        const bool same = k < nt && __double_as_longlong(P.vals[trow + idx + k]) == __double_as_longlong(P.vals[nrow + k]);
                        const uint32_t bad = ~__ballot_sync(VMB_FULL, same);
                        if (bad) { eq += __ffs((int)bad) - 1; break; }
                    }
                    eq = min(eq, nt);
                }
                if (eq > 0) {
                    adv = eq;  // replicated samples at the top are skipped when deduplication is on
                    ncopy = 0;
                } else {
                    // binarySearchTimestamps netstorage.go:646: rows of the top block with timestamp <= ts_next
                    uint32_t c = 0;
                    const uint32_t rem = end - idx;
                    if (P.ts[trow + end - 1] <= ts_next) c = rem;
                    else {
                        for (; c < rem; c += 32) {
                            const uint32_t k = c + lane;
                            const bool le = k < rem && P.ts[trow + idx + k] <= ts_next;
                            const uint32_t gt = ~__ballot_sync(VMB_FULL, le);
                            if (gt) { c += __ffs((int)gt) - 1; break; }
                        }
                        c = min(c, rem);
                    }
                    adv = ncopy = c;
                }
            }
            for (uint32_t k = lane; k < ncopy; k += 32) {
                P.ts[o + k] = P.ts[trow + idx + k];
                P.vals[o + k] = P.vals[trow + idx + k];
            }
            o += ncopy;
            __syncwarp();
            if (lane == 0) H.next[top] = idx + adv;
            __syncwarp();
            if (hn == 1) break;
            if (idx + adv < end) {
                H.down(0, hn);  // heap.Fix(0): up(0) is a no-op
            } else {            // heap.Pop
                H.swap(0, hn - 1);
                H.down(0, hn - 1);
                hn--;
            }
        }
        if (lane == 0) {
            m.n = (uint32_t)(o - m.start);
            P.meta[s] = m;
        }
        __syncwarp();
    }
}

// ---- storage.DeduplicateSamples lib/storage/dedup.go:30, in place, one warp per series.  For non-negative timestamps the
// reference's running tsNext is always the smallest multiple of the interval >= the first timestamp of the current bucket,
// so a row is kept iff it is the last one of its bucket ceil(ts / interval); its value is the maximum over the rows with
// the same timestamp, never a staleness marker when anything else exists (:50-64).  Series with a negative timestamp (Go's %
// truncates toward zero there) replay the sequential loop on lane 0.
__device__ __forceinline__ int64_t dedup_bucket(int64_t t, int64_t d) { return (t + d - 1) / d; }

__device__ double dedup_pick(const int64_t* t, const double* v, uint32_t j) {
    const int64_t tp = t[j];
    double vp = v[j];
    while (j > 0 && t[j - 1] == tp) {
        j--;
        const double x = v[j];
        if (is_stale_nan(x)) continue;
        if (is_stale_nan(vp)) { vp = x; continue; }
        if (x > vp) vp = x;
    }
    return vp;
}

__global__ void __launch_bounds__(128) k_series_dedup(RollupParams P) {
    const int lane = lane_id();
    const int64_t D = P.dedup_interval;
    const uint32_t warps_per_grid = gridDim.x * (blockDim.x >> 5);
    for (uint32_t s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < P.nseries; s += warps_per_grid) {
        SeriesMeta m = P.meta[s];
        const uint32_t n = m.n;
        if (n < 2) continue;
        int64_t* t = P.ts + m.start;
        double* v = P.vals + m.start;
        uint32_t o = 0;
        if (t[0] < 0) {  // timestamps are sorted: the first one decides
            if (lane == 0) {
                int64_t ts_next = t[0] + D - 1;
                ts_next -= ts_next % D;
                bool need = false;  // needsDedup dedup.go:158
                for (uint32_t i = 1; i < n && !need; i++) {
                    if (t[i] <= ts_next) need = true;
                    ts_next += D;
                    if (ts_next < t[i]) { ts_next = t[i] + D - 1; ts_next -= ts_next % D; }
                }
                o = n;
                if (need) {
                    o = 0;
                    ts_next = t[0] + D - 1;
                    ts_next -= ts_next % D;
                    for (uint32_t i = 1; i < n; i++) {
                        const int64_t ti = t[i];
                        if (ti <= ts_next) continue;
                        const double pv = dedup_pick(t, v, i - 1);
                        const int64_t pt = t[i - 1];
                        t[o] = pt; v[o] = pv; o++;
                        ts_next += D;
                        if (ts_next < ti) { ts_next = ti + D - 1; ts_next -= ts_next % D; }
                    }
                    const double pv = dedup_pick(t, v, n - 1);
                    const int64_t pt = t[n - 1];
                    t[o] = pt; v[o] = pv; o++;
                }
            }
            o = __shfl_sync(VMB_FULL, o, 0);
        } else {
            bool need = false;
            for (uint32_t i = 1 + lane; i < n; i += 32) need |= dedup_bucket(t[i], D) == dedup_bucket(t[i - 1], D);
            if (!__any_sync(VMB_FULL, need)) continue;
            for (uint32_t base = 0; base < n; base += 32) {
                const uint32_t i = base + lane;
                bool keep = false;
                int64_t ti = 0;
                double vi = 0.0;
                if (i < n) {
                    ti = t[i];
                    keep = i == n - 1 || dedup_bucket(t[i + 1], D) != dedup_bucket(ti, D);
                    if (keep) vi = dedup_pick(t, v, i);
                }
                const uint32_t bal = __ballot_sync(VMB_FULL, keep);  // also orders the reads above before the writes below
                if (keep) {
                    const uint32_t r = o + __popc(bal & ((1u << lane) - 1u));
                    t[r] = ti;
                    v[r] = vi;
                }
                o += __popc(bal);
                __syncwarp();
            }
        }
        if (lane == 0) {
            m.n = o;
            P.meta[s] = m;
        }
        __syncwarp();
    }
}

struct RcrState {
    double corr, prev_raw, prev_out;
    int64_t prev_ts;
};

// removeCounterResets (rollup.go:921) for one 32-row chunk held one row per lane.  Sequential float semantics are
// preserved: corrections are accumulated in sample order by walking the (rare) reset / staleness-gap events of the chunk;
// the final clamp `values[i] = max(values[i], values[i-1])` is a segmented prefix max (order-independent).  A chunk without
// events (the common case) needs no scan at all: raw values are non-decreasing there, so the clamp is an elementwise max
// with the last output of the previous chunk.
template <class VP>
__device__ __forceinline__ void rcr_chunk(RcrState& st, VP v, uint32_t cb, uint32_t n, double x, int64_t tt,
                                          int64_t max_stale, int lane) {
    const uint32_t i = cb + lane;
    const bool valid = i < n;
    double pv = shfl_up_f64(x, 1);
    int64_t pt = max_stale > 0 ? (int64_t)shfl_up_u64((uint64_t)tt, 1) : 0;
    if (lane == 0) {
        pv = cb == 0 ? x : st.prev_raw;
        pt = cb == 0 ? tt : st.prev_ts;
    }
    const double d = x - pv;
    const bool is_reset = valid && d < 0;
    const bool is_gap = valid && i > 0 && max_stale > 0 && (tt - pt) > max_stale;
    uint32_t ev = __ballot_sync(VMB_FULL, is_reset || is_gap || (valid && (isnan(x) || i == 0)));
    double outv;
    if (ev == 0) {
        double a = x + st.corr;
        outv = (a < st.prev_out) ? st.prev_out : a;
    } else {
        double amt = 0.0;
        if (is_reset) amt = ((-d * 8) < pv) ? (pv - x) : pv;
        uint32_t evs = __ballot_sync(VMB_FULL, is_reset || is_gap);
        double corr = st.corr, my_corr = st.corr;
        while (evs) {
            int b = __ffs((int)evs) - 1;
            evs &= evs - 1;
            double a = shfl_f64(amt, b);
            int flags = __shfl_sync(VMB_FULL, (int)is_reset | ((int)is_gap << 1), b);
            if (flags & 1) corr = corr + a;
            if (flags & 2) corr = 0.0;
            if (lane >= b) my_corr = corr;
        }
        st.corr = corr;
        // element as a function of the previous output: Const(c) or MaxWith(m)
        double mval = is_gap ? x : x + my_corr;
        bool isc = is_gap || i == 0 || isnan(mval) || !valid;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            double am = shfl_up_f64(mval, off);
            int ac = __shfl_up_sync(VMB_FULL, (int)isc, off);
            if (lane >= off && !isc) {
                mval = (mval < am) ? am : mval;
                isc = ac != 0;
            }
        }
        outv = isc ? mval : ((mval < st.prev_out) ? st.prev_out : mval);
    }
    if (valid) v[i] = outv;
    st.prev_out = shfl_f64(outv, 31);
    st.prev_raw = shfl_f64(x, 31);
    if (max_stale > 0) st.prev_ts = (int64_t)shfl_u64((uint64_t)tt, 31);
}

// getScrapeInterval (rollup.go:871) from the k >= 1 intervals it looks at: their 0.6 quantile, `step` when that is not
// positive.  iv(x) is the x-th smallest of the intervals.
template <class IV>
__device__ __forceinline__ int64_t scrape_interval(int64_t step, uint32_t k, IV iv) {
    const double nn = (double)k;
    const double rank = 0.6 * (nn - 1);
    const double lower = fmax(0.0, floor(rank));
    const double upper = fmin(nn - 1, lower + 1);
    const double weight = rank - floor(rank);
    const double q = __dadd_rn(__dmul_rn(iv((int)lower), 1 - weight), __dmul_rn(iv((int)upper), weight));
    const int64_t sq = (int64_t)q;
    return sq > 0 ? sq : step;
}

// maxPrevInterval and the effective window of a series whose scrape interval is si: getMaxPrevInterval (rollup.go:899), the
// lookback / min-staleness clamps and the default-window rules (rollup.go:719-756).  A query of one point ignores si.
struct PrevWindow {
    int64_t max_prev, window;
};
__device__ __forceinline__ PrevWindow prev_interval_window(const vmb_rollup_cfg& rc, int64_t si) {
    int64_t maxPrev = rc.step;
    if (rc.start < rc.end) {
        if (si <= 2 * 1000) maxPrev = si + 4 * si;
        else if (si <= 4 * 1000) maxPrev = si + 2 * si;
        else if (si <= 8 * 1000) maxPrev = si + si;
        else if (si <= 16 * 1000) maxPrev = si + si / 2;
        else if (si <= 32 * 1000) maxPrev = si + si / 4;
        else maxPrev = si + si / 8;
    }
    if (rc.lookback_delta > 0 && maxPrev > rc.lookback_delta) maxPrev = rc.lookback_delta;
    if (rc.min_staleness_ms > 0 && maxPrev < rc.min_staleness_ms) maxPrev = rc.min_staleness_ms;
    int64_t window = rc.window;
    if (window <= 0) {
        window = rc.step;
        if ((rc.flags & VMB_RC_MAY_ADJUST_WINDOW) && window < maxPrev) window = maxPrev;
        if ((rc.flags & VMB_RC_IS_DEFAULT_ROLLUP) && rc.lookback_delta > 0 && window > rc.lookback_delta) window = rc.lookback_delta;
    }
    return PrevWindow{maxPrev, window};
}

// one warp per series
__global__ void __launch_bounds__(128) k_series_prepare(RollupParams P) {
    const int lane = lane_id();
    const uint32_t warps_per_grid = gridDim.x * (blockDim.x >> 5);
    const vmb_rollup_cfg& rc = P.cfg;
    for (uint32_t s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < P.nseries; s += warps_per_grid) {
        SeriesMeta m = P.meta[s];
        double* v = P.vals + m.start;
        int64_t* t = P.ts + m.start;
        uint32_t n = m.n;
        // ---- dropStaleNaNs eval.go:1985
        if ((rc.flags & VMB_RC_DROP_STALE_NANS) && n && (m.flags & VMB_SER_STALE)) {  // decoded batches know whether a marker exists
            bool has = false;
            for (uint32_t i = lane; i < n; i += 32) has |= is_stale_nan(v[i]);
            if (__any_sync(VMB_FULL, has)) {
                uint32_t o = 0;
                for (uint32_t base = 0; base < n; base += 32) {
                    uint32_t i = base + lane;
                    double x = i < n ? v[i] : 0.0;
                    int64_t tt = i < n ? t[i] : 0;
                    bool keep = i < n && !is_stale_nan(x);
                    uint32_t bal = __ballot_sync(VMB_FULL, keep);
                    if (keep) {
                        uint32_t r = o + __popc(bal & ((1u << lane) - 1u));
                        v[r] = x;
                        t[r] = tt;
                    }
                    o += __popc(bal);
                    __syncwarp();
                }
                if (o != n) {  // rows were removed: no arithmetic progression, no known first drop
                    m.flags &= ~VMB_SER_TS_AP;
                    m.set_first_drop(0);
                }
                n = o;
            }
        }
        // ---- removeCounterResets rollup.go:921 (sequential float semantics preserved: corrections are accumulated in
        //      sample order; the final clamp is a segmented prefix "max" which is order-independent)
        // A series whose values never decrease (and hold no NaN) comes out of removeCounterResets unchanged -- the
        // staleness-gap rule only ever zeroes the correction, and without a value drop there is none -- so the pass over its
        // rows is skipped (decoded columns never hold -0.0, so "+ 0.0" is void).  For the same reason the rows before the
        // first value drop of a series are not touched: the pass starts at the 128-row group that holds it, in the state the
        // sequential loop has there (no correction yet, outputs == inputs).
        const int64_t max_stale = rc.lookback_delta != 0 ? rc.lookback_delta + rc.window : 0;  // rollup.go:380-387
        if ((rc.flags & VMB_RC_REMOVE_COUNTER_RESETS) && n && (m.flags & VMB_SER_DROP)) {
            RcrState st;
            st.corr = 0.0; st.prev_raw = 0.0; st.prev_out = 0.0; st.prev_ts = 0;
            const uint32_t r0 = m.first_drop();
            const uint32_t base0 = r0 >= n ? 0u : (r0 & ~127u);
            if (base0) {
                st.prev_raw = st.prev_out = v[base0 - 1];
                st.prev_ts = max_stale > 0 ? t[base0 - 1] : 0;
            }
            // four 32-row chunks per iteration: their loads are issued together (one HBM round trip per 128 rows)
            for (uint32_t base = base0; base < n; base += 128) {
                double x[4];
                int64_t tt[4];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    uint32_t i = base + 32u * u + lane;
                    x[u] = i < n ? v[i] : 0.0;
                    tt[u] = (max_stale > 0 && i < n) ? t[i] : 0;
                }
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    uint32_t cb = base + 32u * u;
                    if (cb < n) rcr_chunk(st, v, cb, n, x[u], tt[u], max_stale, lane);
                }
            }
        }
        // ---- value preFuncs of the multi-output rollups (rollup.go:440-476), in place.  Output i needs inputs i and i+1:
        //      chunks run in ascending order, every lane reads before the chunk writes.
        if ((rc.flags & VMB_RC_PRE_MASK) && n) {
            __syncwarp();
            if (rc.flags & VMB_RC_PRE_DERIV_VALUES) {
                bool dup = false;  // duplicate timestamps make the loop carry state (rollup.go:987): rare, replayed by lane 0
                for (uint32_t i = 1 + lane; i < n; i += 32) dup |= t[i] == t[i - 1];
                if (__any_sync(VMB_FULL, dup)) {
                    if (lane == 0) {
                        double prevDeriv = 0.0, prevValue = v[0];
                        int64_t prevTs = t[0];
                        for (uint32_t i = 0; i + 1 < n; i++) {
                            const double x = v[i + 1];
                            const int64_t ts = t[i + 1];
                            if (ts == prevTs) {
                                v[i] = prevDeriv;
                                continue;
                            }
                            prevDeriv = (x - prevValue) / ((double)(ts - prevTs) / 1e3);
                            v[i] = prevDeriv;
                            prevValue = x;
                            prevTs = ts;
                        }
                        v[n - 1] = prevDeriv;
                    }
                } else {
                    double last = 0.0;
                    for (uint32_t base = 0; base + 1 < n; base += 32) {
                        const uint32_t i = base + lane;
                        double o = 0.0;
                        const bool act = i + 1 < n;
                        if (act) o = (v[i + 1] - v[i]) / ((double)(t[i + 1] - t[i]) / 1e3);
                        __syncwarp();
                        if (act) v[i] = o;
                        if (i + 2 == n) last = o;
                    }
                    last = __shfl_sync(VMB_FULL, last, (int)((n - 2) & 31u));
                    __syncwarp();
                    if (lane == 0) v[n - 1] = n > 1 ? last : 0.0;  // prevDeriv (0 for a single sample)
                }
            } else if (rc.flags & VMB_RC_PRE_DELTA_VALUES) {
                double last = 0.0;
                for (uint32_t base = 0; base + 1 < n; base += 32) {
                    const uint32_t i = base + lane;
                    double o = 0.0;
                    const bool act = i + 1 < n;
                    if (act) o = v[i + 1] - v[i];
                    __syncwarp();
                    if (act) v[i] = o;
                    if (i + 2 == n) last = o;
                }
                last = __shfl_sync(VMB_FULL, last, (int)((n - 2) & 31u));
                __syncwarp();
                if (lane == 0) v[n - 1] = n > 1 ? last : 0.0;  // prevDelta (0 for a single sample)
            } else {  // VMB_RC_PRE_SCRAPE_INTERVAL: values[i] = ts[i]/1000 - ts[i-1]/1000, values[0] = values[1]
                for (uint32_t i = lane; i < n; i += 32) {
                    double o = D_NAN;
                    if (i > 0) o = (double)t[i] / 1000 - (double)t[i - 1] / 1000;
                    else if (n > 1) o = (double)t[1] / 1000 - (double)t[0] / 1000;
                    v[i] = o;
                }
            }
            __syncwarp();
        }
        // ---- maxPrevInterval / window  rollup.go:719-756
        if (lane == 0) {
            int64_t si = rc.step;
            if (rc.start < rc.end && n >= 2) {  // (a query of one point does not look at the scrape interval)
                // getScrapeInterval rollup.go:871: the last <= 20 intervals, sorted
                double iv[20];
                uint32_t m2 = n - 1;
                uint32_t from = m2 > 20 ? m2 - 20 : 0;
                uint32_t k = 0;
                int64_t tsPrev = t[n - 1];
                for (int i = (int)m2 - 1; i >= (int)from; i--) {
                    iv[k++] = (double)(tsPrev - t[i]);
                    tsPrev = t[i];
                }
                for (uint32_t a = 1; a < k; a++) {  // insertion sort
                    double x = iv[a];
                    int b = (int)a - 1;
                    while (b >= 0 && iv[b] > x) {
                        iv[b + 1] = iv[b];
                        b--;
                    }
                    iv[b + 1] = x;
                }
                si = scrape_interval(rc.step, k, [&](int x) { return iv[x]; });
            }
            const PrevWindow pw = prev_interval_window(rc, si);
            m.n = n;
            m.max_prev_interval = pw.max_prev;
            m.window = pw.window;
            P.meta[s] = m;
        }
        __syncwarp();
    }
}

// the window of point p, rows [i, j) of a series of n time-sorted rows t (rollup.go:769-777): i = the first row after
// tEnd - window, j = the first row after tEnd, never below i.  k_rollup's edges of a window it reads from global memory, and
// the windows of vmb_rollup_count_values.
struct WinEdges {
    uint32_t i, j;
};
__device__ __forceinline__ WinEdges window_edges(const vmb_rollup_cfg& rc, const SeriesMeta& m, const int64_t* t, uint32_t n, uint32_t p) {
    const int64_t tEnd = rc.start + (int64_t)p * rc.step;
    const uint32_t i = upper_bound_ts(t, n, tEnd - m.window), j = upper_bound_ts(t, n, tEnd);
    return WinEdges{i, j < i ? i : j};
}

#define ROLLUP_THREADS 256
#define ROLLUP_CAP 2048    /* rows of one series resident in shared memory */
#define ROLLUP_SEEKS 2560  /* window edges of one fill: up to ROLLUP_CAP points + window/step shared left edges */

// first index with ts[idx] > x: interpolation guess + short walk, binary search when the walk does not converge.
// The guess is computed in fp32 from 32-bit offsets when the resident rows span < 2^31 ms (inv_dt > 0 signals that):
// a guess only has to land near the answer, the walk makes it exact.
__device__ __forceinline__ uint32_t seek_after(const int64_t* __restrict__ ts, uint32_t n, int64_t x, float inv_dt) {
    if (n == 0) return 0;
    const int64_t t0 = ts[0];
    if (t0 > x) return 0;
    if (ts[n - 1] <= x) return n;
    uint32_t g;
    if (inv_dt > 0.0f) g = (uint32_t)(__uint2float_rn((uint32_t)(x - t0)) * inv_dt);
    else g = n >> 1;
    if (g >= n) g = n - 1;
    if (ts[g] <= x) {
        uint32_t lim = g + 6 < n ? g + 6 : n;
        do { g++; } while (g < lim && ts[g] <= x);
        if (g < n && ts[g] <= x) g += upper_bound_ts(ts + g, n - g, x);
        return g;
    }
    uint32_t lim = g > 6 ? g - 6 : 0;
    while (g > lim && ts[g - 1] > x) g--;
    if (g > 0 && ts[g - 1] > x) g = upper_bound_ts(ts, g, x);
    return g;
}

// seek_after over the resident rows with the first / last resident timestamps already in registers and the common case
// (regular scrape interval: the guess is the answer or one off) decided from three independent loads.
__device__ __forceinline__ uint32_t seek_resident(const int64_t* __restrict__ ts, uint32_t n, int64_t x, float inv_dt,
                                                  int64_t t_first, int64_t t_last) {
    if (n == 0 || t_first > x) return 0;
    if (t_last <= x) return n;
    if (inv_dt > 0.0f) {  // here n >= 2 and t_first <= x < t_last
        uint32_t g = (uint32_t)(__uint2float_rn((uint32_t)(x - t_first)) * inv_dt) + 1u;
        if (g > n - 1) g = n - 1;
        const uint32_t g2 = g + 1 < n ? g + 1 : g;
        const int64_t a = ts[g - 1], b = ts[g], c = ts[g2];
        if (a <= x) {
            if (x < b) return g;
            if (x < c) return g2;
        }
    }
    return seek_after(ts, n, x, inv_dt);
}

// (double)dt_ms / 1e3 exactly as IEEE division would round it: q = RN(x * RN(1/1000)), rem = x - q * 1000 (exact, FMA),
// RN(q + rem * RN(1/1000)) -- Markstein's division step, valid for every finite x here (1000 is exact, no under/overflow
// for |x| < 2^64).  Same trick as decimal->float in decode.cu; 3 flops instead of a ~25-instruction division sequence.
__device__ __forceinline__ double ms_to_s(int64_t dt_ms) {
    const double x = (double)dt_ms;
    const double r = 1e-3;  // RN(1/1000)
    double q = __dmul_rn(x, r);
    double rem = __fma_rn(-q, 1e3, x);
    return __fma_rn(rem, r, q);
}

// one output point, rollup.go:769-819: the rollupFuncArg of point p from its window edges i, j (absolute rows of a series of
// n rows), and the function applied to it.  v / t reach the rows from `off` on (v[k], t[k] = row off + k); rows [i-1, j] must
// be reachable.
template <int F, class VP, class TP>
__device__ __forceinline__ double window_point(const vmb_rollup_cfg& rc, VP v, TP t, uint32_t off, uint32_t n, uint32_t i, uint32_t j,
                                               uint32_t p, int64_t window, int64_t max_prev, unsigned long long& scanned) {
    const int64_t tEnd = rc.start + (int64_t)p * rc.step;
    const int64_t tStart = tEnd - window;
    if (j < i) j = i;
    WinT<VP, TP> r;
    r.values = v + (i - off);  // the window; [-1] is the row in front of it
    r.timestamps = t + (i - off);
    r.n = j - i;
    r.prevValue = D_NAN;
    r.prevTimestamp = tStart - max_prev;
    r.realPrevValue = D_NAN;
    if (i > 0) {
        const int64_t tp = r.timestamps[-1];
        const double vp = r.values[-1];
        if (i < n && tp > r.prevTimestamp) {
            r.prevValue = vp;
            r.prevTimestamp = tp;
        }
        const int64_t curr = r.n > 0 ? r.timestamps[0] : tStart;
        if (rc.lookback_delta == 0 || (curr - tp) < rc.lookback_delta) r.realPrevValue = vp;
    }
    r.realNextValue = j < n ? r.values[r.n] : D_NAN;
    r.currTimestamp = tEnd;
    r.idx = p;
    r.window = window;
    r.args = rc.args;
    r.args2 = rc.args2;
    scanned += rc.samples_scanned_per_call > 0 ? (unsigned long long)rc.samples_scanned_per_call : (unsigned long long)r.n;
    return call_func(F >= 0 ? F : rc.func_id, r);
}

// rollupDerivFast (rollup.go:1954) of one point from its window edges i <= j (absolute rows of a series of n rows) with selects
// instead of branches, up to the division, which each caller does its own way: result(x / (dt / 1e3)).  v / t reach the rows
// [off, off + cnt) (v[k], t[k] = row off + k), rows [i-1, j) among them; tsp = tStart - maxPrevInterval on the scale of t.
template <class T>
struct RateEdges {
    double x;  // numerator: the last value of the window - the previous sample's value (or the window's first)
    T dt;      // divisor in ms (1000 where the quotient is not used)
    bool prev_ok, fixed;
    __device__ __forceinline__ double result(double q) const { return fixed ? (prev_ok ? 0.0 : D_NAN) : q; }
};
template <class VP, class TP, class T>
__device__ __forceinline__ RateEdges<T> rate_edges(VP v, TP t, uint32_t off, uint32_t n, uint32_t cnt, uint32_t i, uint32_t j, T tsp) {
    const uint32_t ri = i - off, rj = j - off, nw = j - i;
    const bool have_prev = i > 0 && i < n;
    const uint32_t ip = have_prev ? ri - 1 : 0u;
    const uint32_t il = rj ? rj - 1 : 0u;
    const uint32_t i0 = ri < cnt ? ri : il;  // (ri == cnt only for an empty window, whose first row is not used)
    const T tp = t[ip], t0 = t[i0], tl = t[il];
    const double vp = v[ip], v0 = v[i0], vl = v[il];
    RateEdges<T> e;
    e.prev_ok = have_prev && tp > tsp && !isnan(vp);
    e.fixed = e.prev_ok ? nw == 0 : nw < 2;  // no division: 0 with a previous sample, NaN without
    e.x = vl - (e.prev_ok ? vp : v0);
    e.dt = e.fixed ? (T)1000 : tl - (e.prev_ok ? tp : t0);
    return e;
}

// timestamps relative to the first row of a series whose row r sits at r * dt: element k is row base + k
struct RowTs32 {
    uint32_t base;
    int32_t dt;
    __device__ __forceinline__ int32_t operator[](uint32_t k) const { return (int32_t)(base + k) * dt; }
};

// one output point of k_rollup: v / t hold the rows [off, off + cnt) of the series (shared-memory window, or the whole series
// with off == 0 and cnt == n); rows [i-1, j] must be resident
template <int F>
__device__ __forceinline__ double rollup_point(const vmb_rollup_cfg& rc, const SeriesMeta& m, const double* v, const int64_t* t,
                                               uint32_t off, uint32_t n, uint32_t cnt, uint32_t i, uint32_t j, uint32_t p,
                                               unsigned long long& scanned) {
    if (F == VMB_RF_RATE) {
        if (j < i) j = i;
        scanned += rc.samples_scanned_per_call > 0 ? (unsigned long long)rc.samples_scanned_per_call : (unsigned long long)(j - i);
        const RateEdges<int64_t> e =
            rate_edges(v, t, off, n, cnt, i, j, rc.start + (int64_t)p * rc.step - m.window - m.max_prev_interval);
        return e.result(e.x / ms_to_s(e.dt));
    }
    return window_point<F>(rc, v, t, off, n, i, j, p, m.window, m.max_prev_interval, scanned);
}

// rows with timestamp <= t_org + xr when row k sits at t_org + k * dt: exact floor division from a float estimate
__device__ __forceinline__ uint32_t seek_ap(int32_t xr, int32_t dt_row, float inv_row, uint32_t n) {
    if (xr < 0) return 0u;
    if (xr >= (int32_t)(n - 1) * dt_row) return n;  // at or past the last row (also keeps the quotient below 2^14: n <= 16384)
    uint32_t q = (uint32_t)(__int2float_rz(xr) * inv_row);
    int32_t r = xr - (int32_t)q * dt_row;
    if (r < 0) { q--; r += dt_row; }
    if (r >= dt_row) q++;
    return q + 1u < n ? q + 1u : n;
}

// shared memory of k_rollup at file scope: the device functions below index it directly (plain LDS with constant bases)
__shared__ int64_t rs_ts[ROLLUP_CAP];     // timestamps of the resident rows
__shared__ double rs_val[ROLLUP_CAP];     // their values
__shared__ int32_t rs_rt[ROLLUP_CAP];     // timestamps relative to the first row of the series (32-bit fast path)
__shared__ unsigned short rs_seek[ROLLUP_SEEKS];  // window edges of the fill as resident-row indices (<= ROLLUP_CAP)

// first resident row with timestamp > x, timestamps as 32-bit offsets: the interpolation guess is the answer or one off for
// regularly scraped series, decided from three independent loads; anything else falls back to seek_after
__device__ __forceinline__ uint32_t seek32(uint32_t n, int32_t xr, float inv_dt, int32_t r_first, int32_t r_last, int64_t t_org) {
    const int32_t off = xr > r_first ? xr - r_first : 0;
    uint32_t g = (uint32_t)(__int2float_rn(off) * inv_dt) + 1u;
    if (g > n - 1) g = n - 1;
    const uint32_t gm = g ? g - 1 : 0, g2 = g + 1 < n ? g + 1 : g;
    const int32_t a = rs_rt[gm], b = rs_rt[g], c = rs_rt[g2];
    uint32_t res = xr < b ? g : g2;
    const bool ok = a <= xr && (xr < b || xr < c);
    const bool inside = xr >= r_first && xr < r_last;
    if (inside && !ok) res = seek_after(rs_ts, n, t_org + xr, inv_dt);
    res = xr < r_first ? 0u : res;
    res = xr >= r_last ? n : res;
    return res;
}

// Streaming rollup: one CTA walks one series front to back.  Rows are pulled into shared memory once, in order, with
// coalesced loads (no per-tile searches in global memory); the CTA computes every output point whose window lies inside the
// resident rows (threads stride over the points of the fill), then slides the resident range forward keeping only
// the rows the next point still needs.  Both the samples and the output grid are time-ordered, so this visits each row once.
//
// Window seeks: when the window is a multiple of the step (rate(m[5m]) at step 15 s: 20 steps), the left edge of point p is
// the right edge of point p - window/step, so a fill computes ONE seek per grid time (s_seek[]) instead of two per point.
//
// A window that does not fit ROLLUP_CAP rows (huge windows / very dense series) is handled for that tile by reading global
// memory directly.  F >= 0 instantiates the kernel for one rollup function (the switch in call_func folds away).
template <int F>
__global__ void __launch_bounds__(ROLLUP_THREADS, 4) k_rollup(RollupParams P) {
    const vmb_rollup_cfg& rc = P.cfg;
    const uint32_t tid = threadIdx.x;
    unsigned long long scanned = 0;
    for (uint32_t s = blockIdx.x; s < P.nseries; s += gridDim.x) {
        const SeriesMeta m = P.meta[s];
        const double* vg = P.vals + m.start;
        const int64_t* tg = P.ts + m.start;
        const uint32_t n = m.n;
        double* out = P.out + (size_t)(P.out_rows ? P.out_rows[s] : s) * P.npoints;
        if (tid == 0) scanned += n;  // samplesScanned starts at len(values) rollup.go:766
        // window / step and window % step: 32-bit arithmetic when both fit (a 64-bit division is ~100 instructions and every
        // thread of the CTA computes this)
        uint32_t wsteps;
        bool window_is_steps;
        if ((uint64_t)m.window < (1ull << 31) && (uint64_t)rc.step < (1ull << 31)) {
            const uint32_t w32 = (uint32_t)m.window, s32 = (uint32_t)rc.step;
            wsteps = w32 / s32;
            window_is_steps = wsteps * s32 == w32;
        } else {
            wsteps = (uint32_t)(m.window / rc.step);
            window_is_steps = (m.window % rc.step) == 0;
        }
        const bool shared_seeks = window_is_steps && wsteps <= ROLLUP_SEEKS - ROLLUP_CAP;
        const uint32_t wsteps_cap = shared_seeks ? wsteps : 0u;
        // 32-bit fast path (rate): timestamps relative to the first row of the series, when everything fits 2^30 ms
        const int64_t t_org = n ? tg[0] : 0;
        bool fast = false;
        int32_t start_r = 0, step32 = 0, win32 = 0, mpi32 = 0;
        if (F == VMB_RF_RATE && shared_seeks && n) {
            const int64_t lim = (int64_t)1 << 30;
            const int64_t a0 = rc.start - (int64_t)wsteps * rc.step - t_org, a1 = rc.end - t_org;
            fast = (tg[n - 1] - t_org) < lim && a0 > -lim && a0 < lim && a1 > -lim && a1 < lim && m.window < lim &&
                   m.max_prev_interval < lim && rc.step < lim && rc.samples_scanned_per_call < 4096;
            start_r = (int32_t)(rc.start - t_org);
            step32 = (int32_t)rc.step;
            win32 = (int32_t)m.window;
            mpi32 = (int32_t)m.max_prev_interval;
        }
        // arithmetic-progression mode: no timestamp is read at all (rows sit at t_org + row * dt_row)
        int32_t dt_row = 0;
        float inv_row = 0.0f;
        bool ap = false;
        if (fast && (m.flags & VMB_SER_TS_AP) && n >= 2) {
            const int64_t d = tg[1] - tg[0];
            if (d > 0 && d < ((int64_t)1 << 30) && (int64_t)(n - 1) * d < ((int64_t)1 << 30)) {
                ap = true;
                dt_row = (int32_t)d;
                inv_row = 1.0f / (float)dt_row;
            }
        }
        uint32_t base = 0, cnt = 0, p = 0;
        while (p < P.npoints) {
            // ---- fill: rows [base + cnt, min(n, base + CAP))
            __syncthreads();
            const uint32_t want = min(n - base, (uint32_t)ROLLUP_CAP);
            if (ap) {
                for (uint32_t k = cnt + tid; k < want; k += ROLLUP_THREADS) rs_val[k] = vg[base + k];
            } else {
                for (uint32_t k = cnt + tid; k < want; k += ROLLUP_THREADS) {
                    const int64_t t = tg[base + k];
                    rs_ts[k] = t;
                    rs_val[k] = vg[base + k];
                    if (fast) rs_rt[k] = (int32_t)(t - t_org);
                }
            }
            cnt = want;
            __syncthreads();
            // ---- points computable from the resident rows: tEnd < last resident timestamp (so that row j is resident),
            //      or every remaining point once the series end is resident
            uint32_t p_end;
            if (base + cnt == n) p_end = P.npoints;
            else {
                int64_t tl = (ap ? t_org + (int64_t)(base + cnt - 1) * dt_row : rs_ts[cnt - 1]) - 1 - rc.start;
                if (tl < 0) p_end = 0u;
                else if (fast) p_end = min(P.npoints, (uint32_t)tl / (uint32_t)step32 + 1u);  // tl < 2^31 here
                else p_end = (uint32_t)min((int64_t)P.npoints, tl / rc.step + 1);
            }
            float inv_dt = 0.0f;  // rows per millisecond over the resident range (0: no usable slope => bisect)
            {
                const int64_t span = (cnt > 1 && !ap) ? rs_ts[cnt - 1] - rs_ts[0] : 0;
                if (span > 0 && span < (int64_t)0x7fffffff) inv_dt = __fdividef((float)(cnt - 1), (float)span);
            }
            if (p_end <= p) {
                // the window of point p needs more than CAP rows: do one tile from global memory
                p_end = min(p + ROLLUP_THREADS, P.npoints);
                uint32_t q = p + tid;
                if (q < p_end) {
                    const WinEdges w = window_edges(rc, m, tg, n, q);
                    out[q] = rollup_point<F>(rc, m, vg, tg, 0u, n, n, w.i, w.j, q, scanned);
                }
                p = p_end;
                if (p < P.npoints) {  // restart the resident range at the first row the next point needs
                    uint32_t lo = upper_bound_ts(tg, n, rc.start + (int64_t)p * rc.step - m.window);
                    base = lo > 0 ? lo - 1 : 0;
                    cnt = 0;
                }
                continue;
            }
            // ---- while this fill is being evaluated, pull the rows of the next one into L2: the next fill starts at most
            //      ROLLUP_CAP rows after the last resident row.  One 128-byte line per thread (first half of the CTA:
            //      timestamps, second half: values), so the next fill waits for L2 instead of HBM.
            {
                const uint32_t r = base + cnt + (tid & (ROLLUP_THREADS / 2 - 1)) * 16u;
                if (r < n && (!ap || tid >= ROLLUP_THREADS / 2)) {
                    const void* a = tid < ROLLUP_THREADS / 2 ? (const void*)(tg + r) : (const void*)(vg + r);
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(a));
                }
            }
            // ---- the points of this fill, in two passes without barriers inside: every window edge first (shared by the
            //      points when the window is a whole number of steps), then the points.  Iterations are independent, so
            //      the shared-memory latencies of several points of one thread overlap.
            if (p_end - p > ROLLUP_SEEKS - wsteps_cap) p_end = p + (ROLLUP_SEEKS - wsteps_cap);
            const uint32_t np = p_end - p;
            const int64_t t_first = (cnt && !ap) ? rs_ts[0] : 0, t_last = (cnt && !ap) ? rs_ts[cnt - 1] : 0;
            if (fast) {
                // branch-free 32-bit edges, then the rate() points.  Edges and timestamps come from the row arithmetic in
                // arithmetic-progression mode (edges clamped to the resident range), else from the resident rs_rt.
                const int32_t x0r = start_r + ((int32_t)p - (int32_t)wsteps) * step32;
                const int32_t ts0 = start_r + (int32_t)p * step32 - win32 - mpi32;  // tStart - maxPrevInterval of point p
                const uint32_t spc = (uint32_t)rc.samples_scanned_per_call;
                auto rate_fill = [&](auto seek, auto ts) {
#pragma unroll 2
                    for (uint32_t q = tid; q < np + wsteps; q += ROLLUP_THREADS) rs_seek[q] = (unsigned short)seek(x0r + (int32_t)q * step32);
                    __syncthreads();
                    uint32_t sc32 = 0;
#pragma unroll 2
                    for (uint32_t q = tid; q < np; q += ROLLUP_THREADS) {
                        const uint32_t i = base + rs_seek[q];
                        const uint32_t j = max(i, base + rs_seek[q + wsteps]);
                        sc32 += spc ? spc : j - i;
                        const RateEdges<int32_t> e = rate_edges(rs_val, ts, base, n, cnt, i, j, ts0 + (int32_t)q * step32);
                        out[p + q] = e.result(e.x / ms_to_s((int64_t)e.dt));
                    }
                    scanned += sc32;
                };
                if (ap) {
                    rate_fill([&](int32_t x) {
                        const uint32_t e = seek_ap(x, dt_row, inv_row, n);
                        return (e < base ? base : (e > base + cnt ? base + cnt : e)) - base;
                    }, RowTs32{base, dt_row});
                } else {
                    const int32_t r_first = rs_rt[0], r_last = rs_rt[cnt - 1];
                    rate_fill([&](int32_t x) { return seek32(cnt, x, inv_dt, r_first, r_last, t_org); }, (const int32_t*)rs_rt);
                }
            } else if (shared_seeks) {
                const int64_t x0 = rc.start + ((int64_t)p - (int64_t)wsteps) * rc.step;
#pragma unroll 2
                for (uint32_t q = tid; q < np + wsteps; q += ROLLUP_THREADS)
                    rs_seek[q] = (unsigned short)seek_resident(rs_ts, cnt, x0 + (int64_t)q * rc.step, inv_dt, t_first, t_last);
                __syncthreads();
#pragma unroll 2
                for (uint32_t q = tid; q < np; q += ROLLUP_THREADS)
                    out[p + q] = rollup_point<F>(rc, m, rs_val, rs_ts, base, n, cnt, base + rs_seek[q], base + rs_seek[q + wsteps], p + q, scanned);
            } else {
                for (uint32_t q = tid; q < np; q += ROLLUP_THREADS) {
                    const int64_t tEnd = rc.start + (int64_t)(p + q) * rc.step;
                    const uint32_t i = base + seek_resident(rs_ts, cnt, tEnd - m.window, inv_dt, t_first, t_last);
                    const uint32_t j = base + seek_resident(rs_ts, cnt, tEnd, inv_dt, t_first, t_last);
                    // rows before `base` are not resident: the slide rule below keeps row i-1 of the first point resident
                    out[p + q] = rollup_point<F>(rc, m, rs_val, rs_ts, base, n, cnt, i, j, p + q, scanned);
                }
            }
            p = p_end;
            if (p >= P.npoints) break;
            // ---- slide: keep rows from (first row after tStart(p)) - 1
            __syncthreads();
            uint32_t lo;
            if (ap) {
                lo = seek_ap((int32_t)(rc.start + (int64_t)p * rc.step - m.window - t_org), dt_row, inv_row, n);
                lo = lo < base ? base : (lo > base + cnt ? base + cnt : lo);
            } else {
                lo = base + seek_after(rs_ts, cnt, rc.start + (int64_t)p * rc.step - m.window, inv_dt);
            }
            uint32_t nb = lo > base ? lo - 1 : base;
            if (nb > base + cnt - 1) nb = base + cnt - 1;
            const uint32_t shift = nb - base;
            if (shift) {
                const uint32_t keep = cnt - shift;
                for (uint32_t c = 0; c < keep; c += ROLLUP_THREADS) {
                    uint32_t k = c + tid;
                    int64_t a = 0;
                    double b = 0.0;
                    int32_t c32 = 0;
                    if (k < keep) {
                        b = rs_val[k + shift];
                        if (!ap) {
                            a = rs_ts[k + shift];
                            if (fast) c32 = rs_rt[k + shift];
                        }
                    }
                    __syncthreads();
                    if (k < keep) {
                        rs_val[k] = b;
                        if (!ap) {
                            rs_ts[k] = a;
                            if (fast) rs_rt[k] = c32;
                        }
                    }
                }
                base = nb;
                cnt = keep;
            } else if (cnt == ROLLUP_CAP) {
                // no row can be dropped and the buffer is full: the next point's window does not fit; the global-memory
                // branch above will take it on the next iteration (p_end <= p)
            }
        }
    }
    // block reduce -> one atomic per CTA
    __syncthreads();
#pragma unroll
    for (int off = 16; off; off >>= 1) scanned += shfl_u64(scanned, (lane_id() ^ off));
    __shared__ unsigned long long s_part[ROLLUP_THREADS / 32];
    if (lane_id() == 0) s_part[threadIdx.x >> 5] = scanned;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long tot = 0;
        for (int w = 0; w < ROLLUP_THREADS / 32; w++) tot += s_part[w];
        if (tot) atomicAdd(P.scanned, tot);
    }
}

// ---- incremental aggregation (aggr_incremental.go). One thread per (group, point); the series of a group are folded
// in ascending series order, exactly like a single reference worker that receives them in that order.
struct AggrParams {
    const double* rolled;       // [nseries x P]
    const uint32_t* grp_start;  // [ngroups + 1]
    const uint32_t* grp_series; // series indices sorted by (group, series)
    double* values;             // [ngroups x P]
    double* counts;
    uint32_t ngroups, npoints;
    int aggr;
};

__global__ void k_aggr_fold(AggrParams A) {
    uint64_t idx = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (uint64_t)A.ngroups * A.npoints) return;
    uint32_t g = (uint32_t)(idx / A.npoints), p = (uint32_t)(idx % A.npoints);
    double dv = 0.0, dc = 0.0;
    bool any_done = false;
    for (uint32_t k = A.grp_start[g]; k < A.grp_start[g + 1]; k++) {
        double v = A.rolled[(size_t)A.grp_series[k] * A.npoints + p];
        switch (A.aggr) {
            case VMB_AGGR_SUM:
                if (isnan(v)) break;
                if (dc == 0) { dv = v; dc = 1; break; }
                dv += v;
                break;
            case VMB_AGGR_MIN:
                if (isnan(v)) break;
                if (dc == 0) { dv = v; dc = 1; break; }
                if (v < dv) dv = v;
                break;
            case VMB_AGGR_MAX:
                if (isnan(v)) break;
                if (dc == 0) { dv = v; dc = 1; break; }
                if (v > dv) dv = v;
                break;
            case VMB_AGGR_AVG:
                if (isnan(v)) break;
                if (dc == 0) { dv = v; dc = 1; break; }
                dv += v;
                dc += 1;
                break;
            case VMB_AGGR_COUNT:
            case VMB_AGGR_GROUP:
                if (isnan(v)) break;
                dv += 1;
                break;
            case VMB_AGGR_SUM2:
                if (isnan(v)) break;
                if (dc == 0) { dv = __dmul_rn(v, v); dc = 1; break; }
                dv = __dadd_rn(dv, __dmul_rn(v, v));
                break;
            case VMB_AGGR_GEOMEAN:
                if (isnan(v)) break;
                if (dc == 0) { dv = v; dc = 1; break; }
                dv *= v;
                dc += 1;
                break;
            case VMB_AGGR_ANY:  // first series of the group wins, NaNs included (aggr_incremental.go:517)
                if (!any_done) { dv = v; dc = 1; any_done = true; }
                break;
        }
    }
    A.values[idx] = dv;
    A.counts[idx] = dc;
}

__global__ void k_aggr_merge(int aggr, double* dv, double* dc, const double* sv, const double* sc, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double v = sv[i];
    switch (aggr) {
        case VMB_AGGR_COUNT:
        case VMB_AGGR_GROUP: dv[i] += v; break;
        case VMB_AGGR_SUM:
        case VMB_AGGR_SUM2:
            if (sc[i] == 0) break;
            if (dc[i] == 0) { dv[i] = v; dc[i] = 1; break; }
            dv[i] += v;
            break;
        case VMB_AGGR_MIN:
            if (sc[i] == 0) break;
            if (dc[i] == 0) { dv[i] = v; dc[i] = 1; break; }
            if (v < dv[i]) dv[i] = v;
            break;
        case VMB_AGGR_MAX:
            if (sc[i] == 0) break;
            if (dc[i] == 0) { dv[i] = v; dc[i] = 1; break; }
            if (v > dv[i]) dv[i] = v;
            break;
        case VMB_AGGR_AVG:
            if (sc[i] == 0) break;
            if (dc[i] == 0) { dv[i] = v; dc[i] = sc[i]; break; }
            dv[i] += v;
            dc[i] += sc[i];
            break;
        case VMB_AGGR_GEOMEAN:
            if (sc[i] == 0) break;
            if (dc[i] == 0) { dv[i] = v; dc[i] = sc[i]; break; }
            dv[i] *= v;
            dc[i] += sc[i];
            break;
        case VMB_AGGR_ANY:
            if (dc[i] > 0) break;
            dv[i] = v;
            dc[i] = sc[i];
            break;
    }
}

// puts the identity of the all-reduce operator into empty cells: 0 for sum-like, +-Inf for min/max, 1 for geomean
__global__ void k_aggr_prepare_allreduce(int aggr, double* dv, const double* dc, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (aggr == VMB_AGGR_COUNT || aggr == VMB_AGGR_GROUP) return;
    if (dc[i] != 0) return;
    double id = 0.0;
    if (aggr == VMB_AGGR_MIN) id = D_INF;
    else if (aggr == VMB_AGGR_MAX) id = -D_INF;
    else if (aggr == VMB_AGGR_GEOMEAN) id = 1.0;
    dv[i] = id;
}

__global__ void k_aggr_finalize(int aggr, double* dv, const double* dc, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    switch (aggr) {
        case VMB_AGGR_AVG:
            if (dc[i] == 0) dv[i] = D_NAN;
            else dv[i] /= dc[i];
            break;
        case VMB_AGGR_COUNT:
            if (dv[i] == 0) dv[i] = D_NAN;
            break;
        case VMB_AGGR_GROUP:
            dv[i] = dv[i] == 0 ? D_NAN : 1.0;
            break;
        case VMB_AGGR_GEOMEAN:
            if (dc[i] == 0) dv[i] = D_NAN;
            else dv[i] = pow(dv[i], 1 / dc[i]);
            break;
        default:
            if (dc[i] == 0) dv[i] = D_NAN;
            break;
    }
}

void launch_series_assemble(const RollupParams& P, cudaStream_t st) {
    if (!P.nseries) return;
    k_series_assemble<<<(P.nseries + 127) / 128, 128, 0, st>>>(P);
}
void launch_series_merge(const RollupParams& P, cudaStream_t st) {
    if (!P.nseries) return;
    uint32_t grid = (P.nseries + 3) / 4;
    if (grid > VMB_SMS * 16u) grid = VMB_SMS * 16u;
    k_series_merge<<<grid, 128, 0, st>>>(P);
}
void launch_series_dedup(const RollupParams& P, cudaStream_t st) {
    if (!P.nseries) return;
    uint32_t grid = (P.nseries + 3) / 4;
    if (grid > VMB_SMS * 16u) grid = VMB_SMS * 16u;
    k_series_dedup<<<grid, 128, 0, st>>>(P);
}
void launch_series_prepare(const RollupParams& P, cudaStream_t st) {
    if (!P.nseries) return;
    uint32_t grid = (P.nseries + 3) / 4;
    if (grid > VMB_SMS * 16u) grid = VMB_SMS * 16u;
    k_series_prepare<<<grid, 128, 0, st>>>(P);
}
void launch_rollup(const RollupParams& P, cudaStream_t st) {
    if (!P.nseries || !P.npoints) return;
    uint32_t grid = P.nseries > VMB_SMS * 16u ? VMB_SMS * 16u : P.nseries;  // one CTA per series, grid-stride
    switch (P.cfg.func_id) {  // the functions of BASELINE.json's configs get their own instantiation
#define ROLLUP_CASE(F) case F: k_rollup<F><<<grid, ROLLUP_THREADS, 0, st>>>(P); break;
        ROLLUP_CASE(VMB_RF_RATE)
        ROLLUP_CASE(VMB_RF_DELTA)
        ROLLUP_CASE(VMB_RF_AVG)
        ROLLUP_CASE(VMB_RF_MIN)
        ROLLUP_CASE(VMB_RF_MAX)
        ROLLUP_CASE(VMB_RF_SUM)
        ROLLUP_CASE(VMB_RF_COUNT)
        ROLLUP_CASE(VMB_RF_QUANTILE)
        ROLLUP_CASE(VMB_RF_DEFAULT_ROLLUP)
        ROLLUP_CASE(VMB_RF_IDERIV)
#undef ROLLUP_CASE
        default: k_rollup<-1><<<grid, ROLLUP_THREADS, 0, st>>>(P); break;
    }
}
