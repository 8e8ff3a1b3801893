// The bucket of a sample in VictoriaMetrics' log-scale histogram (metrics.Histogram.Update,
// vendor/github.com/VictoriaMetrics/metrics/histogram.go:88), shared by histogram(q) (vmb_aggr_histogram) and histogram_over_time
// (vmb_rollup_histogram).  The bucket is decided by Go's math.Log10, so Go's log is restated here operation for operation:
// math.Log10(x) = math.Log(x) * (1/Ln10) (log10.go), math.Log the fdlibm e_log.c algorithm of log.go written as plain IEEE
// + - * /.  Every operation below is an explicitly rounded intrinsic, so no contraction into an FMA can change a bit whatever
// the build flags; the result is Go's whenever Go evaluates that same sequence without fusing (as the pure-Go log does on amd64).
// Whether the amd64 assembly archLog (log_amd64.s) matches the pure-Go sequence bit for bit is assumed, not verified: its
// reduction computes (f1 - 1) * 2 where log.go computes f1 * 2 - 1 (both exact), and its Frexp does not normalise subnormals
// (every subnormal falls in the lower bucket either way).
#pragma once
#include <stdint.h>

// histogram.go:12-16: e10Min = -9, e10Max = 18, bucketsPerDecimal = 18; 486 decimal buckets between 1e-9 and 1e18
#define VMH_DECIMAL 486u
#define VMH_NB 488u       // bucket numbers of the ABI: 0 the lower bucket "0...1.000e-09", 1 + idx a decimal bucket, 487 the upper
#define VMH_SKIP 0xffffu  // NaN and v < 0: counted nowhere

__device__ __forceinline__ double go_log(double x) {
    // log.go: Ln2Hi, Ln2Lo, L1..L7 (the hex encodings are checked by tests/test_vm_histogram_ref.py)
    const double Ln2Hi = 6.93147180369123816490e-01, Ln2Lo = 1.90821492927058770002e-10;
    const double L1 = 6.666666666666735130e-01, L2 = 3.999999999940941908e-01, L3 = 2.857142874366239149e-01,
                 L4 = 2.222219843214978396e-01, L5 = 1.818357216161805012e-01, L6 = 1.531383769920937332e-01,
                 L7 = 1.479819860511658591e-01;
    if (isnan(x) || x == __longlong_as_double(0x7ff0000000000000ll)) return x;
    if (x < 0) return __longlong_as_double(0x7ff8000000000001ll);  // math.NaN()
    if (x == 0) return __longlong_as_double((long long)0xfff0000000000000ull);
    // Frexp (frexp.go): subnormals are scaled by 2^52 first; f1 in [0.5, 1)
    int ki = 0;
    uint64_t b = (uint64_t)__double_as_longlong(x);
    if ((b >> 52) == 0) {
        b = (uint64_t)__double_as_longlong(__dmul_rn(x, 4503599627370496.0));
        ki = -52;
    }
    ki += (int)((b >> 52) & 0x7ff) - 1022;
    double f1 = __longlong_as_double((long long)((b & ~(0x7ffull << 52)) | (1022ull << 52)));
    if (f1 < 0.70710678118654752440) {  // Sqrt2/2, rounded once
        f1 = __dmul_rn(f1, 2.0);
        ki--;
    }
    const double f = __dsub_rn(f1, 1.0), k = (double)ki;
    const double s = __ddiv_rn(f, __dadd_rn(2.0, f)), s2 = __dmul_rn(s, s), s4 = __dmul_rn(s2, s2);
    const double t1 = __dmul_rn(s2, __dadd_rn(L1, __dmul_rn(s4, __dadd_rn(L3, __dmul_rn(s4, __dadd_rn(L5, __dmul_rn(s4, L7)))))));
    const double t2 = __dmul_rn(s4, __dadd_rn(L2, __dmul_rn(s4, __dadd_rn(L4, __dmul_rn(s4, L6)))));
    const double R = __dadd_rn(t1, t2), hfsq = __dmul_rn(__dmul_rn(0.5, f), f);
    // k*Ln2Hi - ((hfsq - (s*(hfsq+R) + k*Ln2Lo)) - f)
    return __dsub_rn(__dmul_rn(k, Ln2Hi),
                     __dsub_rn(__dsub_rn(hfsq, __dadd_rn(__dmul_rn(s, __dadd_rn(hfsq, R)), __dmul_rn(k, Ln2Lo))), f));
}

// Update: bucketIdx := (Log10(v) - e10Min) * bucketsPerDecimal; < 0 lower, >= 486 upper, else uint(bucketIdx), one lower when
// bucketIdx is a whole number > 0 (a power of ten ends its bucket, as an `le` bound).  -> VMH_SKIP or a bucket number < VMH_NB.
__device__ __forceinline__ uint32_t vmh_bucket(double v) {
    if (isnan(v) || v < 0) return VMH_SKIP;
    const double l10 = __dmul_rn(go_log(v), __longlong_as_double(0x3FDBCB7B1526E50Ell));  // 1/Ln10, Go's constant rounded once
    const double bi = __dmul_rn(__dadd_rn(l10, 9.0), 18.0);
    if (bi < 0) return 0;
    if (bi >= (double)VMH_DECIMAL) return VMH_NB - 1;
    uint32_t idx = (uint32_t)bi;
    if (bi == (double)idx && idx > 0) idx--;
    return 1 + idx;
}
