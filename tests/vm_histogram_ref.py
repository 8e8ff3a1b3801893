"""Restatement of VictoriaMetrics' log-scale histogram (metrics.Histogram, vendor/github.com/VictoriaMetrics/metrics/histogram.go)
and of the two functions built on it, for the tests: histogram(q) by (...) (aggrFuncHistogram app/vmselect/promql/aggr.go:256)
and histogram_over_time(m[d]) (rollupHistogram rollup.go:1526 through rollupConfig.DoTimeseriesMap :693).

The bucket of a sample comes from Go's math.Log10(x) = math.Log(x) * (1/Ln10), and math.Log is the fdlibm e_log.c algorithm as
plain IEEE + - * / (math/log.go).  Python floats are IEEE doubles with round-to-nearest and no fused operations, so go_log below
performs exactly Go's operations and gives Go's bits.  Bucket numbers are the library's: 0 the lower bucket, 1 + idx a decimal
bucket, 487 the upper bucket; None for a skipped sample (NaN, v < 0)."""
import math
import struct
from fractions import Fraction

import numpy as np

import count_values_ref as CV
from vmrange_ref import vmrange_to_le_ref

# math/log.go, with the IEEE 754 encodings of the fdlibm source
CONSTS = dict(Ln2Hi=(6.93147180369123816490e-01, 0x3FE62E42FEE00000), Ln2Lo=(1.90821492927058770002e-10, 0x3DEA39EF35793C76),
              L1=(6.666666666666735130e-01, 0x3FE5555555555593), L2=(3.999999999940941908e-01, 0x3FD999999997FA04),
              L3=(2.857142874366239149e-01, 0x3FD2492494229359), L4=(2.222219843214978396e-01, 0x3FCC71C51D8E78AF),
              L5=(1.818357216161805012e-01, 0x3FC7466496CB03DE), L6=(1.531383769920937332e-01, 0x3FC39A09D078C69F),
              L7=(1.479819860511658591e-01, 0x3FC2F112DF3E5244))
Ln2Hi, Ln2Lo, L1, L2, L3, L4, L5, L6, L7 = (CONSTS[k][0] for k in ("Ln2Hi", "Ln2Lo", "L1", "L2", "L3", "L4", "L5", "L6", "L7"))
# math/const.go: Ln10 and Sqrt2 as Go's untyped constants; Go rounds 1/Ln10 and Sqrt2/2 once, to the nearest float64
LN10 = Fraction("2.30258509299404568401799145468436420760110148862877297603332790")
SQRT2 = Fraction("1.41421356237309504880168872420969807856967187537694807317667974")
INV_LN10 = float(1 / LN10)
HALF_SQRT2 = float(SQRT2 / 2)

E10_MIN, E10_MAX, PER_DECIMAL = -9, 18, 18
DECIMAL = (E10_MAX - E10_MIN) * PER_DECIMAL  # 486
NB = DECIMAL + 2


def bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def from_bits(u):
    return struct.unpack("<d", struct.pack("<Q", u))[0]


def go_log(x):
    """math.Log (log.go): special cases, Frexp (subnormals scaled by 2^52), the reduction and the polynomial"""
    if x != x or x == math.inf:
        return x
    if x < 0:
        return math.nan
    if x == 0:
        return -math.inf
    f1, ki = math.frexp(x)  # exact, f1 in [0.5, 1), as Go's Frexp
    if f1 < HALF_SQRT2:
        f1 *= 2
        ki -= 1
    f = f1 - 1
    k = float(ki)
    s = f / (2 + f)
    s2 = s * s
    s4 = s2 * s2
    t1 = s2 * (L1 + s4 * (L3 + s4 * (L5 + s4 * L7)))
    t2 = s4 * (L2 + s4 * (L4 + s4 * L6))
    R = t1 + t2
    hfsq = 0.5 * f * f
    return k * Ln2Hi - ((hfsq - (s * (hfsq + R) + k * Ln2Lo)) - f)


def go_log10(x):
    return go_log(x) * INV_LN10


def bucket(v, log10=go_log10):
    """Histogram.Update (histogram.go:88) -> bucket number or None"""
    if v != v or v < 0:
        return None
    bi = (log10(v) - E10_MIN) * PER_DECIMAL
    if bi < 0:
        return 0
    if bi >= DECIMAL:
        return NB - 1
    idx = int(bi)
    if bi == float(idx) and idx > 0:
        idx -= 1
    return 1 + idx


def bucket_np(v):
    """bucket() over a float64 array, the same IEEE operations elementwise (numpy rounds every operation, fuses none):
    -> int32 array, -1 for a skipped sample"""
    v = np.asarray(v, dtype=np.float64)
    with np.errstate(all="ignore"):
        skip = np.isnan(v) | (v < 0)
        x = np.where(skip | (v == 0) | np.isinf(v), 1.0, v)
        f1, ki = np.frexp(x)
        low = f1 < HALF_SQRT2
        f1 = np.where(low, f1 * 2, f1)
        k = (ki - low).astype(np.float64)
        f = f1 - 1
        s = f / (2 + f)
        s2 = s * s
        s4 = s2 * s2
        t1 = s2 * (L1 + s4 * (L3 + s4 * (L5 + s4 * L7)))
        t2 = s4 * (L2 + s4 * (L4 + s4 * L6))
        R = t1 + t2
        hfsq = 0.5 * f * f
        lg = k * Ln2Hi - ((hfsq - (s * (hfsq + R) + k * Ln2Lo)) - f)
        bi = (lg * INV_LN10 - E10_MIN) * PER_DECIMAL
        inner = (bi >= 0) & (bi < DECIMAL)
        idx = np.where(inner, bi, 0).astype(np.int64)
        idx = np.where(inner & (bi == idx) & (idx > 0), idx - 1, idx)
        b = np.where(bi < 0, 0, np.where(bi >= DECIMAL, NB - 1, 1 + idx))
    b = np.where(v == 0, 0, np.where(np.isposinf(v), NB - 1, b))
    return np.where(skip, -1, b).astype(np.int32)


def histogram_counts(vals, group_ids, ngroups):
    """histogram_vmrange by numpy: -> (matrix [n x P], groups, buckets) in the library's order"""
    vals = np.asarray(vals, dtype=np.float64)
    S, P = vals.shape
    b = bucket_np(vals)
    ok = b >= 0
    key = (np.asarray(group_ids, dtype=np.int64)[:, None] * NB + b)[ok]  # (group, bucket) of every counted cell
    rows, rid = np.unique(key, return_inverse=True)
    cell = rid.astype(np.int64) * P + np.broadcast_to(np.arange(P), (S, P))[ok]
    c = np.bincount(cell, minlength=rows.size * P).reshape(rows.size, P)
    return c.astype(np.float64), (rows // NB).tolist(), (rows % NB).tolist()


def vmrange_labels(multiplier=None):
    """initBucketRanges (histogram.go:220) and lowerBucketRange / upperBucketRange -> the label of every bucket number"""
    m = 10 ** (1 / PER_DECIMAL) if multiplier is None else multiplier
    v = 1e-9  # math.Pow10(-9)
    start = "%.3e" % v
    labels = ["0...%.3e" % v]
    for _ in range(DECIMAL):
        v *= m
        end = "%.3e" % v
        labels.append(start + "..." + end)
        start = end
    return labels + ["%.3e...+Inf" % 1e18]


LABELS = vmrange_labels()


def histogram_vmrange(vals, group_ids, ngroups):
    """aggrFuncHistogram before vmrangeBucketsToLE, per group: {bucket: counts[P]}, a row zero-filled when it is created"""
    vals = np.asarray(vals, dtype=np.float64)
    P = vals.shape[1]
    gid = np.asarray(group_ids)
    out = {}
    for g in range(ngroups):
        m = {}
        for row in np.flatnonzero(gid == g):
            for i, v in enumerate(vals[row].tolist()):
                b = bucket(v)
                if b is None:
                    continue
                if b not in m:
                    m[b] = np.zeros(P)
                m[b][i] += 1
        if m:
            out[g] = m
    return out


def histogram_rows(vals, group_ids, ngroups):
    """-> (matrix [n x P], groups, buckets) in the library's order: groups ascending, then buckets"""
    h = histogram_vmrange(vals, group_ids, ngroups)
    P = np.asarray(vals).shape[1]
    keys = [(g, b) for g in sorted(h) for b in sorted(h[g])]
    mat = np.array([h[g][b] for g, b in keys]).reshape(len(keys), P)
    return mat, [k[0] for k in keys], [k[1] for k in keys]


def histogram_le(vals, group_ids, ngroups):
    """histogram(q) by (...) with its vmrangeBucketsToLE: [(group, le, values)] in vmrange_to_le_ref's order"""
    mat, groups, buckets = histogram_rows(vals, group_ids, ngroups)
    rows = vmrange_to_le_ref(mat, [LABELS[b] for b in buckets], [None] * len(buckets), groups)
    return [(groups[src], le, v) for src, _, le, v in rows]


def histogram_over_time(values, timestamps, start, end, step, window, lookback_delta=0, drop_stale=True):
    """one series -> ({bucket: counts[P]}, samplesScanned): every point's window through Histogram.Update, a row per bucket met,
    NaN-initialised (a copy of the origin), the count written where it is not zero"""
    v = np.asarray(values, dtype=np.float64)
    t = np.asarray(timestamps, dtype=np.int64)
    if drop_stale:  # dropStaleNaNs eval.go:1985
        keep = np.array([not CV.is_stale(x) for x in v.tolist()], dtype=bool)
        v, t = v[keep], t[keep]
    lo, hi, scanned = CV.rollup_windows(v, t, start, end, step, window, lookback_delta)
    P = lo.size
    vl = v.tolist()
    m = {}
    for p in range(P):
        counts = {}
        for r in range(lo[p], max(lo[p], hi[p])):
            b = bucket(vl[r])
            if b is not None:
                counts[b] = counts.get(b, 0) + 1
        for b, c in counts.items():
            if b not in m:
                m[b] = np.full(P, np.nan)
            m[b][p] = c
    return m, scanned
