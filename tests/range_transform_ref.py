"""numpy restatement of the whole-series transforms of app/vmselect/promql/transform.go, the reference of vmb_transform_range
and of vmb_transform's smooth_exponential.

Row by row as the Go loops go: Welford (rollup.go:1808) and mean() (transform.go:1425) in Python floats (IEEE doubles, no FMA),
the linearRegression sums in Go's evaluation order, and for the order statistics a real sort of the non-NaN values with the
quantileSorted formula of order_aggr_ref.  Elementwise rewrites that have no order (comparisons, one subtraction and one
division per cell) use numpy arrays, so that long rows stay affordable."""
import math

import numpy as np

from order_aggr_ref import quantile, quantile_sorted

NAN, INF = float("nan"), float("inf")
FUNCS = ["range_stddev", "range_stdvar", "range_zscore", "range_trim_zscore", "range_normalize", "range_linear_regression",
         "range_quantile", "range_mad", "range_trim_outliers", "range_trim_spikes"]
ONE_ARG = ["range_trim_zscore", "range_quantile", "range_trim_outliers", "range_trim_spikes"]


def div(a, b):
    """Go's float64 a / b (Python raises on a zero divisor)"""
    with np.errstate(all="ignore"):
        return float(np.float64(a) / np.float64(b))


def stdvar(values):
    """rollup.go:1808: the len(values) == 1 fast path counts NaNs"""
    if len(values) == 0:
        return NAN
    if len(values) == 1:
        return 0.0
    avg = count = q = 0.0
    for v in values:
        if math.isnan(v):
            continue
        count += 1
        avg_new = avg + div(v - avg, count)
        q += (v - avg) * (v - avg_new)
        avg = avg_new
    if count == 0:
        return NAN
    return div(q, count)


def stddev(values):
    """rollup.go:1803"""
    return float(np.sqrt(np.float64(stdvar(values))))


def mean(values):
    """transform.go:1425: a plain sum over n, 0/0 when there is no value"""
    s, n = 0.0, 0
    for v in values:
        if not math.isnan(v):
            s += v
            n += 1
    return div(s, float(n))


def mad(values):
    """rollup.go:1476: the median, then the median of |v - median| (quantile drops the NaNs)"""
    median = quantile(0.5, values)
    with np.errstate(all="ignore"):
        ds = np.abs(np.asarray(values, dtype=np.float64) - median)
    return quantile(0.5, ds.tolist())


def are_const_values(values):
    """rollup.go:1137 on the raw row: NaN != NaN"""
    return len(values) <= 1 or all(values[i] == values[i - 1] for i in range(1, len(values)))


def linear_regression(values, timestamps, intercept):
    """rollup.go:1099"""
    if len(values) == 0:
        return NAN, NAN
    if are_const_values(values):
        return values[0], 0.0
    v_sum = t_sum = tv_sum = tt_sum = 0.0
    n = 0
    for v, t in zip(values, timestamps):
        if math.isnan(v):
            continue
        dt = float(t - intercept) / 1e3
        v_sum += v
        t_sum += dt
        tv_sum += dt * v
        tt_sum += dt * dt
        n += 1
    if n == 0:
        return NAN, NAN
    k = 0.0
    t_diff = tt_sum - div(t_sum * t_sum, float(n))
    if abs(t_diff) >= 1e-6:
        k = div(tv_sum - div(t_sum * v_sum, float(n)), t_diff)
    return div(v_sum, float(n)) - div(k * t_sum, float(n)), k


def set_last_values(row):
    """transform.go:1650"""
    idx = np.flatnonzero(~np.isnan(row))
    if len(idx):
        row[:] = row[idx[-1]]


def range_row(name, row, arg=None, timestamps=None):
    """one series through transform.go's function `name` -> (new row, kept); kept is False only where range_normalize drops
    the series (the row is then returned as it was).  arg: getScalar(...)[0] of the scalar argument; timestamps: the series'
    int64 timestamps (range_linear_regression)."""
    vals = [float(v) for v in row]
    out = np.array(row, dtype=np.float64)
    with np.errstate(all="ignore"):
        if name in ("range_stddev", "range_stdvar"):  # :1550, :1566
            out[:] = stddev(vals) if name == "range_stddev" else stdvar(vals)
        elif name == "range_zscore":  # :1408
            sd, avg = stddev(vals), mean(vals)
            out = (out - avg) / sd
        elif name == "range_trim_zscore":  # :1379
            z = abs(arg)
            sd, avg = stddev(vals), mean(vals)
            out[np.abs(out - avg) / sd > z] = NAN
        elif name == "range_normalize":  # :1347
            v_min, v_max = INF, -INF
            for v in vals:
                if math.isnan(v):
                    continue
                if v < v_min:
                    v_min = v
                if v > v_max:
                    v_max = v
            d = v_max - v_min
            if math.isinf(d):
                return out, False
            out = (out - v_min) / d
        elif name == "range_linear_regression":  # :1513
            ts = [int(t) for t in timestamps]
            v, k = linear_regression(vals, ts, ts[0])
            out = np.array([v + div(k * float(t - ts[0]), 1e3) for t in ts])
        elif name == "range_quantile":  # :1582
            nonnan = np.flatnonzero(~np.isnan(out))
            if len(nonnan):
                out[nonnan[-1]] = quantile_sorted(arg, sorted(out[nonnan].tolist()))
                set_last_values(out)
        elif name == "range_mad":  # :1534
            out[:] = mad(vals)
        elif name == "range_trim_outliers":  # :1437
            d_max = arg * mad(vals)
            median = quantile(0.5, vals)
            out[np.abs(out - median) > d_max] = NAN
        elif name == "range_trim_spikes":  # :1465
            phi = arg / 2
            a = np.sort(out[~np.isnan(out)]).tolist()
            v_max, v_min = quantile_sorted(1 - phi, a), quantile_sorted(phi, a)
            out[(out > v_max) | (out < v_min)] = NAN  # NaN points compare false and stay
        else:
            raise ValueError(name)
    return out, True


def range_transform_ref(name, matrix, arg=None, step=None, start=0):
    """every row of `matrix` through range_row -> (new matrix, kept mask); the series' timestamps are start + j*step"""
    m = np.asarray(matrix, dtype=np.float64)
    P = m.shape[1]
    ts = [start + j * step for j in range(P)] if step is not None else None
    out = np.empty_like(m)
    kept = np.ones(m.shape[0], dtype=bool)
    for r in range(m.shape[0]):
        out[r], kept[r] = range_row(name, m[r], arg, ts)
    return out, kept


def smooth_exponential_row(row, sfs):
    """transform.go:1664"""
    values = [float(v) for v in row]
    P = len(values)
    i0 = 0
    while i0 < P and math.isnan(values[i0]):  # skipLeadingNaNs
        i0 += 1
    for i in range(i0, P):  # then the leading +-Infs, unless nothing but +-Infs follows
        if not math.isinf(values[i]):
            i0 = i
            break
    if i0 >= P:
        return np.array(values)
    avg = values[i0]
    for j in range(i0 + 1, P):  # sfsX = sfs[len(ts.Values)-len(values):]: the absolute index
        v = values[j]
        if math.isnan(v):
            continue
        if math.isinf(v):
            values[j] = avg
            continue
        sf = float(sfs[j])
        if math.isnan(sf):
            sf = 1.0
        if sf < 0:
            sf = 0.0
        if sf > 1:
            sf = 1.0
        avg = avg * (1 - sf) + v * sf
        values[j] = avg
    return np.array(values)


def smooth_exponential_ref(matrix, sf):
    m = np.asarray(matrix, dtype=np.float64)
    sfs = np.broadcast_to(np.asarray(sf, dtype=np.float64), (m.shape[1],))
    return np.array([smooth_exponential_row(r, sfs) for r in m]).reshape(m.shape)
