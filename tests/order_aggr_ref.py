"""numpy restatement of the order-statistic aggregates of app/vmselect/promql/aggr.go (aggrFuncExt :110, aggrPrepareSeries :121,
aggrFuncQuantiles :1162, aggrFuncMAD :942, aggrFuncMode :446, aggrFuncDistinct :423, aggrFuncOutliersIQR :952,
aggrFuncOutliersMAD :1004), the reference of vmb_aggr_order.

Cell by cell as the Go loops go: the group's non-NaN values at a point, sorted; the quantileSorted formula in float64; the
modeNoNaNs loop; a set for distinct (Python's float == and hash put -0.0 and +0.0 in one entry, as Go's map does); mad with a
real second sort of the deviations."""
import math

import numpy as np

NAN = float("nan")
FUNCS = ["quantiles", "mad", "mode", "distinct", "outliers_iqr", "outliers_mad"]
ROW_FUNCS = ["outliers_iqr", "outliers_mad"]


def quantile_sorted(phi, a):
    """aggr.go:922 quantileSorted: a sorted, without NaNs"""
    if len(a) == 0 or math.isnan(phi):
        return NAN
    if phi < 0:
        return -math.inf
    if phi > 1:
        return math.inf
    n = float(len(a))
    rank = phi * (n - 1)
    lower = max(0.0, math.floor(rank))
    upper = min(n - 1, lower + 1)
    weight = rank - math.floor(rank)
    with np.errstate(invalid="ignore", over="ignore"):
        return float(np.float64(a[int(lower)]) * (1 - weight) + np.float64(a[int(upper)]) * weight)


def quantile(phi, values):
    """aggr.go:870 quantile: the NaNs dropped, then sorted"""
    return quantile_sorted(phi, sorted(v for v in values if not math.isnan(v)))


def mode_no_nans(a):
    """aggr.go:541 modeNoNaNs(nan, a)"""
    if len(a) == 0:
        return NAN
    a = sorted(a)
    prev, j, dmax, mode = NAN, -1, 0, NAN
    for i, v in enumerate(a):
        if prev == v:
            continue
        d = i - j
        if d > dmax or math.isnan(mode):
            dmax, mode = d, prev
        j, prev = i, v
    if len(a) - j > dmax or math.isnan(mode):
        mode = prev
    return mode


def distinct(a):
    return float(len(set(a))) if a else NAN


def mad(values):
    """getPerPointMedians :1066 + getPerPointMADs :1088 for one cell -> (median, mad)"""
    med = quantile(0.5, values)
    with np.errstate(invalid="ignore", over="ignore"):
        dev = [float(abs(np.float64(v) - med)) for v in values if not math.isnan(v)]
    return med, quantile(0.5, dev)


def prepare(vals, group_ids, limit):
    """aggrPrepareSeries: rows without a value dropped, groups in order of their first non-empty row -> (order, members, kept)"""
    S, P = vals.shape
    g = np.zeros(S, dtype=np.int64) if group_ids is None else np.asarray(group_ids, dtype=np.int64)
    nonempty = ~np.all(np.isnan(vals), axis=1) if P else np.zeros(S, dtype=bool)
    order, members = [], {}
    for r in range(S):
        if nonempty[r]:
            if g[r] not in members:
                order.append(int(g[r]))
                members[g[r]] = []
            members[g[r]].append(r)
    return g, order, members, (order[:limit] if limit > 0 else order)


def aggr_order_ref(name, vals, group_ids=None, ngroups=1, phis=(0.5,), tolerance=1.0, limit=0):
    """-> (out, returned).  quantiles: out [len(phis) x ngroups x P]; mad / mode / distinct: [ngroups x P]; groups without a
    non-empty row are NaN; returned = the group ids in order of their first non-empty row, cut at `limit`.  outliers_*: out is
    None and returned the mask of the rows the reference returns."""
    vals = np.asarray(vals, dtype=np.float64)
    S, P = vals.shape
    g, order, members, kept = prepare(vals, group_ids, limit)
    if name in ROW_FUNCS:
        tol = np.broadcast_to(np.asarray(tolerance, dtype=np.float64), (P,))
        sel = np.zeros(S, dtype=bool)
        for gid in kept:
            rows = members[gid]
            for p in range(P):
                col = [float(vals[r, p]) for r in rows if not math.isnan(vals[r, p])]
                with np.errstate(invalid="ignore", over="ignore"):
                    if name == "outliers_iqr":  # getPerPointIQRBounds :977
                        a = sorted(col)
                        q25, q75 = quantile_sorted(0.25, a), quantile_sorted(0.75, a)
                        iqr = float(1.5 * (np.float64(q75) - q25))
                        lower, upper = float(np.float64(q25) - iqr), float(np.float64(q75) + iqr)
                        hit = [(vals[r, p] > upper or vals[r, p] < lower) for r in rows]
                    else:
                        med, m = mad(col)
                        bound = float(np.float64(m) * tol[p])
                        hit = [float(abs(np.float64(vals[r, p]) - med)) > bound for r in rows]
                for r, h in zip(rows, hit):
                    sel[r] |= bool(h)
        return None, sel
    phis = [float(x) for x in np.asarray(phis, dtype=np.float64).reshape(-1)]
    out = np.full((len(phis), ngroups, P) if name == "quantiles" else (ngroups, P), NAN)
    for gid in order:
        rows = members[gid]
        for p in range(P):
            col = [float(vals[r, p]) for r in rows if not math.isnan(vals[r, p])]
            if name == "quantiles":
                a = sorted(col)
                for k, phi in enumerate(phis):
                    out[k, gid, p] = quantile_sorted(phi, a)
            elif name == "mad":
                out[gid, p] = mad(col)[1]
            elif name == "mode":
                out[gid, p] = mode_no_nans(col)
            else:
                out[gid, p] = distinct(col)
    return out, np.array(kept, dtype=np.int64)
