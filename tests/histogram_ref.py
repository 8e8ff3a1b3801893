"""numpy restatement of the histogram functions over `le` buckets of app/vmselect/promql/transform.go:634-1169, the reference of
vmb_histogram.

groupLeTimeseries (:1097) puts the rows of every group in row order, sort.Slice orders them by le with the insertion sort Go uses for
up to 12 elements (go_insertion_sort, taken for every group size as the library does), mergeSameLE (:1151) sums equal le into the
first in order, and fixBrokenBuckets (:1122) runs per point.  The Go closures loop over the buckets once per point; here the bucket
loop is vectorised over the points, so every cell sees the same float operations in the same order (numpy's float64 + - * / and
sqrt are IEEE).  fixBrokenBuckets runs at every point although Go skips it where a closure returns before it: no value read at such
a point depends on it."""
import math

import numpy as np

NAN, INF = float("nan"), float("inf")
SKIP = 0xFFFFFFFF  # a row without a parsable `le`
FUNCS = ["histogram_quantile", "histogram_quantiles", "histogram_share", "histogram_fraction", "histogram_avg", "histogram_stddev",
         "histogram_stdvar"]
NARGS = {"histogram_quantile": 1, "histogram_share": 1, "histogram_fraction": 2}  # histogram_quantiles: one per phi


def go_insertion_sort(les):
    """sort.Slice(xss, xss[i].le < xss[j].le) on up to 12 elements (insertionSortLessFunc) -> the new order of the indices.
    A NaN compares false both ways: nothing moves across it."""
    idx = list(range(len(les)))
    for i in range(1, len(idx)):
        j = i
        while j > 0 and les[idx[j]] < les[idx[j - 1]]:
            idx[j], idx[j - 1] = idx[j - 1], idx[j]
            j -= 1
    return idx


def le_groups(group_ids, les, ngroups):
    """groupLeTimeseries + the sort: the rows of every group in row order, then ordered by le -> [rows of group g]"""
    g = np.asarray(group_ids, dtype=np.int64)
    members = [[] for _ in range(ngroups)]
    for r in np.flatnonzero(g != SKIP).tolist():
        members[g[r]].append(r)
    return [[rows[k] for k in go_insertion_sort([float(les[r]) for r in rows])] for rows in members]


def merge_same_le(les, vals):
    """mergeSameLE :1151 on copies: consecutive rows whose le equals the first of their run are added to it in order"""
    out_le, out_v = [les[0]], [vals[0].copy()]
    for le, v in zip(les[1:], vals[1:]):
        if le != out_le[-1]:
            out_le.append(le)
            out_v.append(v.copy())
        else:
            out_v[-1] = out_v[-1] + v
    return out_le, out_v


def fix_broken_buckets(vals):
    """fixBrokenBuckets :1122 at every point: a NaN first bucket becomes 0, a NaN or smaller later one the value before it"""
    if len(vals) < 2:
        return list(vals)
    v = np.where(np.isnan(vals[0]), 0.0, vals[0])
    out, vnext = [v], v
    for x in vals[1:]:
        with np.errstate(invalid="ignore"):
            x = np.where(np.isnan(x) | (vnext > x), vnext, x)
        out.append(x)
        vnext = x
    return out


def last_non_inf(les):
    """lastNonInf :1000"""
    for le in reversed(les):
        if not math.isinf(le):
            return le
    return NAN


def quantile_cells(phi, les, vals):
    """quantile :1010 at every point of one group; les / vals: the merged and fixed buckets -> (q, lower, upper)"""
    P = phi.shape[0]
    q, lo, up = np.full(P, NAN), np.full(P, NAN), np.full(P, NAN)
    vlast = vals[-1]
    with np.errstate(all="ignore"):
        done = np.isnan(phi) | (vlast == 0)
        m = ~done & (phi < 0)
        q[m], lo[m], up[m] = -INF, -INF, vals[0][m]
        done |= m
        m = ~done & (phi > 1)
        q[m], lo[m], up[m] = INF, vlast[m], INF
        done |= m
        vreq = vlast * phi
        vprev, leprev = np.zeros(P), np.zeros(P)
        tail = np.zeros(P, dtype=bool)  # left the loop by the `break` at :1046
        for le, v in zip(les, vals):
            zero = ~done & (v <= 0)
            leprev = np.where(zero, le, leprev)
            below = ~done & ~(v <= 0) & (v < vreq)
            vprev = np.where(below, v, vprev)
            leprev = np.where(below, le, leprev)
            hit = ~done & ~(v <= 0) & ~(v < vreq)
            done |= hit
            if math.isinf(le):
                tail |= hit
                continue
            eq = hit & (v == vprev)
            q[eq], lo[eq], up[eq] = leprev[eq], leprev[eq], v[eq]
            ne = hit & ~(v == vprev)
            interp = leprev + (le - leprev) * (vreq - vprev) / (v - vprev)
            q[ne], lo[ne], up[ne] = interp[ne], leprev[ne], le
        rest = ~done | tail
        vv = last_non_inf(les)
        q[rest], lo[rest], up[rest] = vv, vv, INF
    return q, lo, up


def _share(req, les, vals):
    """the loop of share :673-696 / :771-792 at every point, after its leReq < 0 and +Inf checks"""
    P = req.shape[0]
    q, lo, up = np.ones(P), np.ones(P), np.ones(P)  # :696 leReq > leLast
    vlast = vals[-1]
    with np.errstate(all="ignore"):
        done = req < 0
        q[done], lo[done], up[done] = 0.0, 0.0, 0.0
        m = ~done & (req == INF)
        done |= m  # 1, 1, 1
        vprev, leprev = np.zeros(P), np.zeros(P)
        for le, v in zip(les, vals):
            ge = ~done & (req >= le)
            vprev = np.where(ge, v, vprev)
            leprev = np.where(ge, le, leprev)
            hit = ~done & ~(req >= le)
            done |= hit
            lower = vprev / vlast
            if le == INF:
                q[hit], lo[hit], up[hit] = lower[hit], lower[hit], 1.0
                continue
            eq = hit & (leprev == req)
            q[eq], lo[eq], up[eq] = lower[eq], lower[eq], lower[eq]
            ne = hit & ~(leprev == req)
            upper = v / vlast
            interp = lower + (v - vprev) / vlast * (req - leprev) / (le - leprev)
            q[ne], lo[ne], up[ne] = interp[ne], lower[ne], upper[ne]
    return q, lo, up


def share_cells(req, les, vals):
    """share :661 at every point of one group (merged buckets; the fix happens here) -> (q, lower, upper)"""
    q, lo, up = _share(req, les, fix_broken_buckets(vals))
    nan = np.isnan(req)
    q[nan], lo[nan], up[nan] = NAN, NAN, NAN
    return q, lo, up


def fraction_cells(lower, upper, les, vals):
    """fraction :759: share(upperle) - share(lowerle), NaN where either bound is NaN"""
    fixed = fix_broken_buckets(vals)
    with np.errstate(invalid="ignore"):
        q = _share(upper, les, fixed)[0] - _share(lower, les, fixed)[0]
    q[np.isnan(lower) | np.isnan(upper)] = NAN
    return q


def moments_cells(name, les, vals):
    """avgForLeTimeseries :876 / stdvarForLeTimeseries :900 (+ sqrt for stddev) on the raw rows of one group"""
    P = vals[0].shape[0]
    le_prev, v_prev = 0.0, np.zeros(P)
    s, s2, wt = np.zeros(P), np.zeros(P), np.zeros(P)
    with np.errstate(all="ignore"):
        for le, v in zip(les, vals):
            if math.isinf(le):
                continue
            n = (le + le_prev) / 2
            w = v - v_prev
            s = s + n * w
            s2 = s2 + n * n * w
            wt = wt + w
            le_prev, v_prev = le, v
        avg = s / wt
        if name == "histogram_avg":
            r = avg
        else:
            r = s2 / wt - avg * avg
            r = np.where(r < 0, 0.0, r)
            if name == "histogram_stddev":
                r = np.sqrt(r)
    return np.where(wt == 0, NAN, r)


def histogram_ref(name, buckets, group_ids, les, ngroups, *scalar_args, bounds=False):
    """vmb_histogram's results -> (out, lower, upper, nonempty): out [ngroups x P] ([nphi x ngroups x P] for histogram_quantiles),
    lower / upper [ngroups x P] (None without bounds), nonempty: one bool per output row (out rows, then lower, then upper).
    scalar_args: numbers or per-point arrays as in promql.histogram.  A group without rows is NaN."""
    m = np.asarray(buckets, dtype=np.float64)
    P = m.shape[1]
    les = [float(x) for x in les]
    args = [np.broadcast_to(np.asarray(a, dtype=np.float64), (P,)) for a in scalar_args]
    nphi = len(args) if name == "histogram_quantiles" else 1
    out = np.full((nphi, ngroups, P), NAN)
    lower, upper = np.full((ngroups, P), NAN), np.full((ngroups, P), NAN)
    for g, rows in enumerate(le_groups(group_ids, les, ngroups)):
        if not rows:
            continue
        gl, gv = [les[r] for r in rows], [m[r] for r in rows]
        if name in ("histogram_avg", "histogram_stddev", "histogram_stdvar"):
            out[0, g] = moments_cells(name, gl, gv)
            continue
        ml, mv = merge_same_le(gl, gv)
        if name in ("histogram_quantile", "histogram_quantiles"):
            fixed = fix_broken_buckets(mv)
            for k in range(nphi):
                out[k, g], lower[g], upper[g] = quantile_cells(np.array(args[k]), ml, fixed)
        elif name == "histogram_share":
            out[0, g], lower[g], upper[g] = share_cells(np.array(args[0]), ml, mv)
        elif name == "histogram_fraction":
            out[0, g] = fraction_cells(np.array(args[0]), np.array(args[1]), ml, mv)
        else:
            raise ValueError(name)
    rows_out = [out.reshape(nphi * ngroups, P)] + ([lower, upper] if bounds else [])
    nonempty = np.concatenate([~np.all(np.isnan(r), axis=1) for r in rows_out])
    return (out if name == "histogram_quantiles" else out[0]), (lower if bounds else None), (upper if bounds else None), nonempty
