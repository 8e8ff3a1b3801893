"""numpy restatement of the aggregates of app/vmselect/promql/aggr.go that rank whole series: topk_min ... bottomk_last
(newAggrFuncRangeTopK :677, getRangeTopKTimeseries :704, getRemainingSumTimeseries :751, fillNaNsAtIdx :786, getIntK :793, the
score functions :804-858) and outliersk (aggrFuncOutliersK :1040, getPerPointMedians :1066), the reference of vmb_aggr_rank.

Every chain the reference runs in a loop is run in the same order here: the sums go through np.cumsum (sequential adds) after a
leading 0.0, with 0.0 in place of the skipped NaNs (x + 0.0 is x for every x such a sum can hold, since 0.0 + -0.0 is already +0.0);
min / max / last walk the points one by one.  sort.Slice is restated as a STABLE sort over ascending row order, which is what Go
returns for up to 12 rows and one of the outcomes of its pdqsort beyond."""
import math

import numpy as np

NAN = float("nan")
SCORES = ["min", "max", "avg", "median", "last"]
NAMES = ["topk_" + s for s in SCORES] + ["bottomk_" + s for s in SCORES] + ["outliersk"]


def int_k(k, n):
    """getIntK :793 over floatToIntBounded :1281"""
    if math.isnan(k):
        return 0
    kn = 2 ** 63 - 1 if k > 2 ** 63 - 1 else -2 ** 63 if k < -2 ** 63 else int(k)
    return 0 if kn < 0 else min(kn, n)


def median_rows(a):
    """quantile(0.5, row) :870 for every row of a: the NaNs dropped, sorted, quantileSorted :922"""
    a = np.sort(a, axis=1)  # NaNs last
    cnt = (~np.isnan(a)).sum(axis=1)
    n = cnt.astype(np.float64)
    rank = 0.5 * (n - 1)
    lo = np.maximum(0.0, np.floor(rank))
    hi = np.minimum(n - 1, lo + 1)
    w = rank - np.floor(rank)
    r = np.arange(a.shape[0])
    with np.errstate(invalid="ignore", over="ignore"):
        out = a[r, np.maximum(lo, 0).astype(np.int64)] * (1 - w) + a[r, np.maximum(hi, 0).astype(np.int64)] * w
    out[cnt == 0] = NAN
    return out


def chain_sum(a, axis):
    """0 + a[0] + a[1] ... along axis, in order"""
    pad = np.zeros_like(np.take(a, [0], axis=axis))
    with np.errstate(invalid="ignore", over="ignore"):
        return np.cumsum(np.concatenate([pad, a], axis=axis), axis=axis)


def scores_of(kind, vals):
    """f(ts.Values) for every row (:804-858)"""
    S, P = vals.shape
    nn = ~np.isnan(vals)
    if kind == "avg":
        with np.errstate(invalid="ignore", divide="ignore"):
            return np.where(nn.any(axis=1), chain_sum(np.where(nn, vals, 0.0), 1)[:, -1] / nn.sum(axis=1).astype(np.float64), NAN)
    if kind == "median":
        return median_rows(vals)
    acc = np.full(S, NAN)
    for p in range(P):
        v = vals[:, p]
        with np.errstate(invalid="ignore"):
            if kind == "min":
                acc = np.where(np.isnan(acc) | (v < acc), v, acc)
            elif kind == "max":
                acc = np.where(np.isnan(acc) | (v > acc), v, acc)
            else:
                acc = np.where(nn[:, p], v, acc)
    return acc


def rank_aggr_ref(name, ks, vals, group_ids=None, ngroups=1, remaining=False, limit=0):
    """-> dict:
    masked     [S x P]: the matrix with the survivors masked (fillNaNsAtIdx); every other row as it was (the reference drops them)
    remaining  [ngroups x P] remaining-sum rows (NaN for a group without rows), or None
    remaining_nonempty  bool [ngroups]
    nonempty   bool [S]: rows with a value before the call
    survivors  per group id, the surviving rows from best to worst
    out        the reference's output: groups in order of their first non-empty row, cut at `limit`; per group -(g + 1) for the
               remaining-sum row where it holds a value, then the survivors
    scores     [S]"""
    vals = np.asarray(vals, dtype=np.float64)
    S, P = vals.shape
    g = np.zeros(S, dtype=np.int64) if group_ids is None else np.asarray(group_ids, dtype=np.int64)
    ks = np.broadcast_to(np.asarray(ks, dtype=np.float64), (P,))
    reverse = name.startswith("bottomk_")
    kind = name if name == "outliersk" else name.split("_")[1]
    nonempty = ~np.isnan(vals).all(axis=1) if P else np.zeros(S, dtype=bool)
    if kind == "outliersk":
        scores = np.full(S, NAN)
        for gid in range(ngroups):
            rows = np.flatnonzero(nonempty & (g == gid))
            if len(rows):
                med = median_rows(vals[rows].T)  # getPerPointMedians :1066
                with np.errstate(invalid="ignore", over="ignore"):
                    d = vals[g == gid] - med
                    scores[g == gid] = chain_sum(d * d, 1)[:, -1]
        # a row without a value scores NaN whatever the medians are; groups without any such row have no medians
        scores[~nonempty] = NAN
    else:
        scores = scores_of(kind, vals)
    masked = vals.copy()
    rem = np.full((ngroups, P), NAN) if remaining else None
    survivors = [[] for _ in range(ngroups)]
    for gid in range(ngroups):
        rows = np.flatnonzero(nonempty & (g == gid))
        n = len(rows)
        if n == 0:
            continue
        sc = scores[rows]
        isn = np.isnan(sc)
        key = np.where(isn, 0.0, -sc if reverse else sc)
        srt = rows[np.lexsort((key, ~isn))]  # stable; NaN scores first (lessWithNaNs :1259 / greaterWithNaNs :1270)
        cut = np.array([n - int_k(float(k), n) for k in ks], dtype=np.int64)  # tss[:len(tss)-kn] lose point p
        sv = vals[srt]
        if remaining:
            nn = ~np.isnan(sv)
            sums = chain_sum(np.where(nn, sv, 0.0), 0)
            counts = np.concatenate([np.zeros((1, P), dtype=np.int64), np.cumsum(nn, axis=0)])
            cols = np.arange(P)
            rem[gid] = np.where(counts[cut, cols] > 0, sums[cut, cols], NAN)
        for pos in range(n - 1, int(cut.min()) - 1, -1) if P else ():  # below the cut of every point nothing survives
            row = np.where(pos < cut, NAN, sv[pos])
            if not np.isnan(row).all():
                masked[srt[pos]] = row
                survivors[gid].append(int(srt[pos]))
    rem_ne = ~np.isnan(rem).all(axis=1) if remaining else np.zeros(ngroups, dtype=bool)
    _, first = np.unique(g[nonempty], return_index=True)  # aggrPrepareSeries :121: groups in order of their first non-empty row
    order = [int(x) for x in g[nonempty][np.sort(first)]]
    if limit > 0:
        order = order[:limit]
    out = []
    for gid in order:
        if rem_ne[gid]:
            out.append(-(gid + 1))
        out.extend(survivors[gid])
    return dict(masked=masked, remaining=rem, remaining_nonempty=rem_ne, nonempty=nonempty, survivors=survivors,
                out=np.array(out, dtype=np.int64), scores=scores)
