"""numpy restatement of the non-incremental aggregates of app/vmselect/promql/aggr.go (aggrFuncExt :110, aggrPrepareSeries :121,
aggrFuncSum :185 ... aggrFuncZScore :493), the reference of vmb_aggr_matrix.

Every function loops over the rows of a group in ascending row order and is vectorised over the points, so each cell sees the
same float operations in the same order as the Go loop over `tss`: the results are the reference's bits (numpy's float64 + - * /
and sqrt are IEEE; only geomean's pow is another implementation)."""
import numpy as np

NAN = float("nan")
GROUP_FUNCS = ["sum", "sum2", "min", "max", "avg", "count", "group", "geomean", "stddev", "stdvar"]
ROW_FUNCS = ["share", "zscore"]
FAST_PATH = {"sum", "avg", "min", "max", "geomean"}  # `len(tss) == 1`: the row as it is


def _fold(name, rows):
    """the general path over rows (a list of [P] arrays, non-empty rows only) -> [P]"""
    P = rows[0].shape[0]
    a = np.full(P, NAN) if name in ("min", "max") else np.full(P, 1.0 if name == "geomean" else 0.0)
    q = np.zeros(P)
    n = np.zeros(P)
    with np.errstate(all="ignore"):
        for v in rows:
            m = ~np.isnan(v)
            if name == "min":
                a = np.where(np.isnan(a) | (v < a), v, a)
                continue
            if name == "max":
                a = np.where(np.isnan(a) | (v > a), v, a)
                continue
            n = n + m
            if name in ("sum", "avg"):
                a = np.where(m, a + v, a)
            elif name == "sum2":
                a = np.where(m, a + v * v, a)
            elif name == "geomean":
                a = np.where(m, a * v, a)
            elif name in ("stddev", "stdvar"):
                an = a + (v - a) / n
                q = np.where(m, q + (v - a) * (v - an), q)
                a = np.where(m, an, a)
        if name in ("min", "max"):
            return a
        if name in ("sum", "sum2"):
            return np.where(n > 0, a, NAN)
        if name == "avg":
            return np.where(n > 0, a / n, NAN)
        if name == "count":
            return np.where(n > 0, n, NAN)
        if name == "group":
            return np.where(n > 0, 1.0, NAN)
        if name == "geomean":
            return np.where(n == 0, NAN, np.where(n == 1, a, np.power(a, 1.0 / n)))
        var = np.where(n > 0, q, NAN) / n
        return np.sqrt(var) if name == "stddev" else var


def _share(rows):
    with np.errstate(all="ignore"):
        s = np.zeros(rows[0].shape[0])
        for v in rows:
            s = np.where(np.isnan(v) | (v < 0), s, s + v)
        return [np.where(np.isnan(v) | (v < 0), NAN, v / s) for v in rows]


def _zscore(rows):
    with np.errstate(all="ignore"):
        P = rows[0].shape[0]
        avg, q, n = np.zeros(P), np.zeros(P), np.zeros(P)
        for v in rows:
            m = ~np.isnan(v)
            n = n + m
            an = avg + (v - avg) / n
            q = np.where(m, q + (v - avg) * (v - an), q)
            avg = np.where(m, an, avg)
        sd = np.sqrt(q / n)
        return [np.where(np.isnan(v), v, (v - avg) / sd) for v in rows]


def aggr_matrix_ref(name, vals, group_ids=None, ngroups=1, limit=0):
    """-> (out, returned): out [ngroups x P] (share / zscore: [nseries x P], rows of groups without a value unchanged) and the group
    ids the reference outputs in order of their first non-empty row, cut at `limit` (share / zscore: the mask of the rows)"""
    vals = np.asarray(vals, dtype=np.float64)
    S, P = vals.shape
    g = np.zeros(S, dtype=np.int64) if group_ids is None else np.asarray(group_ids, dtype=np.int64)
    nonempty = ~np.all(np.isnan(vals), axis=1) if P else np.zeros(S, dtype=bool)  # removeEmptySeries
    order, members = [], {}
    for r in range(S):
        if nonempty[r]:
            if g[r] not in members:
                order.append(int(g[r]))
                members[g[r]] = []
            members[g[r]].append(r)
    kept = order[:limit] if limit > 0 else order
    if name in ROW_FUNCS:
        out = vals.copy()
        for gid in order:
            idx = members[gid]
            for r, v in zip(idx, (_share if name == "share" else _zscore)([vals[r] for r in idx])):
                out[r] = v
        return out, nonempty & np.isin(g, kept)
    out = np.full((ngroups, P), NAN)
    for gid in order:
        rows = [vals[r] for r in members[gid]]
        if len(rows) == 1 and name in FAST_PATH:
            out[gid] = rows[0]
        elif len(rows) == 1 and name in ("stddev", "stdvar"):
            out[gid] = np.where(np.isnan(rows[0]), NAN, 0.0)
        else:
            out[gid] = _fold(name, rows)
    return out, np.array(kept, dtype=np.int64)
