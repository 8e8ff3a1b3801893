"""Restatements of the two count_values loops of the reference, for the tests.

count_values (the afe closure of app/vmselect/promql/aggr.go:594): a map keyed by float64 per group, so -0.0 and +0.0 are one key
and the label comes from the first value met (a Python dict keeps its first key object the same way).

count_values_over_time (newRollupCountValues rollup.go:1490 through rollupConfig.DoTimeseriesMap :693): a map keyed by the 'g'
string of every value in every point's window.  The windows come from the oracle's rollupConfig.Do loop (vmo_rollup_do, the code the
rollupConfig.Do known-answer tests pin) run over the row numbers, so that no second copy of the window rules exists here.
"""
import struct

import numpy as np

import oracle_lib as O
from rollup_names import RF
from victoriametrics_b200.promql import go_format_float

STALE_NAN_BITS = 0x7FF0000000000002  # decimal.StaleNaN


def count_values(vals, group_ids, ngroups):
    """-> {group: [(value, counts[P])]} with each group's rows in the order the map first met their values"""
    vals = np.asarray(vals, dtype=np.float64)
    out = {}
    for g in range(ngroups):
        m = {}
        for row in np.flatnonzero(np.asarray(group_ids) == g):
            for i, v in enumerate(vals[row].tolist()):
                if v != v:
                    continue
                if v not in m:
                    m[v] = np.full(vals.shape[1], np.nan)
                c = m[v]
                c[i] = 1 if c[i] != c[i] else c[i] + 1
        if m:
            out[g] = list(m.items())
    return out


def rollup_windows(values, timestamps, start, end, step, window, lookback_delta=0, min_staleness_ms=0):
    """the windows [lo[p], hi[p]) of rollupConfig.Do over one series, and its samplesScanned.  The oracle's own loop finds them:
    over values that are the row numbers, first_over_time gives a non-empty window's first row and last_over_time its last (NaN
    for an empty window, which counts nothing); samplesScanned does not depend on the values."""
    timestamps = np.ascontiguousarray(timestamps, dtype=np.int64)
    rows = np.arange(len(values), dtype=np.float64)
    cfg = dict(lookback_delta=lookback_delta, min_staleness_ms=min_staleness_ms)
    first, scanned = O.rollup_do(RF["first_over_time"], rows, timestamps, start, end, step, window, **cfg)
    last, _ = O.rollup_do(RF["last_over_time"], rows, timestamps, start, end, step, window, **cfg)
    empty = np.isnan(first)
    lo = np.where(empty, 0, np.nan_to_num(first)).astype(np.int64)
    hi = np.where(empty, 0, np.nan_to_num(last) + 1).astype(np.int64)
    return lo, hi, int(scanned)


def is_stale(v):
    return struct.unpack("<Q", struct.pack("<d", v))[0] == STALE_NAN_BITS


def count_values_over_time(values, timestamps, start, end, step, window, lookback_delta=0, drop_stale=True):
    """one series -> ({'g' label: counts[P]} in first-met order, samplesScanned)"""
    v = np.asarray(values, dtype=np.float64)
    t = np.asarray(timestamps, dtype=np.int64)
    if drop_stale:  # dropStaleNaNs eval.go:1985
        keep = np.array([not is_stale(x) for x in v.tolist()], dtype=bool)
        v, t = v[keep], t[keep]
    lo, hi, scanned = rollup_windows(v, t, start, end, step, window, lookback_delta)
    P = lo.size
    m = {}
    vl = v.tolist()
    for p in range(P):
        for r in range(lo[p], max(lo[p], hi[p])):
            k = go_format_float(vl[r], "g")
            if k not in m:
                m[k] = np.full(P, np.nan)
            c = m[k]
            c[p] = 1 if c[p] != c[p] else c[p] + 1
    return m, scanned
