"""Python restatement of the row-set functions of app/vmselect/promql that read values: sort / sort_desc (newTransformFuncSort
transform.go:2557), `or` (binaryOpOr binary_op.go:483 with fillLeftNaNsWithRightValuesOrMerge :542 and createTimeseriesMapByTagSet
:657), removeEmptySeries (exec.go:193), drop_empty_series (transform.go:1939), limit_offset (:2275) and union (:1725), the
reference of vmb_sort_rows, vmb_set_or and vmb_rows_nonempty.

A metric name is a dict of labels, `__name__` included.  sort.Slice is restated as a STABLE sort over ascending row order: what Go
returns for up to 12 rows (its insertion sort) and one of the outcomes of its pdqsort beyond.  sortSeriesByMetricName is restated
the same way."""
import functools
import math

import numpy as np

NAN = float("nan")


def sort_less(a, b, desc):
    """the less function of newTransformFuncSort, word for word"""
    n = len(a) - 1
    while n >= 0:
        if not math.isnan(a[n]):
            if math.isnan(b[n]):
                return False
            if a[n] != b[n]:
                break
        elif not math.isnan(b[n]):
            return True
        n -= 1
    if n < 0:
        return False
    return b[n] < a[n] if desc else a[n] < b[n]


def sort_rows_ref(vals, desc=False):
    """sort(q) / sort_desc(q): the rows of vals in output order"""
    rows = [[float(x) for x in r] for r in np.asarray(vals, dtype=np.float64)]

    def cmp(i, j):
        return -1 if sort_less(rows[i], rows[j], desc) else (1 if sort_less(rows[j], rows[i], desc) else 0)
    return sorted(range(len(rows)), key=functools.cmp_to_key(cmp))


def is_stable_sort(vals, order, desc=False, chunk=4096):
    """order is the stable sort of the rows of vals by sort_less: a permutation in which every adjacent pair is in order, and an
    equal pair in ascending row order.  The same test as sort_rows_ref, vectorised for large matrices."""
    vals = np.asarray(vals, dtype=np.float64)
    S, P = vals.shape
    order = np.asarray(order, dtype=np.int64)
    if order.shape != (S,) or not np.array_equal(np.sort(order), np.arange(S)):
        return False
    for i0 in range(0, max(S - 1, 0), chunk):
        i = np.arange(i0, min(S - 1, i0 + chunk))
        a, b = vals[order[i]], vals[order[i + 1]]
        an, bn = np.isnan(a), np.isnan(b)
        differ = (an != bn) | (~an & ~bn & (a != b))
        anyd = differ.any(axis=1)
        n = P - 1 - np.argmax(differ[:, ::-1], axis=1) if P else np.zeros(len(i), dtype=np.int64)
        k = np.arange(len(i))
        av, bv = (a[k, n], b[k, n]) if P else (np.zeros(len(i)), np.zeros(len(i)))
        with np.errstate(invalid="ignore"):
            less = np.where(np.isnan(av), True, np.where(np.isnan(bv), False, bv < av if desc else av < bv))
        if not np.where(anyd, less, order[i] < order[i + 1]).all():
            return False
    return True


def nonempty(vals):
    """removeEmptySeries: the rows that hold a non-NaN value"""
    vals = np.asarray(vals, dtype=np.float64)
    return (~np.isnan(vals)).any(axis=1) if vals.shape[1] else np.zeros(vals.shape[0], dtype=bool)


def name_key(labels):
    """marshalMetricNameSorted: equal keys are equal names"""
    return tuple(sorted(labels.items()))


def name_order(labels):
    """metricNameLess (exec.go:167): the metric group, then the sorted tags, a prefix first"""
    return (labels.get("__name__", ""), tuple(sorted((k, v) for k, v in labels.items() if k != "__name__")))


def is_scalar(labels_list):
    """isScalar binary_op.go:690"""
    return len(labels_list) == 1 and not labels_list[0]


def tagset_key(labels, on=None, ignoring=(), keep_metric_names=False):
    """the map key of createTimeseriesMapByTagSet :657: RemoveTagsOn / RemoveTagsIgnoring of lib/storage/metric_name.go"""
    d = dict(labels)
    if not keep_metric_names:
        d.pop("__name__", None)
    if on is not None:
        d = {k: v for k, v in d.items() if k in on}
    elif ignoring:
        d = {k: v for k, v in d.items() if k not in ignoring}
    return name_key(d)


def set_or_ref(left, left_labels, right, right_labels, on=None, ignoring=(), keep_metric_names=False):
    """binaryOpOr on copies of the matrices -> (left, right, out): the filled matrices and the output rows, ('l', i) / ('r', i)"""
    L, R = np.array(left, dtype=np.float64), np.array(right, dtype=np.float64)  # [rows x points] each
    m_left, m_right = {}, {}
    for i, lb in enumerate(left_labels):
        m_left.setdefault(tagset_key(lb, on, ignoring, keep_metric_names), []).append(i)
    for i, lb in enumerate(right_labels):
        m_right.setdefault(tagset_key(lb, on, ignoring, keep_metric_names), []).append(i)
    lne = nonempty(L)
    rvs = []
    for k in m_left:
        m_left[k] = [i for i in m_left[k] if lne[i]]
        rvs += m_left[k]
    out = [("l", i) for i in sorted(rvs, key=lambda i: (name_order(left_labels[i]), i))]
    added = []
    for k, rr in m_right.items():
        if k not in m_left:
            added += rr
            continue
        ll = m_left[k]
        scalar = is_scalar([right_labels[r] for r in rr])
        can_scalar = is_scalar([left_labels[i] for i in ll])
        for li in ll:
            left_nan = np.isnan(L[li])
            for r in rr:
                can = can_scalar if scalar else name_key(left_labels[li]) == name_key(right_labels[r])
                if can:
                    L[li] = np.where(left_nan, R[r], L[li])
                R[r] = np.where(~left_nan | can, NAN, R[r])
        rne = nonempty(R)
        added += [r for r in rr if rne[r]]
    out += [("r", i) for i in sorted(added, key=lambda i: (name_order(right_labels[i]), i))]
    return L, R, out


def drop_empty_series_ref(vals):
    return [i for i, ne in enumerate(nonempty(vals)) if ne]


def limit_offset_ref(limit, offset, vals):
    rows = drop_empty_series_ref(vals)
    rows = rows[offset:] if len(rows) >= offset else []
    return rows[:limit] if len(rows) > limit else rows


def union_ref(args):
    """args: [labels of every row] per argument -> [(arg, row)]"""
    if all(is_scalar(a) for a in args):
        return [(j, 0) for j in range(len(args))]
    seen, out = set(), []
    for j, a in enumerate(args):
        for i, lb in enumerate(a):
            k = name_key(lb)
            if k not in seen:
                seen.add(k)
                out.append((j, i))
    return out
