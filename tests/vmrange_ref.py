"""numpy restatement of the `vmrange` histogram functions of app/vmselect/promql/transform.go, the reference of vmb_vmrange_to_le
and vmb_buckets_limit:

  vmrangeBucketsToLE :494-632   (prometheus_buckets :485 and the front of every histogram_*)
  transformBucketsLimit :386-483
  mergeNonOverlappingTimeseries  binary_op.go:367-400

The Go code keys its maps by strings and aliases *timeseries pointers; here every series is a Python object whose values array
is mutated in place, so the same aliasing happens: a gap row's map entry names the SOURCE row, a later equal end merges into that
row, and an `a...a` row after a gap at `a` merges into itself.  Go iterates its group map in random order; here the kept rows come
first, then the groups in ascending id (the library's order).  sort.Slice is restated as the insertion sort Go uses for up to 12
elements, for every group size, as the library does.

go_parse_float restates strconv.ParseFloat(s, 64) acceptance from Go's published documentation (Go's strconv source is not part
of the reference): a scanner in the shape of the documented grammar, independent of the product's regex version."""
import math

import numpy as np

from histogram_ref import go_insertion_sort

NAN, INF = float("nan"), float("inf")
KEEP, DROP = 0xFFFFFFFE, 0xFFFFFFFF
KEPT, BUCKET, GAP, PINF = 0, 1, 2, 3  # enum vmb_vr_kind

_HEX = "0123456789abcdef"


def go_parse_float(s):
    """strconv.ParseFloat(s, 64): the float, or None for ErrSyntax / ErrRange.
    Documented rules: "NaN", and "Inf" / "Infinity" with an optional sign, matched in any case; otherwise a decimal or
    hexadecimal floating-point number in the syntax of Go's floating-point literals -- optional sign, digits with at most one
    '.', at least one digit; decimal: an optional e exponent; hexadecimal (0x prefix): a mandatory p exponent; an exponent is
    an optional sign and digits; an underscore only between two digits or between the 0x prefix and a digit -- and nothing else
    in the string.  Correctly rounded; beyond the float64 range is ErrRange; below it rounds to (signed) zero."""
    low = s.lower()
    body = low[1:] if low[:1] in ("+", "-") else low
    if body in ("inf", "infinity"):
        return -INF if low[0] == "-" else INF
    if low == "nan":
        return NAN
    i, hexa = 0, body.startswith("0x") and len(body) > 2
    digits = _HEX if hexa else _HEX[:10]
    if hexa:
        i = 2
    mant_digits = 0
    dot = False
    while i < len(body):
        c = body[i]
        if c in digits:
            mant_digits += 1
        elif c == "." and not dot:
            dot = True
        elif c != "_":
            break
        i += 1
    if not mant_digits:
        return None
    if i < len(body) and body[i] == ("p" if hexa else "e"):
        i += 1
        if i < len(body) and body[i] in "+-":
            i += 1
        if i >= len(body) or not body[i].isdigit():
            return None
        while i < len(body) and (body[i].isdigit() or body[i] == "_"):
            i += 1
    elif hexa:
        return None
    if i != len(body):
        return None
    # underscores: each one between two digits (the 0x prefix counts as a digit)
    prev = "d" if hexa else "^"
    for c in body[2 if hexa else 0:]:
        if c == "_":
            if prev != "d":
                return None
            prev = "_"
        elif c in digits:
            prev = "d"
        else:
            if prev == "_":
                return None
            prev = "!"
    if prev == "_":
        return None
    t = s.replace("_", "")
    try:
        v = float.fromhex(t) if hexa else float(t)
    except OverflowError:
        return None
    return None if math.isinf(v) else v


class TS:
    """a *timeseries: its input row and its values"""

    def __init__(self, row, values):
        self.row, self.values = row, values


def merge_non_overlapping(dst, src):
    """binary_op.go:367"""
    overlaps = int(np.sum(~np.isnan(src.values) & ~np.isnan(dst.values)))
    if overlaps > 2:
        return False
    if len(src.values) <= 2 and len(dst.values) <= 2:
        return False
    ok = ~np.isnan(src.values)
    dst.values[ok] = src.values[ok]
    return True


def vmrange_to_le_ref(m, vmranges, les, groups):
    """vmrangeBucketsToLE on rows with labels: vmranges[i] (None: no label), les[i] (None or "": no `le`), groups[i] the id of
    the row's labels without vmrange / le.  -> [(src row, kind, le string or None, values)] in output order"""
    m = np.asarray(m, dtype=np.float64)
    P = m.shape[1]
    out, grouped = [], {}
    for i, vr in enumerate(vmranges):
        if not vr:
            if les[i]:
                out.append((i, KEPT, None, m[i].copy()))  # :511
            continue
        n = vr.find("...")
        if n < 0:
            continue
        start_s, end_s = vr[:n], vr[n + 3:]
        start, end = go_parse_float(start_s), go_parse_float(end_s)
        if start is None or end is None:
            continue
        grouped.setdefault(groups[i], []).append(dict(start_s=start_s, end_s=end_s, start=start, end=end,
                                                      ts=TS(i, m[i].copy())))
    for g in sorted(grouped):
        xss = grouped[g]
        xss = [xss[k] for k in go_insertion_sort([x["end"] for x in xss])]  # :565
        new = []  # (x, kind, le string)
        prev = dict(end=0.0, ts=None)
        uniq = {}
        for xs in xss:
            ts = xs["ts"]
            if not np.any(ts.values > 0):  # isZeroTS :556
                continue
            if xs["start"] != prev["end"]:  # :580
                if uniq.get(xs["start_s"]) is None:
                    uniq[xs["start_s"]] = ts
                    new.append((TS(ts.row, np.zeros(P)), GAP, xs["start_s"]))
            prev_ts = uniq.get(xs["end_s"])
            if prev_ts is not None:
                merge_non_overlapping(prev_ts, ts)  # :598
            else:
                new.append((ts, BUCKET, xs["end_s"]))
                uniq[xs["end_s"]] = ts
            prev = xs
        if prev["ts"] is not None and not (prev["end"] == INF) and np.any(prev["ts"].values > 0):  # :605
            new.append((TS(prev["ts"].row, np.zeros(P)), PINF, "+Inf"))
        count = np.zeros(P)
        for ts, _, _ in new:  # :616-626, every point at once
            v = ts.values
            with np.errstate(invalid="ignore"):
                count = np.where(~np.isnan(v) & (v > 0), count + v, count)
            ts.values[:] = count
        out += [(ts.row, kind, le, ts.values) for ts, kind, le in new]
    return out


def vmrange_to_le_arrays(m, vmranges, les, groups):
    """-> (matrix [n x P], src np.int64[n], kinds np.uint8[n], le strings) of vmrange_to_le_ref"""
    rows = vmrange_to_le_ref(m, vmranges, les, groups)
    P = np.asarray(m).shape[1]
    mat = np.array([r[3] for r in rows]).reshape(len(rows), P)
    return (mat, np.array([r[0] for r in rows], dtype=np.int64), np.array([r[1] for r in rows], dtype=np.uint8),
            [r[2] for r in rows])


def buckets_limit_ref(limit, m, group_ids, les, ngroups):
    """transformBucketsLimit :395-481 after vmrangeBucketsToLE: rows with group_ids[i] == DROP have no parsable `le`.
    -> the kept rows in output order (groups in ascending id)"""
    if limit <= 0:
        return []
    limit = max(limit, 3)
    m = np.asarray(m, dtype=np.float64)
    P = m.shape[1]
    members = [[] for _ in range(ngroups)]
    for r, g in enumerate(group_ids):
        if g != DROP:
            members[g].append(r)
    out = []
    for rows in members:
        if len(rows) <= limit:
            out += rows
            continue
        rows = [rows[k] for k in go_insertion_sort([float(les[r]) for r in rows])]
        hits = [0.0] * len(rows)
        for n in range(P):  # :455-463, point by point as Go does
            prev = 0.0
            for i, r in enumerate(rows):
                v = float(m[r, n])
                hits[i] += v - prev
                prev = v
        while len(rows) > limit:  # :464-477
            imin, mmin = 1, hits[1] + hits[2]
            for i in range(len(rows) - 3):
                mh = hits[i + 1] + hits[i + 2]
                if mh < mmin:
                    imin, mmin = i + 1, mh
            hits[imin + 1] += hits[imin]
            del hits[imin], rows[imin]
        out += rows
    return out
