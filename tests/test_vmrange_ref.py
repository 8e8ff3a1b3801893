"""tests/vmrange_ref.py (the reference of vmb_vmrange_to_le and vmb_buckets_limit) pinned on the reference's own tests and on
hand-worked cases:

  - every case of TestVmrangeBucketsToLE (app/vmselect/promql/transform_test.go:70-245), in its output order;
  - the buckets_limit and prometheus_buckets vectors of exec_test.go:4836-5341 (series on the time() grid 1000 ... 2000 s,
    step 200 s; the query's outer sort() makes the comparison order-free, by metric name);
  - each quirk of the string-keyed walk, worked by hand;
  - go_parse_float of the restatement and of the product against Go's documented ParseFloat rules;
  - the ids of include/vmb200.h against the Python ones."""
import os
import re

import numpy as np
import pytest

import vmrange_ref as V

NAN, INF = float("nan"), float("inf")
T = np.arange(1000, 2001, 200, dtype=np.float64)  # time()
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ transform_test.go:70-245
def prom_rows(text):
    """`name{k="v", ...} value ts` lines -> [(labels, value)]"""
    out = []
    for line in text.strip().splitlines():
        m = re.fullmatch(r"\s*(\w+)(?:\{(.*)\})?\s+(\S+)\s+(\S+)\s*", line)
        labels = dict(re.findall(r'(\w+)="([^"]*)"', m.group(2) or ""))
        out.append((labels, float(m.group(3))))
    return out


def to_le(rows, P=1):
    """the rows of one metric through vmrange_to_le_ref -> [(le, value)] in output order"""
    m = np.array([[v] * P for _, v in rows]).reshape(len(rows), P)
    keys = {}
    groups = [keys.setdefault(tuple(sorted((k, v) for k, v in l.items() if k not in ("vmrange", "le"))), len(keys))
              for l, _ in rows]
    out = V.vmrange_to_le_ref(m, [l.get("vmrange") for l, _ in rows], [l.get("le") for l, _ in rows], groups)
    return [(rows[src][0]["le"] if le is None else le, vals[0]) for src, _, le, vals in out]


TRANSFORM_TEST = [  # transform_test.go line, input, expected
    (83, 'foo{vmrange="4.084e+02...4.642e+02"} 2 123', [("4.084e+02", 0), ("4.642e+02", 2), ("+Inf", 2)]),
    (89, 'foo{vmrange="0...+Inf"} 5 123', [("+Inf", 5)]),
    (93, 'foo{vmrange="-Inf...0"} 4 123', [("-Inf", 0), ("0", 4), ("+Inf", 4)]),
    (99, 'foo{vmrange="-Inf...+Inf"} 1.23 456', [("-Inf", 0), ("+Inf", 1.23)]),
    (104, 'foo{vmrange="0...0"} 5.3 0', [("0", 5.3), ("+Inf", 5.3)]),
    (111, 'foo{vmrange="7.743e+05...8.799e+05"} 5 123\nfoo{vmrange="6.813e+05...7.743e+05"} 0 123',
     [("7.743e+05", 0), ("8.799e+05", 5), ("+Inf", 5)]),
    (120, 'foo{vmrange="7.743e+05...8.799e+05"} 5 123\nfoo{vmrange="6.813e+05...7.743e+05"} 0 123\n'
          'foo{vmrange="5.813e+05...6.813e+05"} 0 123', [("7.743e+05", 0), ("8.799e+05", 5), ("+Inf", 5)]),
    (129, 'foo{vmrange="8.799e+05...9.813e+05"} 0 123\nfoo{vmrange="7.743e+05...8.799e+05"} 5 123\n'
          'foo{vmrange="6.813e+05...7.743e+05"} 0 123\nfoo{vmrange="5.813e+05...6.813e+05"} 0 123',
     [("7.743e+05", 0), ("8.799e+05", 5), ("+Inf", 5)]),
    (141, 'foo{vmrange="4.084e+02...4.642e+02"} 2 123\nfoo{vmrange="1.234e+02...4.084e+02"} 3 123',
     [("1.234e+02", 0), ("4.084e+02", 3), ("4.642e+02", 5), ("+Inf", 5)]),
    (152, 'foo{vmrange="1...2"} 2 123\nfoo{vmrange="4...6"} 3 123', [("1", 0), ("2", 2), ("4", 2), ("6", 5), ("+Inf", 5)]),
    (164, 'foo{vmrange="1...5"} 2 123\nfoo{vmrange="4...6"} 3 123', [("1", 0), ("5", 2), ("4", 2), ("6", 5), ("+Inf", 5)]),
    (176, 'foo{vmrange="1...5"} 2 123\nfoo{vmrange="0...5"} 3 123', [("1", 0), ("5", 2), ("0", 2), ("+Inf", 2)]),
    (187, 'foo{vmrange="0...1"} 0 123', []),
    (191, 'foo{vmrange="0...+Inf"} 0 123', []),
    (195, 'foo{vmrange="-Inf...0"} 0 123', []),
    (199, 'foo{vmrange="0...0"} 0 0', []),
    (203, 'foo{vmrange="-Inf...+Inf"} 0 456', []),
    (209, 'foo{vmrange="2...3"} 0 123\nfoo{vmrange="1...2"} 0 123', []),
    (216, 'foo{vmrange="4.084e+02...4.642e+02"} -5 1', []),
    (222, 'foo 3 6', []),
    (228, 'foo{le="456"} 3 6', [("456", 3)]),
    (234, 'foo{vmrange="foo...bar"} 1 1', []),
    (238, 'foo{vmrange="4.084e+02"} 1 1', []),
    (242, 'foo{vmrange="4.084e+02...foo"} 1 1', []),
]


@pytest.mark.parametrize("line,text,want", TRANSFORM_TEST, ids=[str(c[0]) for c in TRANSFORM_TEST])
def test_transform_test_cases(line, text, want):
    got = to_le(prom_rows(text))
    assert [(le, float(v)) for le, v in got] == [(le, float(v)) for le, v in want], line


# ------------------------------------------------------------------------------------------------ exec_test.go:4836-5341
def labelled(*items):
    """alias(label_set(v, k1, v1, ...), name) -> [(values, labels)]; v: a number or ("time", d) for time()/d"""
    out = []
    for v, name, *kv in items:
        vals = T / v[1] if isinstance(v, tuple) else np.full(6, float(v))
        out.append((vals, dict(zip(kv[::2], kv[1::2]), __name__=name)))
    return out


def prometheus_buckets(ss):
    """vmrange_to_le_ref over labelled series -> {(name, sorted labels with the new le): values}"""
    m = np.array([v for v, _ in ss])
    keys = {}
    groups = [keys.setdefault(tuple(sorted((k, v) for k, v in l.items() if k not in ("vmrange", "le"))), len(keys))
              for _, l in ss]
    out = V.vmrange_to_le_ref(m, [l.get("vmrange") for _, l in ss], [l.get("le") for _, l in ss], groups)
    res = {}
    for src, kind, le, vals in out:
        l = dict(ss[src][1])
        l.pop("vmrange", None)
        if kind != V.KEPT:
            l["le"] = le
        res[tuple(sorted(l.items()))] = vals
    return res


def key(name, **kw):
    return tuple(sorted(dict(kw, __name__=name).items()))


def same(got, want):
    assert set(got) == set(want), (sorted(got), sorted(want))
    for k, v in want.items():
        assert np.array_equal(got[k], np.asarray(v, dtype=np.float64)), (k, got[k], v)


def test_exec_prometheus_buckets_missing_vmrange():  # exec_test.go:4948
    ss = labelled((("t", 20), "xyz", "foo", "bar", "le", "0.2"), (("t", 100), "xxx", "foo", "bar", "vmrange", "foobar"),
                  (("t", 100), "xxx", "foo", "bar", "vmrange", "30...foobar"),
                  (("t", 100), "xxx", "foo", "bar", "vmrange", "30...40"),
                  (("t", 80), "yyy", "foo", "bar", "vmrange", "0...900", "le", "54"),
                  (("t", 40), "yyy", "foo", "bar", "vmrange", "900...+Inf", "le", "2343"))
    same(prometheus_buckets(ss), {
        key("xxx", foo="bar", le="30"): [0, 0, 0, 0, 0, 0],
        key("xxx", foo="bar", le="40"): [10, 12, 14, 16, 18, 20],
        key("xxx", foo="bar", le="+Inf"): [10, 12, 14, 16, 18, 20],
        key("yyy", foo="bar", le="900"): [12.5, 15, 17.5, 20, 22.5, 25],
        key("yyy", foo="bar", le="+Inf"): [37.5, 45, 52.5, 60, 67.5, 75],
        key("xyz", foo="bar", le="0.2"): [50, 60, 70, 80, 90, 100]})


def test_exec_prometheus_buckets_zero_vmrange_value():  # exec_test.go:5057
    same(prometheus_buckets([(np.zeros(6), {"vmrange": "0...0"})]), {})


VALID = [(90, "xxx", "foo", "bar", "vmrange", "0...0"), (("t", 20), "xxx", "foo", "bar", "vmrange", "0...0.2"),
         (("t", 100), "xxx", "foo", "bar", "vmrange", "0.2...40"), (("t", 10), "xxx", "foo", "bar", "vmrange", "40...Inf")]


def test_exec_prometheus_buckets_valid():  # exec_test.go:5063
    same(prometheus_buckets(labelled(*VALID)), {
        key("xxx", foo="bar", le="0"): [90] * 6,
        key("xxx", foo="bar", le="0.2"): [140, 150, 160, 170, 180, 190],
        key("xxx", foo="bar", le="40"): [150, 162, 174, 186, 198, 210],
        key("xxx", foo="bar", le="Inf"): [250, 282, 314, 346, 378, 410]})


OVERLAPPED = [(90, "xxx", "foo", "bar", "vmrange", "0...0"), (("t", 20), "xxx", "foo", "bar", "vmrange", "0...0.2"),
              (("t", 20), "xxx", "foo", "bar", "vmrange", "0.2...0.25"), (("t", 20), "xxx", "foo", "bar", "vmrange", "0...0.26"),
              (("t", 100), "xxx", "foo", "bar", "vmrange", "0.2...40"), (("t", 10), "xxx", "foo", "bar", "vmrange", "40...Inf")]
OVERLAPPED_END = [(90, "xxx", "foo", "bar", "vmrange", "0...0"), (("t", 20), "xxx", "foo", "bar", "vmrange", "0...0.2"),
                  (("t", 20), "xxx", "foo", "bar", "vmrange", "0.2...0.25"),
                  (("t", 20), "xxx", "foo", "bar", "vmrange", "0...0.25"),
                  (("t", 100), "xxx", "foo", "bar", "vmrange", "0.2...40"), (("t", 10), "xxx", "foo", "bar", "vmrange", "40...Inf")]


def test_exec_prometheus_buckets_overlapped_ranges():  # exec_test.go:5138
    same(prometheus_buckets(labelled(*OVERLAPPED)), {
        key("xxx", foo="bar", le="0"): [90] * 6,
        key("xxx", foo="bar", le="0.2"): [140, 150, 160, 170, 180, 190],
        key("xxx", foo="bar", le="0.25"): [190, 210, 230, 250, 270, 290],
        key("xxx", foo="bar", le="0.26"): [240, 270, 300, 330, 360, 390],
        key("xxx", foo="bar", le="40"): [250, 282, 314, 346, 378, 410],
        key("xxx", foo="bar", le="Inf"): [350, 402, 454, 506, 558, 610]})


def test_exec_prometheus_buckets_overlapped_at_the_end():  # exec_test.go:5248: the merge of 0...0.25 is refused (6 overlaps)
    same(prometheus_buckets(labelled(*OVERLAPPED_END)), {
        key("xxx", foo="bar", le="0"): [90] * 6,
        key("xxx", foo="bar", le="0.2"): [140, 150, 160, 170, 180, 190],
        key("xxx", foo="bar", le="0.25"): [190, 210, 230, 250, 270, 290],
        key("xxx", foo="bar", le="40"): [200, 222, 244, 266, 288, 310],
        key("xxx", foo="bar", le="Inf"): [300, 342, 384, 426, 468, 510]})


def limit_inputs(ss):
    """buckets_limit's grouping by labels without `le` (unparsable le: dropped) -> (matrix, group ids, les, ngroups)"""
    keys, gids, les = {}, [], []
    for _, l in ss:
        le = V.go_parse_float(l["le"]) if l.get("le") else None
        if le is None:
            gids.append(V.DROP)
            les.append(0.0)
            continue
        gids.append(keys.setdefault(tuple(sorted((k, v) for k, v in l.items() if k != "le")), len(keys)))
        les.append(le)
    return np.array([v for v, _ in ss]), np.array(gids, dtype=np.uint32), np.array(les), len(keys)


LIMIT_USED = [(100, "metric", "le", "inf", "x", "y"), (98, "metric", "le", "300", "x", "y"), (52, "metric", "le", "200", "x", "y"),
              (50, "metric", "le", "120", "x", "y"), (20, "metric", "le", "70", "x", "y"), (10, "metric", "le", "30", "x", "y"),
              (9, "metric", "le", "10", "x", "y")]


def test_exec_buckets_limit():  # exec_test.go:4836, 4845, 4886
    ss = labelled((100, "metric", "le", "inf", "x", "y"), (50, "metric", "le", "120", "x", "y"))
    assert V.buckets_limit_ref(0, *limit_inputs(ss)) == []
    assert V.buckets_limit_ref(5, *limit_inputs(ss)) == [0, 1]  # sort() then gives 50, 100
    ss = labelled(*LIMIT_USED)
    kept = V.buckets_limit_ref(2, *limit_inputs(ss))
    assert sorted(ss[r][1]["le"] for r in kept) == ["10", "300", "inf"]
    assert kept == [6, 1, 0]  # le order: 10, 300, inf


def test_buckets_limit_hand_worked():
    """les 1 ... 5, one point; hits are the bucket increments"""
    les = np.arange(1.0, 6.0)
    g = np.zeros(5, dtype=np.uint32)
    # hits 1 4 1 1 3: merge (2, 3) at index 2 first, then the pair at index 1
    assert V.buckets_limit_ref(3, np.array([[1.0], [5], [6], [7], [10]]), g, les, 1) == [0, 3, 4]
    # hits 1 1 8 NaN NaN: every sum with a NaN compares false, so index 1 goes twice
    assert V.buckets_limit_ref(1, np.array([[1.0], [2], [10], [NAN], [20]]), g, les, 1) == [0, 3, 4]
    # hits 1 8 1 10: merge index 2 (sum 11 > 9 at index 1 -> index 1)
    assert V.buckets_limit_ref(3, np.array([[1.0], [9], [10], [20]]), g[:4], les[:4], 1) == [0, 2, 3]
    assert V.buckets_limit_ref(-1, np.array([[1.0]]), g[:1], les[:1], 1) == []
    # groups at most the limit keep their input order
    assert V.buckets_limit_ref(3, np.array([[3.0], [1], [2]]), g[:3], np.array([3.0, 1, 2]), 1) == [0, 1, 2]


# ------------------------------------------------------------------------------------------------ the quirks, by hand
def walk(rows, P):
    """rows: [(vmrange, values)] of one group -> [(kind, le, values)]"""
    m = np.array([np.broadcast_to(np.asarray(v, dtype=np.float64), (P,)) for _, v in rows])
    out = V.vmrange_to_le_ref(m, [r for r, _ in rows], [None] * len(rows), [0] * len(rows))
    return [(k, le, list(v)) for _, k, le, v in out]


def test_equal_floats_different_strings_do_not_merge():
    assert walk([("0...1e2", 1), ("50...100", 2)], 1) == [
        (V.BUCKET, "1e2", [1]), (V.GAP, "50", [1]), (V.BUCKET, "100", [3]), (V.PINF, "+Inf", [3])]
    # the same strings merge (here refused: P <= 2), so the second row's value is gone
    assert walk([("0...100", 1), ("50...100", 2)], 1) == [(V.BUCKET, "100", [1]), (V.GAP, "50", [1]), (V.PINF, "+Inf", [1])]


def test_end_equal_to_earlier_start_merges_into_its_source_row():
    """7...3 opens a gap at 7 whose map entry names the 7...3 row itself; 1...7 then merges into that row (le 3), not into the
    zero gap row le=7"""
    got = walk([("7...3", [1, NAN, NAN]), ("1...7", [NAN, 4, NAN])], 3)
    assert got == [(V.GAP, "7", [0, 0, 0]), (V.BUCKET, "3", [1, 4, 0]), (V.GAP, "1", [1, 4, 0]), (V.PINF, "+Inf", [1, 4, 0])]


def test_a_to_a_after_a_gap_merges_into_itself_and_is_lost():
    assert walk([("3...3", [2, NAN, NAN])], 3) == [(V.GAP, "3", [0, 0, 0]), (V.PINF, "+Inf", [0, 0, 0])]
    assert walk([("0...0", [2, NAN, NAN])], 3) == [(V.BUCKET, "0", [2, 0, 0]), (V.PINF, "+Inf", [2, 0, 0])]  # no gap at 0


def test_merge_chain_counts_overlaps_against_the_merged_destination():
    """S1 fills points 1, 2 of D; S2 overlaps D at 1 point as D was, at 3 as S1 left it: refused"""
    rows = [("0...5", [1, NAN, NAN, NAN]), ("1...5", [NAN, 2, 3, NAN]), ("2...5", [4, 5, 6, NAN])]
    assert walk(rows, 4) == [(V.BUCKET, "5", [1, 2, 3, 0]), (V.GAP, "1", [1, 2, 3, 0]), (V.GAP, "2", [1, 2, 3, 0]),
                             (V.PINF, "+Inf", [1, 2, 3, 0])]
    # S2 first: 1 overlap, taken; then S1 overlaps the merged D at 2 points: taken too, and overwrites them
    rows = [("0...5", [1, NAN, NAN, NAN]), ("2...5", [4, 5, 6, NAN]), ("1...5", [NAN, 2, 3, NAN])]
    assert walk(rows, 4) == [(V.BUCKET, "5", [4, 2, 3, 0]), (V.GAP, "2", [4, 2, 3, 0]), (V.GAP, "1", [4, 2, 3, 0]),
                             (V.PINF, "+Inf", [4, 2, 3, 0])]
    rows = [("0...5", [1, NAN]), ("1...5", [NAN, 2])]  # P <= 2: never
    assert walk(rows, 2) == [(V.BUCKET, "5", [1, 0]), (V.GAP, "1", [1, 0]), (V.PINF, "+Inf", [1, 0])]


def test_inf_end_spellings_and_minus_inf_start():
    assert walk([("0...Inf", 2)], 1) == [(V.BUCKET, "Inf", [2])]
    assert walk([("0...inf", 2)], 1) == [(V.BUCKET, "inf", [2])]
    assert walk([("-Inf...1", 2)], 1) == [(V.GAP, "-Inf", [0]), (V.BUCKET, "1", [2]), (V.PINF, "+Inf", [2])]


def test_negative_and_nan_values_count_as_zero():
    assert walk([("0...1", [3, -2, NAN]), ("1...2", [1, 1, 1]), ("2...3", [-1, NAN, -5])], 3) == [
        (V.BUCKET, "1", [3, 0, 0]), (V.BUCKET, "2", [4, 1, 1]), (V.PINF, "+Inf", [4, 1, 1])]


def test_kept_le_rows_come_first_and_dropped_rows_vanish():
    m = np.array([[1.0], [2.0], [3.0], [4.0]])
    out = V.vmrange_to_le_ref(m, ["0...1", None, "x", None], [None, "0.5", None, ""], [0, 0, 0, 0])
    assert [(s, k, le) for s, k, le, _ in out] == [(1, V.KEPT, None), (0, V.BUCKET, "1"), (0, V.PINF, "+Inf")]


# ------------------------------------------------------------------------------------------------ go_parse_float
PARSE = [
    ("1", 1.0), ("-2.5", -2.5), ("+1e2", 100.0), (".5", 0.5), ("5.", 5.0), ("4.084e+02", 408.4), ("1E-3", 1e-3),
    (" 1", None), ("1 ", None), (" ", None), ("", None), (".", None), ("e5", None), ("1e", None), ("1e+", None), ("--1", None),
    ("1_0", 10.0), ("1_0.2_5e1_0", 10.25e10), ("_1", None), ("1_", None), ("1__0", None), ("1_.5", None), ("1._5", None),
    ("1e_5", None),
    ("0x1.8p1", 3.0), ("0X1P-2", 0.25), ("-0x.8p1", -1.0), ("0x_1p1", 2.0), ("0x1.8", None), ("0xp1", None), ("0x", None),
    ("0x1_p1", None),
    ("inf", INF), ("+Inf", INF), ("-inf", -INF), ("Infinity", INF), ("-INFINITY", -INF), ("iNfInItY", INF), ("infin", None),
    ("nan", NAN), ("NaN", NAN), ("NAN", NAN), ("+nan", None), ("-NaN", None),
    ("1e400", None), ("-1e400", None), ("0x1p1024", None), ("1e-400", 0.0), ("-1e-400", -0.0), ("1.7976931348623157e308", 1.7976931348623157e308),
]


@pytest.mark.parametrize("s,want", PARSE, ids=[repr(p[0]) for p in PARSE])
def test_go_parse_float(s, want):
    from victoriametrics_b200.promql import go_parse_float
    for f in (V.go_parse_float, go_parse_float):
        got = f(s)
        if want is None:
            assert got is None, (f.__module__, s, got)
        else:
            assert got is not None and np.float64(got).tobytes() == np.float64(want).tobytes(), (f.__module__, s, got)


def test_header_ids():
    from victoriametrics_b200 import promql
    h = open(os.path.join(ROOT, "include", "vmb200.h")).read()
    assert int(re.search(r"#define VMB_VR_KEEP (0x[0-9a-f]+)u", h).group(1), 16) == V.KEEP == promql.VR_KEEP
    body = re.search(r"enum vmb_vr_kind \{([^}]*)\}", h).group(1)
    names = [x.split("=")[0].strip() for x in body.split(",")]
    assert names == ["VMB_VR_KEPT", "VMB_VR_BUCKET", "VMB_VR_GAP", "VMB_VR_INF"]
    assert (V.KEPT, V.BUCKET, V.GAP, V.PINF) == (0, 1, 2, 3) and promql.VR_KINDS == ["kept", "bucket", "gap", "+Inf"]
