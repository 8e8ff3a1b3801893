"""Everything a query does after the rollup, bit for bit: binary and set operators, transforms, quantile / median by,
topk / bottomk, the incremental aggregates on every path, the subquery feed and mergeSeries.

The rule is assert_same_bits of tests/test_gpu_rollup_exact.py: NaN positions match and every other value has the same bits,
so -0.0 and +0.0 differ.  The references are restatements of the Go code in numpy float64 (IEEE: + - * / fmod sqrt and the
comparisons are exact there) or exact arithmetic (decimal at 60 digits, math.fsum).  EXCEPTIONS lists the only places where
a result may differ from its reference, each with its bound and reason.  Shapes go past the grid caps of the kernels, so
that the grid-stride loops run more than once.
"""
import ctypes as C
import math
import zlib
from decimal import Decimal, localcontext

import numpy as np
import pytest

import blockgen
from conftest import SEED0
from rollup_names import AGGR
from test_gpu_rollup_exact import TOLERANCE, assert_same_bits, block_rows, oracle_rows
from test_gpu_transform import _row_ref

pytestmark = pytest.mark.gpu
NAN, INF = float("nan"), float("inf")
DMAX = 1.7976931348623157e308
T0, DT = 1_700_000_000_000, 15000
SMS = 132                    # VMB_SMS (csrc/common.cuh)
ELEM_CAP = SMS * 32 * 256    # k_binary_op, k_transform_elem, k_merge_rows, k_group_first_value: cells per grid pass
ROWS_CAP = SMS * 16 * 4 * 32  # k_transform_rows: rows per grid pass
FEED_CAP = SMS * 16 * 4      # k_series_from_matrix: rows per grid pass
PI = Decimal("3.14159265358979323846264338327950288419716939937510582097494459")

# The only results allowed to differ from their reference.  "ulp": at most that many units in the last place of the reference.
# The CUDA bounds are the maximum ulp errors of the CUDA C++ Programming Guide, appendix "Mathematical Functions", table of
# double-precision functions; the glibc bounds are those of the GNU C Library manual, "Known Maximum Errors in Math Functions"
# (x86_64).  A reference computed in decimal at 60 digits is exact for this purpose, so the bound there is CUDA's alone.
# Largest errors measured on an H100 SXM (80 GB, 400 W): ^ 1.13, atan2 1.00, exp 0.74, ln 0.50, log2 1.18, log10 1.08, sin cos
# tan asin acos atan sinh cosh asinh 1.00, tanh acosh atanh 2.00.
EXCEPTIONS = {
    # binary operators and element transforms that go through CUDA's math library; Go computes them in pure Go
    "^": ("ulp", 2, "CUDA pow: 2 ulp; reference exp(y ln x) in decimal"),
    "atan2": ("ulp", 3, "CUDA atan2: 2 ulp, glibc atan2: 1 ulp"),
    "exp": ("ulp", 1, "CUDA exp: 1 ulp; reference in decimal"),
    "ln": ("ulp", 1, "CUDA log: 1 ulp; reference in decimal"),
    # CUDA documents 1 ulp for log2 and log10, but CUDA 12.9's log2 / log10 measured 1.18 / 1.08 ulp on an H100 (log2 at
    # 7.91686946584097e-231, log10 at 0.0001292109935148567).  The library's -fmad=false is not the cause: the same calls
    # compiled with and without it return the same bits.
    "log2": ("ulp", 2, "CUDA documents 1 ulp; 1.18 ulp measured on an H100; reference in decimal"),
    "log10": ("ulp", 2, "CUDA documents 1 ulp; 1.08 ulp measured on an H100; reference in decimal"),
    "sin": ("ulp", 3, "CUDA sin: 2 ulp, glibc sin: 1 ulp"),
    "cos": ("ulp", 3, "CUDA cos: 2 ulp, glibc cos: 1 ulp"),
    "tan": ("ulp", 3, "CUDA tan: 2 ulp, glibc tan: 1 ulp"),
    "asin": ("ulp", 3, "CUDA asin: 2 ulp, glibc asin: 1 ulp"),
    "acos": ("ulp", 3, "CUDA acos: 2 ulp, glibc acos: 1 ulp"),
    "atan": ("ulp", 3, "CUDA atan: 2 ulp, glibc atan: 1 ulp"),
    "sinh": ("ulp", 4, "CUDA sinh: 2 ulp, glibc sinh: 2 ulp"),
    "cosh": ("ulp", 3, "CUDA cosh: 1 ulp, glibc cosh: 2 ulp"),
    "tanh": ("ulp", 3, "CUDA tanh: 1 ulp, glibc tanh: 2 ulp"),
    "asinh": ("ulp", 5, "CUDA asinh: 3 ulp, glibc asinh: 2 ulp"),
    "acosh": ("ulp", 5, "CUDA acosh: 3 ulp, glibc acosh: 2 ulp"),
    "atanh": ("ulp", 4, "CUDA atanh: 2 ulp, glibc atanh: 2 ulp"),
    # -0.0 == +0.0, so which of them a sorted column holds at a tied rank is the sort's choice (Go's sort.Float64s is not
    # stable, the kernel ranks by counting): the rollup table's reason for quantile_over_time
    "quantile": ("zero sign", 0, TOLERANCE["quantile_over_time"][2]),
    # finalizeAggrGeomean: pow(prod, 1 / count)
    "geomean": TOLERANCE["geomean_over_time"],
    # the fused kernel folds by atomics in scheduling order (so does the reference, one partial state per worker): the sum
    # is within the worst-case error of recursive summation of the exact sum, (n - 1) u sum |v_i|, u = 2^-53
    "fused sum": ("order", 0, "atomicAdd order is scheduling dependent"),
    "fused avg": ("order", 0, "atomicAdd order is scheduling dependent; then one division"),
    "fused sum2": ("order", 0, "atomicAdd order is scheduling dependent; the squares are rounded one by one as in Go"),
    # fu_atomic_min / fu_atomic_max rank -0.0 below +0.0, so a cell whose values are all -0.0 keeps -0.0 (as the reference's
    # fold does); for a mix of the two zeros the result is the one the reference gets when that zero comes first, and which
    # comes first is scheduling dependent there too.  Blocks reach -0.0 through zscore_over_time of values near 1e300: the
    # standard deviation overflows to +Inf and (v - avg) / +Inf is -0.0 for v < avg.
    "fused min": ("zero sign", 0, "the order of equal zeros is scheduling dependent"),
    "fused max": ("zero sign", 0, "the order of equal zeros is scheduling dependent"),
}
ROLLUP_KEY = {"quantile": "quantile_over_time", "geomean": "geomean_over_time"}  # the same exception in the rollup table


def same_bits(got, exp, what, key=None):
    assert_same_bits(got, exp, what, ROLLUP_KEY.get(key))


def worst_ulps(ref_ulps, args):
    """ref_ulps: the error of every value in ulps of its reference (NaN where not measured) -> (largest error, its argument)"""
    e = np.where(np.isnan(ref_ulps), -1.0, ref_ulps)
    i = int(np.argmax(e))
    return float(max(e[i], 0.0)), args[i]


def assert_ulp_bounds(worst):
    """worst: {EXCEPTIONS key: (largest error, argument)}, printed first so that a run shows every function's error"""
    print("largest ulp error per function:", {k: "%.3f at %r" % w for k, w in worst.items()})
    over = {k: w for k, w in worst.items() if w[0] > EXCEPTIONS[k][1]}
    assert not over, "over the bound: %s" % {k: (w, EXCEPTIONS[k]) for k, w in over.items()}


def ulps_vs_decimal(got, exact):
    """|got - exact| in ulps of the double nearest to exact"""
    e = float(exact)
    return float(abs(Decimal(float(got)) - exact) / Decimal(math.ulp(e)))


def ulps_vs_double(got, ref):
    with np.errstate(all="ignore"):
        u = np.vectorize(math.ulp)(ref)
        d = np.abs(got - ref) / u
    d[(got == ref) | (np.isnan(got) & np.isnan(ref))] = 0.0
    return d


def seed(name, k=0):
    return np.random.default_rng(SEED0 + zlib.crc32(("matrix/%s/%d" % (name, k)).encode()))


class Buf:
    def __init__(self, nbytes):
        import torch
        self.t = torch.empty(max(nbytes // 8, 1), dtype=torch.float64, device="cuda")
        self.ptr = self.t.data_ptr()


@pytest.fixture(scope="module")
def vm():
    import victoriametrics_b200 as v
    return v


@pytest.fixture(scope="module")
def dev():
    """numpy -> device tensor and back"""
    import torch

    class D:
        @staticmethod
        def put(a):
            return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()

        @staticmethod
        def get(t):
            torch.cuda.synchronize()
            return t.cpu().numpy()

        @staticmethod
        def empty(*shape):
            return torch.full(shape, -7.0, dtype=torch.float64, device="cuda")
    return D


@pytest.fixture(scope="module")
def tctx(vm):
    ctx = vm.Context(0)
    ctx.enable_stage_timing(True)
    yield ctx
    ctx.close()


# ------------------------------------------------------------------------------------------------ 1. binary operators
SPECIALS = np.array([0.0, -0.0, INF, -INF, NAN, 5e-324, -5e-324, 2.2250738585072014e-308, -1e-310, DMAX, -DMAX, 1.0, -1.0,
                     0.5, 3.0, -2.5, 1e-200, -1e-200, 1e200, -7.0, 1e300])
EXACT_OPS = ["+", "-", "*", "/", "%", "==", "!=", ">", "<", ">=", "<=", "default", "if", "ifnot"]


def ref_binop(op, is_bool, a, b):
    """newBinaryOpFunc binary_op.go:155 with the element functions of metricsql/binaryop"""
    with np.errstate(all="ignore"):
        arith = {"+": np.add, "-": np.subtract, "*": np.multiply, "/": np.divide, "%": np.fmod}  # Go's math.Mod == C fmod
        if op in arith:
            return arith[op](a, b)
        if op == "default":
            return np.where(np.isnan(a), b, a)
        if op == "if":
            return np.where(np.isnan(b), NAN, a)
        if op == "ifnot":
            return np.where(np.isnan(b), a, NAN)
        an, bn = np.isnan(a), np.isnan(b)
        c = {"==": np.where(an, bn, a == b), "!=": np.where(an, ~bn, bn | (a != b)), ">": a > b, "<": a < b, ">=": a >= b,
             "<=": a <= b}[op]
        if not is_bool:
            return np.where(c, a, NAN)
        return np.where(an, NAN, np.where(c, 1.0, 0.0))


def operands(rng, shape):
    m = rng.normal(size=shape) * 10.0 ** rng.integers(-300, 300, shape)
    sel = rng.random(shape) < 0.3
    m[sel] = rng.choice(SPECIALS, int(sel.sum()))
    return m


def run_binop(vm, dev, op, L, R, npairs, P, lrows=None, rrows=None, is_bool=False):
    out = dev.empty(npairs, P)
    vm.promql.binary_op(op, L.data_ptr(), R.data_ptr(), npairs, P, out.data_ptr(), lrows, rrows, is_bool=is_bool)
    return dev.get(out)


@pytest.mark.parametrize("op", EXACT_OPS)
def test_binary_op_bit_exact(vm, dev, op):
    rng = seed(op)
    m = len(SPECIALS)
    pa, pb = np.repeat(SPECIALS, m)[None, :], np.tile(SPECIALS, m)[None, :]  # every pair of special operands
    for is_bool in (False, True):
        got = run_binop(vm, dev, op, dev.put(pa), dev.put(pb), 1, m * m, is_bool=is_bool)
        assert_same_bits(got, ref_binop(op, is_bool, pa, pb), "%s bool=%s special pairs" % (op, is_bool))
    S, P = 41, 211
    left, right = operands(rng, (S, P)), operands(rng, (S // 2 + 1, P))
    lrows, rrows = rng.integers(0, S, 60).astype(np.uint32), rng.integers(0, S // 2 + 1, 60).astype(np.uint32)
    L, R = dev.put(left), dev.put(right)
    for is_bool in (False, True):
        got = run_binop(vm, dev, op, L, R, 60, P, lrows, rrows, is_bool)
        assert_same_bits(got, ref_binop(op, is_bool, left[lrows], right[rrows]), "%s bool=%s row lists" % (op, is_bool))
        # vector op scalar (binary_op.go:218-227): the scalar is a one-row matrix, every pair reads row 0
        for s in (2.0, -0.0, 0.0, INF, NAN, 5e-324, -3.5):
            got = run_binop(vm, dev, op, L, dev.put(np.full((1, P), s)), S, P, None, np.zeros(S, dtype=np.uint32), is_bool)
            assert_same_bits(got, ref_binop(op, is_bool, left, np.full((S, P), s)), "%s bool=%s scalar %r" % (op, is_bool, s))


@pytest.mark.parametrize("op", ["/", "-", "<", "default"])
def test_binary_op_past_the_grid_cap(vm, dev, op):
    """npairs x points above one grid pass, prime point count: the grid-stride loop runs twice"""
    rng = seed(op, 1)
    npairs, P = 2003, 541
    assert npairs * P > ELEM_CAP
    left, right = operands(rng, (npairs, P)), operands(rng, (npairs, P))
    L, R = dev.put(left), dev.put(right)
    assert_same_bits(run_binop(vm, dev, op, L, R, npairs, P), ref_binop(op, False, left, right), op + " plain")
    lr, rr = rng.permutation(npairs).astype(np.uint32), rng.permutation(npairs).astype(np.uint32)
    assert_same_bits(run_binop(vm, dev, op, L, R, npairs, P, lr, rr, True), ref_binop(op, True, left[lr], right[rr]), op + " rows")


def odd_int(y):  # Go's isOddInt (math/pow.go)
    if abs(y) >= 2.0 ** 53 or not math.isfinite(y):
        return False
    return y == math.floor(y) and int(y) % 2 == 1


def go_pow_special(x, y):
    """the special cases of Go's math.Pow, in its order (math/pow.go); None where none applies.  binaryop.Pow first
    returns NaN for a NaN base (NaN ^ 0 included)."""
    if math.isnan(x):
        return NAN
    if y == 0 or x == 1:
        return 1.0
    if y == 1:
        return x
    if math.isnan(y):
        return NAN
    if x == 0:
        neg = math.copysign(1, x) < 0 and odd_int(y)
        return (-INF if neg else INF) if y < 0 else (x if neg else 0.0)
    if math.isinf(y):
        if x == -1:
            return 1.0
        return 0.0 if (abs(x) < 1) == (y > 0) else INF
    if math.isinf(x):
        if x < 0:
            return go_pow_special(-0.0, -y)
        return 0.0 if y < 0 else INF
    if x < 0 and y != math.floor(y):
        return NAN
    return None


def go_atan2_special(y, x):
    """the special cases of Go's math.Atan2 (math/atan2.go); None where none applies"""
    if math.isnan(y) or math.isnan(x):
        return NAN
    if y == 0:
        return math.copysign(0.0, y) if x >= 0 and math.copysign(1, x) > 0 else math.copysign(float(PI), y)
    if x == 0:
        return math.copysign(float(PI / 2), y)
    if math.isinf(x):
        if x > 0:
            return math.copysign(float(PI / 4), y) if math.isinf(y) else math.copysign(0.0, y)
        return math.copysign(float(3 * PI / 4), y) if math.isinf(y) else math.copysign(float(PI), y)
    if math.isinf(y):
        return math.copysign(float(PI / 2), y)
    return None


def test_pow_and_atan2(vm, dev):
    rng = seed("pow")
    sp = np.array([0.0, -0.0, INF, -INF, NAN, 1.0, -1.0, 0.5, -0.5, 2.0, -2.0, 3.0, -3.0, 1.5, -2.5, 0.25, 4.0, 1e-310, -7.0])
    m = len(sp)
    a, b = np.repeat(sp, m), np.tile(sp, m)
    for op, special in (("^", go_pow_special), ("atan2", lambda x, y: go_atan2_special(x, y))):
        got = run_binop(vm, dev, op, dev.put(a[None, :]), dev.put(b[None, :]), 1, m * m)[0]
        want = [special(float(x), float(y)) for x, y in zip(a, b)]
        k = np.array([w is not None for w in want])
        assert k.sum() > m * m // 3, op
        assert_same_bits(got[k], np.array([w for w in want if w is not None]), op + ": Go's special cases")
    # ordinary values: positive bases against exp(y ln x) at 60 digits
    n = 3000
    x = np.concatenate([10.0 ** rng.uniform(-8, 8, n - 600), 1 + rng.uniform(-1e-6, 1e-6, 300), rng.uniform(0.01, 10, 300)])
    y = rng.uniform(-30, 30, n)
    y[:200] = rng.integers(-20, 21, 200)  # integer exponents
    got = run_binop(vm, dev, "^", dev.put(x[None, :]), dev.put(y[None, :]), 1, n)[0]
    err = np.full(n, NAN)
    with localcontext() as c:
        c.prec = 60
        for i in range(n):
            e = (Decimal(float(y[i])) * Decimal(float(x[i])).ln()).exp()
            if Decimal("1e-300") < e < Decimal("1e300"):
                err[i] = ulps_vs_decimal(got[i], e)
    assert np.isfinite(err).sum() > n * 0.9
    worst = {"^": worst_ulps(err, list(zip(x, y)))}
    yy, xx = rng.normal(size=n) * 10.0 ** rng.integers(-5, 6, n), rng.normal(size=n) * 10.0 ** rng.integers(-5, 6, n)
    got = run_binop(vm, dev, "atan2", dev.put(yy[None, :]), dev.put(xx[None, :]), 1, n)[0]
    worst["atan2"] = worst_ulps(ulps_vs_double(got, np.array([math.atan2(p, q) for p, q in zip(yy, xx)])), list(zip(yy, xx)))
    assert_ulp_bounds(worst)


def ref_set_op(op, left, lg, right, rg):
    """binaryOpAnd / binaryOpUnless / binaryOpDefault (binary_op.go:430,610,463), restated loop by loop"""
    want = left.copy()
    for i in range(left.shape[0]):
        rows = np.nonzero(rg == lg[i])[0]
        for j in range(left.shape[1]):
            has = [right[r, j] for r in rows if not np.isnan(right[r, j])]
            if op in ("and", "if") and not has:
                want[i, j] = NAN
            if op in ("unless", "ifnot") and has:
                want[i, j] = NAN
            if op == "default" and np.isnan(want[i, j]) and has:
                want[i, j] = has[0]
    return want


@pytest.mark.parametrize("op", ["and", "unless", "default"])
def test_set_operators_edges(vm, dev, op):
    """right keys whose rows are all NaN, a key with one right row, -0.0 on both sides"""
    rng = seed(op, 2)
    P, G, nl, nr = 97, 12, 50, 40
    left, right = operands(rng, (nl, P)), operands(rng, (nr, P))
    left[rng.random(left.shape) < 0.3] = NAN
    right[rng.random(right.shape) < 0.5] = NAN
    rg = np.concatenate([np.arange(G), rng.integers(2, G, nr - G)]).astype(np.uint32)
    rng.shuffle(rg)
    right[rg == 0] = NAN                  # key 0: every right row NaN
    rg[rg == 1] = 2
    rg[np.nonzero(rg == 2)[0][0]] = 1     # key 1: one right row
    lg = rng.integers(0, G, nl).astype(np.uint32)
    lg[:6] = [0, 0, 1, 1, 1, 0]
    tmp, out, dl, dr = dev.empty(G, P), dev.empty(nl, P), dev.put(left), dev.put(right)
    vm.promql.set_op(op, dl.data_ptr(), lg, nl, dr.data_ptr(), rg, nr, G, P, out.data_ptr(), tmp.data_ptr())
    assert_same_bits(dev.get(out), ref_set_op(op, left, lg, right, rg), op)


# ------------------------------------------------------------------------------------------------ 2. transforms
def run_tf(vm, dev, name, m, *args):
    d = dev.put(m)
    vm.promql.transform(name, d.data_ptr(), m.shape[0], m.shape[1], *args)
    return dev.get(d)


def tf_values(rng, shape):
    m = rng.normal(scale=50.0, size=shape)
    sel = rng.random(shape) < 0.3
    m[sel] = rng.choice(np.array([0.0, -0.0, INF, -INF, NAN, 5e-324, -1e-310, DMAX, -DMAX, 2.5, -2.5, 0.5, -0.5, 1e300, 7.0]),
                        int(sel.sum()))
    return m


def go_round(v, nearest, p10):
    """transform.go:2341 round: the same four float operations, NaN in -> NaN out"""
    with np.errstate(all="ignore"):
        x = v + 0.5 * np.copysign(nearest, v)
        x = x - np.fmod(x, nearest)
        return np.trunc(x * p10) / p10


def test_element_transforms_bit_exact(vm, dev):
    rng = seed("elem")
    S, P = 61, 67
    m = tf_values(rng, (S, P))
    with np.errstate(all="ignore"):
        for name, want in (("abs", np.abs(m)), ("ceil", np.ceil(m)), ("floor", np.floor(m)), ("sqrt", np.sqrt(m)),
                           ("deg", m * 180.0 / float(PI)), ("rad", m * float(PI) / 180.0),
                           ("sgn", np.where(m < 0, -1.0, np.where(m > 0, 1.0, 0.0)))):  # sgn(NaN) = 0 (transform.go:2362)
            assert_same_bits(run_tf(vm, dev, name, m), want, name)
    # per-point arguments: -0.0 / +0.0 bounds, NaN bounds, crossed bounds
    a1 = rng.choice(np.array([-0.0, 0.0, NAN, -10.0, 3.0, -INF, 5e-324]), P)
    a2 = rng.choice(np.array([-0.0, 0.0, NAN, 10.0, -3.0, INF, -5e-324]), P)
    assert_same_bits(run_tf(vm, dev, "clamp", m, a1, a2), np.where(m > a2, a2, np.where(m < a1, a1, m)), "clamp")  # :283
    assert_same_bits(run_tf(vm, dev, "clamp_min", m, a1), np.where(m < a1, a1, m), "clamp_min")
    assert_same_bits(run_tf(vm, dev, "clamp_max", m, a2), np.where(m > a2, a2, m), "clamp_max")
    # round(q, nearest) per point; math.Pow10(-e) of decimal.FromFloat(nearest) is the literal 1e-e for these
    near = np.array([1.0, 0.1, 0.25, 5.0, 100.0, 0.003, 2.0, 0.5])
    exps = {1.0: 0, 0.1: -1, 0.25: -2, 5.0: 0, 100.0: 2, 0.003: -3, 2.0: 0, 0.5: -1}
    nr = near[np.arange(P) % len(near)]
    p10 = np.array([float("1e%d" % -exps[n]) for n in nr])
    mr = rng.normal(scale=300.0, size=(S, P))
    mr[:, :6] = [[-0.0, 0.0, 0.5, -0.5, 2.5, -2.5]] * S
    mr[rng.random(mr.shape) < 0.1] = NAN
    assert_same_bits(run_tf(vm, dev, "round", mr, nr), go_round(mr, nr, p10), "round")


def test_element_transform_past_the_grid_cap(vm, dev):
    """per-point arguments read with the point index of every grid pass"""
    rng = seed("elem", 1)
    S, P = 2003, 541
    assert S * P > ELEM_CAP
    m = rng.normal(scale=10.0, size=(S, P))
    lo, hi = rng.normal(size=P) - 5, rng.normal(size=P) + 5
    assert_same_bits(run_tf(vm, dev, "clamp", m, lo, hi), np.where(m > hi, hi, np.where(m < lo, lo, m)), "clamp")
    assert_same_bits(run_tf(vm, dev, "sqrt", np.abs(m)), np.sqrt(np.abs(m)), "sqrt")


MATH_FUNCS = {"sin": math.sin, "cos": math.cos, "tan": math.tan, "asin": math.asin, "acos": math.acos, "atan": math.atan,
              "sinh": math.sinh, "cosh": math.cosh, "tanh": math.tanh, "asinh": math.asinh, "acosh": math.acosh,
              "atanh": math.atanh}


def test_math_library_transforms_within_ulp_bounds(vm, dev):
    """exp / ln / log2 / log10 against decimal at 60 digits; the trigonometric and hyperbolic functions against the CPU's libm
    through Python's math module (glibc; numpy's SIMD loops have bounds of their own); special arguments exactly"""
    rng = seed("math")
    n = 2000
    worst = {}
    with localcontext() as c:
        c.prec = 60
        ln2, ln10 = Decimal(2).ln(), Decimal(10).ln()
        for name in ("exp", "ln", "log2", "log10"):
            x = rng.uniform(-700, 700, n) if name == "exp" else 10.0 ** rng.uniform(-300, 300, n)
            if name != "exp":
                x[:100] = 1 + rng.uniform(-1e-3, 1e-3, 100)
            got = run_tf(vm, dev, name, x[None, :])[0]
            ex = {"exp": lambda d: d.exp(), "ln": lambda d: d.ln(), "log2": lambda d: d.ln() / ln2, "log10": lambda d: d.log10()}[name]
            err = np.array([ulps_vs_decimal(g, ex(Decimal(float(v)))) if float(v) != 1.0 else (0.0 if g == 0 else INF)
                            for g, v in zip(got, x)])
            worst[name] = worst_ulps(err, x)
    for name, fn in MATH_FUNCS.items():
        x = rng.normal(scale=3.0, size=n) * 10.0 ** rng.integers(-3, 3, n)
        if name in ("asin", "acos", "atanh"):
            x = np.tanh(x)
            x[np.abs(x) >= 1] = 0.5
        elif name == "acosh":
            x = 1.0 + np.abs(x)
        elif name in ("sinh", "cosh"):
            x = np.clip(x, -700, 700)
        got = run_tf(vm, dev, name, x[None, :])[0]
        worst[name] = worst_ulps(ulps_vs_double(got, np.array([fn(v) for v in x])), x)
    assert_ulp_bounds(worst)
    # special arguments: the C99 / Go values are the same for these
    with np.errstate(all="ignore"):
        for name, fn in (("exp", np.exp), ("ln", np.log), ("log2", np.log2), ("log10", np.log10), ("sin", np.sin),
                         ("tan", np.tan), ("atan", np.arctan), ("sinh", np.sinh), ("tanh", np.tanh), ("asinh", np.arcsinh),
                         ("atanh", np.arctanh)):
            sp = np.array([[0.0, -0.0, INF, -INF, NAN] + ([1.0] if name in ("ln", "log2", "log10", "atanh") else [])])
            want = fn(sp)
            assert_same_bits(run_tf(vm, dev, name, sp), want, name + " special arguments")


ROW_FUNCS = ["running_sum", "running_min", "running_max", "running_avg", "range_sum", "range_min", "range_max", "range_avg",
             "range_first", "range_last", "keep_last_value", "keep_next_value", "remove_resets", "interpolate"]


def row_matrix(rng, name, rows, points):
    m = rng.normal(scale=50.0, size=(rows, points))
    m[rng.random(m.shape) < 0.25] = NAN
    sel = rng.random(m.shape) < 0.05
    m[sel] = rng.choice(np.array([0.0, -0.0, -1e-310]), int(sel.sum()))
    if name == "remove_resets":
        m = np.abs(np.cumsum(rng.normal(scale=5.0, size=(rows, points)) ** 2, axis=1))
        for r in range(rows):
            k = int(rng.integers(0, points))
            m[r, k:] -= m[r, k] * float(rng.choice([1.0, 0.05]))
        m[rng.random(m.shape) < 0.2] = NAN
    for r in range(rows):
        if points > 40 and r % 3 == 0:  # a gap over two or more 32-point tiles
            a = int(rng.integers(1, points - 36))
            m[r, a:a + int(rng.integers(34, min(points - a, 80)))] = NAN
        if r % 5 == 1:
            m[r, :int(rng.integers(0, points + 1))] = NAN   # leading NaNs
        if r % 7 == 2:
            m[r, int(rng.integers(0, points)):] = NAN       # trailing NaNs
    m[rows // 2] = NAN
    if rows > 3:
        m[1] = -0.0 if points > 1 else m[1]                 # signed zeros all the way
    if points >= 72:  # one gap that surely crosses two tile boundaries: values at 4 and 71, NaN at 5..70
        m[0, 4], m[0, 5:71], m[0, 71] = 1.5, NAN, -2.25
    return m


@pytest.mark.parametrize("name", ROW_FUNCS)
def test_row_transforms_bit_exact(vm, dev, name):
    rng = seed(name)
    for rows in (31, 32, 33):
        for points in (1, 31, 32, 33, 64, 65, 97):
            m = row_matrix(rng, name, rows, points)
            want = np.stack([_row_ref(name, m[r]) for r in range(rows)])
            assert_same_bits(run_tf(vm, dev, name, m), want, "%s %dx%d" % (name, rows, points))


def ref_rows_vectorized(name, m):
    """running_sum / running_avg / keep_next_value / range_last for many rows at once: the loops of _row_ref, a column at a time"""
    v = m.copy()
    R, P = v.shape
    if name == "keep_next_value":
        nxt = v[:, -1].copy()
        for j in range(P - 1, -1, -1):
            nn = np.isnan(v[:, j])
            nxt = np.where(nn, nxt, v[:, j])
            v[:, j] = nxt
        return v
    if name == "range_last":
        last = np.full(R, NAN)
        for j in range(P):
            last = np.where(np.isnan(v[:, j]), last, v[:, j])
        return np.where(np.isnan(last)[:, None], v, last[:, None])
    started, prev, i0 = np.zeros(R, bool), np.zeros(R), np.zeros(R, np.int64)
    for j in range(P):
        x = v[:, j]
        first = ~started & ~np.isnan(x)
        upd = started & ~np.isnan(x)
        if name == "running_sum":
            nv = prev + x
        else:
            nv = prev + (x - prev) / (j - i0 + 1).astype(np.float64)
        prev = np.where(first, x, np.where(upd, nv, prev))
        i0 = np.where(first, j, i0)
        started |= first
        v[:, j] = np.where(started, prev, x)
    return v


@pytest.mark.parametrize("name", ["running_sum", "running_avg", "keep_next_value", "range_last"])
def test_row_transforms_past_the_grid_cap(vm, dev, name):
    rng = seed(name, 1)
    rows, points = ROWS_CAP + 77, 3
    m = rng.normal(scale=50.0, size=(rows, points))
    m[rng.random(m.shape) < 0.3] = NAN
    m[rng.random(m.shape) < 0.05] = -0.0
    want = ref_rows_vectorized(name, m)
    chk = rng.integers(0, rows, 300)
    assert_same_bits(want[chk], np.stack([_row_ref(name, m[r]) for r in chk]), "vectorized reference " + name)
    assert_same_bits(run_tf(vm, dev, name, m), want, "%s %d rows" % (name, rows))


# ------------------------------------------------------------------------------------------------ 3. quantile / median by
def quantile_sorted(phi, a):
    """quantileSorted aggr.go:922 on a sorted column without NaNs"""
    if len(a) == 0 or math.isnan(phi):
        return NAN
    if phi < 0:
        return -INF
    if phi > 1:
        return INF
    n = float(len(a))
    rank = phi * (n - 1)
    lower = max(0.0, math.floor(rank))
    upper = min(n - 1, lower + 1)
    weight = rank - math.floor(rank)
    return float(a[int(lower)]) * (1 - weight) + float(a[int(upper)]) * weight


def ref_quantile(vals, groups, G, phis):
    out = np.empty((G, vals.shape[1]))
    for g in range(G):
        rows = np.nonzero(groups == g)[0]
        for p in range(vals.shape[1]):
            col = vals[rows, p]
            out[g, p] = quantile_sorted(phis[p], np.sort(col[~np.isnan(col)]))
    return out


def run_quantile(vm, dev, vals, groups, G, phis):
    out, dv = dev.empty(G, vals.shape[1]), dev.put(vals)
    vm.promql.aggr_quantile(phis, dv.data_ptr(), vals.shape[0], vals.shape[1], out.data_ptr(), groups, G)
    return dev.get(out)


def test_quantile_by_bit_exact(vm, dev):
    """groups of 1, 2, 3, 4, 5, 9 and 40 series; phi at the "top two" fast path (n - 1 - floor(phi (n - 1)) <= 1), the "top four"
    and "bottom four" paths and the general rank selection; 0, 1, exact ranks, < 0, > 1, NaN; columns with and without NaNs,
    ties, signed zeros and infinities"""
    rng = seed("quantile")
    sizes = [1, 2, 3, 4, 5, 9, 40, 40]
    G = len(sizes)
    groups = np.repeat(np.arange(G), sizes).astype(np.uint32)
    rng.shuffle(groups)
    S = len(groups)
    phis = np.array([0.0, 1.0, 0.5, 0.99, 0.999, 0.9, 0.75, 0.7, 0.6, 0.25, 0.1, 0.01, 0.05, 1 / 3, 2 / 3, 1 / 39, 38 / 39,
                     36 / 39, 35 / 39, 3 / 39, 4 / 39, 0.125, 7 / 8, -0.5, 1.5, NAN, 1e-300, -0.0])
    phis = np.tile(phis, 4)
    P = len(phis)
    vals = rng.integers(-3, 4, (S, P)).astype(np.float64) * rng.choice([1.0, 0.5, 1e300], (S, P))
    sel = rng.random((S, P)) < 0.1
    vals[sel] = rng.choice(np.array([-0.0, INF, -INF, 5e-324]), int(sel.sum()))
    vals[:, P // 2:][rng.random((S, P - P // 2)) < 0.2] = NAN  # the second half: columns with NaNs
    vals[:, 5] = NAN
    same_bits(run_quantile(vm, dev, vals, groups, G, phis), ref_quantile(vals, groups, G, phis), "quantile", "quantile")
    cont = rng.normal(size=(S, P))  # no ties: the exact interpolation
    same_bits(run_quantile(vm, dev, cont, groups, G, phis), ref_quantile(cont, groups, G, phis), "quantile continuous")
    med = np.full(P, 0.5)
    same_bits(run_quantile(vm, dev, cont, groups, G, med), ref_quantile(cont, groups, G, med), "median")


def test_quantile_group_cap(vm, dev):
    """VMB_QUANTILE_MAX_GROUP = 2048 series per group: 2048 works, 2049 is VMB_ERR_CAP"""
    rng = seed("quantile", 1)
    vals = rng.normal(size=(2049, 3))
    phis = np.array([0.5, 0.99, 0.01])
    g = np.zeros(2048, dtype=np.uint32)
    assert_same_bits(run_quantile(vm, dev, vals[:2048], g, 1, phis), ref_quantile(vals[:2048], g, 1, phis), "2048 series")
    with pytest.raises(vm.VmbError) as ei:
        run_quantile(vm, dev, vals, np.zeros(2049, dtype=np.uint32), 1, phis)
    assert ei.value.code == -54


# ------------------------------------------------------------------------------------------------ 4. incremental aggregates
AGGRS = ["sum", "min", "max", "avg", "count", "sum2", "geomean", "any", "group"]


def oracle_fold(oracle, aggr, rows, groups, G, P, finalize=True):
    """updateTimeseries for every row in ascending series order (one reference worker), then finalize"""
    v, c = np.zeros((G, P)), np.zeros((G, P))
    for s in range(rows.shape[0]):
        r = np.ascontiguousarray(rows[s])
        g = int(groups[s])
        oracle.lib().vmo_aggr_update(AGGR[aggr], v[g].ctypes.data_as(oracle.f64p), c[g].ctypes.data_as(oracle.f64p),
                                     r.ctypes.data_as(oracle.f64p), P)
    if finalize:
        oracle_finalize(oracle, aggr, v, c)
    return v, c


def oracle_finalize(oracle, aggr, v, c):
    for g in range(v.shape[0]):
        oracle.lib().vmo_aggr_finalize(AGGR[aggr], v[g].ctypes.data_as(oracle.f64p), c[g].ctypes.data_as(oracle.f64p), v.shape[1])


def agg_blocks(rng, n, rows=400, regular=False):
    """gauges and counters, a few all-NaN stretches (series that start late), signed values"""
    out = []
    for i in range(n):
        kind = ["gauge", "gauge_small", "counter", "gauge_wide"][i % 4]
        v = blockgen.gen_values(rng, kind, rows)
        if i % 2:
            v = -v
        ts = blockgen.gen_timestamps(rng, "regular" if regular or i % 3 else "jitter", rows, T0 + (0 if i % 5 else 900_000))
        out.append(blockgen.OBlock(ts, v, int(rng.choice([-2, 0, 3])), 64, i))
    return out


def agg_cfg(vm, func):
    return vm.promql.get_rollup_configs(func, T0 + 300_000, T0 + DT * 399, 30_000, 120_000)


def check_aggr(got, want, what, aggr):
    same_bits(got, want, what, aggr)


@pytest.mark.parametrize("aggr", AGGRS)
def test_aggregate_fold_unfused_and_host_series(vm, oracle, tctx, aggr):
    """k_aggr_fold: the un-fused device aggregate and host series through vmb_rollup_aggr_partial, against a sequential fold
    in ascending series order"""
    rng = seed(aggr)
    blocks = agg_blocks(rng, 45)
    G = 6
    groups = rng.integers(0, G, len(blocks)).astype(np.uint32)
    groups[:3] = [5, 5, 5]
    rc = agg_cfg(vm, "avg_over_time")
    want = oracle_fold(oracle, aggr, oracle_rows(oracle, rc, block_rows(blocks))[0], groups, G, rc.points)[0]
    descs, payload = blockgen.to_blockset(blocks)
    B = vm.storage.Blocks(descs, payload, tctx)
    tctx.set_fused(False)
    try:
        ia = vm.promql.IncrementalAggr(aggr, G, rc.points, Buf)
        ia.update_blocks(B, rc, groups)
        check_aggr(ia.finalize(tctx), want, "device aggregate, un-fused [%s]" % aggr, aggr)
    finally:
        tctx.set_fused(True)
        B.close()
    # host rows: -0.0 and +0.0 in the same cells, -0.0 alone, infinities, subnormals
    n, S = 60, 24
    ts_list = [(T0 + DT * np.arange(n)).astype(np.int64)] * S
    v_list = []
    for s in range(S):
        v = np.round(rng.normal(0, 3, n), 1)
        sel = rng.random(n) < 0.3
        v[sel] = rng.choice(np.array([-0.0, 0.0, -0.0, INF, -INF, 5e-324, -5e-324, NAN]), int(sel.sum()))
        if s % 4 == 0:
            v[:] = -0.0
        v_list.append(v)
    hg = (np.arange(S) % 4).astype(np.uint32)  # group 0: -0.0 only
    rc = vm.promql.get_rollup_configs("last_over_time", T0, T0 + DT * (n - 1), DT, DT)
    want = oracle_fold(oracle, aggr, oracle_rows(oracle, rc, list(zip(ts_list, v_list)))[0], hg, 4, rc.points)[0]
    series = vm.storage.Series.from_host(ts_list, v_list, tctx)
    try:
        ia = vm.promql.IncrementalAggr(aggr, 4, rc.points, Buf)
        ia.update(series, rc, hg)
        got = ia.finalize(tctx)
    finally:
        series.close()
    check_aggr(got, want, "host series [%s]" % aggr, aggr)
    if aggr in ("min", "max"):
        assert np.signbit(got[0]).all() and (got[0] == 0).all(), "a group of -0.0 rows folds to -0.0"


@pytest.mark.parametrize("aggr", AGGRS)
def test_aggregate_chunked_host_pipeline(vm, oracle, monkeypatch, aggr):
    """vmb_eval_rollup_aggr_host_partial with chunks of 7 series: each chunk is folded in ascending order and the chunk
    partials are merged in chunk order (aggr_incremental.go's merge of per-worker states)"""
    rng = seed(aggr, 1)
    blocks = agg_blocks(rng, 40)
    G, CH = 5, 7
    groups = rng.integers(0, G, len(blocks)).astype(np.uint32)
    rc = agg_cfg(vm, "avg_over_time")
    rows = oracle_rows(oracle, rc, block_rows(blocks))[0]
    P = rc.points
    tv, tc = np.zeros((G, P)), np.zeros((G, P))
    seen = set()
    for c0 in range(0, len(blocks), CH):
        cv, cc = oracle_fold(oracle, aggr, rows[c0:c0 + CH], groups[c0:c0 + CH], G, P, finalize=False)
        for g in set(groups[c0:c0 + CH].tolist()):
            if g not in seen:  # finalizeTimeseries: the first partial state of a group is taken as it is
                seen.add(g)
                tv[g], tc[g] = cv[g], cc[g]
                continue
            oracle.lib().vmo_aggr_merge(AGGR[aggr], tv[g].ctypes.data_as(oracle.f64p), tc[g].ctypes.data_as(oracle.f64p),
                                        cv[g].ctypes.data_as(oracle.f64p), cc[g].ctypes.data_as(oracle.f64p), P)
    oracle_finalize(oracle, aggr, tv, tc)
    descs, payload = blockgen.to_blockset(blocks)
    ctx = vm.default_context()
    monkeypatch.setenv("VMB_PIPE_CHUNK_BLOCKS", str(CH))
    ia = vm.promql.IncrementalAggr(aggr, G, P, Buf)
    ia.update_host(descs, payload, rc, groups, ctx)
    check_aggr(ia.finalize(ctx), tv, "chunked host pipeline [%s]" % aggr, aggr)


@pytest.mark.parametrize("aggr", ["sum", "avg", "sum2", "count", "group", "min", "max"])
def test_aggregate_fused_atomic_fold(vm, oracle, tctx, aggr):
    """the fold inside the fused kernel: sum / avg / sum2 within the error bound of recursive summation of the exact sum; count,
    group, min and max exact.  Groups hold pairs v, -v that cancel."""
    rng = seed(aggr, 2)
    base = agg_blocks(rng, 24, regular=True)
    blocks = []
    for b in base:  # every series and its negation, in the same group
        for sgn in (1, -1):
            blocks.append(blockgen.OBlock(b.ts, sgn * b.vals, b.scale, 64, len(blocks)))
    G = 5
    groups = (np.arange(len(blocks)) // 2 % G).astype(np.uint32)
    groups[[3, 8, 13]] = 4  # a group without exact cancellation
    rc = agg_cfg(vm, "last_over_time")
    rows = oracle_rows(oracle, rc, block_rows(blocks))[0]
    descs, payload = blockgen.to_blockset(blocks)
    B = vm.storage.Blocks(descs, payload, tctx)
    try:
        ia = vm.promql.IncrementalAggr(aggr, G, rc.points, Buf)
        ia.update_blocks(B, rc, groups)
        st = tctx.stage_ms()
        got = ia.finalize(tctx)
    finally:
        B.close()
    assert st[5] > 0 and st[1] == 0, ("the fused kernel did not fold every series", st)
    want = oracle_fold(oracle, aggr, rows, groups, G, rc.points)[0]
    if aggr in ("count", "group", "min", "max"):
        assert_same_bits(got, want, "fused [%s]" % aggr)
        return
    assert np.array_equal(np.isnan(got), np.isnan(want)), aggr
    u = 2.0 ** -53
    for g in range(G):
        for p in range(rc.points):
            col = rows[groups == g, p]
            col = col[~np.isnan(col)]
            if not len(col):
                continue
            terms = col * col if aggr == "sum2" else col
            n, A, exact = len(terms), float(np.sum(np.abs(terms))), math.fsum(terms)
            bound = (n - 1) * u * A
            if aggr == "avg":  # the sum's bound over n, and the division's own rounding
                exact, bound = exact / n, bound / n + u * abs(exact / n) * 2
            assert abs(got[g, p] - exact) <= bound * (1 + 4 * n * u), (aggr, g, p, got[g, p], exact, bound)


def zero_rank_extreme(col, take_max):
    """min / max under the total order of fu_atomic_min / max: -0.0 just below +0.0"""
    key = [(v, 0 if math.copysign(1, v) < 0 else 1) for v in col]
    return col[key.index(max(key) if take_max else min(key))]


@pytest.mark.parametrize("aggr", ["min", "max"])
def test_aggregate_fused_min_max_signed_zeros(vm, oracle, tctx, aggr):
    """zscore_over_time of values near 1e300 is +-0.0 (the standard deviation overflows): groups whose cells are all -0.0 must
    fold to -0.0 in the fused kernel, as in the reference; a group that mixes the zeros takes the zero-sign exception"""
    pats = [[1, 2, -3, 2, 1, -1, 0] * 6, [5, 5, 5, -5, 5, 5, 5] * 6]
    blocks = []
    for k in range(9):  # groups 0 and 1: one pattern each; group 2: both
        v = np.array(pats[k % 2], dtype=np.int64)
        blocks.append(blockgen.OBlock((T0 + DT * np.arange(len(v))).astype(np.int64), v, 290, 64, k))
    groups = np.array([0, 1, 0, 1, 0, 1, 2, 2, 2], dtype=np.uint32)
    G = 3
    rc = vm.promql.get_rollup_configs("zscore_over_time", T0 + 60_000, T0 + DT * 41, DT, 60_000)
    rows = oracle_rows(oracle, rc, block_rows(blocks))[0]
    fin = ~np.isnan(rows)
    assert (rows[fin] == 0).all() and np.signbit(rows[fin]).any() and (~np.signbit(rows[fin])).any()
    descs, payload = blockgen.to_blockset(blocks)
    B = vm.storage.Blocks(descs, payload, tctx)
    try:
        ia = vm.promql.IncrementalAggr(aggr, G, rc.points, Buf)
        ia.update_blocks(B, rc, groups)
        st = tctx.stage_ms()
        got = ia.finalize(tctx)
    finally:
        B.close()
    assert st[5] > 0 and st[1] == 0, ("the fused kernel did not fold every series", st)
    want = oracle_fold(oracle, aggr, rows, groups, G, rc.points)[0]
    assert_same_bits(got[:2], want[:2], "fused %s, one zero sign per cell" % aggr)
    assert np.signbit(want[:2][want[:2] == 0]).any(), "no cell of -0.0 only"
    # the mixed group: EXCEPTIONS["fused min" / "fused max"] -- equal to the reference's fold up to the sign of a zero, and
    # exactly the extreme under -0.0 < +0.0
    assert np.array_equal(got[2], want[2], equal_nan=True), aggr
    for p in range(rc.points):
        col = rows[groups == 2, p]
        col = col[~np.isnan(col)]
        exp = zero_rank_extreme(col, aggr == "max") if len(col) else NAN
        assert_same_bits(got[2, p], exp, "fused %s, mixed zeros, point %d" % (aggr, p))


# ------------------------------------------------------------------------------------------------ 5. topk / bottomk
def ref_topk(vals, ks, groups, reverse):
    """newAggrFuncTopK: per point the kn = getIntK(k, len(group)) best values survive; equal values (-0.0 == +0.0) rank by
    ascending series id"""
    out = np.full_like(vals, NAN)
    S, P = vals.shape
    for g in np.unique(groups):
        rows = np.nonzero(groups == g)[0]
        for p in range(P):
            k = ks[p]
            kn = 0 if (math.isnan(k) or k < 0) else (len(rows) if k >= len(rows) else int(k))
            live = [r for r in rows if not math.isnan(vals[r, p])]
            live.sort(key=lambda r: ((vals[r, p] if reverse else -vals[r, p]), r))
            for r in live[:kn]:
                out[r, p] = vals[r, p]
    return out, ~np.all(np.isnan(out), axis=1)


def run_topk(vm, dev, vals, ks, groups, G, reverse):
    t = dev.put(vals)
    keep = vm.promql.topk(ks, t.data_ptr(), vals.shape[0], vals.shape[1], Buf, group_ids=groups, ngroups=G, reverse=reverse)
    return dev.get(t), keep


@pytest.mark.parametrize("reverse", [False, True])
def test_topk_ties_and_edges(vm, dev, reverse):
    rng = seed("topk", reverse)
    sizes = [1, 2, 5, 6, 64, 65, 30]
    G = len(sizes)
    groups = np.repeat(np.arange(G), sizes).astype(np.uint32)
    rng.shuffle(groups)
    S = len(groups)
    ks = np.array([0, 1, 2, 2.9, -1, NAN, 5, 6, 7, 64, 30, 31, 0.5, -0.0, 3, 63.5, 64, 4, 1, 65 - 1e-12])
    P = len(ks) * 3
    ks = np.tile(ks, 3)
    vals = rng.integers(-2, 3, (S, P)).astype(np.float64)
    sel = rng.random((S, P)) < 0.25
    vals[sel] = rng.choice(np.array([-0.0, 0.0, INF, -INF, NAN]), int(sel.sum()))
    vals[:, 7] = np.where(np.arange(S) % 2, -0.0, 0.0)  # a column of zeros of both signs only
    got, keep = run_topk(vm, dev, vals, ks, groups, G, reverse)
    want, wkeep = ref_topk(vals, ks, groups, reverse)
    assert_same_bits(got, want, "topk reverse=%s" % reverse)
    assert keep.tolist() == wkeep.tolist()
    with pytest.raises(ValueError):
        run_topk(vm, dev, vals, np.full(P, 65.0), groups, G, reverse)  # 65 > 64 = the largest kmax


def test_topk_apply_checks_k_against_kmax(vm, dev):
    """vmb_topk_apply reads entry kn - 1 of a (group, point) list; k > kmax with a group larger than kmax is an invalid argument,
    and the matrix is left as it was.  The candidate buffer is several lists longer than needed, so that reading past a list
    stays inside the allocation."""
    from victoriametrics_b200 import _lib
    rng = seed("topk", 3)
    S, P, G, KMAX = 10, 8, 1, 2
    vals = rng.normal(size=(S, P))
    t = dev.put(vals)
    cand = Buf(G * P * KMAX * 16 * 8)
    ctx = vm.default_context()
    g = np.zeros(S, dtype=np.uint32)
    gs = np.array([S], dtype=np.uint32)
    _lib.check(_lib.lib().vmb_topk_candidates(ctx.h, C.c_void_p(t.data_ptr()), S, P, g.ctypes.data_as(_lib.u32p), G, KMAX, 0, 0,
                                              C.c_void_p(cand.ptr)))
    flags = np.zeros(S, dtype=np.uint8)
    for k in (3.0, 9.5, 1e300):
        ks = np.full(P, KMAX * 1.0)
        ks[P - 1] = k
        rc = _lib.lib().vmb_topk_apply(ctx.h, C.c_void_p(t.data_ptr()), S, P, g.ctypes.data_as(_lib.u32p), G,
                                       gs.ctypes.data_as(_lib.u32p), C.c_void_p(cand.ptr), KMAX, ks.ctypes.data_as(_lib.f64p), 0,
                                       0, flags.ctypes.data_as(_lib.u8p))
        assert rc == -50, k
        assert_same_bits(dev.get(t), vals, "matrix after the refused call")
    ks = np.array([KMAX, 2.9, 0, NAN, -1, 1, 2, 2.0])  # floor(2.9) = 2 <= kmax
    rc = _lib.lib().vmb_topk_apply(ctx.h, C.c_void_p(t.data_ptr()), S, P, g.ctypes.data_as(_lib.u32p), G,
                                   gs.ctypes.data_as(_lib.u32p), C.c_void_p(cand.ptr), KMAX, ks.ctypes.data_as(_lib.f64p), 0, 0,
                                   flags.ctypes.data_as(_lib.u8p))
    assert rc == 0
    assert_same_bits(dev.get(t), ref_topk(vals, ks, g, False)[0], "k <= kmax")


def test_topk_two_shards_with_ties_across_them(vm, dev):
    from victoriametrics_b200 import _lib
    rng = seed("topk", 4)
    S, P, G, K = 120, 40, 3, 6
    vals = rng.integers(0, 3, (S, P)).astype(np.float64)
    vals[rng.random((S, P)) < 0.3] = -0.0
    vals[rng.random((S, P)) < 0.05] = NAN
    groups = (np.arange(S) % G).astype(np.uint32)
    ks = rng.choice(np.array([0.0, 1, 2, 3, 5, 6]), P)
    ctx = vm.default_context()
    shards = [np.arange(0, S // 2), np.arange(S // 2, S)]  # global series id = row index
    gsz = np.bincount(groups, minlength=G).astype(np.uint32)
    import torch
    cands, devs = [], []
    for base, rows in zip((0, S // 2), shards):
        t = dev.put(vals[rows])
        c = torch.empty(G * P * K * 2, dtype=torch.float64, device="cuda")
        g = np.ascontiguousarray(groups[rows])
        _lib.check(_lib.lib().vmb_topk_candidates(ctx.h, C.c_void_p(t.data_ptr()), len(rows), P, g.ctypes.data_as(_lib.u32p), G,
                                                  K, 0, base, C.c_void_p(c.data_ptr())))
        cands.append(c)
        devs.append((t, g, base))
    gathered = torch.cat(cands)
    merged = torch.empty(G * P * K * 2, dtype=torch.float64, device="cuda")
    _lib.check(_lib.lib().vmb_topk_merge(ctx.h, C.c_void_p(gathered.data_ptr()), 2, G * P, K, 0, C.c_void_p(merged.data_ptr())))
    got = np.empty_like(vals)
    for rows, (t, g, base) in zip(shards, devs):
        flags = np.zeros(len(rows), dtype=np.uint8)
        _lib.check(_lib.lib().vmb_topk_apply(ctx.h, C.c_void_p(t.data_ptr()), len(rows), P, g.ctypes.data_as(_lib.u32p), G,
                                             gsz.ctypes.data_as(_lib.u32p), C.c_void_p(merged.data_ptr()), K,
                                             ks.ctypes.data_as(_lib.f64p), 0, base, flags.ctypes.data_as(_lib.u8p)))
        got[rows] = dev.get(t)
    assert_same_bits(got, ref_topk(vals, ks, groups, False)[0], "two shards")


# ------------------------------------------------------------------------------------------------ 6. subquery feed, mergeSeries
@pytest.mark.parametrize("points", [32, 33, 97])
def test_subquery_feed_past_the_grid_cap(vm, dev, points):
    """vmb_series_from_matrix (removeNanValues eval.go:1027) on 9,000 rows: all-NaN rows, rows of 32 and 33 points (the ballot
    edges), -0.0 kept as a value"""
    rng = seed("feed", points)
    S = 9000
    assert S > FEED_CAP
    m = rng.normal(size=(S, points))
    m[rng.random(m.shape) < 0.3] = NAN
    m[rng.random(m.shape) < 0.05] = -0.0
    m[::7] = NAN
    m[3::11] = rng.normal(size=points)  # rows without a NaN
    start, step = T0, 60_000
    dm = dev.put(m)
    series = vm.storage.Series.from_matrix(dm.data_ptr(), S, points, start, step)
    try:
        got = series.to_lists()
    finally:
        series.close()
    grid = start + step * np.arange(points, dtype=np.int64)
    assert len(got) == S
    for s, (ts, v) in enumerate(got):
        keep = ~np.isnan(m[s])
        assert np.array_equal(ts, grid[keep]), s
        assert_same_bits(v, m[s][keep], "feed row %d" % s)


def test_merge_series_past_the_grid_cap(vm, dev):
    rng = seed("merge")
    pa, pb, n = 270, 271, 2003
    assert n * (pa + pb) > ELEM_CAP
    a, b = rng.normal(size=(n, pa)), rng.normal(size=(n, pb))
    a[rng.random(a.shape) < 0.05] = -0.0
    a_rows = rng.integers(-1, n, n).astype(np.int64)
    b_rows = rng.integers(-1, n, n).astype(np.int64)
    out, da, db = dev.empty(n, pa + pb), dev.put(a), dev.put(b)
    vm.promql.merge_series(da.data_ptr(), a_rows, pa, db.data_ptr(), b_rows, pb, out.data_ptr())
    want = np.concatenate([np.where((a_rows < 0)[:, None], NAN, a[a_rows]), np.where((b_rows < 0)[:, None], NAN, b[b_rows])], axis=1)
    assert_same_bits(dev.get(out), want, "merge_series")
