"""Rollup results bit for bit, on every kernel path, against the CPU oracle and (for the division steps) exact arithmetic.

The kernels are written to give Go's bits: the library is built with -fmad=false, sums and products that Go rounds one by
one are written out with __dadd_rn / __dmul_rn, and the hand-written division steps (ms_to_s, the fused kernel's reciprocal
rate step, Dec's reciprocal for scales -22..-1) are correctly rounded.  The oracle is built with -ffp-contract=off.  So
every function is compared bit for bit; TOLERANCE lists the only exceptions and why.

Paths (each named in the assertion messages):
  F  vmb_eval_rollup_device with the fused decode+rollup kernel on.  A batch of series that all qualify (one block,
     MarshalTypeDeltaConst timestamps at precisionBits 64) must be finished by the kernel: stage 5 (fused kernel) ran and
     stage 1 (the un-fused sub-batch) did not (vmb_ctx_last_stage_ms, vmb200.h).  Cases the kernel hands back assert
     stage 1 instead.
  U  the same blocks with vmb_ctx_set_fused(0): k_rollup in arithmetic-progression and generic mode.
  J  jittered / irregular timestamp columns: k_rollup's resident seeks, shared window edges and global-memory tile.
  H  host series through vmb_rollup (RollupConfig.do_many): values no decimal carries (-0.0, +-Inf, subnormals, DBL_MAX).
"""
import zlib
from fractions import Fraction

import numpy as np
import pytest

import blockgen
from conftest import SEED0, STALE_NAN
from rollup_names import RF, RF_IDS

pytestmark = pytest.mark.gpu

T0, DT = 1_700_000_000_000, 15000
FU_CAP = 4096        # csrc/fused.cu: rows of one series resident in the fused kernel
ROLLUP_CAP = 2048    # csrc/rollup.cu: rows of one series resident in k_rollup
ROLLUP_SEEKS = 2560  # csrc/rollup.cu: shared window edges are used up to ROLLUP_SEEKS - ROLLUP_CAP = 512 steps per window
STALE_BITS = 0x7FF0000000000002
LIM30 = 1 << 30

# every rollup function id, plus the aliases whose rollupConfig differs from their target's (removeCounterResets,
# MayAdjustWindow, samplesScannedPerCall)
FUNCS = RF_IDS + ["increase", "irate", "deriv_fast", "timestamp", "increase_prometheus"]

# The only functions allowed to differ from the oracle in the last bits.  kind "rel": relative to the larger magnitude;
# kind "avg+bound": relative to |avg| + |bound| (the result is avg -+ bound, and only the bound goes through log());
# kind "zero sign": -0.0 for +0.0 or the reverse, nothing else.
TOLERANCE = {
    "geomean_over_time": ("rel", 1e-9, "pow() of CUDA's libdevice and of glibc round differently"),
    "hoeffding_bound_lower": ("avg+bound", 1e-12, "log() of CUDA's libdevice and of glibc round differently"),
    "hoeffding_bound_upper": ("avg+bound", 1e-12, "log() of CUDA's libdevice and of glibc round differently"),
    # -0.0 and +0.0 compare equal, so which of them a sorted window holds at a given rank depends on how the sort orders
    # equal elements; Go's sort.Float64s (pdqsort) is not stable, the oracle uses std::sort and the kernel ranks by counting.
    # Only host series can hold -0.0 (a decimal cannot).
    "quantile_over_time": ("zero sign", 0.0, "the sign of a zero order statistic is the sort's choice"),
    "median_over_time": ("zero sign", 0.0, "the sign of a zero order statistic is the sort's choice"),
    "mode_over_time": ("zero sign", 0.0, "the sign of a zero order statistic is the sort's choice"),
}
FILTER_FUNCS = {f for f in RF_IDS if f.split("_")[0] in ("count", "share", "sum") and f.split("_")[1] in ("le", "gt", "eq", "ne")}


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def assert_same_bits(got, exp, what, func=None, avg=None):
    """got == exp bit for bit: the same NaN pattern, the staleness marker exactly where the oracle returns it, and the same bits
    for every other value (-0.0 != +0.0).  Functions in TOLERANCE may differ by their stated tolerance instead."""
    got = np.asarray(got, dtype=np.float64)
    exp = np.asarray(exp, dtype=np.float64)
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    gn, en = np.isnan(got), np.isnan(exp)
    bad = np.argwhere(gn != en)
    assert not len(bad), "%s: NaN pattern differs at %s: got %r, expected %r" % (
        what, bad[:5].tolist(), got[tuple(bad[0])], exp[tuple(bad[0])])
    gs, es = bits(got) == STALE_BITS, bits(exp) == STALE_BITS
    bad = np.argwhere(gs != es)
    assert not len(bad), "%s: staleness markers differ at %s" % (what, bad[:5].tolist())
    diff = (bits(got) != bits(exp)) & ~en
    if func in TOLERANCE and diff.any():
        kind, tol, _ = TOLERANCE[func]
        g, e = got[diff], exp[diff]
        if kind == "zero sign":
            scale = np.zeros_like(g)
        elif kind == "rel":
            scale = np.maximum(np.abs(g), np.abs(e))
        else:
            a = np.asarray(avg, dtype=np.float64)[diff]
            scale = np.abs(a) + np.abs(e - a)
        with np.errstate(invalid="ignore"):
            ok = np.isfinite(g) & np.isfinite(e) & (np.abs(g - e) <= tol * scale)
        diff[diff] = ~ok
    bad = np.argwhere(diff)
    if len(bad):
        ex = ["%s got %r (%016x) expected %r (%016x)" % (tuple(b), got[tuple(b)], bits(got)[tuple(b)], exp[tuple(b)],
                                                        bits(exp)[tuple(b)]) for b in bad[:4]]
        raise AssertionError("%s: %d values differ in their bits; %s" % (what, len(bad), "; ".join(ex)))


# ------------------------------------------------------------------------------------------------ helpers
def point_args(func, P):
    """args / args2 that change along the grid"""
    q = np.arange(P)

    def cyc(vals):
        return np.asarray(vals, dtype=np.float64)[q % len(vals)]
    if func == "quantile_over_time":
        return cyc([0.0, 1e-300, 0.25, 0.5, 0.75, 0.9, 0.99, 1.0, -1.0, 2.0, np.nan, 1 / 3, 0.1]), None
    if func.startswith("hoeffding_bound"):
        return cyc([0.9, 0.5, 0.0, 1.0, 0.99, -0.5, 1.5, 1e-300]), None
    if func == "predict_linear":
        return cyc([60.0, -30.0, 0.0, 3600.5, 1e-3]), None
    if func == "holt_winters":  # sf, tf at 0, 1, inside and out of range; cycles of 7 and 8 meet in every combination
        return cyc([0.5, 0.0, 1.0, 0.3, -0.1, 1.1, 0.9]), cyc([0.3, 1.0, 0.0, 0.7, 0.5, 2.0, -1.0, 0.1])
    if func == "duration_over_time":  # dMax 15 s equals the scrape interval
        return cyc([DT / 1000, 14.999, 20.0, 0.0, 30.0, 7.5]), None
    if func in FILTER_FUNCS:  # limits equal to values of the windows (gauge_small is -3..3, gauge about 50), +-Inf, NaN
        return cyc([0.0, 1.0, -3.0, 3.0, 50.0, np.inf, -np.inf, np.nan, 2.5, -0.0, 49.99]), None
    return None, None


def rollup_cfg(vm, func, start, end, step, window, lookback=0):
    P = 1 + (end - start) // step
    a1, a2 = point_args(func, P)
    return vm.promql.get_rollup_configs(func, start, end, step, window, lookback, args=a1, args2=a2)


def oracle_rows(oracle, rc, rows, fid=None):
    """the oracle's rollupConfig.Do for every (timestamps, values) series after dropStaleNaNs and removeCounterResets
    -> ([nseries x P], samplesScanned)"""
    out, scanned = [], 0
    for ts, fv in rows:
        ts = np.array(ts, dtype=np.int64)
        fv = np.array(fv, dtype=np.float64)
        n = len(ts)
        if rc.dropStaleNaNs and n:
            n = oracle.lib().vmo_drop_stale_nans(fv.ctypes.data_as(oracle.f64p), ts.ctypes.data_as(oracle.i64p), n)
        ts, fv = ts[:n].copy(), fv[:n].copy()
        if rc.removeCounterResets and n:
            oracle.lib().vmo_remove_counter_resets(fv.ctypes.data_as(oracle.f64p), ts.ctypes.data_as(oracle.i64p), n,
                                                   rc.LookbackDelta + rc.Window if rc.LookbackDelta else 0)
        o, sc = oracle.rollup_do(RF[rc.Func] if fid is None else fid, fv, ts, rc.Start, rc.End, rc.Step, rc.Window,
                                 lookback_delta=rc.LookbackDelta, may_adjust_window=rc.MayAdjustWindow,
                                 is_default_rollup=rc.isDefaultRollup, samples_scanned_per_call=rc.samplesScannedPerCall,
                                 args=rc.args, args2=rc.args2, min_staleness_ms=rc.minStalenessInterval)
        out.append(o)
        scanned += sc
    return np.stack(out), scanned


def expected(oracle, rc, rows):
    """-> (values, samplesScanned, avg_over_time on the same windows for the functions compared relative to it)"""
    exp, sc = oracle_rows(oracle, rc, rows)
    avg = None
    if TOLERANCE.get(rc.Func, ("",))[0] == "avg+bound":
        avg, _ = oracle_rows(oracle, rc, rows, fid=RF["avg_over_time"])
    return exp, sc, avg


def block_rows(blocks):
    out = []
    for b in blocks:
        r, ts, fv, _ = b.oracle_unmarshal()
        assert r == 0
        out.append((ts, fv))
    return out


@pytest.fixture(scope="module")
def vm():
    import victoriametrics_b200 as v
    return v


@pytest.fixture(scope="module")
def tctx(vm):
    """a context of its own with stage timing on, so that every call reports which kernels ran"""
    ctx = vm.Context(0)
    ctx.enable_stage_timing(True)
    yield ctx
    ctx.close()


class DeviceBlocks:
    def __init__(self, vm, ctx, blocks):
        self.vm, self.ctx, self.n = vm, ctx, len(blocks)
        self.descs, self.payload = blockgen.to_blockset(blocks)
        self.B = vm.storage.Blocks(self.descs, self.payload, ctx)

    def run(self, rc, fused):
        """-> (values [nseries x P], samplesScanned, stage_ms)"""
        import torch
        out = torch.full((self.n, rc.points), -7.0, dtype=torch.float64, device="cuda")
        self.ctx.set_fused(fused)
        try:
            _, scanned = self.vm.promql.eval_rollup_func(rc.Func, self.B, rc.Start, rc.End, rc.Step, rc=rc,
                                                         out_dev_ptr=out.data_ptr())
            stages = self.ctx.stage_ms()
        finally:
            self.ctx.set_fused(True)
        torch.cuda.synchronize()
        return out.cpu().numpy(), scanned, stages

    def close(self):
        self.B.close()


def check_fu(oracle, dev, rows, rc, what, fused="taken"):
    """paths F and U of one batch against the oracle.  fused: "taken" = the fused kernel finished every series, "handed back"
    = it gave at least one back to the un-fused pipeline, None = not asserted."""
    exp, esc, avg = expected(oracle, rc, rows)
    for f in (True, False):
        got, sc, st = dev.run(rc, f)
        path = "%s [%s %s]" % (what, rc.Func, "F" if f else "U")
        assert_same_bits(got, exp, path, rc.Func, avg)
        assert sc == esc, (path, "samplesScanned", sc, esc)
        if f and fused == "taken":
            assert st[5] > 0 and st[1] == 0, (path, "the fused kernel did not finish every series", st)
        elif f and fused == "handed back":
            assert st[1] > 0, (path, "expected a hand-back to the un-fused pipeline", st)


def fused_expectation(rc, noisy, dt=DT):
    """what the fused kernel does with a batch of qualifying series.  It removes counter resets (rollup.go:921) from the
    events of one fill, at most FU_MAX_EVENTS = 32 value drops; a noisy gauge has more and is handed back.  The kernel skips
    removeCounterResets when the staleness interval (lookback + window) is below the scrape interval (rollup.go:937)."""
    max_stale = rc.LookbackDelta + rc.Window if rc.LookbackDelta else 0
    removes = rc.removeCounterResets and not (max_stale > 0 and dt > max_stale)
    return "handed back" if noisy and removes else "taken"


def check_j(oracle, dev, rows, rc, what):
    exp, esc, avg = expected(oracle, rc, rows)
    got, sc, _ = dev.run(rc, True)
    path = "%s [%s J]" % (what, rc.Func)
    assert_same_bits(got, exp, path, rc.Func, avg)
    assert sc == esc, (path, "samplesScanned", sc, esc)


def gen(rng, kind, n):
    if kind == "dconst":   # MarshalTypeDeltaConst values with a non-negative delta
        return (int(rng.integers(0, 1000)) + int(rng.integers(0, 50)) * np.arange(n)).astype(np.int64)
    if kind == "big_gauge":  # about 1e15 with small noise: stddev / stdvar / zscore depend on the order of Welford's updates
        return (10 ** 15 + rng.integers(-3, 4, n)).astype(np.int64)
    return blockgen.gen_values(rng, kind, n)


def make_blocks(rng, spec, tkind="regular", dt=DT, first_idx=0):
    out = []
    for i, (kind, n, scale) in enumerate(spec, first_idx):
        if tkind == "regular":
            ts = (T0 + dt * np.arange(n)).astype(np.int64)
        else:
            ts = blockgen.gen_timestamps(rng, tkind, n, T0)
        out.append(blockgen.OBlock(ts, gen(rng, kind, n), scale, 64, i))
    return out


def fseed(func, k):
    return np.random.default_rng(SEED0 + zlib.crc32(("%s/%d" % (func, k)).encode()))


# ------------------------------------------------------------------------------------------------ 2. the path matrix
STEADY_SPEC = [("counter", 8192, -2), ("counter_resets", 5000, -2), ("const", 300, -2), ("dconst", 40, -2),
               ("counter_smooth", 3, -2), ("counter", 2, 1)]
NOISY_SPEC = [("gauge", 700, -2), ("gauge_small", 700, 0), ("gauge", 3, 1)]
END = DT * 8300
# windows stay at or below 240 rows: distinct / mode / mad / the general quantile case are O(window^2) per point on the GPU
GRIDS = [  # (name, start offset, end offset, step, window, lookback)
    ("5m", 300000, END, 15000, 300000, 0),
    ("step%dt!=0", 7777, END, 7001, 33333, 0),                        # fused: no arithmetic window edges, seek_ap
    ("1h", 60000, END, 60000, 3600000, 0),                             # 240 rows per window
    ("window0", 300000, END, 15000, 0, 0),                             # MayAdjustWindow / default window
    ("lookback<si", 300000, END, 15000, 0, 10000),
    ("lookback=si", 300000, END, 30000, 60000, 15000),
    ("lookback>si", 300000, END, 15000, 60000, 20000),
    ("outside", -500000, DT * 8400, 15000, 300000, 0),                 # starts before the series, ends after
    ("512steps", 300000, 300000 + 500 * 3000, 500, 512 * 500, 0),      # k_rollup: shared window edges
    ("513steps", 300000, 300000 + 500 * 3000, 500, 513 * 500, 0),      # k_rollup: one past them
]


@pytest.mark.parametrize("func", FUNCS)
def test_paths_fused_unfused_jittered(vm, oracle, tctx, func):
    rng = fseed(func, 0)
    steady, noisy = make_blocks(rng, STEADY_SPEC), make_blocks(rng, NOISY_SPEC)
    jblocks = make_blocks(rng, STEADY_SPEC[:2] + NOISY_SPEC, "jitter")
    jblocks += make_blocks(rng, STEADY_SPEC[2:], "irregular", first_idx=len(jblocks))
    batches = [(b, block_rows(b), DeviceBlocks(vm, tctx, b)) for b in (steady, noisy, jblocks)]
    try:
        for name, so, eo, step, window, lookback in GRIDS:
            rc = rollup_cfg(vm, func, T0 + so, T0 + eo, step, window, lookback)
            for k, (_, rows, dev) in enumerate(batches):
                if k < 2:
                    check_fu(oracle, dev, rows, rc, name, fused_expectation(rc, noisy=k == 1))
                else:
                    check_j(oracle, dev, rows, rc, name)
    finally:
        for _, _, dev in batches:
            dev.close()


# ------------------------------------------------------------------------------------------------ 3. strategy boundaries
# A point of the fused kernel needs rows i-1 .. j resident (the row in front of its window, the window, the row behind it),
# and the ring holds FU_CAP rows; with the first window starting right after row 0 (tStart = t(row 0)) the ring is full on the
# first fill, so a window of W rows is finished in the kernel iff W + 2 <= FU_CAP.  Wider windows are handed back.
FU_WINDOWS = [FU_CAP - 3, FU_CAP - 2, FU_CAP - 1, FU_CAP, FU_CAP + 1]


@pytest.mark.parametrize("func", FUNCS)
def test_window_capacity_boundaries(vm, oracle, tctx, func):
    rng = fseed(func, 1)
    n = FU_CAP + 104
    # MarshalTypeConst / DeltaConst values: the kernel generates rows one by one, so its ring fills to exactly FU_CAP rows
    blocks = make_blocks(rng, [("dconst", n, -2), ("const", n, -2), ("dconst", n, 0)])
    rows = block_rows(blocks)
    dev = DeviceBlocks(vm, tctx, blocks)
    try:
        for W in FU_WINDOWS:
            rc = rollup_cfg(vm, func, T0 + W * DT, T0 + (n - 1) * DT, 16 * DT, W * DT)
            check_fu(oracle, dev, rows, rc, "fused window %d rows" % W, "taken" if W + 2 <= FU_CAP else "handed back")
    finally:
        dev.close()
    # k_rollup: a window that does not fit ROLLUP_CAP resident rows is read from global memory
    jblocks = make_blocks(rng, [("gauge", 2600, -2), ("counter_resets", 2600, -2), ("gauge_small", 2600, 0)], "jitter")
    jrows = block_rows(jblocks)
    jdev = DeviceBlocks(vm, tctx, jblocks)
    try:
        for W in (ROLLUP_CAP - 2, ROLLUP_CAP - 1, ROLLUP_CAP, ROLLUP_CAP + 1):
            rc = rollup_cfg(vm, func, T0 + W * DT, T0 + 2599 * DT, 32 * DT, W * DT)
            check_j(oracle, jdev, jrows, rc, "k_rollup window %d rows" % W)
    finally:
        jdev.close()


@pytest.mark.parametrize("func", FUNCS)
def test_windows_of_2_31_ms_and_more(vm, oracle, tctx, func):
    """increase(m[30d])-like windows: k_rollup's 64-bit window / step branch; the fused kernel hands them back (its grid
    arithmetic is 32-bit)"""
    rng = fseed(func, 2)
    dt = 3_000_000  # 300 rows over ten days
    blocks = make_blocks(rng, [("counter", 300, -2), ("counter_resets", 300, -2), ("gauge", 300, -2)], dt=dt)
    rows = block_rows(blocks)
    dev = DeviceBlocks(vm, tctx, blocks)
    day = 86_400_000
    try:
        for step, window in ((1 << 24, 1 << 31), (3_600_000, (1 << 31) + 1), (3_600_000, 30 * day), (7_200_001, 30 * day)):
            rc = rollup_cfg(vm, func, T0 + 3_600_000, T0 + 300 * dt + 2 * day, step, window)
            check_fu(oracle, dev, rows, rc, "window %d step %d" % (window, step), "handed back")
    finally:
        dev.close()


# ------------------------------------------------------------------------------------------------ 4. values at the edges
EDGE_SCALES = [-22, -23, -300, 5, 290, -270, 270]


def edge_blocks(rng, with_stale, noisy):
    spec = []
    for s in EDGE_SCALES:
        spec += [("gauge_wide", 400, s), ("big_gauge", 300, s)] if noisy else [("counter", 400, s), ("const", 50, s)]
    spec += [("gauge_small", 300, -23)] if noisy else [("counter_resets", 600, -22)]
    blocks = make_blocks(rng, spec)
    # +-Inf mantissas (decimal.go:406-417) in some of them; staleness markers only in the batch that asks for them
    specials = [(1 << 63) - 1, -(1 << 63)] + ([(1 << 63) - 2] if with_stale else [])
    for k, b in enumerate(blocks):
        if k % 3 == 1 and b.rows > 10:
            v = b.vals.copy()
            v[rng.integers(1, b.rows, 4)] = rng.choice(specials, 4)
            blocks[k] = blockgen.OBlock(b.ts, v, b.scale, 64, k)
    return blocks


@pytest.mark.parametrize("func", FUNCS)
def test_edge_values_through_the_decoder(vm, oracle, tctx, func):
    """scales -22 (Dec through the reciprocal), -23 and -300 (division), 5 and 290 (multiplication; 290 overflows to Inf),
    +-270 (rate / delta / deriv deltas on both sides of 2^-900 and 2^900: the fused Markstein step and its IEEE fallback),
    constant series, values about 1e15; then the same with staleness markers, which the fused kernel takes only where
    nothing drops them"""
    rng = fseed(func, 3)
    for stale in (False, True):
        for noisy in (False, True):
            blocks = edge_blocks(rng, stale, noisy)
            rows = block_rows(blocks)
            dev = DeviceBlocks(vm, tctx, blocks)
            try:
                for step, window in ((15000, 300000), (30000, 0)):
                    rc = rollup_cfg(vm, func, T0 + 300000, T0 + 410 * DT, step, window)
                    expect = fused_expectation(rc, noisy)
                    if stale and rc.dropStaleNaNs or stale and rc.removeCounterResets:
                        expect = "handed back"  # staleness markers that have to be dropped
                    check_fu(oracle, dev, rows, rc, "edges stale=%s noisy=%s" % (stale, noisy), expect)
            finally:
                dev.close()


def _rcr_without_clamp(v):
    """removeCounterResets (rollup.go:921) without its final clamp `if values[i] < values[i-1]`, staleness interval 0"""
    out = np.empty_like(v)
    corr, prev = 0.0, v[0]
    for i, x in enumerate(v.tolist()):
        d = x - prev
        if d < 0:
            corr += (prev - x) if (-d * 8) < prev else prev
        prev = x
        out[i] = x + corr
    return out


@pytest.mark.parametrize("func", ["rate", "increase", "irate", "increase_prometheus", "rate_prometheus", "increase_pure"])
def test_counter_resets_where_rounding_breaks_monotonicity(vm, oracle, tctx, func):
    """counters near 2^55 with small drops after a large one: v + correction rounds below the previous corrected value, so
    the final clamp of removeCounterResets fires (checked here on the CPU) and the fused kernel's parallel correction must
    fall back to its sequential pass"""
    rng = fseed(func, 4)
    blocks = []
    for s in range(6):
        n = 3000
        v = (1 << 55) + np.cumsum(rng.integers(0, 3000, n)).astype(np.int64)
        v[700:] -= v[700] - 1000  # a large reset: the correction becomes about 2^55
        for r in np.sort(rng.choice(np.arange(900, n), 20, replace=False)):
            v[r:] -= v[r] - v[r - 1] + int(rng.integers(1, 40))  # small drops: corrected by prev - v
        blocks.append(blockgen.OBlock((T0 + DT * np.arange(n)).astype(np.int64), v, int(rng.choice([0, -1, 1])), 64, s))
    rows = block_rows(blocks)
    clamped = 0
    for ts, fv in rows:
        e = fv.copy()
        oracle.lib().vmo_remove_counter_resets(e.ctypes.data_as(oracle.f64p), ts.ctypes.data_as(oracle.i64p), len(e), 0)
        clamped += int(np.count_nonzero(bits(e) != bits(_rcr_without_clamp(fv))))
    assert clamped > 0, "the input does not reach the clamp of removeCounterResets"
    dev = DeviceBlocks(vm, tctx, blocks)
    try:
        for step, window in ((15000, 300000), (60000, 3600000)):
            check_fu(oracle, dev, rows, rollup_cfg(vm, func, T0 + 300000, T0 + 3000 * DT, step, window), "rcr clamp")
    finally:
        dev.close()


@pytest.mark.parametrize("func", ["quantile_over_time", "median_over_time", "mad_over_time", "outlier_iqr_over_time",
                                  "mode_over_time", "distinct_over_time"])
def test_quantile_family_small_windows_and_ties(vm, oracle, tctx, func):
    """windows of 1 to 9 values around the top-4 / bottom-4 switches of quantile_tf, heavy ties, phi in
    {0, 1e-300, 0.25, exact ranks, 1, -1, 2, NaN}"""
    rng = fseed(func, 5)
    spec = [("gauge_small", 500, 0), ("gauge_small", 500, -1), ("const", 100, 0), ("gauge", 500, -2), ("counter", 300, -2)]
    blocks = make_blocks(rng, spec)
    tie = blocks[1].vals.copy()
    tie[::2] = 1  # heavier ties
    blocks[1] = blockgen.OBlock(blocks[1].ts, tie, -1, 64, 1)
    rows = block_rows(blocks)
    dev = DeviceBlocks(vm, tctx, blocks)
    try:
        for k in range(1, 10):
            start, end = T0 + k * DT, T0 + 490 * DT  # every window holds k rows
            P = 1 + (end - start) // DT
            # phi * (k - 1) an exact integer for every rank of the window, and the special values
            phis = [0.0, 1e-300, 0.25, 1.0, -1.0, 2.0, np.nan, 0.5] + [r / (k - 1) for r in range(1, k - 1)]
            args = np.array(phis)[np.arange(P) % len(phis)] if func == "quantile_over_time" else None
            rc = vm.promql.get_rollup_configs(func, start, end, DT, k * DT, args=args)
            check_fu(oracle, dev, rows, rc, "window %d rows" % k)
    finally:
        dev.close()


def host_series(rng):
    """values a decimal cannot carry"""
    tiny = 5e-324
    specials = np.array([-0.0, 0.0, np.inf, -np.inf, tiny, -tiny, 2.2250738585072014e-308, 1e-310, -3e-320,
                         1.7976931348623157e308, -1.7976931348623157e308, 8.98846567431158e307, STALE_NAN])
    ts_list, v_list = [], []
    for k, n in enumerate((2, 3, 40, 700, 700, 700)):
        if k % 2:
            ts = T0 + DT * np.arange(n) + rng.integers(-50, 51, n)
        else:
            ts = T0 + DT * np.arange(n)
        if k == 3:    # subnormals and zeros only
            v = rng.choice(specials[[0, 1, 4, 5, 6, 7, 8]], n)
        elif k == 4:  # near DBL_MAX: sums and differences overflow
            v = rng.choice(specials[[9, 10, 11]], n) * rng.choice([1.0, 0.5, 0.75], n)
        else:
            v = np.round(rng.normal(50, 3, n), 2)
            v[rng.integers(0, n, max(n // 10, 1))] = rng.choice(specials, max(n // 10, 1))
        ts_list.append(ts.astype(np.int64))
        v_list.append(v.astype(np.float64))
    return ts_list, v_list


@pytest.mark.parametrize("func", FUNCS)
def test_host_series_special_values(vm, oracle, func):
    rng = fseed(func, 6)
    ts_list, v_list = host_series(rng)
    for name, so, eo, step, window, lookback in (("5m", -30000, 700 * DT, 15000, 300000, 0),
                                                  ("window0", 0, 700 * DT, 30000, 0, 0),
                                                  ("step%dt!=0", 7777, 700 * DT, 7001, 33333, 0)):
        rc = rollup_cfg(vm, func, T0 + so, T0 + eo, step, window, lookback)
        got, sc = rc.do_many(ts_list, v_list)
        exp, esc, avg = expected(oracle, rc, list(zip(ts_list, v_list)))
        assert_same_bits(got, exp, "%s [%s H]" % (name, func), func, avg)
        assert sc == esc, (name, func, "samplesScanned", sc, esc)


# ------------------------------------------------------------------------------------------------ 5. exact division
DIV_DTS = sorted({1, 3, 7, 999, 1001, LIM30 - 1} | {(1 << k) + d for k in range(2, 30) for d in (-1, 1)})
DIV_MANTISSAS = [  # (scale, m0, m1): dv = v(m1) - v(m0) about 2^900 and 2^-900 on both sides of the fused kernel's guard, zero
    (255, 10 ** 16, 10 ** 16 + 8_400_000_000_000_000), (255, 10 ** 16, 10 ** 16 + 8_500_000_000_000_000), (255, 7, 7),
    (-288, 10 ** 17, 10 ** 17 + 117_000_000_000_000_000), (-288, 10 ** 17, 10 ** 17 + 119_000_000_000_000_000),
    (-288, 123456789, 123456790), (-2, 100, 1234567), (-2, 5, 5), (-3, 1, 2), (0, 0, 1)]
H_PAIRS = [(0.0, 2.0 ** 900), (-0.0, 2.0 ** 901), (2.0 ** -900, 1.25 * 2.0 ** -899), (0.0, 5e-324), (-0.0, 3e-320),
           (1e-310, 2e-310), (0.0, 0.0), (0.0, -0.0), (-0.0, -0.0), (2.0 ** 900, 0.0), (3e-320, -1e-310)]


def go_div(dv, dt_ms):
    """Go's dv / (float64(dt) / 1e3), both divisions correctly rounded: from exact rationals"""
    D = float(Fraction(dt_ms, 1000))
    if dv == 0:
        return dv / D  # (a signed zero)
    return float(Fraction(dv) / Fraction(D))


@pytest.mark.parametrize("func", ["rate", "irate", "deriv_fast"])
def test_rate_division_matches_exact_arithmetic(vm, oracle, tctx, func):
    """two- and three-row series, dt from 1 ms to 2^30 - 1 ms, one point at the last row with a window of one interval: the
    result is (v[n-1] - v[n-2]) / (dt / 1e3).  F (the fused kernel's reciprocal step), U (ms_to_s) and H against a quotient
    computed from exact rationals, and the oracle against the same"""
    rcr = func != "deriv_fast"
    for dt in DIV_DTS:
        ts3 = (T0 + dt * np.arange(3)).astype(np.int64)
        for n in (2, 3):
            blocks = []
            for scale, m0, m1 in DIV_MANTISSAS:
                vals = np.array([m0, m1] if n == 2 else [m0 - (m1 - m0) // 3, m0, m1], dtype=np.int64)
                if not rcr and (m1 + dt) % 2:
                    vals = vals[::-1].copy()  # negative deltas for deriv_fast (rate / irate would remove a counter reset)
                blocks.append(blockgen.OBlock(ts3[:n], vals, scale, 64, len(blocks)))
            rows = block_rows(blocks)
            want = np.array([[go_div(fv[-1] - fv[-2], dt)] for _, fv in rows])
            tend = int(ts3[n - 1])
            rc = rollup_cfg(vm, func, tend, tend, dt, dt)
            what = "dt=%d n=%d" % (dt, n)
            assert_same_bits(expected(oracle, rc, rows)[0], want, "oracle vs exact " + what)
            # the fused kernel takes these while its grid stays inside +-2^30 ms (maxPrevInterval = step = dt here) and the
            # values column is not a decreasing MarshalTypeDeltaConst one
            taken = (n - 1) * dt < LIM30 and all(b.vmt != 2 or b.vals[-1] >= b.vals[0] for b in blocks)
            dev = DeviceBlocks(vm, tctx, blocks)
            try:
                check_fu(oracle, dev, rows, rc, what, "taken" if taken else None)
                for f in (True, False):
                    assert_same_bits(dev.run(rc, f)[0], want, "exact %s %s" % (what, "F" if f else "U"))
            finally:
                dev.close()
        # H: host values, including subnormal quotients and signed zeros
        pairs = [(a, b) for a, b in H_PAIRS if not (rcr and b < a)]
        ts_list = [ts3[:2]] * len(pairs)
        v_list = [np.array(p) for p in pairs]
        rc = rollup_cfg(vm, func, int(ts3[1]), int(ts3[1]), dt, dt)
        got, _ = rc.do_many(ts_list, v_list)
        # removeCounterResets adds a correction of +0.0 to every value: -0.0 becomes +0.0
        want = np.array([[go_div((b + 0.0) - (a + 0.0) if rcr else b - a, dt)] for a, b in pairs])
        assert_same_bits(got, want, "exact dt=%d H" % dt)
        assert_same_bits(expected(oracle, rc, list(zip(ts_list, v_list)))[0], want, "oracle vs exact dt=%d H" % dt)
