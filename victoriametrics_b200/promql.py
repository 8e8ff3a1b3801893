"""app/vmselect/promql mirror: rollupConfig.Do, getRollupConfigs, evalRollupFunc*, incremental aggregates.

Names follow the reference (rollup.go / eval.go / aggr_incremental.go); every compute call goes to libvmb200.
"""
import ctypes as C
import math
import re
import string

import numpy as np

from . import _lib, decimal, storage
from ._lib import RollupCfg, check, lib

# enum vmb_rollup_func order (include/vmb200.h); keys are the MetricsQL names of rollup.go:24-108
_RF_ORDER = ["default_rollup", "rate", "delta", "avg_over_time", "min_over_time", "max_over_time", "sum_over_time",
             "count_over_time", "quantile_over_time", "first_over_time", "last_over_time", "range_over_time",
             "sum2_over_time", "stddev_over_time", "stdvar_over_time", "ideriv", "idelta", "deriv", "increase_pure",
             "changes", "changes_prometheus", "resets", "increases_over_time", "integrate", "lag", "lifetime",
             "scrape_interval", "tmin_over_time", "tmax_over_time", "tfirst_over_time", "tlast_over_time",
             "tlast_change_over_time", "mode_over_time", "mad_over_time", "outlier_iqr_over_time", "zscore_over_time",
             "ascent_over_time", "descent_over_time", "distinct_over_time", "geomean_over_time", "predict_linear",
             "holt_winters", "hoeffding_bound_lower", "hoeffding_bound_upper", "duration_over_time",
             "count_le_over_time", "count_gt_over_time", "count_eq_over_time", "count_ne_over_time",
             "share_le_over_time", "share_gt_over_time", "share_eq_over_time", "sum_le_over_time", "sum_gt_over_time",
             "sum_eq_over_time", "present_over_time", "absent_over_time", "stale_samples_over_time",
             "median_over_time", "rate_over_sum", "delta_prometheus", "rate_prometheus", "rollup_open", "rollup_close",
             "rollup_high", "rollup_low"]
ROLLUP_FUNCS = {n: i for i, n in enumerate(_RF_ORDER)}
for _a, _b in {"deriv_fast": "rate", "increase": "delta", "irate": "ideriv", "decreases_over_time": "resets",
               "timestamp": "tlast_over_time", "timestamp_with_name": "tlast_over_time",
               "increase_prometheus": "delta_prometheus", "iqr_over_time": "outlier_iqr_over_time"}.items():
    ROLLUP_FUNCS[_a] = ROLLUP_FUNCS[_b]

# rollup.go:199 rollupFuncsCanAdjustWindow
ROLLUP_FUNCS_CAN_ADJUST_WINDOW = {"default_rollup", "deriv", "deriv_fast", "ideriv", "irate", "rate", "rate_over_sum",
                                  "rollup", "rollup_candlestick", "rollup_deriv", "rollup_rate",
                                  "rollup_scrape_interval", "scrape_interval", "timestamp"}
# rollup.go:223 rollupFuncsRemoveCounterResets
ROLLUP_FUNCS_REMOVE_COUNTER_RESETS = {"increase", "increase_prometheus", "increase_pure", "irate", "rate",
                                      "rate_prometheus", "rollup_increase", "rollup_rate"}
# rollup.go:238 rollupFuncsSamplesScannedPerCall
ROLLUP_FUNCS_SAMPLES_SCANNED_PER_CALL = {
    "absent_over_time": 1, "count_over_time": 1, "default_rollup": 1, "delta": 2, "delta_prometheus": 2, "deriv_fast": 2,
    "first_over_time": 1, "idelta": 2, "ideriv": 2, "increase": 2, "increase_prometheus": 2, "increase_pure": 2,
    "irate": 2, "lag": 1, "last_over_time": 1, "lifetime": 2, "present_over_time": 1, "rate": 2, "rate_prometheus": 2,
    "scrape_interval": 2, "tfirst_over_time": 1, "timestamp": 1, "timestamp_with_name": 1, "tlast_over_time": 1}

RC_MAY_ADJUST_WINDOW, RC_IS_DEFAULT_ROLLUP, RC_REMOVE_COUNTER_RESETS, RC_DROP_STALE_NANS = 1, 2, 4, 8
RC_PRE = {None: 0, "delta": 16, "deriv": 32, "scrape_interval": 64}  # value preFuncs of the multi-output rollups
# rollup.go:147 rollupAggrFuncs: what aggr_over_time() accepts
ROLLUP_AGGR_FUNCS = {"absent_over_time", "ascent_over_time", "avg_over_time", "changes", "count_over_time",
                     "decreases_over_time", "default_rollup", "delta", "deriv", "deriv_fast", "descent_over_time",
                     "distinct_over_time", "first_over_time", "geomean_over_time", "idelta", "ideriv", "increase",
                     "increase_pure", "increases_over_time", "integrate", "irate", "iqr_over_time", "lag", "last_over_time",
                     "lifetime", "mad_over_time", "max_over_time", "median_over_time", "min_over_time", "mode_over_time",
                     "present_over_time", "range_over_time", "rate", "rate_over_sum", "resets", "scrape_interval",
                     "stale_samples_over_time", "stddev_over_time", "stdvar_over_time", "sum_over_time", "sum2_over_time",
                     "tfirst_over_time", "timestamp", "timestamp_with_name", "tlast_change_over_time", "tlast_over_time",
                     "tmax_over_time", "tmin_over_time", "zscore_over_time"}
AGGR_FUNCS = {"sum": 0, "min": 1, "max": 2, "avg": 3, "count": 4, "sum2": 5, "geomean": 6, "any": 7, "group": 8}


def get_timestamps(start, end, step):
    """eval.go:230 getTimestamps"""
    if step <= 0:
        raise ValueError("BUG: Step must be bigger than 0; got %d" % step)
    if start > end:
        raise ValueError("BUG: Start cannot exceed End; got %d vs %d" % (start, end))
    return start + step * np.arange(1 + (end - start) // step, dtype=np.int64)


class RollupConfig:
    """rollupConfig rollup.go:574.  Func is the MetricsQL function name."""

    def __init__(self, Func, Start, End, Step, Window=0, LookbackDelta=0, MayAdjustWindow=False, isDefaultRollup=False,
                 samplesScannedPerCall=0, args=None, args2=None, removeCounterResets=False, dropStaleNaNs=False,
                 minStalenessInterval=0, TagValue="", preFunc=None):
        self.Func, self.Start, self.End, self.Step, self.Window = Func, int(Start), int(End), int(Step), int(Window)
        self.LookbackDelta, self.MayAdjustWindow, self.isDefaultRollup = int(LookbackDelta), MayAdjustWindow, isDefaultRollup
        self.samplesScannedPerCall, self.args, self.args2 = samplesScannedPerCall, args, args2
        self.removeCounterResets, self.dropStaleNaNs = removeCounterResets, dropStaleNaNs
        self.minStalenessInterval = int(minStalenessInterval)
        self.TagValue, self.preFunc = TagValue, preFunc  # rollup.go:576 TagValue; preFunc in (None, "delta", "deriv", "scrape_interval")
        if self.Step <= 0 or self.Start > self.End or self.Window < 0:  # rollup.go:703-711 logger.Panicf("BUG: ...")
            raise ValueError("BUG: invalid rollupConfig: Step=%d Start=%d End=%d Window=%d" % (Step, Start, End, Window))
        self.Timestamps = get_timestamps(self.Start, self.End, self.Step)
        self._keep = []

    @property
    def points(self):
        return int(self.Timestamps.size)

    def _cfg(self):
        flags = (RC_MAY_ADJUST_WINDOW if self.MayAdjustWindow else 0) | (RC_IS_DEFAULT_ROLLUP if self.isDefaultRollup else 0) \
            | (RC_REMOVE_COUNTER_RESETS if self.removeCounterResets else 0) | (RC_DROP_STALE_NANS if self.dropStaleNaNs else 0) \
            | RC_PRE[self.preFunc]
        cfg = RollupCfg(ROLLUP_FUNCS[self.Func], flags, self.Start, self.End, self.Step, self.Window, self.LookbackDelta,
                        self.minStalenessInterval, self.samplesScannedPerCall, 0, None, None)
        self._keep = []
        for name, a in (("args", self.args), ("args2", self.args2)):
            if a is not None:
                arr = np.ascontiguousarray(np.broadcast_to(np.asarray(a, dtype=np.float64), (self.points,)))
                self._keep.append(arr)
                setattr(cfg, name, arr.ctypes.data_as(_lib.f64p))
        return cfg

    def do(self, values, timestamps, ctx=None):
        """rollupConfig.Do rollup.go:688 for ONE series (kept for compatibility/tests; the batched forms are the fast path)
        -> (dstValues np.float64[points], samplesScanned)"""
        out, scanned = self.do_many([timestamps], [values], ctx)
        return out[0], scanned

    def do_many(self, timestamps_list, values_list, ctx=None):
        s = storage.Series.from_host(timestamps_list, values_list, ctx)
        try:
            return self.do_series(s)
        finally:
            s.close()

    def do_series(self, series, out_dev_ptr=None):
        """rollup over a device batch -> ([nseries x points] np.float64 (or None when out_dev_ptr is given), samplesScanned)"""
        cfg = self._cfg()
        scanned = C.c_uint64(0)
        if out_dev_ptr is not None:
            check(lib().vmb_rollup(series.ctx.h, series.h, C.byref(cfg), C.c_void_p(int(out_dev_ptr)), 1, C.byref(scanned)))
            return None, scanned.value
        out = np.empty((series.count, self.points), dtype=np.float64)
        check(lib().vmb_rollup(series.ctx.h, series.h, C.byref(cfg), C.c_void_p(out.ctypes.data), 0, C.byref(scanned)))
        return out, scanned.value


def get_rollup_configs(func_name, start, end, step, window=0, lookback_delta=0, args=None, args2=None,
                       no_stale_markers=False, min_staleness_interval=0):
    """getRollupConfigs rollup.go:374 for the single-config functions + the preFunc / dropStaleNaNs decisions of
    eval.go:1855-1866, :1985.  (rollup*(), aggr_over_time(), *_values_over_time() produce several series per input
    and stay on the host: SURVEY.md 8(a) a23.)"""
    name = func_name.lower()
    if name not in ROLLUP_FUNCS:
        raise KeyError("unsupported rollup function %r" % func_name)
    drop_stale = not (no_stale_markers or name in ("default_rollup", "stale_samples_over_time"))
    return RollupConfig(name, start, end, step, window, lookback_delta,
                        MayAdjustWindow=name in ROLLUP_FUNCS_CAN_ADJUST_WINDOW, isDefaultRollup=name == "default_rollup",
                        samplesScannedPerCall=ROLLUP_FUNCS_SAMPLES_SCANNED_PER_CALL.get(name, 0), args=args, args2=args2,
                        removeCounterResets=name in ROLLUP_FUNCS_REMOVE_COUNTER_RESETS, dropStaleNaNs=drop_stale,
                        minStalenessInterval=min_staleness_interval)


def eval_rollup_func(func_name, blocks, start, end, step, window=0, lookback_delta=0, args=None, args2=None,
                     tr_min=storage.INT64_MIN, tr_max=storage.INT64_MAX, out_dev_ptr=None, rc=None):
    """evalRollupFuncNoCache eval.go:1680 -> evalRollupNoIncrementalAggregate eval.go:1845 on device-resident blocks:
    decode, per-series preamble, rollupConfig.Do for every series.
    -> ([nseries x points] np.float64 or None, samplesScanned).  `rc`: a RollupConfig to use instead of the one
    getRollupConfigs derives from func_name."""
    rc = rc or get_rollup_configs(func_name, start, end, step, window, lookback_delta, args, args2)
    cfg = rc._cfg()
    scanned = C.c_uint64(0)
    if out_dev_ptr is not None:
        check(lib().vmb_eval_rollup_device(blocks.ctx.h, blocks.h, tr_min, tr_max, C.byref(cfg), C.c_void_p(int(out_dev_ptr)),
                                           C.byref(scanned)))
        return None, scanned.value
    series, _ = storage.decode_blocks(blocks, tr_min, tr_max)
    try:
        return rc.do_series(series)[0], None
    finally:
        series.close()


def eval_rollup_func_with_subquery(func_name, inner_dev_ptr, nseries, sq_start, sq_end, sq_step, start, end, step, window,
                                   lookback_delta=0, args=None, args2=None, out_dev_ptr=None, ctx=None):
    """evalRollupFuncWithSubquery eval.go:910 with the inner result resident on the device: `inner_dev_ptr` = [nseries x Psq] float64
    on the subquery grid sq_start..sq_end step sq_step (already aligned by the caller, eval.go:932); every row loses its NaN points
    (removeNanValues), goes through the outer function's preFunc and rollupConfig.Do on the outer grid.
    -> ([nseries x points] np.float64 or None, samplesScanned)"""
    rc = get_rollup_configs(func_name, start, end, step, window, lookback_delta, args, args2)
    rc.dropStaleNaNs = False  # the subquery path has no dropStaleNaNs (eval.go:958-964)
    psq = 1 + (sq_end - sq_start) // sq_step
    series = storage.Series.from_matrix(inner_dev_ptr, nseries, psq, sq_start, sq_step, ctx)
    try:
        return rc.do_series(series, out_dev_ptr)
    finally:
        series.close()


def eval_rollup_func_host(func_name, descs, payload, start, end, step, window=0, lookback_delta=0, args=None, args2=None,
                          tr_min=storage.INT64_MIN, tr_max=storage.INT64_MAX, out=None, nseries=None, ctx=None, rc=None):
    """the whole path with HOST buffers in one call (vmb_eval_rollup_host): H2D, decode, rollup, D2H."""
    ctx = ctx or _lib.default_context()
    rc = rc or get_rollup_configs(func_name, start, end, step, window, lookback_delta, args, args2)
    cfg = rc._cfg()
    if isinstance(descs, np.ndarray):
        dptr, n = descs.ctypes.data_as(C.POINTER(_lib.BlockDesc)), descs.shape[0]
        if nseries is None:
            nseries = int(np.count_nonzero(np.diff(descs["series_idx"])) + 1) if n else 0
    else:
        dptr, n = descs, len(descs)
        if nseries is None:
            nseries = len({d.series_idx for d in descs})
    if out is None:
        out = np.empty((nseries, rc.points), dtype=np.float64)
    payload = np.ascontiguousarray(payload, dtype=np.uint8)
    scanned = C.c_uint64(0)
    check(lib().vmb_eval_rollup_host(ctx.h, dptr, n, payload.ctypes.data_as(_lib.u8p), payload.size, tr_min, tr_max,
                                     C.byref(cfg), out.ctypes.data_as(_lib.f64p), None, C.byref(scanned)))
    return out, scanned.value


def eval_rollup_aggr_host(aggr_name, func_name, descs, payload, group_ids, ngroups, start, end, step, window=0,
                          lookback_delta=0, args=None, args2=None, tr_min=storage.INT64_MIN, tr_max=storage.INT64_MAX,
                          out=None, ctx=None, rc=None):
    """aggr(rollup(m[d])) by (...) with HOST buffers in one call (vmb_eval_rollup_aggr_host): H2D, decode, rollup and the
    incremental aggregate on the GPU, D2H of the [ngroups x points] result only -> (np.float64[ngroups, points], samplesScanned)"""
    ctx = ctx or _lib.default_context()
    rc = rc or get_rollup_configs(func_name, start, end, step, window, lookback_delta, args, args2)
    cfg = rc._cfg()
    if isinstance(descs, np.ndarray):
        dptr, n = descs.ctypes.data_as(C.POINTER(_lib.BlockDesc)), descs.shape[0]
    else:
        dptr, n = descs, len(descs)
    if out is None:
        out = np.empty((int(ngroups), rc.points), dtype=np.float64)
    g = np.ascontiguousarray(group_ids, dtype=np.uint32)
    payload = np.ascontiguousarray(payload, dtype=np.uint8)
    scanned = C.c_uint64(0)
    check(lib().vmb_eval_rollup_aggr_host(ctx.h, dptr, n, payload.ctypes.data_as(_lib.u8p), payload.size, tr_min, tr_max,
                                          C.byref(cfg), AGGR_FUNCS[aggr_name.lower()], g.ctypes.data_as(_lib.u32p), int(ngroups),
                                          out.ctypes.data_as(_lib.f64p), None, C.byref(scanned)))
    return out, scanned.value


def eval_rollup_aggr_dist(aggr_name, func_name, blocks, group_ids, ngroups, start, end, step, window=0, lookback_delta=0, args=None,
                          args2=None, tr_min=storage.INT64_MIN, tr_max=storage.INT64_MAX, out=None, rc=None):
    """aggr(rollup(m[d])) by (...) over every rank of the ctx's communicator in ONE library call (vmb_eval_rollup_aggr_dist): this
    rank's device-resident blocks are folded on the GPU, the partial states are merged by the library's NCCL all-reduce, every rank
    finalizes -> (np.float64[ngroups, points], this rank's samplesScanned).  Without a communicator: the single-GPU result."""
    rc = rc or get_rollup_configs(func_name, start, end, step, window, lookback_delta, args, args2)
    cfg = rc._cfg()
    if out is None:
        out = np.empty((int(ngroups), rc.points), dtype=np.float64)
    g = np.ascontiguousarray(group_ids, dtype=np.uint32)
    scanned = C.c_uint64(0)
    check(lib().vmb_eval_rollup_aggr_dist(blocks.ctx.h, blocks.h, tr_min, tr_max, C.byref(cfg), AGGR_FUNCS[aggr_name.lower()],
                                          g.ctypes.data_as(_lib.u32p), int(ngroups), out.ctypes.data_as(_lib.f64p), C.byref(scanned)))
    return out, scanned.value


class IncrementalAggr:
    """incrementalAggrFuncContext aggr_incremental.go:73: aggr(rollup(m[d])) by (...) without keeping [series x points]
    on the host.  update() == updateTimeseries for every series of a device batch (per-GPU partial state);
    finalize() == finalizeTimeseries.  With torch.distributed initialised, finalize(all_reduce=True) merges the per-rank
    partial states with one NCCL all-reduce of values and one of counts (SURVEY.md 8e)."""

    def __init__(self, aggr_name, ngroups, points, device_alloc):
        """device_alloc(nbytes) -> object with .ptr (device address); e.g. a torch.empty(..., device='cuda') wrapper"""
        self.aggr = AGGR_FUNCS[aggr_name.lower()]
        self.name = aggr_name.lower()
        self.ngroups, self.points = int(ngroups), int(points)
        self.values = device_alloc(self.ngroups * self.points * 8)
        self.counts = device_alloc(self.ngroups * self.points * 8)

    def update(self, series, rc, group_ids, rolled_scratch_ptr=None):
        g = np.ascontiguousarray(group_ids, dtype=np.uint32)
        cfg = rc._cfg()
        scanned = C.c_uint64(0)
        check(lib().vmb_rollup_aggr_partial(series.ctx.h, series.h, C.byref(cfg), self.aggr, g.ctypes.data_as(_lib.u32p),
                                            self.ngroups, C.c_void_p(self.values.ptr), C.c_void_p(self.counts.ptr),
                                            C.c_void_p(rolled_scratch_ptr or 0), C.byref(scanned)))
        return scanned.value

    def update_blocks(self, blocks, rc, group_ids, tr_min=storage.INT64_MIN, tr_max=storage.INT64_MAX):
        """decode + preamble + rollup + fold of device-resident compressed blocks in one library call
        (vmb_eval_rollup_aggr_device); the decoded columns stay in a library-side cache"""
        g = np.ascontiguousarray(group_ids, dtype=np.uint32)
        cfg = rc._cfg()
        scanned = C.c_uint64(0)
        check(lib().vmb_eval_rollup_aggr_device(blocks.ctx.h, blocks.h, tr_min, tr_max, C.byref(cfg), self.aggr,
                                                g.ctypes.data_as(_lib.u32p), self.ngroups, C.c_void_p(self.values.ptr),
                                                C.c_void_p(self.counts.ptr), C.byref(scanned)))
        return scanned.value

    def update_host(self, descs, payload, rc, group_ids, ctx, tr_min=storage.INT64_MIN, tr_max=storage.INT64_MAX):
        """the same from HOST buffers through the chunked pipeline (vmb_eval_rollup_aggr_host_partial): the partial state of
        the batch replaces this object's state"""
        g = np.ascontiguousarray(group_ids, dtype=np.uint32)
        cfg = rc._cfg()
        scanned = C.c_uint64(0)
        if isinstance(descs, np.ndarray):
            dptr, n = descs.ctypes.data_as(C.POINTER(_lib.BlockDesc)), descs.shape[0]
        else:
            dptr, n = descs, len(descs)
        payload = np.ascontiguousarray(payload, dtype=np.uint8)
        check(lib().vmb_eval_rollup_aggr_host_partial(ctx.h, dptr, n, payload.ctypes.data_as(_lib.u8p), payload.size, tr_min,
                                                      tr_max, C.byref(cfg), self.aggr, g.ctypes.data_as(_lib.u32p), self.ngroups,
                                                      C.c_void_p(self.values.ptr), C.c_void_p(self.counts.ptr), None,
                                                      C.byref(scanned)))
        return scanned.value

    def finalize(self, ctx, all_reduce=None, out=None):
        """all_reduce(values_buf, counts_buf, op) is called between prepare and finalize when given; `out` may be a
        preallocated (ideally pinned, vmb_host_alloc) [ngroups x points] float64 array"""
        n = self.ngroups * self.points
        if all_reduce is not None:
            check(lib().vmb_aggr_prepare_allreduce(ctx.h, self.aggr, C.c_void_p(self.values.ptr), C.c_void_p(self.counts.ptr), n))
            ctx.synchronize()
            op = {"min": "min", "max": "max", "geomean": "prod"}.get(self.name, "sum")
            all_reduce(self.values, self.counts, op)
        if out is None:
            out = np.empty((self.ngroups, self.points), dtype=np.float64)
        assert out.dtype == np.float64 and out.size == n and out.flags.c_contiguous
        check(lib().vmb_aggr_finalize(ctx.h, self.aggr, C.c_void_p(self.values.ptr), C.c_void_p(self.counts.ptr), n,
                                      out.ctypes.data_as(_lib.f64p)))
        return out


# ---- multi-GPU protocol for aggr(rollup(...)) by (...)  (SURVEY.md 8e) -------------------------------------------------
# all-reduce operator and the identity vmb_aggr_prepare_allreduce writes into empty cells (count == 0), per aggregate
ALLREDUCE_OP = {"sum": "sum", "avg": "sum", "count": "sum", "sum2": "sum", "group": "sum", "min": "min", "max": "max",
                "geomean": "prod"}
ALLREDUCE_IDENTITY = {"sum": 0.0, "avg": 0.0, "count": 0.0, "sum2": 0.0, "group": 0.0, "min": float("inf"),
                      "max": float("-inf"), "geomean": 1.0}


def shard_series(nseries, rank, world):
    """series owned by `rank`: MetricID mod world (independent series => no exchange for decode + rollup)"""
    return np.arange(rank, nseries, world)


def dense_group_ids(group_keys):
    """dense group ids from the marshaled group-by label sets (aggr_incremental.go:113 marshalMetricNameSorted);
    every rank must call this on the SAME global key list so that ids agree across ranks -> (ids, ngroups)"""
    uniq = {}
    ids = np.empty(len(group_keys), dtype=np.uint32)
    for i, k in enumerate(group_keys):
        ids[i] = uniq.setdefault(k, len(uniq))
    return ids, len(uniq)


def torch_all_reduce(values_t, counts_t, op):
    """the `all_reduce` callback for IncrementalAggr.finalize: NCCL (or gloo) all-reduce of values with the aggregate's
    operator and of counts with sum"""
    import torch.distributed as dist
    ops = {"sum": dist.ReduceOp.SUM, "min": dist.ReduceOp.MIN, "max": dist.ReduceOp.MAX, "prod": dist.ReduceOp.PRODUCT}
    dist.all_reduce(values_t, op=ops[op])
    dist.all_reduce(counts_t, op=dist.ReduceOp.SUM)


# ---- multi-output rollups (getRollupConfigs rollup.go:416-504): one input series -> several output series --------------
def get_rollup_configs_multi(func_name, start, end, step, window=0, lookback_delta=0, tag=None, aggr_funcs=None, phis=None,
                             no_stale_markers=False, min_staleness_interval=0):
    """getRollupConfigs rollup.go:374 for rollup(), rollup_rate/deriv/increase/delta(), rollup_scrape_interval(),
    rollup_candlestick(), aggr_over_time() and quantiles_over_time(): -> [RollupConfig], one per output series, TagValue =
    the value of the `rollup` (or phi) label.  The value preFunc (deltaValues / derivValues / intervals) and
    removeCounterResets are shared by the configs and run once per decoded batch."""
    name = func_name.lower()
    rcr = name in ROLLUP_FUNCS_REMOVE_COUNTER_RESETS
    pre = None
    spc = ROLLUP_FUNCS_SAMPLES_SCANNED_PER_CALL.get(name, 0)
    if name in ("rollup", "rollup_rate", "rollup_deriv", "rollup_increase", "rollup_delta", "rollup_scrape_interval"):
        pre = {"rollup_rate": "deriv", "rollup_deriv": "deriv", "rollup_increase": "delta", "rollup_delta": "delta",
               "rollup_scrape_interval": "scrape_interval"}.get(name)
        funcs = {"min": "min_over_time", "max": "max_over_time", "avg": "avg_over_time"}
        if tag in (None, ""):
            pairs = [(funcs[t], t, None) for t in ("min", "max", "avg")]
        elif tag in funcs:
            pairs = [(funcs[tag], "", None)]
        else:
            raise ValueError("unexpected second arg for %s: %r; want `min`, `max` or `avg`" % (func_name, tag))
    elif name == "rollup_candlestick":
        funcs = {"open": "rollup_open", "close": "rollup_close", "low": "rollup_low", "high": "rollup_high"}
        if tag in (None, ""):
            pairs = [(funcs[t], t, None) for t in ("open", "close", "low", "high")]
        elif tag in funcs:
            pairs = [(funcs[tag], tag, None)]
        else:
            raise ValueError("unexpected second arg for %s: %r; want `open`, `close`, `low` or `high`" % (func_name, tag))
    elif name == "aggr_over_time":
        if not aggr_funcs:
            raise ValueError("aggr_over_time() needs at least one aggregate function name")
        pairs = []
        for f in aggr_funcs:
            f = f.lower()
            if f not in ROLLUP_AGGR_FUNCS:
                raise ValueError("%r cannot be used in `aggr_over_time` function" % f)
            rcr = rcr or f in ROLLUP_FUNCS_REMOVE_COUNTER_RESETS
            pairs.append((f, f, None))
    elif name == "quantiles_over_time":
        if not phis:
            raise ValueError("quantiles_over_time() needs at least one phi")
        pairs = [("quantile_over_time", repr(float(p)).rstrip("0").rstrip(".") if float(p) != int(p) else str(int(p)), float(p))
                 for p in phis]
    else:
        raise KeyError("%r is not a multi-output rollup function" % func_name)
    drop_stale = not no_stale_markers
    return [RollupConfig(f, start, end, step, window, lookback_delta,
                         MayAdjustWindow=name in ROLLUP_FUNCS_CAN_ADJUST_WINDOW, isDefaultRollup=False,
                         samplesScannedPerCall=spc, args=arg, removeCounterResets=rcr, dropStaleNaNs=drop_stale,
                         minStalenessInterval=min_staleness_interval, TagValue=t, preFunc=pre) for f, t, arg in pairs]


def eval_rollup_func_multi(func_name, blocks, start, end, step, window=0, lookback_delta=0, tr_min=storage.INT64_MIN,
                           tr_max=storage.INT64_MAX, **kw):
    """evalRollupNoIncrementalAggregate eval.go:1845 for a multi-output rollup on device-resident blocks: decode once, run
    the shared preFunc once, then one rollup per config -> ({TagValue: [nseries x points] np.float64}, samplesScanned)"""
    rcs = get_rollup_configs_multi(func_name, start, end, step, window, lookback_delta, **kw)
    series, _ = storage.decode_blocks(blocks, tr_min, tr_max)
    try:
        out, scanned = {}, 0
        for rc in rcs:
            m, sc = rc.do_series(series)
            out[rc.TagValue] = m
            scanned += sc
        return out, scanned
    finally:
        series.close()


# ---- topk / bottomk over the [series x points] matrix (aggr.go:646 newAggrFuncTopK) -------------------------------------
def topk(ks, vals_dev_ptr, nseries, points, device_alloc, group_ids=None, ngroups=1, reverse=False, ctx=None,
         all_gather=None, group_sizes=None, series_id_base=0):
    """topk(k, q) (reverse=True: bottomk) on a DEVICE matrix [nseries x points] of float64, masked in place: per group and
    point only the k best values survive (fillNaNsAtIdx aggr.go:786).  ks: scalar or one k per point.
    device_alloc(nbytes) -> object with .ptr.  Several processes (series sharded by rank): all_gather(buf, nbytes) ->
    (gathered_buf, nparts) over the candidate lists (all_gather="nccl": the library's own ncclAllGather over the ctx's communicator),
    group_sizes = series per group over ALL processes, series_id_base = global id of this process's row 0 (equal values rank by
    ascending global series id: exactly k survive per group and point).
    -> np.bool_[nseries]: rows that still hold a value (removeEmptySeries drops the others)"""
    ctx = ctx or _lib.default_context()
    g = np.zeros(nseries, dtype=np.uint32) if group_ids is None else np.ascontiguousarray(group_ids, dtype=np.uint32)
    if group_sizes is None:
        group_sizes = np.bincount(g, minlength=ngroups)
    gs = np.ascontiguousarray(group_sizes, dtype=np.uint32)
    kk = np.ascontiguousarray(np.broadcast_to(np.asarray(ks, dtype=np.float64), (points,)))
    kclean = np.where(np.isnan(kk) | (kk < 0), 0.0, kk)
    kmax = int(min(np.floor(kclean.max()) if points else 0, gs.max() if ngroups else 0))
    kmax = max(kmax, 1)
    if kmax > 64:
        raise ValueError("topk on the GPU supports k <= 64 (got %d)" % kmax)
    cells = int(ngroups) * int(points)
    cand = device_alloc(cells * kmax * 16)  # {value, global series id} per entry
    rev = 1 if reverse else 0
    check(lib().vmb_topk_candidates(ctx.h, C.c_void_p(int(vals_dev_ptr)), nseries, points, g.ctypes.data_as(_lib.u32p), int(ngroups),
                                    kmax, rev, int(series_id_base), C.c_void_p(cand.ptr)))
    if all_gather == "nccl":
        nparts = ctx.comm_size
        parts = device_alloc(nparts * cells * kmax * 16)
        check(lib().vmb_topk_allgather(ctx.h, C.c_void_p(cand.ptr), cells * kmax * 2, C.c_void_p(parts.ptr)))
        check(lib().vmb_topk_merge(ctx.h, C.c_void_p(parts.ptr), int(nparts), cells, kmax, rev, C.c_void_p(cand.ptr)))
    elif all_gather is not None:
        ctx.synchronize()
        parts, nparts = all_gather(cand, cells * kmax * 16)
        check(lib().vmb_topk_merge(ctx.h, C.c_void_p(parts.ptr), int(nparts), cells, kmax, rev, C.c_void_p(cand.ptr)))
    flags = np.zeros(max(nseries, 1), dtype=np.uint8)
    check(lib().vmb_topk_apply(ctx.h, C.c_void_p(int(vals_dev_ptr)), nseries, points, g.ctypes.data_as(_lib.u32p), int(ngroups),
                               gs.ctypes.data_as(_lib.u32p), C.c_void_p(cand.ptr), kmax, kk.ctypes.data_as(_lib.f64p), rev,
                               int(series_id_base), flags.ctypes.data_as(_lib.u8p)))
    return flags[:nseries].astype(bool)


# ---- post-rollup operations on device matrices (binary_op.go, aggr.go:1217 quantile, rollup_result_cache.go:618 mergeSeries) ----------
BINARY_OPS = {"+": 0, "-": 1, "*": 2, "/": 3, "%": 4, "^": 5, "atan2": 6, "==": 7, "!=": 8, ">": 9, "<": 10, ">=": 11, "<=": 12,
              "default": 13, "if": 14, "ifnot": 15}


def binary_op(op, left_dev_ptr, right_dev_ptr, npairs, points, dst_dev_ptr, left_rows=None, right_rows=None, is_bool=False, ctx=None):
    """newBinaryOpFunc binary_op.go:155: dst[i] = left[left_rows[i]] op right[right_rows[i]] element by element on DEVICE matrices;
    the row lists come from the host's tag matching (adjustBinaryOpTags), a scalar operand is a one-row matrix with rows all 0"""
    ctx = ctx or _lib.default_context()
    lr = None if left_rows is None else np.ascontiguousarray(left_rows, dtype=np.uint32)
    rr = None if right_rows is None else np.ascontiguousarray(right_rows, dtype=np.uint32)
    check(lib().vmb_binary_op(ctx.h, BINARY_OPS[op.lower()], int(bool(is_bool)), C.c_void_p(int(left_dev_ptr)),
                              lr.ctypes.data_as(_lib.u32p) if lr is not None else None, C.c_void_p(int(right_dev_ptr)),
                              rr.ctypes.data_as(_lib.u32p) if rr is not None else None, int(npairs), int(points), C.c_void_p(int(dst_dev_ptr))))


def merge_series(a_dev_ptr, a_rows, pa, b_dev_ptr, b_rows, pb, dst_dev_ptr, ctx=None):
    """mergeSeries rollup_result_cache.go:618 on DEVICE matrices: dst row i = a[a_rows[i]] ++ b[b_rows[i]], -1 = series missing (NaNs)"""
    ctx = ctx or _lib.default_context()
    ar = np.ascontiguousarray(a_rows, dtype=np.int64)
    br = np.ascontiguousarray(b_rows, dtype=np.int64)
    assert ar.size == br.size
    check(lib().vmb_matrix_merge_rows(ctx.h, C.c_void_p(int(a_dev_ptr)), ar.ctypes.data_as(_lib.i64p), int(pa), C.c_void_p(int(b_dev_ptr)),
                                      br.ctypes.data_as(_lib.i64p), int(pb), ar.size, C.c_void_p(int(dst_dev_ptr))))


def group_first_value(vals_dev_ptr, nseries, points, group_ids, ngroups, out_dev_ptr, ctx=None):
    """the right-hand side of a set operator reduced per tag-set group (vmb_group_first_value): out[g][j] = first non-NaN value of
    the group's rows at point j, in row order"""
    ctx = ctx or _lib.default_context()
    g = np.ascontiguousarray(group_ids, dtype=np.uint32)
    check(lib().vmb_group_first_value(ctx.h, C.c_void_p(int(vals_dev_ptr)), int(nseries), int(points), g.ctypes.data_as(_lib.u32p), int(ngroups),
                                      C.c_void_p(int(out_dev_ptr))))


def set_op(op, left_dev_ptr, left_groups, nleft, right_dev_ptr, right_groups, nright, ngroups, points, dst_dev_ptr, tmp_dev_ptr, ctx=None):
    """`and` (binaryOpAnd binary_op.go:430), `unless` (:610), `if` (:416), `ifnot` (:595), `default` (:463) between two DEVICE matrices
    whose rows the host has keyed by tag set (left_groups / right_groups: dense key ids < ngroups, every left key present on the
    right): the right side is reduced per key into tmp_dev_ptr [ngroups x points], then one element pass over the left rows"""
    el = {"and": "if", "if": "if", "unless": "ifnot", "ifnot": "ifnot", "default": "default"}[op.lower()]
    group_first_value(right_dev_ptr, nright, points, right_groups, ngroups, tmp_dev_ptr, ctx=ctx)
    binary_op(el, left_dev_ptr, tmp_dev_ptr, nleft, points, dst_dev_ptr, right_rows=np.asarray(left_groups, dtype=np.uint32), ctx=ctx)


TRANSFORM_FUNCS = {n: i for i, n in enumerate(
    ["abs", "ceil", "floor", "sqrt", "exp", "ln", "log2", "log10", "sin", "cos", "tan", "asin", "acos", "atan", "sinh", "cosh", "tanh", "asinh",
     "acosh", "atanh", "deg", "rad", "sgn", "clamp", "clamp_min", "clamp_max", "round"])}
TRANSFORM_FUNCS.update({n: 32 + i for i, n in enumerate(
    ["running_sum", "running_min", "running_max", "running_avg", "range_sum", "range_min", "range_max", "range_avg", "range_first",
     "range_last", "keep_last_value", "keep_next_value", "remove_resets", "interpolate", "smooth_exponential"])})
TRANSFORM_FUNCS.update({n: 64 + i for i, n in enumerate(
    ["hour", "minute", "day_of_month", "day_of_week", "day_of_year", "days_in_month", "month", "year", "bitmap_and", "bitmap_or",
     "bitmap_xor"])})


def _go_pow10(n):
    """Go's math.Pow10 (src/math/pow10.go): a PRODUCT / QUOTIENT of two table literals, not the literal 1eN itself for |n| >= 32"""
    if 0 <= n <= 308:
        return float("1e%d" % (n // 32 * 32)) * float("1e%d" % (n % 32))
    if -323 <= n <= 0:
        return float("1e-%d" % ((-n) // 32 * 32)) / float("1e%d" % ((-n) % 32))
    return 0.0 if n < 0 else float("inf")


def transform(name, dev_ptr, nrows, points, *scalar_args, ctx=None):
    """transform.go value functions in place on a DEVICE matrix [nrows x points] (vmb_transform).  scalar_args: the function's scalar
    arguments (numbers or per-point arrays, getScalar): clamp(min, max), clamp_min(min), clamp_max(max), round(nearest = 1),
    smooth_exponential(sf), bitmap_and / bitmap_or / bitmap_xor(w).  The zero-argument date-time forms (`hour()` = `hour(time())`)
    are this call on a one-row matrix of float64(ts) / 1e3 over the query's timestamps (evalTime, eval.go:1959)."""
    ctx = ctx or _lib.default_context()
    name = name.lower()
    bc = lambda x: np.ascontiguousarray(np.broadcast_to(np.asarray(x, dtype=np.float64), (points,)))
    a1 = a2 = None
    if name == "clamp":
        a1, a2 = bc(scalar_args[0]), bc(scalar_args[1])
    elif name in ("clamp_min", "clamp_max", "smooth_exponential", "bitmap_and", "bitmap_or", "bitmap_xor"):
        a1 = bc(scalar_args[0])
    elif name == "round":
        a1 = bc(scalar_args[0] if scalar_args else 1.0)
        # p10 = math.Pow10(-e), (_, e) = decimal.FromFloat(nearest)  transform.go:2341
        uniq, inv = np.unique(a1, return_inverse=True)
        p10u = np.empty(uniq.size)
        for k, n in enumerate(uniq):
            if np.isnan(n) or np.isinf(n) or n == 0:
                p10u[k] = 1.0
                continue
            _, e = decimal.append_float_to_decimal(np.array([n], dtype=np.float64))
            p10u[k] = _go_pow10(-int(e))
        a2 = np.ascontiguousarray(p10u[inv])
    fp = lambda a: a.ctypes.data_as(_lib.f64p) if a is not None else None
    check(lib().vmb_transform(ctx.h, TRANSFORM_FUNCS[name], C.c_void_p(int(dev_ptr)), int(nrows), int(points), fp(a1), fp(a2)))


RANGE_FUNCS = {n: i for i, n in enumerate(
    ["range_stddev", "range_stdvar", "range_zscore", "range_trim_zscore", "range_normalize", "range_linear_regression",
     "range_quantile", "range_mad", "range_trim_outliers", "range_trim_spikes"])}
_RANGE_ONE_ARG = ("range_trim_zscore", "range_quantile", "range_trim_outliers", "range_trim_spikes")


def transform_range(name, dev_ptr, nrows, points, *scalar_args, step=None, ctx=None):
    """transform.go functions that reduce a whole series and rewrite it, in place on a DEVICE matrix [nrows x points]
    (vmb_transform_range).  scalar_args: range_quantile(phi), range_trim_spikes(phi), range_trim_outliers(k), range_trim_zscore(z),
    each a number or a per-point array of which the first value counts (getScalar(...)[0]); range_linear_regression needs the
    query's step in ms.  Returns the np.bool_[nrows] mask of the rows range_normalize keeps, None for the others."""
    ctx = ctx or _lib.default_context()
    name = name.lower()
    args = None
    if name in _RANGE_ONE_ARG:
        args = np.ascontiguousarray(np.asarray(scalar_args[0], dtype=np.float64).reshape(-1)[:1])
    elif name == "range_linear_regression":
        args = np.array([step], dtype=np.float64)
    kept = np.zeros(max(int(nrows), 1), dtype=np.uint8) if name == "range_normalize" else None
    check(lib().vmb_transform_range(ctx.h, RANGE_FUNCS[name], C.c_void_p(int(dev_ptr)), int(nrows), int(points),
                                    args.ctypes.data_as(_lib.f64p) if args is not None else None, 0 if args is None else args.size,
                                    kept.ctypes.data_as(_lib.u8p) if kept is not None else None))
    return kept[:nrows].astype(bool) if kept is not None else None


HISTOGRAM_FUNCS = {"histogram_quantile": 0, "histogram_quantiles": 0, "histogram_share": 1, "histogram_fraction": 2,
                   "histogram_avg": 3, "histogram_stddev": 4, "histogram_stdvar": 5}
_HISTOGRAM_NARGS = {"histogram_quantile": 1, "histogram_share": 1, "histogram_fraction": 2}


def histogram(name, vals_dev_ptr, nrows, points, group_ids, les, ngroups, out_dev_ptr, *scalar_args, lower_dev_ptr=None,
              upper_dev_ptr=None, ctx=None):
    """The histogram functions over `le` buckets (transform.go:634-1169, vmb_histogram) on a DEVICE matrix [nrows x points] of
    bucket series.  group_ids: the dense id of every row's label set without `le`, 0xffffffff for a row without a parsable `le`;
    les: every row's parsed `le`.  scalar_args (numbers or per-point arrays, getScalar): histogram_quantile(phi),
    histogram_quantiles(phi, ...), histogram_share(le), histogram_fraction(lower, upper); none for histogram_avg / stddev / stdvar.
    -> out_dev_ptr [ngroups x points] (histogram_quantiles: [len(phis) x ngroups x points], phi-major); lower_dev_ptr /
    upper_dev_ptr (histogram_quantile and histogram_share, both or neither): the boundsLabel series [ngroups x points].
    Returns the np.bool_ mask of the output rows -- out rows, then lower, then upper -- that hold a value (removeEmptySeries)."""
    ctx = ctx or _lib.default_context()
    name = name.lower()
    g = np.ascontiguousarray(group_ids, dtype=np.uint32)
    le = np.ascontiguousarray(les, dtype=np.float64)
    if g.size != int(nrows) or le.size != int(nrows):
        raise ValueError("%s: need one group id and one le per row (%d rows)" % (name, nrows))
    want = len(scalar_args) if name == "histogram_quantiles" else _HISTOGRAM_NARGS.get(name, 0)
    if len(scalar_args) != want or (name == "histogram_quantiles" and not want):
        raise ValueError("%s: unexpected number of scalar args: %d" % (name, len(scalar_args)))
    args = None
    if want:
        args = np.ascontiguousarray(np.concatenate([np.broadcast_to(np.asarray(a, dtype=np.float64), (points,)) for a in scalar_args]))
    bounds = lower_dev_ptr is not None or upper_dev_ptr is not None
    nout = (want if name == "histogram_quantiles" else 1) * int(ngroups) + (2 * int(ngroups) if bounds else 0)
    flags = np.zeros(max(nout, 1), dtype=np.uint8)
    ptr = lambda p: C.c_void_p(int(p)) if p is not None else None
    check(lib().vmb_histogram(ctx.h, HISTOGRAM_FUNCS[name], C.c_void_p(int(vals_dev_ptr)), int(nrows), int(points),
                              g.ctypes.data_as(_lib.u32p), le.ctypes.data_as(_lib.f64p), int(ngroups),
                              args.ctypes.data_as(_lib.f64p) if args is not None else None, 0 if args is None else args.size,
                              C.c_void_p(int(out_dev_ptr)), ptr(lower_dev_ptr), ptr(upper_dev_ptr), flags.ctypes.data_as(_lib.u8p)))
    return flags[:nout].astype(bool)


_GO_SPECIAL = re.compile(r"[+-]?(inf|infinity)|nan", re.I)
_GO_DEC = re.compile(r"[+-]?([0-9_]+\.?[0-9_]*|\.[0-9_]+)([eE][+-]?[0-9][0-9_]*)?")
_GO_HEX = re.compile(r"[+-]?0[xX]([0-9a-fA-F_]+\.?[0-9a-fA-F_]*|\.[0-9a-fA-F_]+)[pP][+-]?[0-9][0-9_]*")


def _go_underscores_ok(s):
    """underscores only between digits, or between the base prefix and a digit, as in Go's number literals"""
    s = s[1:] if s[:1] in "+-" else s
    saw, i, hexa = "^", 0, False
    if len(s) >= 2 and s[0] == "0" and s[1] in "xX":
        saw, i, hexa = "0", 2, True
    for c in s[i:]:
        if c.isdigit() or (hexa and c in "abcdefABCDEF"):
            saw = "0"
        elif c == "_":
            if saw != "0":
                return False
            saw = "_"
        elif saw == "_":
            return False
        else:
            saw = "!"
    return saw != "_"


def go_parse_float(s):
    """strconv.ParseFloat(s, 64) -> the float, or None where Go returns an error.  Go's strconv source is not part of the
    reference, so this restates Go's published documentation of ParseFloat: decimal and hexadecimal floating-point numbers in
    the syntax of Go's floating-point literals (a hexadecimal one needs its p exponent; underscores may separate digits, as
    in Go literals), rounded to nearest even; "NaN", and "Inf" / "Infinity" with an optional sign, in any case; nothing
    around the number (no spaces).  A number beyond the float64 range is ErrRange (None); one below it rounds to 0."""
    if _GO_SPECIAL.fullmatch(s):
        low = s.lower()
        return float("nan") if low == "nan" else float("-inf") if low[0] == "-" else float("inf")
    hexa = _GO_HEX.fullmatch(s) or None
    m = hexa or _GO_DEC.fullmatch(s)
    if not m or not any(c in string.hexdigits if hexa else c.isdigit() for c in m.group(1)):  # a mantissa digit
        return None
    if "_" in s and not _go_underscores_ok(s):
        return None
    t = s.replace("_", "")
    try:
        v = float.fromhex(t) if hexa else float(t)
    except (OverflowError, ValueError):
        return None
    return None if math.isinf(v) else v


def go_format_float(v, fmt):
    """strconv.FormatFloat(v, fmt, -1, 64) for fmt 'f' and 'g', restated from Go's published documentation: the shortest digits
    that round-trip (Python's repr digits); 'g' uses %e when the decimal exponent is < -4 or >= 6 (the exponent with at least two
    digits, as in 1e+06 and 1.5e-05), 'f' never does (772424014, 0.0000001); NaN, +Inf, -Inf and -0."""
    v = float(v)
    if math.isnan(v):
        return "NaN"
    if math.isinf(v):
        return "+Inf" if v > 0 else "-Inf"
    neg = "-" if math.copysign(1.0, v) < 0 else ""
    if v == 0:
        return neg + "0"
    mant, _, ex = repr(abs(v)).partition("e")
    ip, _, fp = mant.partition(".")
    digits = ip + fp
    ds = digits.rstrip("0")
    e = int(ex or 0) - len(fp) + len(digits) - len(ds)
    ds = ds.lstrip("0")
    dp = len(ds) + e  # value = 0.ds x 10^dp
    if fmt == "g" and not -4 <= dp - 1 < 6:
        x = dp - 1
        return "%s%s%s%se%s%02d" % (neg, ds[0], "." if len(ds) > 1 else "", ds[1:], "-" if x < 0 else "+", abs(x))
    if fmt not in ("f", "g"):
        raise ValueError("go_format_float: format %r" % fmt)
    ip = ds[:dp].ljust(dp, "0") if dp > 0 else "0"
    frac = ("0" * -dp + ds) if dp < 0 else ds[dp:]
    return neg + ip + ("." + frac if frac else "")


def count_values(label, vals_dev_ptr, nseries, points, group_ids, ngroups, device_alloc, ctx=None):
    """count_values("label", q) by (...) (the afe closure of aggr.go:594, vmb_count_values) on a DEVICE matrix [nseries x points].
    group_ids: the dense id of every row's label set after removing `label` from by (...) or adding it to without (...).
    device_alloc(nbytes) -> object with .ptr.  -> (out, n, groups, tags): out holds [n x points] (sized by a first call that only
    counts, which a caller compares with -search.maxSeriesPerAggrFunc), groups the group of every output row (np.int64), tags the
    (label, strconv.FormatFloat(v, 'f', -1, 64)) tag every output row adds to its group's labels."""
    ctx = ctx or _lib.default_context()
    g = np.ascontiguousarray(group_ids, dtype=np.uint32)
    if g.size != int(nseries):
        raise ValueError("count_values: need one group id per series (%d series)" % nseries)
    nout = C.c_size_t(0)
    grp, val = np.zeros(1, dtype=np.uint32), np.zeros(1)

    def call(out_ptr):
        return lib().vmb_count_values(ctx.h, C.c_void_p(int(vals_dev_ptr)), int(nseries), int(points), g.ctypes.data_as(_lib.u32p),
                                      int(ngroups), out_ptr, C.byref(nout), grp.ctypes.data_as(_lib.u32p), val.ctypes.data_as(_lib.f64p))
    check(call(None), allow=(-54,))  # VMB_ERR_CAP: the count
    rows = nout.value
    grp, val = np.zeros(max(rows, 1), dtype=np.uint32), np.zeros(max(rows, 1))
    out = device_alloc(max(rows * int(points) * 8, 8))
    if rows:
        check(call(C.c_void_p(int(out.ptr))))
    return out, rows, grp[:rows].astype(np.int64), [(label, go_format_float(v, "f")) for v in val[:rows].tolist()]


def count_values_over_time_config(start, end, step, window=0, lookback_delta=0, no_stale_markers=False, min_staleness_interval=0):
    """the rollupConfig getRollupConfigs (rollup.go:374) makes for count_values_over_time: no window adjustment, no preFunc,
    dropStaleNaNs unless the series hold no staleness markers.  func_id is not read by vmb_rollup_count_values."""
    flags = 0 if no_stale_markers else RC_DROP_STALE_NANS
    if int(step) <= 0 or int(start) > int(end) or int(window) < 0:
        raise ValueError("BUG: invalid rollupConfig: Step=%d Start=%d End=%d Window=%d" % (step, start, end, window))
    return RollupCfg(0, flags, int(start), int(end), int(step), int(window), int(lookback_delta), int(min_staleness_interval), 0, 0,
                     None, None)


def count_values_over_time(label, series, start, end, step, window, lookback_delta=0, device_alloc=None, ctx=None,
                           no_stale_markers=False):
    """count_values_over_time("label", m[window]) (newRollupCountValues rollup.go:1490 through rollupConfig.DoTimeseriesMap,
    vmb_rollup_count_values) on a device batch (storage.Series); the series preamble runs in place on it.
    device_alloc(nbytes) -> object with .ptr.  -> (out, n, series_idx, tags, samples_scanned): out holds [n x points], series_idx
    the input series of every output row (np.int64), tags the (label, strconv.FormatFloat(v, 'g', -1, 64)) tag it adds to that
    series' labels."""
    if device_alloc is None:
        raise ValueError("count_values_over_time: device_alloc is required")
    ctx = ctx or series.ctx
    cfg = count_values_over_time_config(start, end, step, window, lookback_delta, no_stale_markers)
    points = 1 + (int(end) - int(start)) // int(step)
    nout = C.c_size_t(0)
    scanned = C.c_uint64(0)
    ser, val = np.zeros(1, dtype=np.uint32), np.zeros(1)

    def call(out_ptr):
        return lib().vmb_rollup_count_values(ctx.h, series.h, C.byref(cfg), out_ptr, C.byref(nout), ser.ctypes.data_as(_lib.u32p),
                                             val.ctypes.data_as(_lib.f64p), C.byref(scanned))
    check(call(None), allow=(-54,))
    rows = nout.value
    ser, val = np.zeros(max(rows, 1), dtype=np.uint32), np.zeros(max(rows, 1))
    out = device_alloc(max(rows * points * 8, 8))
    check(call(C.c_void_p(int(out.ptr))))
    return out, rows, ser[:rows].astype(np.int64), [(label, go_format_float(v, "g")) for v in val[:rows].tolist()], scanned.value


VR_KEEP = 0xFFFFFFFE  # VMB_VR_KEEP
VR_KINDS = ["kept", "bucket", "gap", "+Inf"]  # enum vmb_vr_kind


def prometheus_buckets(vals_dev_ptr, nrows, points, vmranges, has_le, group_ids, device_alloc, ctx=None):
    """prometheus_buckets (vmrangeBucketsToLE, transform.go:494, vmb_vmrange_to_le) on a DEVICE matrix [nrows x points].
    vmranges: every row's `vmrange` label, None (or "") where it has none; has_le: whether the row has a non-empty `le`;
    group_ids: the dense id of every row's label set without `vmrange` and `le` (read for rows with a valid vmrange).
    device_alloc(nbytes) -> object with .ptr.  -> (out, n, src, kinds, les): out holds [n x points] (sized by a first call that
    only counts); per output row: src, the input row it comes from (a gap or +Inf row takes its labels); kinds, an index into
    VR_KINDS; les, its `le` string (None for a kept row, which keeps its own `le`)."""
    ctx = ctx or _lib.default_context()
    n = int(nrows)
    if len(vmranges) != n or len(has_le) != n or len(group_ids) != n:
        raise ValueError("prometheus_buckets: need one vmrange, has_le and group id per row (%d rows)" % n)
    gids = np.full(n, 0xFFFFFFFF, dtype=np.uint32)
    starts, ends = np.zeros(n), np.zeros(n)
    skeys, ekeys = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint32)
    strings, ids = [], {}

    def key(s):
        if s not in ids:
            ids[s] = len(strings)
            strings.append(s)
        return ids[s]
    for i, vr in enumerate(vmranges):
        if not vr:
            if has_le[i]:
                gids[i] = VR_KEEP
            continue
        k = vr.find("...")
        if k < 0:
            continue
        a, b = vr[:k], vr[k + 3:]
        fa, fb = go_parse_float(a), go_parse_float(b)
        if fa is None or fb is None:
            continue
        gids[i], starts[i], ends[i], skeys[i], ekeys[i] = int(group_ids[i]), fa, fb, key(a), key(b)
    return _vmrange_to_le(vals_dev_ptr, n, points, gids, starts, ends, skeys, ekeys, strings, device_alloc, ctx)


def _vmrange_to_le(vals_dev_ptr, n, points, gids, starts, ends, skeys, ekeys, strings, device_alloc, ctx):
    """vmb_vmrange_to_le with the rows' group ids, parsed bounds and string ids -> what prometheus_buckets returns"""
    grouped = gids[gids < VR_KEEP]
    ngroups = int(grouped.max()) + 1 if grouped.size else 0
    nout = C.c_size_t(0)
    src, kind, le = (np.zeros(1, dtype=np.uint32), np.zeros(1, dtype=np.uint8), np.zeros(1, dtype=np.uint32))
    u32 = lambda a: a.ctypes.data_as(_lib.u32p)
    f64 = lambda a: a.ctypes.data_as(_lib.f64p)

    def call(out_ptr):
        return lib().vmb_vmrange_to_le(ctx.h, C.c_void_p(int(vals_dev_ptr)), n, int(points), u32(gids), f64(starts), f64(ends),
                                       u32(skeys), u32(ekeys), ngroups, out_ptr, C.byref(nout), u32(src),
                                       kind.ctypes.data_as(_lib.u8p), u32(le))
    check(call(None), allow=(-54,))  # VMB_ERR_CAP: the count
    rows = nout.value
    src, kind, le = (np.zeros(max(rows, 1), dtype=np.uint32), np.zeros(max(rows, 1), dtype=np.uint8),
                     np.zeros(max(rows, 1), dtype=np.uint32))
    out = device_alloc(max(rows * int(points) * 8, 8))
    if rows:
        check(call(C.c_void_p(int(out.ptr))))
    les = [None if k == 0 else "+Inf" if k == 3 else strings[x] for k, x in zip(kind[:rows].tolist(), le[:rows].tolist())]
    return out, rows, src[:rows].astype(np.int64), kind[:rows].copy(), les


VMH_NB = 488  # bucket numbers of vmb_aggr_histogram / vmb_rollup_histogram: 0 lower, 1 + idx decimal, 487 upper
_VMRANGE_TABLE = None


def vmrange_table():
    """The `vmrange` label of every bucket number, as metrics.Histogram names its buckets (histogram.go:220, initBucketRanges:
    v = Pow10(-9), then v *= Pow(10, 1/18) once per bucket, every bound formatted %.3e; lowerBucketRange "0...1.000e-09" and
    upperBucketRange "1.000e+18...+Inf").  Built once.  -> dict with
      labels[488]                    the label of every bucket number
      strings                        the distinct bound strings: "0", the 487 decimal bounds (adjacent buckets share one), "+Inf"
      start_ids, end_ids  uint32[488] every bucket's start / end as an index into strings (the ids vmb_vmrange_to_le takes)
      starts, ends       float64[488] those strings parsed by strconv.ParseFloat, as vmrangeBucketsToLE parses them"""
    global _VMRANGE_TABLE
    if _VMRANGE_TABLE is None:
        v, mult = 1e-9, 10.0 ** (1.0 / 18)
        bounds = ["%.3e" % v]
        for _ in range(VMH_NB - 2):
            v *= mult
            bounds.append("%.3e" % v)
        strings = ["0"] + bounds + ["+Inf"]
        start_ids = np.arange(VMH_NB, dtype=np.uint32)  # bucket b starts at strings[b] ("0" for the lower bucket)
        end_ids = start_ids + 1
        parsed = np.array([go_parse_float(x) for x in strings])
        _VMRANGE_TABLE = dict(labels=[strings[a] + "..." + strings[a + 1] for a in range(VMH_NB)], strings=strings,
                              start_ids=start_ids, end_ids=end_ids, starts=parsed[start_ids], ends=parsed[end_ids])
    return _VMRANGE_TABLE


def aggr_histogram_vmrange(vals_dev_ptr, nseries, points, group_ids, ngroups, device_alloc, ctx=None):
    """histogram(q) by (...) up to its vmrangeBucketsToLE (aggrFuncHistogram aggr.go:256, vmb_aggr_histogram) on a DEVICE matrix
    [nseries x points].  group_ids: the dense id of every row's label set after the by (...) / without (...) grouping.
    device_alloc(nbytes) -> object with .ptr.  -> (out, n, groups, buckets): out holds [n x points] counts (0 where none), groups
    and buckets (np.int64) the group and bucket number of every row; vmrange_table()["labels"] names the buckets."""
    ctx = ctx or _lib.default_context()
    g = np.ascontiguousarray(group_ids, dtype=np.uint32)
    if g.size != int(nseries):
        raise ValueError("histogram: need one group id per series (%d series)" % nseries)
    nout = C.c_size_t(0)
    grp, bkt = np.zeros(1, dtype=np.uint32), np.zeros(1, dtype=np.uint32)

    def call(out_ptr):
        return lib().vmb_aggr_histogram(ctx.h, C.c_void_p(int(vals_dev_ptr)), int(nseries), int(points), g.ctypes.data_as(_lib.u32p),
                                        int(ngroups), out_ptr, C.byref(nout), grp.ctypes.data_as(_lib.u32p),
                                        bkt.ctypes.data_as(_lib.u32p))
    check(call(None), allow=(-54,))  # VMB_ERR_CAP: the count
    rows = nout.value
    grp, bkt = np.zeros(max(rows, 1), dtype=np.uint32), np.zeros(max(rows, 1), dtype=np.uint32)
    out = device_alloc(max(rows * int(points) * 8, 8))
    if rows:
        check(call(C.c_void_p(int(out.ptr))))
    return out, rows, grp[:rows].astype(np.int64), bkt[:rows].astype(np.int64)


def aggr_histogram(vals_dev_ptr, nseries, points, group_ids, ngroups, device_alloc, ctx=None):
    """histogram(q) by (...) (aggrFuncHistogram aggr.go:256) on a DEVICE matrix [nseries x points]: vmb_aggr_histogram, then its
    vmrangeBucketsToLE through vmb_vmrange_to_le as prometheus_buckets runs it, the bounds' string ids from vmrange_table().
    -> (out, n, groups, les): out holds the [n x points] `le` rows, groups the group of every row (np.int64), les its `le`."""
    ctx = ctx or _lib.default_context()
    vr, n, groups, buckets = aggr_histogram_vmrange(vals_dev_ptr, nseries, points, group_ids, ngroups, device_alloc, ctx)
    t = vmrange_table()
    out, rows, src, _, les = _vmrange_to_le(vr.ptr, n, points, groups.astype(np.uint32), t["starts"][buckets], t["ends"][buckets],
                                            t["start_ids"][buckets], t["end_ids"][buckets], t["strings"], device_alloc, ctx)
    return out, rows, groups[src], les


def histogram_over_time(series, start, end, step, window, lookback_delta=0, device_alloc=None, ctx=None, no_stale_markers=False):
    """histogram_over_time(m[window]) (rollupHistogram rollup.go:1526 through rollupConfig.DoTimeseriesMap, vmb_rollup_histogram)
    on a device batch (storage.Series); the series preamble runs in place on it.  Its rollupConfig is count_values_over_time's.
    device_alloc(nbytes) -> object with .ptr.  -> (out, n, series_idx, vmranges, samples_scanned): out holds [n x points] (NaN
    where a bucket has no sample in the window), series_idx the input series of every output row (np.int64), vmranges the
    `vmrange` label it adds to that series' labels."""
    if device_alloc is None:
        raise ValueError("histogram_over_time: device_alloc is required")
    ctx = ctx or series.ctx
    cfg = count_values_over_time_config(start, end, step, window, lookback_delta, no_stale_markers)
    points = 1 + (int(end) - int(start)) // int(step)
    nout = C.c_size_t(0)
    scanned = C.c_uint64(0)
    ser, bkt = np.zeros(1, dtype=np.uint32), np.zeros(1, dtype=np.uint32)

    def call(out_ptr):
        return lib().vmb_rollup_histogram(ctx.h, series.h, C.byref(cfg), out_ptr, C.byref(nout), ser.ctypes.data_as(_lib.u32p),
                                          bkt.ctypes.data_as(_lib.u32p), C.byref(scanned))
    check(call(None), allow=(-54,))
    rows = nout.value
    ser, bkt = np.zeros(max(rows, 1), dtype=np.uint32), np.zeros(max(rows, 1), dtype=np.uint32)
    out = device_alloc(max(rows * points * 8, 8))
    check(call(C.c_void_p(int(out.ptr))))
    labels = vmrange_table()["labels"]
    return out, rows, ser[:rows].astype(np.int64), [labels[b] for b in bkt[:rows].tolist()], scanned.value


def buckets_limit(limit, vals_dev_ptr, nrows, points, group_ids, les, ngroups, ctx=None):
    """buckets_limit(limit, buckets) (transform.go:386, vmb_buckets_limit) on a DEVICE `le` matrix [nrows x points], usually
    the output of prometheus_buckets.  group_ids: the dense id of every row's label set without `le`, 0xffffffff for a row
    without a parsable `le`; les: every row's parsed `le`.  -> the rows kept, in output order (np.int64); the matrix is not
    changed."""
    ctx = ctx or _lib.default_context()
    g = np.ascontiguousarray(group_ids, dtype=np.uint32)
    le = np.ascontiguousarray(les, dtype=np.float64)
    if g.size != int(nrows) or le.size != int(nrows):
        raise ValueError("buckets_limit: need one group id and one le per row (%d rows)" % nrows)
    rows = np.zeros(max(int(nrows), 1), dtype=np.uint32)
    nout = C.c_size_t(rows.size)
    check(lib().vmb_buckets_limit(ctx.h, C.c_void_p(int(vals_dev_ptr)), int(nrows), int(points), g.ctypes.data_as(_lib.u32p),
                                  le.ctypes.data_as(_lib.f64p), int(ngroups), int(limit), rows.ctypes.data_as(_lib.u32p),
                                  C.byref(nout)))
    return rows[:nout.value].astype(np.int64)


MATRIX_AGGR_FUNCS ={n: i for i, n in enumerate(
    ["sum", "sum2", "min", "max", "avg", "count", "group", "geomean", "stddev", "stdvar", "share", "zscore"])}


def aggr_matrix(name, vals_dev_ptr, nseries, points, out_dev_ptr, group_ids=None, ngroups=1, limit=0, ctx=None):
    """aggr(q) by (...) [limit N] (aggrFuncExt aggr.go:110) on a DEVICE matrix [nseries x points] for any argument q: sum, sum2, min,
    max, avg, count, group, geomean, stddev, stdvar -> out_dev_ptr [ngroups x points]; share, zscore -> out_dev_ptr [nseries x points]
    (may be vals_dev_ptr).  Returns the ids of the groups the reference outputs (those with a non-empty row), in order of their first
    non-empty row and cut at `limit` (0 = no limit); for share / zscore the np.bool_[nseries] mask of the rows it returns instead."""
    ctx = ctx or _lib.default_context()
    g = np.zeros(nseries, dtype=np.uint32) if group_ids is None else np.ascontiguousarray(group_ids, dtype=np.uint32)
    flags = np.zeros(max(nseries, 1), dtype=np.uint8)
    check(lib().vmb_aggr_matrix(ctx.h, MATRIX_AGGR_FUNCS[name.lower()], C.c_void_p(int(vals_dev_ptr)), int(nseries), int(points),
                                g.ctypes.data_as(_lib.u32p), int(ngroups), C.c_void_p(int(out_dev_ptr)), flags.ctypes.data_as(_lib.u8p)))
    nonempty = flags[:nseries].astype(bool)
    _, first = np.unique(g[nonempty], return_index=True)  # aggrPrepareSeries aggr.go:139: groups in order of first non-empty row
    groups = g[nonempty][np.sort(first)]
    if limit > 0:
        groups = groups[:limit]
    if name.lower() in ("share", "zscore"):
        return nonempty & np.isin(g, groups)
    return groups


ORDER_AGGR_FUNCS = {n: i for i, n in enumerate(["quantiles", "mad", "mode", "distinct", "outliers_iqr", "outliers_mad"])}


def aggr_order(name, vals_dev_ptr, nseries, points, out_dev_ptr=None, group_ids=None, ngroups=1, phis=None, tolerance=None, limit=0,
               ctx=None):
    """The order-statistic aggregates by (...) [limit N] (aggrFuncExt aggr.go:110) on a DEVICE matrix [nseries x points], any group
    size: quantiles(phis) -> out_dev_ptr [len(phis) x ngroups x points] (phi-major); mad, mode, distinct -> out_dev_ptr [ngroups x
    points]; outliers_iqr, outliers_mad(tolerance) write no matrix.  phis and tolerance: a number or an array (tolerance: one per
    point).  Returns the ids of the groups the reference outputs, in order of their first non-empty row and cut at `limit` (0 = no
    limit); for outliers_iqr / outliers_mad the np.bool_[nseries] mask of the rows it returns instead."""
    ctx = ctx or _lib.default_context()
    name = name.lower()
    g = np.zeros(nseries, dtype=np.uint32) if group_ids is None else np.ascontiguousarray(group_ids, dtype=np.uint32)
    args = None
    if name == "quantiles":
        args = np.ascontiguousarray(np.asarray(phis, dtype=np.float64).reshape(-1))
    elif name == "outliers_mad":
        args = np.ascontiguousarray(np.broadcast_to(np.asarray(tolerance, dtype=np.float64), (points,)))
    nonempty = np.zeros(max(nseries, 1), dtype=np.uint8)
    selected = np.zeros(max(nseries, 1), dtype=np.uint8)
    check(lib().vmb_aggr_order(ctx.h, ORDER_AGGR_FUNCS[name], C.c_void_p(int(vals_dev_ptr)), int(nseries), int(points),
                               g.ctypes.data_as(_lib.u32p), int(ngroups), args.ctypes.data_as(_lib.f64p) if args is not None else None,
                               0 if args is None else args.size, C.c_void_p(int(out_dev_ptr or 0)), nonempty.ctypes.data_as(_lib.u8p),
                               selected.ctypes.data_as(_lib.u8p)))
    ne = nonempty[:nseries].astype(bool)
    _, first = np.unique(g[ne], return_index=True)  # aggrPrepareSeries aggr.go:139: groups in order of first non-empty row
    groups = g[ne][np.sort(first)]
    if limit > 0:
        groups = groups[:limit]
    if name in ("outliers_iqr", "outliers_mad"):
        return selected[:nseries].astype(bool) & np.isin(g, groups)
    return groups


RANK_FUNCS = {n: i for i, n in enumerate(["min", "max", "avg", "median", "last", "outliersk"])}
RANK_AGGR_NAMES = ["%s_%s" % (t, s) for t in ("topk", "bottomk") for s in ("min", "max", "avg", "median", "last")] + ["outliersk"]


def aggr_rank(name, ks, vals_dev_ptr, nseries, points, group_ids=None, ngroups=1, remaining_dev_ptr=None, limit=0, ctx=None):
    """topk_min / topk_max / topk_avg / topk_median / topk_last(k, q [, "remaining_sum"]) by (...) [limit N], their bottomk_* twins
    (getRangeTopKTimeseries aggr.go:704) and outliersk(k, q) (:1040) on a DEVICE matrix [nseries x points] (vmb_aggr_rank).  ks: a
    number or one k per point.  The surviving rows are masked in place (NaN where a row is not among the point's k best of its
    group); every other row stays as it was.  remaining_dev_ptr: [ngroups x points] for the remaining-sum rows (the third argument;
    not for outliersk).  -> (out, scores): out (np.int64) lists the reference's output, groups in order of their first non-empty
    row and cut at `limit` (0 = no limit), per group -(g + 1) for the remaining-sum row of group g where it holds a value, then
    the surviving rows from best to worst; scores: every row's score."""
    ctx = ctx or _lib.default_context()
    name = name.lower()
    if name not in RANK_AGGR_NAMES:
        raise ValueError("aggr_rank: unknown function %r" % name)
    g = np.zeros(nseries, dtype=np.uint32) if group_ids is None else np.ascontiguousarray(group_ids, dtype=np.uint32)
    k = np.ascontiguousarray(np.broadcast_to(np.asarray(ks, dtype=np.float64), (points,)))
    rem_ne = np.zeros(max(int(ngroups), 1), dtype=np.uint8)
    nonempty = np.zeros(max(nseries, 1), dtype=np.uint8)
    rows = np.zeros(max(nseries, 1), dtype=np.uint32)
    counts = np.zeros(max(int(ngroups), 1), dtype=np.uint32)
    scores = np.full(max(nseries, 1), np.nan)
    u8 = lambda a: a.ctypes.data_as(_lib.u8p)
    u32 = lambda a: a.ctypes.data_as(_lib.u32p)
    check(lib().vmb_aggr_rank(ctx.h, RANK_FUNCS[name.split("_")[-1]], int(name.startswith("bottomk_")), C.c_void_p(int(vals_dev_ptr)),
                              int(nseries), int(points), u32(g), int(ngroups), k.ctypes.data_as(_lib.f64p),
                              C.c_void_p(int(remaining_dev_ptr or 0)), u8(rem_ne) if remaining_dev_ptr else None, u8(nonempty),
                              u32(rows), u32(counts), scores.ctypes.data_as(_lib.f64p)))
    ne = nonempty[:nseries].astype(bool)
    _, first = np.unique(g[ne], return_index=True)  # aggrPrepareSeries aggr.go:139: groups in order of first non-empty row
    groups = g[ne][np.sort(first)]
    if limit > 0:
        groups = groups[:limit]
    starts = np.concatenate([[0], np.cumsum(counts[:ngroups], dtype=np.int64)])
    out = []
    for gid in groups.tolist():
        if rem_ne[gid]:
            out.append(-(gid + 1))
        out.extend(rows[starts[gid]:starts[gid + 1]].tolist())
    return np.array(out, dtype=np.int64), scores[:nseries]


def aggr_quantile(phis, vals_dev_ptr, nseries, points, out_dev_ptr, group_ids=None, ngroups=1, ctx=None):
    """quantile(phi, q) by (...) / median (phi = 0.5)  aggr.go:1217 on a DEVICE matrix -> out_dev_ptr [ngroups x points]"""
    ctx = ctx or _lib.default_context()
    g = np.zeros(nseries, dtype=np.uint32) if group_ids is None else np.ascontiguousarray(group_ids, dtype=np.uint32)
    ph = np.ascontiguousarray(np.broadcast_to(np.asarray(phis, dtype=np.float64), (points,)))
    check(lib().vmb_aggr_quantile(ctx.h, C.c_void_p(int(vals_dev_ptr)), int(nseries), int(points), g.ctypes.data_as(_lib.u32p), int(ngroups),
                                  ph.ctypes.data_as(_lib.f64p), C.c_void_p(int(out_dev_ptr))))


def _metric_name_key(labels):
    """marshalMetricNameSorted (binary_op.go): labels, `__name__` included, as one comparable key"""
    return tuple(sorted(labels.items()))


def _metric_name_order(labels):
    """metricNameLess exec.go:167: the metric group, then the sorted tags (a prefix first)"""
    return (labels.get("__name__", ""), tuple(sorted((k, v) for k, v in labels.items() if k != "__name__")))


def _gather(src_dev_ptr, rows, points, out_dev_ptr, ctx):
    """out rows = src rows `rows` (vmb_matrix_merge_rows with pb = 0)"""
    rows = np.asarray(rows, dtype=np.int64)
    if rows.size and points:
        merge_series(src_dev_ptr, rows, points, 0, np.zeros(rows.size, dtype=np.int64), 0, out_dev_ptr, ctx=ctx)


def rows_nonempty(vals_dev_ptr, nrows, points, ctx=None):
    """removeEmptySeries exec.go:193 on a DEVICE matrix [nrows x points] (vmb_rows_nonempty): np.bool_[nrows], True where the
    row holds a non-NaN value"""
    ctx = ctx or _lib.default_context()
    flags = np.zeros(max(int(nrows), 1), dtype=np.uint8)
    check(lib().vmb_rows_nonempty(ctx.h, C.c_void_p(int(vals_dev_ptr or 0)), int(nrows), int(points), flags.ctypes.data_as(_lib.u8p)))
    return flags[:int(nrows)].astype(bool)


def sort_rows(vals_dev_ptr, nrows, points, desc=False, out_dev_ptr=None, ctx=None):
    """sort(q) / sort_desc(q) (newTransformFuncSort transform.go:2557, vmb_sort_rows) on a DEVICE matrix [nrows x points]:
    -> the rows in output order (np.int64), gathered into out_dev_ptr [nrows x points] when it is given"""
    ctx = ctx or _lib.default_context()
    order = np.zeros(max(int(nrows), 1), dtype=np.uint32)
    check(lib().vmb_sort_rows(ctx.h, C.c_void_p(int(vals_dev_ptr or 0)), int(nrows), int(points), int(bool(desc)),
                              order.ctypes.data_as(_lib.u32p)))
    order = order[:int(nrows)].astype(np.int64)
    if out_dev_ptr is not None:
        _gather(vals_dev_ptr, order, points, out_dev_ptr, ctx)
    return order


def drop_empty_series(vals_dev_ptr, nrows, points, out_dev_ptr=None, ctx=None):
    """drop_empty_series(q) transform.go:1939: -> the rows that hold a value (np.int64), gathered into out_dev_ptr if given"""
    rows = np.flatnonzero(rows_nonempty(vals_dev_ptr, nrows, points, ctx=ctx)).astype(np.int64)
    if out_dev_ptr is not None:
        _gather(vals_dev_ptr, rows, points, out_dev_ptr, ctx or _lib.default_context())
    return rows


def limit_offset(limit, offset, vals_dev_ptr, nrows, points, out_dev_ptr=None, ctx=None):
    """limit_offset(limit, offset, q) transform.go:2275: the empty rows removed first, then `offset` rows skipped, then at most
    `limit` kept -> those rows (np.int64), gathered into out_dev_ptr if given"""
    if int(limit) < 0 or int(offset) < 0:
        raise ValueError("limit_offset: limit and offset must not be negative")
    rows = np.flatnonzero(rows_nonempty(vals_dev_ptr, nrows, points, ctx=ctx)).astype(np.int64)
    rows = rows[int(offset):int(offset) + int(limit)]
    if out_dev_ptr is not None:
        _gather(vals_dev_ptr, rows, points, out_dev_ptr, ctx or _lib.default_context())
    return rows


def union(args, points, out_dev_ptr=None, ctx=None):
    """union(q1, ...) transform.go:1725.  args: one (dev_ptr, labels of every row) per argument, labels a dict with `__name__`.
    -> [(arg, row)]: every scalar argument (one unnamed row each) when all of them are scalars, else the first row of every metric
    name in argument order; gathered into out_dev_ptr [len x points] if given"""
    ctx = ctx or _lib.default_context()
    if all(len(lb) == 1 and not lb[0] for _, lb in args):
        out = [(j, 0) for j in range(len(args))]
    else:
        seen, out = set(), []
        for j, (_, labels) in enumerate(args):
            for i, lb in enumerate(labels):
                k = _metric_name_key(lb)
                if k not in seen:
                    seen.add(k)
                    out.append((j, i))
    if out_dev_ptr is not None:
        at = 0
        for j, (ptr, _) in enumerate(args):
            rows = [i for a, i in out if a == j]
            _gather(ptr, rows, points, int(out_dev_ptr) + at * int(points) * 8, ctx)
            at += len(rows)
    return out


def _tagset_key(labels, on, ignoring, keep_metric_names):
    """the map key of createTimeseriesMapByTagSet binary_op.go:657 (RemoveTagsOn / RemoveTagsIgnoring)"""
    d = dict(labels)
    if not keep_metric_names:
        d.pop("__name__", None)
    if on is not None:
        d = {k: v for k, v in d.items() if k in on}
    elif ignoring:
        d = {k: v for k, v in d.items() if k not in ignoring}
    return _metric_name_key(d)


def set_or(left_dev_ptr, left_labels, right_dev_ptr, right_labels, points, out_dev_ptr=None, on=None, ignoring=(),
           keep_metric_names=False, ctx=None):
    """q1 or q2 (binaryOpOr binary_op.go:483, vmb_set_or) on two DEVICE matrices, filled in place.  left_labels / right_labels: a
    dict per row, `__name__` included; on / ignoring: the group modifier's labels.  -> [(side, row)] in output order, side 0 for
    the left matrix and 1 for the right: the left rows with a value sorted by metric name, then the right rows added (all of a key
    the left side lacks, the ones still holding a value of the others) sorted by metric name.  Gathered into out_dev_ptr
    [len x points] if given."""
    ctx = ctx or _lib.default_context()
    nl, nr = len(left_labels), len(right_labels)
    keys, names = {}, {}
    kid = lambda lb: keys.setdefault(_tagset_key(lb, on, ignoring, keep_metric_names), len(keys))
    nid = lambda lb: names.setdefault(_metric_name_key(lb), len(names))
    lk = np.array([kid(lb) for lb in left_labels], dtype=np.uint32)
    rk = np.array([kid(lb) for lb in right_labels], dtype=np.uint32)
    ln = np.array([nid(lb) for lb in left_labels], dtype=np.uint32)
    rn = np.array([nid(lb) for lb in right_labels], dtype=np.uint32)
    # the scalar fast path (:543): a key whose right side is one unnamed row merges only with a single unnamed non-empty left row
    rcount = np.bincount(rk, minlength=len(keys)) if nr else np.zeros(len(keys), dtype=np.int64)
    unnamed = nid({})
    lne_pre = None
    for r in range(nr):
        k = rk[r]
        if rcount[k] != 1 or right_labels[r]:
            continue
        left_rows = np.flatnonzero(lk == k)
        if not (ln[left_rows] == unnamed).any():
            continue  # no left row has the id: nothing merges either way
        if lne_pre is None:
            lne_pre = rows_nonempty(left_dev_ptr, nl, points, ctx=ctx)
        live = left_rows[lne_pre[left_rows]]
        if not (live.size == 1 and ln[live[0]] == unnamed):
            rn[r] = len(names) + r  # an id no left row has
    lne, rne = np.zeros(max(nl, 1), dtype=np.uint8), np.zeros(max(nr, 1), dtype=np.uint8)
    u32 = lambda a: np.ascontiguousarray(a, dtype=np.uint32).ctypes.data_as(_lib.u32p)
    check(lib().vmb_set_or(ctx.h, C.c_void_p(int(left_dev_ptr or 0)), nl, u32(lk), u32(ln), C.c_void_p(int(right_dev_ptr or 0)), nr,
                           u32(rk), u32(rn), len(keys), int(points), lne.ctypes.data_as(_lib.u8p), rne.ctypes.data_as(_lib.u8p)))
    left_keys = set(lk.tolist())
    kept = [i for i in range(nl) if lne[i]]
    added = [i for i in range(nr) if rk[i] not in left_keys or rne[i]]
    kept.sort(key=lambda i: (_metric_name_order(left_labels[i]), i))
    added.sort(key=lambda i: (_metric_name_order(right_labels[i]), i))
    if out_dev_ptr is not None:
        _gather(left_dev_ptr, kept, points, out_dev_ptr, ctx)
        _gather(right_dev_ptr, added, points, int(out_dev_ptr) + len(kept) * int(points) * 8, ctx)
    return [(0, i) for i in kept] + [(1, i) for i in added]
