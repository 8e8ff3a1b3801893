"""evalRollupFuncWithSubquery (eval.go:910) on the device: max_over_time(rate(m[5m])[30m:1m]) -- the inner rollup's result stays in
HBM, vmb_series_from_matrix turns its rows into series (removeNanValues eval.go:1027 drops NaN points with their timestamps), the
outer rollup runs on those.  Checked against the oracle doing the same three steps on the CPU."""
import numpy as np
import pytest

import blockgen
from conftest import SEED0
from rollup_names import RF
from test_baseline_configs import _oracle_rollup_matrix
from test_gpu_rollup_exact import assert_same_bits

pytestmark = pytest.mark.gpu
T0 = 1_700_000_000_000


@pytest.mark.parametrize("outer,inner", [("max_over_time", "rate"), ("avg_over_time", "increase"), ("rate", "sum_over_time"),
                                         ("quantile_over_time", "rate"), ("count_over_time", "rate")])
def test_subquery_outer_rollup_over_device_matrix(oracle, outer, inner):
    import torch
    import victoriametrics_b200 as vm
    rng = np.random.default_rng(SEED0 + 9090)
    blocks = []
    for i in range(24):
        rows = [4096, 700, 2500][i % 3]  # short series leave NaN points at the end of the inner grid
        t0 = T0 + (0 if i % 4 else 15000 * 900)  # ... and late starters at its beginning
        blocks.append(blockgen.OBlock(blockgen.gen_timestamps(rng, "regular" if i % 5 else "jitter", rows, t0),
                                      blockgen.gen_values(rng, ["counter", "gauge", "counter_resets"][i % 3], rows), -2, 64, i))
    descs, payload = blockgen.to_blockset(blocks)
    ctx = vm.default_context()
    B = vm.storage.Blocks(descs, payload, ctx)
    # outer grid and the subquery grid derived from it (eval.go:924-932: start -= window + step, end += step, aligned to the step)
    start, end, step = T0 + 3_600_000, T0 + 15000 * 4000, 120_000
    sq_step, sq_window, in_window = 60_000, 1_800_000, 300_000
    sq_start = start - (sq_window + sq_step)
    sq_start -= sq_start % sq_step
    sq_end = end + sq_step
    sq_end -= sq_end % sq_step
    psq = 1 + (sq_end - sq_start) // sq_step
    inner_dev = torch.empty((len(blocks), psq), dtype=torch.float64, device="cuda")
    vm.promql.eval_rollup_func(inner, B, sq_start, sq_end, sq_step, in_window, out_dev_ptr=inner_dev.data_ptr())
    P = 1 + (end - start) // step
    args = np.full(P, 0.9) if outer == "quantile_over_time" else None
    got, scanned = vm.promql.eval_rollup_func_with_subquery(outer, inner_dev.data_ptr(), len(blocks), sq_start, sq_end, sq_step, start, end,
                                                            step, sq_window, args=args, ctx=ctx)
    # oracle: inner matrix, removeNanValues per row, outer preFunc + Do
    inner_exp = _oracle_rollup_matrix(oracle, blocks, inner, sq_start, sq_end, sq_step, in_window)
    assert_same_bits(inner_dev.cpu().numpy(), inner_exp, "inner " + inner, inner)
    assert np.isnan(inner_exp).any() and (~np.isnan(inner_exp)).any()
    grid = sq_start + sq_step * np.arange(psq, dtype=np.int64)
    rc = vm.promql.get_rollup_configs(outer, start, end, step, sq_window)
    total = 0
    for s in range(len(blocks)):
        row = inner_dev[s].cpu().numpy()  # the GPU's own inner values: the outer step is checked on identical input
        keep = ~np.isnan(row)
        v, t = np.ascontiguousarray(row[keep]), np.ascontiguousarray(grid[keep])
        if rc.removeCounterResets and len(v):
            oracle.lib().vmo_remove_counter_resets(v.ctypes.data_as(oracle.f64p), t.ctypes.data_as(oracle.i64p), len(v), 0)
        exp, sc = oracle.rollup_do(RF[outer], v, t, start, end, step, sq_window, may_adjust_window=rc.MayAdjustWindow,
                                   samples_scanned_per_call=rc.samplesScannedPerCall, args=args)
        total += sc
        assert_same_bits(got[s], exp, "%s row %d" % (outer, s), outer)
    assert scanned == total
