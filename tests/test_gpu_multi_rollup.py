"""multi-output rollups (getRollupConfigs rollup.go:416-504): rollup(), rollup_rate/deriv/increase/delta(),
rollup_scrape_interval(), rollup_candlestick(), aggr_over_time(), quantiles_over_time() through the CUDA path (shared value
preFunc: deltaValues rollup.go:960, derivValues :976, scrape intervals :462) against the oracle"""
import numpy as np

from conftest import SEED0
import pytest

import blockgen
from rollup_names import RF
from test_gpu_rollup_exact import assert_same_bits

pytestmark = pytest.mark.gpu
T0 = 1_700_000_000_000


def _pre_oracle(oracle, name, ts, fv):
    L = oracle.lib()
    if name in ("rollup_rate", "rollup_deriv"):
        L.vmo_deriv_values(fv.ctypes.data_as(oracle.f64p), ts.ctypes.data_as(oracle.i64p), len(fv))
    elif name in ("rollup_increase", "rollup_delta"):
        L.vmo_delta_values(fv.ctypes.data_as(oracle.f64p), len(fv))
    elif name == "rollup_scrape_interval":  # rollup.go:462-474
        secs = ts.astype(np.float64) / 1000
        out = np.empty_like(fv)
        out[0] = np.nan
        out[1:] = secs[1:] - secs[:-1]
        if len(out) > 1:
            out[0] = out[1]
        fv[:] = out


@pytest.mark.parametrize("name,kw", [
    ("rollup", {}), ("rollup", {"tag": "max"}), ("rollup_rate", {}), ("rollup_deriv", {}), ("rollup_increase", {}),
    ("rollup_delta", {"tag": "avg"}), ("rollup_scrape_interval", {}), ("rollup_candlestick", {}),
    ("rollup_candlestick", {"tag": "high"}), ("aggr_over_time", {"aggr_funcs": ["min_over_time", "rate", "count_over_time"]}),
    ("quantiles_over_time", {"phis": [0.1, 0.5, 0.99]})])
def test_multi_output_rollups(oracle, name, kw):
    import victoriametrics_b200 as vm
    import zlib
    rng = np.random.default_rng(SEED0 + zlib.crc32(name.encode()) % 1000 + len(kw))
    blocks = []
    for i in range(36):
        n = int(rng.choice([1, 2, 3, 40, 600, 4096]))
        tkind = ("regular", "jitter", "irregular", "dups")[i % 4]   # "dups": derivValues' carried state
        vkind = ("counter_resets", "gauge", "counter", "special")[(i // 4) % 4]
        vals = blockgen.gen_values(rng, vkind, n)
        if vkind != "special":
            vals = np.abs(vals)
        blocks.append(blockgen.OBlock(blockgen.gen_timestamps(rng, tkind, n, T0), vals, -2, 64, i))
    descs, payload = blockgen.to_blockset(blocks)
    B = vm.storage.Blocks(descs, payload)
    start, end, step, window = T0 + 60_000, T0 + 15_000 * 700, 30_000, 120_000
    got, gscanned = vm.promql.eval_rollup_func_multi(name, B, start, end, step, window, **kw)
    rcs = vm.promql.get_rollup_configs_multi(name, start, end, step, window, **kw)
    assert list(got) == [rc.TagValue for rc in rcs]
    escanned = 0
    for rc in rcs:
        exp = []
        for b in blocks:
            r, ts, fv, _ = b.oracle_unmarshal()
            assert r == 0
            ts, fv = ts.copy(), fv.copy()
            n = oracle.lib().vmo_drop_stale_nans(fv.ctypes.data_as(oracle.f64p), ts.ctypes.data_as(oracle.i64p), len(ts))
            ts, fv = ts[:n].copy(), fv[:n].copy()
            if n and rc.removeCounterResets:
                oracle.lib().vmo_remove_counter_resets(fv.ctypes.data_as(oracle.f64p), ts.ctypes.data_as(oracle.i64p), n, 0)
            if n:
                _pre_oracle(oracle, name, ts, fv)
            o, sc = oracle.rollup_do(RF[rc.Func], fv, ts, start, end, step, window, may_adjust_window=rc.MayAdjustWindow,
                                     samples_scanned_per_call=rc.samplesScannedPerCall, args=rc.args)
            exp.append(o)
            escanned += sc
        exp = np.stack(exp)
        g = got[rc.TagValue]
        assert_same_bits(g, exp, "%s %s" % (name, rc.TagValue), rc.Func)
    assert gscanned == escanned
