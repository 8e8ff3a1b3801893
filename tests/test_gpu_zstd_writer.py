"""The library's zstd writer on the GPU: vmb_zstd_compress_batch == vmb_zstd_compress byte for byte (and the digests of
tests/golden/zstd_writer_frames.json), every frame decodes to its source, and vmb_marshal_columns_gpu -- now with its zstd stage,
the 0.9 rule and the compaction on the device -- == vmb_marshal_columns."""
import hashlib
import json
import os

import numpy as np
import pytest

import blockgen
import zstd_writer_corpus as Z
from conftest import SEED0

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "zstd_writer_frames.json")
FAM = {1: "d2", 5: "d2", 4: "d", 6: "d", 2: "dc", 3: "c"}
VMB_ERR_INVALID_ARG, VMB_ERR_CAP = -50, -54


def _compressed_block_over_128k(frame, n):
    """the writer's known limit: one Compressed block for a compressible source of 128 KiB < n <= 262143, whose literals regenerate
    more than Block_Maximum_Size -- libzstd (and klauspost) reject the frame; the oracle's decoder and the library's accept it"""
    fh = {0x20: 6, 0x60: 7, 0xA0: 9}[int(frame[4])]
    return n > (1 << 17) and (int(frame[fh]) >> 1) & 3 == 2


def _decodes(oracle, frames, sources):
    """every frame decodes to its source through the oracle and vmb_zstd_decompress_batch; through libzstd every frame but those of
    the known limit, which libzstd must reject.  Returns how many frames hit the limit."""
    import victoriametrics_b200 as vm
    have_ref = bool(oracle.lib().vmo_zstd_ref_available())
    over = 0
    for f, raw in zip(frames, sources):
        rc, d = oracle.zstd_decompress(f)
        assert rc == 0 and np.array_equal(d, raw), raw.size
        if have_ref:
            n, r = oracle.zstd_ref_decompress_rc(f, raw.size)
            if _compressed_block_over_128k(f, raw.size):
                assert n < 0, raw.size
                over += 1
            else:
                assert n == raw.size and np.array_equal(r[:n], raw), raw.size
    got = vm.encoding.decompress_zstd_batch(frames)
    for g, raw in zip(got, sources):
        assert np.array_equal(g, raw), raw.size
    return over


def test_batch_equals_host_writer_and_digests_one_frame_per_call(oracle):
    import victoriametrics_b200 as vm
    with open(GOLDEN) as fh:
        golden = json.load(fh)
    corpus = Z.corpus()
    assert [e["name"] for e in golden] == [name for name, _ in corpus]
    ctx = vm.default_context()
    frames = []
    for e, (name, raw) in zip(golden, corpus):
        [f] = vm.encoding.zstd_compress_batch([raw], ctx=ctx)
        assert np.array_equal(f, vm.encoding.zstd_compress(raw)), name
        assert hashlib.sha256(f.tobytes()).hexdigest() == e["frame_sha256"], name
        frames.append(f)
    over = _decodes(oracle, frames, [raw for _, raw in corpus])
    assert over > 0 or not oracle.lib().vmo_zstd_ref_available()  # the corpus reaches the known limit


def test_batch_of_thousands_of_mixed_sizes_in_one_call(oracle):
    import victoriametrics_b200 as vm
    rng = np.random.default_rng(SEED0 + 700)
    corpus = [raw for _, raw in Z.corpus()]
    srcs = list(corpus)
    while len(srcs) < 4000:
        n = int(rng.choice([rng.integers(1, 200), rng.integers(100, 2000), rng.integers(1000, 40000), rng.integers(1, 300000)],
                           p=[0.3, 0.3, 0.35, 0.05]))
        kind = Z.CONTENTS[int(rng.integers(len(Z.CONTENTS)))]
        srcs.append(Z._content(rng, kind, n).astype(np.uint8))
    perm = rng.permutation(len(srcs))
    srcs = [srcs[i] for i in perm]
    got = vm.encoding.zstd_compress_batch(srcs, ctx=vm.default_context())
    assert len(got) == len(srcs)
    for g, raw in zip(got, srcs):
        assert np.array_equal(g, vm.encoding.zstd_compress(raw)), raw.size
    _decodes(oracle, got[:600], srcs[:600])


def test_batch_error_contract():
    import victoriametrics_b200 as vm
    from victoriametrics_b200 import _lib
    L = _lib.lib()
    ctx = vm.default_context()
    u8, u64 = _lib.u8p, _lib.u64p
    srcs = [np.arange(300, dtype=np.uint8), np.full(5000, 9, dtype=np.uint8), np.random.default_rng(1).integers(0, 4, 9000).astype(np.uint8)]
    arena = np.concatenate(srcs)
    offs = np.array([0, 300, 5300, 14300], dtype=np.uint64)
    need = sum(vm.encoding.zstd_compress(s).size for s in srcs)
    doffs = np.zeros(4, dtype=np.uint64)
    dst = np.full(need, 0xAB, dtype=np.uint8)
    # too small: VMB_ERR_CAP, the bytes needed, dst untouched
    rc = L.vmb_zstd_compress_batch(ctx.h, arena.ctypes.data_as(u8), offs.ctypes.data_as(u64), 3, dst.ctypes.data_as(u8), need - 1,
                                   doffs.ctypes.data_as(u64))
    assert rc == VMB_ERR_CAP and int(doffs[3]) == need and (dst == 0xAB).all()
    rc = L.vmb_zstd_compress_batch(ctx.h, arena.ctypes.data_as(u8), offs.ctypes.data_as(u64), 3, dst.ctypes.data_as(u8), need,
                                   doffs.ctypes.data_as(u64))
    assert rc == 0 and int(doffs[3]) == need
    assert np.array_equal(dst, np.concatenate([vm.encoding.zstd_compress(s) for s in srcs]))
    # an empty source, NULL pointers
    bad = np.array([0, 300, 300, 14300], dtype=np.uint64)
    assert L.vmb_zstd_compress_batch(ctx.h, arena.ctypes.data_as(u8), bad.ctypes.data_as(u64), 3, dst.ctypes.data_as(u8), need,
                                     doffs.ctypes.data_as(u64)) == VMB_ERR_INVALID_ARG
    assert L.vmb_zstd_compress_batch(ctx.h, None, offs.ctypes.data_as(u64), 3, dst.ctypes.data_as(u8), need,
                                     doffs.ctypes.data_as(u64)) == VMB_ERR_INVALID_ARG
    assert L.vmb_zstd_compress_batch(ctx.h, arena.ctypes.data_as(u8), offs.ctypes.data_as(u64), 3, dst.ctypes.data_as(u8), need,
                                     None) == VMB_ERR_INVALID_ARG
    # a source of more than 128 MiB: rejected before anything is copied
    big = np.array([0, (128 << 20) + 1], dtype=np.uint64)
    assert L.vmb_zstd_compress_batch(ctx.h, arena.ctypes.data_as(u8), big.ctypes.data_as(u64), 1, dst.ctypes.data_as(u8), need,
                                     doffs.ctypes.data_as(u64)) == VMB_ERR_INVALID_ARG
    # n == 0
    doffs[:] = 77
    assert L.vmb_zstd_compress_batch(ctx.h, None, offs.ctypes.data_as(u64), 0, None, 0, doffs.ctypes.data_as(u64)) == 0
    assert int(doffs[0]) == 0
    with pytest.raises(_lib.VmbError):
        vm.encoding.zstd_compress_batch([np.zeros(0, dtype=np.uint8)], ctx=ctx)
    assert vm.encoding.zstd_compress_batch([], ctx=ctx) == []


def _check_marshal(oracle, a, pb=64, decode_cols=None):
    import victoriametrics_b200 as vm
    p_gpu, o_gpu, mt_gpu, f_gpu = vm.encoding.marshal_columns(a, pb, ctx=vm.default_context())
    p_cpu, o_cpu, mt_cpu, f_cpu = vm.encoding.marshal_columns(a, pb)
    assert np.array_equal(mt_gpu, mt_cpu) and np.array_equal(f_gpu, f_cpu) and np.array_equal(o_gpu, o_cpu)
    assert np.array_equal(p_gpu, p_cpu)
    cols = range(a.shape[0]) if decode_cols is None else decode_cols
    for c in cols:
        b = p_gpu[int(o_gpu[c]):int(o_gpu[c + 1])]
        rc, out = oracle.unmarshal_int64_array(b, int(mt_gpu[c]), int(f_gpu[c]), a.shape[1])
        assert rc == 0, c
        if pb == 64:
            assert np.array_equal(out, a[c]), c
        else:
            ob, omt, ofirst = oracle.marshal_int64_array(a[c], pb)
            rc2, oout = oracle.unmarshal_int64_array(ob, omt, ofirst, a.shape[1])
            assert rc2 == 0 and np.array_equal(out, oout) and FAM[omt] == FAM[int(mt_gpu[c])], c
    return mt_gpu


@pytest.mark.parametrize("rows", [1, 2, 130, 8192, 16384])
def test_marshal_gpu_every_kind(oracle, rows):
    rng = np.random.default_rng(SEED0 + 710 + rows)
    cols = []
    for kind in blockgen.VALUE_KINDS:
        cols += [blockgen.gen_values(rng, kind, rows) for _ in range(4)]
    for kind in blockgen.TS_KINDS:
        cols += [blockgen.gen_timestamps(rng, kind, rows) for _ in range(4)]
    _check_marshal(oracle, np.stack(cols))


def test_marshal_gpu_streams_over_128k(oracle):
    """16384 rows of 9- and 10-byte varints: streams over 128 KiB.  Random ones get a Raw-block frame split at 128 KiB and then
    type 6; the wrapped sums of large steps compress, into one Compressed block of more than 128 KiB (type 4)"""
    rng = np.random.default_rng(SEED0 + 720)
    rows = 16384
    a = np.stack([rng.integers(-(1 << 62), 1 << 62, rows).astype(np.int64) for _ in range(6)] +
                 [np.cumsum(rng.integers(1 << 58, 1 << 59, rows)).astype(np.int64) for _ in range(2)])
    mts = _check_marshal(oracle, a)
    assert (mts[:6] == 6).all() and (mts[6:] == 4).all()


def test_marshal_gpu_streams_of_127_and_128_bytes(oracle):
    """the largest stream the zstd stage leaves alone (encoding.go:15) and the smallest it takes"""
    rng = np.random.default_rng(SEED0 + 730)
    for target in (127, 128):
        rows = target + 1
        # first value < 0: a gauge (delta coding), every delta in [-60, 60]: one varint byte each
        a = np.stack([-5 + np.cumsum(np.r_[0, rng.integers(-60, 61, rows - 1)]) for _ in range(16)]).astype(np.int64)
        for c in a:
            assert oracle.marshal_nearest_delta(c, 64)[0].size == target
        mts = _check_marshal(oracle, a)
        if target == 127:
            assert (mts == 6).all()


def test_marshal_gpu_frames_at_the_09_cut(oracle):
    """columns whose frame lands within a few bytes of 0.9 x the stream, on both sides, found by a seeded search"""
    import victoriametrics_b200 as vm
    rng = np.random.default_rng(SEED0 + 740)
    rows = 600
    near = []
    for _ in range(4000):
        spread = int(rng.integers(20, 4000))
        v = np.cumsum(rng.integers(0, spread, rows)).astype(np.int64)
        raw, _ = oracle.marshal_nearest_delta(v, 64, delta2=True)
        f = vm.encoding.zstd_compress(raw)
        if abs(f.size - 0.9 * raw.size) <= 4:
            near.append(v)
        if len(near) >= 64:
            break
    assert len(near) >= 8
    mts = _check_marshal(oracle, np.stack(near))
    assert 1 in mts.tolist() and 5 in mts.tolist()


@pytest.mark.parametrize("pb", [1, 5, 12, 33])
def test_marshal_gpu_lossy(oracle, pb):
    rng = np.random.default_rng(SEED0 + 750 + pb)
    cols = []
    for kind in ("counter", "counter_resets", "gauge", "gauge_wide", "counter_big", "counter_smooth", "special"):
        cols += [blockgen.gen_values(rng, kind, 2000) for _ in range(6)]
    _check_marshal(oracle, np.stack(cols), pb=pb)


def test_marshal_gpu_100k_mixed_columns(oracle):
    rng = np.random.default_rng(SEED0 + 760)
    rows = 130
    kinds = blockgen.VALUE_KINDS
    a = np.empty((100_000, rows), dtype=np.int64)
    for c in range(a.shape[0]):
        a[c] = blockgen.gen_values(rng, kinds[c % len(kinds)], rows)
    _check_marshal(oracle, a, decode_cols=range(0, a.shape[0], 97))


def test_marshal_gpu_cap_too_small():
    import victoriametrics_b200 as vm
    from victoriametrics_b200 import _lib
    rng = np.random.default_rng(SEED0 + 770)
    a = np.stack([blockgen.gen_values(rng, "counter", 1000) for _ in range(8)])
    payload, _, _, _ = vm.encoding.marshal_columns(a)
    need = payload.size
    dst = np.empty(need, dtype=np.uint8)
    offs, mts, firsts = np.zeros(9, dtype=np.uint64), np.zeros(8, dtype=np.uint8), np.zeros(8, dtype=np.int64)
    args = (offs.ctypes.data_as(_lib.u64p), mts.ctypes.data_as(_lib.u8p), firsts.ctypes.data_as(_lib.i64p), a.ctypes.data_as(_lib.i64p),
            8, 1000, 64, 1)
    ctx = vm.default_context()
    assert _lib.lib().vmb_marshal_columns_gpu(ctx.h, dst.ctypes.data_as(_lib.u8p), need - 1, *args) == VMB_ERR_CAP
    assert int(offs[8]) == need
    assert _lib.lib().vmb_marshal_columns_gpu(ctx.h, dst.ctypes.data_as(_lib.u8p), need, *args) == 0
    assert np.array_equal(dst, payload)
