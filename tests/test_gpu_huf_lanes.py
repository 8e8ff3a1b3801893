"""The lane-packed Huffman literal decoder (k_huf_decode) on batches shaped after its lane mapping: 8 frames per warp, lane
4f + s decoding stream s of frame f.

Frames are literals-only blocks made by the reference's libzstd (oracle/_ref) from dictated sequences, so the literal count
of every frame -- and with it the four segment lengths -- is chosen here.  Expected bytes are the frame's source, which
libzstd decodes back to.  A damaged frame is one whose stream ends in a zero byte: no final-bit marker, a corrupt stream
by RFC 8878 4.1, which the oracle's decoder rejects (libzstd 1.5.7's literal decoder does not look)."""
import numpy as np
import pytest

from conftest import SEED0
import oracle_lib as O
import zstd_shapes as Z
from test_gpu_zstd_shapes import _batch


def _factory():
    return O.lib().vmo_zstd_ref_factory_available()


def _literals(rng, n, kind):
    """n literal bytes whose Huffman table depth depends on kind: ("uniform", k) over 2^k symbols (table log k), or
    ("geometric", p) over 40 symbols (deep, skewed trees up to the 11-bit limit)"""
    what, a = kind
    if what == "uniform":
        return rng.integers(0, 1 << a, n).astype(np.uint8)
    return np.minimum(rng.geometric(a, n) - 1, 39).astype(np.uint8)


KINDS = [("uniform", 1), ("geometric", 0.5), ("uniform", 3), ("geometric", 0.3), ("uniform", 2), ("geometric", 0.7),
         ("uniform", 5), ("geometric", 0.15), ("uniform", 7), ("geometric", 0.9), ("uniform", 4), ("uniform", 6)]


def _frame(rng, n, kind):
    src = _literals(rng, n, kind)
    frame = O.zstd_ref_compress_sequences(src, [(0, n, 0)])
    return src, frame


def _streams(frame):
    """-> byte offsets [begin, end) of the Huffman streams of a prepared literals-only frame"""
    info = Z.parse_frame(frame)
    b = bytes(frame)
    pos = 4 + 1 + (0 if info["single"] else 1) + info["fcs_size"] + 3  # magic, FHD, WD, FCS, block header
    sf = (b[pos] >> 2) & 3
    hs = 3 if sf < 2 else sf + 2
    v = int.from_bytes(b[pos:pos + hs], "little")
    bits = (10, 10, 14, 18)[sf]
    csize = (v >> (4 + bits)) & ((1 << bits) - 1)
    p = pos + hs
    hb = b[p]
    tree = 1 + (hb if hb < 128 else (hb - 127 + 1) // 2)
    lit_end = p + csize
    p += tree
    if sf == 0:
        return [(p, lit_end)]
    s1, s2, s3 = (int.from_bytes(b[p + 2 * k:p + 2 * k + 2], "little") for k in range(3))
    p += 6
    out = []
    for s in (s1, s2, s3):
        out.append((p, p + s))
        p += s
    out.append((p, lit_end))
    return out


def _check(frames, srcs, bad=()):
    rc, st, got, _ = _batch(frames)
    assert (rc == 0) == (not bad)
    for i, (s, g) in enumerate(zip(srcs, got)):
        if i in bad:
            assert st[i] != 0, i
        else:
            assert st[i] == 0, (i, int(st[i]))
            assert np.array_equal(g, s), i


def _need_ref():
    if not _factory():
        pytest.skip("oracle/_ref (the reference's libzstd with the frame factory) was not built")


@pytest.mark.gpu
@pytest.mark.parametrize("nframes", [1, 7, 8, 9, 17, 33])
def test_frame_counts(nframes):
    """partial warps, literal counts of every residue mod 16 in each segment, neighbouring table depths"""
    _need_ref()
    rng = np.random.default_rng(SEED0 + 7300 + nframes)
    frames, srcs = [], []
    for i in range(nframes):
        n = 1024 + 37 * i + int(rng.integers(0, 64))
        src, frame = _frame(rng, n, KINDS[i % len(KINDS)])
        assert "prepared_4_stream" in Z.shapes(frame), i
        frames.append(frame)
        srcs.append(src)
    _check(frames, srcs)


@pytest.mark.gpu
def test_segment_lengths():
    """regenerated sizes n = 4k .. 4k + 3 (the last segment n - 3 * ceil(n / 4) up to 3 symbols shorter than the others),
    so every stream length modulo 16 and every destination alignment meet head, body and tail"""
    _need_ref()
    rng = np.random.default_rng(SEED0 + 7310)
    frames, srcs = [], []
    for i, n in enumerate(range(1000, 1000 + 64)):
        src, frame = _frame(rng, n, KINDS[i % len(KINDS)])
        assert "prepared_4_stream" in Z.shapes(frame), n
        frames.append(frame)
        srcs.append(src)
    # libzstd's decode of the same frames is the source
    for s, f in zip(srcs[:4], frames[:4]):
        assert np.array_equal(O.zstd_ref_decompress(f, s.size), s)
    _check(frames, srcs)


@pytest.mark.gpu
def test_single_stream_beside_four_stream():
    """single-stream literals (one lane of the frame's four decodes, the other three idle) in the same warps as 4-stream
    frames"""
    _need_ref()
    rng = np.random.default_rng(SEED0 + 7320)
    frames, srcs = [], []
    for i in range(40):
        n = int(rng.integers(100, 256)) if i % 3 == 0 else int(rng.integers(600, 3000))
        src, frame = _frame(rng, n, KINDS[i % 6])  # (libzstd stores 6- and 7-bit uniform literals of < 256 bytes raw)
        want = "prepared_1_stream" if i % 3 == 0 else "prepared_4_stream"
        assert want in Z.shapes(frame), (i, n)
        frames.append(frame)
        srcs.append(src)
    _check(frames, srcs)


@pytest.mark.gpu
@pytest.mark.parametrize("stream", [0, 1, 2, 3])
def test_damaged_stream(stream):
    """a stream without its final-bit marker fails its frame, whichever of the four it is, and only that frame: the rest of
    the warp decodes"""
    _need_ref()
    rng = np.random.default_rng(SEED0 + 7330 + stream)
    frames, srcs = [], []
    for i in range(20):
        src, frame = _frame(rng, 2000 + 53 * i, KINDS[i % len(KINDS)])
        frames.append(frame)
        srcs.append(src)
    bad = (5, 8)  # inside the first warp, and the first frame of the second
    for i in bad:
        f = frames[i].copy()
        spans = _streams(f)
        assert len(spans) == 4
        b, e = spans[stream]
        assert f[e - 1] != 0
        f[e - 1] = 0
        assert O.zstd_decompress(f)[0] < 0, "the oracle accepts the damaged frame"
        frames[i] = f
    _check(frames, srcs, bad=bad)
