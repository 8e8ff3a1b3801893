"""The seeded corpus that pins the library's zstd writer (vmb_zstd_compress, vmb_zstd_compress_batch): byte sources at the sizes
where the writer changes its frame (literals-header forms, one stream / four streams, the 128 KiB block limit, the 262143-byte
Huffman limit, the FCS widths), with contents that reach every branch of the code-length and weight rules, and the varint
streams of every blockgen column kind.  tests/golden/make_zstd_writer_frames.py records the SHA-256 of each frame."""
import numpy as np

import blockgen
import oracle_lib as O

SEED = 20261018
SIZES = (1, 2, 31, 32, 33, 127, 128, 1023, 1024, 1025, 16383, 16384, 16385, 65535, 65791, 65792, 131071, 131072, 131073,
         163830, 262143, 262144, 300000)


def _content(rng, kind, n):
    if kind == "uniform":
        return rng.integers(0, 256, n)
    if kind == "two":
        return rng.choice(np.array([17, 201]), n)
    if kind == "three":
        return rng.integers(0, 3, n)
    if kind == "high":      # every symbol above 128: more than 128 weights, so only the FSE-compressed tree description fits
        return rng.integers(129, 256, n)
    if kind == "rle":
        return np.full(n, 7)
    if kind == "geo_steep":  # code lengths beyond 11 bits: the lengthening loop, then the shortening loop
        return np.minimum(rng.geometric(0.45, n), 255)
    if kind == "geo_mild":
        return np.minimum(rng.geometric(0.08, n), 255)
    if kind == "ties":      # all 256 symbols at equal counts: every order decision is a tie-break
        return rng.permutation(np.resize(np.arange(256), n))
    if kind == "dominant":  # one symbol and 255 rare ones
        a = np.full(n, 42)
        k = min(n, 255)
        a[rng.choice(n, k, replace=False)] = np.delete(np.arange(256), 42)[:k]
        return a
    raise KeyError(kind)


CONTENTS = ("uniform", "two", "three", "high", "rle", "geo_steep", "geo_mild", "ties", "dominant")


def varint_stream(vals, delta2):
    """the MarshalType 1 (delta2) / 4 (delta) varint stream of a column at precisionBits 64"""
    raw, _ = O.marshal_nearest_delta(vals, 64, delta2=delta2)
    return raw


def corpus():
    """[(name, np.uint8 source)], in a fixed order; every source has at least one byte"""
    rng = np.random.default_rng(SEED)
    out = []
    for n in SIZES:
        for kind in CONTENTS:
            out.append(("%s_%d" % (kind, n), _content(rng, kind, n).astype(np.uint8)))
    for rows in (130, 8192, 16384):
        for kind in blockgen.VALUE_KINDS:
            v = blockgen.gen_values(rng, kind, rows)
            for delta2 in (False, True):
                out.append(("%s_d%d_%d" % (kind, 2 if delta2 else 1, rows), varint_stream(v, delta2)))
        for kind in blockgen.TS_KINDS:
            t = blockgen.gen_timestamps(rng, kind, rows)
            for delta2 in (False, True):
                out.append(("ts_%s_d%d_%d" % (kind, 2 if delta2 else 1, rows), varint_stream(t, delta2)))
    return out
