"""The library's zstd writer (vmb_zstd_compress) held to the frame digests of tests/golden/zstd_writer_frames.json: the code-length,
weight-table and header rules are shared by the host writer and the device writer (csrc/zstd_writer.cuh), and these digests,
taken before they were shared, prove that no byte of any frame changed."""
import hashlib
import json
import os

import numpy as np
import pytest

import zstd_writer_corpus as Z
from victoriametrics_b200 import encoding

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "zstd_writer_frames.json")


def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def test_corpus_is_the_one_the_digests_were_taken_of():
    g = golden()
    c = Z.corpus()
    assert [e["name"] for e in g] == [name for name, _ in c]
    for e, (_, raw) in zip(g, c):
        assert e["n"] == raw.size and e["src_sha256"] == hashlib.sha256(raw.tobytes()).hexdigest(), e["name"]


def test_host_writer_matches_the_digests(oracle):
    bad = []
    for e, (name, raw) in zip(golden(), Z.corpus()):
        frame = encoding.zstd_compress(raw)
        if frame.size != e["frame_len"] or hashlib.sha256(frame.tobytes()).hexdigest() != e["frame_sha256"]:
            bad.append(name)
            continue
        rc, d = oracle.zstd_decompress(frame)
        assert rc == 0 and np.array_equal(d, raw), name
    assert not bad, bad


def test_host_writer_frames_libzstd_accepts_and_the_known_limit(oracle):
    """libzstd decodes every corpus frame except the writer's known limit: a compressible source of 128 KiB < n <= 262143 bytes
    gets one Compressed block whose literals regenerate more than Block_Maximum_Size, which libzstd rejects"""
    if not oracle.lib().vmo_zstd_ref_available():
        pytest.skip("oracle/_ref/libzstd_ref.so not built")
    over = []
    for name, raw in Z.corpus():
        frame = encoding.zstd_compress(raw)
        fh = {0x20: 6, 0x60: 7, 0xA0: 9}[int(frame[4])]
        n, r = oracle.zstd_ref_decompress_rc(frame, raw.size)
        if raw.size > (1 << 17) and (int(frame[fh]) >> 1) & 3 == 2:
            assert n < 0, name
            over.append((name, raw.size))
        else:
            assert n == raw.size and np.array_equal(r[:n], raw), name
    assert over and all(n <= 262143 for _, n in over), over
