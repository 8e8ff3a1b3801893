#!/usr/bin/env python3
"""Generate tests/golden/zstd_writer_frames.json: the SHA-256 of every frame the library's zstd writer (vmb_zstd_compress)
makes of the seeded corpus of tests/zstd_writer_corpus.py, with the source's SHA-256 and both lengths.  The digests were taken
before the writer's rules moved into shared host / device code and pin it byte for byte; tests/test_zstd_writer_frames.py
(host writer) and tests/test_gpu_zstd_writer.py (vmb_zstd_compress_batch) read the JSON.  Needs a built libvmb200.so."""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import zstd_writer_corpus as Z  # noqa: E402
from victoriametrics_b200 import encoding  # noqa: E402


def main():
    out = []
    for name, raw in Z.corpus():
        frame = encoding.zstd_compress(raw)
        out.append(dict(name=name, n=int(raw.size), src_sha256=hashlib.sha256(raw.tobytes()).hexdigest(),
                        frame_len=int(frame.size), frame_sha256=hashlib.sha256(frame.tobytes()).hexdigest()))
    path = os.path.join(HERE, "zstd_writer_frames.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0, separators=(",", ":"))
    print("frames:", len(out), "bytes:", os.path.getsize(path))


if __name__ == "__main__":
    main()
