#!/usr/bin/env python3
"""Generate tests/golden/zstd_shapes.json: varint columns (MarshalType 1 / 4 payloads) in the zstd frame shapes the
reference's writers produce, made by the reference's own libzstd 1.5.7 (oracle/_ref) -- the pure-Go writer's headers (no
Frame_Content_Size below 256 bytes, a Window_Descriptor up to 1024), every level the storage uses, dictated repeat-offset
sequences, and frames libzstd or the varint check rejects.  Each entry carries the raw varint stream and the sha256 of both
byte strings.  Run in the build container only (needs oracle/_ref); tests/test_gpu_zstd_shapes.py reads the JSON."""
import base64
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import oracle_lib as O  # noqa: E402
import zstd_shapes as Z  # noqa: E402


def main():
    assert O.lib().vmo_zstd_ref_factory_available(), "oracle/_ref/libzstd_ref.so missing or stale: run `make -C oracle ref`"
    rng = np.random.default_rng(20261016)
    cases = (Z.pure_go_cases(rng) + Z.level_cases(rng, Z.STORAGE_LEVELS, rows_choices=(13, 100, 257, 600)) +
             Z.sequence_cases(rng, nseq=48) + Z.error_cases(rng))
    # small blocks of one stream: treeless literals and Repeat_Mode tables (the Huffman / FSE tables of an earlier block)
    for kind in ("counter", "counter_smooth", "gauge", "counter_resets"):
        mt, first, raw = Z.varint_column(rng, kind, 8192, True)
        f = O.zstd_ref_compress_params(raw, targetCBlockSize=1340)
        if {"lit_treeless", "repeat_mode"} <= Z.shapes(f):
            cases.append(Z.case("treeless_repeat_mode_%s" % kind, mt, 8192, first, raw, f))
            break
    else:
        raise AssertionError("no frame with treeless literals and Repeat_Mode tables")
    out = []
    for c in cases:
        raw, frame = c["raw"].tobytes(), c["frame"].tobytes()
        out.append(dict(name=c["name"], mt=c["mt"], rows=c["rows"], first=c["first"], zstd_ok=c["zstd_ok"],
                        raw=base64.b64encode(raw).decode(), raw_sha256=hashlib.sha256(raw).hexdigest(),
                        frame=base64.b64encode(frame).decode(), frame_sha256=hashlib.sha256(frame).hexdigest()))
    path = os.path.join(HERE, "zstd_shapes.json")
    with open(path, "w") as f:
        json.dump(out, f, separators=(",", ":"))
    print("cases:", len(out), "bytes:", os.path.getsize(path))


if __name__ == "__main__":
    main()
