"""Test-only zstd frame shapes (RFC 8878): a header walker that names the shape of a frame, the pure-Go writer's header
layout, and frames whose sequences are dictated.  Frames come from the reference's libzstd (oracle/_ref); nothing here
decodes a frame's content, so expected values never depend on the decoders under test."""
import numpy as np

import oracle_lib as O

LIT_TYPES = ("raw", "rle", "compressed", "treeless")
BLOCK_TYPES = ("raw", "rle", "compressed", "reserved")


def parse_frame(frame):
    """-> dict: the frame header fields and, per block, its type and (compressed blocks) the literals / sequences headers"""
    b = bytes(frame)
    assert b[:4] == b"\x28\xb5\x2f\xfd", "not a zstd frame"
    fhd = b[4]
    fcs_flag, single, checksum, did = fhd >> 6, (fhd >> 5) & 1, (fhd >> 2) & 1, fhd & 3
    pos = 5
    wd = None
    if not single:
        wd = b[pos]
        pos += 1
    pos += (0, 1, 2, 4)[did]
    fcs_size = (1 if single else 0) if fcs_flag == 0 else (1 << fcs_flag)
    fcs = int.from_bytes(b[pos:pos + fcs_size], "little") + (256 if fcs_size == 2 else 0) if fcs_size else None
    pos += fcs_size
    info = dict(single=bool(single), fcs=fcs, fcs_size=fcs_size, window_descriptor=wd, checksum=bool(checksum), blocks=[])
    while True:
        bh = int.from_bytes(b[pos:pos + 3], "little")
        pos += 3
        last, btype, bsize = bh & 1, (bh >> 1) & 3, bh >> 3
        blk = dict(type=BLOCK_TYPES[btype], size=bsize)
        if btype == 2:
            blk.update(_compressed_block(b[pos:pos + bsize]))
        pos += 1 if btype == 1 else bsize
        info["blocks"].append(blk)
        if last:
            break
    info["trailing"] = len(b) - pos - (4 if checksum else 0)
    return info


def _compressed_block(blk):
    lt, sf = blk[0] & 3, (blk[0] >> 2) & 3
    out = dict(lit=LIT_TYPES[lt])
    if lt < 2:
        hs = (1, 2, 1, 3)[sf]
        regen = blk[0] >> 3 if hs == 1 else (int.from_bytes(blk[:hs], "little") >> 4)
        p = hs + (regen if lt == 0 else 1)
        out.update(streams=0, lit_regen=regen)
    else:
        if sf in (0, 1):
            v, hs, bits = int.from_bytes(blk[:3], "little"), 3, 10
        elif sf == 2:
            v, hs, bits = int.from_bytes(blk[:4], "little"), 4, 14
        else:
            v, hs, bits = int.from_bytes(blk[:5], "little"), 5, 18
        regen, csize = (v >> 4) & ((1 << bits) - 1), (v >> (4 + bits)) & ((1 << bits) - 1)
        out.update(streams=1 if sf == 0 else 4, lit_regen=regen)
        p = hs + csize
    b0 = blk[p]
    nseq = b0 if b0 < 128 else (((b0 - 128) << 8) + blk[p + 1] if b0 < 255 else blk[p + 1] + (blk[p + 2] << 8) + 0x7F00)
    p += 1 if b0 < 128 else (2 if b0 < 255 else 3)
    out["nseq"] = nseq
    out["seq_modes"] = (blk[p] >> 6 & 3, blk[p] >> 4 & 3, blk[p] >> 2 & 3) if nseq else ()
    return out


def shapes(frame):
    """the set of shape names a frame shows (the decoder paths it takes are named after them)"""
    f = parse_frame(frame)
    s = set()
    blocks = f["blocks"]
    comp = [b for b in blocks if b["type"] == "compressed"]
    s.add("fcs" if f["fcs"] is not None else "no_fcs")
    if f["window_descriptor"] is not None:
        s.add("window_descriptor")
    if f["fcs_size"] == 2:
        s.add("fcs2")
    if f["checksum"]:
        s.add("checksum")
    if len(blocks) > 1:
        s.add("multi_block")
    for b in blocks:
        if b["type"] != "compressed":
            s.add(b["type"] + "_block")
    for b in comp:
        s.add("lit_" + b["lit"])
        if b["lit"] in ("raw", "rle") and b["nseq"]:
            s.add("lit_%s_with_sequences" % b["lit"])
        if 3 in b["seq_modes"]:
            s.add("repeat_mode")
    # what the library's host classifier sends to the lane-packed (prepared) path: one last Compressed block with Huffman
    # literals, a Frame_Content_Size and no checksum
    if f["fcs"] is not None and not f["checksum"] and len(blocks) == 1 and comp and comp[0]["lit"] == "compressed":
        s.add("prepared")
        s.add("prepared_%d_stream" % comp[0]["streams"])
        s.add("prepared_with_sequences" if comp[0]["nseq"] else "prepared_literals_only")
    else:
        s.add("serial")
    return s


def pure_go_frame(raw, **params):
    """a libzstd frame in the header layout of klauspost/compress EncodeAll (the reference's writer when built without cgo):
    one segment with a Frame_Content_Size when 1024 < len <= window, else a Window_Descriptor and a Frame_Content_Size only
    from 256 bytes on (frameenc.go: 'framessizes < 256 are not stored').  The blocks are libzstd's; Window_Size >= len."""
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    n = raw.size
    if n > 1024:
        return O.zstd_ref_compress_params(raw, **params)
    f = O.zstd_ref_compress_params(raw, contentSizeFlag=0, **params)
    assert f[4] == 0x00 and f[5] == 0x00, "expected no FCS and a 1 KiB window: FHD %02x WD %02x" % (f[4], f[5])
    if n < 256:
        return f
    # Frame_Content_Size_Flag 1: a 2-byte field holding len - 256 behind the Window_Descriptor
    return np.concatenate([f[:4], np.array([0x40, 0x00], np.uint8), np.frombuffer((n - 256).to_bytes(2, "little"), np.uint8),
                           f[6:]])


def run_sequences(seqs, lit_alphabet, rng, tail=0):
    """the bytes a list of (offset, literal length, match length) sequences produces with random literals from lit_alphabet
    (repeat offsets already resolved to plain ones), plus `tail` trailing literals"""
    out = []
    for off, ll, ml in seqs:
        out.extend(int(x) for x in rng.choice(lit_alphabet, ll))
        assert 0 < off <= len(out), (off, len(out))
        for _ in range(ml):
            out.append(out[-off])
    out.extend(int(x) for x in rng.choice(lit_alphabet, tail))
    return np.array(out, dtype=np.uint8)


def repcode_sequences(rng, nseq, lit_alphabet=np.arange(0, 16), max_off=64):
    """sequences that exercise every repeat-offset form: after a literal run, sequences with ll = 0 whose offset equals
    rep2, rep3 or rep1 - 1 (and rep1 with ll > 0); short offsets 1..7 that overlap their own output; long matches.
    -> (seqs as (offset, ll, ml), the source bytes)"""
    seqs, rep = [], [1, 4, 8]
    produced = 0

    def push(off, ll, ml):
        nonlocal produced
        seqs.append((off, ll, ml))
        produced += ll + ml

    push(1, 16, 4)
    rep = [1, 4, 8]
    for i in range(nseq):
        kind = i % 8
        ll = 0 if kind in (1, 2, 3) else int(rng.integers(1, 6))
        if kind == 1:
            off = rep[1]
        elif kind == 2:
            off = rep[2]
        elif kind == 3:
            off = rep[0] - 1
        elif kind == 4:
            off = int(rng.integers(1, 8))
        elif kind == 5:
            off = rep[0]
        else:
            off = int(rng.integers(8, max_off))
        if off < 1 or off > produced + ll:
            off = int(rng.integers(1, 8))
        ml = int(rng.integers(3, 12)) if kind != 6 else int(rng.integers(40, 300))
        ml = max(ml, 3)
        push(off, ll, ml)
        # repeat-offset history as RFC 8878 3.1.1.5 updates it (the compressor resolves offsets the same way)
        if ll == 0:
            if off == rep[1]:
                rep = [rep[1], rep[0], rep[2]]
            elif off == rep[2]:
                rep = [rep[2], rep[0], rep[1]]
            elif off == rep[0] - 1:
                rep = [off, rep[0], rep[1]]
            else:  # (with ll = 0 an offset equal to rep1 has no repeat code: it is written as a new offset)
                rep = [off, rep[0], rep[1]]
        else:
            if off == rep[0]:
                pass
            elif off == rep[1]:
                rep = [rep[1], rep[0], rep[2]]
            elif off == rep[2]:
                rep = [rep[2], rep[0], rep[1]]
            else:
                rep = [off, rep[0], rep[1]]
    src = run_sequences(seqs, lit_alphabet, rng, tail=5)
    return seqs, src


# ---- the corpus: varint columns (MarshalType 1 / 4 payloads) in every frame shape
LEVELS = tuple(range(-7, 23))
STORAGE_LEVELS = (-5, -2, -1, 1, 2, 3, 4, 5)  # encoding.go getCompressLevel and partition.go:1705 (index blocks)
ROWS = (13, 40, 100, 257, 1000, 2048, 4096, 8192)
PARAM_SETS = (
    dict(contentSizeFlag=0),                                  # no Frame_Content_Size: a Window_Descriptor instead
    dict(contentSizeFlag=0, compressionLevel=19),
    dict(checksumFlag=1),
    dict(checksumFlag=1, contentSizeFlag=0),
    dict(windowLog=10),                                       # blocks smaller than the content
    dict(windowLog=10, contentSizeFlag=0, compressionLevel=7),
    dict(literalCompressionMode=O.ZSTD_LCM_UNCOMPRESSED),   # raw literals beside sequences
    dict(maxBlockSize=1024),
    dict(maxBlockSize=2048, compressionLevel=9),
    dict(targetCBlockSize=1340),                              # treeless literals, Repeat_Mode tables
    dict(targetCBlockSize=1340, compressionLevel=12, contentSizeFlag=0),
    dict(strategy=1), dict(strategy=2), dict(strategy=4, compressionLevel=8), dict(strategy=6, compressionLevel=14),
    dict(strategy=9, compressionLevel=19),
)


def case(name, mt, rows, first, raw, frame, zstd_ok=True):
    return dict(name=name, mt=int(mt), rows=rows, first=int(first), raw=np.ascontiguousarray(raw, dtype=np.uint8),
                frame=np.ascontiguousarray(frame, dtype=np.uint8), zstd_ok=bool(zstd_ok))


def varint_column(rng, kind, rows, delta2):
    """a MarshalType 1 (delta2) / 4 (delta) column's varint stream -> (mt, first value, raw bytes)"""
    import blockgen
    vals = blockgen.gen_values(rng, kind, rows)
    raw, first = O.marshal_nearest_delta(vals, 64, delta2=delta2)
    return (1 if delta2 else 4), first, raw


def sequence_cases(rng, nseq=120):
    """frames whose sequences are dictated (every repeat-offset form, overlapping short offsets, long matches), as columns:
    the literals are bytes < 0x80, so the content is a stream of one-byte varints"""
    out = []
    seqs, src = repcode_sequences(rng, nseq)
    seqs = [tuple(s) for s in seqs]
    delim = [(0, 5, 0)]
    half = len(seqs) // 2
    n_half = sum(ll + ml for _, ll, ml in seqs[:half])
    variants = [
        ("seq_one_block", seqs + delim, {}),
        ("seq_checksum", seqs + delim, dict(checksumFlag=1)),
        ("seq_no_fcs", seqs + delim, dict(contentSizeFlag=0)),
        ("seq_two_blocks", seqs[:half] + [(0, 0, 0)] + seqs[half:] + delim, {}),
        # the first half of the content as one block of literals only; the second half's offsets reach back into it
        ("seq_literals_only_block", [(0, n_half, 0)] + seqs[half:] + delim, {}),
    ]
    for name, s, p in variants:
        out.append(case(name, 4, len(src) + 1, 0, src, O.zstd_ref_compress_sequences(src, s, **p)))
    # literals all one byte: RLE literals beside sequences
    rseqs = [(1, 3, 6), (2, 1, 9), (4, 0, 5)] * 40
    rsrc = run_sequences(rseqs, np.array([5]), rng, tail=2)
    for name, p in (("seq_rle_literals", {}), ("seq_rle_literals_no_fcs", dict(contentSizeFlag=0))):
        out.append(case(name, 4, len(rsrc) + 1, 0, rsrc, O.zstd_ref_compress_sequences(rsrc, rseqs + [(0, 2, 0)], **p)))
    return out


def error_cases(rng):
    """frames libzstd or the reference's varint check rejects, each with a Window_Descriptor and no Frame_Content_Size"""
    out = []
    mt, first, raw = varint_column(rng, "gauge", 100, False)
    f = pure_go_frame(raw)
    assert len(raw) < 256 and 0x00 == f[4]
    out.append(case("err_no_fcs_truncated", mt, 100, first, raw, f[:-3], zstd_ok=False))
    # content over 10 bytes per row: libzstd decodes it, the varint decode of rows - 1 values leaves a tail
    out.append(case("err_no_fcs_over_10_bytes_per_row", mt, len(raw) // 10 - 1, first, raw, f))
    # a Compressed block larger than the declared window (2 KiB of content under a 1 KiB Window_Descriptor)
    for _ in range(20):
        mt, first, raw = varint_column(rng, "counter", 700, True)
        if 1024 < len(raw) <= 2048:
            break
    f = O.zstd_ref_compress_params(raw, contentSizeFlag=0, windowLog=11).copy()
    assert f[4] == 0x00 and f[5] == 0x08 and (f[6] >> 1) & 3 == 2 and f[6] & 1, "one Compressed block under a 2 KiB window"
    f[5] = 0x00
    out.append(case("err_block_over_window", mt, 700, first, raw, f, zstd_ok=False))
    return out


def pure_go_cases(rng):
    """varint streams of 128..1024 bytes in the pure-Go writer's header layouts"""
    out = []
    for kind, rows in (("gauge", 60), ("counter", 90), ("gauge_small", 130), ("counter_resets", 200), ("gauge", 300),
                       ("counter", 400), ("gauge_wide", 120)):
        for delta2 in (False, True):
            mt, first, raw = varint_column(rng, kind, rows, delta2)
            if not 128 <= len(raw) <= 1024:
                continue
            for level in (1, 3):
                out.append(case("pure_go_%s_r%d_n%d_l%d" % (kind, rows, len(raw), level), mt, rows, first, raw,
                                pure_go_frame(raw, compressionLevel=level)))
    return out


def level_cases(rng, levels, rows_choices=ROWS):
    import blockgen
    out = []
    kinds = [k for k in blockgen.VALUE_KINDS if k not in ("const",)]
    for i, level in enumerate(levels):
        rows = rows_choices[i % len(rows_choices)]
        kind = kinds[i % len(kinds)]
        mt, first, raw = varint_column(rng, kind, rows, i % 2 == 0)
        out.append(case("level%d_%s_r%d" % (level, kind, rows), mt, rows, first, raw, O.zstd_ref_compress_params(raw, compressionLevel=level)))
    return out


def param_cases(rng, rows_choices=ROWS):
    import blockgen
    out = []
    kinds = [k for k in blockgen.VALUE_KINDS if k not in ("const",)]
    for i, p in enumerate(PARAM_SETS):
        for j, rows in enumerate((rows_choices[i % len(rows_choices)], 8192)):
            kind = kinds[(i + j) % len(kinds)]
            mt, first, raw = varint_column(rng, kind, rows, (i + j) % 2 == 0)
            name = "params_" + "_".join("%s%d" % kv for kv in p.items()) + "_%s_r%d" % (kind, rows)
            out.append(case(name, mt, rows, first, raw, O.zstd_ref_compress_params(raw, **p)))
    return out


def live_corpus(seed):
    """the full sweep (needs oracle/_ref): levels -7..22, the parameter sets, pure-Go headers, dictated sequences, errors"""
    rng = np.random.default_rng(seed)
    return (level_cases(rng, LEVELS) + level_cases(rng, LEVELS, rows_choices=ROWS[::-1]) + param_cases(rng) +
            pure_go_cases(rng) + sequence_cases(rng) + error_cases(rng))
