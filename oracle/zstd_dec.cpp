// ORACLE (test infrastructure, not product code): a from-the-spec zstd frame decoder.
//
// The reference decompresses MarshalType 1/4 columns with libzstd 1.5.7 through cgo
// (/root/reference/lib/encoding/compress.go:27 -> lib/encoding/zstd/zstd_cgo.go:13 ->
// vendor/github.com/valyala/gozstd/gozstd.go:187 -> ZSTD_decompressDCtx).  libzstd's C sources are
// NOT vendored in the reference (only the prebuilt .a), so this file restates the published format
// (RFC 8878 "Zstandard Compression and the 'application/zstd' Media Type") and is pinned against the
// reference's own libzstd through oracle/_ref (tests/test_oracle_zstd.py: frames produced by
// ZSTD_compressCCtx at levels -5..5 on the codec's varint streams must decode byte-identically).
#include <string.h>

#include <algorithm>
#include <vector>

#include "vm_oracle.h"

namespace {

struct Err {};

inline int highbit32(uint32_t v) { return 31 - __builtin_clz(v); }

// ---- forward (LSB-first) bit reader: FSE table descriptions (RFC 8878 4.1.1)
struct FwdBits {
    const uint8_t* p;
    size_t len;
    size_t bitpos = 0;
    uint32_t peek(int nb) const {
        uint64_t v = 0;
        size_t byte = bitpos >> 3;
        for (int i = 0; i < 5; i++)
            if (byte + i < len) v |= (uint64_t)p[byte + i] << (8 * i);
        return (uint32_t)((v >> (bitpos & 7)) & ((1ull << nb) - 1));
    }
    void skip(int nb) { bitpos += nb; }
    size_t bytes_consumed() const { return (bitpos + 7) >> 3; }
};

// ---- backward bit reader (RFC 8878 4.1 "Bitstreams"): the last byte holds a final-bit marker
struct BackBits {
    const uint8_t* p;
    int64_t bits_left;  // number of unread payload bits; may go negative (reads zeros) => corruption if final < 0
    void init(const uint8_t* src, size_t len) {
        if (len == 0) throw Err();
        p = src;
        uint8_t last = src[len - 1];
        if (last == 0) throw Err();
        bits_left = (int64_t)(len - 1) * 8 + highbit32(last);
    }
    // read nb bits (nb <= 32), most significant first from the stream end
    uint32_t read(int nb) {
        if (nb == 0) return 0;
        uint32_t v = peek(nb);
        bits_left -= nb;
        return v;
    }
    uint32_t peek(int nb) const {
        // bits [bits_left-nb, bits_left) ; positions below 0 read as zero
        uint64_t acc = 0;
        int64_t lo = bits_left - nb;
        for (int i = 0; i < nb; i++) {
            int64_t pos = lo + i;
            uint32_t bit = 0;
            if (pos >= 0) bit = (p[pos >> 3] >> (pos & 7)) & 1u;
            acc |= (uint64_t)bit << i;
        }
        return (uint32_t)acc;
    }
};

// ---- FSE decoding table (RFC 8878 4.1.1)
struct FseEntry {
    uint8_t symbol;
    uint8_t nbits;
    uint16_t base;
};
struct FseTable {
    int log = 0;
    std::vector<FseEntry> e;
};

void fse_build(FseTable& t, const int16_t* norm, int nsym, int log) {
    int size = 1 << log;
    t.log = log;
    t.e.assign(size, FseEntry{0, 0, 0});
    std::vector<uint16_t> next(nsym);
    int high = size - 1;
    for (int s = 0; s < nsym; s++) {
        if (norm[s] == -1) {
            t.e[high--].symbol = (uint8_t)s;
            next[s] = 1;
        } else {
            next[s] = (uint16_t)norm[s];
        }
    }
    int step = (size >> 1) + (size >> 3) + 3;
    int mask = size - 1;
    int pos = 0;
    for (int s = 0; s < nsym; s++) {
        for (int i = 0; i < norm[s]; i++) {
            t.e[pos].symbol = (uint8_t)s;
            do {
                pos = (pos + step) & mask;
            } while (pos > high);
        }
    }
    if (pos != 0) throw Err();
    for (int i = 0; i < size; i++) {
        int s = t.e[i].symbol;
        uint16_t ns = next[s]++;
        int nb = log - highbit32(ns);
        t.e[i].nbits = (uint8_t)nb;
        t.e[i].base = (uint16_t)((ns << nb) - size);
    }
}

// reads a normalized-count header; returns bytes consumed
size_t fse_read_ncount(int16_t* norm, int* nsym_out, int* log_out, int max_sym, int max_log, const uint8_t* src,
                       size_t len) {
    FwdBits b{src, len};
    int log = (int)b.peek(4) + 5;
    b.skip(4);
    if (log > max_log) throw Err();
    int remaining = (1 << log) + 1;
    int threshold = 1 << log;
    int nbits = log + 1;
    int sym = 0;
    bool prev0 = false;
    while (remaining > 1 && sym <= max_sym) {
        if (prev0) {
            // repeat flags: 2 bits each, value 3 means "continue"
            for (;;) {
                int r = (int)b.peek(2);
                b.skip(2);
                for (int k = 0; k < r; k++) {
                    if (sym > max_sym) throw Err();
                    norm[sym++] = 0;
                }
                if (r != 3) break;
            }
            prev0 = false;
            continue;
        }
        int max = (2 * threshold - 1) - remaining;
        int count;
        uint32_t bits = b.peek(nbits);
        if ((int)(bits & (uint32_t)(threshold - 1)) < max) {
            count = (int)(bits & (uint32_t)(threshold - 1));
            b.skip(nbits - 1);
        } else {
            count = (int)(bits & (uint32_t)(2 * threshold - 1));
            if (count >= threshold) count -= max;
            b.skip(nbits);
        }
        count--;  // -1 == "less than 1"
        remaining -= count < 0 ? -count : count;
        if (sym > max_sym) throw Err();
        norm[sym++] = (int16_t)count;
        prev0 = (count == 0);
        while (remaining < threshold) {
            nbits--;
            threshold >>= 1;
        }
    }
    if (remaining != 1) throw Err();
    if (b.bytes_consumed() > len) throw Err();
    *nsym_out = sym;
    *log_out = log;
    return b.bytes_consumed();
}

// ---- Huffman (RFC 8878 4.2)
struct HufTable {
    int log = 0;              // Max_Number_of_Bits
    std::vector<uint16_t> e;  // (nbits << 8) | symbol
    bool valid = false;
};

size_t huf_read_table(HufTable& t, const uint8_t* src, size_t len) {
    if (len < 1) throw Err();
    uint8_t weights[256];
    int nw = 0;
    size_t consumed;
    uint8_t hb = src[0];
    if (hb >= 128) {
        nw = hb - 127;
        size_t nbytes = (size_t)(nw + 1) / 2;
        if (1 + nbytes > len) throw Err();
        for (int i = 0; i < nw; i++) {
            uint8_t b = src[1 + i / 2];
            weights[i] = (i & 1) ? (b & 15) : (b >> 4);
        }
        consumed = 1 + nbytes;
    } else {
        size_t csize = hb;
        if (1 + csize > len || csize < 2) throw Err();
        int16_t norm[256];
        int nsym, log;
        size_t hdr = fse_read_ncount(norm, &nsym, &log, 255, 6, src + 1, csize);
        FseTable ft;
        fse_build(ft, norm, nsym, log);
        BackBits bb;
        bb.init(src + 1 + hdr, csize - hdr);
        uint32_t s1 = bb.read(log), s2 = bb.read(log);
        // two interleaved states (RFC 8878 4.2.1.2)
        for (;;) {
            if (nw >= 255) throw Err();
            weights[nw++] = ft.e[s1].symbol;
            if (bb.bits_left < ft.e[s1].nbits) {  // cannot update state 1 any more
                if (nw >= 255) throw Err();
                weights[nw++] = ft.e[s2].symbol;
                break;
            }
            s1 = ft.e[s1].base + bb.read(ft.e[s1].nbits);
            if (nw >= 255) throw Err();
            weights[nw++] = ft.e[s2].symbol;
            if (bb.bits_left < ft.e[s2].nbits) {
                if (nw >= 255) throw Err();
                weights[nw++] = ft.e[s1].symbol;
                break;
            }
            s2 = ft.e[s2].base + bb.read(ft.e[s2].nbits);
        }
        consumed = 1 + csize;
    }
    // implicit last weight
    uint32_t total = 0;
    for (int i = 0; i < nw; i++) {
        if (weights[i] > 11) throw Err();
        if (weights[i]) total += 1u << (weights[i] - 1);
    }
    if (total == 0) throw Err();
    int log = highbit32(total) + 1;
    if (log > 11) throw Err();
    uint32_t rest = (1u << log) - total;
    if (rest == 0 || (rest & (rest - 1))) throw Err();
    weights[nw++] = (uint8_t)(highbit32(rest) + 1);
    // table fill: weight ascending, symbol ascending within a weight
    t.log = log;
    t.e.assign((size_t)1 << log, 0);
    uint32_t pos = 0;
    for (int w = 1; w <= log; w++) {
        for (int s = 0; s < nw; s++) {
            if (weights[s] != w) continue;
            uint32_t span = 1u << (w - 1);
            uint16_t ent = (uint16_t)(((log + 1 - w) << 8) | s);
            for (uint32_t k = 0; k < span; k++) t.e[pos + k] = ent;
            pos += span;
        }
    }
    if (pos != (1u << log)) throw Err();
    t.valid = true;
    return consumed;
}

void huf_decode_stream(const HufTable& t, uint8_t* dst, size_t n, const uint8_t* src, size_t len) {
    BackBits bb;
    bb.init(src, len);
    for (size_t i = 0; i < n; i++) {
        uint16_t ent = t.e[bb.peek(t.log)];
        dst[i] = (uint8_t)ent;
        bb.bits_left -= ent >> 8;
    }
    if (bb.bits_left != 0) throw Err();  // stream must be consumed exactly
}

// ---- sequences (RFC 8878 3.1.1.3.2)
const int16_t LL_DEFAULT[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2,
                                2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1};
const int16_t ML_DEFAULT[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                                1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
const int16_t OF_DEFAULT[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};
const uint32_t LL_BASE[36] = {0,  1,  2,  3,  4,  5,  6,  7,  8,  9,   10,  11,  12,   13,   14,   15,   16,   18,
                              20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536};
const uint8_t LL_BITS[36] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1,
                             1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
const uint32_t ML_BASE[53] = {3,  4,  5,  6,  7,  8,  9,  10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20,
                              21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33, 34, 35, 37, 39, 41,
                              43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539};
const uint8_t ML_BITS[53] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
                             0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};

struct FrameCtx {
    HufTable huf;
    FseTable ll, of, ml;
    bool have_ll = false, have_of = false, have_ml = false;
    uint64_t rep[3] = {1, 4, 8};
};

// reads one table per its mode; returns bytes consumed
size_t read_seq_table(FseTable& t, bool& have, int mode, const int16_t* defnorm, int defn, int deflog, int max_sym,
                      int max_log, const uint8_t* src, size_t len) {
    switch (mode) {
        case 0:
            fse_build(t, defnorm, defn, deflog);
            have = true;
            return 0;
        case 1: {
            if (len < 1) throw Err();
            if (src[0] > max_sym) throw Err();
            t.log = 0;
            t.e.assign(1, FseEntry{src[0], 0, 0});
            have = true;
            return 1;
        }
        case 2: {
            int16_t norm[64];
            int nsym, log;
            size_t used = fse_read_ncount(norm, &nsym, &log, max_sym, max_log, src, len);
            fse_build(t, norm, nsym, log);
            have = true;
            return used;
        }
        default:
            if (!have) throw Err();
            return 0;
    }
}

size_t decode_block(FrameCtx& fc, uint8_t* out_base, size_t out_pos, size_t out_cap, const uint8_t* src, size_t len) {
    if (len < 1) throw Err();
    // ---- literals section
    std::vector<uint8_t> lits;
    size_t pos = 0;
    {
        uint8_t b0 = src[0];
        int type = b0 & 3;
        int sf = (b0 >> 2) & 3;
        if (type == 0 || type == 1) {
            size_t regen, hdr;
            if ((sf & 1) == 0) {
                regen = b0 >> 3;
                hdr = 1;
            } else if (sf == 1) {
                if (len < 2) throw Err();
                regen = (b0 >> 4) | ((size_t)src[1] << 4);
                hdr = 2;
            } else {
                if (len < 3) throw Err();
                regen = (b0 >> 4) | ((size_t)src[1] << 4) | ((size_t)src[2] << 12);
                hdr = 3;
            }
            pos = hdr;
            lits.resize(regen);
            if (type == 0) {
                if (pos + regen > len) throw Err();
                memcpy(lits.data(), src + pos, regen);
                pos += regen;
            } else {
                if (pos + 1 > len) throw Err();
                memset(lits.data(), src[pos], regen);
                pos += 1;
            }
        } else {
            size_t regen, csize, hdr;
            int streams = 4;
            if (sf == 0 || sf == 1) {
                if (len < 3) throw Err();
                uint32_t v = src[0] | ((uint32_t)src[1] << 8) | ((uint32_t)src[2] << 16);
                regen = (v >> 4) & 0x3ff;
                csize = (v >> 14) & 0x3ff;
                hdr = 3;
                if (sf == 0) streams = 1;
            } else if (sf == 2) {
                if (len < 4) throw Err();
                uint32_t v = src[0] | ((uint32_t)src[1] << 8) | ((uint32_t)src[2] << 16) | ((uint32_t)src[3] << 24);
                regen = (v >> 4) & 0x3fff;
                csize = (v >> 18) & 0x3fff;
                hdr = 4;
            } else {
                if (len < 5) throw Err();
                uint64_t v = src[0] | ((uint64_t)src[1] << 8) | ((uint64_t)src[2] << 16) | ((uint64_t)src[3] << 24) |
                             ((uint64_t)src[4] << 32);
                regen = (v >> 4) & 0x3ffff;
                csize = (v >> 22) & 0x3ffff;
                hdr = 5;
            }
            pos = hdr;
            if (pos + csize > len) throw Err();
            const uint8_t* lp = src + pos;
            size_t lrem = csize;
            if (type == 2) {
                size_t used = huf_read_table(fc.huf, lp, lrem);
                lp += used;
                lrem -= used;
            } else if (!fc.huf.valid) {
                throw Err();
            }
            lits.resize(regen);
            if (streams == 1) {
                huf_decode_stream(fc.huf, lits.data(), regen, lp, lrem);
            } else {
                if (lrem < 6) throw Err();
                size_t s1 = lp[0] | (lp[1] << 8), s2 = lp[2] | (lp[3] << 8), s3 = lp[4] | (lp[5] << 8);
                if (6 + s1 + s2 + s3 > lrem) throw Err();
                size_t s4 = lrem - 6 - s1 - s2 - s3;
                size_t seg = (regen + 3) / 4;
                if (seg * 3 > regen) throw Err();
                const uint8_t* q = lp + 6;
                huf_decode_stream(fc.huf, lits.data(), seg, q, s1);
                huf_decode_stream(fc.huf, lits.data() + seg, seg, q + s1, s2);
                huf_decode_stream(fc.huf, lits.data() + 2 * seg, seg, q + s1 + s2, s3);
                huf_decode_stream(fc.huf, lits.data() + 3 * seg, regen - 3 * seg, q + s1 + s2 + s3, s4);
            }
            pos += csize;
        }
    }
    // ---- sequences section
    if (pos >= len) throw Err();
    size_t nseq;
    {
        uint8_t b0 = src[pos];
        if (b0 == 0) {
            nseq = 0;
            pos += 1;
        } else if (b0 < 128) {
            nseq = b0;
            pos += 1;
        } else if (b0 < 255) {
            if (pos + 2 > len) throw Err();
            nseq = ((size_t)(b0 - 128) << 8) + src[pos + 1];
            pos += 2;
        } else {
            if (pos + 3 > len) throw Err();
            nseq = (size_t)src[pos + 1] + ((size_t)src[pos + 2] << 8) + 0x7F00;
            pos += 3;
        }
    }
    size_t o = out_pos;
    size_t lit_pos = 0;
    if (nseq > 0) {
        if (pos >= len) throw Err();
        uint8_t modes = src[pos++];
        if (modes & 3) throw Err();
        pos += read_seq_table(fc.ll, fc.have_ll, (modes >> 6) & 3, LL_DEFAULT, 36, 6, 35, 9, src + pos, len - pos);
        pos += read_seq_table(fc.of, fc.have_of, (modes >> 4) & 3, OF_DEFAULT, 29, 5, 31, 8, src + pos, len - pos);
        pos += read_seq_table(fc.ml, fc.have_ml, (modes >> 2) & 3, ML_DEFAULT, 53, 6, 52, 9, src + pos, len - pos);
        if (pos >= len) throw Err();
        BackBits bb;
        bb.init(src + pos, len - pos);
        uint32_t sll = bb.read(fc.ll.log), sof = bb.read(fc.of.log), sml = bb.read(fc.ml.log);
        for (size_t i = 0; i < nseq; i++) {
            uint8_t ofc = fc.of.e[sof].symbol, mlc = fc.ml.e[sml].symbol, llc = fc.ll.e[sll].symbol;
            if (ofc > 31 || mlc > 52 || llc > 35) throw Err();
            uint64_t ofv = ((uint64_t)1 << ofc) + bb.read(ofc);
            uint32_t mlen = ML_BASE[mlc] + bb.read(ML_BITS[mlc]);
            uint32_t llen = LL_BASE[llc] + bb.read(LL_BITS[llc]);
            if (i + 1 < nseq) {
                sll = fc.ll.e[sll].base + bb.read(fc.ll.e[sll].nbits);
                sml = fc.ml.e[sml].base + bb.read(fc.ml.e[sml].nbits);
                sof = fc.of.e[sof].base + bb.read(fc.of.e[sof].nbits);
            }
            if (bb.bits_left < 0) throw Err();
            // repeat offsets (RFC 8878 3.1.1.5)
            uint64_t offset;
            if (ofv > 3) {
                offset = ofv - 3;
                fc.rep[2] = fc.rep[1];
                fc.rep[1] = fc.rep[0];
                fc.rep[0] = offset;
            } else {
                uint64_t idx = ofv - 1 + (llen == 0 ? 1 : 0);
                if (idx == 0) {
                    offset = fc.rep[0];
                } else {
                    offset = idx < 3 ? fc.rep[idx] : fc.rep[0] - 1;
                    if (offset == 0) throw Err();
                    if (idx > 1) fc.rep[2] = fc.rep[1];
                    fc.rep[1] = fc.rep[0];
                    fc.rep[0] = offset;
                }
            }
            if (lit_pos + llen > lits.size()) throw Err();
            if (o + llen + mlen > out_cap) throw Err();
            memcpy(out_base + o, lits.data() + lit_pos, llen);
            o += llen;
            lit_pos += llen;
            if (offset > o) throw Err();  // no dictionary / no window beyond the frame start
            for (uint32_t k = 0; k < mlen; k++) out_base[o + k] = out_base[o + k - offset];
            o += mlen;
        }
        if (bb.bits_left != 0) throw Err();
    } else if (pos != len) {
        throw Err();
    }
    size_t rest = lits.size() - lit_pos;
    if (o + rest > out_cap) throw Err();
    memcpy(out_base + o, lits.data() + lit_pos, rest);
    o += rest;
    return o - out_pos;
}

struct FrameHdr {
    size_t hdr_size;
    bool has_fcs;
    uint64_t fcs;
    bool checksum;
    uint64_t block_max;  // Block_Maximum_Size = min(Window_Size, 128 KiB)
};

FrameHdr parse_frame_header(const uint8_t* src, size_t len) {
    if (len < 5) throw Err();
    if (!(src[0] == 0x28 && src[1] == 0xB5 && src[2] == 0x2F && src[3] == 0xFD)) throw Err();
    uint8_t fhd = src[4];
    int fcs_flag = fhd >> 6;
    bool single = (fhd >> 5) & 1;
    if (fhd & 0x08) throw Err();  // reserved bit
    bool checksum = (fhd >> 2) & 1;
    int did_flag = fhd & 3;
    size_t pos = 5;
    if (!single) pos += 1;  // window descriptor
    static const int did_sizes[4] = {0, 1, 2, 4};
    if (did_flag != 0) {
        // dictionaries are never used on this path (gozstd.Decompress passes dd=nil)
        uint64_t did = 0;
        if (pos + did_sizes[did_flag] > len) throw Err();
        for (int i = 0; i < did_sizes[did_flag]; i++) did |= (uint64_t)src[pos + i] << (8 * i);
        if (did != 0) throw Err();
        pos += did_sizes[did_flag];
    }
    int fcs_size = 0;
    if (fcs_flag == 0) fcs_size = single ? 1 : 0;
    else fcs_size = 1 << fcs_flag;
    if (pos + fcs_size > len) throw Err();
    uint64_t fcs = 0;
    for (int i = 0; i < fcs_size; i++) fcs |= (uint64_t)src[pos + i] << (8 * i);
    if (fcs_size == 2) fcs += 256;
    pos += fcs_size;
    uint64_t window = fcs;  // Single_Segment_Flag: the window is the content
    if (!single) {
        // Window_Descriptor (RFC 8878 3.1.1.1.2)
        const int wlog = 10 + (src[5] >> 3);
        window = (1ull << wlog) + ((1ull << wlog) / 8) * (src[5] & 7);
    }
    return FrameHdr{pos, fcs_size != 0, fcs, checksum, std::min<uint64_t>(window, 128 << 10)};
}

}  // namespace

extern "C" {

int64_t vmo_zstd_content_size(const uint8_t* src, size_t len) {
    try {
        FrameHdr h = parse_frame_header(src, len);
        if (!h.has_fcs) return VMO_ERR_ZSTD;
        return (int64_t)h.fcs;
    } catch (Err&) {
        return VMO_ERR_ZSTD;
    }
}

// Frame_Content_Size when the frame has one; otherwise an upper bound of the content from the block headers (Raw and RLE
// blocks exactly, a Compressed block at most Block_Maximum_Size).  Errors when the block headers run past the frame.
int64_t vmo_zstd_content_bound(const uint8_t* src, size_t len) {
    try {
        FrameHdr h = parse_frame_header(src, len);
        if (h.has_fcs) return (int64_t)h.fcs;
        uint64_t bound = 0;
        size_t pos = h.hdr_size;
        for (;;) {
            if (pos + 3 > len) throw Err();
            uint32_t bh = src[pos] | ((uint32_t)src[pos + 1] << 8) | ((uint32_t)src[pos + 2] << 16);
            pos += 3;
            int type = (bh >> 1) & 3;
            size_t bsize = bh >> 3;
            if (type == 3) throw Err();
            size_t stored = type == 1 ? 1 : bsize;
            if (pos + stored > len) throw Err();
            pos += stored;
            bound += type == 2 ? h.block_max : bsize;
            if (bh & 1) break;
        }
        return (int64_t)bound;
    } catch (Err&) {
        return VMO_ERR_ZSTD;
    }
}

int64_t vmo_zstd_decompress(uint8_t* dst, size_t cap, const uint8_t* src, size_t len) {
    try {
        FrameHdr h = parse_frame_header(src, len);
        size_t pos = h.hdr_size;
        size_t o = 0;
        FrameCtx fc;
        for (;;) {
            if (pos + 3 > len) throw Err();
            uint32_t bh = src[pos] | ((uint32_t)src[pos + 1] << 8) | ((uint32_t)src[pos + 2] << 16);
            pos += 3;
            bool last = bh & 1;
            int type = (bh >> 1) & 3;
            size_t bsize = bh >> 3;
            if (type == 0) {
                if (pos + bsize > len || o + bsize > cap) throw Err();
                memcpy(dst + o, src + pos, bsize);
                pos += bsize;
                o += bsize;
            } else if (type == 1) {
                if (pos + 1 > len || o + bsize > cap) throw Err();
                memset(dst + o, src[pos], bsize);
                pos += 1;
                o += bsize;
            } else if (type == 2) {
                if (pos + bsize > len) throw Err();
                size_t regen = decode_block(fc, dst, o, cap, src + pos, bsize);
                if (!h.has_fcs && regen > h.block_max) throw Err();  // libzstd: a block larger than the window is corrupt
                o += regen;
                pos += bsize;
            } else {
                throw Err();
            }
            if (last) break;
        }
        if (h.checksum) pos += 4;  // XXH64 low 32 bits: not verified (gozstd frames carry none)
        if (pos != len) throw Err();
        if (h.has_fcs && h.fcs != o) throw Err();
        return (int64_t)o;
    } catch (Err&) {
        return VMO_ERR_ZSTD;
    }
}

}  // extern "C"
