// In-kernel zstd frame decoding for MarshalType 1/4 columns.
//
// Replaces lib/encoding/compress.go:27 DecompressZSTD -> lib/encoding/zstd/zstd_cgo.go:13 -> gozstd.Decompress
// (vendor/github.com/valyala/gozstd/gozstd.go:187 -> libzstd ZSTD_decompressDCtx) for every compressed column of a
// batch at once.  The format is the published one (RFC 8878); frames written by the reference are single-segment,
// checksum-less, dictionary-less and (for <=128 KiB columns) single-block (SURVEY.md section 7, "Measured frame shapes").
//
// Three kernels:
//   k_zstd_prepare : one thread per frame of the common shape (one Compressed block, Huffman-coded literals):
//                    parses headers + the Huffman tree description into a HufJob.
//   k_huf_decode   : the hot one. Lane-packed: every lane owns ONE Huffman bitstream (4 per frame => 8 frames per
//                    warp); decode tables (symbol by code prefix, length by symbol) live in shared memory; the
//                    compressed stream reaches the lane through a private shared-memory ring that is filled by
//                    warp-uniform 16-byte loads issued two phases ahead; output is staged in shared memory and written
//                    out by the whole warp, 4 streams x 128 contiguous bytes per store instruction.
//   k_zstd_serial  : one thread per frame: (a) executes the sequences section of prepared frames, (b) decodes any
//                    frame of another shape (raw/RLE blocks, multi-block, raw/RLE/treeless literals) completely.
#include "common.cuh"
#include <mutex>

// ------------------------------------------------------------------------------------------------ shared pieces
namespace {

__device__ __forceinline__ int hb32(uint32_t v) { return 31 - __clz((int)v); }

// backward bitstream (RFC 8878 4.1): MSB-aligned 64-bit window
struct BitR {
    const uint8_t* base;
    int pos;        // bytes of the stream not yet pulled into the window
    uint64_t buf;   // next bits at the top
    int cnt;        // bits in buf (may count zero padding pulled from before the stream start)
    long long left; // payload bits not yet consumed; < 0 => the stream was over-read (corruption)

    __device__ __forceinline__ void refill() {  // requires cnt <= 32
        uint32_t w;
        if (pos >= 4) {
            w = load_u32_unaligned(base + pos - 4);
            pos -= 4;
        } else {
            w = 0;
            for (int i = 0; i < pos; i++) w |= (uint32_t)base[i] << (8 * i);
            w = pos ? (w << (8 * (4 - pos))) : 0u;
            pos = 0;
        }
        buf |= (uint64_t)w << (32 - cnt);
        cnt += 32;
    }
    __device__ bool init(const uint8_t* src, uint32_t len) {
        if (len == 0) return false;
        uint32_t last = src[len - 1];
        if (last == 0) return false;
        base = src;
        pos = (int)len;
        buf = 0;
        cnt = 0;
        left = (long long)(len - 1) * 8 + hb32(last);
        refill();
        int skip = 8 - hb32(last);  // zero padding + the final-bit marker
        buf <<= skip;
        cnt -= skip;
        return true;
    }
    __device__ __forceinline__ uint32_t peek(int nb) {  // 1 <= nb <= 32
        if (cnt < nb) refill();
        return (uint32_t)(buf >> (64 - nb));
    }
    __device__ __forceinline__ void skip(int nb) {
        buf <<= nb;
        cnt -= nb;
        left -= nb;
    }
    __device__ __forceinline__ uint32_t read(int nb) {  // 0 <= nb <= 32
        if (nb == 0) return 0;
        uint32_t v = peek(nb);
        skip(nb);
        return v;
    }
};

// forward LSB-first bit reader for FSE table descriptions (RFC 8878 4.1.1)
struct FwdR {
    const uint8_t* p;
    uint32_t len;
    uint32_t bitpos;
    __device__ uint32_t peek(int nb) const {
        uint32_t byte = bitpos >> 3;
        uint64_t v = 0;
        for (int i = 0; i < 5; i++)
            if (byte + i < len) v |= (uint64_t)p[byte + i] << (8 * i);
        return (uint32_t)((v >> (bitpos & 7)) & ((1ull << nb) - 1));
    }
};

// FSE decoding table entry: base(16) | nbits(8) | symbol(8)
__device__ __forceinline__ uint32_t fse_pack(uint32_t base, uint32_t nbits, uint32_t sym) {
    return (base << 16) | (nbits << 8) | sym;
}
#define FSE_SYM(e) ((e) & 0xffu)
#define FSE_NB(e) (((e) >> 8) & 0xffu)
#define FSE_BASE(e) ((e) >> 16)

// returns bytes consumed or 0 on error
__device__ uint32_t fse_read_ncount(short* norm, int* nsym_out, int* log_out, int max_sym, int max_log,
                                    const uint8_t* src, uint32_t len) {
    FwdR b{src, len, 0};
    int log = (int)b.peek(4) + 5;
    b.bitpos += 4;
    if (log > max_log) return 0;
    int remaining = (1 << log) + 1, threshold = 1 << log, nbits = log + 1, sym = 0;
    bool prev0 = false;
    while (remaining > 1 && sym <= max_sym) {
        if (prev0) {
            for (;;) {
                int r = (int)b.peek(2);
                b.bitpos += 2;
                for (int k = 0; k < r; k++) {
                    if (sym > max_sym) return 0;
                    norm[sym++] = 0;
                }
                if (r != 3) break;
                if (b.bitpos > len * 8u + 16u) return 0;
            }
            prev0 = false;
            continue;
        }
        int maxv = (2 * threshold - 1) - remaining;
        int count;
        uint32_t bits = b.peek(nbits);
        if ((int)(bits & (uint32_t)(threshold - 1)) < maxv) {
            count = (int)(bits & (uint32_t)(threshold - 1));
            b.bitpos += nbits - 1;
        } else {
            count = (int)(bits & (uint32_t)(2 * threshold - 1));
            if (count >= threshold) count -= maxv;
            b.bitpos += nbits;
        }
        count--;
        remaining -= count < 0 ? -count : count;
        if (sym > max_sym) return 0;
        norm[sym++] = (short)count;
        prev0 = (count == 0);
        while (remaining < threshold) {
            nbits--;
            threshold >>= 1;
        }
    }
    if (remaining != 1) return 0;
    uint32_t used = (b.bitpos + 7) >> 3;
    if (used > len) return 0;
    *nsym_out = sym;
    *log_out = log;
    return used;
}

// builds the decoding table (size 1<<log entries) ; `next` is scratch for nsym uint16. returns false on error
__device__ bool fse_build(uint32_t* table, const short* norm, int nsym, int log, unsigned short* next) {
    int size = 1 << log;
    int high = size - 1;
    for (int s = 0; s < nsym; s++) {
        if (norm[s] == -1) {
            table[high--] = (uint32_t)s;
            next[s] = 1;
        } else {
            next[s] = (unsigned short)norm[s];
        }
    }
    int step = (size >> 1) + (size >> 3) + 3, mask = size - 1, pos = 0;
    for (int s = 0; s < nsym; s++) {
        for (int i = 0; i < norm[s]; i++) {
            table[pos] = (uint32_t)s;
            do {
                pos = (pos + step) & mask;
            } while (pos > high);
        }
    }
    if (pos != 0) return false;
    for (int i = 0; i < size; i++) {
        uint32_t s = table[i];
        uint32_t ns = next[s]++;
        int nb = log - hb32(ns);
        table[i] = fse_pack((ns << nb) - (uint32_t)size, (uint32_t)nb, s);
    }
    return true;
}

// Huffman tree description (RFC 8878 4.2.1) -> code length per symbol.  `ftab` : scratch for 64 uint32 + 256 shorts.
// returns bytes consumed, 0 on error
__device__ uint32_t huf_read_weights(uint8_t* nbits_out /*256*/, int* table_log, const uint8_t* src, uint32_t len,
                                     uint32_t* ftab, short* norm, unsigned short* next) {
    if (len < 1) return 0;
    uint8_t* weights = nbits_out;  // reuse: weights first, converted to code lengths at the end
    int nw = 0;
    uint32_t consumed;
    uint32_t hb = src[0];
    if (hb >= 128) {
        nw = (int)hb - 127;
        uint32_t nbytes = (uint32_t)(nw + 1) / 2;
        if (1 + nbytes > len) return 0;
        for (int i = 0; i < nw; i++) {
            uint32_t b = src[1 + i / 2];
            weights[i] = (uint8_t)((i & 1) ? (b & 15) : (b >> 4));
        }
        consumed = 1 + nbytes;
    } else {
        uint32_t csize = hb;
        if (1 + csize > len || csize < 2) return 0;
        int nsym, log;
        uint32_t hdr = fse_read_ncount(norm, &nsym, &log, 255, 6, src + 1, csize);
        if (!hdr) return 0;
        if (!fse_build(ftab, norm, nsym, log, next)) return 0;
        BitR bb;
        if (hdr >= csize || !bb.init(src + 1 + hdr, csize - hdr)) return 0;
        uint32_t s1 = bb.read(log), s2 = bb.read(log);
        for (;;) {  // two interleaved states (RFC 8878 4.2.1.2)
            if (nw >= 255) return 0;
            uint32_t e1 = ftab[s1];
            weights[nw++] = (uint8_t)FSE_SYM(e1);
            if (bb.left < (long long)FSE_NB(e1)) {
                if (nw >= 255) return 0;
                weights[nw++] = (uint8_t)FSE_SYM(ftab[s2]);
                break;
            }
            s1 = FSE_BASE(e1) + bb.read((int)FSE_NB(e1));
            if (nw >= 255) return 0;
            uint32_t e2 = ftab[s2];
            weights[nw++] = (uint8_t)FSE_SYM(e2);
            if (bb.left < (long long)FSE_NB(e2)) {
                if (nw >= 255) return 0;
                weights[nw++] = (uint8_t)FSE_SYM(ftab[s1]);
                break;
            }
            s2 = FSE_BASE(e2) + bb.read((int)FSE_NB(e2));
        }
        consumed = 1 + csize;
    }
    uint32_t total = 0;
    for (int i = 0; i < nw; i++) {
        if (weights[i] > 11) return 0;
        if (weights[i]) total += 1u << (weights[i] - 1);
    }
    if (total == 0) return 0;
    int log = hb32(total) + 1;
    if (log > 11) return 0;
    uint32_t rest = (1u << log) - total;
    if (rest == 0 || (rest & (rest - 1))) return 0;
    weights[nw++] = (uint8_t)(hb32(rest) + 1);
    for (int i = 0; i < nw; i++) nbits_out[i] = weights[i] ? (uint8_t)(log + 1 - weights[i]) : 0;
    for (int i = nw; i < 256; i++) nbits_out[i] = 0;
    *table_log = log;
    return consumed;
}

// fills a (1<<log)-entry decode table: entry = (nbits << 8) | symbol; codes are assigned in (weight asc, symbol asc)
// order, i.e. (nbits desc, symbol asc).  Serial version for the per-thread decoder.
__device__ bool huf_fill_table_serial(unsigned short* table, const uint8_t* nbits, int log) {
    uint32_t pos = 0;
    for (int nb = log; nb >= 1; nb--) {
        uint32_t span = 1u << (log - nb);
        for (int s = 0; s < 256; s++) {
            if (nbits[s] != nb) continue;
            unsigned short ent = (unsigned short)((nb << 8) | s);
            if (pos + span > (1u << log)) return false;
            for (uint32_t k = 0; k < span; k++) table[pos + k] = ent;
            pos += span;
        }
    }
    return pos == (1u << log);
}

__device__ bool huf_decode_stream_serial(const unsigned short* table, int log, uint8_t* dst, uint32_t n,
                                         const uint8_t* src, uint32_t len) {
    BitR bb;
    if (!bb.init(src, len)) return false;
    for (uint32_t i = 0; i < n; i++) {
        unsigned short ent = table[bb.peek(log)];
        dst[i] = (uint8_t)ent;
        bb.skip(ent >> 8);
    }
    return bb.left == 0;
}

__constant__ short c_ll_default[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2,
                                       2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1};
__constant__ short c_ml_default[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                                       1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
__constant__ short c_of_default[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1,
                                       1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};
__constant__ uint32_t c_ll_base[36] = {0,  1,  2,  3,  4,  5,  6,  7,  8,  9,   10,  11,  12,   13,   14,   15,   16,   18,
                                       20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536};
__constant__ uint8_t c_ll_bits[36] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1,
                                      1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
__constant__ uint32_t c_ml_base[53] = {3,  4,  5,  6,  7,  8,  9,  10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20,
                                       21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33, 34, 35, 37, 39, 41,
                                       43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539};
__constant__ uint8_t c_ml_bits[53] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
                                      0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};

// per-thread workspace of the serial decoder (global memory)
struct SerialWs {
    uint32_t ll[512];
    uint32_t ml[512];
    uint32_t of[256];
    unsigned short huf[2048];
    short norm[256];
    unsigned short next[256];
    uint8_t nbits[256];
    int ll_log, ml_log, of_log, huf_log;
    int have_ll, have_ml, have_of, have_huf;
    unsigned long long rep[3];
};

__device__ uint32_t read_seq_table(uint32_t* table, int* tlog, int* have, int mode, const short* defnorm, int defn,
                                   int deflog, int max_sym, int max_log, const uint8_t* src, uint32_t len, SerialWs* ws,
                                   bool* ok) {
    *ok = true;
    switch (mode) {
        case 0: {
            for (int i = 0; i < defn; i++) ws->norm[i] = defnorm[i];
            if (!fse_build(table, ws->norm, defn, deflog, ws->next)) *ok = false;
            *tlog = deflog;
            *have = 1;
            return 0;
        }
        case 1: {
            if (len < 1 || src[0] > max_sym) {
                *ok = false;
                return 0;
            }
            table[0] = fse_pack(0, 0, src[0]);
            *tlog = 0;
            *have = 1;
            return 1;
        }
        case 2: {
            int nsym, log;
            uint32_t used = fse_read_ncount(ws->norm, &nsym, &log, max_sym, max_log, src, len);
            if (!used || !fse_build(table, ws->norm, nsym, log, ws->next)) {
                *ok = false;
                return 0;
            }
            *tlog = log;
            *have = 1;
            return used;
        }
        default:
            if (!*have) *ok = false;
            return 0;
    }
}

// sequences section (RFC 8878 3.1.1.3.2) + execution.  lits/lit_len: decoded literals of this block.
// Writes at out[o...]; returns new o or -1.
__device__ long long run_sequences(SerialWs* ws, uint8_t* out, long long o, long long out_cap, const uint8_t* lits,
                                   uint32_t lit_len, const uint8_t* src, uint32_t len) {
    if (len < 1) return -1;
    uint32_t pos = 0, nseq;
    uint32_t b0 = src[0];
    if (b0 == 0) { nseq = 0; pos = 1; }
    else if (b0 < 128) { nseq = b0; pos = 1; }
    else if (b0 < 255) {
        if (len < 2) return -1;
        nseq = ((b0 - 128) << 8) + src[1];
        pos = 2;
    } else {
        if (len < 3) return -1;
        nseq = (uint32_t)src[1] + ((uint32_t)src[2] << 8) + 0x7F00u;
        pos = 3;
    }
    uint32_t lit_pos = 0;
    if (nseq > 0) {
        if (pos >= len) return -1;
        uint32_t modes = src[pos++];
        if (modes & 3) return -1;
        bool ok;
        pos += read_seq_table(ws->ll, &ws->ll_log, &ws->have_ll, (modes >> 6) & 3, c_ll_default, 36, 6, 35, 9, src + pos,
                              len - pos, ws, &ok);
        if (!ok) return -1;
        pos += read_seq_table(ws->of, &ws->of_log, &ws->have_of, (modes >> 4) & 3, c_of_default, 29, 5, 31, 8, src + pos,
                              len - pos, ws, &ok);
        if (!ok) return -1;
        pos += read_seq_table(ws->ml, &ws->ml_log, &ws->have_ml, (modes >> 2) & 3, c_ml_default, 53, 6, 52, 9, src + pos,
                              len - pos, ws, &ok);
        if (!ok || pos >= len) return -1;
        BitR bb;
        if (!bb.init(src + pos, len - pos)) return -1;
        uint32_t sll = bb.read(ws->ll_log), sof = bb.read(ws->of_log), sml = bb.read(ws->ml_log);
        for (uint32_t i = 0; i < nseq; i++) {
            uint32_t ell = ws->ll[sll], eof = ws->of[sof], eml = ws->ml[sml];
            uint32_t ofc = FSE_SYM(eof), mlc = FSE_SYM(eml), llc = FSE_SYM(ell);
            if (ofc > 31 || mlc > 52 || llc > 35) return -1;
            unsigned long long ofv = (1ull << ofc) + bb.read((int)ofc);
            uint32_t mlen = c_ml_base[mlc] + bb.read(c_ml_bits[mlc]);
            uint32_t llen = c_ll_base[llc] + bb.read(c_ll_bits[llc]);
            if (i + 1 < nseq) {
                sll = FSE_BASE(ell) + bb.read((int)FSE_NB(ell));
                sml = FSE_BASE(eml) + bb.read((int)FSE_NB(eml));
                sof = FSE_BASE(eof) + bb.read((int)FSE_NB(eof));
            }
            if (bb.left < 0) return -1;
            unsigned long long offset;
            if (ofv > 3) {
                offset = ofv - 3;
                ws->rep[2] = ws->rep[1];
                ws->rep[1] = ws->rep[0];
                ws->rep[0] = offset;
            } else {
                unsigned long long idx = ofv - 1 + (llen == 0 ? 1 : 0);
                if (idx == 0) offset = ws->rep[0];
                else {
                    offset = idx < 3 ? ws->rep[idx] : ws->rep[0] - 1;
                    if (offset == 0) return -1;
                    if (idx > 1) ws->rep[2] = ws->rep[1];
                    ws->rep[1] = ws->rep[0];
                    ws->rep[0] = offset;
                }
            }
            if (lit_pos + llen > lit_len) return -1;
            if (o + llen + mlen > out_cap) return -1;
            for (uint32_t k = 0; k < llen; k++) out[o + k] = lits[lit_pos + k];
            o += llen;
            lit_pos += llen;
            if ((long long)offset > o) return -1;
            for (uint32_t k = 0; k < mlen; k++) out[o + k] = out[o + k - (long long)offset];
            o += mlen;
        }
        if (bb.left != 0) return -1;
    } else if (pos != len) {
        return -1;
    }
    uint32_t rest = lit_len - lit_pos;
    if (o + rest > out_cap) return -1;
    for (uint32_t k = 0; k < rest; k++) out[o + k] = lits[lit_pos + k];
    return o + rest;
}

// one Compressed block, fully serial (generic shapes). returns new o or -1
__device__ long long decode_block_serial(SerialWs* ws, uint8_t* out, long long o, long long out_cap, uint8_t* litbuf,
                                         const uint8_t* src, uint32_t len) {
    if (len < 1) return -1;
    uint32_t b0 = src[0];
    int type = b0 & 3, sf = (b0 >> 2) & 3;
    uint32_t pos, regen;
    const uint8_t* lits;
    if (type == 0 || type == 1) {
        if ((sf & 1) == 0) { regen = b0 >> 3; pos = 1; }
        else if (sf == 1) {
            if (len < 2) return -1;
            regen = (b0 >> 4) | ((uint32_t)src[1] << 4);
            pos = 2;
        } else {
            if (len < 3) return -1;
            regen = (b0 >> 4) | ((uint32_t)src[1] << 4) | ((uint32_t)src[2] << 12);
            pos = 3;
        }
        if ((long long)regen > out_cap) return -1;
        if (type == 0) {
            if (pos + regen > len) return -1;
            lits = src + pos;
            pos += regen;
        } else {
            if (pos + 1 > len) return -1;
            for (uint32_t k = 0; k < regen; k++) litbuf[k] = src[pos];
            lits = litbuf;
            pos += 1;
        }
    } else {
        uint32_t csize, hdr;
        int streams = 4;
        if (sf == 0 || sf == 1) {
            if (len < 3) return -1;
            uint32_t v = src[0] | ((uint32_t)src[1] << 8) | ((uint32_t)src[2] << 16);
            regen = (v >> 4) & 0x3ff;
            csize = (v >> 14) & 0x3ff;
            hdr = 3;
            if (sf == 0) streams = 1;
        } else if (sf == 2) {
            if (len < 4) return -1;
            uint32_t v = src[0] | ((uint32_t)src[1] << 8) | ((uint32_t)src[2] << 16) | ((uint32_t)src[3] << 24);
            regen = (v >> 4) & 0x3fff;
            csize = (v >> 18) & 0x3fff;
            hdr = 4;
        } else {
            if (len < 5) return -1;
            unsigned long long v = src[0] | ((unsigned long long)src[1] << 8) | ((unsigned long long)src[2] << 16) |
                                   ((unsigned long long)src[3] << 24) | ((unsigned long long)src[4] << 32);
            regen = (uint32_t)((v >> 4) & 0x3ffff);
            csize = (uint32_t)((v >> 22) & 0x3ffff);
            hdr = 5;
        }
        pos = hdr;
        if (pos + csize > len || (long long)regen > out_cap) return -1;
        const uint8_t* lp = src + pos;
        uint32_t lrem = csize;
        if (type == 2) {
            uint32_t used = huf_read_weights(ws->nbits, &ws->huf_log, lp, lrem, ws->ll /*scratch*/, ws->norm, ws->next);
            if (!used || !huf_fill_table_serial(ws->huf, ws->nbits, ws->huf_log)) return -1;
            ws->have_huf = 1;
            lp += used;
            lrem -= used;
        } else if (!ws->have_huf) {
            return -1;
        }
        if (streams == 1) {
            if (!huf_decode_stream_serial(ws->huf, ws->huf_log, litbuf, regen, lp, lrem)) return -1;
        } else {
            if (lrem < 6) return -1;
            uint32_t s1 = lp[0] | (lp[1] << 8), s2 = lp[2] | (lp[3] << 8), s3 = lp[4] | (lp[5] << 8);
            if (6 + s1 + s2 + s3 > lrem) return -1;
            uint32_t s4 = lrem - 6 - s1 - s2 - s3;
            uint32_t seg = (regen + 3) / 4;
            if (seg * 3 > regen) return -1;
            const uint8_t* q = lp + 6;
            if (!huf_decode_stream_serial(ws->huf, ws->huf_log, litbuf, seg, q, s1)) return -1;
            if (!huf_decode_stream_serial(ws->huf, ws->huf_log, litbuf + seg, seg, q + s1, s2)) return -1;
            if (!huf_decode_stream_serial(ws->huf, ws->huf_log, litbuf + 2 * seg, seg, q + s1 + s2, s3)) return -1;
            if (!huf_decode_stream_serial(ws->huf, ws->huf_log, litbuf + 3 * seg, regen - 3 * seg, q + s1 + s2 + s3, s4))
                return -1;
        }
        lits = litbuf;
        pos += csize;
    }
    if (pos >= len) return -1;
    return run_sequences(ws, out, o, out_cap, lits, regen, src + pos, len - pos);
}

struct FrameHdr {
    uint32_t hdr_size;
    bool has_fcs, checksum;
    unsigned long long fcs;
    unsigned long long block_max;  // Block_Maximum_Size = min(Window_Size, 128 KiB) (RFC 8878 3.1.1.1.2)
};

__host__ __device__ inline bool parse_frame_header(FrameHdr* h, const uint8_t* src, uint32_t len) {
    if (len < 5) return false;
    if (!(src[0] == 0x28 && src[1] == 0xB5 && src[2] == 0x2F && src[3] == 0xFD)) return false;
    uint32_t fhd = src[4];
    int fcs_flag = fhd >> 6;
    bool single = (fhd >> 5) & 1;
    if (fhd & 0x08) return false;
    h->checksum = (fhd >> 2) & 1;
    int did_flag = fhd & 3;
    uint32_t pos = 5;
    if (!single) pos += 1;
    const int did_sizes[4] = {0, 1, 2, 4};
    if (did_flag) {
        unsigned long long did = 0;
        if (pos + did_sizes[did_flag] > len) return false;
        for (int i = 0; i < did_sizes[did_flag]; i++) did |= (unsigned long long)src[pos + i] << (8 * i);
        if (did != 0) return false;  // dictionaries are never used on this path (gozstd.Decompress, dd == nil)
        pos += did_sizes[did_flag];
    }
    int fcs_size = fcs_flag == 0 ? (single ? 1 : 0) : (1 << fcs_flag);
    if (pos + fcs_size > len) return false;
    unsigned long long fcs = 0;
    for (int i = 0; i < fcs_size; i++) fcs |= (unsigned long long)src[pos + i] << (8 * i);
    if (fcs_size == 2) fcs += 256;
    pos += fcs_size;
    h->hdr_size = pos;
    h->has_fcs = fcs_size != 0;
    h->fcs = fcs;
    unsigned long long window = fcs;  // Single_Segment: Window_Size = Frame_Content_Size
    if (!single) {
        const uint32_t wd = src[5], wlog = 10 + (wd >> 3);
        window = (1ull << wlog) + ((1ull << wlog) >> 3) * (wd & 7);
    }
    h->block_max = window < (128u << 10) ? window : (128u << 10);
    return true;
}

// XXH64 (seed 0) of the decompressed content: RFC 8878 3.1.1 Content_Checksum = its low 32 bits.  Frames that carry one are
// rare on this path (gozstd and klauspost/compress write none) and always take the serial decoder, which verifies it.
__device__ __forceinline__ unsigned long long xxh_rotl(unsigned long long x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ unsigned long long xxh_read64(const uint8_t* p) {
    unsigned long long v = 0;
    for (int i = 0; i < 8; i++) v |= (unsigned long long)p[i] << (8 * i);
    return v;
}
__device__ unsigned long long xxh64(const uint8_t* p, unsigned long long len) {
    const unsigned long long P1 = 11400714785074694791ULL, P2 = 14029467366897019727ULL, P3 = 1609587929392839161ULL,
                             P4 = 9650029242287828579ULL, P5 = 2870177450012600261ULL;
    const uint8_t* const end = p + len;
    unsigned long long h;
    auto round = [&](unsigned long long acc, unsigned long long in) { return xxh_rotl(acc + in * P2, 31) * P1; };
    auto merge = [&](unsigned long long acc, unsigned long long v) { return (acc ^ round(0, v)) * P1 + P4; };
    if (len >= 32) {
        unsigned long long v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0ULL - P1;
        const uint8_t* const lim = end - 32;
        do {
            v1 = round(v1, xxh_read64(p));
            v2 = round(v2, xxh_read64(p + 8));
            v3 = round(v3, xxh_read64(p + 16));
            v4 = round(v4, xxh_read64(p + 24));
            p += 32;
        } while (p <= lim);
        h = xxh_rotl(v1, 1) + xxh_rotl(v2, 7) + xxh_rotl(v3, 12) + xxh_rotl(v4, 18);
        h = merge(h, v1);
        h = merge(h, v2);
        h = merge(h, v3);
        h = merge(h, v4);
    } else {
        h = P5;
    }
    h += len;
    while (p + 8 <= end) {
        h ^= round(0, xxh_read64(p));
        h = xxh_rotl(h, 27) * P1 + P4;
        p += 8;
    }
    if (p + 4 <= end) {
        unsigned long long w = (unsigned long long)p[0] | ((unsigned long long)p[1] << 8) | ((unsigned long long)p[2] << 16) | ((unsigned long long)p[3] << 24);
        h ^= w * P1;
        h = xxh_rotl(h, 23) * P2 + P3;
        p += 4;
    }
    while (p < end) {
        h ^= (unsigned long long)(*p) * P5;
        h = xxh_rotl(h, 11) * P1;
        p++;
    }
    h ^= h >> 33;
    h *= P2;
    h ^= h >> 29;
    h *= P3;
    h ^= h >> 32;
    return h;
}

// A frame with a Frame_Content_Size must fill out_cap exactly; one without it may produce up to out_cap bytes, and each of its
// Compressed blocks at most Block_Maximum_Size (what libzstd enforces).  Returns the bytes produced, or -1.
__device__ long long decode_frame_serial(SerialWs* ws, uint8_t* out, uint32_t out_cap, uint8_t* litbuf, const uint8_t* src,
                                         uint32_t len) {
    FrameHdr h;
    if (!parse_frame_header(&h, src, len)) return -1;
    uint32_t pos = h.hdr_size;
    long long o = 0;
    ws->have_ll = ws->have_ml = ws->have_of = ws->have_huf = 0;
    ws->rep[0] = 1;
    ws->rep[1] = 4;
    ws->rep[2] = 8;
    for (;;) {
        if (pos + 3 > len) return -1;
        uint32_t bh = src[pos] | ((uint32_t)src[pos + 1] << 8) | ((uint32_t)src[pos + 2] << 16);
        pos += 3;
        bool last = bh & 1;
        int type = (bh >> 1) & 3;
        uint32_t bsize = bh >> 3;
        if (type == 0) {
            if (pos + bsize > len || o + bsize > out_cap) return -1;
            for (uint32_t k = 0; k < bsize; k++) out[o + k] = src[pos + k];
            pos += bsize;
            o += bsize;
        } else if (type == 1) {
            if (pos + 1 > len || o + bsize > out_cap) return -1;
            for (uint32_t k = 0; k < bsize; k++) out[o + k] = src[pos];
            pos += 1;
            o += bsize;
        } else if (type == 2) {
            if (pos + bsize > len) return -1;
            const long long o0 = o;
            o = decode_block_serial(ws, out, o, out_cap, litbuf, src + pos, bsize);
            if (o < 0) return -1;
            if (!h.has_fcs && (unsigned long long)(o - o0) > h.block_max) return -1;
            pos += bsize;
        } else {
            return -1;
        }
        if (last) break;
    }
    if (h.has_fcs && (unsigned long long)o != (unsigned long long)out_cap) return -1;
    if (h.checksum) {
        if (pos + 4 > len) return -1;
        const uint32_t want = src[pos] | ((uint32_t)src[pos + 1] << 8) | ((uint32_t)src[pos + 2] << 16) | ((uint32_t)src[pos + 3] << 24);
        if ((uint32_t)xxh64(out, (unsigned long long)o) != want) return -1;  // corrupted content
        pos += 4;
    }
    return pos == len ? o : -1;
}

}  // namespace

// ------------------------------------------------------------------------------------------------ kernels
struct ZstdParams {
    const vmb_block_desc* descs;
    ColInfo* cols;         // (k_zstd_serial writes content_size of frames without Frame_Content_Size)
    const uint8_t* payload;
    uint8_t* scratch;      // decompressed varint bytes
    uint8_t* lit;          // literal arena (same offsets as scratch) or nullptr
    int32_t* status;       // per column
    const uint32_t* list;  // column indices to process
    uint32_t count;
    HufJob* jobs;          // one per list entry (prepare -> huf)
    void* ws;              // SerialWs array, one per resident thread of k_zstd_serial
    uint32_t ws_count;
    unsigned long long* seq_rec;  // decoded sequences (literal length | match length | offset), ColInfo::seq_rec_off
};

__device__ __forceinline__ void col_src(const ZstdParams& P, uint32_t col, const uint8_t** src, uint32_t* len) {
    const vmb_block_desc& d = P.descs[col >> 1];
    if (col & 1) { *src = P.payload + d.val_off; *len = d.val_size; }
    else { *src = P.payload + d.ts_off; *len = d.ts_size; }
}

// one thread per VMB_ZK_HUF column
__global__ void k_zstd_prepare(ZstdParams P) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.count) return;
    uint32_t col = P.list[i];
    HufJob* job = &P.jobs[i];
    job->col = col;
    job->nstreams = 0;  // = invalid until proven otherwise
    const uint8_t* src;
    uint32_t len;
    col_src(P, col, &src, &len);
    const ColInfo ci = P.cols[col];
    int rc = VMB_ERR_ZSTD;
    do {
        FrameHdr h;
        if (!parse_frame_header(&h, src, len)) break;
        uint32_t pos = h.hdr_size;
        if (pos + 3 > len) break;
        uint32_t bh = src[pos] | ((uint32_t)src[pos + 1] << 8) | ((uint32_t)src[pos + 2] << 16);
        pos += 3;
        uint32_t bsize = bh >> 3;
        if (!(bh & 1) || ((bh >> 1) & 3) != 2) break;  // host classified it as one last Compressed block
        if (pos + bsize + (h.checksum ? 4u : 0u) != len) break;
        const uint8_t* blk = src + pos;
        if (bsize < 3) break;
        uint32_t b0 = blk[0];
        int type = b0 & 3, sf = (b0 >> 2) & 3;
        if (type != 2) break;
        uint32_t regen, csize, hdr;
        int streams = 4;
        if (sf == 0 || sf == 1) {
            uint32_t v = blk[0] | ((uint32_t)blk[1] << 8) | ((uint32_t)blk[2] << 16);
            regen = (v >> 4) & 0x3ff;
            csize = (v >> 14) & 0x3ff;
            hdr = 3;
            if (sf == 0) streams = 1;
        } else if (sf == 2) {
            if (bsize < 4) break;
            uint32_t v = blk[0] | ((uint32_t)blk[1] << 8) | ((uint32_t)blk[2] << 16) | ((uint32_t)blk[3] << 24);
            regen = (v >> 4) & 0x3fff;
            csize = (v >> 18) & 0x3fff;
            hdr = 4;
        } else {
            if (bsize < 5) break;
            unsigned long long v = blk[0] | ((unsigned long long)blk[1] << 8) | ((unsigned long long)blk[2] << 16) |
                                   ((unsigned long long)blk[3] << 24) | ((unsigned long long)blk[4] << 32);
            regen = (uint32_t)((v >> 4) & 0x3ffff);
            csize = (uint32_t)((v >> 22) & 0x3ffff);
            hdr = 5;
        }
        if (hdr + csize >= bsize) break;  // a sequences section (>= 1 byte) must follow
        if (regen > ci.content_size) break;
        // Huffman tree description; scratch tables live on the thread's local stack (small: 64 + 256 + 256 entries)
        uint32_t ftab[64];
        short norm[256];
        unsigned short next[256];
        int tlog = 0;
        __align__(16) uint8_t nb_local[256];  // weights / code lengths are built on the thread's stack (L1), not in the job record
        uint32_t used = huf_read_weights(nb_local, &tlog, blk + hdr, csize, ftab, norm, next);
        if (!used) break;
#pragma unroll
        for (int k = 0; k < 32; k++) ((uint64_t*)job->nbits)[k] = ((const uint64_t*)nb_local)[k];  // (records are 8-byte aligned)
        uint32_t lrem = csize - used;
        const uint8_t* lp = blk + hdr + used;
        if (streams == 1) {
            job->stream_size[0] = lrem;
            job->stream_size[1] = job->stream_size[2] = job->stream_size[3] = 0;
            job->src_off = (uint64_t)(lp - P.payload);
        } else {
            if (lrem < 6) break;
            uint32_t s1 = lp[0] | (lp[1] << 8), s2 = lp[2] | (lp[3] << 8), s3 = lp[4] | (lp[5] << 8);
            if (6 + s1 + s2 + s3 > lrem) break;
            uint32_t seg = (regen + 3) / 4;
            if (seg * 3 > regen) break;
            job->stream_size[0] = s1;
            job->stream_size[1] = s2;
            job->stream_size[2] = s3;
            job->stream_size[3] = lrem - 6 - s1 - s2 - s3;
            job->src_off = (uint64_t)(lp + 6 - P.payload);
        }
        job->regen_size = regen;
        job->table_log = (uint8_t)tlog;
        uint32_t seq_off = hdr + csize;
        job->seq_off = (uint32_t)(blk - src) + seq_off;
        job->seq_size = bsize - seq_off;
        bool has_seq = blk[seq_off] != 0;
        if (!has_seq && (job->seq_size != 1 || regen != ci.content_size)) break;
        if (has_seq && !P.lit) break;
        job->dst_is_lit = has_seq ? 1 : 0;
        job->seq_big = 0;
        job->dst_off = ci.scratch_off;
        job->nstreams = (uint8_t)streams;
        rc = 0;
    } while (0);
    P.status[col] = rc;
}

// ---- lane-packed Huffman decode: 8 frames x 4 streams per warp
#define HUF_WARPS 2
#define HUF_FRAMES_PER_WARP 8
#define HUF_MAX_LOG 11
// Words of compressed input resident in shared memory per lane (power of two).  16 is enough: priming leaves 12..15 words
// and a head takes <= 6; a phase of 8 symbols takes <= 3 (4 only as the first after an empty head, with >= 12 resident), and a
// block is fetched only while the ring has room for it and the other pending one.  Enumerating those bounds, every phase finds
// >= 3 words once its block has landed and a tail (<= 6 words) finds >= 6, so a phase re-reads the candidate word after the
// block lands (the refill before may have read that slot before it was written).
#define HUF_RING 16
#define HUF_FRAME_BYTES (256 + 64) /* per frame: symbols in canonical order, then 10 thresholds (f32) + 12 index offsets (i16) */
#define HUF_WARP_TABLE_BYTES (HUF_FRAMES_PER_WARP * HUF_FRAME_BYTES)
// Output pieces (16 bytes) staged per lane before the warp writes them out together: HUF_STAGE per lane, slot (q, l) of a warp's
// HUF_STAGE x 32 at q * 32 + (l ^ q * (8 / HUF_STAGE)) -- a step's 32 stores and a write-out's 8-lane groups are conflict-free.
#ifndef HUF_STAGE
#define HUF_STAGE 8
#endif
#define HUF_STAGE_SLOT(q, l) ((q) * 32 + ((l) ^ ((q) * (8 / HUF_STAGE))))
#define HUF_FBIAS 0x4B000000u /* bits of 2^23: (HUF_FBIAS | v) is the float 2^23 + v for v < 2^23 */
#define HUF_CTAS_PER_SM 12u   /* grid cap (VMB_HUF_CTAS_PER_SM overrides it, for measurements) */

// Attribution builds (-DVMB_HUF_EXP=<mask>, scripts/exp_huf_bound.py; never the product): each bit takes one suspect off the
// symbol loop and keeps the rest of it live.  Their outputs are wrong; they are for timing only.  Without the macro every test
// below is `if (0)` and the kernel compiles to the product's SASS.
#ifndef VMB_HUF_EXP
#define VMB_HUF_EXP 0
#endif
#define HUF_EXP_STORE 1     /* no STG.128: the 16-byte pieces are XOR-folded per lane and written once per stream */
#define HUF_EXP_LOOKUP 2    /* the symbol is cut from the code bits: no perm / adj loads */
#define HUF_EXP_CONVERT 4   /* the code length from integer compares on packed thresholds: no I2F / F2I */
#define HUF_EXP_INPUT 8     /* the ring is refilled from registers: no input LDG in the loop */
#define HUF_EXP_L1 16       /* input loads bypass L1 (ld.global.nc.L1::no_allocate) */
#define HUF_EXP_PHASES 32   /* clock64() at lane 0 around table build, stream set-up + priming, head, body, tail */
#define HUF_EXP_CARVEOUT 64 /* shared-memory carveout just large enough for the grid cap: the rest of the SM's 256 KB is L1 */
#define HUF_EXP(bit) ((VMB_HUF_EXP & (bit)) != 0)
enum { HUF_PH_BUILD, HUF_PH_PRIME, HUF_PH_HEAD, HUF_PH_BODY, HUF_PH_TAIL, HUF_PH_N, HUF_PH_SYMS = HUF_PH_N, HUF_PH_SLOTS };
#if HUF_EXP(HUF_EXP_PHASES)
__device__ unsigned long long huf_phase_cyc[HUF_PH_SLOTS];
#define HUF_PH(k)                                                                              \
    do {                                                                                       \
        const long long ph_c = clock64();                                                      \
        ph[(k)] += (unsigned long long)(ph_c - ph_t);                                          \
        ph_t = ph_c;                                                                           \
    } while (0)
#else
#define HUF_PH(k) \
    do {          \
    } while (0)
#endif

// input block load of k_huf_decode (attribution builds may bypass L1)
__device__ __forceinline__ uint4 huf_ldg(const uint4* p) {
    if (HUF_EXP(HUF_EXP_L1)) {
        uint4 r;
        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                     : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                     : "l"(p));
        return r;
    }
    return *p;
}

__global__ void __launch_bounds__(HUF_WARPS * 32) k_huf_decode(ZstdParams P) {
    // Canonical decode without a 2^log-entry lookup table.  zstd lays a frame's codes out by descending length over the
    // 11-bit (left-aligned) code space, so the length of the next code is 1 + #{k : v < S_k} where S_k is the position
    // where the k-bit codes start: ten register-resident thresholds, ten compares, an add tree -- arithmetic only, no
    // shared-memory access on the loop-carried path (the bit buffer advances as soon as the length is known).  The symbol
    // is perm[(v >> (11 - L)) + adj[L]]: two small lookups off the critical path.  Per frame that is 320 bytes of shared
    // memory instead of a 2048-entry table, so the SM holds every warp the grid has instead of two per scheduler.
    extern __shared__ __align__(16) uint8_t s_smem[];
    const int lane = lane_id();
    const int warp = threadIdx.x >> 5;
    const uint32_t groups = (P.count + HUF_FRAMES_PER_WARP - 1) / HUF_FRAMES_PER_WARP;
    uint8_t* wtab = s_smem + (size_t)warp * HUF_WARP_TABLE_BYTES;
    // per-warp input rings behind the tables: HUF_RING words per lane, word-interleaved across lanes
    uint32_t* wring = (uint32_t*)(s_smem + (size_t)HUF_WARPS * HUF_WARP_TABLE_BYTES) + (size_t)warp * HUF_RING * 32;
#if HUF_EXP(HUF_EXP_PHASES)
    unsigned long long ph[HUF_PH_SLOTS] = {};
    long long ph_t = clock64();
#endif
    for (uint32_t g = blockIdx.x * HUF_WARPS + warp; g < groups; g += gridDim.x * HUF_WARPS) {
        // ---- build the 8 canonical tables cooperatively: symbols in (nbits desc, symbol asc) order
        for (int f = 0; f < HUF_FRAMES_PER_WARP; f++) {
            uint32_t ji = g * HUF_FRAMES_PER_WARP + f;
            if (ji >= P.count) break;
            const HufJob* job = &P.jobs[ji];
            if (job->nstreams == 0) continue;
            const int log = job->table_log;
            uint8_t* perm = wtab + f * HUF_FRAME_BYTES;
            float* thr = (float*)(perm + 256);   // thr[k-1] = 2^23 + S_k, k = 1..10
            short* adj = (short*)(perm + 256 + 40);  // adj[L], L = 1..11
            // each lane owns 8 symbols
            uint32_t nb[8];
            uint64_t packed = *(const uint64_t*)(job->nbits + lane * 8);
#pragma unroll
            for (int k = 0; k < 8; k++) nb[k] = (uint32_t)(packed >> (8 * k)) & 0xff;
            uint32_t start = 0;  // S_len in the 11-bit code space
            uint32_t rank = 0;   // symbols with longer codes
            if (lane < 10) thr[lane] = __uint_as_float(HUF_FBIAS);  // k >= log: no k-bit codes above v, never counted
            __syncwarp();
            for (int len = log; len >= 1; len--) {
                uint32_t mine = 0;
#pragma unroll
                for (int k = 0; k < 8; k++) mine += (nb[k] == (uint32_t)len);
                uint32_t inc = mine;
#pragma unroll
                for (int off = 1; off < 32; off <<= 1) {
                    uint32_t t = __shfl_up_sync(VMB_FULL, inc, off);
                    if (lane >= off) inc += t;
                }
                uint32_t tot = __shfl_sync(VMB_FULL, inc, 31);
                if (lane == 0) {
                    if (len <= 10) thr[len - 1] = __uint_as_float(HUF_FBIAS | start);
                    adj[len] = (short)((int)rank - (int)(start >> (HUF_MAX_LOG - len)));
                }
                uint32_t r = rank + inc - mine;
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    if (nb[k] == (uint32_t)len) perm[r++ & 255u] = (uint8_t)(lane * 8 + k);
                }
                rank += tot;
                start += tot << (HUF_MAX_LOG - len);
            }
        }
        __syncwarp();
        HUF_PH(HUF_PH_BUILD);
        // ---- every lane decodes one stream
        {
            const int f = lane >> 2, s = lane & 3;
            uint32_t ji = g * HUF_FRAMES_PER_WARP + f;
            bool active = ji < P.count;
            const HufJob* job = active ? &P.jobs[ji] : nullptr;
            if (active && (job->nstreams == 0 || s >= job->nstreams)) active = false;
            bool ok = true;
            // Decoder state, declared here because the body runs as a warp-uniform loop (its stores are cooperative): a lane
            // that decodes no stream (live == false) runs the loop's votes and stores but none of its decoding.
            bool live = false;
            const uint8_t* perm = wtab + f * HUF_FRAME_BYTES;
            const short* adj = (const short*)(perm + 256 + 40);
            __half2 th2[5];
            uint32_t th_i[5] = {0, 0, 0, 0, 0};
            uint32_t count = 0, total_bits = 0, wr = 0, rd = 0, cand = 0, i = 0;
            uint8_t* dst = nullptr;
            const uint4* blk = nullptr;
            const uint4* blk_min = nullptr;
            uint32_t* ring = wring + lane;  // slot i -> ring[(i & (HUF_RING - 1)) * 32]
            uint64_t buf = 0;               // bit buffer, next bit at the top
            int cnt = 0, cnt_init = 0;      // valid bits in buf; payload bits consumed so far = cnt_init + 32 * rd - cnt
            uint4 pendA = make_uint4(0, 0, 0, 0), pendB = make_uint4(0, 0, 0, 0);
            bool hasA = false, hasB = false;
            uint4 xo = make_uint4(0, 0, 0, 0);  // HUF_EXP_STORE
            if (active) {
                // the ten thresholds S_k (0..2048, exact in fp16) as five half2 registers: two compares per instruction
                {
                    const float* tf = (const float*)(perm + 256);
#pragma unroll
                    for (int j = 0; j < 5; j++) {
                        const uint32_t a = __float_as_uint(tf[2 * j]) & 0x7fffffu, b = __float_as_uint(tf[2 * j + 1]) & 0x7fffffu;
                        th2[j] = __halves2half2(__ushort2half_rn((unsigned short)a), __ushort2half_rn((unsigned short)b));
                    }
                }
                // integer variant: 0x1000 + S_k in each 16-bit half; (th_i[j] - (v + 1) * 0x10001) has bit 12 (28) set iff v < S_k
                if (HUF_EXP(HUF_EXP_CONVERT)) {
                    const float* tf = (const float*)(perm + 256);
#pragma unroll
                    for (int j = 0; j < 5; j++)
                        th_i[j] = ((0x1000u + (__float_as_uint(tf[2 * j + 1]) & 0x7fffffu)) << 16) |
                                  (0x1000u + (__float_as_uint(tf[2 * j]) & 0x7fffffu));
                }
                uint32_t regen = job->regen_size;
                uint32_t seg = job->nstreams == 1 ? regen : (regen + 3) / 4;
                count = job->nstreams == 1 ? regen : (s < 3 ? seg : regen - 3 * seg);
                uint64_t soff = job->src_off;
                for (int k = 0; k < s; k++) soff += job->stream_size[k];
                uint32_t slen = job->stream_size[s];
                dst = (job->dst_is_lit ? P.lit : P.scratch) + job->dst_off + (size_t)s * seg;
                const uint8_t* base = P.payload + soff;
                uint32_t last = slen ? base[slen - 1] : 0;
                if (count == 0) {
                    // an empty last segment: nothing to write (the stream holds just the final-bit marker)
                } else if (slen == 0 || last == 0) {
                    ok = false;
                } else {
                    live = true;
                    // Backward bitstream, lane-private, with every memory access at a warp-uniform program point:
                    //   * the stream is pulled in as aligned 16-byte blocks (LDG.128) that land in registers and are moved
                    //     into the lane's shared-memory ring TWO phases (16 symbols) later -- the HBM round trip is covered
                    //     by decoding, and no lane ever makes the other 31 wait on its own load;
                    //   * 32-bit words are popped from the ring into an MSB-aligned 64-bit bit buffer; the candidate word is
                    //     re-read (LDS) at every refill check by all lanes, so that read is uniform too.
                    // The ring is word-interleaved across lanes (word w of lane l at [w*32 + l]): conflict-free.
                    total_bits = (slen - 1) * 8 + (uint32_t)hb32(last);
                    const uint8_t* endp = base + slen - 1;                                 // byte holding the final-bit marker
                    blk = (const uint4*)((uintptr_t)endp & ~(uintptr_t)15);   // aligned block that holds it
                    blk_min = (const uint4*)(((uintptr_t)base & ~(uintptr_t)15) - 32);  // never read below this
                    {
                        uint4 q = *blk;
                        uint64_t qlo = ((uint64_t)q.y << 32) | q.x, qhi = ((uint64_t)q.w << 32) | q.z;
                        uint32_t nbytes = (uint32_t)((uintptr_t)endp & 15) + 1;  // valid bytes of this block: 1..16
                        uint32_t drop = (16 - nbytes) * 8;                       // bits above the marker byte (next stream's data)
                        if (drop >= 64) { qhi = qlo; qlo = 0; drop -= 64; }
                        if (drop) { qhi = (qhi << drop) | (qlo >> (64 - drop)); qlo <<= drop; }
                        uint32_t r = nbytes & 3;  // the odd 1..3 (or 4) top bytes go straight into the bit buffer: whole words remain
                        if (r == 0) r = 4;
                        buf = qhi & ~(~0ull >> (8 * r));
                        cnt = (int)(8 * r);
                        qhi = (qhi << (8 * r)) | (r == 8 ? 0 : (qlo >> (64 - 8 * r)));
                        qlo <<= (8 * r);
                        uint32_t nw = (nbytes - r) >> 2;
                        for (uint32_t k = 0; k < nw; k++) {
                            ring[(wr & (HUF_RING - 1)) * 32] = (uint32_t)(qhi >> 32);
                            wr++;
                            qhi = (qhi << 32) | (qlo >> 32);
                            qlo <<= 32;
                        }
                        int skip = 8 - hb32(last);  // zero padding + the final-bit marker
                        buf <<= skip;
                        cnt -= skip;
                        // prime the ring: 3 more blocks (reads below the stream start return bytes that are never consumed)
#pragma unroll
                        for (int k = 0; k < 3; k++) {
                            if (blk > blk_min) blk--;
                            uint4 b = huf_ldg(blk);
                            ring[((wr + 0) & (HUF_RING - 1)) * 32] = b.w;
                            ring[((wr + 1) & (HUF_RING - 1)) * 32] = b.z;
                            ring[((wr + 2) & (HUF_RING - 1)) * 32] = b.y;
                            ring[((wr + 3) & (HUF_RING - 1)) * 32] = b.x;
                            wr += 4;
                        }
                    }
                    cnt_init = cnt;
                    cand = ring[(rd & (HUF_RING - 1)) * 32];
#define HUF_PHASE(pend, has)                                                               \
    do {                                                                                   \
        if (has) { /* block fetched two phases ago: now in registers for sure */           \
            ring[((wr + 0) & (HUF_RING - 1)) * 32] = pend.w;                               \
            ring[((wr + 1) & (HUF_RING - 1)) * 32] = pend.z;                               \
            ring[((wr + 2) & (HUF_RING - 1)) * 32] = pend.y;                               \
            ring[((wr + 3) & (HUF_RING - 1)) * 32] = pend.x;                               \
            wr += 4;                                                                       \
        }                                                                                  \
        /* room for this block even when the other pending block lands first? */           \
        has = (wr - rd) + 8u <= (uint32_t)HUF_RING;                                        \
        if (has) {                                                                         \
            if (blk > blk_min) blk--;                                                      \
            if (HUF_EXP(HUF_EXP_INPUT)) pend = make_uint4(rd, wr, (uint32_t)cnt, (uint32_t)(uintptr_t)blk); \
            else pend = huf_ldg(blk);                                                      \
        }                                                                                  \
        cand = ring[(rd & (HUF_RING - 1)) * 32]; /* the slot may have been written just now */ \
    } while (0)
#define HUF_REFILL()                                                                       \
    do {                                                                                   \
        if (cnt <= 32) {                                                                   \
            buf |= (uint64_t)cand << (32 - cnt);                                           \
            cnt += 32;                                                                     \
            rd++;                                                                          \
        }                                                                                  \
        cand = ring[(rd & (HUF_RING - 1)) * 32];                                           \
    } while (0)
#define HUF_LT(k) __hlt2(vv_, th2[k]) /* (1.0, 0.0) per half */
#define HUF_LTI(j) ((th_i[j] - v1_) & 0x10001000u)
#define HUF_SYM(outv, shift)                                                               \
    do {                                                                                   \
        const uint32_t v_ = (uint32_t)(buf >> 53);                                         \
        uint32_t nb_;                                                                      \
        if (HUF_EXP(HUF_EXP_CONVERT)) {                                                    \
            const uint32_t v1_ = (v_ + 1u) * 0x10001u;                                     \
            const uint32_t a_ = HUF_LTI(0) + HUF_LTI(1) + HUF_LTI(2) + HUF_LTI(3) + HUF_LTI(4); \
            nb_ = 1u + ((a_ * 0x10001u) >> 28);                                            \
        } else {                                                                           \
            const __half2 vv_ = __half2half2(__ushort2half_rn((unsigned short)v_));        \
            /* code length = 1 + #{k : v < S_k}; the count (<= 10) is exact in fp16 */      \
            const __half2 c_ = __hadd2(__hadd2(__hadd2(HUF_LT(0), HUF_LT(1)), __hadd2(HUF_LT(2), HUF_LT(3))), HUF_LT(4)); \
            nb_ = 1u + (uint32_t)__half2ushort_rz(__hadd(__low2half(c_), __high2half(c_))); \
        }                                                                                  \
        buf <<= nb_;                                                                       \
        cnt -= (int)nb_;                                                                   \
        const uint32_t sym_ = HUF_EXP(HUF_EXP_LOOKUP) ? ((v_ >> (HUF_MAX_LOG - nb_)) & 255u)  \
            : perm[((v_ >> (HUF_MAX_LOG - nb_)) + (uint32_t)(int)adj[nb_]) & 255u];         \
        outv |= sym_ << (shift);                                                           \
    } while (0)
                    HUF_PH(HUF_PH_PRIME);
                    // head: single bytes until dst is 16-byte aligned (<= 15 symbols <= 6 words: covered by the primed ring)
                    while (i < count && (((uintptr_t)(dst + i)) & 15)) {
                        HUF_REFILL();
                        uint32_t o = 0;
                        HUF_SYM(o, 0);
                        dst[i++] = (uint8_t)o;
                    }
                    HUF_PH(HUF_PH_HEAD);
                }
            }
            // body: 16 symbols per aligned 16-byte piece = two phases of 8 symbols (<= 88 bits <= 3 words each).  A lane's
            // pieces are staged in shared memory; every HUF_STAGE steps the warp writes them out, each store instruction
            // covering 32 / HUF_STAGE streams with HUF_STAGE consecutive pieces each, instead of 32 streams with one piece.
            {
                uint4* stage = (uint4*)(s_smem + (size_t)HUF_WARPS * (HUF_WARP_TABLE_BYTES + HUF_RING * 32 * sizeof(uint32_t))) +
                               warp * HUF_STAGE * 32;
                uint32_t k = 0, bi = i;  // steps of this batch; the lane's output index at the batch's start
                for (;;) {
                    const bool more = live && i + 16 <= count;
                    if (more) {
                        uint32_t o[4];
                        HUF_PHASE(pendA, hasA);
#pragma unroll
                        for (int q = 0; q < 2; q++) {
                            o[q] = 0;
                            HUF_REFILL();
                            HUF_SYM(o[q], 0);
                            HUF_SYM(o[q], 8);
                            HUF_REFILL();
                            HUF_SYM(o[q], 16);
                            HUF_SYM(o[q], 24);
                        }
                        HUF_PHASE(pendB, hasB);
#pragma unroll
                        for (int q = 2; q < 4; q++) {
                            o[q] = 0;
                            HUF_REFILL();
                            HUF_SYM(o[q], 0);
                            HUF_SYM(o[q], 8);
                            HUF_REFILL();
                            HUF_SYM(o[q], 16);
                            HUF_SYM(o[q], 24);
                        }
                        if (HUF_EXP(HUF_EXP_STORE)) {
                            xo.x ^= o[0]; xo.y ^= o[1]; xo.z ^= o[2]; xo.w ^= o[3];
                        } else {
                            stage[HUF_STAGE_SLOT(k, lane)] = make_uint4(o[0], o[1], o[2], o[3]);
                        }
                        i += 16;
                    }
                    const bool any = __any_sync(VMB_FULL, more);
                    if (++k == HUF_STAGE || !any) {  // write the batch: piece q of stream l goes to dst_l + bi_l + 16 q
                        __syncwarp();
                        const uint32_t n_l = (i - bi) >> 4;
                        const uintptr_t p_l = (uintptr_t)(dst + bi);
#pragma unroll
                        for (int j = 0; j < HUF_STAGE; j++) {
                            const int l = (j * 32 + lane) / HUF_STAGE, q = (j * 32 + lane) % HUF_STAGE;
                            const uint32_t n = __shfl_sync(VMB_FULL, n_l, l);
                            const uintptr_t pp = (uintptr_t)__shfl_sync(VMB_FULL, (unsigned long long)p_l, l);
                            if ((uint32_t)q < n && !HUF_EXP(HUF_EXP_STORE)) *(uint4*)(pp + 16 * q) = stage[HUF_STAGE_SLOT(q, l)];
                        }
                        __syncwarp();
                        k = 0;
                        bi = i;
                    }
                    if (!any) break;
                }
            }
            if (HUF_EXP(HUF_EXP_STORE) && live && i >= 16) *(uint4*)(dst + i - 16) = xo;
            if (live) {
                {
                    HUF_PH(HUF_PH_BODY);
                    // tail (<= 15 symbols <= 6 words): what is already in the ring plus the pending blocks is enough
                    if (i < count) {
                        HUF_PHASE(pendA, hasA);
                        HUF_PHASE(pendB, hasB);
                        hasA = hasB = false;
                    }
                    for (; i < count; i++) {
                        HUF_REFILL();
                        uint32_t o = 0;
                        HUF_SYM(o, 0);
                        dst[i] = (uint8_t)o;
                    }
                    HUF_PH(HUF_PH_TAIL);
#if HUF_EXP(HUF_EXP_PHASES)
                    ph[HUF_PH_SYMS] += count;
#endif
#undef HUF_PHASE
#undef HUF_REFILL
#undef HUF_SYM
#undef HUF_LT
#undef HUF_LTI
                    ok = (long long)cnt_init + 32ll * (long long)rd - (long long)cnt == (long long)total_bits;
                }
            }
            // a frame fails if any of its streams failed
            // variants that write wrong literals fail every frame, so that no later kernel reads them
            if (HUF_EXP(HUF_EXP_STORE | HUF_EXP_LOOKUP | HUF_EXP_INPUT)) ok = false;
            uint32_t bad = __ballot_sync(VMB_FULL, active && !ok);
            if (HUF_EXP(HUF_EXP_STORE | HUF_EXP_LOOKUP | HUF_EXP_INPUT) && ji < P.count && s == 0) bad |= 1u << (f * 4);
            if (ji < P.count && s == 0 && ((bad >> (f * 4)) & 0xf)) P.status[P.jobs[ji].col] = VMB_ERR_ZSTD;
        }
        __syncwarp();
    }
#if HUF_EXP(HUF_EXP_PHASES)
    if (lane == 0)  // lane 0's cycles; the wait for the warp's slower lanes lands in the next table build
        for (int k = 0; k < HUF_PH_SLOTS; k++) atomicAdd(&huf_phase_cyc[k], ph[k]);
#endif
}

// ---- sequences of prepared frames, in two kernels.
// k_zstd_seq_decode: the FSE bitstream of a frame is inherently serial, and its latency (table lookup -> extra bits -> next
//   state) is what bounds the step; so it runs apart from the copies, SEQ_G lanes per frame (redundantly: same registers,
//   broadcast loads, the three decoding tables in shared memory), 32 / SEQ_G frames per warp, and leaves one 8-byte record
//   per sequence: literal length | match length | offset.
// k_zstd_seq_exec: one warp per frame turns the records into bytes -- positions by warp scans, every literal run
//   independent of the rest, the matches in order (32 lanes per copy; out[o+k] = out[o-offset + k % offset] when a match
//   overlaps itself).
#define SEQ_G 4
#define SEQ_FPW (32 / SEQ_G)
#define SEQ_WARPS 1
#define SEQ_REC(ll, ml, of) (((unsigned long long)(ll) << 44) | ((unsigned long long)(ml) << 24) | (unsigned long long)(of))
#define SEQ_REC_LL(r) ((uint32_t)((r) >> 44))
#define SEQ_REC_ML(r) ((uint32_t)((r) >> 24) & 0xfffffu)
#define SEQ_REC_OF(r) ((uint32_t)(r) & 0xffffffu)
// decoding tables of one frame, 3 bytes per state (16-bit nbits|base + 8-bit symbol) so that more frames fit an SM.  Two
// capacities: libzstd picks accuracy log 8 for the ~1300 sequences of an 8192-row column (measured; the format allows 9 / 8 / 9),
// so the kernel runs first with 256-state tables (2304 B per frame: twelve warps of eight frames per SM) and frames whose
// tables are larger are flagged (HufJob::seq_big) for a second launch with full-size tables.
template <int LLC, int MLC, int OFC>
struct SeqTablesT {
    unsigned short ll_nb[LLC], ml_nb[MLC], of_nb[OFC];  // (nbits << 12) | base, base < 512
    uint8_t ll_sym[LLC], ml_sym[MLC], of_sym[OFC];
};

// fse_build for the packed layout (same spreading, RFC 8878 4.1.1)
__device__ bool fse_build_packed(uint8_t* sym, unsigned short* nbbase, const short* norm, int nsym, int log, unsigned short* next) {
    const int size = 1 << log;
    int high = size - 1;
    for (int s = 0; s < nsym; s++) {
        if (norm[s] == -1) {
            sym[high--] = (uint8_t)s;
            next[s] = 1;
        } else {
            next[s] = (unsigned short)norm[s];
        }
    }
    const int step = (size >> 1) + (size >> 3) + 3, mask = size - 1;
    int pos = 0;
    for (int s = 0; s < nsym; s++) {
        for (int i = 0; i < norm[s]; i++) {
            sym[pos] = (uint8_t)s;
            do {
                pos = (pos + step) & mask;
            } while (pos > high);
        }
    }
    if (pos != 0) return false;
    for (int i = 0; i < size; i++) {
        const uint32_t s = sym[i];
        const uint32_t ns = next[s]++;
        const int nb = log - hb32(ns);
        nbbase[i] = (unsigned short)(((uint32_t)nb << 12) | ((ns << nb) - (uint32_t)size));
    }
    return true;
}

// Symbol_Compression_Mode of one sequence table (RFC 8878 3.1.1.3.2.1) -> packed table; returns bytes consumed.
// Repeat mode is invalid here: a prepared frame holds a single block.  *big: the table has more than 2^cap_log states
// (nothing is built; the frame belongs to the launch with full-size tables).
// The three predefined distributions (RFC 8878 3.1.1.3.2.2) as packed decoding tables, built once per device
// (k_zstd_seq_defaults): frames that use Predefined_Mode copy 160 states instead of running the builder.
#define SEQ_DEF_LL 0
#define SEQ_DEF_OF 64
#define SEQ_DEF_ML 96
__device__ unsigned short g_seq_def_nb[160];
__device__ uint8_t g_seq_def_sym[160];
__global__ void k_zstd_seq_defaults() {
    if (blockIdx.x || threadIdx.x) return;
    short norm[64];
    unsigned short next[64];
    for (int i = 0; i < 36; i++) norm[i] = c_ll_default[i];
    fse_build_packed(g_seq_def_sym + SEQ_DEF_LL, g_seq_def_nb + SEQ_DEF_LL, norm, 36, 6, next);
    for (int i = 0; i < 29; i++) norm[i] = c_of_default[i];
    fse_build_packed(g_seq_def_sym + SEQ_DEF_OF, g_seq_def_nb + SEQ_DEF_OF, norm, 29, 5, next);
    for (int i = 0; i < 53; i++) norm[i] = c_ml_default[i];
    fse_build_packed(g_seq_def_sym + SEQ_DEF_ML, g_seq_def_nb + SEQ_DEF_ML, norm, 53, 6, next);
}

struct SeqWs {  // scratch of the table builder (global memory, one per frame group of the grid)
    short norm[256];
    unsigned short next[256];
};
__device__ uint32_t read_seq_table_packed(uint8_t* sym, unsigned short* nbbase, int* tlog, int mode, int def_off, int deflog, int max_sym,
                                          int max_log, int cap_log, const uint8_t* src, uint32_t len, SeqWs* ws, bool* ok, bool* big) {
    *ok = true;
    if (mode == 0) {
        for (int i = 0; i < (1 << deflog); i++) {
            sym[i] = g_seq_def_sym[def_off + i];
            nbbase[i] = g_seq_def_nb[def_off + i];
        }
        *tlog = deflog;
        return 0;
    }
    if (mode == 1) {
        if (len < 1 || src[0] > max_sym) {
            *ok = false;
            return 0;
        }
        sym[0] = src[0];
        nbbase[0] = 0;
        *tlog = 0;
        return 1;
    }
    if (mode == 2) {
        int nsym, log;
        const uint32_t used = fse_read_ncount(ws->norm, &nsym, &log, max_sym, max_log, src, len);
        if (!used) {
            *ok = false;
            return 0;
        }
        if (log > cap_log) {
            *big = true;
            return used;
        }
        if (!fse_build_packed(sym, nbbase, ws->norm, nsym, log, ws->next)) {
            *ok = false;
            return 0;
        }
        *tlog = log;
        return used;
    }
    *ok = false;
    return 0;
}

// Backward bitstream of the sequences section for the decode loop: MSB-aligned 64-bit window in two registers (every field is
// cut with funnel shifts, no 64-bit variable shifts), fed by ALIGNED 32-bit words loaded one refill ahead (the load's latency
// is covered by the sequences decoded in between).  Words in front of the stream start hold other bytes of the frame: they can
// only be consumed by a stream that over-reads, which `left` < 0 reports.
struct SeqBits {
    const uint32_t* wbase;  // aligned word that holds the byte 4 in front of the stream start: never read below it
    uint32_t widx;          // word index (from wbase) that the NEXT prefetch reads
    uint32_t w_hi, w_lo;    // aligned words around the next 4 stream bytes
    uint32_t w_next;        // the word below them, loaded one refill ahead (may still be in flight: touched by the next refill only)
    uint32_t sh;            // (address of the stream bytes & 3) * 8
    uint32_t hi, lo;        // the window, next bit at the top of hi
    int cnt;                // bits in the window
    int left;               // payload bits not yet consumed; < 0 => over-read

    __device__ __forceinline__ void refill() {  // requires cnt <= 32
        const uint32_t w = __funnelshift_r(w_lo, w_hi, sh);
        hi |= __funnelshift_rc(w, 0u, (uint32_t)cnt);
        lo = __funnelshift_lc(0u, w, 32u - (uint32_t)cnt);
        cnt += 32;
        w_hi = w_lo;
        w_lo = w_next;
        w_next = wbase[widx];
        // The eight frames of a warp refill at different steps, so nearly every step of the warp carries this load for somebody;
        // the stream is walked backwards (no hardware prefetch), and a sector that misses L1 would stall all eight: ask for the
        // sector 96 bytes further down now (no destination register, nothing waits)
        asm volatile("prefetch.global.L1 [%0];" ::"l"(wbase + (widx > 24u ? widx - 24u : 0u)));
        widx -= (widx != 0u);
    }
    __device__ bool init(const uint8_t* src, uint32_t len) {
        if (len == 0) return false;
        const uint32_t last = src[len - 1];
        if (last == 0) return false;
        const uintptr_t a = (uintptr_t)(src + len) - 4;  // the first four bytes to pull (the stream's last four)
        sh = (uint32_t)(a & 3u) * 8u;
        const uint32_t* w0 = (const uint32_t*)(a & ~(uintptr_t)3);
        wbase = (const uint32_t*)(((uintptr_t)src - 4) & ~(uintptr_t)3);
        w_hi = sh ? w0[1] : 0u;
        w_lo = w0[0];
        const uint32_t i0 = (uint32_t)(w0 - wbase);  // >= 0: w0 holds byte src + len - 4 >= src - 3
        widx = i0 ? i0 - 1u : 0u;
        w_next = wbase[widx];
        widx -= (widx != 0u);
        hi = lo = 0;
        cnt = 0;
        left = (int)((len - 1) * 8u) + hb32(last);
        refill();
        if (len < 4) {  // bytes in front of the section ended up in the low end of the first word: zero them like padding
            const uint32_t keep = 8u * len;
            hi &= ~(0xffffffffu >> keep);
        }
        const uint32_t skip = 8u - (uint32_t)hb32(last);  // zero padding + the final-bit marker
        hi = __funnelshift_lc(lo, hi, skip);
        lo = __funnelshift_lc(0u, lo, skip);
        cnt -= (int)skip;
        return true;
    }
    __device__ __forceinline__ uint32_t take(uint32_t nb) {  // 0 <= nb <= 32, nb <= cnt
        const uint32_t x = __funnelshift_rc(hi, 0u, 32u - nb);
        hi = __funnelshift_lc(lo, hi, nb);
        lo = __funnelshift_lc(0u, lo, nb);
        return x;
    }
    __device__ __forceinline__ uint32_t read_slow(uint32_t nb) {  // any window state
        if (cnt < (int)nb) refill();
        const uint32_t x = take(nb);
        cnt -= (int)nb;
        left -= (int)nb;
        return x;
    }
};

template <bool BIG>
__global__ void __launch_bounds__(SEQ_WARPS * 32) k_zstd_seq_decode(ZstdParams P) {
    typedef SeqTablesT<BIG ? 512 : 256, BIG ? 512 : 256, 256> Tables;
    constexpr int LL_CAP = BIG ? 9 : 8, ML_CAP = BIG ? 9 : 8, OF_CAP = 8;
    __shared__ Tables s_tab[SEQ_WARPS * SEQ_FPW];
    // code -> (base value, extra bits): copies in shared memory, because the groups of a warp index them with different codes
    // (constant memory would serve one address per pass)
    __shared__ uint32_t s_ll_base[36], s_ml_base[53];
    __shared__ uint8_t s_ll_bits[36], s_ml_bits[53];
    for (uint32_t t = threadIdx.x; t < 53; t += blockDim.x) {
        if (t < 36) { s_ll_base[t] = c_ll_base[t]; s_ll_bits[t] = c_ll_bits[t]; }
        s_ml_base[t] = c_ml_base[t];
        s_ml_bits[t] = c_ml_bits[t];
    }
    __syncthreads();
    const int lane = lane_id(), warp = threadIdx.x >> 5;
    const int grp = lane / SEQ_G, sub = lane % SEQ_G;
    const uint32_t gslot = (blockIdx.x * SEQ_WARPS + warp) * SEQ_FPW + grp;  // this group's workspace slot
    const uint32_t nslots = gridDim.x * SEQ_WARPS * SEQ_FPW;
    SeqWs* ws = (SeqWs*)P.ws + gslot;  // scratch of the table builder (the launch guarantees the slot exists)
    Tables* T = &s_tab[warp * SEQ_FPW + grp];
    for (uint32_t i0 = (blockIdx.x * SEQ_WARPS + warp) * SEQ_FPW; i0 < P.count; i0 += nslots) {
        const uint32_t i = i0 + grp;
        // ---- per group: locate the frame, read the section header, expand the table descriptions (group leader)
        bool act = i < P.count;
        HufJob* job = act ? &P.jobs[i] : nullptr;
        if (act && (job->nstreams == 0 || !job->dst_is_lit)) act = false;
        if (act && (job->seq_big != 0) != BIG) act = false;  // the other launch's frame
        uint32_t col = 0;
        if (act) {
            col = job->col;
            if (P.status[col]) act = false;
        }
        bool ok = true;
        const uint8_t* src = nullptr;
        uint32_t len = 0, lit_len = 0, nseq = 0, pos = 0, out_cap = 0;
        unsigned long long* rec = nullptr;
        int ll_log = 0, of_log = 0, ml_log = 0;
        bool big = false;
        if (act) {
            const ColInfo ci = P.cols[col];
            const uint8_t* fsrc;
            uint32_t flen;
            col_src(P, col, &fsrc, &flen);
            src = fsrc + job->seq_off;
            len = job->seq_size;
            out_cap = ci.content_size;  // (<= 163840: everything below fits 32 bits)
            lit_len = job->regen_size;
            rec = P.seq_rec + ci.seq_rec_off;
            if (len < 1) ok = false;
            else {
                const uint32_t b0 = src[0];
                if (b0 < 128) { nseq = b0; pos = 1; }
                else if (b0 < 255) {
                    if (len < 2) ok = false;
                    else { nseq = ((b0 - 128) << 8) + src[1]; pos = 2; }
                } else {
                    if (len < 3) ok = false;
                    else { nseq = (uint32_t)src[1] + ((uint32_t)src[2] << 8) + 0x7F00u; pos = 3; }
                }
            }
            if (ok && nseq != ci.nseq) ok = false;  // the record arena was sized by the host from the same byte(s)
            if (ok && (nseq == 0 || pos >= len)) ok = false;
            if (ok) {
                const uint32_t modes = src[pos++];
                if (modes & 3) ok = false;
                if (ok && sub == 0) {
                    bool tok;
                    pos += read_seq_table_packed(T->ll_sym, T->ll_nb, &ll_log, (modes >> 6) & 3, SEQ_DEF_LL, 6, 35, 9, LL_CAP,
                                                 src + pos, len - pos, ws, &tok, &big);
                    if (tok)
                        pos += read_seq_table_packed(T->of_sym, T->of_nb, &of_log, (modes >> 4) & 3, SEQ_DEF_OF, 5, 31, 8, OF_CAP,
                                                     src + pos, len - pos, ws, &tok, &big);
                    if (tok)
                        pos += read_seq_table_packed(T->ml_sym, T->ml_nb, &ml_log, (modes >> 2) & 3, SEQ_DEF_ML, 6, 52, 9, ML_CAP,
                                                     src + pos, len - pos, ws, &tok, &big);
                    if (!tok || pos >= len) ok = false;  // (leader only; the group learns it from the broadcast below)
                    if (tok && big) job->seq_big = 1;    // (BIG launch: cannot happen, its tables hold every legal log)
                }
            }
        }
        {   // broadcast the leader's view inside each group (uniform code: all 32 lanes execute the shuffles)
            const int leader = grp * SEQ_G;
            ok = __shfl_sync(VMB_FULL, (int)ok, leader) != 0;
            big = __shfl_sync(VMB_FULL, (int)big, leader) != 0;
            pos = __shfl_sync(VMB_FULL, pos, leader);
            ll_log = __shfl_sync(VMB_FULL, ll_log, leader);
            of_log = __shfl_sync(VMB_FULL, of_log, leader);
            ml_log = __shfl_sync(VMB_FULL, ml_log, leader);
        }
        if (big) act = false;  // decoded by the launch with full-size tables
        __syncwarp();
        SeqBits bb;
        bb.wbase = (const uint32_t*)P.payload;
        bb.widx = 0;
        bb.w_hi = bb.w_lo = bb.w_next = bb.sh = bb.hi = bb.lo = 0;
        bb.cnt = 64;  // (idle groups never refill)
        bb.left = 0;
        uint32_t sll = 0, sof = 0, sml = 0;
        if (act && ok) {
            if (!bb.init(src + pos, len - pos)) ok = false;
            else {
                sll = bb.read_slow((uint32_t)ll_log);
                sof = bb.read_slow((uint32_t)of_log);
                sml = bb.read_slow((uint32_t)ml_log);
            }
        }
        uint32_t rep0 = 1, rep1 = 4, rep2 = 8;  // one block per prepared frame: the repeat offsets start fresh
        uint32_t o = 0, lit_pos = 0;
        uint32_t bad = 0, last_state_bits = 0;
        // The loop is the same for every group of the warp (trip count = the longest frame, work predicated, no early
        // exit): groups that left a loop at different times would never run in lockstep again, and the redundant
        // instruction stream would be issued once per group instead of once per warp.  Inside, everything but the rare
        // "fields do not fit the window" case is branch-free for the same reason.
        uint32_t nmax = (act && ok) ? nseq : 0u;
#pragma unroll
        for (int off = 16; off; off >>= 1) nmax = max(nmax, __shfl_xor_sync(VMB_FULL, nmax, off));
        const bool live = act && ok;
        if (!live) nseq = 0;
        for (uint32_t q = 0; q < nmax; q++) {
            const bool run = q < nseq;
            if (run) {
                const uint32_t ell = T->ll_nb[sll], eof = T->of_nb[sof], eml = T->ml_nb[sml];  // (nbits << 12) | base
                const uint32_t yll = T->ll_sym[sll], yof = T->of_sym[sof], yml = T->ml_sym[sml];  // (<= 35 / 31 / 52 by construction)
                const uint32_t b_of = yof, b_ml = s_ml_bits[yml], b_ll = s_ll_bits[yll];
                // (the last sequence reads no state bits; the loop reads them anyway and the totals are put right after it)
                const uint32_t n_ll = ell >> 12, n_ml = eml >> 12, n_of = eof >> 12;
                const uint32_t need = b_of + b_ml + b_ll + n_ll + n_ml + n_of;
                last_state_bits = n_ll + n_ml + n_of;
                if (bb.cnt <= 32) bb.refill();
                uint32_t x_of, x_ml, x_ll, x_sl, x_sm, x_so;
                if ((int)need <= bb.cnt) {
                    // all the bits of this sequence are in the window (nearly always): six funnel-shift cuts
                    x_of = bb.take(b_of);
                    x_ml = bb.take(b_ml);
                    x_ll = bb.take(b_ll);
                    x_sl = bb.take(n_ll);
                    x_sm = bb.take(n_ml);
                    x_so = bb.take(n_of);
                    bb.cnt -= (int)need;
                    bb.left -= (int)need;
                } else {
                    x_of = bb.read_slow(b_of);
                    x_ml = bb.read_slow(b_ml);
                    x_ll = bb.read_slow(b_ll);
                    x_sl = bb.read_slow(n_ll);
                    x_sm = bb.read_slow(n_ml);
                    x_so = bb.read_slow(n_of);
                }
                sll = (ell & 0xfffu) + x_sl;
                sml = (eml & 0xfffu) + x_sm;
                sof = (eof & 0xfffu) + x_so;
                const uint32_t ofv = (1u << (yof & 31u)) + x_of;
                const uint32_t mlen = s_ml_base[yml] + x_ml, llen = s_ll_base[yll] + x_ll;
                // offset codes > 24 cannot be valid here (the window is at most the column)
                bad |= (uint32_t)(yof > 24u);
                // repeat offsets (RFC 8878 3.1.1.5), as selects: idx 0 = rep0 unchanged, 1 = swap in rep1, 2 = rotate in rep2,
                // 3 = rep0 - 1 or a new offset (both push the history down)
                const bool is_new = ofv > 3u;
                const uint32_t idx = is_new ? 3u : ofv - 1u + (llen == 0u ? 1u : 0u);
                const uint32_t from_hist = idx == 0u ? rep0 : (idx == 1u ? rep1 : (idx == 2u ? rep2 : rep0 - 1u));
                const uint32_t offset = is_new ? ofv - 3u : from_hist;
                rep2 = idx >= 2u ? rep1 : rep2;
                rep1 = idx >= 1u ? rep0 : rep1;
                rep0 = offset;
                o += llen;
                bad |= (uint32_t)(offset > o) | (uint32_t)(offset == 0u);
                o += mlen;
                bad |= (uint32_t)(o > out_cap);  // (sticky, so o stays within 2^32; lit_pos <= o: its bound is checked after the loop)
                lit_pos += llen;
                if (sub == 0) rec[q] = SEQ_REC(llen, mlen, offset);
            }
        }
        bb.left += (int)last_state_bits;  // the state update behind the last sequence does not exist in the stream
        if (lit_pos > lit_len) bad = 1;
        if (bad) ok = false;
        if (live && ok) {
            if (bb.left != 0) ok = false;
            if (ok && o + (lit_len - lit_pos) != out_cap) ok = false;
        }
        if (live && sub == 0 && !ok) P.status[col] = VMB_ERR_ZSTD;
        if (act && !live && sub == 0 && !ok) P.status[col] = VMB_ERR_ZSTD;
        __syncwarp();
    }
}

#define SEQX_WARPS 4
// n bytes src -> dst by the whole warp (no overlap between the two ranges within n): long runs go 16 bytes per lane and step
// -- destination aligned to 16, the source read as five aligned words and funnel-shifted into place
__device__ __forceinline__ void warp_copy(uint8_t* dst, const uint8_t* src, uint32_t n, int lane) {
    if (n >= 64u) {
        uint32_t head = (uint32_t)((16u - ((uintptr_t)dst & 15u)) & 15u);
        if ((uint32_t)lane < head) dst[lane] = src[lane];
        const uint32_t chunks = (n - head) >> 4;
        const uint8_t* s0 = src + head;
        const uint32_t sh = (uint32_t)((uintptr_t)s0 & 3u) * 8u;
        const uint32_t* sw = (const uint32_t*)((uintptr_t)s0 & ~(uintptr_t)3);
        uint4* d4 = (uint4*)(dst + head);
        for (uint32_t c = lane; c < chunks; c += 32) {
            const uint32_t* w = sw + 4 * c;
            const uint32_t w0 = w[0], w1 = w[1], w2 = w[2], w3 = w[3], w4 = sh ? w[4] : 0u;
            uint4 v;
            v.x = __funnelshift_r(w0, w1, sh);
            v.y = __funnelshift_r(w1, w2, sh);
            v.z = __funnelshift_r(w2, w3, sh);
            v.w = __funnelshift_r(w3, w4, sh);
            d4[c] = v;
        }
        const uint32_t done = head + 16u * chunks;
        if (done + lane < n) dst[done + lane] = src[done + lane];  // <= 15 tail bytes
        return;
    }
    for (uint32_t k = lane; k < n; k += 32) dst[k] = src[k];
}

// One warp per frame, 32 sequences per step, one sequence per lane: positions by two warp scans; every lane copies its own
// literal run (independent of everything else) and, when its match reads only bytes in front of the step's first output byte
// -- final since the previous step --, its own match too; the remaining matches (sources inside the step's own output) follow
// in order, each copied by the whole warp.  Matches of smooth series are short (4-13 bytes) and reach a few hundred bytes
// back: three quarters of them are of the first kind.
__global__ void __launch_bounds__(SEQX_WARPS * 32) k_zstd_seq_exec(ZstdParams P) {
    const int lane = lane_id();
    const uint32_t wi = blockIdx.x * SEQX_WARPS + (threadIdx.x >> 5), nw = gridDim.x * SEQX_WARPS;
    for (uint32_t i = wi; i < P.count; i += nw) {
        const HufJob* job = &P.jobs[i];
        if (job->nstreams == 0 || !job->dst_is_lit) continue;
        const uint32_t col = job->col;
        if (P.status[col]) continue;
        const ColInfo ci = P.cols[col];
        const unsigned long long* rec = P.seq_rec + ci.seq_rec_off;
        const uint32_t nseq = ci.nseq;
        uint8_t* out = P.scratch + ci.scratch_off;
        const uint8_t* lits = P.lit + ci.scratch_off;
        uint32_t o_base = 0, l_base = 0;
        for (uint32_t c = 0; c < nseq; c += 32) {
            const uint32_t q = c + lane;
            const unsigned long long r = q < nseq ? rec[q] : 0ull;
            const uint32_t ll = SEQ_REC_LL(r), ml = SEQ_REC_ML(r), of = SEQ_REC_OF(r);
            const uint32_t tot = ll + ml;
            uint32_t so = tot, sl = ll;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
                const uint32_t a = __shfl_up_sync(VMB_FULL, so, off), b = __shfl_up_sync(VMB_FULL, sl, off);
                if (lane >= off) { so += a; sl += b; }
            }
            const uint32_t o = o_base + so - tot, lp = l_base + sl - ll;  // where this sequence's literals go / come from
            const uint32_t d = o + ll;                                    // first byte of its match
            // ---- literal runs
            const uint32_t long_ll = __ballot_sync(VMB_FULL, ll > 16u);
            if (ll <= 16u)
                for (uint32_t k = 0; k < ll; k++) out[o + k] = lits[lp + k];
            for (uint32_t mm = long_ll; mm; mm &= mm - 1u) {
                const int j = __ffs((int)mm) - 1;
                warp_copy(out + __shfl_sync(VMB_FULL, o, j), lits + __shfl_sync(VMB_FULL, lp, j), __shfl_sync(VMB_FULL, ll, j), lane);
            }
            // ---- matches whose source is final already: one per lane
            const bool early = ml && d - of + ml <= o_base;  // (offset <= d was checked by the decoder)
            __syncwarp();
            if (early)
                for (uint32_t k = 0; k < ml; k++) out[d + k] = out[d - of + k];
            __syncwarp();
            // ---- the others, in order
            for (uint32_t mm = __ballot_sync(VMB_FULL, ml && !early); mm; mm &= mm - 1u) {
                const int j = __ffs((int)mm) - 1;
                const uint32_t dj = __shfl_sync(VMB_FULL, d, j), m = __shfl_sync(VMB_FULL, ml, j), f = __shfl_sync(VMB_FULL, of, j);
                if (m <= 32u) {  // the common case: one byte per lane, one step
                    if ((uint32_t)lane < m) out[dj + lane] = out[dj - f + (f >= m ? (uint32_t)lane : (uint32_t)lane % f)];
                } else if (f >= m) {
                    warp_copy(out + dj, out + dj - f, m, lane);
                } else {
                    const uint8_t* pat = out + dj - f;  // the match overlaps itself: a pattern of f bytes, all written before
                    for (uint32_t k = lane; k < m; k += 32) out[dj + k] = pat[k % f];
                }
                __syncwarp();
            }
            o_base += __shfl_sync(VMB_FULL, so, 31);
            l_base += __shfl_sync(VMB_FULL, sl, 31);
        }
        warp_copy(out + o_base, lits + l_base, job->regen_size - l_base, lane);  // literals after the last sequence
        __syncwarp();
    }
}

// ---- serial kernel: (mode 0) sequences of prepared frames, (mode 1) complete generic frames
__global__ void k_zstd_serial(ZstdParams P, int mode) {
    uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= P.ws_count) return;
    SerialWs* ws = (SerialWs*)P.ws + tid;
    for (uint32_t i = tid; i < P.count; i += P.ws_count) {
        if (mode == 0) {
            const HufJob* job = &P.jobs[i];
            if (job->nstreams == 0 || !job->dst_is_lit) continue;
            uint32_t col = job->col;
            if (P.status[col]) continue;
            const ColInfo ci = P.cols[col];
            const uint8_t* src;
            uint32_t len;
            col_src(P, col, &src, &len);
            ws->have_ll = ws->have_ml = ws->have_of = 0;
            ws->rep[0] = 1;
            ws->rep[1] = 4;
            ws->rep[2] = 8;
            long long o = run_sequences(ws, P.scratch + ci.scratch_off, 0, ci.content_size, P.lit + ci.scratch_off,
                                        job->regen_size, src + job->seq_off, job->seq_size);
            if (o != (long long)ci.content_size) P.status[col] = VMB_ERR_ZSTD;
        } else {
            uint32_t col = P.list[i];
            const ColInfo ci = P.cols[col];
            const uint8_t* src;
            uint32_t len;
            col_src(P, col, &src, &len);
            const long long o = P.lit ? decode_frame_serial(ws, P.scratch + ci.scratch_off, ci.content_size,
                                                            P.lit + ci.scratch_off, src, len)
                                      : -1;
            P.status[col] = o >= 0 ? 0 : VMB_ERR_ZSTD;
            // a frame without Frame_Content_Size was given the host's bound of its content: what the column decoders read is
            // the length it actually produced
            if (o >= 0 && o != (long long)ci.content_size) P.cols[col].content_size = (uint32_t)o;
        }
    }
}

size_t zstd_serial_ws_bytes() { return sizeof(SerialWs); }

void launch_zstd_prepare(const ZstdParams& P, cudaStream_t st) {
    if (!P.count) return;
    k_zstd_prepare<<<(P.count + 63) / 64, 64, 0, st>>>(P);
}

// ctas_per_sm: grid cap per SM, 0 = HUF_CTAS_PER_SM
void launch_huf_decode(const ZstdParams& P, uint32_t ctas_per_sm, cudaStream_t st) {
    if (!P.count) return;
    // 17 KB per CTA (tables, input rings, output staging): below the 48 KB that need no opt-in.  The grid is capped at 12 CTAs
    // (24 warps) per SM: with the cooperative stores the flagship's one-shot k_huf_decode measured 3.31 ms at 12, 3.23 at 4 and
    // 3.40 at 16 (H100 SXM, 700 W; DESIGN.md section 8).
    constexpr size_t smem = (size_t)HUF_WARPS * HUF_WARP_TABLE_BYTES + (size_t)HUF_WARPS * HUF_RING * 32 * sizeof(uint32_t) +
                            (size_t)HUF_WARPS * HUF_STAGE * 32 * sizeof(uint4);
    static_assert(smem <= 48 * 1024, "k_huf_decode would need cudaFuncAttributeMaxDynamicSharedMemorySize");
    const uint32_t cap = ctas_per_sm ? ctas_per_sm : HUF_CTAS_PER_SM;
    if (HUF_EXP(HUF_EXP_CARVEOUT)) {  // percent of the 228 KB maximum; each CTA also takes 1 KB the system reserves
        const int pct = (int)((cap * (smem + 1024) * 100 + 228 * 1024 - 1) / (228 * 1024));
        cudaFuncSetAttribute(k_huf_decode, cudaFuncAttributePreferredSharedMemoryCarveout, pct > 100 ? 100 : pct);
    }
    uint32_t groups = (P.count + HUF_FRAMES_PER_WARP - 1) / HUF_FRAMES_PER_WARP;
    uint32_t grid = (groups + HUF_WARPS - 1) / HUF_WARPS;
    if (grid > VMB_SMS * cap) grid = VMB_SMS * cap;
    k_huf_decode<<<grid, HUF_WARPS * 32, smem, st>>>(P);
}

#if HUF_EXP(HUF_EXP_PHASES)
// phase-clock build only: copies huf_phase_cyc (lane 0's cycles summed over all warps, then lane 0's symbols) to `out`, then
// zeroes it (reset != 0); returns HUF_PH_SLOTS so that the caller can check the layout
extern "C" int vmb_huf_phase_cycles(unsigned long long* out, int reset) {
    if (out && cudaMemcpyFromSymbol(out, huf_phase_cyc, sizeof(huf_phase_cyc)) != cudaSuccess) return -1;
    if (reset) {
        static const unsigned long long zero[HUF_PH_SLOTS] = {};
        if (cudaMemcpyToSymbol(huf_phase_cyc, zero, sizeof(zero)) != cudaSuccess) return -1;
    }
    return HUF_PH_SLOTS;
}
#endif

void launch_zstd_sequences(const ZstdParams& P, cudaStream_t st) {
    if (!P.count || !P.ws_count || !P.seq_rec) return;
    const uint32_t per_cta = SEQ_WARPS * SEQ_FPW;
    // one SeqWs slot per frame group of the grid, carved out of the serial kernel's workspace
    const uint64_t slots = (uint64_t)P.ws_count * sizeof(SerialWs) / sizeof(SeqWs);
    uint64_t groups = P.count < slots ? P.count : slots;
    uint32_t grid = (uint32_t)((groups + per_cta - 1) / per_cta);
    if ((uint64_t)grid * per_cta > slots) grid = (uint32_t)(slots / per_cta);
    if (grid == 0) grid = 1;
    {   // the predefined tables, once per device (a second context of the same device must not run ahead of the build)
        static std::mutex mu;
        static bool built[64] = {};
        int dev = 0;
        cudaGetDevice(&dev);
        std::lock_guard<std::mutex> lk(mu);
        if (!built[dev & 63]) {
            k_zstd_seq_defaults<<<1, 32, 0, st>>>();
            if (cudaStreamSynchronize(st) == cudaSuccess) built[dev & 63] = true;
        }
    }
    k_zstd_seq_decode<false><<<grid, SEQ_WARPS * 32, 0, st>>>(P);
    k_zstd_seq_decode<true><<<grid, SEQ_WARPS * 32, 0, st>>>(P);  // frames flagged by the first launch (normally none)
    uint32_t xgrid = (P.count + SEQX_WARPS - 1) / SEQX_WARPS;
    if (xgrid > VMB_SMS * 64u) xgrid = VMB_SMS * 64u;
    k_zstd_seq_exec<<<xgrid, SEQX_WARPS * 32, 0, st>>>(P);
}

void launch_zstd_serial(const ZstdParams& P, int mode, cudaStream_t st) {
    if (!P.count || !P.ws_count) return;
    uint32_t threads = P.ws_count < P.count ? P.ws_count : P.count;
    k_zstd_serial<<<(threads + 31) / 32, 32, 0, st>>>(P, mode);
}

// ---- host-side classification at upload time: reads only the frame / block / literals headers

// A frame without Frame_Content_Size (klauspost/compress, the reference's writer in builds without cgo, omits it below 256
// bytes): an upper bound of its content from the block headers.  Raw and RLE blocks are exact; a Compressed block
// regenerates at most Block_Maximum_Size.  false: the block headers run past the end of the frame.
static bool zstd_content_bound_host(const FrameHdr& h, const uint8_t* src, uint32_t len, unsigned long long* bound) {
    unsigned long long b = 0;
    uint32_t pos = h.hdr_size;
    for (;;) {
        if (pos + 3 > len) return false;
        const uint32_t bh = src[pos] | ((uint32_t)src[pos + 1] << 8) | ((uint32_t)src[pos + 2] << 16);
        pos += 3;
        const uint32_t bsize = bh >> 3, type = (bh >> 1) & 3;
        if (type == 3) return false;
        const uint32_t stored = type == 1 ? 1u : bsize;
        if ((unsigned long long)pos + stored > len) return false;
        pos += stored;
        b += type == 2 ? h.block_max : bsize;
        if (bh & 1) break;
    }
    *bound = b;
    return true;
}

// returns kind; fills content_size; *needs_lit = the literal arena is required for this column
// content_bound = 0: a block payload, at most 10 bytes per row; else the caller's cap on Frame_Content_Size
// A frame without Frame_Content_Size always takes the serial decoder, with content_size = the bound of its content; the
// decoder replaces that with the length it produced.
uint8_t zstd_classify_host(const uint8_t* src, uint32_t len, uint32_t rows, uint32_t* content_size, bool* needs_lit,
                           uint32_t* nseq, unsigned long long content_bound = 0) {
    *needs_lit = false;
    *content_size = 0;
    *nseq = 0;
    FrameHdr h;
    if (!parse_frame_header(&h, src, len)) return VMB_ZK_BAD;
    // a valid payload holds rows-1 varints of <= 10 bytes
    unsigned long long bound = content_bound ? content_bound : (unsigned long long)rows * 10ull;
    if (!h.has_fcs) {
        unsigned long long cb;
        if (!zstd_content_bound_host(h, src, len, &cb)) return VMB_ZK_BAD;
        *content_size = (uint32_t)(cb < bound ? cb : bound);
        *needs_lit = true;
        return VMB_ZK_GENERIC;
    }
    if (h.fcs > bound) return VMB_ZK_BAD;
    *content_size = (uint32_t)h.fcs;
    uint32_t pos = h.hdr_size;
    if (pos + 3 > len) return VMB_ZK_BAD;
    uint32_t bh = src[pos] | ((uint32_t)src[pos + 1] << 8) | ((uint32_t)src[pos + 2] << 16);
    pos += 3;
    uint32_t bsize = bh >> 3;
    bool last = bh & 1;
    int btype = (bh >> 1) & 3;
    *needs_lit = true;
    if (!last || btype != 2 || h.checksum) return VMB_ZK_GENERIC;  // (a content checksum is verified by the serial decoder)
    if (pos + bsize + (h.checksum ? 4u : 0u) != len || bsize < 3) return VMB_ZK_GENERIC;
    const uint8_t* blk = src + pos;
    int type = blk[0] & 3, sf = (blk[0] >> 2) & 3;
    if (type != 2) return VMB_ZK_GENERIC;
    uint32_t csize, hdr;
    if (sf == 0 || sf == 1) {
        uint32_t v = blk[0] | ((uint32_t)blk[1] << 8) | ((uint32_t)blk[2] << 16);
        csize = (v >> 14) & 0x3ff;
        hdr = 3;
    } else if (sf == 2) {
        if (bsize < 4) return VMB_ZK_GENERIC;
        uint32_t v = blk[0] | ((uint32_t)blk[1] << 8) | ((uint32_t)blk[2] << 16) | ((uint32_t)blk[3] << 24);
        csize = (v >> 18) & 0x3fff;
        hdr = 4;
    } else {
        if (bsize < 5) return VMB_ZK_GENERIC;
        unsigned long long v = blk[0] | ((unsigned long long)blk[1] << 8) | ((unsigned long long)blk[2] << 16) |
                               ((unsigned long long)blk[3] << 24) | ((unsigned long long)blk[4] << 32);
        csize = (uint32_t)((v >> 22) & 0x3ffff);
        hdr = 5;
    }
    if (hdr + csize >= bsize) return VMB_ZK_GENERIC;
    const uint8_t* sq = blk + hdr + csize;  // Number_of_Sequences (RFC 8878 3.1.1.3.2.1)
    const uint32_t avail = bsize - hdr - csize;
    uint32_t ns = sq[0];
    if (ns >= 128) {
        if (ns < 255) {
            if (avail < 2) return VMB_ZK_GENERIC;
            ns = ((ns - 128) << 8) + sq[1];
        } else {
            if (avail < 3) return VMB_ZK_GENERIC;
            ns = (uint32_t)sq[1] + ((uint32_t)sq[2] << 8) + 0x7F00u;
        }
    }
    if (ns == 0 && sq[0] != 0) return VMB_ZK_GENERIC;  // zero sequences spelled in the long form: leave it to the serial decoder
    *nseq = ns;
    *needs_lit = ns != 0;
    return VMB_ZK_HUF;
}
