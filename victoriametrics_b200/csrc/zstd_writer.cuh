// The library's zstd writer (stands for encoding.CompressZSTDLevel, lib/encoding/compress.go:13): Huffman literals only -- one
// Compressed block with zero sequences, an RLE block, or Raw blocks.  This file holds the rules that decide every byte of a
// frame, written once for both sides: the host writer (marshal.inc zstd_compress_huf: vmb_zstd_compress, vmb_marshal_columns,
// vmb_marshal_int64) and the device writer (encode.cu k_zstd_frames: vmb_zstd_compress_batch, vmb_marshal_columns_gpu) call the
// same plan_table / plan_layout, so both write the same frame byte for byte.
//
//   plan_table:  byte histogram -> RLE? Huffman code lengths (<= 11 bits, complete), the tree description (FSE-compressed or
//                direct weights) -- the serial part, one thread;
//   plan_layout: code bits per stream -> stream sizes, jump table, literals header, block header, or the Raw fallback.
//
// Device writer: one CTA per frame.  Per-warp shared histograms of each stream segment; the plan on thread 0; canonical codes
// one symbol per thread; then each segment's backward LSB-first bit stream: a tile of symbols is staged in shared memory in
// stream order (last byte first), a block-wide exclusive scan of the code lengths gives every thread the bit offset of its run
// of symbols, and each thread stores the 32-bit words it fills alone and merges only its first and last word (atomicOr into the
// zeroed frame).
#pragma once

namespace zw {

constexpr int kHufMaxBits = 11;
constexpr uint32_t kMaxBlock = 1u << 17;        // Block_Maximum_Size
constexpr uint64_t kHufMaxSrc = 262143;         // 18-bit Regenerated_Size of the 5-byte literals header
constexpr uint64_t kSingleStreamMax = 1023;     // up to here one stream, beyond it four
enum : uint8_t { kRaw = 0, kRle = 1, kHuf = 2 };

struct HufWork {  // scratch of huf_lengths: at most 256 leaves + 255 internal nodes
    uint32_t w[511];
    int16_t l[511], r[511];
    uint16_t q1[256], q2[256], tmp[256];
    uint8_t depth[511];
};

struct FramePlan {
    uint64_t n, frame_len;
    uint8_t mode, nseg, maxbits, fh;     // fh: bytes of the frame header
    uint16_t head_len;                   // kHuf / kRle: bytes before the first stream (the RLE byte); kRaw: the frame header
    uint16_t tree_len;
    uint32_t stream_off[4];              // kHuf: offset of stream k in the frame
    uint32_t seg_bits[4];                // kHuf: code bits of the symbols of segment k
    uint8_t lens[256];
    uint8_t tree[129];
    uint8_t head[9 + 3 + 5 + 129 + 6];   // frame header | block header | literals header | tree description | jump table
};

struct BitBuf {  // LSB-first bit writer into a fixed buffer; `bad` once it passes cap
    uint8_t* p;
    int cap, len = 0, cnt = 0;
    uint64_t acc = 0;
    bool bad = false;
    __host__ __device__ BitBuf(uint8_t* p_, int cap_) : p(p_), cap(cap_) {}
    __host__ __device__ void put(uint8_t b) {
        if (len < cap) p[len] = b;
        else bad = true;
        len++;
    }
    __host__ __device__ void add(uint32_t v, int nb) {
        acc |= (uint64_t)v << cnt;
        cnt += nb;
        while (cnt >= 8) {
            put((uint8_t)acc);
            acc >>= 8;
            cnt -= 8;
        }
    }
    __host__ __device__ void flush() {
        if (cnt) put((uint8_t)acc);
        acc = 0;
        cnt = 0;
    }
    __host__ __device__ void finish_with_mark() {  // final-bit marker, then pad with zeros
        add(1, 1);
        flush();
    }
};

__host__ __device__ inline int hb32(uint32_t v) {
#ifdef __CUDA_ARCH__
    return 31 - __clz(v);
#else
    return 31 - __builtin_clz(v);
#endif
}

// FSE-compresses the Huffman weights (RFC 8878 4.2.1.2) into out[0..cap).  Returns the bytes written, or -1 when the weights are
// not representable or need more than cap bytes (the caller falls back to direct weights).
__host__ __device__ inline int fse_compress_weights(uint8_t* out, int cap, const uint8_t* w, int nw) {
    const int tlog = 6, tsize = 64;
    int maxsym = 0;
    uint32_t cnt[13] = {0};
    for (int i = 0; i < nw; i++) {
        if (w[i] > 12) return -1;
        cnt[w[i]]++;
        if (w[i] > maxsym) maxsym = w[i];
    }
    int present = 0;
    for (int s = 0; s <= maxsym; s++) present += cnt[s] != 0;
    if (present < 2 || nw < 2) return -1;
    // normalize to sum == 64, every present symbol >= 1 (largest-remainder, then fix up: the first best symbol in ascending order)
    int norm[13] = {0};
    int total = 0;
    for (int s = 0; s <= maxsym; s++) {
        if (!cnt[s]) continue;
        int v = (int)((uint64_t)cnt[s] * tsize / (uint32_t)nw);
        if (v < 1) v = 1;
        norm[s] = v;
        total += v;
    }
    while (total != tsize) {
        int best = -1;
        for (int s = 0; s <= maxsym; s++) {
            if (!cnt[s]) continue;
            if (total < tsize) {  // grow the most under-represented symbol (largest cnt/norm)
                if (best < 0 || (uint64_t)cnt[s] * (uint32_t)norm[best] > (uint64_t)cnt[best] * (uint32_t)norm[s]) best = s;
            } else {              // shrink the most over-represented symbol that can still shrink (smallest cnt/norm)
                if (norm[s] <= 1) continue;
                if (best < 0 || (uint64_t)cnt[s] * (uint32_t)norm[best] < (uint64_t)cnt[best] * (uint32_t)norm[s]) best = s;
            }
        }
        if (best < 0) return -1;
        if (total < tsize) { norm[best]++; total++; }
        else { norm[best]--; total--; }
    }
    BitBuf bw(out, cap);
    // ---- header (FSE_writeNCount)
    {
        bw.add((uint32_t)(tlog - 5), 4);
        int remaining = tsize + 1, threshold = tsize, nbits = tlog + 1, sym = 0;
        bool prev0 = false;
        const int alphabet = maxsym + 1;
        while (sym < alphabet && remaining > 1) {
            if (prev0) {
                int start = sym;
                while (sym < alphabet && norm[sym] == 0) sym++;
                if (sym == alphabet) break;
                int run = sym - start;
                while (run >= 3) { bw.add(3, 2); run -= 3; }
                bw.add((uint32_t)run, 2);
            }
            int count = norm[sym++];
            int maxv = (2 * threshold - 1) - remaining;
            remaining -= count < 0 ? -count : count;
            count++;
            if (count >= threshold) count += maxv;
            bw.add((uint32_t)count, count < maxv ? nbits - 1 : nbits);
            prev0 = (count == 1);
            if (remaining < 1) return -1;
            while (remaining < threshold) { nbits--; threshold >>= 1; }
        }
        if (remaining != 1) return -1;
        bw.flush();
    }
    // ---- encoding tables (FSE_buildCTable)
    uint8_t tsym[64];
    {
        int pos = 0, step = (tsize >> 1) + (tsize >> 3) + 3, mask = tsize - 1;
        for (int s = 0; s <= maxsym; s++)
            for (int i = 0; i < norm[s]; i++) {
                tsym[pos] = (uint8_t)s;
                pos = (pos + step) & mask;
            }
        if (pos != 0) return -1;
    }
    int cumul[14];
    cumul[0] = 0;
    for (int s = 0; s <= maxsym; s++) cumul[s + 1] = cumul[s] + norm[s];
    uint16_t state_tab[64];
    {
        int c2[14];
        for (int s = 0; s < 14; s++) c2[s] = cumul[s];
        for (int u = 0; u < tsize; u++) state_tab[c2[tsym[u]]++] = (uint16_t)(tsize + u);
    }
    int delta_nb[13], delta_fs[13];
    {
        int tot = 0;
        for (int s = 0; s <= maxsym; s++) {
            if (norm[s] == 0) { delta_nb[s] = ((tlog + 1) << 16) - tsize; delta_fs[s] = 0; continue; }
            if (norm[s] == 1) {
                delta_nb[s] = (tlog << 16) - tsize;
                delta_fs[s] = tot - 1;
                tot++;
            } else {
                int mbo = tlog - hb32((uint32_t)norm[s] - 1);
                delta_nb[s] = (mbo << 16) - (norm[s] << mbo);
                delta_fs[s] = tot - norm[s];
                tot += norm[s];
            }
        }
    }
    // FSE_initCState2 / FSE_encodeSymbol; symbols with even index belong to state 1, odd index to state 2; from the end
    auto init_state = [&](int s) -> uint32_t {
        uint32_t nbo = (uint32_t)(delta_nb[s] + (1 << 15)) >> 16;
        uint32_t value = (nbo << 16) - (uint32_t)delta_nb[s];
        return state_tab[(value >> nbo) + delta_fs[s]];
    };
    auto encode = [&](uint32_t& st, int s) {
        uint32_t nbo = (uint32_t)(st + delta_nb[s]) >> 16;
        bw.add(st & ((1u << nbo) - 1), (int)nbo);
        st = state_tab[(st >> nbo) + delta_fs[s]];
    };
    int ip = nw;
    uint32_t st1, st2;
    if (nw & 1) {
        st1 = init_state(w[--ip]);
        st2 = init_state(w[--ip]);
        encode(st1, w[--ip]);
    } else {
        st2 = init_state(w[--ip]);
        st1 = init_state(w[--ip]);
    }
    while (ip > 0) {
        encode(st2, w[--ip]);
        if (ip == 0) return -1;  // parity guarantees pairs
        encode(st1, w[--ip]);
    }
    bw.add(st2 - tsize, tlog);
    bw.add(st1 - tsize, tlog);
    bw.finish_with_mark();
    return bw.bad ? -1 : bw.len;
}

// Huffman code lengths (<= 11 bits, complete code) for byte histogram `cnt` (at least two symbols present, total < 2^32).
// Leaves sorted by (count, symbol); the two-queue pop takes the leaf queue on equal weight; the lengthening loop picks the
// longest code < 11, then the lower count, then the lowest symbol; the shortening loop the highest count, then the lowest symbol.
__host__ __device__ inline bool huf_lengths(uint8_t* lens, const uint32_t* cnt, HufWork& W) {
    int nl = 0;
    for (int s = 0; s < 256; s++) {
        lens[s] = 0;
        if (cnt[s]) {
            W.w[nl] = cnt[s];
            W.l[nl] = -1;
            W.r[nl] = (int16_t)s;
            W.q1[nl] = (uint16_t)nl;
            nl++;
        }
    }
    if (nl < 2) return false;
    // leaves are in symbol order: a stable merge sort by count gives the (count, symbol) order
    for (int width = 1; width < nl; width *= 2) {
        for (int lo = 0; lo < nl; lo += 2 * width) {
            const int mid = lo + width < nl ? lo + width : nl, hi = lo + 2 * width < nl ? lo + 2 * width : nl;
            int a = lo, b = mid, o = lo;
            while (a < mid && b < hi) W.tmp[o++] = W.w[W.q1[b]] < W.w[W.q1[a]] ? W.q1[b++] : W.q1[a++];
            while (a < mid) W.tmp[o++] = W.q1[a++];
            while (b < hi) W.tmp[o++] = W.q1[b++];
        }
        for (int i = 0; i < nl; i++) W.q1[i] = W.tmp[i];
    }
    // two-queue construction
    int i1 = 0, i2 = 0, n2 = 0, nn = nl;
    while ((nl - i1) + (n2 - i2) > 1) {
        int ab[2];
        for (int k = 0; k < 2; k++)
            ab[k] = (i1 < nl && (i2 >= n2 || W.w[W.q1[i1]] <= W.w[W.q2[i2]])) ? W.q1[i1++] : W.q2[i2++];
        W.w[nn] = W.w[ab[0]] + W.w[ab[1]];
        W.l[nn] = (int16_t)ab[0];
        W.r[nn] = (int16_t)ab[1];
        W.q2[n2++] = (uint16_t)nn;
        nn++;
    }
    // depths: the root is the last node made, and every node is made after its children
    W.depth[nn - 1] = 0;
    for (int k = nn - 1; k >= nl; k--) W.depth[W.l[k]] = W.depth[W.r[k]] = (uint8_t)(W.depth[k] + 1);
    for (int k = 0; k < nl; k++) lens[W.r[k]] = W.depth[k];
    // limit to 11 bits keeping the code complete (Kraft sum == 2^11)
    const int L = kHufMaxBits;
    long long kraft = 0;
    for (int s = 0; s < 256; s++) {
        if (!lens[s]) continue;
        if (lens[s] > L) lens[s] = L;
        kraft += 1ll << (L - lens[s]);
    }
    while (kraft > (1ll << L)) {  // lengthen the longest code that is still < L
        int best = -1;
        for (int s = 0; s < 256; s++)
            if (lens[s] && lens[s] < L && (best < 0 || lens[s] > lens[best] || (lens[s] == lens[best] && cnt[s] < cnt[best]))) best = s;
        if (best < 0) return false;
        kraft -= 1ll << (L - lens[best] - 1);
        lens[best]++;
    }
    while (kraft < (1ll << L)) {  // shorten: pick the most frequent symbol whose shortening still fits
        int best = -1;
        for (int s = 0; s < 256; s++) {
            if (lens[s] < 2) continue;
            long long gain = 1ll << (L - lens[s]);
            if (kraft + gain > (1ll << L)) continue;
            if (best < 0 || cnt[s] > cnt[best]) best = s;
        }
        if (best < 0) return false;
        kraft += 1ll << (L - lens[best]);
        lens[best]--;
    }
    return true;
}

// Huffman tree description (RFC 8878 4.2.1): weights of symbols 0..lastsym-1 (the last one is implicit), FSE-compressed when
// that is shorter, else direct 4-bit weights.  Returns its bytes, or -1 when neither form fits.
__host__ __device__ inline int tree_description(uint8_t* tree, const uint8_t* lens, int lastsym, int maxbits) {
    uint8_t weights[256];
    const int nw = lastsym;
    for (int s = 0; s < nw; s++) weights[s] = lens[s] ? (uint8_t)(maxbits + 1 - lens[s]) : 0;
    const int f = nw >= 2 ? fse_compress_weights(tree + 1, 127, weights, nw) : -1;
    if (f >= 0 && (nw > 128 || f < (nw + 1) / 2)) {
        tree[0] = (uint8_t)f;
        return 1 + f;
    }
    if (nw > 128) return -1;
    tree[0] = (uint8_t)(127 + nw);
    for (int i = 0; i < nw; i += 2) tree[1 + i / 2] = (uint8_t)((weights[i] << 4) | (i + 1 < nw ? weights[i + 1] : 0));
    return 1 + (nw + 1) / 2;
}

__host__ __device__ inline int frame_header(uint8_t* o, uint64_t content) {  // single segment, no checksum, no dictionary
    o[0] = 0x28; o[1] = 0xB5; o[2] = 0x2F; o[3] = 0xFD;
    if (content < 256) {
        o[4] = 0x20;  // 1-byte FCS
        o[5] = (uint8_t)content;
        return 6;
    }
    if (content < 65536 + 256) {
        o[4] = 0x60;  // 2-byte FCS
        const uint32_t v = (uint32_t)content - 256;
        o[5] = (uint8_t)v;
        o[6] = (uint8_t)(v >> 8);
        return 7;
    }
    o[4] = 0xA0;  // 4-byte FCS
    for (int i = 0; i < 4; i++) o[5 + i] = (uint8_t)(content >> (8 * i));
    return 9;
}
__host__ __device__ inline void block_header(uint8_t* o, bool last, int type, uint32_t size) {
    const uint32_t bh = (last ? 1u : 0u) | ((uint32_t)type << 1) | (size << 3);
    o[0] = (uint8_t)bh;
    o[1] = (uint8_t)(bh >> 8);
    o[2] = (uint8_t)(bh >> 16);
}
__host__ __device__ inline uint64_t raw_frame_len(uint64_t n, int fh) { return fh + n + 3 * ((n + kMaxBlock - 1) / kMaxBlock); }
// the symbols [b, e) of stream k
__host__ __device__ inline void segment(uint64_t n, int nseg, int k, uint64_t* b, uint64_t* e) {
    if (nseg == 1) { *b = 0; *e = n; return; }
    const uint64_t seg = (n + 3) / 4;
    *b = k * seg;
    *e = k == 3 ? n : (k + 1) * seg;
}

// Step 1 of a frame: everything that follows from the byte histogram.  P.mode = kRle, kRaw, or kHuf (still subject to
// plan_layout); for kHuf, P.lens, P.maxbits and the tree description.
__host__ __device__ inline void plan_table(FramePlan& P, uint64_t n, const uint32_t* cnt, HufWork& W) {
    P.n = n;
    P.fh = (uint8_t)frame_header(P.head, n);
    int distinct = 0, lastsym = 0;
    for (int s = 0; s < 256; s++)
        if (cnt[s]) { distinct++; lastsym = s; }
    P.nseg = n <= kSingleStreamMax ? 1 : 4;
    if (distinct == 1) {  // RLE block
        P.mode = kRle;
        block_header(P.head + P.fh, true, 1, (uint32_t)n);
        P.head_len = (uint16_t)(P.fh + 3);
        P.frame_len = P.head_len + 1;
        return;
    }
    P.mode = kRaw;
    P.head_len = P.fh;
    P.frame_len = raw_frame_len(n, P.fh);
    if (n < 32 || n > kHufMaxSrc || !huf_lengths(P.lens, cnt, W)) return;
    int maxbits = 0;
    for (int s = 0; s < 256; s++) maxbits = P.lens[s] > maxbits ? P.lens[s] : maxbits;
    P.maxbits = (uint8_t)maxbits;
    const int t = tree_description(P.tree, P.lens, lastsym, maxbits);
    if (t < 0) return;
    P.tree_len = (uint16_t)t;
    P.mode = kHuf;
}

// Step 2 (P.mode == kHuf): P.seg_bits[k] = the code bits of the symbols of segment k.  Either the Compressed block's layout
// (literals header, jump table, stream offsets, P.head, P.frame_len) or the fall-back to Raw blocks.
__host__ __device__ inline void plan_layout(FramePlan& P) {
    const uint64_t n = P.n;
    const bool single = P.nseg == 1;
    uint32_t ssz[4] = {0, 0, 0, 0};
    uint64_t csize = P.tree_len + (single ? 0 : 6);
    for (int k = 0; k < P.nseg; k++) {
        ssz[k] = (P.seg_bits[k] + 8) / 8;  // the bits, the end mark, zero padding
        csize += ssz[k];
    }
    P.mode = kRaw;
    if (!single && (ssz[0] > 65535 || ssz[1] > 65535 || ssz[2] > 65535)) return;
    if (!(csize < n)) return;
    uint8_t lh[5];
    int lhn;
    if (single && csize <= 1023) {  // literals section header, type 2 = Compressed
        const uint32_t v = 2u | (0u << 2) | ((uint32_t)n << 4) | ((uint32_t)csize << 14);
        lhn = 3;
        for (int i = 0; i < 3; i++) lh[i] = (uint8_t)(v >> (8 * i));
    } else if (!single && n <= 16383 && csize <= 16383) {
        const uint32_t v = 2u | (2u << 2) | ((uint32_t)n << 4) | ((uint32_t)csize << 18);
        lhn = 4;
        for (int i = 0; i < 4; i++) lh[i] = (uint8_t)(v >> (8 * i));
    } else if (!single) {
        const uint64_t v = 2u | (3u << 2) | ((uint64_t)n << 4) | ((uint64_t)csize << 22);
        lhn = 5;
        for (int i = 0; i < 5; i++) lh[i] = (uint8_t)(v >> (8 * i));
    } else {
        return;
    }
    const uint64_t blk = lhn + csize + 1;  // + Number_of_Sequences = 0
    if (!(blk < n && blk < kMaxBlock)) return;
    P.mode = kHuf;
    int o = P.fh;
    block_header(P.head + o, true, 2, (uint32_t)blk);
    o += 3;
    for (int i = 0; i < lhn; i++) P.head[o++] = lh[i];
    for (int i = 0; i < P.tree_len; i++) P.head[o++] = P.tree[i];
    if (!single)
        for (int k = 0; k < 3; k++) {
            P.head[o++] = (uint8_t)ssz[k];
            P.head[o++] = (uint8_t)(ssz[k] >> 8);
        }
    P.head_len = (uint16_t)o;
    P.stream_off[0] = (uint32_t)o;
    for (int k = 1; k < P.nseg; k++) P.stream_off[k] = P.stream_off[k - 1] + ssz[k - 1];
    P.frame_len = P.fh + 3 + blk;
}

// canonical codes, (nbits desc, symbol asc) order == decode-table order: start[nb] = the first position of the codes of nb bits
__host__ __device__ inline void code_starts(uint32_t* start, const uint8_t* lens, int maxbits) {
    uint32_t numl[kHufMaxBits + 1] = {0};
    for (int s = 0; s < 256; s++) numl[lens[s]]++;
    uint32_t pos = 0;
    for (int nb = maxbits; nb >= 1; nb--) {
        start[nb] = pos;
        pos += numl[nb] << (maxbits - nb);
    }
}
// the code of the symbol of `nb` bits that has `rank` smaller symbols of nb bits before it
__host__ __device__ inline uint32_t canonical_code(const uint32_t* start, int nb, uint32_t rank, int maxbits) {
    return (start[nb] + (rank << (maxbits - nb))) >> (maxbits - nb);
}

}  // namespace zw
