// ORACLE (test infrastructure, not product code): CPU restatement of the reference block codec.
// Follows /root/reference/lib/encoding/{int.go,nearest_delta.go,nearest_delta2.go,encoding.go},
// lib/decimal/decimal.go, lib/storage/{block.go,block_header.go}.  See vm_oracle.h for the pinning status.
#include "vm_oracle.h"

#include <dlfcn.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

namespace {

inline uint64_t zigzag(int64_t v) { return (uint64_t)((v << 1) ^ (v >> 63)); }  // int.go:88
inline int64_t unzigzag(uint64_t u) { return (int64_t)(u >> 1) ^ ((int64_t)(u << 63) >> 63); }  // int.go:82

inline int bitlen64(uint64_t x) { return x == 0 ? 0 : 64 - __builtin_clzll(x); }  // math/bits.Len64

// marshalVarInt64sSlow int.go:119 -- plain LEB128 of the zig-zag value (1..10 bytes)
inline size_t put_varuint(uint8_t* dst, uint64_t u) {
    size_t n = 0;
    while (u >= 0x80) {
        dst[n++] = (uint8_t)(u | 0x80);
        u >>= 7;
    }
    dst[n++] = (uint8_t)u;
    return n;
}

}  // namespace

extern "C" {

// MarshalVarInt64s int.go:107 (fast 1-byte path and slow path emit identical bytes)
int64_t vmo_marshal_varint64s(uint8_t* dst, size_t cap, const int64_t* vs, size_t n) {
    size_t o = 0;
    for (size_t i = 0; i < n; i++) {
        if (o + 10 > cap) return VMO_ERR_CAP;
        o += put_varuint(dst + o, zigzag(vs[i]));
    }
    return (int64_t)o;
}

// UnmarshalVarInt64s int.go:182 + unmarshalVarInt64sSlow int.go:196
int vmo_unmarshal_varint64s(int64_t* dst, size_t n, const uint8_t* src, size_t src_len, size_t* consumed) {
    if (consumed) *consumed = 0;
    if (src_len < n) return VMO_ERR_SHORT_SRC;  // int.go:183
    size_t idx = 0;
    for (size_t i = 0; i < n; i++) {
        if (idx >= src_len) return VMO_ERR_SHORT_SRC;  // int.go:199
        uint8_t c = src[idx++];
        if (c < 0x80) {
            dst[i] = (int64_t)(int8_t)((int8_t)(c >> 1) ^ ((int8_t)(c << 7) >> 7));  // int.go:206
            continue;
        }
        uint64_t u = c & 0x7f;
        unsigned nbytes = 1;
        for (;;) {
            if (idx >= src_len) return VMO_ERR_SHORT_SRC;  // int.go:211,223,240
            uint8_t b = src[idx++];
            nbytes++;
            if (nbytes > 10) {
                // int.go:276: more than 7 bytes after the first three => "too long encoded varint".
                // The Go code first scans to the terminating byte (returning "unexpected end" if the
                // source runs out); reproduce that precedence.
                while (b >= 0x80) {
                    if (idx >= src_len) return VMO_ERR_SHORT_SRC;
                    b = src[idx++];
                }
                return VMO_ERR_VARINT_TOO_LONG;
            }
            if (nbytes == 10) {
                if (b >= 0x80) continue;  // keep scanning: will be "too long" (or short src)
                if (b > 1) return VMO_ERR_VARINT_TOO_BIG;  // int.go:271
                u |= (uint64_t)1 << 63;  // int.go:275 sets bit 63 unconditionally
                break;
            }
            if (b < 0x80) {
                u |= (uint64_t)b << (7 * (nbytes - 1));
                break;
            }
            u |= (uint64_t)(b & 0x7f) << (7 * (nbytes - 1));
        }
        dst[i] = unzigzag(u);
    }
    if (consumed) *consumed = idx;
    return VMO_OK;
}

int64_t vmo_marshal_int64_be(uint8_t* dst, int64_t v) {  // int.go:69
    uint64_t u = zigzag(v);
    for (int i = 0; i < 8; i++) dst[i] = (uint8_t)(u >> (56 - 8 * i));
    return 8;
}
int64_t vmo_unmarshal_int64_be(const uint8_t* src) {  // int.go:79
    uint64_t u = 0;
    for (int i = 0; i < 8; i++) u = (u << 8) | src[i];
    return unzigzag(u);
}

// getTrailingZeros nearest_delta.go:134
uint8_t vmo_get_trailing_zeros(int64_t v, uint8_t pb) {
    uint64_t a = v < 0 ? (uint64_t)0 - (uint64_t)v : (uint64_t)v;
    if (v < 0 && (int64_t)a < 0) a = (uint64_t)v;  // -(-1<<63) wraps to itself in Go
    uint8_t vbits = (uint8_t)bitlen64(a);
    if (vbits <= pb) return 0;
    return (uint8_t)(vbits - pb);
}

static inline uint8_t dec_if_nonzero(uint8_t n) { return n == 0 ? 0 : (uint8_t)(n - 1); }

// nearestDelta nearest_delta.go:83
void vmo_nearest_delta(int64_t next, int64_t prev, uint8_t pb, uint8_t prev_tz, int64_t* dout, uint8_t* tzout) {
    int64_t d = (int64_t)((uint64_t)next - (uint64_t)prev);
    if (d == 0) {
        *dout = 0;
        *tzout = dec_if_nonzero(prev_tz);
        return;
    }
    int64_t origin = next;
    if (origin < 0) origin = (int64_t)((uint64_t)0 - (uint64_t)origin);
    uint8_t origin_bits = (uint8_t)bitlen64((uint64_t)origin);
    if (origin_bits <= pb) {
        *dout = d;
        *tzout = dec_if_nonzero(prev_tz);
        return;
    }
    uint8_t tz = (uint8_t)(origin_bits - pb);
    // Go: uint8 arithmetic `trailingZeros > prevTrailingZeros+4` (uint8 wrap is impossible here: values <= 64+4)
    if (tz > (uint8_t)(prev_tz + 4)) {
        *dout = d;
        *tzout = (uint8_t)(prev_tz + 2);
        return;
    }
    if ((uint8_t)(tz + 4) < prev_tz) {
        *dout = d;
        *tzout = (uint8_t)(prev_tz - 2);
        return;
    }
    bool minus = false;
    if (d < 0) {
        minus = true;
        d = (int64_t)((uint64_t)0 - (uint64_t)d);
    }
    // uint64(1<<64-1) << trailingZeros ; Go shifts >= 64 yield 0
    uint64_t mask = tz >= 64 ? 0 : (~(uint64_t)0 << tz);
    int64_t nd = (int64_t)((uint64_t)d & mask);
    if (minus) nd = (int64_t)((uint64_t)0 - (uint64_t)nd);
    *dout = nd;
    *tzout = tz;
}

// marshalInt64NearestDelta nearest_delta.go:15
int64_t vmo_marshal_nearest_delta(uint8_t* dst, size_t cap, const int64_t* src, size_t n, uint8_t pb, int64_t* first) {
    if (n < 1 || pb < 1 || pb > 64) return VMO_ERR_BUG;
    *first = src[0];
    int64_t v = src[0];
    std::vector<int64_t> is(n - 1);
    if (pb == 64) {
        for (size_t i = 1; i < n; i++) {
            int64_t d = (int64_t)((uint64_t)src[i] - (uint64_t)v);
            v = (int64_t)((uint64_t)v + (uint64_t)d);
            is[i - 1] = d;
        }
    } else {
        uint8_t tz = vmo_get_trailing_zeros(v, pb);
        for (size_t i = 1; i < n; i++) {
            int64_t d;
            uint8_t tzs;
            vmo_nearest_delta(src[i], v, pb, tz, &d, &tzs);
            tz = tzs;
            v = (int64_t)((uint64_t)v + (uint64_t)d);
            is[i - 1] = d;
        }
    }
    return vmo_marshal_varint64s(dst, cap, is.data(), is.size());
}

// marshalInt64NearestDelta2 nearest_delta2.go:15
int64_t vmo_marshal_nearest_delta2(uint8_t* dst, size_t cap, const int64_t* src, size_t n, uint8_t pb, int64_t* first) {
    if (n < 2 || pb < 1 || pb > 64) return VMO_ERR_BUG;
    *first = src[0];
    int64_t d1 = (int64_t)((uint64_t)src[1] - (uint64_t)src[0]);
    int64_t w0 = vmo_marshal_varint64s(dst, cap, &d1, 1);
    if (w0 < 0) return w0;
    int64_t v = src[1];
    std::vector<int64_t> is(n - 2);
    if (pb == 64) {
        for (size_t i = 2; i < n; i++) {
            int64_t d2 = (int64_t)((uint64_t)src[i] - (uint64_t)v - (uint64_t)d1);
            d1 = (int64_t)((uint64_t)d1 + (uint64_t)d2);
            v = (int64_t)((uint64_t)v + (uint64_t)d1);
            is[i - 2] = d2;
        }
    } else {
        uint8_t tz = vmo_get_trailing_zeros(v, pb);
        for (size_t i = 2; i < n; i++) {
            int64_t d2;
            uint8_t tzs;
            vmo_nearest_delta((int64_t)((uint64_t)src[i] - (uint64_t)v), d1, pb, tz, &d2, &tzs);
            tz = tzs;
            d1 = (int64_t)((uint64_t)d1 + (uint64_t)d2);
            v = (int64_t)((uint64_t)v + (uint64_t)d1);
            is[i - 2] = d2;
        }
    }
    int64_t w1 = vmo_marshal_varint64s(dst + w0, cap - (size_t)w0, is.data(), is.size());
    if (w1 < 0) return w1;
    return w0 + w1;
}

// unmarshalInt64NearestDelta nearest_delta.go:53
int vmo_unmarshal_nearest_delta(int64_t* dst, const uint8_t* src, size_t src_len, int64_t first, size_t n) {
    if (n < 1) return VMO_ERR_BUG;
    std::vector<int64_t> is(n - 1);
    size_t consumed = 0;
    int rc = vmo_unmarshal_varint64s(is.data(), n - 1, src, src_len, &consumed);
    if (rc != VMO_OK) return rc;
    if (consumed < src_len) return VMO_ERR_TAIL;
    uint64_t v = (uint64_t)first;
    dst[0] = (int64_t)v;
    for (size_t i = 0; i + 1 < n; i++) {
        v += (uint64_t)is[i];
        dst[i + 1] = (int64_t)v;
    }
    return VMO_OK;
}

// unmarshalInt64NearestDelta2 nearest_delta2.go:57
int vmo_unmarshal_nearest_delta2(int64_t* dst, const uint8_t* src, size_t src_len, int64_t first, size_t n) {
    if (n < 2) return VMO_ERR_BUG;
    std::vector<int64_t> is(n - 1);
    size_t consumed = 0;
    int rc = vmo_unmarshal_varint64s(is.data(), n - 1, src, src_len, &consumed);
    if (rc != VMO_OK) return rc;
    if (consumed < src_len) return VMO_ERR_TAIL;
    uint64_t v = (uint64_t)first;
    uint64_t d1 = (uint64_t)is[0];
    dst[0] = (int64_t)v;
    v += d1;
    dst[1] = (int64_t)v;
    for (size_t i = 1; i + 1 < n; i++) {
        d1 += (uint64_t)is[i];
        v += d1;
        dst[i + 1] = (int64_t)v;
    }
    return VMO_OK;
}

// isConst encoding.go:289
int vmo_is_const(const int64_t* a, size_t n) {
    if (n == 0) return 0;
    for (size_t i = 0; i < n; i++)
        if (a[i] != a[0]) return 0;
    return 1;
}
// isDeltaConst encoding.go:311
int vmo_is_delta_const(const int64_t* a, size_t n) {
    if (n < 2) return 0;
    uint64_t d1 = (uint64_t)a[1] - (uint64_t)a[0];
    for (size_t i = 2; i < n; i++)
        if ((uint64_t)a[i] - (uint64_t)a[i - 1] != d1) return 0;
    return 1;
}
// isGauge encoding.go:331
int vmo_is_gauge(const int64_t* a, size_t n) {
    if (n < 2) return 0;
    size_t resets = 0;
    int64_t prev = a[0];
    if (prev < 0) return 1;
    for (size_t i = 1; i < n; i++) {
        int64_t v = a[i];
        if (v < prev) {
            if (v < 0) return 1;
            if (v > (prev >> 3)) return 1;
            resets++;
        }
        prev = v;
    }
    if (resets <= 2) return 0;
    return resets > (n >> 3);
}
// getCompressLevel encoding.go:371
int vmo_get_compress_level(size_t n) {
    if (n <= (1u << 6)) return 1;
    if (n <= (1u << 8)) return 2;
    if (n <= (1u << 10)) return 3;
    if (n <= (1u << 12)) return 4;
    return 5;
}

// EnsureNonDecreasingSequence encoding.go:258
void vmo_ensure_non_decreasing(int64_t* a, size_t n, int64_t vmin, int64_t vmax) {
    if (n == 0) return;
    if (a[0] != vmin) a[0] = vmin;
    int64_t prev = a[0];
    for (size_t i = 1; i < n; i++) {
        if (a[i] < prev) a[i] = prev;
        prev = a[i];
    }
    ptrdiff_t i = (ptrdiff_t)n - 1;
    if (a[i] != vmax) {
        a[i] = vmax;
        i--;
        while (i >= 0 && a[i] > vmax) {
            a[i] = vmax;
            i--;
        }
    }
}

// checkTimestampsBounds block.go:298
int vmo_check_timestamps_bounds(const int64_t* ts, size_t n, int64_t tmin, int64_t tmax) {
    if (n == 0) return VMO_OK;
    int64_t prev = ts[0];
    if (prev < tmin) return VMO_ERR_TS_BOUNDS;
    for (size_t i = 1; i < n; i++) {
        if (ts[i] < prev) return VMO_ERR_TS_BOUNDS;
        prev = ts[i];
    }
    if (prev > tmax) return VMO_ERR_TS_BOUNDS;
    return VMO_OK;
}

// ---------------------------------------------------------------- zstd reference (libzstd 1.5.7) via oracle/_ref
typedef size_t (*ref_compress_fn)(void*, size_t, const void*, size_t, int);
typedef size_t (*ref_decompress_fn)(void*, size_t, const void*, size_t);
typedef unsigned (*ref_iserr_fn)(size_t);
typedef size_t (*ref_compress_params_fn)(void*, size_t, const void*, size_t, const int*, int);
typedef size_t (*ref_compress_seq_fn)(void*, size_t, const void*, size_t, const unsigned*, size_t, const int*, int);
static ref_compress_fn g_ref_compress;
static ref_decompress_fn g_ref_decompress;
static ref_compress_fn g_ref_compress_ck;
static ref_compress_params_fn g_ref_compress_params;
static ref_compress_seq_fn g_ref_compress_seq;
static ref_iserr_fn g_ref_iserr;
static int g_ref_state;  // 0 = not tried, 1 = ok, -1 = unavailable

static void load_ref() {
    if (g_ref_state != 0) return;
    g_ref_state = -1;
    Dl_info info;
    std::string dir = ".";
    if (dladdr((void*)&load_ref, &info) && info.dli_fname) {
        std::string p(info.dli_fname);
        size_t s = p.rfind('/');
        if (s != std::string::npos) dir = p.substr(0, s);
    }
    std::string path = dir + "/_ref/libzstd_ref.so";
    void* h = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    if (!h) return;
    g_ref_compress = (ref_compress_fn)dlsym(h, "ref_zstd_compress");
    g_ref_decompress = (ref_decompress_fn)dlsym(h, "ref_zstd_decompress");
    g_ref_compress_ck = (ref_compress_fn)dlsym(h, "ref_zstd_compress_checksum");
    g_ref_compress_params = (ref_compress_params_fn)dlsym(h, "ref_zstd_compress_params");
    g_ref_compress_seq = (ref_compress_seq_fn)dlsym(h, "ref_zstd_compress_sequences");
    g_ref_iserr = (ref_iserr_fn)dlsym(h, "ref_zstd_is_error");
    if (g_ref_compress && g_ref_decompress && g_ref_iserr) g_ref_state = 1;
}
int vmo_zstd_ref_available(void) {
    load_ref();
    return g_ref_state == 1;
}
// the frame factory (ref_zstd_compress_params / ref_zstd_compress_sequences): absent from an oracle/_ref built by an older
// recipe, which still serves everything else
int vmo_zstd_ref_factory_available(void) {
    return vmo_zstd_ref_available() && g_ref_compress_params && g_ref_compress_seq;
}
int64_t vmo_zstd_ref_compress(uint8_t* dst, size_t cap, const uint8_t* src, size_t n, int level) {
    load_ref();
    if (g_ref_state != 1) return VMO_ERR_NO_ZSTD_REF;
    size_t r = g_ref_compress(dst, cap, src, n, level);
    if (g_ref_iserr(r)) return VMO_ERR_ZSTD;
    return (int64_t)r;
}
int64_t vmo_zstd_ref_compress_checksum(uint8_t* dst, size_t cap, const uint8_t* src, size_t n, int level) {
    if (!vmo_zstd_ref_available() || !g_ref_compress_ck) return VMO_ERR_NO_ZSTD_REF;
    size_t r = g_ref_compress_ck(dst, cap, src, n, level);
    if (g_ref_iserr(r)) return VMO_ERR_ZSTD;
    return (int64_t)r;
}
// ZSTD_compress2 after ZSTD_CCtx_setParameter of each (param, value) pair in kv[0 .. 2 * nkv)
int64_t vmo_zstd_ref_compress_params(uint8_t* dst, size_t cap, const uint8_t* src, size_t n, const int* kv, int nkv) {
    if (!vmo_zstd_ref_factory_available()) return VMO_ERR_NO_ZSTD_REF;
    size_t r = g_ref_compress_params(dst, cap, src, n, kv, nkv);
    if (g_ref_iserr(r)) return VMO_ERR_ZSTD;
    return (int64_t)r;
}
// ZSTD_compressSequences, explicit block delimiters: seq = nseq (offset, literal length, match length) triples
int64_t vmo_zstd_ref_compress_sequences(uint8_t* dst, size_t cap, const uint8_t* src, size_t n, const uint32_t* seq, size_t nseq,
                                        const int* kv, int nkv) {
    if (!vmo_zstd_ref_factory_available()) return VMO_ERR_NO_ZSTD_REF;
    size_t r = g_ref_compress_seq(dst, cap, src, n, seq, nseq, kv, nkv);
    if (g_ref_iserr(r)) return VMO_ERR_ZSTD;
    return (int64_t)r;
}
int64_t vmo_zstd_ref_decompress(uint8_t* dst, size_t cap, const uint8_t* src, size_t n) {
    load_ref();
    if (g_ref_state != 1) return VMO_ERR_NO_ZSTD_REF;
    size_t r = g_ref_decompress(dst, cap, src, n);
    if (g_ref_iserr(r)) return VMO_ERR_ZSTD;
    return (int64_t)r;
}

// marshalInt64Array encoding.go:119
int64_t vmo_marshal_int64_array(uint8_t* dst, size_t cap, const int64_t* a, size_t n, uint8_t pb, int* mt, int64_t* first) {
    if (n == 0) return VMO_ERR_BUG;
    if (vmo_is_const(a, n)) {
        *first = a[0];
        *mt = 3;
        return 0;
    }
    if (vmo_is_delta_const(a, n)) {
        *first = a[0];
        *mt = 2;
        int64_t d = (int64_t)((uint64_t)a[1] - (uint64_t)a[0]);
        return vmo_marshal_varint64s(dst, cap, &d, 1);
    }
    std::vector<uint8_t> bb(n * 10 + 16);
    int64_t blen;
    if (vmo_is_gauge(a, n)) {
        *mt = 4;
        uint8_t p = pb;
        if (p < 6) p += 2;
        blen = vmo_marshal_nearest_delta(bb.data(), bb.size(), a, n, p, first);
    } else {
        *mt = 1;
        blen = vmo_marshal_nearest_delta2(bb.data(), bb.size(), a, n, pb, first);
    }
    if (blen < 0) return blen;
    int64_t clen = 0;
    const int64_t min_compressible = 128;  // encoding.go:15
    if (blen >= min_compressible) {
        clen = vmo_zstd_ref_compress(dst, cap, bb.data(), (size_t)blen, vmo_get_compress_level(n));
        if (clen < 0) return clen;
    }
    if (blen < min_compressible || (double)clen > 0.9 * (double)blen) {  // encoding.go:156
        *mt = (*mt == 1) ? 5 : 6;
        if ((size_t)blen > cap) return VMO_ERR_CAP;
        memcpy(dst, bb.data(), (size_t)blen);
        return blen;
    }
    return clen;
}

// unmarshalInt64Array encoding.go:173
int vmo_unmarshal_int64_array(int64_t* dst, const uint8_t* src, size_t src_len, int mt, int64_t first, size_t n) {
    switch (mt) {
        case 4:
        case 1: {
            // Frame_Content_Size, or for a frame without one (klauspost/compress omits it below 256 bytes) the bound of its
            // content from the block headers, capped at 10 bytes per row (the varint decode rejects anything longer);
            // the decoded length is what the frame produced
            int64_t cs = vmo_zstd_content_bound(src, src_len);
            if (cs < 0) return VMO_ERR_ZSTD;
            if (vmo_zstd_content_size(src, src_len) < 0) cs = std::min<int64_t>(cs, (int64_t)n * 10);
            std::vector<uint8_t> bb((size_t)cs + 8);
            int64_t r = vmo_zstd_decompress(bb.data(), (size_t)cs, src, src_len);
            if (r < 0) return VMO_ERR_ZSTD;
            return mt == 4 ? vmo_unmarshal_nearest_delta(dst, bb.data(), (size_t)r, first, n)
                           : vmo_unmarshal_nearest_delta2(dst, bb.data(), (size_t)r, first, n);
        }
        case 6:
            return vmo_unmarshal_nearest_delta(dst, src, src_len, first, n);
        case 5:
            return vmo_unmarshal_nearest_delta2(dst, src, src_len, first, n);
        case 3:
            if (src_len > 0) return VMO_ERR_CONST_TAIL;
            for (size_t i = 0; i < n; i++) dst[i] = first;
            return VMO_OK;
        case 2: {
            // UnmarshalVarInt64 int.go:173 = binary.Uvarint + zig-zag
            uint64_t u = 0;
            size_t i = 0;
            unsigned shift = 0;
            bool ok = false;
            for (; i < src_len; i++) {
                uint8_t b = src[i];
                if (i == 10) break;  // binary.Uvarint overflow: returns n<0
                if (b < 0x80) {
                    if (i == 9 && b > 1) break;  // overflow
                    u |= (uint64_t)b << shift;
                    ok = true;
                    i++;
                    break;
                }
                u |= (uint64_t)(b & 0x7f) << shift;
                shift += 7;
            }
            if (!ok) return VMO_ERR_DELTA_CONST;
            if (i < src_len) return VMO_ERR_TAIL;
            uint64_t d = (uint64_t)unzigzag(u);
            uint64_t v = (uint64_t)first;
            for (size_t k = 0; k < n; k++) {
                dst[k] = (int64_t)v;
                v += d;
            }
            return VMO_OK;
        }
        default:
            return VMO_ERR_MARSHAL_TYPE;
    }
}

// ---------------------------------------------------------------- lib/decimal/decimal.go
static const double kPow10Tab[32] = {1e00, 1e01, 1e02, 1e03, 1e04, 1e05, 1e06, 1e07, 1e08, 1e09, 1e10,
                                     1e11, 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21,
                                     1e22, 1e23, 1e24, 1e25, 1e26, 1e27, 1e28, 1e29, 1e30, 1e31};
static const double kPow10PosTab32[10] = {1e00, 1e32, 1e64, 1e96, 1e128, 1e160, 1e192, 1e224, 1e256, 1e288};
static const double kPow10NegTab32[11] = {1e-00,  1e-32,  1e-64,  1e-96,  1e-128, 1e-160,
                                          1e-192, 1e-224, 1e-256, 1e-288, 1e-320};
// Go stdlib math.Pow10 (src/math/pow10.go): table product, NOT pow().
double vmo_pow10(int n) {
    if (0 <= n && n <= 308) return kPow10PosTab32[(unsigned)n / 32] * kPow10Tab[(unsigned)n % 32];
    if (-323 <= n && n <= 0) return kPow10NegTab32[(unsigned)(-n) / 32] / kPow10Tab[(unsigned)(-n) % 32];
    if (n > 0) return INFINITY;
    return 0;
}

static const int64_t vInfPos = INT64_MAX;           // decimal.go:404
static const int64_t vInfNeg = INT64_MIN;           // decimal.go:405
static const int64_t vStaleNaN = INT64_MAX - 1;     // decimal.go:406
static const int64_t vMax = INT64_MAX - 2;          // decimal.go:408
static const int64_t vMin = INT64_MIN + 1;          // decimal.go:409
static const uint64_t staleNaNBits = 0x7ff0000000000002ULL;  // decimal.go:414
static inline bool is_special(int64_t v) { return v > vMax || v < vMin; }  // decimal.go:417
static inline double stale_nan() {
    double d;
    uint64_t b = staleNaNBits;
    memcpy(&d, &b, 8);
    return d;
}
static inline bool is_stale_nan(double f) {
    uint64_t b;
    memcpy(&b, &f, 8);
    return b == staleNaNBits;
}

// AppendDecimalToFloat decimal.go:100 (the all-zeros / all-ones fast paths produce the same bits)
void vmo_decimal_to_float(double* dst, const int64_t* va, size_t n, int16_t e) {
    double e10 = 1;
    if (e < 0) e10 = vmo_pow10(-(int)e);
    if (e > 0) e10 = vmo_pow10((int)e);
    for (size_t i = 0; i < n; i++) {
        int64_t v = va[i];
        double f = (double)v;
        if (e < 0) f = f / e10;
        else if (e > 0) f = f * e10;
        if (is_special(v)) {
            if (v == vInfPos) f = INFINITY;
            else if (v == vInfNeg) f = -INFINITY;
            else f = stale_nan();
        }
        dst[i] = f;
    }
}

// ToFloat decimal.go:376
double vmo_to_float(int64_t v, int16_t e) {
    if (is_special(v)) {
        if (v == vInfPos) return INFINITY;
        if (v == vInfNeg) return -INFINITY;
        return stale_nan();
    }
    double f = (double)v;
    if (e < 0) return f / vmo_pow10(-(int)e);
    return f * vmo_pow10((int)e);
}

// Go's uint64(f) on amd64 for out-of-range f yields 1<<63
static inline uint64_t go_f2u(double f) {
    if (!(f < 18446744073709551616.0)) return (uint64_t)1 << 63;
    if (f < 0) return (uint64_t)(int64_t)f;
    return (uint64_t)f;
}

// getDecimalAndScale decimal.go:480
static void get_decimal_and_scale(uint64_t u, int64_t* v, int16_t* e) {
    int16_t scale = 0;
    while (u >= ((uint64_t)1 << 55)) {
        u /= 10;
        scale++;
    }
    if (u % 10 != 0) {
        *v = (int64_t)u;
        *e = scale;
        return;
    }
    u /= 10;
    scale++;
    while (u != 0 && u % 10 == 0) {
        u /= 10;
        scale++;
    }
    *v = (int64_t)u;
    *e = scale;
}

// positiveFloatToDecimalSlow decimal.go:502
static void positive_float_to_decimal_slow(double f, int64_t* v, int16_t* e) {
    int16_t scale = 0;
    double prec = 1e12;  // conversionPrecision decimal.go:552
    if (f > 1e6 || f < 1e-6) {
        if (f > 1e6) prec = 1e15;
        int exp;
        frexp(f, &exp);
        if (exp < -1022) exp = -1022;
        else if (exp > 1023) exp = 1023;
        // math.Ln2/math.Ln10 is an exact Go constant expression rounded once to float64 = log10(2)
        scale = (int16_t)((double)exp * 0.301029995663981195213738894724493026768189881462108541310);
        f *= vmo_pow10(-(int)scale);
    }
    while (f < prec) {
        double x;
        double frac = modf(f, &x);
        if (frac * prec < x) {
            f = x;
            break;
        }
        if ((1 - frac) * prec < x) {
            f = x + 1;
            break;
        }
        f *= 100;
        scale -= 2;
    }
    uint64_t u = go_f2u(f);
    if (u % 10 != 0) {
        *v = (int64_t)u;
        *e = scale;
        return;
    }
    u /= 10;
    scale++;
    *v = (int64_t)u;
    *e = scale;
}

// positiveFloatToDecimal decimal.go:467
void vmo_positive_float_to_decimal(double f, int64_t* v, int16_t* e) {
    uint64_t u = go_f2u(f);
    if ((double)u != f) {
        positive_float_to_decimal_slow(f, v, e);
        return;
    }
    if (u < ((uint64_t)1 << 55) && u % 10 != 0) {
        *v = (int64_t)u;
        *e = 0;
        return;
    }
    get_decimal_and_scale(u, v, e);
}

// FromFloat decimal.go:437
void vmo_from_float(double f, int64_t* v, int16_t* e) {
    if (f == 0) {
        *v = 0;
        *e = 0;
        return;
    }
    if (is_stale_nan(f)) {
        *v = vStaleNaN;
        *e = 0;
        return;
    }
    if (isinf(f)) {
        *v = f > 0 ? vInfPos : vInfNeg;
        *e = 0;
        return;
    }
    if (f > 0) {
        vmo_positive_float_to_decimal(f, v, e);
        if (*v > vMax) *v = vMax;
        return;
    }
    vmo_positive_float_to_decimal(-f, v, e);
    int64_t nv = (int64_t)((uint64_t)0 - (uint64_t)*v);
    *v = nv > vMin ? nv : vMin;
}

// maxUpExponent decimal.go:268
static int16_t max_up_exponent(int64_t v) {
    if (v == 0 || is_special(v)) return 1024;
    if (v < 0) v = (int64_t)((uint64_t)0 - (uint64_t)v);
    if (v < 0) return 0;
    static const int64_t lim[19] = {INT64_MAX,          INT64_MAX / 10,          INT64_MAX / 100,
                                    INT64_MAX / 1000,   INT64_MAX / 10000,       INT64_MAX / 100000,
                                    INT64_MAX / 1000000, INT64_MAX / 10000000,   INT64_MAX / 100000000,
                                    INT64_MAX / 1000000000LL, INT64_MAX / 10000000000LL, INT64_MAX / 100000000000LL,
                                    INT64_MAX / 1000000000000LL, INT64_MAX / 10000000000000LL,
                                    INT64_MAX / 100000000000000LL, INT64_MAX / 1000000000000000LL,
                                    INT64_MAX / 10000000000000000LL, INT64_MAX / 100000000000000000LL,
                                    INT64_MAX / 1000000000000000000LL};
    for (int k = 18; k >= 1; k--)
        if (v <= lim[k]) return (int16_t)k;
    return 0;
}

// AppendFloatToDecimal decimal.go:173
int16_t vmo_float_to_decimal(int64_t* dst, const double* src, size_t n) {
    if (n == 0) return 0;
    bool zeros = true, ones = true;
    for (size_t i = 0; i < n; i++) {
        uint64_t b;
        memcpy(&b, &src[i], 8);
        if (b != 0) zeros = false;            // fastnum.IsFloat64Zeros compares raw bytes with +0
        if (b != 0x3ff0000000000000ULL) ones = false;
    }
    if (zeros) {
        for (size_t i = 0; i < n; i++) dst[i] = 0;
        return 0;
    }
    if (ones) {
        for (size_t i = 0; i < n; i++) dst[i] = 1;
        return 0;
    }
    std::vector<int64_t> va(n);
    std::vector<int16_t> ea(n);
    int16_t min_exp = (int16_t)((1 << 15) - 1);
    for (size_t i = 0; i < n; i++) {
        vmo_from_float(src[i], &va[i], &ea[i]);
        if (ea[i] < min_exp && !is_special(va[i])) min_exp = ea[i];
    }
    int16_t down_exp = 0;
    for (size_t i = 0; i < n; i++) {
        int16_t up_exp = (int16_t)(ea[i] - min_exp);
        int16_t mue = max_up_exponent(va[i]);
        if ((int16_t)(up_exp - mue) > down_exp) down_exp = (int16_t)(up_exp - mue);
    }
    min_exp = (int16_t)(min_exp + down_exp);
    for (size_t i = 0; i < n; i++) {
        int64_t v = va[i];
        if (is_special(v)) {
            dst[i] = v;
            continue;
        }
        int16_t adj = (int16_t)(ea[i] - min_exp);
        while (adj > 0) {
            v = (int64_t)((uint64_t)v * 10u);
            adj--;
        }
        while (adj < 0) {
            v /= 10;
            adj++;
        }
        dst[i] = v;
    }
    return min_exp;
}

// CalibrateScale decimal.go:13
int16_t vmo_calibrate_scale(int64_t* a, size_t na, int16_t ae, int64_t* b, size_t nb, int16_t be) {
    if (ae == be) return ae;
    if (na == 0) return be;
    if (nb == 0) return ae;
    if (ae < be) {
        int64_t* t = a; a = b; b = t;
        size_t tn = na; na = nb; nb = tn;
        int16_t te = ae; ae = be; be = te;
    }
    static const int64_t mult[19] = {1LL, 10LL, 100LL, 1000LL, 10000LL, 100000LL, 1000000LL, 10000000LL, 100000000LL,
                                     1000000000LL, 10000000000LL, 100000000000LL, 1000000000000LL, 10000000000000LL,
                                     100000000000000LL, 1000000000000000LL, 10000000000000000LL,
                                     100000000000000000LL, 1000000000000000000LL};
    int16_t up_exp = (int16_t)(ae - be);
    int16_t down_exp = 0;
    for (size_t i = 0; i < na; i++) {
        int16_t mue = max_up_exponent(a[i]);
        if ((int16_t)(up_exp - mue) > down_exp) down_exp = (int16_t)(up_exp - mue);
    }
    up_exp = (int16_t)(up_exp - down_exp);
    if (up_exp > 0) {
        int64_t m = (uint16_t)up_exp >= 19 ? 1 : mult[up_exp];
        for (size_t i = 0; i < na; i++)
            if (!is_special(a[i])) a[i] = (int64_t)((uint64_t)a[i] * (uint64_t)m);
    }
    if (down_exp > 0) {
        if (down_exp > 18) {
            for (size_t i = 0; i < nb; i++)
                if (!is_special(b[i])) b[i] = 0;
        } else {
            int64_t m = mult[down_exp];
            for (size_t i = 0; i < nb; i++)
                if (!is_special(b[i])) b[i] = b[i] / m;
        }
    }
    return (int16_t)(be + down_exp);
}

// ---------------------------------------------------------------- lib/storage/block_header.go:104 (81 bytes, big endian)
static void put_be(uint8_t* d, uint64_t v, int nbytes) {
    for (int i = 0; i < nbytes; i++) d[i] = (uint8_t)(v >> (8 * (nbytes - 1 - i)));
}
static uint64_t get_be(const uint8_t* s, int nbytes) {
    uint64_t v = 0;
    for (int i = 0; i < nbytes; i++) v = (v << 8) | s[i];
    return v;
}
void vmo_block_header_marshal(uint8_t dst[81], const vmo_block_header* bh) {
    memcpy(dst, bh->tsid, 24);  // TSID.Marshal: 3 x BE u32 + 3 x BE u64, opaque here
    vmo_marshal_int64_be(dst + 24, bh->min_ts);
    vmo_marshal_int64_be(dst + 32, bh->max_ts);
    vmo_marshal_int64_be(dst + 40, bh->first_value);
    put_be(dst + 48, bh->ts_off, 8);
    put_be(dst + 56, bh->val_off, 8);
    put_be(dst + 64, bh->ts_size, 4);
    put_be(dst + 68, bh->val_size, 4);
    put_be(dst + 72, bh->rows, 4);
    uint16_t zz = (uint16_t)(((int16_t)(bh->scale << 1)) ^ (bh->scale >> 15));  // MarshalInt16 int.go:51
    put_be(dst + 76, zz, 2);
    dst[78] = bh->ts_mt;
    dst[79] = bh->val_mt;
    dst[80] = bh->precision_bits;
}
void vmo_block_header_unmarshal(vmo_block_header* bh, const uint8_t src[81]) {
    memcpy(bh->tsid, src, 24);
    bh->min_ts = vmo_unmarshal_int64_be(src + 24);
    bh->max_ts = vmo_unmarshal_int64_be(src + 32);
    bh->first_value = vmo_unmarshal_int64_be(src + 40);
    bh->ts_off = get_be(src + 48, 8);
    bh->val_off = get_be(src + 56, 8);
    bh->ts_size = (uint32_t)get_be(src + 64, 4);
    bh->val_size = (uint32_t)get_be(src + 68, 4);
    bh->rows = (uint32_t)get_be(src + 72, 4);
    uint16_t u = (uint16_t)get_be(src + 76, 2);
    bh->scale = (int16_t)((int16_t)(u >> 1) ^ ((int16_t)(u << 15) >> 15));  // UnmarshalInt16 int.go:61
    bh->ts_mt = src[78];
    bh->val_mt = src[79];
    bh->precision_bits = src[80];
}

// Block.UnmarshalData block.go:250 + AppendRowsWithTimeRangeFilter block.go:324
int64_t vmo_block_unmarshal(int64_t* ts_out, double* val_out, int64_t* ival, const vmo_block_header* bh,
                            const uint8_t* ts_data, const uint8_t* val_data, int64_t tr_min, int64_t tr_max) {
    size_t n = bh->rows;
    if (n == 0) return VMO_ERR_BUG;
    std::vector<int64_t> ts(n);
    int rc = vmo_unmarshal_int64_array(ts.data(), ts_data, bh->ts_size, bh->ts_mt, bh->min_ts, n);
    if (rc != VMO_OK) return rc;
    if (bh->precision_bits < 64) {
        vmo_ensure_non_decreasing(ts.data(), n, bh->min_ts, bh->max_ts);
    } else if (bh->ts_mt == 5 || bh->ts_mt == 6) {
        rc = vmo_check_timestamps_bounds(ts.data(), n, bh->min_ts, bh->max_ts);
        if (rc != VMO_OK) return rc;
    }
    rc = vmo_unmarshal_int64_array(ival, val_data, bh->val_size, bh->val_mt, bh->first_value, n);
    if (rc != VMO_OK) return rc;
    // filterTimestamps block.go:331
    size_t i = 0;
    while (i < n && ts[i] < tr_min) i++;
    size_t j = n;
    while (j > i && ts[j - 1] > tr_max) j--;
    if (i == j) return 0;
    memcpy(ts_out, ts.data() + i, (j - i) * sizeof(int64_t));
    vmo_decimal_to_float(val_out, ival + i, j - i, bh->scale);
    if (i > 0) memmove(ival, ival + i, (j - i) * sizeof(int64_t));
    return (int64_t)(j - i);
}

}  // extern "C"
