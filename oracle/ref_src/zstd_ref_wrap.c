/* ORACLE support (test infrastructure): thin C wrapper over the reference's own libzstd 1.5.7
 * (vendor/github.com/valyala/gozstd/libzstd_linux_amd64.a), calling it exactly as gozstd does
 * (gozstd.go:171 ZSTD_compressCCtx, gozstd.go:331 ZSTD_decompressDCtx).  Contexts are reused per thread, like gozstd's
 * sync.Pool of cctx/dctx wrappers (gozstd.go:93, :222).  Built into oracle/_ref/. */
#define ZSTD_STATIC_LINKING_ONLY /* ZSTD_compressSequences and the experimental parameters (the .a is the same 1.5.7) */
#include <stdlib.h>

#include "zstd.h"
static __thread ZSTD_CCtx* t_cctx;
static __thread ZSTD_DCtx* t_dctx;
size_t ref_zstd_compress(void* dst, size_t cap, const void* src, size_t n, int level) {
    if (!t_cctx) t_cctx = ZSTD_createCCtx();
    return ZSTD_compressCCtx(t_cctx, dst, cap, src, n, level);
}
size_t ref_zstd_decompress(void* dst, size_t cap, const void* src, size_t n) {
    if (!t_dctx) t_dctx = ZSTD_createDCtx();
    return ZSTD_decompressDCtx(t_dctx, dst, cap, src, n);
}
/* a frame WITH a content checksum (ZSTD_c_checksumFlag): gozstd never writes one; used to test that the decoders verify it */
size_t ref_zstd_compress_checksum(void* dst, size_t cap, const void* src, size_t n, int level) {
    if (!t_cctx) t_cctx = ZSTD_createCCtx();
    ZSTD_CCtx_reset(t_cctx, ZSTD_reset_session_and_parameters);
    ZSTD_CCtx_setParameter(t_cctx, ZSTD_c_compressionLevel, level);
    ZSTD_CCtx_setParameter(t_cctx, ZSTD_c_checksumFlag, 1);
    size_t r = ZSTD_compress2(t_cctx, dst, cap, src, n);
    ZSTD_CCtx_reset(t_cctx, ZSTD_reset_session_and_parameters);
    return r;
}

/* fresh parameters, then the caller's nkv (ZSTD_cParameter, value) pairs from kv; returns 0 or a zstd error code */
static size_t set_params(const int* kv, int nkv) {
    if (!t_cctx) t_cctx = ZSTD_createCCtx();
    ZSTD_CCtx_reset(t_cctx, ZSTD_reset_session_and_parameters);
    for (int i = 0; i < nkv; i++) {
        size_t r = ZSTD_CCtx_setParameter(t_cctx, (ZSTD_cParameter)kv[2 * i], kv[2 * i + 1]);
        if (ZSTD_isError(r)) return r;
    }
    return 0;
}

/* frames in the shapes other writers produce (no Frame_Content_Size, a small window, raw literals, small blocks, high
 * levels ...): ZSTD_compress2 under explicit parameters */
size_t ref_zstd_compress_params(void* dst, size_t cap, const void* src, size_t n, const int* kv, int nkv) {
    size_t r = set_params(kv, nkv);
    if (!ZSTD_isError(r)) r = ZSTD_compress2(t_cctx, dst, cap, src, n);
    ZSTD_CCtx_reset(t_cctx, ZSTD_reset_session_and_parameters);
    return r;
}

/* a frame whose sequences the caller dictates: ZSTD_compressSequences with explicit block delimiters.  seq holds nseq
 * (offset, literal length, match length) triples over src; (0, ll, 0) ends a block with ll trailing literals.  Offsets
 * that equal a repeat offset (with ll = 0: rep2, rep3 or rep1 - 1) are written as repeat codes. */
size_t ref_zstd_compress_sequences(void* dst, size_t cap, const void* src, size_t n, const unsigned* seq, size_t nseq,
                                   const int* kv, int nkv) {
    size_t r = set_params(kv, nkv);
    if (ZSTD_isError(r)) return r;
    ZSTD_CCtx_setParameter(t_cctx, ZSTD_c_blockDelimiters, ZSTD_sf_explicitBlockDelimiters);
    ZSTD_CCtx_setParameter(t_cctx, ZSTD_c_repcodeResolution, ZSTD_ps_enable);
    ZSTD_CCtx_setParameter(t_cctx, ZSTD_c_validateSequences, 1);
    ZSTD_Sequence* s = (ZSTD_Sequence*)calloc(nseq ? nseq : 1, sizeof(ZSTD_Sequence));
    if (!s) return (size_t)-ZSTD_error_memory_allocation;
    for (size_t i = 0; i < nseq; i++) {
        s[i].offset = seq[3 * i];
        s[i].litLength = seq[3 * i + 1];
        s[i].matchLength = seq[3 * i + 2];
    }
    r = ZSTD_compressSequences(t_cctx, dst, cap, s, nseq, src, n);
    free(s);
    ZSTD_CCtx_reset(t_cctx, ZSTD_reset_session_and_parameters);
    return r;
}
unsigned ref_zstd_is_error(size_t r) { return ZSTD_isError(r); }
unsigned ref_zstd_version(void) { return ZSTD_versionNumber(); }
