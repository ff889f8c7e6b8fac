/* vp8l_enc_core.h -- the rules of the lossless WebP (VP8L) encoder, written once for every party that has to agree on them: the
 * device kernels (vp8l_kernels.cu), the host writer (vp8l_encode.cpp), the decoder (vp8l_decode.cpp: pixel helpers and predictors),
 * the ALPH coder (vp8l_alpha.cpp: prefix coding of values, the neighbourhood distance map), the CPU emulation (tests/emul) and the
 * scalar oracle (oracle/vp8l_oracle.c, plain C -- hence no namespace and no C++ in this file).
 *
 * The bitstream this encoder writes (the VP8L specification's terms): subtract-green, then a predictor transform with one of the
 * 14 modes per 16x16 tile, then one entropy-coded image with an optional colour cache, LZ77 copies at the first VP8L_NCAND
 * neighbourhood distance codes, and one prefix-code group.
 *   tile mode    the mode with the lowest sum over the four channels of N log2 N - sum n log2 n of the tile's residuals (integer
 *                fixed-point log2, so every party agrees bit for bit); ties to the lower mode
 *   copies       at pixel i, candidate code c (1..VP8L_NCAND) at distance max(1, dy * width + dx) runs while the residual pixels
 *                are equal, up to VP8L_MAX_COPY and the end of i's parse chunk; the longest run wins, ties to the smaller code;
 *                runs shorter than VP8L_MIN_COPY are no copy
 *   parse        per chunk of VP8L_CHUNK pixels from its first pixel: greedy, one-step lazy (a copy at i yields to a literal when
 *                the copy at i + 1 inside the chunk is longer)
 *   colour cache a literal at i is a cache hit for cache bits b iff the last pixel before i with the same key holds the same value
 *                (a decoder inserts every pixel it produces, copies included, into a cache that starts all zeros), so hits depend
 *                on the image only; the cache size is the candidate with the lowest integer size estimate, ties to the smaller */
#ifndef VP8L_ENC_CORE_H
#define VP8L_ENC_CORE_H
#include <stdint.h>

#if defined(__CUDACC__)
#define VP8L_HD static __host__ __device__ __forceinline__
#else
#define VP8L_HD static inline
#endif

#ifdef __cplusplus
namespace b200 {
#endif

enum {
    VP8L_TILE_BITS = 4, VP8L_TILE = 1 << VP8L_TILE_BITS,   /* predictor tiles of 16 x 16 pixels */
    VP8L_NMODES = 14,
    VP8L_NCAND = 4,                                         /* distance codes 1..4: up, left, up-left, up-right */
    VP8L_MIN_COPY = 3, VP8L_MAX_COPY = 4096,
    VP8L_CHUNK = 4096,                                      /* parse chunk; no copy crosses a chunk end */
    VP8L_NCACHE = 4,                                        /* cache-size candidates: vp8l_cache_bits(0..3) = 0, 6, 8, 10 */
    VP8L_MAX_CACHE_BITS = 10,
    VP8L_NGREEN = 256 + 24 + (1 << VP8L_MAX_CACHE_BITS),    /* green + length prefixes + cache keys, at the largest cache */
    VP8L_NDIST = 40,
    VP8L_HIST = VP8L_NGREEN + 3 * 256 + VP8L_NDIST          /* one candidate's histograms: green | red | blue | alpha | distance */
};
#define VP8L_HIST_RED (VP8L_NGREEN)
#define VP8L_HIST_BLUE (VP8L_NGREEN + 256)
#define VP8L_HIST_ALPHA (VP8L_NGREEN + 512)
#define VP8L_HIST_DIST (VP8L_NGREEN + 768)

VP8L_HD int vp8l_cache_bits(int cand) { return cand ? 4 + 2 * cand : 0; }

/* ---- pixel helpers and the 14 predictors (specification section 4.1) ------------------------------------------------------- */
VP8L_HD uint32_t vp8l_add_px(uint32_t a, uint32_t b)
{   /* per-component sum mod 256 */
    const uint32_t ag = (a & 0xFF00FF00u) + (b & 0xFF00FF00u), rb = (a & 0x00FF00FFu) + (b & 0x00FF00FFu);
    return (ag & 0xFF00FF00u) | (rb & 0x00FF00FFu);
}
VP8L_HD uint32_t vp8l_sub_px(uint32_t a, uint32_t b)
{   /* per-component difference mod 256 */
    const uint32_t ag = 0x00FF00FFu + (a & 0xFF00FF00u) - (b & 0xFF00FF00u), rb = 0xFF00FF00u + (a & 0x00FF00FFu) - (b & 0x00FF00FFu);
    return (ag & 0xFF00FF00u) | (rb & 0x00FF00FFu);
}
VP8L_HD uint32_t vp8l_avg2(uint32_t a, uint32_t b) { return (((a ^ b) & 0xFEFEFEFEu) >> 1) + (a & b); }
VP8L_HD int vp8l_clip255(int v) { return v < 0 ? 0 : v > 255 ? 255 : v; }
VP8L_HD uint32_t vp8l_select(uint32_t T, uint32_t L, uint32_t TL)
{
    int s = 0, sh;
    for (sh = 0; sh < 32; sh += 8) {
        const int t = (T >> sh) & 0xFF, l = (L >> sh) & 0xFF, c = (TL >> sh) & 0xFF;
        const int pb = l - c, pa = t - c;
        s += (pb < 0 ? -pb : pb) - (pa < 0 ? -pa : pa);
    }
    return s <= 0 ? T : L;
}
VP8L_HD uint32_t vp8l_clamp_add_sub_full(uint32_t a, uint32_t b, uint32_t c)
{
    uint32_t o = 0; int sh;
    for (sh = 0; sh < 32; sh += 8) o |= (uint32_t)vp8l_clip255((int)((a >> sh) & 0xFF) + (int)((b >> sh) & 0xFF) - (int)((c >> sh) & 0xFF)) << sh;
    return o;
}
VP8L_HD uint32_t vp8l_clamp_add_sub_half(uint32_t a, uint32_t b)
{
    uint32_t o = 0; int sh;
    for (sh = 0; sh < 32; sh += 8) { const int x = (a >> sh) & 0xFF, y = (b >> sh) & 0xFF; o |= (uint32_t)vp8l_clip255(x + (x - y) / 2) << sh; }
    return o;
}
VP8L_HD uint32_t vp8l_predict(int mode, uint32_t L, uint32_t T, uint32_t TR, uint32_t TL)
{
    switch (mode) {
        case 1: return L;
        case 2: return T;
        case 3: return TR;
        case 4: return TL;
        case 5: return vp8l_avg2(vp8l_avg2(L, TR), T);
        case 6: return vp8l_avg2(L, TL);
        case 7: return vp8l_avg2(L, T);
        case 8: return vp8l_avg2(TL, T);
        case 9: return vp8l_avg2(T, TR);
        case 10: return vp8l_avg2(vp8l_avg2(L, TL), vp8l_avg2(T, TR));
        case 11: return vp8l_select(T, L, TL);
        case 12: return vp8l_clamp_add_sub_full(L, T, TL);
        case 13: return vp8l_clamp_add_sub_half(vp8l_avg2(L, T), TL);
        default: return 0xFF000000u;
    }
}
/* the prediction of pixel (x, y) of a w-wide image under `mode`, with the edge rules: pixel 0 is 0xff000000, row 0 is predicted
 * from L, column 0 from T; TR of the last column is the first pixel of the current row (linear addressing: cur[-w + 1]) */
VP8L_HD uint32_t vp8l_predict_at(int mode, const uint32_t *img, int w, int x, int y)
{
    const uint32_t *cur = img + (long long)y * w + x;
    if (y == 0) return x ? cur[-1] : 0xFF000000u;
    if (x == 0) return cur[-w];
    return vp8l_predict(mode, cur[-1], cur[-w], cur[-w + 1], cur[-w - 1]);
}

VP8L_HD uint32_t vp8l_sub_green(uint32_t p)
{
    const uint32_t g = (p >> 8) & 0xFFu;
    return (p & 0xFF00FF00u) | ((0x01000100u + (p & 0x00FF00FFu) - ((g << 16) | g)) & 0x00FF00FFu);
}

VP8L_HD uint32_t vp8l_cache_key(uint32_t argb, int bits) { return (0x1e35a7bdu * argb) >> (32 - bits); }

/* ---- integer fixed-point log2 ------------------------------------------------------------------------------------------------ */
/* floor(log2(v) * 1024) for v >= 1 (0 for v = 0): the integer part from the top bit, ten fraction bits by repeated squaring of the
 * normalised mantissa (exact integer arithmetic) */
VP8L_HD uint32_t vp8l_log2_q10(uint32_t v)
{
    uint32_t e = 0, m, r, k;
    if (v == 0) return 0;
    while ((v >> e) > 1u) e++;
    m = e >= 15 ? v >> (e - 15) : v << (15 - e);                  /* in [2^15, 2^16): 1.15 fixed point */
    r = e << 10;
    for (k = 0; k < 10; k++) {
        m = (m * m) >> 15;                                          /* < 2^17 */
        if (m >= (1u << 16)) { m >>= 1; r |= 1u << (9 - k); }
    }
    return r;
}
/* n * log2(n) in 1/1024 bit */
VP8L_HD uint64_t vp8l_nlog2_q10(uint32_t n) { return (uint64_t)n * vp8l_log2_q10(n); }

/* ---- prefix coding of values and the neighbourhood distance map (specification sections 5.2.2, 6.2.x) ------------------------ */
/* value >= 1 -> (prefix symbol, extra bit count, extra bits) */
VP8L_HD void vp8l_prefix_of(uint32_t v, int *sym, int *nx, uint32_t *xv)
{
    const uint32_t d = v - 1;
    int hb = 0;
    if (d < 4) { *sym = (int)d; *nx = 0; *xv = 0; return; }
    while ((d >> hb) > 1u) hb++;
    *sym = 2 * hb + (int)((d >> (hb - 1)) & 1u); *nx = hb - 1; *xv = d & ((1u << *nx) - 1u);
}

/* distance codes 1..120 name a pixel of the neighbourhood: (dy << 4) | (8 - dx)  (table of the specification, section 5.2.2) */
VP8L_HD int vp8l_code_to_plane(int code /* 1..120 */)
{
    const uint8_t t[120] = {
        0x18, 0x07, 0x17, 0x19, 0x28, 0x06, 0x27, 0x29, 0x16, 0x1a, 0x26, 0x2a, 0x38, 0x05, 0x37, 0x39, 0x15, 0x1b, 0x36, 0x3a,
        0x25, 0x2b, 0x48, 0x04, 0x47, 0x49, 0x14, 0x1c, 0x35, 0x3b, 0x46, 0x4a, 0x24, 0x2c, 0x58, 0x45, 0x4b, 0x34, 0x3c, 0x03,
        0x57, 0x59, 0x13, 0x1d, 0x56, 0x5a, 0x23, 0x2d, 0x44, 0x4c, 0x55, 0x5b, 0x33, 0x3d, 0x68, 0x02, 0x67, 0x69, 0x12, 0x1e,
        0x66, 0x6a, 0x22, 0x2e, 0x54, 0x5c, 0x43, 0x4d, 0x65, 0x6b, 0x32, 0x3e, 0x78, 0x01, 0x77, 0x79, 0x53, 0x5d, 0x11, 0x1f,
        0x64, 0x6c, 0x42, 0x4e, 0x76, 0x7a, 0x21, 0x2f, 0x75, 0x7b, 0x31, 0x3f, 0x63, 0x6d, 0x52, 0x5e, 0x00, 0x74, 0x7c, 0x41,
        0x4f, 0x10, 0x20, 0x62, 0x6e, 0x30, 0x73, 0x7d, 0x51, 0x5f, 0x40, 0x72, 0x7e, 0x61, 0x6f, 0x50, 0x71, 0x7f, 0x60, 0x70};
    return t[code - 1];
}
/* the pixel distance of a code for one image width, as a decoder resolves it (codes that point forward clamp to 1); 0 when the
 * code points forward (the ALPH coder's map: such a code is never chosen for a distance) */
VP8L_HD long long vp8l_code_dist_raw(int code, int width)
{
    const int c = vp8l_code_to_plane(code);
    return (long long)(c >> 4) * width + (8 - (c & 15));
}
VP8L_HD uint32_t vp8l_code_dist(int code, int width) { const long long d = vp8l_code_dist_raw(code, width); return d >= 1 ? (uint32_t)d : 1u; }

/* pixel distance -> distance code for one image width (the ALPH coder's copies come at arbitrary distances) */
typedef struct { int width; uint32_t near_dist[120]; } Vp8lPlaneCodes;
VP8L_HD void vp8l_plane_codes_init(Vp8lPlaneCodes *pc, int w)
{
    int i;
    pc->width = w;
    for (i = 0; i < 120; i++) { const long long d = vp8l_code_dist_raw(i + 1, w); pc->near_dist[i] = d >= 1 ? (uint32_t)d : 0u; }
}
VP8L_HD uint32_t vp8l_plane_code_of(const Vp8lPlaneCodes *pc, uint32_t dist)
{
    int i;
    if (dist <= 7u * (uint32_t)pc->width + 8u)
        for (i = 0; i < 120; i++) if (pc->near_dist[i] == dist) return (uint32_t)i + 1u;
    return dist + 120u;
}

/* ---- matches and the parse ------------------------------------------------------------------------------------------------- */
/* best copy at pixel i of the residual image res[0..n): (length << 8) | code, or 0; the definition the device's bit-array search
 * and the oracle's loops must equal */
VP8L_HD uint32_t vp8l_best_copy(const uint32_t *res, uint32_t n, int width, uint32_t i)
{
    const uint32_t chunk_end = (i / VP8L_CHUNK + 1) * VP8L_CHUNK, end = chunk_end < n ? chunk_end : n;
    const uint32_t maxlen = end - i < (uint32_t)VP8L_MAX_COPY ? end - i : (uint32_t)VP8L_MAX_COPY;
    uint32_t best = 0, bl = 0, l;
    int c;
    for (c = 1; c <= VP8L_NCAND; c++) {
        const uint32_t d = vp8l_code_dist(c, width);
        if (d > i) continue;
        for (l = 0; l < maxlen && res[i + l] == res[i + l - d]; l++) {}
        if (l > bl) { bl = l; best = (l << 8) | (uint32_t)c; }
    }
    return bl >= VP8L_MIN_COPY ? best : 0u;
}
/* the step the parse takes at i given best copies at i and i + 1 (next = 0 when i + 1 is past the chunk or the image): a copy's
 * length, or 1 for a literal */
VP8L_HD uint32_t vp8l_parse_step(uint32_t here, uint32_t next)
{
    const uint32_t len = here >> 8;
    if (!len || (next >> 8) > len) return 1;
    return len;
}
/* a token as a copy or a literal: the copy it takes (0 = literal) */
VP8L_HD uint32_t vp8l_token_copy(uint32_t here, uint32_t next) { return vp8l_parse_step(here, next) > 1 ? here : 0u; }

/* ---- sizes ----------------------------------------------------------------------------------------------------------------- */
/* sum n * (log2 N - log2 n) of one histogram, 1/1024 bit */
VP8L_HD uint64_t vp8l_entropy_q10(const uint32_t *h, int n)
{
    uint64_t total = 0, s = 0; int i;
    for (i = 0; i < n; i++) { total += h[i]; s += vp8l_nlog2_q10(h[i]); }
    if (!total) return 0;
    return (total > 0xFFFFFFFFull ? 0 : (uint64_t)(uint32_t)total * vp8l_log2_q10((uint32_t)total)) - s;
}
/* the size estimate of one cache candidate from its histograms (layout VP8L_HIST): the entropy of the five alphabets plus four bits
 * of code description per used cache key */
VP8L_HD uint64_t vp8l_cache_estimate(const uint32_t *h, int bits)
{
    const int ngreen = 256 + 24 + (bits ? 1 << bits : 0);
    uint64_t e = vp8l_entropy_q10(h, ngreen) + vp8l_entropy_q10(h + VP8L_HIST_RED, 256) + vp8l_entropy_q10(h + VP8L_HIST_BLUE, 256) +
                 vp8l_entropy_q10(h + VP8L_HIST_ALPHA, 256) + vp8l_entropy_q10(h + VP8L_HIST_DIST, VP8L_NDIST);
    int k;
    for (k = 280; k < ngreen; k++) if (h[k]) e += 4 * 1024;
    return e;
}
/* the chosen candidate: the lowest estimate, ties to the smaller cache */
VP8L_HD int vp8l_choose_cache(const uint32_t *hists /* VP8L_NCACHE x VP8L_HIST */)
{
    int best = 0, c; uint64_t be = 0;
    for (c = 0; c < VP8L_NCACHE; c++) {
        const uint64_t e = vp8l_cache_estimate(hists + (long long)c * VP8L_HIST, vp8l_cache_bits(c));
        if (c == 0 || e < be) { be = e; best = c; }
    }
    return best;
}

/* the tile score of one mode: per channel N log2 N - sum n log2 n over the channel's 256-bin histogram of the tile's residuals */
VP8L_HD uint64_t vp8l_tile_cost(const uint32_t *hist /* 4 x 256 */, uint32_t npix)
{
    uint64_t cost = 0; int ch, v;
    for (ch = 0; ch < 4; ch++) {
        cost += vp8l_nlog2_q10(npix);
        for (v = 0; v < 256; v++) cost -= vp8l_nlog2_q10(hist[ch * 256 + v]);
    }
    return cost;
}

#ifdef __cplusplus
} /* namespace b200 */
#endif
#endif
