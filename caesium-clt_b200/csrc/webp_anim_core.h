/* webp_anim_core.h -- the rules of the animated WebP re-encoder, written once for every party that has to agree on them: the
 * device kernels and their host driver (webp_anim_kernels.cu, webp_anim_device.cu), the host decoder hook (webp_anim_host.cpp)
 * and the scalar oracle (oracle/webp_anim_oracle.c, plain C -- hence no namespace and no C++ in this file).
 *
 * Pixels are RGBA words, R in the low byte, A in the high byte.
 *
 *   compositing   libwebp's WebPAnimDecoder (what Pillow shows).  The canvas starts as 0x00000000; the ANIM background colour is
 *                 not painted.  A keyframe (webp_anim_is_keyframe) starts from a zeroed canvas and draws its rectangle without
 *                 blending.  Any other frame starts from the previous canvas with the previous frame's rectangle cleared when that
 *                 frame was disposed to background; a no-blend frame replaces its rectangle, a blend frame blends every pixel that
 *                 lies outside the cleared rectangle (webp_anim_blend) and copies the ones inside it.
 *   frames        a canvas equal to the previous one is dropped and its duration added to the previous output frame (at most
 *                 2^24 - 1 ms); frame 0 covers the whole canvas, frame j the bounding box of the pixels that differ from the
 *                 previous kept canvas with x0 and y0 rounded down to even numbers (ANMF offsets count in 2-pixel units).
 *   flags         every output frame is no-blend and dispose-none, so decoding the output gives every kept canvas back exactly
 *                 when the frames are lossless.
 *   container     RIFF, VP8X (animation flag; alpha flag iff some kept pixel has alpha below 255), ANIM with the source's
 *                 background bytes and loop count, then one ANMF per frame; no ICCP, EXIF or XMP. */
#ifndef WEBP_ANIM_CORE_H
#define WEBP_ANIM_CORE_H
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define WA_HD static __host__ __device__ __forceinline__
#else
#define WA_HD static inline
#endif

#ifdef __cplusplus
namespace b200 {
#endif

enum {
    WA_MAX_DURATION = (1 << 24) - 1,   /* ANMF durations are 24-bit */
    WA_MAX_SIDE = 16383,               /* the largest canvas side this leg takes (a VP8 / VP8L frame cannot be wider) */
    WA_DISPOSE_BG = 1,                 /* ANMF flag bit 0: dispose to background */
    WA_NO_BLEND = 2                    /* ANMF flag bit 1: do not blend */
};

/* a rectangle at (x, y) of w x h pixels; empty when w == 0 */
typedef struct { int x, y, w, h; } WaRect;

WA_HD int wa_in_rect(WaRect r, int x, int y) { return x >= r.x && x < r.x + r.w && y >= r.y && y < r.y + r.h; }

/* libwebp's BlendPixelNonPremult: src over dst, non-premultiplied, in uint32 arithmetic */
WA_HD uint32_t webp_anim_blend(uint32_t src, uint32_t dst)
{
    const uint32_t sa = src >> 24;
    if (sa == 255u) return src;
    if (sa == 0u) return dst;
    const uint32_t da = dst >> 24, dfa = (da * (256u - sa)) >> 8, ba = sa + dfa, scale = (1u << 24) / ba;
    uint32_t out = ba << 24;
    for (int s = 0; s < 24; s += 8) {
        const uint32_t sc = (src >> s) & 255u, dc = (dst >> s) & 255u;
        out |= (((sc * sa + dc * dfa) * scale) >> 24) << s;
    }
    return out;
}

/* libwebp's IsKeyFrame: frame k (0-based) of rectangle r with the frame's alpha feature (an ALPH chunk, or a VP8L header with
 * its alpha bit) and flags; prev / prev_flags / prev_key describe frame k - 1 */
WA_HD int webp_anim_is_keyframe(int k, WaRect r, int has_alpha, int flags, WaRect prev, int prev_flags, int prev_key, int W, int H)
{
    if (k == 0) return 1;
    if ((!has_alpha || (flags & WA_NO_BLEND)) && r.x == 0 && r.y == 0 && r.w == W && r.h == H) return 1;
    return (prev_flags & WA_DISPOSE_BG) && ((prev.x == 0 && prev.y == 0 && prev.w == W && prev.h == H) || prev_key);
}

/* How one frame changes the canvas, everything the per-pixel rule needs */
typedef struct {
    WaRect rect;          /* the frame's rectangle */
    WaRect cleared;       /* the previous frame's rectangle when it was disposed to background, else empty */
    int keyframe, blend;
} WaStep;

/* the canvas pixel at (x, y) after the step: old = the canvas before it, src = the frame's pixel there (read only inside rect) */
WA_HD uint32_t webp_anim_pixel(const WaStep *s, int x, int y, uint32_t old, uint32_t src)
{
    const int cleared = s->cleared.w > 0 && wa_in_rect(s->cleared, x, y);
    const uint32_t base = s->keyframe || cleared ? 0u : old;
    if (!wa_in_rect(s->rect, x, y)) return base;
    return s->blend && !s->keyframe && !cleared ? webp_anim_blend(src, base) : src;
}

/* the step of frame k given the previous frame's rectangle, flags and keyframe-ness (k == 0: none) */
WA_HD WaStep webp_anim_step(int k, WaRect r, int has_alpha, int flags, WaRect prev, int prev_flags, int prev_key, int W, int H)
{
    WaStep s;
    s.rect = r;
    s.keyframe = webp_anim_is_keyframe(k, r, has_alpha, flags, prev, prev_flags, prev_key, W, H);
    s.blend = !(flags & WA_NO_BLEND);
    s.cleared = r;
    s.cleared.w = 0;
    if (k > 0 && (prev_flags & WA_DISPOSE_BG)) s.cleared = prev;
    return s;
}

/* the output rectangle of a changed box [x0, x1) x [y0, y1): offsets rounded down to even numbers */
WA_HD WaRect webp_anim_out_rect(int x0, int y0, int x1, int y1)
{
    WaRect r;
    r.x = x0 & ~1; r.y = y0 & ~1; r.w = x1 - r.x; r.h = y1 - r.y;
    return r;
}

WA_HD uint32_t webp_anim_add_duration(uint32_t a, uint32_t b) { return a + b > (uint32_t)WA_MAX_DURATION ? (uint32_t)WA_MAX_DURATION : a + b; }

/* ---- container (host side) ----------------------------------------------------------------------------------------------------- */
static inline uint8_t *wa_put24(uint8_t *o, uint32_t v) { o[0] = (uint8_t)v; o[1] = (uint8_t)(v >> 8); o[2] = (uint8_t)(v >> 16); return o + 3; }
static inline uint8_t *wa_put32(uint8_t *o, uint32_t v) { o = wa_put24(o, v); *o++ = (uint8_t)(v >> 24); return o; }

/* RIFF header (its size is patched by webp_anim_finish), VP8X and ANIM; returns bytes written (42) */
static inline int webp_anim_put_header(uint8_t *o, int W, int H, int alpha, const uint8_t bg[4], int loop)
{
    uint8_t *p = o;
    const char *riff = "RIFF\0\0\0\0WEBPVP8X";
    for (int i = 0; i < 16; i++) *p++ = (uint8_t)riff[i];
    p = wa_put32(p, 10);
    *p++ = (uint8_t)(0x02 | (alpha ? 0x10 : 0)); *p++ = 0; *p++ = 0; *p++ = 0;
    p = wa_put24(p, (uint32_t)(W - 1)); p = wa_put24(p, (uint32_t)(H - 1));
    *p++ = 'A'; *p++ = 'N'; *p++ = 'I'; *p++ = 'M';
    p = wa_put32(p, 6);
    for (int i = 0; i < 4; i++) *p++ = bg[i];
    *p++ = (uint8_t)loop; *p++ = (uint8_t)(loop >> 8);
    return (int)(p - o);
}

/* the ANMF chunk header and frame header of a no-blend, dispose-none frame whose sub-chunks take `payload` bytes; returns 24 */
static inline int webp_anim_put_frame_head(uint8_t *o, WaRect r, uint32_t duration, size_t payload)
{
    uint8_t *p = o;
    *p++ = 'A'; *p++ = 'N'; *p++ = 'M'; *p++ = 'F';
    p = wa_put32(p, (uint32_t)(16 + payload));
    p = wa_put24(p, (uint32_t)(r.x / 2)); p = wa_put24(p, (uint32_t)(r.y / 2));
    p = wa_put24(p, (uint32_t)(r.w - 1)); p = wa_put24(p, (uint32_t)(r.h - 1));
    p = wa_put24(p, duration);
    *p++ = WA_NO_BLEND;
    return (int)(p - o);
}

/* the RIFF size field of a finished file of n bytes */
static inline void webp_anim_finish(uint8_t *o, size_t n) { wa_put32(o + 4, (uint32_t)(n - 8)); }

#ifdef __cplusplus
}
#endif
#endif /* WEBP_ANIM_CORE_H */
