/* vp8l_palette_core.h -- the rules of the lossless WebP (VP8L) encoder's colour-indexing (palette) variant, written once for every
 * party that has to agree on them: the device kernels (vp8l_palette.cu), the host writer (vp8l_encode.cpp), the CPU emulation
 * (tests/emul/vp8l_palette_emul.cpp) and the scalar oracle (oracle/vp8l_palette_oracle.c, plain C -- hence no C++ in this file).
 *
 *   colour       the full ARGB word (a << 24) | (r << 16) | (g << 8) | b, so distinct RGB under alpha 0 are distinct colours and the
 *                file decodes to the exact pixels; the encoder's buffer holds subtract-green pixels, so green is added back first
 *   palette      every colour of the image, ascending by that 32-bit value, when there are at most VP8L_PAL_MAX of them
 *   bundling     vp8l_pal_xbits(count) indices per packed pixel: 1 << xbits of them, index k of a bundle at bit k * (8 >> xbits) of
 *                the green channel; the packed image is ((w + (1 << xbits) - 1) >> xbits) x h, alpha 255, red and blue 0
 *   palette image the count x 1 entropy-coded image without a colour cache, each entry minus the previous one per channel mod 256
 *   the choice   with at most VP8L_PAL_MAX colours the encoder codes the image both ways and keeps the smaller file, the one without
 *                the palette on a tie, so a file is never larger than without the palette
 *   collection   per CTA a shared-memory set of the colours of VP8L_PAL_CTA_PIXELS pixels, merged into one global set; VP8L_PAL_MAX + 1
 *                distinct colours anywhere raise the overflow flag, which every CTA reads at entry and before each step */
#ifndef VP8L_PALETTE_CORE_H
#define VP8L_PALETTE_CORE_H
#include <stdint.h>
#include "vp8l_enc_core.h"

#if defined(__CUDACC__)
#define VP8L_PAL_HD static __host__ __device__ __forceinline__
#else
#define VP8L_PAL_HD static inline
#endif

#ifdef __cplusplus
namespace b200 {
#endif

enum {
    VP8L_PAL_MAX = 256,                     /* colours a palette can hold */
    VP8L_PAL_THREADS = 256,                 /* collect: threads per CTA, one pixel each per step */
    VP8L_PAL_STEPS = 16,                    /* collect: steps per CTA */
    VP8L_PAL_CTA_PIXELS = VP8L_PAL_THREADS * VP8L_PAL_STEPS,
    VP8L_PAL_SET_BITS = 10,                 /* the per-CTA and the global set: 1024 slots, never more than 512 of them taken */
    VP8L_PAL_SET = 1 << VP8L_PAL_SET_BITS,
    VP8L_PAL_INFO = 2 + VP8L_PAL_MAX        /* what the sort hands the host: count, overflow flag, the palette */
};

/* the true ARGB colour of a subtract-green pixel */
VP8L_PAL_HD uint32_t vp8l_add_green(uint32_t p)
{
    const uint32_t g = (p >> 8) & 0xFFu;
    return (p & 0xFF00FF00u) | (((p & 0x00FF00FFu) + ((g << 16) | g)) & 0x00FF00FFu);
}

/* a colour's home slot in a VP8L_PAL_SET-slot set (probing goes on linearly, wrapping) */
VP8L_PAL_HD uint32_t vp8l_pal_hash(uint32_t c) { return (c * 0x9E3779B1u) >> (32 - VP8L_PAL_SET_BITS); }

/* index bits per packed pixel's bundle: 3 for <= 2 colours, 2 for <= 4, 1 for <= 16, 0 otherwise */
VP8L_PAL_HD int vp8l_pal_xbits(int count) { return count <= 2 ? 3 : count <= 4 ? 2 : count <= 16 ? 1 : 0; }
VP8L_PAL_HD int vp8l_pal_width(int w, int xbits) { return (w + (1 << xbits) - 1) >> xbits; }

/* the index of colour c in the ascending palette pal[0 .. count) (c is in it) */
VP8L_PAL_HD int vp8l_pal_index(const uint32_t *pal, int count, uint32_t c)
{
    int lo = 0, hi = count - 1;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (pal[mid] < c) lo = mid + 1; else hi = mid; }
    return lo;
}

/* packed pixel xp of row `row` (w subtract-green pixels): the bundle of indices of pixels xp << xbits .. in green, alpha 255 */
VP8L_PAL_HD uint32_t vp8l_pal_pack(const uint32_t *row, int w, int xp, const uint32_t *pal, int count, int xbits)
{
    const int per = 1 << xbits, shift = 8 >> xbits;
    uint32_t bundle = 0; int k;
    for (k = 0; k < per; k++) {
        const int x = (xp << xbits) + k;
        if (x >= w) break;
        bundle |= (uint32_t)vp8l_pal_index(pal, count, vp8l_add_green(row[x])) << (k * shift);
    }
    return 0xFF000000u | (bundle << 8);
}

/* palette entry i as the palette image stores it: minus entry i - 1 per channel mod 256 (entry 0 as it is) */
VP8L_PAL_HD uint32_t vp8l_pal_delta(const uint32_t *pal, int i) { return i ? vp8l_sub_px(pal[i], pal[i - 1]) : pal[0]; }

#ifdef __cplusplus
} /* namespace b200 */
#endif
#endif
