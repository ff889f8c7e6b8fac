/* webp_anim_oracle.c -- scalar twin of the animated WebP leg (caesium-clt_b200/csrc/webp_anim_device.cu, webp_anim_kernels.cu)
 * over the same rules (webp_anim_core.h): decoded frame rectangles in, composited canvases out; composited canvases in, the output
 * frames (which canvases are kept, their rectangles and durations) out.  TEST INFRASTRUCTURE, NOT PRODUCT CODE. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "../caesium-clt_b200/csrc/webp_anim_core.h"

/* n frames: rects[4k..4k+3] = x, y, w, h; flags[k] ANMF flags; has_alpha[k] the bitstream's alpha feature; pixels: every frame's
 * w * h RGBA words one after the other.  canvases: n * W * H words.  Returns 0, or -1 for a frame outside the canvas. */
int orc_webp_anim_compose(int W, int H, int n, const int *rects, const int *flags, const int *has_alpha, const uint32_t *pixels, uint32_t *canvases)
{
    const size_t np = (size_t)W * H;
    uint32_t *canvas = (uint32_t *)calloc(np ? np : 1, 4);
    if (!canvas) return -1;
    WaRect prev = {0, 0, 0, 0};
    int prev_flags = 0, prev_key = 0;
    for (int k = 0; k < n; k++) {
        const WaRect r = {rects[4 * k], rects[4 * k + 1], rects[4 * k + 2], rects[4 * k + 3]};
        if (r.x < 0 || r.y < 0 || r.w < 1 || r.h < 1 || r.x + r.w > W || r.y + r.h > H) { free(canvas); return -1; }
        const WaStep s = webp_anim_step(k, r, has_alpha[k], flags[k], prev, prev_flags, prev_key, W, H);
        /* the cleared rectangle and the keyframe fill first, then the frame's own pixels */
        for (int y = 0; y < H; y++)
            for (int x = 0; x < W; x++) {
                uint32_t *c = canvas + (size_t)y * W + x;
                if (s.keyframe || (s.cleared.w > 0 && wa_in_rect(s.cleared, x, y))) *c = 0u;
            }
        for (int y = 0; y < r.h; y++)
            for (int x = 0; x < r.w; x++) {
                const int cx = r.x + x, cy = r.y + y;
                uint32_t *c = canvas + (size_t)cy * W + cx;
                const uint32_t src = pixels[(size_t)y * r.w + x];
                const int cleared = s.cleared.w > 0 && wa_in_rect(s.cleared, cx, cy);
                *c = s.blend && !s.keyframe && !cleared ? webp_anim_blend(src, *c) : src;
            }
        memcpy(canvases + np * k, canvas, np * 4);
        pixels += (size_t)r.w * r.h;
        prev = r; prev_flags = flags[k]; prev_key = s.keyframe;
    }
    free(canvas);
    return 0;
}

/* n canvases of W x H words with their durations -> the output frames: kept[j] the index of the canvas frame j shows, rects[4j..]
 * its rectangle, dur[j] its duration.  Returns the number of output frames. */
int orc_webp_anim_frames(int W, int H, int n, const uint32_t *canvases, const uint32_t *durations, int *kept, int *rects, uint32_t *dur)
{
    const size_t np = (size_t)W * H;
    int m = 0, last = -1;
    for (int k = 0; k < n; k++) {
        const uint32_t *c = canvases + np * k;
        int x0 = W, y0 = H, x1 = 0, y1 = 0;
        if (last < 0) { x0 = 0; y0 = 0; x1 = W; y1 = H; }
        else {
            const uint32_t *p = canvases + np * last;
            for (int y = 0; y < H; y++)
                for (int x = 0; x < W; x++)
                    if (c[(size_t)y * W + x] != p[(size_t)y * W + x]) {
                        if (x < x0) x0 = x;
                        if (y < y0) y0 = y;
                        if (x + 1 > x1) x1 = x + 1;
                        if (y + 1 > y1) y1 = y + 1;
                    }
        }
        if (x1 == 0) { dur[m - 1] = webp_anim_add_duration(dur[m - 1], durations[k]); continue; }
        const WaRect r = webp_anim_out_rect(x0, y0, x1, y1);
        kept[m] = k;
        rects[4 * m] = r.x; rects[4 * m + 1] = r.y; rects[4 * m + 2] = r.w; rects[4 * m + 3] = r.h;
        dur[m] = durations[k] > (uint32_t)WA_MAX_DURATION ? (uint32_t)WA_MAX_DURATION : durations[k];
        m++;
        last = k;
    }
    return m;
}
