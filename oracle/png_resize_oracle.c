/*
 * oracle/png_resize_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the PNG resize leg: libcaesium png::compress_in_memory with width / height set decodes through
 * image::load_from_memory (the png crate with EXPAND), calls resize_exact(w, h, Lanczos3) and re-encodes.  Two halves here:
 *  - the decoded type of every PNG colour type / depth / tRNS (every channel kept, 16 bits stay 16 bits):
 *      grey 1/2/4/8 -> L8 (sub-byte v * 255 / (2^d - 1)), grey 16 -> L16, a grey tRNS key -> LA (alpha 0 where the UNSCALED
 *      sample equals the key, else the maximum); grey+alpha -> LA8/16; RGB -> RGB8/16, an RGB key -> RGBA; RGBA -> RGBA8/16;
 *      palette -> RGB8, palette + tRNS -> RGBA8 (entries past tRNS opaque, indices past PLTE opaque black);
 *  - Lanczos3 over u16 planes, the same two passes as orc_resize_plane_lanczos3 (resize_oracle.c) with the clamp at 65535, over
 *    the oracle's own weights (orc_resize_weights).
 * Alpha is resampled as an independent channel (not premultiplied), as the JPEG / WebP legs do.
 * Compile with -ffp-contract=off (oracle/Makefile): every multiply and add rounds separately.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

int orc_resize_weights(int in_size, int out_size, int *left, int *count, float *weights, int max_taps_cap);

/* decoded type: *color_type, *channels and *depth (8 or 16) of the image crate's buffer */
void orc_png_decoded_type(int ct, int bd, size_t ntrns, int *out_ct, int *channels, int *depth)
{
    const int d = bd == 16 ? 16 : 8;
    switch (ct) {
        case 0: if (ntrns >= 2) { *out_ct = 4; *channels = 2; } else { *out_ct = 0; *channels = 1; } *depth = d; break;
        case 2: if (ntrns >= 6) { *out_ct = 6; *channels = 4; } else { *out_ct = 2; *channels = 3; } *depth = d; break;
        case 3: if (ntrns) { *out_ct = 6; *channels = 4; } else { *out_ct = 2; *channels = 3; } *depth = 8; break;
        case 4: *out_ct = 4; *channels = 2; *depth = d; break;
        default: *out_ct = 6; *channels = 4; *depth = d; break;
    }
}

static unsigned sample_at(const uint8_t *row, size_t k, int bd)
{
    if (bd == 16) return (unsigned)row[2 * k] << 8 | row[2 * k + 1];
    if (bd == 8) return row[k];
    const size_t bit = k * (size_t)bd;
    return (row[bit / 8] >> (8 - bd - (int)(bit % 8))) & ((1u << bd) - 1);
}

/* un-filtered rows [h][rb] -> planes [channels][h][w] as u16 values (0..255 for the 8-bit types).  Returns the channel count. */
int orc_png_expand_planes(const uint8_t *raw, size_t rb, int w, int h, int ct, int bd, const uint8_t *plte, size_t nplte,
                          const uint8_t *trns, size_t ntrns, uint16_t *planes)
{
    int oct, ch, depth;
    orc_png_decoded_type(ct, bd, ntrns, &oct, &ch, &depth);
    const unsigned amax = depth == 16 ? 65535u : 255u;
    const size_t n = (size_t)w * h;
    for (int y = 0; y < h; y++) {
        const uint8_t *row = raw + (size_t)y * rb;
        for (int x = 0; x < w; x++) {
            const size_t i = (size_t)y * w + x;
            if (ct == 3) {
                const unsigned v = sample_at(row, (size_t)x, bd);
                for (int c = 0; c < 3; c++) planes[c * n + i] = (uint16_t)(3 * v + 2 < nplte ? plte[3 * v + c] : 0);
                if (ch == 4) planes[3 * n + i] = (uint16_t)(v < ntrns ? trns[v] : 255);
            } else if (ct == 0) {
                const unsigned v = sample_at(row, (size_t)x, bd);
                planes[i] = (uint16_t)(bd < 8 ? v * 255 / ((1u << bd) - 1) : v);
                if (ch == 2) planes[n + i] = (uint16_t)(v == ((unsigned)trns[0] << 8 | trns[1]) ? 0 : amax);
            } else {
                const int nin = ct == 2 ? 3 : ct == 4 ? 2 : 4;
                unsigned s[4];
                for (int c = 0; c < nin; c++) { s[c] = sample_at(row, (size_t)x * nin + c, bd); planes[c * n + i] = (uint16_t)s[c]; }
                if (ct == 2 && ch == 4) {
                    int key = 1;
                    for (int c = 0; c < 3; c++) key &= s[c] == ((unsigned)trns[2 * c] << 8 | trns[2 * c + 1]);
                    planes[3 * n + i] = (uint16_t)(key ? 0 : amax);
                }
            }
        }
    }
    return ch;
}

/* one u16 channel plane: vertical pass to f32, horizontal pass clamped to [0, 65535] and rounded half away from zero */
int orc_resize_plane_lanczos3_u16(const uint16_t *in, int w, int h, int stride, uint16_t *out, int nw, int nh, int ostride)
{
    if (nw == w && nh == h) { for (int y = 0; y < h; y++) memcpy(out + (size_t)y * ostride, in + (size_t)y * stride, (size_t)w * 2); return 0; }
    int cap_v = (int)(2 * 3 * ((float)h / nh < 1 ? 1 : (float)h / nh)) + 4, cap_h = (int)(2 * 3 * ((float)w / nw < 1 ? 1 : (float)w / nw)) + 4;
    int *lv = malloc(sizeof(int) * nh), *cv = malloc(sizeof(int) * nh), *lh = malloc(sizeof(int) * nw), *chh = malloc(sizeof(int) * nw);
    float *wv = malloc(sizeof(float) * (size_t)nh * cap_v), *wh = malloc(sizeof(float) * (size_t)nw * cap_h);
    float *tmp = malloc(sizeof(float) * (size_t)nh * w);
    int rc = -1;
    if (!lv || !cv || !lh || !chh || !wv || !wh || !tmp) goto done;
    orc_resize_weights(h, nh, lv, cv, wv, cap_v);
    orc_resize_weights(w, nw, lh, chh, wh, cap_h);
    for (int oy = 0; oy < nh; oy++) {
        const float *ws = wv + (size_t)oy * cap_v;
        for (int x = 0; x < w; x++) {
            float t = 0.0f;
            for (int i = 0; i < cv[oy]; i++) t += (float)in[(size_t)(lv[oy] + i) * stride + x] * ws[i];
            tmp[(size_t)oy * w + x] = t;
        }
    }
    for (int y = 0; y < nh; y++) for (int ox = 0; ox < nw; ox++) {
        const float *ws = wh + (size_t)ox * cap_h;
        float t = 0.0f;
        for (int i = 0; i < chh[ox]; i++) t += tmp[(size_t)y * w + lh[ox] + i] * ws[i];
        t = t < 0.0f ? 0.0f : (t > 65535.0f ? 65535.0f : t);
        out[(size_t)y * ostride + ox] = (uint16_t)roundf(t);
    }
    rc = 0;
done:
    free(lv); free(cv); free(lh); free(chh); free(wv); free(wh); free(tmp);
    return rc;
}
