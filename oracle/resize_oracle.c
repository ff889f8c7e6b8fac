/*
 * oracle/resize_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the resize leg reached through CSParameters.width/height
 * (caesium-clt's src/compressor.rs:439-443, :503-536): libcaesium's resize::resize_image calls
 * image 0.25.9 `resize_exact(w, h, FilterType::Lanczos3)` (Cargo.lock:701).  The crate source is not vendored; this
 * follows its published algorithm (imageops/sample.rs: vertical_sample into an f32 image, then horizontal_sample
 * with clamp + round-half-away to u8; lanczos3_kernel = sinc(x) * sinc(x/3) in f32), plus libjpeg's fixed-point
 * colour conversion (jdcolor.c ycc_rgb_convert, jccolor.c rgb_ycc_convert) either side of it.
 * PARITY STATUS: unpinned against the true crate (no Rust toolchain); pinned by properties and a float64 reference
 * in tests/test_oracle_resize.py.  Compile with -ffp-contract=off (oracle/Makefile) so that every multiply and add
 * rounds separately, which is what the product kernels reproduce bit for bit.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static float sincf_(float t) { float a = t * 3.14159265358979323846f; return t == 0.0f ? 1.0f : sinf(a) / a; }
float orc_lanczos3_kernel(float x) { return fabsf(x) < 3.0f ? sincf_(x) * sincf_(x / 3.0f) : 0.0f; }

/* libcaesium resize.rs compute_dimensions: the missing side follows the aspect ratio, rounded in f32 */
void orc_compute_dimensions(uint32_t ow, uint32_t oh, uint32_t dw, uint32_t dh, uint32_t *nw, uint32_t *nh)
{
    if (dw > 0 && dh > 0) { *nw = dw; *nh = dh; return; }
    float n_width = (float)dw, n_height = (float)dh;
    float ratio = (float)ow / (float)oh;
    if (dh == 0) n_height = roundf(n_width / ratio);
    if (dw == 0) n_width = roundf(n_height * ratio);
    *nw = (uint32_t)n_width; *nh = (uint32_t)n_height;
}

/* per-output-coordinate tap window and normalised weights, shared by both passes (sample.rs horizontal_sample /
 * vertical_sample).  left[i], count[i], and weights packed at stride max_taps.  Returns max_taps. */
int orc_resize_weights(int in_size, int out_size, int *left, int *count, float *weights, int max_taps_cap)
{
    float ratio = (float)in_size / (float)out_size;
    float sratio = ratio < 1.0f ? 1.0f : ratio;
    float src_support = 3.0f * sratio;
    int max_taps = 0;
    for (int o = 0; o < out_size; o++) {
        float inputx = ((float)o + 0.5f) * ratio;
        long l = (long)floorf(inputx - src_support);
        if (l < 0) l = 0;
        if (l > in_size - 1) l = in_size - 1;
        long r = (long)ceilf(inputx + src_support);
        if (r < l + 1) r = l + 1;
        if (r > in_size) r = in_size;
        inputx = inputx - 0.5f;
        int n = (int)(r - l);
        if (n > max_taps) max_taps = n;
        left[o] = (int)l; count[o] = n;
        if (weights && n <= max_taps_cap) {
            float *w = weights + (size_t)o * max_taps_cap, sum = 0.0f;
            for (int i = 0; i < n; i++) { w[i] = orc_lanczos3_kernel(((float)(l + i) - inputx) / sratio); sum += w[i]; }
            for (int i = 0; i < n; i++) w[i] /= sum;
        }
    }
    return max_taps;
}

/* one u8 channel plane: vertical pass to f32, horizontal pass to u8 */
int orc_resize_plane_lanczos3(const uint8_t *in, int w, int h, int stride, uint8_t *out, int nw, int nh, int ostride)
{
    if (nw == w && nh == h) { for (int y = 0; y < h; y++) memcpy(out + (size_t)y * ostride, in + (size_t)y * stride, w); return 0; }
    int cap_v = (int)(2 * 3 * ((float)h / nh < 1 ? 1 : (float)h / nh)) + 4, cap_h = (int)(2 * 3 * ((float)w / nw < 1 ? 1 : (float)w / nw)) + 4;
    int *lv = malloc(sizeof(int) * nh), *cv = malloc(sizeof(int) * nh), *lh = malloc(sizeof(int) * nw), *ch = malloc(sizeof(int) * nw);
    float *wv = malloc(sizeof(float) * (size_t)nh * cap_v), *wh = malloc(sizeof(float) * (size_t)nw * cap_h);
    float *tmp = malloc(sizeof(float) * (size_t)nh * w);
    if (!lv || !cv || !lh || !ch || !wv || !wh || !tmp) return -1;
    orc_resize_weights(h, nh, lv, cv, wv, cap_v);
    orc_resize_weights(w, nw, lh, ch, wh, cap_h);
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
        for (int i = 0; i < ch[ox]; i++) t += tmp[(size_t)y * w + lh[ox] + i] * ws[i];
        t = t < 0.0f ? 0.0f : (t > 255.0f ? 255.0f : t);
        out[(size_t)y * ostride + ox] = (uint8_t)roundf(t);
    }
    free(lv); free(cv); free(lh); free(ch); free(wv); free(wh); free(tmp);
    return 0;
}

/* jdcolor.c ycc_rgb_convert (SCALEBITS 16 tables) on planar data */
#define FIXC(x) ((int32_t)((x) * 65536.0 + 0.5))
static inline uint8_t clamp8(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }
void orc_ycc_to_rgb(const uint8_t *y, const uint8_t *cb, const uint8_t *cr, uint8_t *r, uint8_t *g, uint8_t *b, size_t n)
{
    for (size_t i = 0; i < n; i++) {
        int Y = y[i], xb = cb[i] - 128, xr = cr[i] - 128;
        int cr_r = (FIXC(1.40200) * xr + 32768) >> 16;
        int cb_b = (FIXC(1.77200) * xb + 32768) >> 16;
        int g_off = ((-FIXC(0.34414)) * xb + 32768 + (-FIXC(0.71414)) * xr) >> 16;
        r[i] = clamp8(Y + cr_r); g[i] = clamp8(Y + g_off); b[i] = clamp8(Y + cb_b);
    }
}
/* jccolor.c rgb_ycc_convert */
void orc_rgb_to_ycc(const uint8_t *r, const uint8_t *g, const uint8_t *b, uint8_t *y, uint8_t *cb, uint8_t *cr, size_t n)
{
    for (size_t i = 0; i < n; i++) {
        int R = r[i], G = g[i], B = b[i];
        y[i]  = (uint8_t)((FIXC(0.29900) * R + FIXC(0.58700) * G + FIXC(0.11400) * B + 32768) >> 16);
        cb[i] = (uint8_t)(((-FIXC(0.16874)) * R + (-FIXC(0.33126)) * G + FIXC(0.50000) * B + (128 << 16) + 32767) >> 16);
        cr[i] = (uint8_t)((FIXC(0.50000) * R + (-FIXC(0.41869)) * G + (-FIXC(0.08131)) * B + (128 << 16) + 32767) >> 16);
    }
}

/* ---- whole path: libcaesium jpeg compress with CSParameters.width/height set ---------------------------------
 * decode (native YCbCr, fancy upsampling) -> RGB -> Lanczos3 -> YCbCr -> the same forward path as the no-resize case */
#include "jpeg_oracle.h"
int orc_jpeg_lossy_resized(const uint8_t *data, size_t len, const orc_jpeg_params *p, uint32_t want_w, uint32_t want_h,
                           uint8_t **out, size_t *out_len, char err[256])
{
    orc_jpeg in, fw; int rc = -1;
    if (orc_jpeg_read(data, len, &in, err)) return -1;
    memset(&fw, 0, sizeof(fw));
    uint32_t nw, nh;
    orc_compute_dimensions((uint32_t)in.width, (uint32_t)in.height, want_w, want_h, &nw, &nh);
    if (nw == 0 || nh == 0 || nw > ORC_JPEG_MAX_DIMENSION || nh > ORC_JPEG_MAX_DIMENSION) { if (err) strcpy(err, "invalid target dimensions"); orc_jpeg_free(&in); return -1; }
    size_t n = (size_t)in.width * in.height, m = (size_t)nw * nh;
    uint8_t *src[4] = {0, 0, 0, 0}, *rgb[3] = {0, 0, 0}, *dst[3] = {0, 0, 0}, *ycc[4] = {0, 0, 0, 0};
    for (int c = 0; c < in.ncomp; c++) { src[c] = malloc(n); ycc[c] = malloc(m); }
    if (orc_jpeg_decode_native(&in, src, err)) goto done;
    if (in.ncomp == 3) {
        for (int c = 0; c < 3; c++) { rgb[c] = malloc(n); dst[c] = malloc(m); }
        orc_ycc_to_rgb(src[0], src[1], src[2], rgb[0], rgb[1], rgb[2], n);
        for (int c = 0; c < 3; c++) if (orc_resize_plane_lanczos3(rgb[c], in.width, in.height, in.width, dst[c], (int)nw, (int)nh, (int)nw)) goto done;
        orc_rgb_to_ycc(dst[0], dst[1], dst[2], ycc[0], ycc[1], ycc[2], m);
    } else if (orc_resize_plane_lanczos3(src[0], in.width, in.height, in.width, ycc[0], (int)nw, (int)nh, (int)nw)) goto done;
    if (orc_jpeg_forward((const uint8_t *const *)ycc, (int)nw, (int)nh, in.ncomp, p, &fw, err)) goto done;
    rc = orc_jpeg_write(&fw, p, &in, out, out_len, err);
done:
    for (int c = 0; c < 4; c++) { free(src[c]); free(ycc[c]); }
    for (int c = 0; c < 3; c++) { free(rgb[c]); free(dst[c]); }
    orc_jpeg_free(&fw); orc_jpeg_free(&in);
    return rc;
}
