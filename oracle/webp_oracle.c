/* webp_oracle.c -- TEST INFRASTRUCTURE ONLY (never linked into or called by the product).
 *
 * CPU restatement of the WebP leg of the hot path: caesium::convert_in_memory(.., SupportedFileTypes::WebP)
 * (caesium-clt's src/compressor.rs:288-292 -> libcaesium webp::compress -> libwebp, lossy VP8 key frame at
 * `parameters.webp.quality`).  libwebp is a Cargo/C dependency that is NOT vendored under the caesium-clt sources; the VP8
 * bitstream, its arithmetic ("bool") coder, token tree, transforms and intra predictors are normative (RFC 6386), so the
 * decoder side of every function below is fixed by the standard.  The ENCODER decisions are this project's profile:
 * 16x16 luma prediction only (DC / TM / V / H by least squared error), one segment, token probabilities re-estimated per
 * frame where the update pays for itself, the simple loop filter at level qindex/2, libwebp's forward transforms and
 * quality -> quantiser-index curve, quantiser bias 3/8.  Documented deviation (DESIGN.md): no 4x4 intra modes, no RD
 * optimisation, no segmentation, simple instead of normal deblocking filter, no alpha plane.
 * Parity status: "pinned by decode" -- files made here must decode in libwebp (through Pillow) to exactly this encoder's
 * own reconstruction (tests/test_webp_host.py); byte-identity with libwebp's encoder output is not claimed.
 * Plain scalar C, macroblock by macroblock in raster order.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "vp8_tables_oracle.h"

enum { M_DC = 0, M_TM = 1, M_V = 2, M_H = 3 };
static const uint8_t kZig[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};
static const uint8_t kBand[17] = {0, 1, 2, 3, 6, 4, 5, 6, 6, 6, 6, 6, 6, 6, 6, 7, 0};

static int clip8(int v) { return v < 0 ? 0 : v > 255 ? 255 : v; }

/* libwebp config: quality (0..100) -> base quantiser index, one segment, sns contribution zero */
int orc_vp8_qindex(int quality)
{
    double c = quality / 100.0;
    double lin = c < 0.75 ? c * (2.0 / 3.0) : 2.0 * c - 1.0;
    double v = pow(lin, 1.0 / 3.0);
    int q = (int)(127.0 * (1.0 - v));
    return q < 0 ? 0 : q > 127 ? 127 : q;
}

/* RFC 6386 14.1 / 9.6: dequantisation factors from the index: [0] y1 dc, [1] y1 ac, [2] y2 dc, [3] y2 ac, [4] uv dc, [5] uv ac */
void orc_vp8_quant_factors(int q, int f[6])
{
    f[0] = ORC_VP8_DC_Q[q]; f[1] = ORC_VP8_AC_Q[q];
    f[2] = ORC_VP8_DC_Q[q] * 2; f[3] = ORC_VP8_AC_Q[q] * 155 / 100; if (f[3] < 8) f[3] = 8;
    f[4] = ORC_VP8_DC_Q[q > 117 ? 117 : q]; f[5] = ORC_VP8_AC_Q[q];
}

/* ---- colour: RGB -> Y'CbCr 4:2:0, BT.601 studio range, libwebp's 16-bit fixed-point weights; chroma from the 2x2 box sum
 *      (edges replicated).  Planes are written at macroblock-padded size (replicating the last column / row). */
void orc_webp_rgb_to_yuv(const uint8_t *r, const uint8_t *g, const uint8_t *b, int w, int h, uint8_t *Y, uint8_t *U, uint8_t *V)
{
    const int mbw = (w + 15) >> 4, mbh = (h + 15) >> 4, ys = mbw * 16, cs = mbw * 8;
    for (int y = 0; y < mbh * 16; y++) for (int x = 0; x < ys; x++) {
        int sx = x < w ? x : w - 1, sy = y < h ? y : h - 1; size_t i = (size_t)sy * w + sx;
        Y[(size_t)y * ys + x] = (uint8_t)((16839 * r[i] + 33059 * g[i] + 6420 * b[i] + (1 << 15) + (16 << 16)) >> 16);
    }
    for (int y = 0; y < mbh * 8; y++) for (int x = 0; x < cs; x++) {
        int R = 0, G = 0, B = 0;
        for (int dy = 0; dy < 2; dy++) for (int dx = 0; dx < 2; dx++) {
            int sx = 2 * x + dx, sy = 2 * y + dy; if (sx > w - 1) sx = w - 1; if (sy > h - 1) sy = h - 1;
            size_t i = (size_t)sy * w + sx; R += r[i]; G += g[i]; B += b[i];
        }
        U[(size_t)y * cs + x] = (uint8_t)clip8((-9719 * R - 19081 * G + 28800 * B + (128 << 18) + (1 << 17)) >> 18);
        V[(size_t)y * cs + x] = (uint8_t)clip8((28800 * R - 24116 * G - 4684 * B + (128 << 18) + (1 << 17)) >> 18);
    }
}

/* ---- transforms ---------------------------------------------------------------------------------------------------- */
/* forward 4x4 DCT of (src - pred), libwebp FTransform */
static void fdct4(const uint8_t *src, int ss, const uint8_t *pred, int ps, int16_t out[16])
{
    int tmp[16];
    for (int i = 0; i < 4; i++, src += ss, pred += ps) {
        int d0 = src[0] - pred[0], d1 = src[1] - pred[1], d2 = src[2] - pred[2], d3 = src[3] - pred[3];
        int a0 = d0 + d3, a1 = d1 + d2, a2 = d1 - d2, a3 = d0 - d3;
        tmp[0 + i * 4] = (a0 + a1) * 8;
        tmp[1 + i * 4] = (a2 * 2217 + a3 * 5352 + 1812) >> 9;
        tmp[2 + i * 4] = (a0 - a1) * 8;
        tmp[3 + i * 4] = (a3 * 2217 - a2 * 5352 + 937) >> 9;
    }
    for (int i = 0; i < 4; i++) {
        int a0 = tmp[0 + i] + tmp[12 + i], a1 = tmp[4 + i] + tmp[8 + i], a2 = tmp[4 + i] - tmp[8 + i], a3 = tmp[0 + i] - tmp[12 + i];
        out[0 + i] = (int16_t)((a0 + a1 + 7) >> 4);
        out[4 + i] = (int16_t)(((a2 * 2217 + a3 * 5352 + 12000) >> 16) + (a3 != 0));
        out[8 + i] = (int16_t)((a0 - a1 + 7) >> 4);
        out[12 + i] = (int16_t)((a3 * 2217 - a2 * 5352 + 51000) >> 16);
    }
}
/* forward Walsh-Hadamard of the 16 luma DCs, libwebp FTransformWHT */
static void fwht(const int16_t dc[16], int16_t out[16])
{
    int tmp[16];
    for (int i = 0; i < 4; i++) {
        int a0 = dc[4 * i + 0] + dc[4 * i + 2], a1 = dc[4 * i + 1] + dc[4 * i + 3], a2 = dc[4 * i + 1] - dc[4 * i + 3], a3 = dc[4 * i + 0] - dc[4 * i + 2];
        tmp[0 + i * 4] = a0 + a1; tmp[1 + i * 4] = a3 + a2; tmp[2 + i * 4] = a3 - a2; tmp[3 + i * 4] = a0 - a1;
    }
    for (int i = 0; i < 4; i++) {
        int a0 = tmp[0 + i] + tmp[8 + i], a1 = tmp[4 + i] + tmp[12 + i], a2 = tmp[4 + i] - tmp[12 + i], a3 = tmp[0 + i] - tmp[8 + i];
        out[0 + i] = (int16_t)((a0 + a1) >> 1); out[4 + i] = (int16_t)((a3 + a2) >> 1); out[8 + i] = (int16_t)((a3 - a2) >> 1); out[12 + i] = (int16_t)((a0 - a1) >> 1);
    }
}
/* RFC 6386 14.3: inverse WHT -> the 16 luma DCs */
static void iwht(const int16_t in[16], int16_t dc[16])
{
    int tmp[16];
    for (int i = 0; i < 4; i++) {
        int a0 = in[0 + i] + in[12 + i], a1 = in[4 + i] + in[8 + i], a2 = in[4 + i] - in[8 + i], a3 = in[0 + i] - in[12 + i];
        tmp[0 + i] = a0 + a1; tmp[8 + i] = a0 - a1; tmp[4 + i] = a3 + a2; tmp[12 + i] = a3 - a2;
    }
    for (int i = 0; i < 4; i++) {
        int d = tmp[0 + i * 4] + 3, a0 = d + tmp[3 + i * 4], a1 = tmp[1 + i * 4] + tmp[2 + i * 4], a2 = tmp[1 + i * 4] - tmp[2 + i * 4], a3 = d - tmp[3 + i * 4];
        dc[4 * i + 0] = (int16_t)((a0 + a1) >> 3); dc[4 * i + 1] = (int16_t)((a3 + a2) >> 3); dc[4 * i + 2] = (int16_t)((a0 - a1) >> 3); dc[4 * i + 3] = (int16_t)((a3 - a2) >> 3);
    }
}
/* RFC 6386 14.4: inverse DCT added to the prediction, result clamped */
#define MUL1(a) ((((a) * 20091) >> 16) + (a))
#define MUL2(a) (((a) * 35468) >> 16)
static void idct4_add(const int16_t in[16], const uint8_t *pred, int ps, uint8_t *dst, int ds)
{
    int tmp[16];
    for (int i = 0; i < 4; i++) {
        int a = in[i] + in[8 + i], b = in[i] - in[8 + i];
        int c = MUL2(in[4 + i]) - MUL1(in[12 + i]), d = MUL1(in[4 + i]) + MUL2(in[12 + i]);
        tmp[4 * i + 0] = a + d; tmp[4 * i + 1] = b + c; tmp[4 * i + 2] = b - c; tmp[4 * i + 3] = a - d;
    }
    for (int i = 0; i < 4; i++) {
        int dc = tmp[i] + 4, a = dc + tmp[8 + i], b = dc - tmp[8 + i];
        int c = MUL2(tmp[4 + i]) - MUL1(tmp[12 + i]), d = MUL1(tmp[4 + i]) + MUL2(tmp[12 + i]);
        dst[i * ds + 0] = (uint8_t)clip8(pred[i * ps + 0] + ((a + d) >> 3));
        dst[i * ds + 1] = (uint8_t)clip8(pred[i * ps + 1] + ((b + c) >> 3));
        dst[i * ds + 2] = (uint8_t)clip8(pred[i * ps + 2] + ((b - c) >> 3));
        dst[i * ds + 3] = (uint8_t)clip8(pred[i * ps + 3] + ((a - d) >> 3));
    }
}

/* level = sign * min(2047, (|c| + 3q/8) / q) */
static int quantize(int c, int q)
{
    int a = c < 0 ? -c : c, l = (a + ((q * 3) >> 3)) / q;
    if (l > 2047) l = 2047;
    return c < 0 ? -l : l;
}

/* ---- intra prediction (RFC 6386 12.2/12.3); n = 16 (luma) or 8 (chroma); rec = reconstructed plane, stride s --------------- */
static void predict(const uint8_t *rec, int s, int mbx, int mby, int n, int mode, uint8_t *pred /* n x n, pitch n */)
{
    uint8_t top[16], left[16]; int tl;
    const uint8_t *p = rec + (size_t)mby * n * s + (size_t)mbx * n;
    for (int i = 0; i < n; i++) { top[i] = mby ? p[-s + i] : 127; left[i] = mbx ? p[i * s - 1] : 129; }
    tl = mby ? (mbx ? p[-s - 1] : 129) : 127;
    const int sh = n == 16 ? 4 : 3;
    for (int y = 0; y < n; y++) for (int x = 0; x < n; x++) {
        int v;
        switch (mode) {
            case M_V: v = top[x]; break;
            case M_H: v = left[y]; break;
            case M_TM: v = clip8(left[y] + top[x] - tl); break;
            default: {
                int sum = 0;
                if (mby && mbx) { for (int i = 0; i < n; i++) sum += top[i] + left[i]; v = (sum + n) >> (sh + 1); }
                else if (mby) { for (int i = 0; i < n; i++) sum += top[i]; v = (sum + (n >> 1)) >> sh; }
                else if (mbx) { for (int i = 0; i < n; i++) sum += left[i]; v = (sum + (n >> 1)) >> sh; }
                else v = 128;
            }
        }
        pred[y * n + x] = (uint8_t)v;
    }
}
static long sse(const uint8_t *src, int ss, const uint8_t *pred, int n)
{
    long e = 0;
    for (int y = 0; y < n; y++) for (int x = 0; x < n; x++) { int d = src[y * ss + x] - pred[y * n + x]; e += d * d; }
    return e;
}

/* ---- macroblock analysis + reconstruction ------------------------------------------------------------------------------ */
typedef struct { uint8_t ymode, uvmode, skip, inner /* decoder filters the inner 4x4 edges */; int16_t y2[16], y[16][16], u[4][16], v[4][16]; /* levels, ZIGZAG order */ } MbCoded;

static void code_block(const int16_t coef[16], int first, int qdc, int qac, int16_t levels_zz[16], int16_t deq[16])
{
    for (int n = 0; n < 16; n++) {
        int pos = kZig[n], l = n < first ? 0 : quantize(coef[pos], n == 0 ? qdc : qac);
        levels_zz[n] = (int16_t)l; deq[pos] = (int16_t)(l * (n == 0 ? qdc : qac));
    }
}

static void encode_mb(const uint8_t *Y, const uint8_t *U, const uint8_t *V, uint8_t *RY, uint8_t *RU, uint8_t *RV, int mbw, int mbx, int mby, const int f[6], MbCoded *mb)
{
    const int ys = mbw * 16, cs = mbw * 8;
    uint8_t pred[4][256]; int16_t coef[16][16], dcs[16], wht[16], deq[16], y2deq[16], dcrec[16];
    const uint8_t *sy = Y + (size_t)mby * 16 * ys + mbx * 16;
    /* luma mode: least squared error, first of equals in the order DC, TM, V, H */
    long best = -1; int bm = 0;
    for (int m = 0; m < 4; m++) { predict(RY, ys, mbx, mby, 16, m, pred[m]); long e = sse(sy, ys, pred[m], 16); if (best < 0 || e < best) { best = e; bm = m; } }
    mb->ymode = (uint8_t)bm;
    for (int k = 0; k < 16; k++) { fdct4(sy + (k >> 2) * 4 * ys + (k & 3) * 4, ys, pred[bm] + (k >> 2) * 64 + (k & 3) * 4, 16, coef[k]); dcs[k] = coef[k][0]; }
    fwht(dcs, wht);
    code_block(wht, 0, f[2], f[3], mb->y2, y2deq);
    iwht(y2deq, dcrec);
    int nz = 0, inner = 0;      /* inner: some block carries a non-zero coefficient AFTER the inverse WHT (what the decoder's filter looks at) */
    for (int n = 0; n < 16; n++) nz |= mb->y2[n];
    uint8_t *ry = RY + (size_t)mby * 16 * ys + mbx * 16;
    for (int k = 0; k < 16; k++) {
        code_block(coef[k], 1, f[0], f[1], mb->y[k], deq);
        deq[0] = dcrec[k];
        inner |= dcrec[k] != 0;
        for (int n = 1; n < 16; n++) nz |= mb->y[k][n];
        idct4_add(deq, pred[bm] + (k >> 2) * 64 + (k & 3) * 4, 16, ry + (k >> 2) * 4 * ys + (k & 3) * 4, ys);
    }
    /* chroma mode: U and V share it */
    const uint8_t *su = U + (size_t)mby * 8 * cs + mbx * 8, *sv = V + (size_t)mby * 8 * cs + mbx * 8;
    uint8_t pu[4][64], pv[4][64];
    best = -1; bm = 0;
    for (int m = 0; m < 4; m++) {
        predict(RU, cs, mbx, mby, 8, m, pu[m]); predict(RV, cs, mbx, mby, 8, m, pv[m]);
        long e = sse(su, cs, pu[m], 8) + sse(sv, cs, pv[m], 8);
        if (best < 0 || e < best) { best = e; bm = m; }
    }
    mb->uvmode = (uint8_t)bm;
    uint8_t *ru = RU + (size_t)mby * 8 * cs + mbx * 8, *rv = RV + (size_t)mby * 8 * cs + mbx * 8;
    for (int k = 0; k < 4; k++) {
        int16_t c[16]; const int o = (k >> 1) * 4 * cs + (k & 1) * 4, po = (k >> 1) * 32 + (k & 1) * 4;
        fdct4(su + o, cs, pu[bm] + po, 8, c); code_block(c, 0, f[4], f[5], mb->u[k], deq);
        for (int n = 0; n < 16; n++) nz |= mb->u[k][n];
        idct4_add(deq, pu[bm] + po, 8, ru + o, cs);
        fdct4(sv + o, cs, pv[bm] + po, 8, c); code_block(c, 0, f[4], f[5], mb->v[k], deq);
        for (int n = 0; n < 16; n++) nz |= mb->v[k][n];
        idct4_add(deq, pv[bm] + po, 8, rv + o, cs);
    }
    mb->skip = nz == 0;
    {   /* Y2 levels alone do not make an inner edge: only what reaches the 4x4 blocks counts */
        int ac_or_uv = 0;
        for (int k = 0; k < 16; k++) for (int n = 1; n < 16; n++) ac_or_uv |= mb->y[k][n];
        for (int k = 0; k < 4; k++) for (int n = 0; n < 16; n++) ac_or_uv |= mb->u[k][n] | mb->v[k][n];
        mb->inner = (uint8_t)(inner || ac_or_uv);
    }
}

/* ---- RFC 6386 15.2: the decoder's SIMPLE loop filter (luma only), macroblocks in raster order, in place.  The encoder never
 *      looks at filtered samples (intra prediction uses the unfiltered reconstruction); this is here so that the tests know what
 *      a decoder must output. */
static int sclip(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }
static void simple_edge(uint8_t *p, int step, int thresh)
{
    const int p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step];
    if (4 * abs(p0 - q0) + abs(p1 - q1) > 2 * thresh + 1) return;
    const int a = 3 * (q0 - p0) + sclip(p1 - q1, -128, 127);
    const int a1 = sclip((a + 4) >> 3, -16, 15), a2 = sclip((a + 3) >> 3, -16, 15);
    p[-step] = (uint8_t)clip8(p0 + a2); p[0] = (uint8_t)clip8(q0 - a1);
}
static void loop_filter_simple(uint8_t *Yp, int mbw, int mbh, int level, const MbCoded *mbs)
{
    if (level <= 0) return;
    const int ys = mbw * 16, limit = 2 * level + (level < 1 ? 1 : level);      /* sharpness 0: interior level = level */
    for (int my = 0; my < mbh; my++) for (int mx = 0; mx < mbw; mx++) {
        uint8_t *p = Yp + (size_t)my * 16 * ys + mx * 16;
        const int inner = mbs[my * mbw + mx].inner;
        if (mx > 0) for (int i = 0; i < 16; i++) simple_edge(p + i * ys, 1, limit + 4);
        if (inner) for (int e = 4; e < 16; e += 4) for (int i = 0; i < 16; i++) simple_edge(p + i * ys + e, 1, limit);
        if (my > 0) for (int i = 0; i < 16; i++) simple_edge(p + i, ys, limit + 4);
        if (inner) for (int e = 4; e < 16; e += 4) for (int i = 0; i < 16; i++) simple_edge(p + e * ys + i, ys, limit);
    }
}

/* loop filter strength this encoder asks the decoder for: none at the finest quantisers, rising with the step size */
int orc_vp8_filter_level(int qindex) { int l = qindex / 2; return l > 63 ? 63 : l; }

/* ---- RFC 6386 section 7: the boolean entropy encoder ---------------------------------------------------------------------- */
typedef struct { uint8_t *buf; size_t n, cap; uint32_t range, bottom; int bit_count; } Bool;
static void bool_init(Bool *e) { e->buf = NULL; e->n = e->cap = 0; e->range = 255; e->bottom = 0; e->bit_count = 24; }
static void bool_byte(Bool *e, uint8_t v) { if (e->n == e->cap) { e->cap = e->cap ? e->cap * 2 : 4096; e->buf = (uint8_t *)realloc(e->buf, e->cap); } e->buf[e->n++] = v; }
static void bool_carry(Bool *e) { size_t i = e->n; while (i > 0 && e->buf[i - 1] == 255) e->buf[--i] = 0; if (i > 0) e->buf[i - 1]++; }
static int bool_put(Bool *e, int bit, int prob)
{
    uint32_t split = 1 + (((e->range - 1) * (uint32_t)prob) >> 8);
    if (bit) { e->bottom += split; e->range -= split; }
    else e->range = split;
    while (e->range < 128) {
        e->range <<= 1;
        if (e->bottom & 0x80000000u) bool_carry(e);
        e->bottom <<= 1;
        if (!--e->bit_count) { bool_byte(e, (uint8_t)(e->bottom >> 24)); e->bottom &= 0xFFFFFFu; e->bit_count = 8; }
    }
    return bit;
}
static void bool_bits(Bool *e, int v, int n) { for (int i = n - 1; i >= 0; i--) bool_put(e, (v >> i) & 1, 128); }
static void bool_flush(Bool *e)
{
    int c = e->bit_count; uint32_t v = e->bottom;
    if (v & (1u << (32 - c))) bool_carry(e);
    v <<= c & 7; c >>= 3;
    while (--c >= 0) v <<= 8;
    for (c = 0; c < 4; c++) { bool_byte(e, (uint8_t)(v >> 24)); v <<= 8; }
}

/* ---- RFC 6386 13: token coding of one block; returns 1 if anything but an immediate end-of-block was coded.
 *      The same walk either writes bits (k->e set) or only counts the 0/1 decisions per probability slot (k->stats set):
 *      the counting pass feeds the probability update below. */
typedef struct { Bool *e; uint32_t *stats /* [1056][2] */; const uint8_t *probs /* [1056] */; } Coder;
static int node(Coder *k, int slot, int bit)
{
    if (k->stats) k->stats[2 * slot + (bit ? 1 : 0)]++;
    else bool_put(k->e, bit, k->probs[slot]);
    return bit;
}
static void fixed(Coder *k, int bit, int prob) { if (!k->stats) bool_put(k->e, bit, prob); }

static int put_coeffs(Coder *k, const int16_t lv[16], int type, int first, int ctx)
{
    static const uint8_t cat3[] = {173, 148, 140}, cat4[] = {176, 155, 140, 135}, cat5[] = {180, 157, 141, 134, 130}, cat6[] = {254, 254, 243, 230, 196, 177, 153, 140, 133, 130, 129};
    int last = -1, n = first;
    for (int i = first; i < 16; i++) if (lv[i]) last = i;
    int p = ((type * 8 + kBand[n]) * 3 + ctx) * 11;                 /* slot of node 0 for the current (band, context) */
    if (!node(k, p + 0, last >= 0)) return 0;
    while (n < 16) {
        int c = lv[n++], sign = c < 0, v = sign ? -c : c;
        const int base = (type * 8 + kBand[n]) * 3 * 11;
        if (!node(k, p + 1, v != 0)) { p = base; continue; }
        if (!node(k, p + 2, v > 1)) p = base + 11;
        else {
            if (!node(k, p + 3, v > 4)) { if (node(k, p + 4, v != 2)) node(k, p + 5, v == 4); }
            else if (!node(k, p + 6, v > 10)) {
                if (!node(k, p + 7, v > 6)) fixed(k, v == 6, 159);
                else { fixed(k, v >= 9, 165); fixed(k, !(v & 1), 145); }
            } else {
                const uint8_t *tab; int nb, residue;
                if (v < 19) { node(k, p + 8, 0); node(k, p + 9, 0); residue = v - 11; nb = 3; tab = cat3; }
                else if (v < 35) { node(k, p + 8, 0); node(k, p + 9, 1); residue = v - 19; nb = 4; tab = cat4; }
                else if (v < 67) { node(k, p + 8, 1); node(k, p + 10, 0); residue = v - 35; nb = 5; tab = cat5; }
                else { node(k, p + 8, 1); node(k, p + 10, 1); residue = v - 67; nb = 11; tab = cat6; }
                for (int i = nb - 1; i >= 0; i--) fixed(k, (residue >> i) & 1, *tab++);
            }
            p = base + 22;
        }
        fixed(k, sign, 128);
        if (n == 16 || !node(k, p + 0, n <= last)) return 1;
    }
    return 1;
}

/* all residual tokens of the frame in coding order, through `k` */
static void code_frame_tokens(Coder *k, const MbCoded *mbs, int mbw, int mbh, int use_skip)
{
    uint8_t *top_nz = (uint8_t *)calloc((size_t)mbw, 9), left_nz[9];
    for (int mby = 0; mby < mbh; mby++) {
        memset(left_nz, 0, 9);
        for (int mbx = 0; mbx < mbw; mbx++) {
            const MbCoded *m = &mbs[mby * mbw + mbx];
            uint8_t *t = top_nz + (size_t)mbx * 9, *l = left_nz;
            if (use_skip && m->skip) { memset(t, 0, 9); memset(l, 0, 9); continue; }
            t[8] = l[8] = (uint8_t)put_coeffs(k, m->y2, 1, 0, t[8] + l[8]);
            for (int y = 0; y < 4; y++) for (int x = 0; x < 4; x++) t[x] = l[y] = (uint8_t)put_coeffs(k, m->y[y * 4 + x], 0, 1, t[x] + l[y]);
            for (int y = 0; y < 2; y++) for (int x = 0; x < 2; x++) t[4 + x] = l[4 + y] = (uint8_t)put_coeffs(k, m->u[y * 2 + x], 2, 0, t[4 + x] + l[4 + y]);
            for (int y = 0; y < 2; y++) for (int x = 0; x < 2; x++) t[6 + x] = l[6 + y] = (uint8_t)put_coeffs(k, m->v[y * 2 + x], 2, 0, t[6 + x] + l[6 + y]);
        }
    }
    free(top_nz);
}

/* cost of coding one decision with probability-of-zero p/256, in 1/256 bit */
static int bit_cost(int p) { return p <= 0 ? 1 << 20 : (int)(-log2(p / 256.0) * 256.0 + 0.5); }

/* RFC 6386 13.4: per slot, replace the default probability by the frame's own estimate when that pays for the 8-bit update
 * (libwebp's estimate: 255 - ones * 255 / total).  probs[] in: defaults, out: the table the tokens are coded with. */
static void choose_probs(const uint32_t *stats, uint8_t *probs, uint8_t *updated)
{
    for (int i = 0; i < 4 * 8 * 3 * 11; i++) {
        const uint64_t c0 = stats[2 * i], c1 = stats[2 * i + 1], total = c0 + c1;
        const int oldp = probs[i], u = ORC_VP8_COEF_UPDATE_PROBS[i];
        updated[i] = 0;
        if (!total) continue;
        int newp = 255 - (int)(c1 * 255 / total); if (newp < 1) newp = 1;
        const uint64_t old_cost = c0 * bit_cost(oldp) + c1 * bit_cost(256 - oldp) + bit_cost(u);
        const uint64_t new_cost = c0 * bit_cost(newp) + c1 * bit_cost(256 - newp) + bit_cost(256 - u) + 8 * 256;
        if (newp != oldp && new_cost < old_cost) { probs[i] = (uint8_t)newp; updated[i] = 1; }
    }
}

/* Stage view for the parity tests: per macroblock the 25 x 16 quantised levels (Y2, 16 Y, 4 U, 4 V; zigzag order) and
 * {ymode, uvmode, skip, 0} -- the exact layout the product's K8 kernel hands to its host writer. */
int orc_webp_analyze(const uint8_t *r, const uint8_t *g, const uint8_t *b, int w, int h, int quality, int16_t *levels, uint8_t *modes)
{
    if (w < 1 || h < 1 || w > 16383 || h > 16383) return -1;
    const int mbw = (w + 15) >> 4, mbh = (h + 15) >> 4, ys = mbw * 16, cs = mbw * 8;
    const size_t ny = (size_t)ys * mbh * 16, nc = (size_t)cs * mbh * 8;
    uint8_t *Y = (uint8_t *)malloc(ny), *U = (uint8_t *)malloc(nc), *V = (uint8_t *)malloc(nc);
    uint8_t *RY = (uint8_t *)calloc(ny, 1), *RU = (uint8_t *)calloc(nc, 1), *RV = (uint8_t *)calloc(nc, 1);
    orc_webp_rgb_to_yuv(r, g, b, w, h, Y, U, V);
    int f[6]; orc_vp8_quant_factors(orc_vp8_qindex(quality), f);
    for (int mby = 0; mby < mbh; mby++) for (int mbx = 0; mbx < mbw; mbx++) {
        MbCoded m; encode_mb(Y, U, V, RY, RU, RV, mbw, mbx, mby, f, &m);
        int16_t *lv = levels + ((size_t)mby * mbw + mbx) * 400; uint8_t *md = modes + ((size_t)mby * mbw + mbx) * 4;
        memcpy(lv, m.y2, 32);
        for (int k = 0; k < 16; k++) memcpy(lv + 16 * (1 + k), m.y[k], 32);
        for (int k = 0; k < 4; k++) { memcpy(lv + 16 * (17 + k), m.u[k], 32); memcpy(lv + 16 * (21 + k), m.v[k], 32); }
        md[0] = m.ymode; md[1] = m.uvmode; md[2] = m.skip; md[3] = 0;
    }
    free(Y); free(U); free(V); free(RY); free(RU); free(RV);
    return 0;
}

/* ---- the encoder ------------------------------------------------------------------------------------------------------------ */
/* RGB planes -> a complete .webp file (simple format: RIFF + one 'VP8 ' chunk).  Optional recon_* receive the encoder's own
 * reconstruction at macroblock-padded size; a conforming decoder must reproduce it exactly. */
int orc_webp_encode(const uint8_t *r, const uint8_t *g, const uint8_t *b, int w, int h, int quality,
                    uint8_t **out, size_t *out_len, uint8_t *recon_y, uint8_t *recon_u, uint8_t *recon_v)
{
    if (w < 1 || h < 1 || w > 16383 || h > 16383) return -1;
    const int mbw = (w + 15) >> 4, mbh = (h + 15) >> 4, nmb = mbw * mbh, ys = mbw * 16, cs = mbw * 8;
    const size_t ny = (size_t)ys * mbh * 16, nc = (size_t)cs * mbh * 8;
    uint8_t *Y = (uint8_t *)malloc(ny), *U = (uint8_t *)malloc(nc), *V = (uint8_t *)malloc(nc);
    uint8_t *RY = (uint8_t *)calloc(ny, 1), *RU = (uint8_t *)calloc(nc, 1), *RV = (uint8_t *)calloc(nc, 1);
    MbCoded *mbs = (MbCoded *)malloc(sizeof(MbCoded) * (size_t)nmb);
    orc_webp_rgb_to_yuv(r, g, b, w, h, Y, U, V);
    const int q = orc_vp8_qindex(quality);
    const int flevel = orc_vp8_filter_level(q);
    int f[6]; orc_vp8_quant_factors(q, f);
    int nskip = 0;
    for (int mby = 0; mby < mbh; mby++) for (int mbx = 0; mbx < mbw; mbx++) { encode_mb(Y, U, V, RY, RU, RV, mbw, mbx, mby, f, &mbs[mby * mbw + mbx]); nskip += mbs[mby * mbw + mbx].skip; }
    /* ---- first partition: frame header + per-macroblock modes */
    Bool h0, tk; bool_init(&h0); bool_init(&tk);
    const int use_skip = nskip > 0;
    /* counting pass over the tokens -> which default probabilities are worth replacing */
    uint8_t probs[4 * 8 * 3 * 11], updated[4 * 8 * 3 * 11];
    memcpy(probs, ORC_VP8_COEF_PROBS, sizeof(probs));
    {
        uint32_t *stats = (uint32_t *)calloc(4 * 8 * 3 * 11 * 2, sizeof(uint32_t));
        Coder k = {NULL, stats, probs};
        code_frame_tokens(&k, mbs, mbw, mbh, use_skip);
        choose_probs(stats, probs, updated);
        free(stats);
    }
    int skip_p = (int)(((long)(nmb - nskip) * 255) / nmb); if (skip_p < 1) skip_p = 1; if (skip_p > 255) skip_p = 255;
    bool_bits(&h0, 0, 1);             /* color_space */
    bool_bits(&h0, 0, 1);             /* clamping_type: clamping needed */
    bool_bits(&h0, 0, 1);             /* segmentation_enabled */
    bool_bits(&h0, 1, 1);             /* filter_type: simple */
    bool_bits(&h0, flevel, 6);        /* loop_filter_level */
    bool_bits(&h0, 0, 3);             /* sharpness_level */
    bool_bits(&h0, 0, 1);             /* loop_filter_adj_enable */
    bool_bits(&h0, 0, 2);             /* log2_nbr_of_dct_partitions */
    bool_bits(&h0, q, 7);             /* y_ac_qi */
    for (int i = 0; i < 5; i++) bool_bits(&h0, 0, 1);   /* y_dc, y2_dc, y2_ac, uv_dc, uv_ac deltas absent */
    bool_bits(&h0, 0, 1);             /* refresh_entropy_probs */
    for (int i = 0; i < 4 * 8 * 3 * 11; i++) {                                                /* token probability updates */
        if (bool_put(&h0, updated[i], ORC_VP8_COEF_UPDATE_PROBS[i])) bool_bits(&h0, probs[i], 8);
    }
    bool_bits(&h0, use_skip, 1);      /* mb_no_coeff_skip */
    if (use_skip) bool_bits(&h0, skip_p, 8);
    for (int i = 0; i < nmb; i++) {
        const MbCoded *m = &mbs[i];
        if (use_skip) bool_put(&h0, m->skip, skip_p);
        bool_put(&h0, 1, 145);                                                              /* not B_PRED */
        if (bool_put(&h0, m->ymode == M_TM || m->ymode == M_H, 156)) bool_put(&h0, m->ymode == M_TM, 128);
        else bool_put(&h0, m->ymode == M_V, 163);
        if (bool_put(&h0, m->uvmode != M_DC, 142)) if (bool_put(&h0, m->uvmode != M_V, 114)) bool_put(&h0, m->uvmode != M_H, 183);
    }
    bool_flush(&h0);
    /* ---- token partition */
    { Coder k = {&tk, NULL, probs}; code_frame_tokens(&k, mbs, mbw, mbh, use_skip); }
    bool_flush(&tk);
    /* ---- container */
    const size_t vp8_size = 10 + h0.n + tk.n, riff_payload = 4 + 8 + vp8_size + (vp8_size & 1);
    uint8_t *o = (uint8_t *)malloc(8 + riff_payload), *p = o;
    memcpy(p, "RIFF", 4); p += 4;
    *p++ = (uint8_t)riff_payload; *p++ = (uint8_t)(riff_payload >> 8); *p++ = (uint8_t)(riff_payload >> 16); *p++ = (uint8_t)(riff_payload >> 24);
    memcpy(p, "WEBPVP8 ", 8); p += 8;
    *p++ = (uint8_t)vp8_size; *p++ = (uint8_t)(vp8_size >> 8); *p++ = (uint8_t)(vp8_size >> 16); *p++ = (uint8_t)(vp8_size >> 24);
    const uint32_t tag = 0u | (0u << 1) | (1u << 4) | ((uint32_t)h0.n << 5);     /* key frame, version 0, show_frame, first partition size */
    *p++ = (uint8_t)tag; *p++ = (uint8_t)(tag >> 8); *p++ = (uint8_t)(tag >> 16);
    *p++ = 0x9d; *p++ = 0x01; *p++ = 0x2a;
    *p++ = (uint8_t)w; *p++ = (uint8_t)(w >> 8); *p++ = (uint8_t)h; *p++ = (uint8_t)(h >> 8);
    memcpy(p, h0.buf, h0.n); p += h0.n; memcpy(p, tk.buf, tk.n); p += tk.n;
    if (vp8_size & 1) *p++ = 0;
    *out = o; *out_len = (size_t)(p - o);
    if (recon_y) { loop_filter_simple(RY, mbw, mbh, flevel, mbs); memcpy(recon_y, RY, ny); }      /* what a decoder shows */
    if (recon_u) memcpy(recon_u, RU, nc);
    if (recon_v) memcpy(recon_v, RV, nc);
    free(Y); free(U); free(V); free(RY); free(RU); free(RV); free(mbs); free(h0.buf); free(tk.buf);
    return h0.n >= (1u << 19) ? -2 : 0;
}
