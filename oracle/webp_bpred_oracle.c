/* webp_bpred_oracle.c -- TEST INFRASTRUCTURE ONLY (never linked into or called by the product).
 *
 * Scalar twin of the lossy WebP encoder with 4x4 intra prediction (B_PRED) switched on (k_vp8_encode_bpred + the host writer).  It
 * shares the rules of vp8_bpred_core.h (predictors, edges, rates, mode costs, lambda) and restates everything else: the 16x16 arm
 * and chroma of oracle/webp_oracle.c, every sub-block coded in raster order, and the token and mode partitions with the decoder's
 * own running contexts (the Y2 flag updated on 16x16 macroblocks only), not the device's carried masks.
 * Files made here must decode in libwebp and in the project's decoder to exactly this encoder's reconstruction
 * (tests/test_webp_bpred_host.py).  Plain scalar C, macroblock by macroblock in raster order. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "vp8_tables_oracle.h"
#include "../caesium-clt_b200/csrc/vp8_bpred_core.h"

int orc_vp8_qindex(int quality);
void orc_vp8_quant_factors(int q, int f[6]);
void orc_webp_rgb_to_yuv(const uint8_t *r, const uint8_t *g, const uint8_t *b, int w, int h, uint8_t *Y, uint8_t *U, uint8_t *V);
int orc_vp8_filter_level(int qindex);

static const uint8_t kZig[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};
static const uint8_t kBand[17] = {0, 1, 2, 3, 6, 4, 5, 6, 6, 6, 6, 6, 6, 6, 6, 7, 0};
static int clip8(int v) { return v < 0 ? 0 : v > 255 ? 255 : v; }

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
static int quantize(int c, int q)
{
    int a = c < 0 ? -c : c, l = (a + ((q * 3) >> 3)) / q;
    if (l > 2047) l = 2047;
    return c < 0 ? -l : l;
}
static void code_block(const int16_t coef[16], int first, int qdc, int qac, int16_t levels_zz[16], int16_t deq[16])
{
    for (int n = 0; n < 16; n++) {
        int pos = kZig[n], l = n < first ? 0 : quantize(coef[pos], n == 0 ? qdc : qac);
        levels_zz[n] = (int16_t)l; deq[pos] = (int16_t)(l * (n == 0 ? qdc : qac));
    }
}
/* 16x16 / 8x8 prediction (RFC 6386 12.2) */
static void predict(const uint8_t *rec, int s, int mbx, int mby, int n, int mode, uint8_t *pred)
{
    uint8_t top[16], left[16]; int tl;
    const uint8_t *p = rec + (size_t)mby * n * s + (size_t)mbx * n;
    for (int i = 0; i < n; i++) { top[i] = mby ? p[-s + i] : 127; left[i] = mbx ? p[i * s - 1] : 129; }
    tl = mby ? (mbx ? p[-s - 1] : 129) : 127;
    const int sh = n == 16 ? 4 : 3;
    for (int y = 0; y < n; y++) for (int x = 0; x < n; x++) {
        int v, sum = 0;
        switch (mode) {
            case 2: v = top[x]; break;
            case 3: v = left[y]; break;
            case 1: v = clip8(left[y] + top[x] - tl); break;
            default:
                if (mby && mbx) { for (int i = 0; i < n; i++) sum += top[i] + left[i]; v = (sum + n) >> (sh + 1); }
                else if (mby) { for (int i = 0; i < n; i++) sum += top[i]; v = (sum + (n >> 1)) >> sh; }
                else if (mbx) { for (int i = 0; i < n; i++) sum += left[i]; v = (sum + (n >> 1)) >> sh; }
                else v = 128;
        }
        pred[y * n + x] = (uint8_t)v;
    }
}
static uint32_t sse(const uint8_t *a, int as, const uint8_t *b, int bs, int w, int h)
{
    uint32_t e = 0;
    for (int y = 0; y < h; y++) for (int x = 0; x < w; x++) { int d = a[y * as + x] - b[y * bs + x]; e += (uint32_t)(d * d); }
    return e;
}

typedef struct { uint8_t ymode, uvmode, skip, inner, bmodes[16]; int16_t y2[16], y[16][16], u[4][16], v[4][16]; } MbCoded;

/* one macroblock: both luma arms, the rate-distortion choice, chroma */
static void encode_mb(const uint8_t *Y, const uint8_t *U, const uint8_t *V, uint8_t *RY, uint8_t *RU, uint8_t *RV, int mbw, int mbx, int mby,
                      const int f[6], const uint8_t *above_modes /* 4 */, const uint8_t *left_modes /* 4 */, MbCoded *mb)
{
    const int ys = mbw * 16, cs = mbw * 8, lam = vp8bp_lambda(f[1]);
    const uint8_t *sy = Y + (size_t)mby * 16 * ys + mbx * 16;
    uint8_t *ry = RY + (size_t)mby * 16 * ys + mbx * 16;
    /* ---- 16x16 arm */
    uint8_t pred[4][256], rec16[256];
    int16_t coef[16][16], dcs[16], wht[16], deq[16], y2deq[16], dcrec[16], y2[16], y16[16][16];
    uint32_t best = 0; int bm = 0;
    for (int m = 0; m < 4; m++) { predict(RY, ys, mbx, mby, 16, m, pred[m]); uint32_t e = sse(sy, ys, pred[m], 16, 16, 16); if (m == 0 || e < best) { best = e; bm = m; } }
    for (int k = 0; k < 16; k++) { fdct4(sy + (k >> 2) * 4 * ys + (k & 3) * 4, ys, pred[bm] + (k >> 2) * 64 + (k & 3) * 4, 16, coef[k]); dcs[k] = coef[k][0]; }
    fwht(dcs, wht);
    code_block(wht, 0, f[2], f[3], y2, y2deq);
    iwht(y2deq, dcrec);
    int nz16 = 0, inner16 = 0, dummy;
    for (int n = 0; n < 16; n++) nz16 |= y2[n];
    uint32_t rate16 = vp8bp_block_rate(y2, 1, 0, 0, &dummy) + vp8bp_i16_cost(bm);
    int acnz[16];
    for (int k = 0; k < 16; k++) {
        code_block(coef[k], 1, f[0], f[1], y16[k], deq);
        deq[0] = dcrec[k];
        inner16 |= dcrec[k] != 0;
        for (int n = 1; n < 16; n++) nz16 |= y16[k][n], inner16 |= y16[k][n];
        idct4_add(deq, pred[bm] + (k >> 2) * 64 + (k & 3) * 4, 16, rec16 + (k >> 2) * 64 + (k & 3) * 4, 16);
        const int x = k & 3, yy = k >> 2;
        rate16 += vp8bp_block_rate(y16[k], 0, 1, (yy ? acnz[k - 4] : 0) + (x ? acnz[k - 1] : 0), &acnz[k]);
    }
    const uint64_t score16 = vp8bp_score(sse(sy, ys, rec16, 16, 16, 16), rate16, lam);
    /* ---- B_PRED arm, sub-blocks in raster order */
    uint8_t top[21], left[16], rec4[256], modes4[16];
    int16_t y4[16][16];
    int nz4[16];
    uint64_t sum4 = (uint64_t)lam * vp8bp_bit(0, VP8BP_FLAG_PROB);
    vp8bp_mb_border(RY, ys, mbx, mby, mbw, top, left);
    for (int k = 0; k < 16; k++) {
        const int x = k & 3, yy = k >> 2;
        const uint8_t *sb = sy + yy * 4 * ys + x * 4;
        uint8_t e[13];
        vp8bp_edges(top, left, rec4, 16, x, yy, e);
        const int ctx = (yy ? nz4[k - 4] : 0) + (x ? nz4[k - 1] : 0);
        const int am = yy ? modes4[k - 4] : above_modes[x], lm = x ? modes4[k - 1] : left_modes[yy];
        uint64_t bs = 0;
        for (int m = 0; m < VP8BP_NMODES; m++) {
            uint8_t p[16], r[16]; int16_t c[16], lv[16], dq[16]; int nz;
            vp8bp_pred4(m, e, p);
            fdct4(sb, ys, p, 4, c);
            code_block(c, 0, f[0], f[1], lv, dq);
            idct4_add(dq, p, 4, r, 4);
            const uint64_t s = vp8bp_score(sse(sb, ys, r, 4, 4, 4), vp8bp_block_rate(lv, 3, 0, ctx, &nz) + vp8bp_bmode_cost(am, lm, m), lam);
            if (m == 0 || s < bs) {
                bs = s; modes4[k] = (uint8_t)m; nz4[k] = nz; memcpy(y4[k], lv, sizeof(lv));
                for (int j = 0; j < 4; j++) memcpy(rec4 + (yy * 4 + j) * 16 + x * 4, r + 4 * j, 4);
            }
        }
        sum4 += bs;
    }
    const int bp = sum4 < score16;
    int nz = 0;
    if (bp) {
        mb->ymode = VP8BP_YMODE; memset(mb->y2, 0, sizeof(mb->y2)); memcpy(mb->y, y4, sizeof(y4)); memcpy(mb->bmodes, modes4, 16);
        for (int k = 0; k < 16; k++) for (int n = 0; n < 16; n++) nz |= y4[k][n];
        for (int j = 0; j < 16; j++) memcpy(ry + j * ys, rec4 + j * 16, 16);
    } else {
        mb->ymode = (uint8_t)bm; memcpy(mb->y2, y2, sizeof(y2)); memcpy(mb->y, y16, sizeof(y16)); memset(mb->bmodes, bm, 16);
        nz = nz16;
        for (int j = 0; j < 16; j++) memcpy(ry + j * ys, rec16 + j * 16, 16);
    }
    /* ---- chroma */
    const uint8_t *su = U + (size_t)mby * 8 * cs + mbx * 8, *sv = V + (size_t)mby * 8 * cs + mbx * 8;
    uint8_t pu[4][64], pv[4][64];
    best = 0; bm = 0;
    for (int m = 0; m < 4; m++) {
        predict(RU, cs, mbx, mby, 8, m, pu[m]); predict(RV, cs, mbx, mby, 8, m, pv[m]);
        uint32_t e = sse(su, cs, pu[m], 8, 8, 8) + sse(sv, cs, pv[m], 8, 8, 8);
        if (m == 0 || e < best) { best = e; bm = m; }
    }
    mb->uvmode = (uint8_t)bm;
    int uvnz = 0;
    uint8_t *ru = RU + (size_t)mby * 8 * cs + mbx * 8, *rv = RV + (size_t)mby * 8 * cs + mbx * 8;
    for (int k = 0; k < 4; k++) {
        int16_t c[16]; const int o = (k >> 1) * 4 * cs + (k & 1) * 4, po = (k >> 1) * 32 + (k & 1) * 4;
        fdct4(su + o, cs, pu[bm] + po, 8, c); code_block(c, 0, f[4], f[5], mb->u[k], deq);
        idct4_add(deq, pu[bm] + po, 8, ru + o, cs);
        fdct4(sv + o, cs, pv[bm] + po, 8, c); code_block(c, 0, f[4], f[5], mb->v[k], deq);
        idct4_add(deq, pv[bm] + po, 8, rv + o, cs);
        for (int n = 0; n < 16; n++) uvnz |= mb->u[k][n] | mb->v[k][n];
    }
    mb->skip = (nz | uvnz) == 0;
    mb->inner = (uint8_t)(bp || inner16 || uvnz);      /* the decoder always filters a B_PRED macroblock's inner edges */
}

/* ---- the decoder's simple loop filter (luma), as in webp_oracle.c */
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
    const int ys = mbw * 16, limit = 2 * level + level;
    for (int my = 0; my < mbh; my++) for (int mx = 0; mx < mbw; mx++) {
        uint8_t *p = Yp + (size_t)my * 16 * ys + mx * 16;
        const int inner = mbs[my * mbw + mx].inner;
        if (mx > 0) for (int i = 0; i < 16; i++) simple_edge(p + i * ys, 1, limit + 4);
        if (inner) for (int e = 4; e < 16; e += 4) for (int i = 0; i < 16; i++) simple_edge(p + i * ys + e, 1, limit);
        if (my > 0) for (int i = 0; i < 16; i++) simple_edge(p + i, ys, limit + 4);
        if (inner) for (int e = 4; e < 16; e += 4) for (int i = 0; i < 16; i++) simple_edge(p + e * ys + i, ys, limit);
    }
}

/* ---- boolean encoder (RFC 6386 section 7) */
typedef struct { uint8_t *buf; size_t n, cap; uint32_t range, bottom; int bit_count; } Bool;
static void bool_init(Bool *e) { e->buf = NULL; e->n = e->cap = 0; e->range = 255; e->bottom = 0; e->bit_count = 24; }
static void bool_byte(Bool *e, uint8_t v) { if (e->n == e->cap) { e->cap = e->cap ? e->cap * 2 : 4096; e->buf = (uint8_t *)realloc(e->buf, e->cap); } e->buf[e->n++] = v; }
static void bool_carry(Bool *e) { size_t i = e->n; while (i > 0 && e->buf[i - 1] == 255) e->buf[--i] = 0; if (i > 0) e->buf[i - 1]++; }
static int bool_put(Bool *e, int bit, int prob)
{
    uint32_t split = 1 + (((e->range - 1) * (uint32_t)prob) >> 8);
    if (bit) { e->bottom += split; e->range -= split; } else e->range = split;
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

/* ---- tokens: counting or writing, with the decoder's running contexts */
typedef struct { Bool *e; uint32_t *stats; const uint8_t *probs; } Coder;
static int node(Coder *k, int slot, int bit) { if (k->stats) k->stats[2 * slot + (bit ? 1 : 0)]++; else bool_put(k->e, bit, k->probs[slot]); return bit; }
static void fixed(Coder *k, int bit, int prob) { if (!k->stats) bool_put(k->e, bit, prob); }
static int put_coeffs(Coder *k, const int16_t lv[16], int type, int first, int ctx)
{
    static const uint8_t cat3[] = {173, 148, 140}, cat4[] = {176, 155, 140, 135}, cat5[] = {180, 157, 141, 134, 130}, cat6[] = {254, 254, 243, 230, 196, 177, 153, 140, 133, 130, 129};
    int last = -1, n = first;
    for (int i = first; i < 16; i++) if (lv[i]) last = i;
    int p = ((type * 8 + kBand[n]) * 3 + ctx) * 11;
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
/* t[8] / l[8] is the decoder's Y2 flag: written by 16x16 macroblocks only (a skipped one clears it), left alone by B_PRED ones */
static void code_frame_tokens(Coder *k, const MbCoded *mbs, int mbw, int mbh, int use_skip)
{
    uint8_t *top_nz = (uint8_t *)calloc((size_t)mbw, 9), left_nz[9];
    for (int mby = 0; mby < mbh; mby++) {
        memset(left_nz, 0, 9);
        for (int mbx = 0; mbx < mbw; mbx++) {
            const MbCoded *m = &mbs[mby * mbw + mbx];
            const int bp = m->ymode == VP8BP_YMODE;
            uint8_t *t = top_nz + (size_t)mbx * 9, *l = left_nz;
            if (use_skip && m->skip) { memset(t, 0, 8); memset(l, 0, 8); if (!bp) t[8] = l[8] = 0; continue; }
            if (!bp) t[8] = l[8] = (uint8_t)put_coeffs(k, m->y2, 1, 0, t[8] + l[8]);
            for (int y = 0; y < 4; y++) for (int x = 0; x < 4; x++) t[x] = l[y] = (uint8_t)put_coeffs(k, m->y[y * 4 + x], bp ? 3 : 0, bp ? 0 : 1, t[x] + l[y]);
            for (int y = 0; y < 2; y++) for (int x = 0; x < 2; x++) t[4 + x] = l[4 + y] = (uint8_t)put_coeffs(k, m->u[y * 2 + x], 2, 0, t[4 + x] + l[4 + y]);
            for (int y = 0; y < 2; y++) for (int x = 0; x < 2; x++) t[6 + x] = l[6 + y] = (uint8_t)put_coeffs(k, m->v[y * 2 + x], 2, 0, t[6 + x] + l[6 + y]);
        }
    }
    free(top_nz);
}
static int bit_cost_f(int p) { return p <= 0 ? 1 << 20 : (int)(-log2(p / 256.0) * 256.0 + 0.5); }
static void choose_probs(const uint32_t *stats, uint8_t *probs, uint8_t *updated)
{   /* the rule of webp_oracle.c */
    for (int i = 0; i < 4 * 8 * 3 * 11; i++) {
        const uint64_t c0 = stats[2 * i], c1 = stats[2 * i + 1], total = c0 + c1;
        const int oldp = probs[i], u = ORC_VP8_COEF_UPDATE_PROBS[i];
        updated[i] = 0;
        if (!total) continue;
        int newp = 255 - (int)(c1 * 255 / total); if (newp < 1) newp = 1;
        const uint64_t old_cost = c0 * bit_cost_f(oldp) + c1 * bit_cost_f(256 - oldp) + bit_cost_f(u);
        const uint64_t new_cost = c0 * bit_cost_f(newp) + c1 * bit_cost_f(256 - newp) + bit_cost_f(256 - u) + 8 * 256;
        if (newp != oldp && new_cost < old_cost) { probs[i] = (uint8_t)newp; updated[i] = 1; }
    }
}

/* RGB planes -> .webp file with B_PRED.  Optional stage outputs: levels [nmb][25][16], modes [nmb][4], bmodes [nmb][16], and the
 * reconstruction a decoder shows (Y after the loop filter, U, V; macroblock-padded) and the encoder's own (raw_y: Y before the filter).  Returns 0, -1 on bad dimensions, -2 when the
 * first partition does not fit in 19 bits (the file is then still returned, for the tests). */
int orc_webp_bpred_encode(const uint8_t *r, const uint8_t *g, const uint8_t *b, int w, int h, int quality, uint8_t **out, size_t *out_len,
                          int16_t *levels, uint8_t *modes, uint8_t *bmodes, uint8_t *recon_y, uint8_t *recon_u, uint8_t *recon_v, uint8_t *raw_y)
{
    if (w < 1 || h < 1 || w > 16383 || h > 16383) return -1;
    const int mbw = (w + 15) >> 4, mbh = (h + 15) >> 4, nmb = mbw * mbh, ys = mbw * 16, cs = mbw * 8;
    const size_t ny = (size_t)ys * mbh * 16, nc = (size_t)cs * mbh * 8;
    uint8_t *Y = (uint8_t *)malloc(ny), *U = (uint8_t *)malloc(nc), *V = (uint8_t *)malloc(nc);
    uint8_t *RY = (uint8_t *)calloc(ny, 1), *RU = (uint8_t *)calloc(nc, 1), *RV = (uint8_t *)calloc(nc, 1);
    MbCoded *mbs = (MbCoded *)malloc(sizeof(MbCoded) * (size_t)nmb);
    orc_webp_rgb_to_yuv(r, g, b, w, h, Y, U, V);
    const int q = orc_vp8_qindex(quality), flevel = orc_vp8_filter_level(q);
    int f[6]; orc_vp8_quant_factors(q, f);
    int nskip = 0;
    const uint8_t zero4[4] = {0, 0, 0, 0};
    for (int mby = 0; mby < mbh; mby++) for (int mbx = 0; mbx < mbw; mbx++) {
        MbCoded *m = &mbs[mby * mbw + mbx];
        uint8_t left4[4];
        if (mbx) for (int y = 0; y < 4; y++) left4[y] = m[-1].bmodes[4 * y + 3];
        encode_mb(Y, U, V, RY, RU, RV, mbw, mbx, mby, f, mby ? mbs[(mby - 1) * mbw + mbx].bmodes + 12 : zero4, mbx ? left4 : zero4, m);
        nskip += m->skip;
    }
    const int use_skip = nskip > 0;
    uint8_t probs[4 * 8 * 3 * 11], updated[4 * 8 * 3 * 11];
    memcpy(probs, ORC_VP8_COEF_PROBS, sizeof(probs));
    {
        uint32_t *stats = (uint32_t *)calloc(4 * 8 * 3 * 11 * 2, sizeof(uint32_t));
        Coder k = {NULL, stats, probs};
        code_frame_tokens(&k, mbs, mbw, mbh, use_skip);
        choose_probs(stats, probs, updated);
        free(stats);
    }
    Bool h0, tk; bool_init(&h0); bool_init(&tk);
    int skip_p = (int)(((long)(nmb - nskip) * 255) / nmb); if (skip_p < 1) skip_p = 1; if (skip_p > 255) skip_p = 255;
    bool_bits(&h0, 0, 1); bool_bits(&h0, 0, 1); bool_bits(&h0, 0, 1);     /* colour space, clamping, no segmentation */
    bool_bits(&h0, 1, 1); bool_bits(&h0, flevel, 6); bool_bits(&h0, 0, 3); /* simple filter, level, sharpness */
    bool_bits(&h0, 0, 1); bool_bits(&h0, 0, 2); bool_bits(&h0, q, 7);     /* no filter deltas, one partition, y_ac_qi */
    for (int i = 0; i < 5; i++) bool_bits(&h0, 0, 1);
    bool_bits(&h0, 0, 1);                                                   /* refresh_entropy_probs */
    for (int i = 0; i < 4 * 8 * 3 * 11; i++) if (bool_put(&h0, updated[i], ORC_VP8_COEF_UPDATE_PROBS[i])) bool_bits(&h0, probs[i], 8);
    bool_bits(&h0, use_skip, 1);
    if (use_skip) bool_bits(&h0, skip_p, 8);
    uint8_t *top_modes = (uint8_t *)calloc((size_t)mbw, 4), left_modes[4];
    for (int i = 0; i < nmb; i++) {
        const MbCoded *m = &mbs[i];
        uint8_t *tm = top_modes + (size_t)(i % mbw) * 4;
        if (i % mbw == 0) memset(left_modes, 0, 4);
        if (use_skip) bool_put(&h0, m->skip, skip_p);
        if (m->ymode == VP8BP_YMODE) {
            bool_put(&h0, 0, 145);
            for (int k = 0; k < 16; k++) {
                /* the decoder's tree walk run backwards: from the root, the branch whose subtree holds the mode */
                const uint8_t *pr = VP8_BMODES_PROBA[tm[k & 3]][left_modes[k >> 2]];
                const int mode = m->bmodes[k];
                int nd = 0;
                for (;;) {
                    int bit = -1;
                    for (int side = 0; side < 2 && bit < 0; side++) {      /* search the subtree under entry 2 * nd + side */
                        int stack[16], sp = 0; stack[sp++] = VP8_YMODES_INTRA4[2 * nd + side];
                        while (sp) { const int v = stack[--sp]; if (v <= 0) { if (-v == mode) bit = side; } else { stack[sp++] = VP8_YMODES_INTRA4[2 * v]; stack[sp++] = VP8_YMODES_INTRA4[2 * v + 1]; } }
                    }
                    bool_put(&h0, bit, pr[nd]);
                    const int next = VP8_YMODES_INTRA4[2 * nd + bit];
                    if (next <= 0) break;
                    nd = next;
                }
                tm[k & 3] = left_modes[k >> 2] = (uint8_t)mode;
            }
        } else {
            bool_put(&h0, 1, 145);
            if (bool_put(&h0, m->ymode == 1 || m->ymode == 3, 156)) bool_put(&h0, m->ymode == 1, 128);
            else bool_put(&h0, m->ymode == 2, 163);
            memset(tm, m->ymode, 4); memset(left_modes, m->ymode, 4);
        }
        if (bool_put(&h0, m->uvmode != 0, 142)) if (bool_put(&h0, m->uvmode != 2, 114)) bool_put(&h0, m->uvmode != 3, 183);
    }
    free(top_modes);
    bool_flush(&h0);
    { Coder k = {&tk, NULL, probs}; code_frame_tokens(&k, mbs, mbw, mbh, use_skip); }
    bool_flush(&tk);
    const size_t vp8_size = 10 + h0.n + tk.n, riff_payload = 4 + 8 + vp8_size + (vp8_size & 1);
    uint8_t *o = (uint8_t *)malloc(8 + riff_payload), *p = o;
    memcpy(p, "RIFF", 4); p += 4;
    *p++ = (uint8_t)riff_payload; *p++ = (uint8_t)(riff_payload >> 8); *p++ = (uint8_t)(riff_payload >> 16); *p++ = (uint8_t)(riff_payload >> 24);
    memcpy(p, "WEBPVP8 ", 8); p += 8;
    *p++ = (uint8_t)vp8_size; *p++ = (uint8_t)(vp8_size >> 8); *p++ = (uint8_t)(vp8_size >> 16); *p++ = (uint8_t)(vp8_size >> 24);
    const uint32_t tag = (1u << 4) | ((uint32_t)h0.n << 5);
    *p++ = (uint8_t)tag; *p++ = (uint8_t)(tag >> 8); *p++ = (uint8_t)(tag >> 16);
    *p++ = 0x9d; *p++ = 0x01; *p++ = 0x2a;
    *p++ = (uint8_t)w; *p++ = (uint8_t)(w >> 8); *p++ = (uint8_t)h; *p++ = (uint8_t)(h >> 8);
    memcpy(p, h0.buf, h0.n); p += h0.n; memcpy(p, tk.buf, tk.n); p += tk.n;
    if (vp8_size & 1) *p++ = 0;
    *out = o; *out_len = (size_t)(p - o);
    for (int i = 0; i < nmb; i++) {
        const MbCoded *m = &mbs[i];
        if (levels) {
            int16_t *lv = levels + (size_t)i * 400;
            memcpy(lv, m->y2, 32);
            for (int k = 0; k < 16; k++) memcpy(lv + 16 * (1 + k), m->y[k], 32);
            for (int k = 0; k < 4; k++) { memcpy(lv + 16 * (17 + k), m->u[k], 32); memcpy(lv + 16 * (21 + k), m->v[k], 32); }
        }
        if (modes) { modes[4 * i] = m->ymode; modes[4 * i + 1] = m->uvmode; modes[4 * i + 2] = m->skip; modes[4 * i + 3] = 0; }
        if (bmodes) memcpy(bmodes + 16 * (size_t)i, m->bmodes, 16);
    }
    if (raw_y) memcpy(raw_y, RY, ny);
    if (recon_y) { loop_filter_simple(RY, mbw, mbh, flevel, mbs); memcpy(recon_y, RY, ny); }
    if (recon_u) memcpy(recon_u, RU, nc);
    if (recon_v) memcpy(recon_v, RV, nc);
    const int big = h0.n >= (1u << 19);
    free(Y); free(U); free(V); free(RY); free(RU); free(RV); free(mbs); free(h0.buf); free(tk.buf);
    return big ? -2 : 0;
}
