/*
 * oracle/jpeg_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE (see jpeg_oracle.h).
 *
 * Plain-C restatement of the JPEG path below caesiumclt's codec boundary
 * (caesium-clt's src/compressor.rs:287-306 -> caesium::compress_in_memory).
 * Upstream routine names (mozjpeg 4.x / libjpeg-turbo lineage, pinned by
 * caesium-clt's Cargo.lock:1035 mozjpeg-sys 2.2.1) are cited per function; the
 * sources are not vendored under the caesium-clt sources, so each block restates the
 * published IJG algorithm and is pinned by tests/test_oracle_jpeg.py against
 * libjpeg-turbo (Pillow) and the fixtures' DQT / scan-script known answers.
 */
#include "jpeg_oracle.h"
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define SETERR(...) do { if (err) snprintf(err, 256, __VA_ARGS__); } while (0)

static const uint8_t ZZ[64] = { /* zigzag index k -> natural (row-major) position; jutils.c jpeg_natural_order */
     0,  1,  8, 16,  9,  2,  3, 10, 17, 24, 32, 25, 18, 11,  4,  5,
    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,  6,  7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63 };

/* ------------------------------------------------------------------------- */
/* Quantisation tables: mozjpeg jcparam.c, base table index 3 ("ImageMagick   */
/* table by N. Robidoux"), the JCP_MAX_COMPRESSION default; luma == chroma.   */
/* Values fitted to samples/j0.JPG's DQT (SURVEY.md KAT-1).                   */
/* ------------------------------------------------------------------------- */
static const uint16_t ROBIDOUX[64] = {
    16, 16, 16, 18, 25, 37, 56, 85,
    16, 17, 20, 27, 34, 40, 53, 75,
    16, 20, 24, 31, 43, 62, 91, 135,
    18, 27, 31, 40, 53, 74, 106, 156,
    25, 34, 43, 53, 69, 94, 131, 189,
    37, 40, 62, 74, 94, 124, 169, 238,
    56, 53, 91, 106, 131, 169, 226, 311,
    85, 75, 135, 156, 189, 238, 311, 418 };

/* jcparam.c jpeg_quality_scaling + jpeg_add_quant_table(force_baseline = FALSE) */
void orc_quant_table(int quality, int which, uint16_t out[64])
{
    (void)which; /* table idx 3 is identical for luma and chroma */
    int q = quality;
    if (q <= 0) q = 1;
    if (q > 100) q = 100;
    int scale = q < 50 ? 5000 / q : 200 - q * 2;
    for (int i = 0; i < 64; i++) {
        long t = ((long)ROBIDOUX[i] * scale + 50L) / 100L;
        if (t <= 0) t = 1;
        if (t > 32767) t = 32767;
        out[i] = (uint16_t)t;
    }
}

/* ------------------------------------------------------------------------- */
/* jidctint.c jpeg_idct_islow: CONST_BITS = 13, PASS1_BITS = 2                */
/* ------------------------------------------------------------------------- */
#define CONST_BITS 13
#define PASS1_BITS 2
#define FIX_0_298631336 2446
#define FIX_0_390180644 3196
#define FIX_0_541196100 4433
#define FIX_0_765366865 6270
#define FIX_0_899976223 7373
#define FIX_1_175875602 9633
#define FIX_1_501321110 12299
#define FIX_1_847759065 15137
#define FIX_1_961570560 16069
#define FIX_2_053119869 16819
#define FIX_2_562915447 20995
#define FIX_3_072711026 25172
#define DESCALE(x, n) (((x) + (1 << ((n)-1))) >> (n))

/* jdmaster.c prepare_range_limit_table, indexed as IDCT_range_limit[x & RANGE_MASK] */
static inline uint8_t range_limit_idct(int32_t x)
{
    int v = x & 1023;
    if (v < 128) return (uint8_t)(v + 128);
    if (v < 512) return 255;
    if (v < 896) return 0;
    return (uint8_t)(v - 896);
}

void orc_idct_islow(const int16_t coef[64], const uint16_t q[64], uint8_t out[64])
{
    int32_t ws[64];
    for (int c = 0; c < 8; c++) { /* pass 1: columns */
        int32_t in0 = coef[c] * (int32_t)q[c], in1 = coef[8 + c] * (int32_t)q[8 + c];
        int32_t in2 = coef[16 + c] * (int32_t)q[16 + c], in3 = coef[24 + c] * (int32_t)q[24 + c];
        int32_t in4 = coef[32 + c] * (int32_t)q[32 + c], in5 = coef[40 + c] * (int32_t)q[40 + c];
        int32_t in6 = coef[48 + c] * (int32_t)q[48 + c], in7 = coef[56 + c] * (int32_t)q[56 + c];
        int32_t z1, z2, z3, z4, z5, t0, t1, t2, t3, t10, t11, t12, t13;
        z2 = in2; z3 = in6;
        z1 = (z2 + z3) * FIX_0_541196100;
        t2 = z1 + z3 * (-FIX_1_847759065);
        t3 = z1 + z2 * FIX_0_765366865;
        z2 = in0; z3 = in4;
        t0 = (z2 + z3) * (1 << CONST_BITS);
        t1 = (z2 - z3) * (1 << CONST_BITS);
        t10 = t0 + t3; t13 = t0 - t3; t11 = t1 + t2; t12 = t1 - t2;
        t0 = in7; t1 = in5; t2 = in3; t3 = in1;
        z1 = t0 + t3; z2 = t1 + t2; z3 = t0 + t2; z4 = t1 + t3;
        z5 = (z3 + z4) * FIX_1_175875602;
        t0 *= FIX_0_298631336; t1 *= FIX_2_053119869; t2 *= FIX_3_072711026; t3 *= FIX_1_501321110;
        z1 *= -FIX_0_899976223; z2 *= -FIX_2_562915447; z3 *= -FIX_1_961570560; z4 *= -FIX_0_390180644;
        z3 += z5; z4 += z5;
        t0 += z1 + z3; t1 += z2 + z4; t2 += z2 + z3; t3 += z1 + z4;
        ws[c]      = DESCALE(t10 + t3, CONST_BITS - PASS1_BITS);
        ws[56 + c] = DESCALE(t10 - t3, CONST_BITS - PASS1_BITS);
        ws[8 + c]  = DESCALE(t11 + t2, CONST_BITS - PASS1_BITS);
        ws[48 + c] = DESCALE(t11 - t2, CONST_BITS - PASS1_BITS);
        ws[16 + c] = DESCALE(t12 + t1, CONST_BITS - PASS1_BITS);
        ws[40 + c] = DESCALE(t12 - t1, CONST_BITS - PASS1_BITS);
        ws[24 + c] = DESCALE(t13 + t0, CONST_BITS - PASS1_BITS);
        ws[32 + c] = DESCALE(t13 - t0, CONST_BITS - PASS1_BITS);
    }
    for (int r = 0; r < 8; r++) { /* pass 2: rows */
        const int32_t *w = ws + 8 * r;
        int32_t z1, z2, z3, z4, z5, t0, t1, t2, t3, t10, t11, t12, t13;
        z2 = w[2]; z3 = w[6];
        z1 = (z2 + z3) * FIX_0_541196100;
        t2 = z1 + z3 * (-FIX_1_847759065);
        t3 = z1 + z2 * FIX_0_765366865;
        t0 = (w[0] + w[4]) * (1 << CONST_BITS);
        t1 = (w[0] - w[4]) * (1 << CONST_BITS);
        t10 = t0 + t3; t13 = t0 - t3; t11 = t1 + t2; t12 = t1 - t2;
        t0 = w[7]; t1 = w[5]; t2 = w[3]; t3 = w[1];
        z1 = t0 + t3; z2 = t1 + t2; z3 = t0 + t2; z4 = t1 + t3;
        z5 = (z3 + z4) * FIX_1_175875602;
        t0 *= FIX_0_298631336; t1 *= FIX_2_053119869; t2 *= FIX_3_072711026; t3 *= FIX_1_501321110;
        z1 *= -FIX_0_899976223; z2 *= -FIX_2_562915447; z3 *= -FIX_1_961570560; z4 *= -FIX_0_390180644;
        z3 += z5; z4 += z5;
        t0 += z1 + z3; t1 += z2 + z4; t2 += z2 + z3; t3 += z1 + z4;
        uint8_t *o = out + 8 * r;
        o[0] = range_limit_idct(DESCALE(t10 + t3, CONST_BITS + PASS1_BITS + 3));
        o[7] = range_limit_idct(DESCALE(t10 - t3, CONST_BITS + PASS1_BITS + 3));
        o[1] = range_limit_idct(DESCALE(t11 + t2, CONST_BITS + PASS1_BITS + 3));
        o[6] = range_limit_idct(DESCALE(t11 - t2, CONST_BITS + PASS1_BITS + 3));
        o[2] = range_limit_idct(DESCALE(t12 + t1, CONST_BITS + PASS1_BITS + 3));
        o[5] = range_limit_idct(DESCALE(t12 - t1, CONST_BITS + PASS1_BITS + 3));
        o[3] = range_limit_idct(DESCALE(t13 + t0, CONST_BITS + PASS1_BITS + 3));
        o[4] = range_limit_idct(DESCALE(t13 - t0, CONST_BITS + PASS1_BITS + 3));
    }
}

/* jfdctint.c jpeg_fdct_islow preceded by jcdctmgr.c convsamp (sample - CENTERJSAMPLE) */
void orc_fdct_islow(const uint8_t px[64], int32_t d[64])
{
    for (int i = 0; i < 64; i++) d[i] = (int32_t)px[i] - 128;
    for (int r = 0; r < 8; r++) { /* pass 1: rows */
        int32_t *p = d + 8 * r;
        int32_t t0 = p[0] + p[7], t7 = p[0] - p[7], t1 = p[1] + p[6], t6 = p[1] - p[6];
        int32_t t2 = p[2] + p[5], t5 = p[2] - p[5], t3 = p[3] + p[4], t4 = p[3] - p[4];
        int32_t t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
        p[0] = (t10 + t11) * (1 << PASS1_BITS);
        p[4] = (t10 - t11) * (1 << PASS1_BITS);
        int32_t z1 = (t12 + t13) * FIX_0_541196100;
        p[2] = DESCALE(z1 + t13 * FIX_0_765366865, CONST_BITS - PASS1_BITS);
        p[6] = DESCALE(z1 + t12 * (-FIX_1_847759065), CONST_BITS - PASS1_BITS);
        z1 = t4 + t7; int32_t z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
        int32_t z5 = (z3 + z4) * FIX_1_175875602;
        t4 *= FIX_0_298631336; t5 *= FIX_2_053119869; t6 *= FIX_3_072711026; t7 *= FIX_1_501321110;
        z1 *= -FIX_0_899976223; z2 *= -FIX_2_562915447; z3 *= -FIX_1_961570560; z4 *= -FIX_0_390180644;
        z3 += z5; z4 += z5;
        p[7] = DESCALE(t4 + z1 + z3, CONST_BITS - PASS1_BITS);
        p[5] = DESCALE(t5 + z2 + z4, CONST_BITS - PASS1_BITS);
        p[3] = DESCALE(t6 + z2 + z3, CONST_BITS - PASS1_BITS);
        p[1] = DESCALE(t7 + z1 + z4, CONST_BITS - PASS1_BITS);
    }
    for (int c = 0; c < 8; c++) { /* pass 2: columns */
        int32_t *p = d + c;
        int32_t t0 = p[0] + p[56], t7 = p[0] - p[56], t1 = p[8] + p[48], t6 = p[8] - p[48];
        int32_t t2 = p[16] + p[40], t5 = p[16] - p[40], t3 = p[24] + p[32], t4 = p[24] - p[32];
        int32_t t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
        p[0]  = DESCALE(t10 + t11, PASS1_BITS);
        p[32] = DESCALE(t10 - t11, PASS1_BITS);
        int32_t z1 = (t12 + t13) * FIX_0_541196100;
        p[16] = DESCALE(z1 + t13 * FIX_0_765366865, CONST_BITS + PASS1_BITS);
        p[48] = DESCALE(z1 + t12 * (-FIX_1_847759065), CONST_BITS + PASS1_BITS);
        z1 = t4 + t7; int32_t z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
        int32_t z5 = (z3 + z4) * FIX_1_175875602;
        t4 *= FIX_0_298631336; t5 *= FIX_2_053119869; t6 *= FIX_3_072711026; t7 *= FIX_1_501321110;
        z1 *= -FIX_0_899976223; z2 *= -FIX_2_562915447; z3 *= -FIX_1_961570560; z4 *= -FIX_0_390180644;
        z3 += z5; z4 += z5;
        p[56] = DESCALE(t4 + z1 + z3, CONST_BITS + PASS1_BITS);
        p[40] = DESCALE(t5 + z2 + z4, CONST_BITS + PASS1_BITS);
        p[24] = DESCALE(t6 + z2 + z3, CONST_BITS + PASS1_BITS);
        p[8]  = DESCALE(t7 + z1 + z4, CONST_BITS + PASS1_BITS);
    }
}

/* jcdctmgr.c quantize(): divisor = quantval << 3 for ISLOW; round half away from zero */
void orc_quantize(const int32_t dct[64], const uint16_t q[64], int16_t out[64])
{
    for (int i = 0; i < 64; i++) {
        int32_t qv = (int32_t)q[i] << 3, t = dct[i];
        if (t < 0) { t = -t; t += qv >> 1; t = t >= qv ? t / qv : 0; t = -t; }
        else       { t += qv >> 1; t = t >= qv ? t / qv : 0; }
        out[i] = (int16_t)t;
    }
}

/* ------------------------------------------------------------------------- */
/* jdsample.c upsamplers.  Edge columns/rows use the nearest sample as the    */
/* missing neighbour, which reproduces the "special case" first/last column  */
/* formulas and jdmainct.c's top/bottom row replication exactly.             */
/* ------------------------------------------------------------------------- */
static inline int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

void orc_upsample_box(const uint8_t *in, int cw, int ch, int stride, int hx, int vx, uint8_t *out, int ow, int oh, int ostride)
{   /* int_upsample / h2v1_upsample / h2v2_upsample: pixel replication */
    for (int y = 0; y < oh; y++) {
        const uint8_t *r = in + (size_t)clampi(y / vx, 0, ch - 1) * stride;
        for (int x = 0; x < ow; x++) out[(size_t)y * ostride + x] = r[clampi(x / hx, 0, cw - 1)];
    }
}

void orc_upsample_h2v1_fancy(const uint8_t *in, int cw, int ch, int stride, uint8_t *out, int ow, int oh, int ostride)
{   /* h2v1_fancy_upsample: 3/4 nearest + 1/4 further, rounding bias 1 (left) / 2 (right) */
    if (cw <= 2) { orc_upsample_box(in, cw, ch, stride, 2, 1, out, ow, oh, ostride); return; } /* jinit_upsampler: fancy needs downsampled_width > 2 */
    for (int y = 0; y < oh; y++) {
        const uint8_t *r = in + (size_t)clampi(y, 0, ch - 1) * stride;
        for (int x = 0; x < ow; x++) {
            int c = x >> 1, v = 3 * r[c];
            if (x & 1) v = (v + r[clampi(c + 1, 0, cw - 1)] + 2) >> 2;
            else       v = (v + r[clampi(c - 1, 0, cw - 1)] + 1) >> 2;
            out[(size_t)y * ostride + x] = (uint8_t)v;
        }
    }
}

void orc_upsample_h1v2_fancy(const uint8_t *in, int cw, int ch, int stride, uint8_t *out, int ow, int oh, int ostride)
{   /* h1v2_fancy_upsample (libjpeg-turbo >= 2.0): bias 1 for the upper output row, 2 for the lower */
    for (int y = 0; y < oh; y++) {
        int r = y >> 1;
        const uint8_t *r0 = in + (size_t)clampi(r, 0, ch - 1) * stride;
        const uint8_t *r1 = in + (size_t)clampi((y & 1) ? r + 1 : r - 1, 0, ch - 1) * stride;
        int bias = (y & 1) ? 2 : 1;
        for (int x = 0; x < ow; x++) {
            int c = clampi(x, 0, cw - 1);
            out[(size_t)y * ostride + x] = (uint8_t)((3 * r0[c] + r1[c] + bias) >> 2);
        }
    }
}

void orc_upsample_h2v2_fancy(const uint8_t *in, int cw, int ch, int stride, uint8_t *out, int ow, int oh, int ostride)
{   /* h2v2_fancy_upsample: triangle filter, 9/16 3/16 3/16 1/16; bias 8 (even col) / 7 (odd col) */
    if (cw <= 2) { orc_upsample_box(in, cw, ch, stride, 2, 2, out, ow, oh, ostride); return; }
    for (int y = 0; y < oh; y++) {
        int r = y >> 1;
        const uint8_t *r0 = in + (size_t)clampi(r, 0, ch - 1) * stride;
        const uint8_t *r1 = in + (size_t)clampi((y & 1) ? r + 1 : r - 1, 0, ch - 1) * stride;
        for (int x = 0; x < ow; x++) {
            int c = x >> 1;
            int cn = clampi((x & 1) ? c + 1 : c - 1, 0, cw - 1);
            int thiscol = 3 * r0[c] + r1[c], othercol = 3 * r0[cn] + r1[cn];
            out[(size_t)y * ostride + x] = (uint8_t)((3 * thiscol + othercol + ((x & 1) ? 7 : 8)) >> 4);
        }
    }
}

/* jcsample.c h2v1_downsample / h2v2_downsample / int_downsample / fullsize_downsample,
 * with jcprepct.c expand_bottom_edge and jcsample.c expand_right_edge padding rules.
 * (hx, vx) = box size; out is pw x ph where pw, ph are multiples of 8 covering the real blocks. */
void orc_downsample(const uint8_t *in, int w, int h, int stride, int hx, int vx, uint8_t *out, int pw, int ph)
{
    /* input is first padded at the bottom to a whole "row group" (max_v_samp rows; vx == vmax/vs and the
     * component keeps vs rows per group); downsampled rows past the last group replicate the last row. */
    int nreal = ((h + vx - 1) / vx);           /* rows this component really has after downsampling */
    for (int y = 0; y < ph; y++) {
        int yy = y < nreal ? y : nreal - 1;
        for (int x = 0; x < pw; x++) {
            int sum = 0;
            for (int dy = 0; dy < vx; dy++) {
                const uint8_t *r = in + (size_t)clampi(yy * vx + dy, 0, h - 1) * stride;
                for (int dx = 0; dx < hx; dx++) sum += r[clampi(x * hx + dx, 0, w - 1)];
            }
            int v;
            if (hx == 1 && vx == 1) v = sum;
            else if (hx == 2 && vx == 1) v = (sum + (x & 1)) >> 1;            /* bias 0,1,0,1 */
            else if (hx == 2 && vx == 2) v = (sum + 1 + (x & 1)) >> 2;        /* bias 1,2,1,2 */
            else { int n = hx * vx; v = (sum + n / 2) / n; }                   /* int_downsample */
            out[(size_t)y * pw + x] = (uint8_t)v;
        }
    }
}

/* ------------------------------------------------------------------------- */
/* Marker parsing + Huffman decoding (jdmarker.c, jdhuff.c, jdphuff.c)        */
/* ------------------------------------------------------------------------- */
typedef struct { uint8_t bits[17]; uint8_t vals[256]; int present; uint16_t *look; /* 65536 entries: len<<8|sym, 0 = invalid */ } hufftab;

static void huff_build(hufftab *t)
{
    if (!t->look) t->look = (uint16_t *)malloc(65536 * sizeof(uint16_t));
    memset(t->look, 0, 65536 * sizeof(uint16_t));
    uint32_t code = 0; int p = 0;
    for (int l = 1; l <= 16; l++) {
        for (int i = 0; i < t->bits[l]; i++, p++) {
            uint32_t first = code << (16 - l), n = 1u << (16 - l);
            if (first + n > 65536) return; /* over-subscribed table: leave the rest invalid */
            uint16_t e = (uint16_t)((l << 8) | t->vals[p]);
            for (uint32_t k = 0; k < n; k++) t->look[first + k] = e;
            code++;
        }
        code <<= 1;
    }
}

typedef struct { const uint8_t *p, *end; uint64_t acc; int nbits; int marker; } bitrd;

static void br_fill(bitrd *b)
{
    while (b->nbits <= 56) {
        unsigned c = 0;
        if (!b->marker && b->p < b->end) {
            c = *b->p++;
            if (c == 0xFF) {
                unsigned c2 = b->p < b->end ? *b->p : 0xD9;
                if (c2 == 0) b->p++;
                else { b->p--; b->marker = 1; c = 0; } /* stop at marker; feed zeros like jdhuff.c's "insert_fake_zeros" */
            }
        }
        b->acc |= (uint64_t)c << (56 - b->nbits);
        b->nbits += 8;
    }
}
static inline unsigned br_peek16(bitrd *b) { if (b->nbits < 16) br_fill(b); return (unsigned)(b->acc >> 48); }
static inline void br_drop(bitrd *b, int n) { b->acc <<= n; b->nbits -= n; }
static inline int br_get(bitrd *b, int n) { if (n == 0) return 0; if (b->nbits < n) br_fill(b); int v = (int)(b->acc >> (64 - n)); br_drop(b, n); return v; }
static inline int huff_decode(bitrd *b, const hufftab *t) { unsigned e = t->look[br_peek16(b)]; if (!e) return -1; br_drop(b, e >> 8); return e & 0xFF; }
static inline int huff_extend(int v, int s) { return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v; }

static int ceil_div(int a, int b) { return (a + b - 1) / b; }

typedef struct {
    hufftab dc[4], ac[4];
} huffset;

typedef struct { int ns; int ci[4]; int td[4], ta[4]; int Ss, Se, Ah, Al; } scanhdr;

/* decode one entropy-coded segment (one scan) into j->coef */
static int decode_scan(orc_jpeg *j, const scanhdr *s, huffset *hs, const uint8_t *p, const uint8_t *end, const uint8_t **next, char *err)
{
    bitrd b = { p, end, 0, 0, 0 };
    int pred[4] = { 0, 0, 0, 0 };
    int eobrun = 0;
    int interleaved = s->ns > 1;
    int c0 = s->ci[0];
    int mcus_x = interleaved ? j->mcux : j->rbw[c0];
    int mcus_y = interleaved ? j->mcuy : j->rbh[c0];
    int restart_in = j->restart_interval, rst_count = 0;
    for (int i = 0; i < s->ns; i++) {
        if (s->Ss == 0 && (!j->progressive || s->Ah == 0) && !hs->dc[s->td[i]].present) { SETERR("missing DC Huffman table %d", s->td[i]); return -1; }
        if ((s->Se > 0) && !hs->ac[s->ta[i]].present) { SETERR("missing AC Huffman table %d", s->ta[i]); return -1; }
    }
    for (int my = 0; my < mcus_y; my++) for (int mx = 0; mx < mcus_x; mx++) {
        if (restart_in && rst_count == restart_in) {
            /* jdhuff.c process_restart: discard partial byte, expect RSTn */
            b.nbits = 0; b.acc = 0;
            const uint8_t *q = b.p;
            while (q + 1 < end && !(q[0] == 0xFF && q[1] >= 0xD0 && q[1] <= 0xD7)) {
                if (q[0] == 0xFF && q[1] != 0 && q[1] != 0xFF) break;
                q++;
            }
            if (q + 1 < end && q[0] == 0xFF && q[1] >= 0xD0 && q[1] <= 0xD7) q += 2;
            b.p = q; b.marker = 0;
            pred[0] = pred[1] = pred[2] = pred[3] = 0; eobrun = 0; rst_count = 0;
        }
        rst_count++;
        for (int i = 0; i < s->ns; i++) {
            int c = s->ci[i];
            int nbx = interleaved ? j->hs[c] : 1, nby = interleaved ? j->vs[c] : 1;
            for (int by = 0; by < nby; by++) for (int bx = 0; bx < nbx; bx++) {
                int row = interleaved ? my * j->vs[c] + by : my;
                int col = interleaved ? mx * j->hs[c] + bx : mx;
                int16_t *blk = j->coef[c] + ((size_t)row * j->bw[c] + col) * 64;
                if (!j->progressive) {
                    /* jdhuff.c decode_mcu_slow */
                    int sz = huff_decode(&b, &hs->dc[s->td[i]]);
                    if (sz < 0 || sz > 16) { SETERR("bad DC code"); return -1; }
                    int diff = sz ? huff_extend(br_get(&b, sz), sz) : 0;
                    pred[i] += diff; blk[0] = (int16_t)pred[i];
                    for (int k = 1; k < 64; k++) {
                        int rs = huff_decode(&b, &hs->ac[s->ta[i]]);
                        if (rs < 0) { SETERR("bad AC code"); return -1; }
                        int r = rs >> 4, sz2 = rs & 15;
                        if (sz2) { k += r; if (k > 63) break; blk[ZZ[k]] = (int16_t)huff_extend(br_get(&b, sz2), sz2); }
                        else { if (r != 15) break; k += 15; }
                    }
                } else if (s->Ss == 0) {
                    if (s->Ah == 0) { /* jdphuff.c decode_mcu_DC_first */
                        int sz = huff_decode(&b, &hs->dc[s->td[i]]);
                        if (sz < 0 || sz > 16) { SETERR("bad DC code"); return -1; }
                        int diff = sz ? huff_extend(br_get(&b, sz), sz) : 0;
                        pred[i] += diff; blk[0] = (int16_t)(pred[i] * (1 << s->Al));
                    } else {          /* decode_mcu_DC_refine */
                        if (br_get(&b, 1)) blk[0] |= (int16_t)(1 << s->Al);
                    }
                } else if (s->Ah == 0) { /* decode_mcu_AC_first */
                    if (eobrun > 0) eobrun--;
                    else for (int k = s->Ss; k <= s->Se; k++) {
                        int rs = huff_decode(&b, &hs->ac[s->ta[i]]);
                        if (rs < 0) { SETERR("bad AC code"); return -1; }
                        int r = rs >> 4, sz = rs & 15;
                        if (sz) { k += r; if (k > 63) break; blk[ZZ[k]] = (int16_t)(huff_extend(br_get(&b, sz), sz) * (1 << s->Al)); }
                        else if (r == 15) k += 15;
                        else { eobrun = 1 << r; if (r) eobrun += br_get(&b, r); eobrun--; break; }
                    }
                } else {               /* decode_mcu_AC_refine */
                    int p1 = 1 << s->Al, m1 = -(1 << s->Al);
                    int k = s->Ss;
                    if (eobrun == 0) {
                        for (; k <= s->Se; k++) {
                            int rs = huff_decode(&b, &hs->ac[s->ta[i]]);
                            if (rs < 0) { SETERR("bad AC code"); return -1; }
                            int r = rs >> 4, sz = rs & 15, val = 0;
                            if (sz) { val = br_get(&b, 1) ? p1 : m1; }
                            else if (r != 15) { eobrun = 1 << r; if (r) eobrun += br_get(&b, r); break; }
                            do {
                                int16_t *cf = blk + ZZ[k];
                                if (*cf != 0) {
                                    if (br_get(&b, 1)) { if ((*cf & p1) == 0) *cf = (int16_t)(*cf >= 0 ? *cf + p1 : *cf + m1); }
                                } else { if (--r < 0) break; }
                                k++;
                            } while (k <= s->Se);
                            if (val && k <= 63) blk[ZZ[k]] = (int16_t)val;
                        }
                    }
                    if (eobrun > 0) {
                        for (; k <= s->Se; k++) {
                            int16_t *cf = blk + ZZ[k];
                            if (*cf != 0 && br_get(&b, 1)) { if ((*cf & p1) == 0) *cf = (int16_t)(*cf >= 0 ? *cf + p1 : *cf + m1); }
                        }
                        eobrun--;
                    }
                }
            }
        }
    }
    /* advance to the next marker */
    const uint8_t *q = b.p;
    if (!b.marker) { while (q + 1 < end && !(q[0] == 0xFF && q[1] != 0 && q[1] != 0xFF && !(q[1] >= 0xD0 && q[1] <= 0xD7))) q++; }
    *next = q;
    return 0;
}

static void append_bytes(uint8_t **buf, size_t *len, const uint8_t *src, size_t n)
{
    *buf = (uint8_t *)realloc(*buf, *len + n + 1);
    memcpy(*buf + *len, src, n); *len += n;
}

void orc_jpeg_free(orc_jpeg *j)
{
    for (int c = 0; c < ORC_MAX_COMP; c++) { free(j->coef[c]); j->coef[c] = NULL; }
    free(j->markers); j->markers = NULL; free(j->icc_markers); j->icc_markers = NULL;
}
void orc_free(void *p) { free(p); }

static void setup_geometry(orc_jpeg *j)
{   /* jdmaster.c / jcmaster.c initial_setup + per_scan_setup geometry */
    j->hmax = j->vmax = 1;
    for (int c = 0; c < j->ncomp; c++) { if (j->hs[c] > j->hmax) j->hmax = j->hs[c]; if (j->vs[c] > j->vmax) j->vmax = j->vs[c]; }
    j->mcux = ceil_div(j->width, 8 * j->hmax); j->mcuy = ceil_div(j->height, 8 * j->vmax);
    for (int c = 0; c < j->ncomp; c++) {
        j->cw[c] = ceil_div(j->width * j->hs[c], j->hmax); j->ch[c] = ceil_div(j->height * j->vs[c], j->vmax);
        j->rbw[c] = ceil_div(j->cw[c], 8); j->rbh[c] = ceil_div(j->ch[c], 8);
        j->bw[c] = j->mcux * j->hs[c]; j->bh[c] = j->mcuy * j->vs[c];
    }
}

int orc_jpeg_read(const uint8_t *d, size_t len, orc_jpeg *j, char err[256])
{
    memset(j, 0, sizeof(*j));
    huffset *hs = (huffset *)calloc(1, sizeof(huffset));
    int rc = -1, have_sof = 0;
    if (len < 4 || d[0] != 0xFF || d[1] != 0xD8) { SETERR("not a JPEG (no SOI)"); goto done; }
    size_t i = 2;
    while (i + 3 < len) {
        if (d[i] != 0xFF) { i++; continue; }
        unsigned m = d[i + 1];
        if (m == 0xFF) { i++; continue; }
        if (m == 0x00 || m == 0x01 || (m >= 0xD0 && m <= 0xD8)) { i += 2; continue; }
        if (m == 0xD9) break;
        size_t L = ((size_t)d[i + 2] << 8) | d[i + 3];
        if (L < 2 || i + 2 + L > len) { SETERR("truncated marker segment %02X", m); goto done; }
        const uint8_t *seg = d + i + 4; size_t sl = L - 2;
        if (m == 0xDB) { /* jdmarker.c get_dqt */
            size_t k = 0;
            while (k < sl) {
                int pq = seg[k] >> 4, tq = seg[k] & 15; k++;
                if (tq > 3) { SETERR("bad DQT index"); goto done; }
                if (k + (pq ? 128 : 64) > sl) { SETERR("truncated DQT"); goto done; }
                for (int z = 0; z < 64; z++) {
                    unsigned v = pq ? ((seg[k] << 8) | seg[k + 1]) : seg[k];
                    k += pq ? 2 : 1;
                    j->qt[tq][ZZ[z]] = (uint16_t)v;
                }
                j->qt_present[tq] = 1;
            }
        } else if (m == 0xC4) { /* get_dht */
            size_t k = 0;
            while (k + 17 <= sl) {
                int tc = seg[k] >> 4, th = seg[k] & 15; k++;
                if (th > 3 || tc > 1) { SETERR("bad DHT index"); goto done; }
                hufftab *t = tc ? &hs->ac[th] : &hs->dc[th];
                int n = 0; t->bits[0] = 0;
                for (int l = 1; l <= 16; l++) { t->bits[l] = seg[k++]; n += t->bits[l]; }
                if (n > 256 || k + n > sl) { SETERR("bad DHT counts"); goto done; }
                memcpy(t->vals, seg + k, n); k += n;
                t->present = 1; huff_build(t);
            }
        } else if (m == 0xC0 || m == 0xC1 || m == 0xC2) { /* get_sof */
            if (have_sof) { SETERR("duplicate SOF"); goto done; }
            if (sl < 6) { SETERR("short SOF"); goto done; }
            if (seg[0] != 8) { SETERR("unsupported sample precision %d", seg[0]); goto done; }
            j->progressive = (m == 0xC2);
            j->height = (seg[1] << 8) | seg[2]; j->width = (seg[3] << 8) | seg[4]; j->ncomp = seg[5];
            if (j->width <= 0 || j->height <= 0) { SETERR("empty image"); goto done; }
            if (j->width > ORC_JPEG_MAX_DIMENSION || j->height > ORC_JPEG_MAX_DIMENSION) { SETERR("Maximum supported image dimension is %d pixels", ORC_JPEG_MAX_DIMENSION); goto done; }
            if (j->ncomp != 1 && j->ncomp != 3) { SETERR("unsupported component count %d", j->ncomp); goto done; }
            if (sl < (size_t)(6 + 3 * j->ncomp)) { SETERR("short SOF"); goto done; }
            for (int c = 0; c < j->ncomp; c++) {
                j->cid[c] = seg[6 + 3 * c]; j->hs[c] = seg[7 + 3 * c] >> 4; j->vs[c] = seg[7 + 3 * c] & 15; j->tq[c] = seg[8 + 3 * c];
                if (j->hs[c] < 1 || j->hs[c] > 4 || j->vs[c] < 1 || j->vs[c] > 4 || j->tq[c] > 3) { SETERR("bad sampling factors"); goto done; }
            }
            if (j->ncomp == 1) { j->hs[0] = j->vs[0] = 1; } /* single-component: MCU is one block whatever the header says */
            setup_geometry(j);
            for (int c = 0; c < j->ncomp; c++) {
                j->coef[c] = (int16_t *)calloc((size_t)j->bw[c] * j->bh[c] * 64, sizeof(int16_t));
                if (!j->coef[c]) { SETERR("out of memory"); goto done; }
            }
            have_sof = 1;
        } else if (m == 0xDD) {
            if (sl >= 2) j->restart_interval = (seg[0] << 8) | seg[1];
        } else if (m == 0xDA) { /* get_sos + entropy-coded segment */
            if (!have_sof) { SETERR("SOS before SOF"); goto done; }
            scanhdr s; memset(&s, 0, sizeof(s));
            s.ns = seg[0];
            if (s.ns < 1 || s.ns > j->ncomp || sl < (size_t)(4 + 2 * s.ns)) { SETERR("bad SOS"); goto done; }
            for (int k = 0; k < s.ns; k++) {
                int id = seg[1 + 2 * k], ci = -1;
                for (int c = 0; c < j->ncomp; c++) if (j->cid[c] == id) ci = c;
                if (ci < 0) { SETERR("SOS names unknown component"); goto done; }
                s.ci[k] = ci; s.td[k] = seg[2 + 2 * k] >> 4; s.ta[k] = seg[2 + 2 * k] & 15;
                if (s.td[k] > 3 || s.ta[k] > 3) { SETERR("bad table selector"); goto done; }
            }
            if (s.ns > 1) { /* jdinput.c per_scan_setup: an interleaved MCU holds at most D_MAX_BLOCKS_IN_MCU (10) blocks */
                int blocks = 0;
                for (int k = 0; k < s.ns; k++) blocks += j->hs[s.ci[k]] * j->vs[s.ci[k]];
                if (blocks > 10) { SETERR("bad MCU size: %d blocks in an interleaved MCU", blocks); goto done; }
            }
            s.Ss = seg[1 + 2 * s.ns]; s.Se = seg[2 + 2 * s.ns]; s.Ah = seg[3 + 2 * s.ns] >> 4; s.Al = seg[3 + 2 * s.ns] & 15;
            if (!j->progressive) { s.Ss = 0; s.Se = 63; s.Ah = s.Al = 0; }
            else if (s.Ss > s.Se || s.Se > 63 || (s.Ss == 0 && s.Se != 0) || (s.Ss > 0 && s.ns != 1) || s.Al > 13) { SETERR("bad progressive scan parameters"); goto done; }
            if (j->nscans < 64) {
                int *e = j->scan_script[j->nscans++];
                e[0] = s.ns; e[1] = s.Ss; e[2] = s.Se; e[3] = s.Ah; e[4] = s.Al;
                e[5] = s.ci[0]; e[6] = s.ns > 1 ? s.ci[1] : -1; e[7] = s.ns > 2 ? s.ci[2] : -1;
            }
            const uint8_t *next = NULL;
            if (decode_scan(j, &s, hs, d + i + 2 + L, d + len, &next, err)) goto done;
            i = (size_t)(next - d);
            continue;
        } else if ((m >= 0xE0 && m <= 0xEF) || m == 0xFE) {
            if (m == 0xE0 && sl >= 5 && !memcmp(seg, "JFIF\0", 5)) j->jfif = 1;
            if (m == 0xEE && sl >= 12 && !memcmp(seg, "Adobe", 5)) { j->adobe = 1; j->adobe_transform = seg[11]; }
            if (m == 0xE2 && sl >= 12 && !memcmp(seg, "ICC_PROFILE\0", 12)) append_bytes(&j->icc_markers, &j->icc_len, d + i, 2 + L);
            else if (!(m == 0xE0 && j->jfif) && m != 0xEE) append_bytes(&j->markers, &j->markers_len, d + i, 2 + L);
        } else if (m >= 0xC3 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {
            SETERR("unsupported JPEG process (SOF%d)", m - 0xC0); goto done;
        }
        i += 2 + L;
    }
    if (!have_sof || j->nscans == 0) { SETERR("no image data"); goto done; }
    for (int c = 0; c < j->ncomp; c++) if (!j->qt_present[j->tq[c]]) { SETERR("missing quantisation table %d", j->tq[c]); goto done; }
    rc = 0;
done:
    for (int t = 0; t < 4; t++) { free(hs->dc[t].look); free(hs->ac[t].look); }
    free(hs);
    if (rc) orc_jpeg_free(j);
    return rc;
}

void orc_jpeg_idct_component(const orc_jpeg *j, int c, uint8_t *plane)
{
    int stride = j->bw[c] * 8;
    uint8_t px[64];
    for (int by = 0; by < j->bh[c]; by++) for (int bx = 0; bx < j->bw[c]; bx++) {
        orc_idct_islow(j->coef[c] + ((size_t)by * j->bw[c] + bx) * 64, j->qt[j->tq[c]], px);
        for (int y = 0; y < 8; y++) memcpy(plane + (size_t)(by * 8 + y) * stride + bx * 8, px + 8 * y, 8);
    }
}

/* jdapimin/jdmaster with out_color_space = jpeg_color_space, do_fancy_upsampling = TRUE:
 * what libcaesium's jpeg::lossy hands to the compressor (SURVEY.md §3.4-i). */
int orc_jpeg_decode_native(const orc_jpeg *j, uint8_t *planes[ORC_MAX_COMP], char err[256])
{
    for (int c = 0; c < j->ncomp; c++) {
        int stride = j->bw[c] * 8;
        uint8_t *tmp = (uint8_t *)malloc((size_t)stride * j->bh[c] * 8);
        if (!tmp) { SETERR("out of memory"); return -1; }
        orc_jpeg_idct_component(j, c, tmp);
        int hx = j->hmax / j->hs[c], vx = j->vmax / j->vs[c];
        if (j->hmax % j->hs[c] || j->vmax % j->vs[c]) { free(tmp); SETERR("fractional sampling ratio unsupported"); return -1; }
        uint8_t *o = planes[c]; int W = j->width, H = j->height;
        if (hx == 1 && vx == 1) { for (int y = 0; y < H; y++) memcpy(o + (size_t)y * W, tmp + (size_t)y * stride, W); }
        else if (hx == 2 && vx == 1) orc_upsample_h2v1_fancy(tmp, j->cw[c], j->ch[c], stride, o, W, H, W);
        else if (hx == 2 && vx == 2) orc_upsample_h2v2_fancy(tmp, j->cw[c], j->ch[c], stride, o, W, H, W);
        else if (hx == 1 && vx == 2) orc_upsample_h1v2_fancy(tmp, j->cw[c], j->ch[c], stride, o, W, H, W);
        else orc_upsample_box(tmp, j->cw[c], j->ch[c], stride, hx, vx, o, W, H, W);
        free(tmp);
    }
    return 0;
}

/* jccoefct.c compress_first_pass / jctrans.c compress_output dummy-block rule:
 * AC = 0, DC = DC of the previous block of the same MCU row group. */
static void fill_dummy_blocks(orc_jpeg *j)
{
    for (int c = 0; c < j->ncomp; c++) {
        int bw = j->bw[c], hsf = j->hs[c];
        for (int r = 0; r < j->bh[c]; r++) {
            int16_t *row = j->coef[c] + (size_t)r * bw * 64;
            if (r < j->rbh[c]) {
                for (int x = j->rbw[c]; x < bw; x++) { memset(row + (size_t)x * 64, 0, 128); row[(size_t)x * 64] = row[(size_t)(x - 1) * 64]; }
            } else {
                const int16_t *prev = row - (size_t)bw * 64;
                for (int m = 0; m < bw / hsf; m++) {
                    int16_t dc = prev[(size_t)(m * hsf + hsf - 1) * 64];
                    for (int b = 0; b < hsf; b++) { memset(row + (size_t)(m * hsf + b) * 64, 0, 128); row[(size_t)(m * hsf + b) * 64] = dc; }
                }
            }
        }
    }
}

/* jcparam.c jpeg_set_defaults/jpeg_set_colorspace + libcaesium set_chroma_subsampling,
 * then jcsample -> jcdctmgr forward_DCT for every real block. */
int orc_jpeg_forward(const uint8_t *const planes[ORC_MAX_COMP], int width, int height, int ncomp,
                     const orc_jpeg_params *p, orc_jpeg *o, char err[256])
{
    memset(o, 0, sizeof(*o));
    if (width < 1 || height < 1 || width > ORC_JPEG_MAX_DIMENSION || height > ORC_JPEG_MAX_DIMENSION) { SETERR("invalid target dimensions"); return -1; }  /* jcinit.c initial_setup */
    o->width = width; o->height = height; o->ncomp = ncomp; o->progressive = p->progressive;
    int lh = 1, lv = 1;
    if (ncomp == 3) {
        switch (p->subsampling) {
            case 444: lh = 1; lv = 1; break;
            case 422: lh = 2; lv = 1; break;
            case 411: lh = 4; lv = 1; break;
            case 420: case 0: lh = 2; lv = 2; break;
            default: SETERR("bad chroma subsampling %d", p->subsampling); return -1;
        }
    } else if (ncomp != 1) { SETERR("unsupported component count %d", ncomp); return -1; }
    for (int c = 0; c < ncomp; c++) { o->cid[c] = c + 1; o->hs[c] = c ? 1 : lh; o->vs[c] = c ? 1 : lv; o->tq[c] = c ? 1 : 0; }
    orc_quant_table(p->quality, 0, o->qt[0]); o->qt_present[0] = 1;
    if (ncomp == 3) { orc_quant_table(p->quality, 1, o->qt[1]); o->qt_present[1] = 1; }
    setup_geometry(o);
    o->jfif = 1;
    for (int c = 0; c < ncomp; c++) {
        o->coef[c] = (int16_t *)calloc((size_t)o->bw[c] * o->bh[c] * 64, sizeof(int16_t));
        int pw = o->rbw[c] * 8, ph = o->rbh[c] * 8;
        uint8_t *ds = (uint8_t *)malloc((size_t)pw * ph);
        if (!o->coef[c] || !ds) { free(ds); orc_jpeg_free(o); SETERR("out of memory"); return -1; }
        orc_downsample(planes[c], width, height, width, o->hmax / o->hs[c], o->vmax / o->vs[c], ds, pw, ph);
        uint8_t px[64]; int32_t dct[64];
        for (int by = 0; by < o->rbh[c]; by++) for (int bx = 0; bx < o->rbw[c]; bx++) {
            for (int y = 0; y < 8; y++) memcpy(px + 8 * y, ds + (size_t)(by * 8 + y) * pw + bx * 8, 8);
            orc_fdct_islow(px, dct);
            orc_quantize(dct, o->qt[o->tq[c]], o->coef[c] + ((size_t)by * o->bw[c] + bx) * 64);
        }
        free(ds);
    }
    fill_dummy_blocks(o);
    return 0;
}

/* ------------------------------------------------------------------------- */
/* Entropy encoder: jchuff.c (sequential) + jcphuff.c (progressive), always   */
/* with optimize_coding (two passes: gather statistics, emit).               */
/* ------------------------------------------------------------------------- */
typedef struct { uint8_t *buf; size_t len, cap; uint64_t acc; int nbits; } bitwr;

static void bw_byte(bitwr *w, unsigned c)
{
    if (w->len + 2 > w->cap) { w->cap = w->cap ? w->cap * 2 : 1 << 16; w->buf = (uint8_t *)realloc(w->buf, w->cap); }
    w->buf[w->len++] = (uint8_t)c;
}
static void bw_raw(bitwr *w, const void *src, size_t n) { const uint8_t *s = (const uint8_t *)src; for (size_t i = 0; i < n; i++) bw_byte(w, s[i]); }
static void bw_u16(bitwr *w, unsigned v) { bw_byte(w, v >> 8); bw_byte(w, v & 0xFF); }
static void bw_bits(bitwr *w, unsigned code, int size)
{   /* jchuff.c emit_bits: MSB first, 0xFF byte-stuffed with 0x00 */
    if (size == 0) return;
    w->acc = (w->acc << size) | (code & ((1u << size) - 1)); w->nbits += size;
    while (w->nbits >= 8) { unsigned c = (unsigned)(w->acc >> (w->nbits - 8)) & 0xFF; bw_byte(w, c); if (c == 0xFF) bw_byte(w, 0); w->nbits -= 8; }
}
static void bw_flush(bitwr *w) { if (w->nbits) bw_bits(w, 0x7F, 8 - w->nbits); w->acc = 0; w->nbits = 0; } /* flush_bits: pad with ones */

typedef struct { uint8_t bits[17]; uint8_t vals[256]; unsigned code[256]; uint8_t size[256]; int nvals; } enctab;

/* jchuff.c jpeg_gen_optimal_table (Annex K.2 with the IJG 16-bit length limiter) */
static void gen_optimal_table(enctab *t, const long freq_in[257])
{
    uint8_t bits[33]; int codesize[257], others[257]; long freq[257];
    memset(bits, 0, sizeof(bits)); memset(codesize, 0, sizeof(codesize));
    memcpy(freq, freq_in, sizeof(freq));
    for (int i = 0; i < 257; i++) others[i] = -1;
    freq[256] = 1;
    for (;;) {
        int c1 = -1, c2 = -1; long v = 1000000000L;
        for (int i = 0; i <= 256; i++) if (freq[i] && freq[i] <= v) { v = freq[i]; c1 = i; }
        v = 1000000000L;
        for (int i = 0; i <= 256; i++) if (freq[i] && freq[i] <= v && i != c1) { v = freq[i]; c2 = i; }
        if (c2 < 0) break;
        freq[c1] += freq[c2]; freq[c2] = 0;
        codesize[c1]++; while (others[c1] >= 0) { c1 = others[c1]; codesize[c1]++; }
        others[c1] = c2;
        codesize[c2]++; while (others[c2] >= 0) { c2 = others[c2]; codesize[c2]++; }
    }
    for (int i = 0; i <= 256; i++) if (codesize[i]) bits[codesize[i] > 32 ? 32 : codesize[i]]++;
    for (int i = 32; i > 16; i--) while (bits[i] > 0) {
        int jx = i - 2; while (bits[jx] == 0) jx--;
        bits[i] -= 2; bits[i - 1]++; bits[jx + 1] += 2; bits[jx]--;
    }
    int i = 16; while (bits[i] == 0) i--; bits[i]--;
    memset(t, 0, sizeof(*t));
    memcpy(t->bits, bits, 17);
    int pidx = 0;
    for (int l = 1; l <= 32; l++) for (int s = 0; s <= 255; s++) if (codesize[s] == l) t->vals[pidx++] = (uint8_t)s;
    t->nvals = pidx;
    /* jchuff.c jpeg_make_c_derived_tbl */
    unsigned code = 0; int k = 0;
    for (int l = 1; l <= 16; l++) { for (int n = 0; n < t->bits[l]; n++, k++) { t->code[t->vals[k]] = code++; t->size[t->vals[k]] = (uint8_t)l; } code <<= 1; }
}

static inline int nbits_of(int v) { int n = 0; while (v) { n++; v >>= 1; } return n; }

typedef struct {
    int gather; bitwr *w;
    long *dc_freq[4], *ac_freq[4]; const enctab *dc_tab[4], *ac_tab[4];
    int last_dc[4];
    /* progressive state (jcphuff.c phuff_entropy_encoder) */
    int Ss, Se, Ah, Al, ac_tbl; unsigned eobrun; unsigned BE; uint8_t corr[1000 + 64];
} encstate;

static inline void emit_sym(encstate *e, int is_ac, int tbl, int sym)
{
    if (e->gather) { (is_ac ? e->ac_freq[tbl] : e->dc_freq[tbl])[sym]++; }
    else { const enctab *t = is_ac ? e->ac_tab[tbl] : e->dc_tab[tbl]; bw_bits(e->w, t->code[sym], t->size[sym]); }
}
static inline void emit_bits_e(encstate *e, unsigned v, int n) { if (!e->gather) bw_bits(e->w, v, n); }
static void emit_buffered(encstate *e, const uint8_t *b, unsigned n) { if (e->gather) return; for (unsigned i = 0; i < n; i++) bw_bits(e->w, b[i], 1); }
static void emit_eobrun(encstate *e)
{   /* jcphuff.c emit_eobrun */
    if (e->eobrun > 0) {
        int nb = nbits_of((int)e->eobrun) - 1;
        emit_sym(e, 1, e->ac_tbl, nb << 4);
        if (nb) emit_bits_e(e, e->eobrun, nb);
        e->eobrun = 0;
        emit_buffered(e, e->corr, e->BE); e->BE = 0;
    }
}

/* jchuff.c encode_one_block / htest_one_block */
static void enc_block_seq(encstate *e, const int16_t *blk, int ci, int dctbl, int actbl)
{
    int temp = blk[0] - e->last_dc[ci], temp2 = temp; e->last_dc[ci] = blk[0];
    if (temp < 0) { temp = -temp; temp2--; }
    int nb = nbits_of(temp);
    emit_sym(e, 0, dctbl, nb);
    if (nb) emit_bits_e(e, (unsigned)temp2, nb);
    int r = 0;
    for (int k = 1; k < 64; k++) {
        temp = blk[ZZ[k]];
        if (temp == 0) { r++; continue; }
        while (r > 15) { emit_sym(e, 1, actbl, 0xF0); r -= 16; }
        temp2 = temp; if (temp < 0) { temp = -temp; temp2--; }
        nb = nbits_of(temp);
        emit_sym(e, 1, actbl, (r << 4) + nb);
        emit_bits_e(e, (unsigned)temp2, nb);
        r = 0;
    }
    if (r > 0) emit_sym(e, 1, actbl, 0);
}

static void enc_block_dc_first(encstate *e, const int16_t *blk, int ci, int dctbl)
{   /* jcphuff.c encode_mcu_DC_first */
    int t2 = blk[0] >> e->Al; /* arithmetic shift (IRIGHT_SHIFT) */
    int temp = t2 - e->last_dc[ci]; e->last_dc[ci] = t2;
    t2 = temp; if (temp < 0) { temp = -temp; t2--; }
    int nb = nbits_of(temp);
    emit_sym(e, 0, dctbl, nb);
    if (nb) emit_bits_e(e, (unsigned)t2, nb);
}

static void enc_block_ac_first(encstate *e, const int16_t *blk)
{   /* jcphuff.c encode_mcu_AC_first */
    int r = 0;
    for (int k = e->Ss; k <= e->Se; k++) {
        int temp = blk[ZZ[k]], temp2;
        if (temp == 0) { r++; continue; }
        if (temp < 0) { temp = -temp; temp >>= e->Al; temp2 = ~temp; } else { temp >>= e->Al; temp2 = temp; }
        if (temp == 0) { r++; continue; }
        if (e->eobrun > 0) emit_eobrun(e);
        while (r > 15) { emit_sym(e, 1, e->ac_tbl, 0xF0); r -= 16; }
        int nb = nbits_of(temp);
        emit_sym(e, 1, e->ac_tbl, (r << 4) + nb);
        emit_bits_e(e, (unsigned)temp2, nb);
        r = 0;
    }
    if (r > 0) { e->eobrun++; if (e->eobrun == 0x7FFF) emit_eobrun(e); }
}

static void enc_block_ac_refine(encstate *e, const int16_t *blk)
{   /* jcphuff.c encode_mcu_AC_refine */
    int absv[64], EOB = 0;
    for (int k = e->Ss; k <= e->Se; k++) { int t = blk[ZZ[k]]; if (t < 0) t = -t; t >>= e->Al; absv[k] = t; if (t == 1) EOB = k; }
    int r = 0; unsigned BR = 0; uint8_t *BRbuf = e->corr + e->BE;
    for (int k = e->Ss; k <= e->Se; k++) {
        int t = absv[k];
        if (t == 0) { r++; continue; }
        while (r > 15 && k <= EOB) {
            emit_eobrun(e);
            emit_sym(e, 1, e->ac_tbl, 0xF0); r -= 16;
            emit_buffered(e, BRbuf, BR); BRbuf = e->corr; BR = 0;
        }
        if (t > 1) { BRbuf[BR++] = (uint8_t)(t & 1); continue; }
        emit_eobrun(e);
        emit_sym(e, 1, e->ac_tbl, (r << 4) + 1);
        emit_bits_e(e, blk[ZZ[k]] < 0 ? 0 : 1, 1);
        emit_buffered(e, BRbuf, BR); BRbuf = e->corr; BR = 0;
        r = 0;
    }
    if (r > 0 || BR > 0) {
        e->eobrun++; e->BE += BR;
        if (e->eobrun == 0x7FFF || e->BE > (1000 - 64 + 1)) emit_eobrun(e);
    }
}

typedef struct { int ns, ci[3], Ss, Se, Ah, Al; } scandef;

/* run one scan in gather or emit mode */
static void run_scan(const orc_jpeg *j, const scandef *s, encstate *e)
{
    memset(e->last_dc, 0, sizeof(e->last_dc)); e->eobrun = 0; e->BE = 0;
    e->Ss = s->Ss; e->Se = s->Se; e->Ah = s->Ah; e->Al = s->Al;
    int inter = s->ns > 1, c0 = s->ci[0];
    int mx_n = inter ? j->mcux : j->rbw[c0], my_n = inter ? j->mcuy : j->rbh[c0];
    for (int my = 0; my < my_n; my++) for (int mx = 0; mx < mx_n; mx++)
        for (int i = 0; i < s->ns; i++) {
            int c = s->ci[i], nbx = inter ? j->hs[c] : 1, nby = inter ? j->vs[c] : 1, tbl = c ? 1 : 0;
            for (int by = 0; by < nby; by++) for (int bx = 0; bx < nbx; bx++) {
                int row = inter ? my * j->vs[c] + by : my, col = inter ? mx * j->hs[c] + bx : mx;
                const int16_t *blk = j->coef[c] + ((size_t)row * j->bw[c] + col) * 64;
                if (!j->progressive) enc_block_seq(e, blk, c, tbl, tbl);
                else if (s->Ss == 0) { if (s->Ah == 0) enc_block_dc_first(e, blk, c, tbl); else emit_bits_e(e, (unsigned)(blk[0] >> s->Al) & 1, 1); }
                else { e->ac_tbl = tbl; if (s->Ah == 0) enc_block_ac_first(e, blk); else enc_block_ac_refine(e, blk); }
            }
        }
    if (j->progressive && s->Ss > 0) emit_eobrun(e);
}

static void write_dht(bitwr *w, int tc, int th, const enctab *t)
{   /* jcmarker.c emit_dht */
    bw_u16(w, 0xFFC4); bw_u16(w, 2 + 1 + 16 + t->nvals);
    bw_byte(w, (tc << 4) | th);
    for (int l = 1; l <= 16; l++) bw_byte(w, t->bits[l]);
    bw_raw(w, t->vals, t->nvals);
}

int orc_jpeg_write(const orc_jpeg *j, const orc_jpeg_params *p, const orc_jpeg *meta, uint8_t **out, size_t *out_len, char err[256])
{
    bitwr w; memset(&w, 0, sizeof(w));
    orc_jpeg jj = *j; jj.progressive = p->progressive; /* geometry identical; coefficient arrays shared, not owned */
    /* jcmarker.c write_file_header: SOI + JFIF APP0 (version 1.01, density 1:1 aspect) */
    bw_u16(&w, 0xFFD8);
    { static const uint8_t jfif[] = { 0xFF, 0xE0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0 }; bw_raw(&w, jfif, sizeof(jfif)); }
    if (meta) {
        if (p->keep_metadata && meta->markers_len) bw_raw(&w, meta->markers, meta->markers_len);
        if ((p->keep_metadata || p->preserve_icc) && meta->icc_len) bw_raw(&w, meta->icc_markers, meta->icc_len);
    }
    /* write_frame_header: all quantisation tables in one DQT segment (mozjpeg emit_multi_dqt; matches samples/j0.JPG) */
    {
        int used[4] = { 0, 0, 0, 0 }, seglen = 2;
        for (int c = 0; c < j->ncomp; c++) used[j->tq[c]] = 1;
        int prec[4];
        for (int t = 0; t < 4; t++) { prec[t] = 0; if (used[t]) { for (int i = 0; i < 64; i++) if (j->qt[t][i] > 255) prec[t] = 1; seglen += 1 + (prec[t] ? 128 : 64); } }
        bw_u16(&w, 0xFFDB); bw_u16(&w, seglen);
        for (int t = 0; t < 4; t++) if (used[t]) {
            bw_byte(&w, (prec[t] << 4) | t);
            for (int z = 0; z < 64; z++) { unsigned v = j->qt[t][ZZ[z]]; if (prec[t]) bw_byte(&w, v >> 8); bw_byte(&w, v & 0xFF); }
        }
    }
    bw_u16(&w, p->progressive ? 0xFFC2 : 0xFFC0); bw_u16(&w, 8 + 3 * j->ncomp); bw_byte(&w, 8);
    bw_u16(&w, j->height); bw_u16(&w, j->width); bw_byte(&w, j->ncomp);
    for (int c = 0; c < j->ncomp; c++) { bw_byte(&w, j->cid[c]); bw_byte(&w, (j->hs[c] << 4) | j->vs[c]); bw_byte(&w, j->tq[c]); }

    /* scan script: sequential = one interleaved scan; progressive = the 8-scan mozjpeg-style script of samples/j0.JPG */
    scandef sc[16]; int ns = 0;
    if (!p->progressive) { sc[0].ns = j->ncomp; for (int c = 0; c < j->ncomp; c++) sc[0].ci[c] = c; sc[0].Ss = 0; sc[0].Se = 63; sc[0].Ah = sc[0].Al = 0; ns = 1; }
    else {
        sc[ns].ns = j->ncomp; for (int c = 0; c < j->ncomp; c++) sc[ns].ci[c] = c; sc[ns].Ss = 0; sc[ns].Se = 0; sc[ns].Ah = 0; sc[ns].Al = 0; ns++;
        sc[ns] = (scandef){ 1, { 0, 0, 0 }, 1, 2, 0, 1 }; ns++;
        sc[ns] = (scandef){ 1, { 0, 0, 0 }, 3, 63, 0, 1 }; ns++;
        for (int c = 1; c < j->ncomp; c++) { sc[ns] = (scandef){ 1, { c, 0, 0 }, 1, 63, 0, 1 }; ns++; }
        for (int c = 0; c < j->ncomp; c++) { sc[ns] = (scandef){ 1, { c, 0, 0 }, 1, 63, 1, 0 }; ns++; }
    }
    long *freq = (long *)malloc(sizeof(long) * 257 * 4);
    for (int si = 0; si < ns; si++) {
        const scandef *s = &sc[si];
        encstate e; memset(&e, 0, sizeof(e));
        enctab dct[2], act[2]; int need_dc[2] = { 0, 0 }, need_ac[2] = { 0, 0 };
        memset(freq, 0, sizeof(long) * 257 * 4);
        e.dc_freq[0] = freq; e.dc_freq[1] = freq + 257; e.ac_freq[0] = freq + 514; e.ac_freq[1] = freq + 771;
        int dc_refine = p->progressive && s->Ss == 0 && s->Ah != 0;
        if (!dc_refine) {
            e.gather = 1; run_scan(&jj, s, &e);
            for (int i = 0; i < s->ns; i++) {
                int t = s->ci[i] ? 1 : 0;
                if (!p->progressive || s->Ss == 0) need_dc[t] = 1;
                if (!p->progressive || s->Ss > 0) need_ac[t] = 1;
            }
            for (int t = 0; t < 2; t++) {
                if (need_dc[t]) { gen_optimal_table(&dct[t], e.dc_freq[t]); write_dht(&w, 0, t, &dct[t]); }
                if (need_ac[t]) { gen_optimal_table(&act[t], e.ac_freq[t]); write_dht(&w, 1, t, &act[t]); }
            }
        }
        /* jcmarker.c emit_sos */
        bw_u16(&w, 0xFFDA); bw_u16(&w, 6 + 2 * s->ns); bw_byte(&w, s->ns);
        for (int i = 0; i < s->ns; i++) {
            int c = s->ci[i], td = c ? 1 : 0, ta = c ? 1 : 0;
            if (p->progressive) { if (s->Ss == 0) { ta = 0; if (s->Ah != 0) td = 0; } else td = 0; }
            bw_byte(&w, j->cid[c]); bw_byte(&w, (td << 4) | ta);
        }
        bw_byte(&w, s->Ss); bw_byte(&w, s->Se); bw_byte(&w, (s->Ah << 4) | s->Al);
        e.gather = 0; e.w = &w; e.dc_tab[0] = &dct[0]; e.dc_tab[1] = &dct[1]; e.ac_tab[0] = &act[0]; e.ac_tab[1] = &act[1];
        run_scan(&jj, s, &e);
        bw_flush(&w);
    }
    free(freq);
    bw_u16(&w, 0xFFD9);
    if (!w.buf) { SETERR("out of memory"); return -1; }
    *out = w.buf; *out_len = w.len;
    return 0;
}

int orc_jpeg_lossy(const uint8_t *data, size_t len, const orc_jpeg_params *p, uint8_t **out, size_t *out_len, char err[256])
{
    orc_jpeg in, fw; int rc = -1;
    if (orc_jpeg_read(data, len, &in, err)) return -1;
    uint8_t *planes[ORC_MAX_COMP] = { 0, 0, 0, 0 };
    for (int c = 0; c < in.ncomp; c++) planes[c] = (uint8_t *)malloc((size_t)in.width * in.height);
    memset(&fw, 0, sizeof(fw));
    if (orc_jpeg_decode_native(&in, planes, err)) goto done;
    if (orc_jpeg_forward((const uint8_t *const *)planes, in.width, in.height, in.ncomp, p, &fw, err)) goto done;
    rc = orc_jpeg_write(&fw, p, &in, out, out_len, err);
done:
    for (int c = 0; c < ORC_MAX_COMP; c++) free(planes[c]);
    orc_jpeg_free(&fw); orc_jpeg_free(&in);
    return rc;
}

int orc_jpeg_lossless(const uint8_t *data, size_t len, const orc_jpeg_params *p, uint8_t **out, size_t *out_len, char err[256])
{   /* jpegtran-style: jpeg_read_coefficients -> jpeg_copy_critical_parameters -> jpeg_write_coefficients */
    orc_jpeg in;
    if (orc_jpeg_read(data, len, &in, err)) return -1;
    fill_dummy_blocks(&in);
    int rc = orc_jpeg_write(&in, p, &in, out, out_len, err);
    orc_jpeg_free(&in);
    /* jpeg_copy_critical_parameters also copies the source's JFIF version (major 1 or 2) and density: patch them into the
       APP0 orc_jpeg_write put at out[2] (version at +9, units at +11, X / Y density at +12 / +14) */
    for (size_t i = 2; rc == 0 && i + 4 <= len && data[i] == 0xFF; ) {
        unsigned m = data[i + 1];
        if (m == 0xFF) { i++; continue; }
        size_t L = ((size_t)data[i + 2] << 8) | data[i + 3];
        if (m == 0xDA || m == 0xD9 || L < 2 || i + 2 + L > len) break;
        if (m == 0xE0 && L >= 16 && !memcmp(data + i + 4, "JFIF\0", 5)) {
            if (data[i + 9] == 1 || data[i + 9] == 2) memcpy(*out + 11, data + i + 9, 2);
            memcpy(*out + 13, data + i + 11, 5);
            break;
        }
        i += 2 + L;
    }
    return rc;
}
