/* jpeg_trellis_core.h -- the rule of the JPEG encoder's rate-distortion (trellis) quantiser, written once for every party that
 * has to agree on it: the device kernel and its host driver (jpeg_kernels.cu, jpeg_device.cu) and the scalar oracle
 * (oracle/jpeg_oracle.c, plain C -- hence no namespace and no C++ in this file).  All arithmetic is integer (64-bit
 * accumulators, fixed-point lambda and weights), so device and oracle agree bit for bit whatever the compiler contracts.
 *
 * One 8x8 block at a time, in zigzag order k = 0..63, with one quantisation table Q[k] (1..32767):
 *   x[k]      the ISLOW FDCT output (scaled by 8), |x| <= 2^13 for 8-bit samples
 *   p[k]      the plain level, round half away from zero: sign(x) * floor((|x| + 4 Q) / (8 Q))   (jcdctmgr.c quantize)
 *   DC        t[0] = p[0]; DC is never traded across blocks
 *   AC        t[k] = 0 where p[k] = 0; where p[k] != 0 the candidates are 0, |p[k]| and 2^s - 1 for 1 <= s < nbits(|p[k]|)
 *             (the largest magnitude of each smaller size category), each with the sign of x[k]
 *   weight    W[k]   = floor(2^31 / Q[k]^2)
 *   lambda    S      = sum_{k>=1} x[k]^2,   lam = floor(63 * JT_LAMBDA_A * 2^24 / (63 * JT_LAMBDA_B + S))
 *             (lambda = A / (B + S / 63) in units of 2^-24)
 *   distortion dist(k, c) = ((((x[k] - 8 c Q[k])^2 * W[k]) >> 20) * lam) >> 19     (unsigned 64-bit; about
 *             2^16 * lambda * (x - 8 c Q)^2 / Q^2, i.e. in units of 2^-16 bit)
 *   rate      a non-zero level c at k after a run of r zeros since the previous non-zero AC level (or since DC) costs
 *             floor(r / 16) * L(0xF0) + L(((r mod 16) << 4) | size(c)) + size(c) bits, and the block pays L(0x00) (EOB) when
 *             its last non-zero AC level is below 63 (also when it has none); L is the code length of the JPEG standard's
 *             Annex K AC table -- K.5 for component 0, K.6 for the others -- and 16 for a symbol those tables do not list.
 *             Progressive output is costed with the same sequential model.  Rate is counted in units of 2^-16 bit (JT_RATE_SHIFT).
 *   result    the AC levels that minimise  sum_{k>=1} dist(k, t[k]) + rate , by dynamic programming over the position of the
 *             previous non-zero level.  Ties: positions are visited in increasing k; at each, candidates from the largest
 *             magnitude down and predecessors from the nearest back to DC, and the end of block from the last non-zero level
 *             back to DC; a later option replaces the kept one only when strictly cheaper.
 * Hence DC = p[0], every AC level is 0 or has the sign of p[k] and |t[k]| <= |p[k]|, and a block whose plain AC levels are all
 * zero comes out as the plain block.
 *
 * B = round(2^16.5) is the value commonly documented as mozjpeg's default (lambda_log_scale2 = 16.5).  A = 2^20 is tuned: with
 * mozjpeg's documented A = 2^14.75 and this rule (Annex K rates, 1/Q^2 weights) files shrink by 6-13 % but lose 1-1.5 dB of PSNR,
 * a BD-rate (bytes at equal PSNR) of +5 to +6 % on the 1280x720 synthetic seeds 0-2 it was tuned on; A = 2^20 gives
 * -0.2 to -0.3 % there (DESIGN.md §4.10).  Every
 * product above fits 64 bits for A <= 2^20: (e^2 W >> 20) * lam <= x^2 2^11 * 63 A 2^24 / S <= 2^61. */
#ifndef JPEG_TRELLIS_CORE_H
#define JPEG_TRELLIS_CORE_H
#include <stdint.h>

#if defined(__CUDACC__)
#define JT_HD static __host__ __device__ __forceinline__
#else
#define JT_HD static inline
#endif
#define JT_H static inline          /* host only: the table set-up */

#define JT_LAMBDA_A 1048576
#define JT_LAMBDA_B 92682
#define JT_RATE_SHIFT 16

/* per quantisation table: the weights, the table itself and the Annex K AC code lengths of its component class */
typedef struct {
    uint32_t w[64];         /* zigzag: floor(2^31 / Q^2) */
    uint16_t q[64];         /* zigzag */
    uint8_t len[256];       /* AC symbol -> Annex K code length */
} JtTable;

/* Annex K.5 (luminance) and K.6 (chrominance) AC tables: symbols with codes shorter than 16 bits, by increasing length; every
 * other symbol has a 16-bit code (or none) */
JT_H void jt_ac_lengths(int chroma, uint8_t len[256])
{
    static const uint8_t lum_n[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0};
    static const uint8_t lum_v[37] = {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61,
                                      0x07, 0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52,
                                      0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82};
    static const uint8_t chr_n[16] = {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0};
    static const uint8_t chr_v[43] = {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61,
                                      0x71, 0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33,
                                      0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1};
    const uint8_t *n = chroma ? chr_n : lum_n, *v = chroma ? chr_v : lum_v;
    for (int i = 0; i < 256; i++) len[i] = 16;
    int j = 0;
    for (int l = 1; l <= 16; l++)
        for (int i = 0; i < n[l - 1]; i++) len[v[j++]] = (uint8_t)l;
}

/* qt_zigzag: the table in zigzag order; chroma: 0 for component 0's table, 1 otherwise */
JT_H void jt_make_table(const uint16_t qt_zigzag[64], int chroma, JtTable *t)
{
    for (int k = 0; k < 64; k++) {
        const uint32_t q = qt_zigzag[k] ? qt_zigzag[k] : 1;
        t->q[k] = (uint16_t)q;
        t->w[k] = (uint32_t)((1ull << 31) / ((unsigned long long)q * q));
    }
    jt_ac_lengths(chroma, t->len);
}

JT_HD int jt_nbits(int v) { int n = 0; while (v) { n++; v >>= 1; } return n; }

JT_HD int jt_plain(int x, int q)
{
    const int ax = x < 0 ? -x : x, l = (ax + 4 * q) / (8 * q);
    return x < 0 ? -l : l;
}

JT_HD uint32_t jt_lambda(unsigned long long S)
{
    return (uint32_t)((63ull * JT_LAMBDA_A << 24) / (63ull * JT_LAMBDA_B + S));
}

/* c >= 0 is a magnitude; the error is taken against |x| */
JT_HD unsigned long long jt_dist(int ax, int c, int q, uint32_t w, uint32_t lam)
{
    const long long e = (long long)ax - 8ll * c * q;
    return ((((unsigned long long)(e * e) * w) >> 20) * lam) >> 19;
}

/* The trellis over one block.  x (zigzag, read) and out (zigzag, written) may be the same array: every x[k] is read before
 * out[k] is written.  The scratch arrays hold one entry per visited non-zero position (at most 64) at index i * stride, so a
 * device caller can interleave the blocks of its threads ([position][thread]); G is int64, pos / pred / size are bytes. */
JT_HD void jt_trellis_block(const int16_t *x, const JtTable *t, int16_t *out,
                            long long *G, uint8_t *pos, uint8_t *pred, uint8_t *size, int stride)
{
    const int dc = jt_plain(x[0], t->q[0]);
    unsigned long long S = 0;
    int any = 0;
    for (int k = 1; k < 64; k++) { const int v = x[k]; S += (unsigned long long)((long long)v * v); any |= jt_plain(v, t->q[k]); }
    if (!any) {                         /* all plain AC levels are zero: the plain block */
        for (int k = 1; k < 64; k++) out[k] = 0;
        out[0] = (int16_t)dc;
        return;
    }
    const uint32_t lam = jt_lambda(S);
    const long long U = 1ll << JT_RATE_SHIFT, zrl = (long long)t->len[0xF0] << JT_RATE_SHIFT;
    int n = 0;                          /* entry 0 = DC (position 0) */
    G[0] = 0; pos[0] = 0; pred[0] = 0; size[0] = 0;
    long long Z = 0;                    /* sum of dist(m, 0) over 1 <= m < k */
    for (int k = 1; k < 64; k++) {
        const int v = x[k], q = t->q[k], av = v < 0 ? -v : v;
        const uint32_t w = t->w[k];
        const long long d0 = (long long)jt_dist(av, 0, q, w, lam);
        const int ap = (av + 4 * q) / (8 * q);
        if (ap) {
            const int nb = jt_nbits(ap);
            long long best = 0; int bb = -1, bs = 0;
            for (int s = nb; s >= 1; s--) {
                const int c = s == nb ? ap : (1 << s) - 1;
                const long long dc_ = (long long)jt_dist(av, c, q, w, lam) + ((long long)s << JT_RATE_SHIFT);
                for (int b = n; b >= 0; b--) {
                    const int r = k - pos[b * stride] - 1;
                    const long long cost = G[b * stride] + Z + dc_ + (r >> 4) * zrl + ((long long)t->len[((r & 15) << 4) | s] << JT_RATE_SHIFT);
                    if (bb < 0 || cost < best) { best = cost; bb = b; bs = s; }
                }
            }
            n++;
            G[n * stride] = best - (Z + d0);
            pos[n * stride] = (uint8_t)k; pred[n * stride] = (uint8_t)bb; size[n * stride] = (uint8_t)bs;
        }
        Z += d0;
    }
    const long long eob = (long long)t->len[0x00] * U;
    long long best = 0; int bb = -1;
    for (int b = n; b >= 0; b--) {
        const long long cost = G[b * stride] + (pos[b * stride] < 63 ? eob : 0);
        if (bb < 0 || cost < best) { best = cost; bb = b; }
    }
    int cur = 63;                       /* out[cur + 1 ..] are written */
    for (int b = bb; b > 0; b = pred[b * stride]) {
        const int k = pos[b * stride], s = size[b * stride];
        const int v = x[k], ap = ((v < 0 ? -v : v) + 4 * t->q[k]) / (8 * t->q[k]);
        const int c = s == jt_nbits(ap) ? ap : (1 << s) - 1;
        for (int m = cur; m > k; m--) out[m] = 0;
        out[k] = (int16_t)(v < 0 ? -c : c);
        cur = k - 1;
    }
    for (int m = cur; m >= 1; m--) out[m] = 0;
    out[0] = (int16_t)dc;
}

#endif /* JPEG_TRELLIS_CORE_H */
