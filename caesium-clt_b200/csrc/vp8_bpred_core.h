/* vp8_bpred_core.h -- the rules of 4x4 intra prediction (B_PRED) in VP8 key frames, written once for every party that has to agree
 * on them: the decoder (vp8_decode.cpp: predictors and edges), the device encoder (vp8_kernels.cu, k_vp8_encode_bpred), the host
 * writer (vp8_host.cpp: the sub-block mode tree), the CPU emulation (tests/emul) and the scalar twin (oracle/webp_bpred_oracle.c,
 * plain C -- hence no namespace and no C++ in this file).
 *
 * Sub-block modes, in the decoder's numbering: 0 DC, 1 TM, 2 VE, 3 HE, 4 RD, 5 VR, 6 LD, 7 VL, 8 HD, 9 HU.  A 16x16-coded
 * macroblock gives its neighbours the sub-block mode context of its luma mode (DC, TM, V, H = 0, 1, 2, 3), and the frame's edges give DC.
 *
 * The encoder's decision, all in integers so that the device and every host restatement agree bit for bit:
 *   rate        vp8bp_block_rate: the token tree of one block (vt::put_block's walk) priced with VP8BP_BIT_COST over the DEFAULT
 *               coefficient probabilities, with the real non-zero contexts inside the macroblock and context 0 across its edges;
 *               the Y2 block takes context 0
 *   sub-block   score = 256 * SSE(source - reconstruction) + lambda * (rate + cost of the mode in the tree of its (above, left)
 *               context); the lowest score wins, a tie goes to the lower mode
 *   macroblock  B_PRED iff the sum of its 16 sub-block scores + lambda * cost(B_PRED flag) < the 16x16 score, where the 16x16 mode is
 *               the one the i16-only encoder picks (least prediction SSE) and its score is 256 * SSE + lambda * (Y2 + 16 AC block
 *               rates + the mode's tree and flag); chroma is the same in both arms and stays out of the comparison
 *   lambda      vp8bp_lambda(y1 AC quantiser) = max(1, 3 q^2 >> 7) */
#ifndef VP8_BPRED_CORE_H
#define VP8_BPRED_CORE_H
#include <stdint.h>
#include "vp8_tables.h"

#if defined(__CUDACC__)
#define VP8BP_HD static __host__ __device__ __forceinline__
#else
#define VP8BP_HD static inline
#endif

#ifdef __cplusplus
namespace b200 {
#endif

enum { VP8BP_NMODES = 10, VP8BP_YMODE = 4 /* modes[mb][0] of a B_PRED macroblock */, VP8BP_FLAG_PROB = 145 };

/* cost of a decision coded with probability-of-zero p / 256: VP8BP_BIT_COST[p] for a 0, [256 - p] for a 1, in 1/256 bit
 * (round(-256 log2(p / 256)); entry 0 is never read) */
VP8_TABLE(uint16_t, VP8BP_BIT_COST, [256], {
    2048, 2048, 1792, 1642, 1536, 1454, 1386, 1329, 1280, 1236, 1198, 1162, 1130, 1101, 1073, 1048,
    1024, 1002,  980,  961,  942,  924,  906,  890,  874,  859,  845,  831,  817,  804,  792,  780,
     768,  757,  746,  735,  724,  714,  705,  695,  686,  676,  668,  659,  650,  642,  634,  626,
     618,  611,  603,  596,  589,  582,  575,  568,  561,  555,  548,  542,  536,  530,  524,  518,
     512,  506,  501,  495,  490,  484,  479,  474,  468,  463,  458,  453,  449,  444,  439,  434,
     430,  425,  420,  416,  412,  407,  403,  399,  394,  390,  386,  382,  378,  374,  370,  366,
     362,  358,  355,  351,  347,  343,  340,  336,  333,  329,  326,  322,  319,  315,  312,  309,
     305,  302,  299,  296,  292,  289,  286,  283,  280,  277,  274,  271,  268,  265,  262,  259,
     256,  253,  250,  247,  245,  242,  239,  236,  234,  231,  228,  226,  223,  220,  218,  215,
     212,  210,  207,  205,  202,  200,  197,  195,  193,  190,  188,  185,  183,  181,  178,  176,
     174,  171,  169,  167,  164,  162,  160,  158,  156,  153,  151,  149,  147,  145,  143,  140,
     138,  136,  134,  132,  130,  128,  126,  124,  122,  120,  118,  116,  114,  112,  110,  108,
     106,  104,  102,  101,   99,   97,   95,   93,   91,   89,   87,   86,   84,   82,   80,   78,
      77,   75,   73,   71,   70,   68,   66,   64,   63,   61,   59,   58,   56,   54,   53,   51,
      49,   48,   46,   44,   43,   41,   40,   38,   36,   35,   33,   32,   30,   28,   27,   25,
      24,   22,   21,   19,   18,   16,   15,   13,   12,   10,    9,    7,    6,    4,    3,    1,
})
/* per node of VP8_YMODES_INTRA4, the modes (bit m) that lie under its 1 branch: encoding mode m codes bit (mask >> m) & 1 */
VP8_TABLE(uint16_t, VP8BP_TREE_ONES, [9], {0x3FE, 0x3FC, 0x3F8, 0x3C0, 0x030, 0x020, 0x380, 0x300, 0x200})

VP8BP_HD uint32_t vp8bp_bit(int bit, int p) { return VP8_TAB(VP8BP_BIT_COST)[bit ? 256 - p : p]; }
VP8BP_HD int vp8bp_lambda(int q_ac) { const int l = (3 * q_ac * q_ac) >> 7; return l < 1 ? 1 : l; }
VP8BP_HD uint64_t vp8bp_score(uint32_t sse, uint32_t rate, int lambda) { return 256ull * sse + (uint64_t)lambda * rate; }

/* ---- the 10 sub-block predictors -----------------------------------------------------------------------------------------------
 * e[0] = X (top-left), e[1..8] = A..H (the row above and the four above-right), e[9..12] = I..L (the left column); out = 4x4 raster */
#define VP8BP_AVG3(a, b, c) ((uint8_t)(((a) + 2 * (b) + (c) + 2) >> 2))
#define VP8BP_AVG2(a, b) ((uint8_t)(((a) + (b) + 1) >> 1))
VP8BP_HD void vp8bp_pred4(int mode, const uint8_t *e, uint8_t *out)
{
    const int X = e[0], A = e[1], B = e[2], C = e[3], D = e[4], E = e[5], F = e[6], G = e[7], H = e[8], I = e[9], J = e[10], K = e[11], L = e[12];
#define DST(x, y) out[(x) + 4 * (y)]
    switch (mode) {
        case 0: { const uint8_t dc = (uint8_t)((A + B + C + D + I + J + K + L + 4) >> 3); for (int i = 0; i < 16; i++) out[i] = dc; break; }
        case 1:
            for (int y = 0; y < 4; y++) for (int x = 0; x < 4; x++) { const int v = e[1 + x] + e[9 + y] - X; DST(x, y) = (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v); }
            break;
        case 2: {
            const uint8_t v0 = VP8BP_AVG3(X, A, B), v1 = VP8BP_AVG3(A, B, C), v2 = VP8BP_AVG3(B, C, D), v3 = VP8BP_AVG3(C, D, E);
            for (int y = 0; y < 4; y++) { DST(0, y) = v0; DST(1, y) = v1; DST(2, y) = v2; DST(3, y) = v3; }
            break;
        }
        case 3: {
            const uint8_t v0 = VP8BP_AVG3(X, I, J), v1 = VP8BP_AVG3(I, J, K), v2 = VP8BP_AVG3(J, K, L), v3 = VP8BP_AVG3(K, L, L);
            for (int x = 0; x < 4; x++) { DST(x, 0) = v0; DST(x, 1) = v1; DST(x, 2) = v2; DST(x, 3) = v3; }
            break;
        }
        case 4:
            DST(0, 3) = VP8BP_AVG3(J, K, L); DST(1, 3) = DST(0, 2) = VP8BP_AVG3(I, J, K); DST(2, 3) = DST(1, 2) = DST(0, 1) = VP8BP_AVG3(X, I, J);
            DST(3, 3) = DST(2, 2) = DST(1, 1) = DST(0, 0) = VP8BP_AVG3(A, X, I); DST(3, 2) = DST(2, 1) = DST(1, 0) = VP8BP_AVG3(B, A, X);
            DST(3, 1) = DST(2, 0) = VP8BP_AVG3(C, B, A); DST(3, 0) = VP8BP_AVG3(D, C, B); break;
        case 5:
            DST(0, 0) = DST(1, 2) = VP8BP_AVG2(X, A); DST(1, 0) = DST(2, 2) = VP8BP_AVG2(A, B); DST(2, 0) = DST(3, 2) = VP8BP_AVG2(B, C); DST(3, 0) = VP8BP_AVG2(C, D);
            DST(0, 3) = VP8BP_AVG3(K, J, I); DST(0, 2) = VP8BP_AVG3(J, I, X); DST(0, 1) = DST(1, 3) = VP8BP_AVG3(I, X, A); DST(1, 1) = DST(2, 3) = VP8BP_AVG3(X, A, B);
            DST(2, 1) = DST(3, 3) = VP8BP_AVG3(A, B, C); DST(3, 1) = VP8BP_AVG3(B, C, D); break;
        case 6:
            DST(0, 0) = VP8BP_AVG3(A, B, C); DST(1, 0) = DST(0, 1) = VP8BP_AVG3(B, C, D); DST(2, 0) = DST(1, 1) = DST(0, 2) = VP8BP_AVG3(C, D, E);
            DST(3, 0) = DST(2, 1) = DST(1, 2) = DST(0, 3) = VP8BP_AVG3(D, E, F); DST(3, 1) = DST(2, 2) = DST(1, 3) = VP8BP_AVG3(E, F, G);
            DST(3, 2) = DST(2, 3) = VP8BP_AVG3(F, G, H); DST(3, 3) = VP8BP_AVG3(G, H, H); break;
        case 7:
            DST(0, 0) = VP8BP_AVG2(A, B); DST(1, 0) = DST(0, 2) = VP8BP_AVG2(B, C); DST(2, 0) = DST(1, 2) = VP8BP_AVG2(C, D); DST(3, 0) = DST(2, 2) = VP8BP_AVG2(D, E);
            DST(0, 1) = VP8BP_AVG3(A, B, C); DST(1, 1) = DST(0, 3) = VP8BP_AVG3(B, C, D); DST(2, 1) = DST(1, 3) = VP8BP_AVG3(C, D, E); DST(3, 1) = DST(2, 3) = VP8BP_AVG3(D, E, F);
            DST(3, 2) = VP8BP_AVG3(E, F, G); DST(3, 3) = VP8BP_AVG3(F, G, H); break;
        case 8:
            DST(0, 0) = DST(2, 1) = VP8BP_AVG2(I, X); DST(0, 1) = DST(2, 2) = VP8BP_AVG2(J, I); DST(0, 2) = DST(2, 3) = VP8BP_AVG2(K, J); DST(0, 3) = VP8BP_AVG2(L, K);
            DST(3, 0) = VP8BP_AVG3(A, B, C); DST(2, 0) = VP8BP_AVG3(X, A, B); DST(1, 0) = DST(3, 1) = VP8BP_AVG3(I, X, A); DST(1, 1) = DST(3, 2) = VP8BP_AVG3(J, I, X);
            DST(1, 2) = DST(3, 3) = VP8BP_AVG3(K, J, I); DST(1, 3) = VP8BP_AVG3(L, K, J); break;
        default: /* 9: HU */
            DST(0, 0) = VP8BP_AVG2(I, J); DST(2, 0) = DST(0, 1) = VP8BP_AVG2(J, K); DST(2, 1) = DST(0, 2) = VP8BP_AVG2(K, L); DST(1, 0) = VP8BP_AVG3(I, J, K);
            DST(3, 0) = DST(1, 1) = VP8BP_AVG3(J, K, L); DST(3, 1) = DST(1, 2) = VP8BP_AVG3(K, L, L);
            DST(3, 2) = DST(2, 2) = DST(0, 3) = DST(1, 3) = DST(2, 3) = DST(3, 3) = (uint8_t)L; break;
    }
#undef DST
}

/* ---- edges ---------------------------------------------------------------------------------------------------------------------
 * The macroblock's border from the (unfiltered) reconstruction R of luma stride `s`: top[0] = top-left, top[1..16] = the row above,
 * top[17..20] = above-right; left[0..15].  Frame top row: 127 everywhere, top-left and above-right included.  Left frame edge: 129
 * (so also the top-left below the top row).  Last macroblock column: the above-right is the above row's pixel 15 repeated. */
VP8BP_HD void vp8bp_mb_border(const uint8_t *R, int s, int mbx, int mby, int mbw, uint8_t *top, uint8_t *left)
{
    const uint8_t *p = R + (long)mby * 16 * s + mbx * 16;
    if (mby == 0) { for (int i = 0; i < 21; i++) top[i] = 127; }
    else {
        top[0] = mbx ? p[-s - 1] : 129;
        for (int i = 0; i < 16; i++) top[1 + i] = p[-s + i];
        for (int i = 0; i < 4; i++) top[17 + i] = mbx < mbw - 1 ? p[-s + 16 + i] : p[-s + 15];
    }
    for (int j = 0; j < 16; j++) left[j] = mbx ? p[j * s - 1] : 129;
}
/* the 13 edge samples of sub-block (bx, by) (layout of vp8bp_pred4) from the border and the macroblock's reconstruction so far
 * (`cur`, stride cs).  For sub-block rows 1..3 of column 3 the above-right comes from the row above the MACROBLOCK (top[17..20]). */
VP8BP_HD void vp8bp_edges(const uint8_t *top, const uint8_t *left, const uint8_t *cur, int cs, int bx, int by, uint8_t *e)
{
    const int x0 = 4 * bx, y0 = 4 * by;
    if (by == 0) { for (int i = 0; i < 9; i++) e[i] = top[x0 + i]; }
    else {
        const uint8_t *a = cur + (y0 - 1) * cs;
        e[0] = bx ? a[x0 - 1] : left[y0 - 1];
        for (int i = 0; i < 4; i++) e[1 + i] = a[x0 + i];
        for (int i = 0; i < 4; i++) e[5 + i] = bx < 3 ? a[x0 + 4 + i] : top[17 + i];
    }
    for (int j = 0; j < 4; j++) e[9 + j] = bx ? cur[(y0 + j) * cs + x0 - 1] : left[y0 + j];
}

/* ---- rates ---------------------------------------------------------------------------------------------------------------------- */
VP8BP_HD int vp8bp_band(int n) { return n < 4 ? n : n == 4 ? 6 : n == 5 ? 4 : n == 6 ? 5 : n < 15 ? 6 : n == 15 ? 7 : 0; }
/* the tokens of one block (16 levels in zigzag order; type 0 = Y after Y2, 1 = Y2, 2 = chroma, 3 = Y with its DC), in 1/256 bit,
 * over the default probabilities; *nz = the block's "has coded coefficients" flag */
VP8BP_HD uint32_t vp8bp_block_rate(const int16_t *lv, int type, int first, int ctx, int *nz)
{
    const uint8_t *P = VP8_TAB(VP8_COEF_PROBS);
    int last = -1;
    for (int i = 15; i >= first; i--) if (lv[i]) { last = i; break; }
    int p = ((type * 8 + vp8bp_band(first)) * 3 + ctx) * 11;
    uint32_t r = vp8bp_bit(last >= 0, P[p]);
    *nz = last >= 0;
    if (last < 0) return r;
    for (int n = first; n < 16;) {
        const int c = lv[n++], v = c < 0 ? -c : c;
        r += vp8bp_bit(v != 0, P[p + 1]);
        if (!v) { p = ((type * 8 + vp8bp_band(n)) * 3 + 0) * 11; continue; }
        r += vp8bp_bit(v > 1, P[p + 2]);
        if (v == 1) p = ((type * 8 + vp8bp_band(n)) * 3 + 1) * 11;
        else {
            r += vp8bp_bit(v > 4, P[p + 3]);
            if (v <= 4) { r += vp8bp_bit(v != 2, P[p + 4]); if (v != 2) r += vp8bp_bit(v == 4, P[p + 5]); }
            else {
                r += vp8bp_bit(v > 10, P[p + 6]);
                if (v <= 10) {
                    r += vp8bp_bit(v > 6, P[p + 7]);
                    if (v <= 6) r += vp8bp_bit(v == 6, 159); else r += vp8bp_bit(v >= 9, 165) + vp8bp_bit(!(v & 1), 145);
                } else {
                    const int cat = v < 19 ? 0 : v < 35 ? 1 : v < 67 ? 2 : 3;
                    const int nbits = cat == 0 ? 3 : cat == 1 ? 4 : cat == 2 ? 5 : 11, base = cat == 0 ? 11 : cat == 1 ? 19 : cat == 2 ? 35 : 67;
                    r += vp8bp_bit(cat >> 1, P[p + 8]) + vp8bp_bit(cat & 1, P[p + 9 + (cat >> 1)]);
                    for (int i = nbits - 1, t = 0; i >= 0; i--, t++) {
                        int pr;
                        if (cat == 0) pr = t == 0 ? 173 : t == 1 ? 148 : 140;
                        else if (cat == 1) pr = t == 0 ? 176 : t == 1 ? 155 : t == 2 ? 140 : 135;
                        else if (cat == 2) pr = t == 0 ? 180 : t == 1 ? 157 : t == 2 ? 141 : t == 3 ? 134 : 130;
                        else pr = t < 2 ? 254 : t == 2 ? 243 : t == 3 ? 230 : t == 4 ? 196 : t == 5 ? 177 : t == 6 ? 153 : t == 7 ? 140 : t == 8 ? 133 : t == 9 ? 130 : 129;
                        r += vp8bp_bit(((v - base) >> i) & 1, pr);
                    }
                }
            }
            p = ((type * 8 + vp8bp_band(n)) * 3 + 2) * 11;
        }
        r += vp8bp_bit(c < 0, 128);
        if (n == 16) break;
        r += vp8bp_bit(n <= last, P[p]);
        if (n > last) break;
    }
    return r;
}

/* ---- modes ---------------------------------------------------------------------------------------------------------------------
 * Sub-block mode `mode` in the tree of context (above, left): calls emit(node probability, bit) for each decision.  The writer codes
 * these decisions; the cost below sums them. */
VP8BP_HD int vp8bp_bmode_bits(int above, int left, int mode, uint8_t *probs, uint8_t *bits)
{
    const uint8_t *pr = VP8_TAB(VP8_BMODES_PROBA)[above][left];
    int n = 0, node = 0;
    for (;;) {
        const int b = (VP8_TAB(VP8BP_TREE_ONES)[node] >> mode) & 1, next = VP8_TAB(VP8_YMODES_INTRA4)[2 * node + b];
        probs[n] = pr[node]; bits[n] = (uint8_t)b; n++;
        if (next <= 0) return n;
        node = next;
    }
}
VP8BP_HD uint32_t vp8bp_bmode_cost(int above, int left, int mode)
{
    uint8_t p[8], b[8];
    const int n = vp8bp_bmode_bits(above, left, mode, p, b);
    uint32_t r = 0;
    for (int i = 0; i < n; i++) r += vp8bp_bit(b[i], p[i]);
    return r;
}
/* a 16x16 luma mode (0 DC, 1 TM, 2 V, 3 H) with its "not B_PRED" flag */
VP8BP_HD uint32_t vp8bp_i16_cost(int ymode)
{
    const int tm_or_h = ymode == 1 || ymode == 3;
    return vp8bp_bit(1, VP8BP_FLAG_PROB) + vp8bp_bit(tm_or_h, 156) + (tm_or_h ? vp8bp_bit(ymode == 1, 128) : vp8bp_bit(ymode == 2, 163));
}

#ifdef __cplusplus
} /* namespace b200 */
#endif
#endif /* VP8_BPRED_CORE_H */
