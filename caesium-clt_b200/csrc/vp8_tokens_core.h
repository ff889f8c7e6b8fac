// vp8_tokens_core.h -- the residual tokens of a VP8 key frame (RFC 6386 section 13: coefficient token tree, bands, contexts) written once
// as __host__ __device__ code: the device generates the frame's decisions in parallel, one thread per macroblock (vp8_kernels.cu,
// k_vp8_tokens), the host writer (vp8_host.cpp) runs the same bodies when it is handed levels instead of tokens (the stage entry
// points and the CPU tests), so both produce the same decision list.  WebP leg of caesium::convert_in_memory
// (caesium-clt's src/compressor.rs:288-292 -> libcaesium webp::compress -> libwebp's token pass).
//
// What makes the pass parallel: a block's context is "did the block above / to the left have coded coefficients", which is a
// property of those blocks' levels alone -- a 25-bit mask per macroblock (mb_mask), computable before any token exists.  With the
// masks of the macroblock above and to the left in hand, a macroblock's decisions depend on nothing else.
//
// A decision is recorded as 16 bits: bit 0 = the decision; bit 15 clear: bits 1..11 = probability slot ((type * 8 + band) * 3 + ctx)
// * 11 + node; bit 15 set: bits 1..8 = a fixed probability (extra bits of the large categories, signs).
#pragma once
#include <cstdint>
#if defined(__SSE2__) && !defined(__CUDACC__)
#include <emmintrin.h>
#endif

#if defined(__CUDACC__)
#define VT_HD __host__ __device__ __forceinline__
#else
#define VT_HD inline
#endif

namespace b200 {
namespace vt {

constexpr int kNumProbs = 4 * 8 * 3 * 11;
constexpr int kMaxDecisionsPerMb = 7300;             // 25 blocks x at most 1 + 16 x 18 decisions

VT_HD int band_of(int n)
{   // coefficient index -> band (RFC 6386 13.3); index 16 is only ever used to pick a context that is not read
    return n < 4 ? n : n == 4 ? 6 : n == 5 ? 4 : n == 6 ? 5 : n < 15 ? 6 : n == 15 ? 7 : 0;
}
VT_HD int slot(int type, int band, int ctx) { return ((type * 8 + band) * 3 + ctx) * 11; }

// index of the last non-zero level at or after `first`, -1 if none
VT_HD int last_nonzero(const int16_t *lv, int first)
{
#if defined(__SSE2__) && !defined(__CUDACC__)
    const __m128i z = _mm_setzero_si128();
    const __m128i a = _mm_cmpeq_epi16(_mm_loadu_si128(reinterpret_cast<const __m128i *>(lv)), z), b = _mm_cmpeq_epi16(_mm_loadu_si128(reinterpret_cast<const __m128i *>(lv + 8)), z);
    unsigned nz = ~(unsigned)_mm_movemask_epi8(_mm_packs_epi16(a, b)) & 0xFFFFu;        // bit i: lv[i] != 0
    nz &= ~((1u << first) - 1u);
    return nz ? 31 - __builtin_clz(nz) : -1;
#else
    for (int i = 15; i >= first; i--) if (lv[i]) return i;
    return -1;
#endif
}

// Sink interface: node(slot, bit) for a tree decision coded with the frame's probability of that slot, fixed(bit, prob) for a
// decision with a constant probability.
// One block's tokens; `lv` = 16 levels in zigzag order.  Returns the "has coded coefficients" flag (the neighbours' context).
template <class Sink> VT_HD int put_block(Sink &w, const int16_t *lv, int type, int first, int ctx)
{
    const int last = last_nonzero(lv, first);
    int p = slot(type, band_of(first), ctx);
    w.node(p, last >= 0);
    if (last < 0) return 0;
    for (int n = first; n < 16;) {
        const int c = lv[n++], v = c < 0 ? -c : c;
        w.node(p + 1, v != 0);
        if (!v) { p = slot(type, band_of(n), 0); continue; }           // a zero is never followed by an end-of-block check
        w.node(p + 2, v > 1);
        if (v == 1) p = slot(type, band_of(n), 1);
        else {
            w.node(p + 3, v > 4);
            if (v <= 4) { w.node(p + 4, v != 2); if (v != 2) w.node(p + 5, v == 4); }
            else {
                w.node(p + 6, v > 10);
                if (v <= 10) {
                    w.node(p + 7, v > 6);
                    if (v <= 6) w.fixed(v == 6, 159); else { w.fixed(v >= 9, 165); w.fixed(!(v & 1), 145); }
                } else {
                    // DCT_CAT3..6: bases 11, 19, 35, 67; extra-bit probabilities of RFC 6386 13.2
                    const int cat = v < 19 ? 0 : v < 35 ? 1 : v < 67 ? 2 : 3;
                    const int nbits = cat == 0 ? 3 : cat == 1 ? 4 : cat == 2 ? 5 : 11, base = cat == 0 ? 11 : cat == 1 ? 19 : cat == 2 ? 35 : 67;
                    w.node(p + 8, cat >> 1); w.node(p + 9 + (cat >> 1), cat & 1);
                    for (int i = nbits - 1, t = 0; i >= 0; i--, t++) {
                        int pr;
                        if (cat == 0) pr = t == 0 ? 173 : t == 1 ? 148 : 140;
                        else if (cat == 1) pr = t == 0 ? 176 : t == 1 ? 155 : t == 2 ? 140 : 135;
                        else if (cat == 2) pr = t == 0 ? 180 : t == 1 ? 157 : t == 2 ? 141 : t == 3 ? 134 : 130;
                        else pr = t < 2 ? 254 : t == 2 ? 243 : t == 3 ? 230 : t == 4 ? 196 : t == 5 ? 177 : t == 6 ? 153 : t == 7 ? 140 : t == 8 ? 133 : t == 9 ? 130 : 129;
                        w.fixed(((v - base) >> i) & 1, pr);
                    }
                }
            }
            p = slot(type, band_of(n), 2);
        }
        w.fixed(c < 0, 128);
        if (n == 16) break;
        w.node(p, n <= last);
        if (n > last) break;
    }
    return 1;
}

// which of a macroblock's 25 blocks have coded coefficients: bit 0 Y2, bits 1..16 the Y blocks (AC only: their DC lives in Y2; all
// 16 coefficients in a B_PRED macroblock, which has no Y2), bits 17..20 U, 21..24 V
VT_HD uint32_t mb_mask(const int16_t *lv, bool bpred = false)
{
    uint32_t m = !bpred && last_nonzero(lv, 0) >= 0 ? 1u : 0u;
    for (int b = 0; b < 16; b++) if (last_nonzero(lv + 16 * (1 + b), bpred ? 0 : 1) >= 0) m |= 1u << (1 + b);
    for (int b = 0; b < 8; b++) if (last_nonzero(lv + 16 * (17 + b), 0) >= 0) m |= 1u << (17 + b);
    return m;
}

// every residual block of one macroblock in coding order (13): the contexts of its first row / column of blocks come from the masks
// of the macroblock above / to the left (0 at the frame edge and for a skipped macroblock).  Bit 0 of `top` / `left_mask` is the Y2
// context, which is NOT the neighbour's own bit 0: a decoder updates it on 16x16-coded macroblocks only (y2_carry).  A B_PRED
// macroblock codes no Y2 and its luma blocks as type 3 from coefficient 0.
template <class Sink> VT_HD void walk_mb(Sink &sk, const int16_t *lv, uint32_t top, uint32_t left_mask, bool bpred = false)
{
    uint8_t t[9], l[9];
    for (int x = 0; x < 4; x++) { t[x] = (uint8_t)((top >> (1 + 12 + x)) & 1u); l[x] = (uint8_t)((left_mask >> (1 + 4 * x + 3)) & 1u); }
    for (int x = 0; x < 2; x++) {
        t[4 + x] = (uint8_t)((top >> (17 + 2 + x)) & 1u); l[4 + x] = (uint8_t)((left_mask >> (17 + 2 * x + 1)) & 1u);
        t[6 + x] = (uint8_t)((top >> (21 + 2 + x)) & 1u); l[6 + x] = (uint8_t)((left_mask >> (21 + 2 * x + 1)) & 1u);
    }
    t[8] = (uint8_t)(top & 1u); l[8] = (uint8_t)(left_mask & 1u);
    if (!bpred) t[8] = l[8] = (uint8_t)put_block(sk, lv, 1, 0, t[8] + l[8]);
    for (int b = 0; b < 16; b++) { const int x = b & 3, y = b >> 2; t[x] = l[y] = (uint8_t)put_block(sk, lv + 16 * (1 + b), bpred ? 3 : 0, bpred ? 0 : 1, t[x] + l[y]); }
    for (int c = 0; c < 2; c++)
        for (int b = 0; b < 4; b++) { const int x = 4 + 2 * c + (b & 1), y = 4 + 2 * c + (b >> 1); t[x] = l[y] = (uint8_t)put_block(sk, lv + 16 * (17 + 4 * c + b), 2, 0, t[x] + l[y]); }
}

// The Y2 contexts of macroblock mb = y * mbw + x: the Y2 flag of the nearest 16x16-coded macroblock above in the same column
// (y2top[mb]) and to the left in the same row (y2left[mb]), 0 if there is none.  A skipped 16x16 macroblock's flag is 0 (its mask
// is); a B_PRED macroblock, skipped or not, leaves the flag alone.  modes[4 * mb] == 4 marks B_PRED.  Every column and every row
// is an independent walk: the device runs one thread per column and one per row.
VT_HD void y2_carry_col(const uint32_t *mask, const uint8_t *modes, int mbw, int mbh, int col, uint8_t *y2top)
{
    uint8_t c = 0;
    for (int y = 0; y < mbh; y++) {
        const int mb = y * mbw + col;
        y2top[mb] = c;
        if (modes[4 * mb] != 4) c = (uint8_t)(mask[mb] & 1u);
    }
}
VT_HD void y2_carry_row(const uint32_t *mask, const uint8_t *modes, int mbw, int row, uint8_t *y2left)
{
    uint8_t c = 0;
    for (int x = 0; x < mbw; x++) {
        const int mb = row * mbw + x;
        y2left[mb] = c;
        if (modes[4 * mb] != 4) c = (uint8_t)(mask[mb] & 1u);
    }
}
// a neighbour's mask with bit 0 replaced by the carried Y2 context
VT_HD uint32_t with_y2(uint32_t mask, uint8_t y2) { return (mask & ~1u) | (y2 & 1u); }

VT_HD uint16_t rec_node(int s, bool bit) { return (uint16_t)((s << 1) | (bit ? 1 : 0)); }
VT_HD uint16_t rec_fixed(bool bit, int prob) { return (uint16_t)(0x8000u | ((unsigned)prob << 1) | (bit ? 1u : 0u)); }

} // namespace vt
} // namespace b200
