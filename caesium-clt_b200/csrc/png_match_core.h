// png_match_core.h -- K7 phase 1 (fixed pixel / row candidates, SURVEY.md §8a row a8; libcaesium png::lossless -> oxipng -> deflate,
// caesium-clt's src/compressor.rs:428,436-437) written once as __host__ __device__ code: png_kernels.cu's k_png_match and the CPU
// emulation in tests/emul/match_emul.cpp run the same bodies.
//
// One CTA owns MATCH_T consecutive positions of the filtered stream.  For every candidate distance the comparison "byte q of the
// CTA's stretch equals the byte `distance` before it" is evaluated ONCE per byte and kept as a bit array (MATCH_WORDS 32-bit words:
// the stretch plus the 258 bytes a match may run past it); the match length at a position is then the run of ones that starts at
// its bit -- a funnel shift and a count-trailing-zeros instead of a byte-compare loop per position and candidate.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define PM_HD __host__ __device__ __forceinline__
#else
#define PM_HD inline
#endif

namespace b200 {
namespace pm {

constexpr int MATCH_T = 256;                         // positions per CTA
constexpr int MATCH_MAX = 258;                       // longest DEFLATE match
constexpr int MATCH_WORDS = 18;                      // bits 0 .. 575: position 255 may look at bits 255 .. 255 + 257 + 31, and word k + 1 is read with word k
constexpr int MATCH_BITS = MATCH_WORDS * 32;
constexpr int NCAND = 10;
constexpr int NEAR_BACK = 24;                        // the near window starts this many bytes before the stretch (distances up to 3 pixels of 8 bytes)
constexpr int ROW_SLACK = 8;                         // the row-above window starts stride + 8 before the stretch (distance stride + bpp)
constexpr int WIN0 = NEAR_BACK + MATCH_BITS, WIN1 = 2 * ROW_SLACK + MATCH_BITS, WIN2 = MATCH_BITS;

// the candidate distances, in the order ties are resolved (earlier wins)
PM_HD void candidates(int bpp, int stride, int (&cand)[NCAND])
{
    cand[0] = bpp; cand[1] = 1; cand[2] = 2 * bpp; cand[3] = stride; cand[4] = stride - bpp; cand[5] = stride + bpp; cand[6] = 3 * bpp; cand[7] = 2; cand[8] = 3; cand[9] = 2 * stride;
}
// offset of the byte `cand[c]` before stretch byte 0 inside its window (w0: near, w1: row above, w2: two rows up) and which window
PM_HD int window_of(int c) { return (c >= 3 && c <= 5) ? 1 : c == 9 ? 2 : 0; }
PM_HD int window_base(int c, int d, int stride) { return (c >= 3 && c <= 5) ? ROW_SLACK + (stride - d) : c == 9 ? 0 : NEAR_BACK - d; }

// four byte comparisons at once: bit b of the result is set iff byte b of x equals byte b of y
PM_HD uint32_t eq_nibble(uint32_t x, uint32_t y)
{
    const uint32_t d = x ^ y;                                         // zero bytes = equal bytes
    const uint32_t z = ~((((d & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | d) | 0x7F7F7F7Fu);   // 0x80 in every zero byte of d
    return ((z >> 7) * 0x01020408u) >> 24;                            // bits 0, 8, 16, 24 gathered into bits 0..3 (no carries: the partial products do not overlap)
}

PM_HD int ctz32(uint32_t v)
{
#if defined(__CUDA_ARCH__)
    return __ffs((int)v) - 1;
#else
    return __builtin_ctz(v);
#endif
}
PM_HD uint32_t bits_from(const uint32_t *words, int j)
{   // 32 bits of the array starting at bit j
    const int k = j >> 5, b = j & 31;
#if defined(__CUDA_ARCH__)
    return __funnelshift_r(words[k], words[k + 1], b);
#else
    return b ? (uint32_t)((((uint64_t)words[k + 1] << 32) | words[k]) >> b) : words[k];
#endif
}
// length of the run of ones starting at bit j, at most maxlen (maxlen <= MATCH_MAX, j < MATCH_T)
PM_HD int run_from(const uint32_t *words, int j, int maxlen)
{
    int len = 0;
    while (len < maxlen) {
        const uint32_t t = ~bits_from(words, j + len);
        if (t) { len += ctz32(t); break; }
        len += 32;
    }
    return len < maxlen ? len : maxlen;
}
// best (length << 16 | distance) of stretch position t (stream position i), 0 if no candidate reaches length 3.  Written without
// early exits: a later candidate replaces the best only if it is strictly longer, so evaluating all ten gives the same answer as
// stopping at the first one that reaches maxlen, and the common case (a run shorter than 32) is one funnel shift and one bit scan.
PM_HD uint32_t best_of(const uint32_t (*eq)[MATCH_WORDS], const int (&cand)[NCAND], int t, unsigned long long i, int maxlen)
{
    int bl = 0, bd = 0;
    const int reach = i > 32768ull ? 32768 : (int)i;                  // the largest usable distance at this position
    if (maxlen >= 3) {
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int c = 0; c < NCAND; c++) {
            const int d = cand[c];
            const uint32_t inv = ~bits_from(eq[c], t);
            int l = inv ? ctz32(inv) : run_from(eq[c], t, maxlen);
            l = l < maxlen ? l : maxlen;
            const bool better = d >= 1 && d <= reach && l > bl;       // earlier candidate wins ties
            bl = better ? l : bl; bd = better ? d : bd;
        }
    }
    return bl >= 3 ? ((uint32_t)bl << 16) | (uint32_t)bd : 0u;
}

} // namespace pm
} // namespace b200
