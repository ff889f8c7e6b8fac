// png_kernels.cu -- K6 (row-filter selection) and K7 (LZ77 match finding) for the lossless PNG path, SURVEY.md §8a row a8:
// the device side of what oxipng 9.1.5 does behind libcaesium png::lossless (caesium-clt's src/compressor.rs:428,
// 436-437): for every filter strategy of the optimisation preset, filter all rows and run the compressor over them.
// Filtering reads only RAW neighbours (left, up, up-left), so unlike un-filtering it is embarrassingly parallel: one CTA
// per row scores the five candidate filters (MinSum / Entropy / Bigrams / BigEnt heuristics as histograms in shared
// memory) and writes the winner.  Match finding is per position over a fixed candidate set that suits filtered image data
// (pixel-multiple distances and the row above); parsing is sequential inside 4 KiB chunks, parallel across them.
// All integer/byte work, HBM-bound; no tensor cores.
#include <cuda_runtime.h>
#include <algorithm>
#include <cub/block/block_radix_sort.cuh>
#include <cmath>
#include <cstdint>
#include "png_kernels.h"
#include "png_match_core.h"
#include "png_zopfli_core.h"
#include "launch_timer.h"

namespace b200 {

void png_make_tlog(uint32_t *tlog, size_t n)
{
    tlog[0] = 0;
    for (size_t c = 1; c <= n; c++) tlog[c] = (uint32_t)llround((double)c * std::log2((double)c) * 1024.0);
}

__device__ __forceinline__ int paeth_pred(int a, int b, int c)
{
    const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}
// the five PNG filters of byte x of a row (PNG 9.2), computed from raw neighbours
__device__ __forceinline__ void five_filters(const uint8_t *__restrict__ row, const uint8_t *__restrict__ up, int x, int bpp, uint8_t v[5])
{
    const int cur = row[x], a = x >= bpp ? row[x - bpp] : 0, b = up ? up[x] : 0, c = (up && x >= bpp) ? up[x - bpp] : 0;
    v[0] = (uint8_t)cur; v[1] = (uint8_t)(cur - a); v[2] = (uint8_t)(cur - b); v[3] = (uint8_t)(cur - ((a + b) >> 1)); v[4] = (uint8_t)(cur - paeth_pred(a, b, c));
}

// One CTA per row.  The row and the row above are staged in shared memory with 16-byte loads (the five candidate filters read
// four neighbours per byte: from global memory that was four scattered byte loads per byte and kept the kernel at 1 % of the HBM
// roofline); scoring and the final write then work out of shared memory.
__device__ __forceinline__ void five_filters_sm(const uint8_t *__restrict__ row, const uint8_t *__restrict__ up, int x, int bpp, uint8_t v[5])
{   // row / up point at byte 0 of the staged rows, which are preceded by 16 zero bytes (so x - bpp may run off the left edge)
    const int cur = row[x], a = row[x - bpp], b = up[x], c = up[x - bpp];
    v[0] = (uint8_t)cur; v[1] = (uint8_t)(cur - a); v[2] = (uint8_t)(cur - b); v[3] = (uint8_t)(cur - ((a + b) >> 1)); v[4] = (uint8_t)(cur - paeth_pred(a, b, c));
}
__global__ void __launch_bounds__(1024) k_png_filter(const uint8_t *__restrict__ raw, uint8_t *__restrict__ filt, int h, int rb, int bpp, int strategy, const uint32_t *__restrict__ tlog,
                                                    int row_pitch)
{
    extern __shared__ __align__(16) uint32_t sm_all[];
    __shared__ unsigned long long score[5];
    __shared__ int chosen;
    uint8_t *srow = reinterpret_cast<uint8_t *>(sm_all) + 16, *sup = srow + row_pitch;       // 16 zero bytes in front of each staged row
    uint32_t *sm = reinterpret_cast<uint32_t *>(reinterpret_cast<uint8_t *>(sm_all) + 2 * row_pitch);
    const int y = blockIdx.x;
    const uint8_t *grow = raw + (size_t)y * rb, *gup = y ? grow - rb : nullptr;
    // stage with aligned 32-bit loads (rows start at arbitrary byte offsets: align the global side down, drop the bytes outside)
    for (int i = threadIdx.x; i < 4; i += blockDim.x) { reinterpret_cast<uint32_t *>(srow - 16)[i] = 0; reinterpret_cast<uint32_t *>(sup - 16)[i] = 0; }
    {
        const int lead = (int)((uintptr_t)grow & 3), nwords = (lead + rb + 3) / 4;
        const uint32_t *gw = reinterpret_cast<const uint32_t *>(grow - lead);
        for (int j = threadIdx.x; j < nwords; j += blockDim.x) {
            const uint32_t w = gw[j];
#pragma unroll
            for (int k = 0; k < 4; k++) { const int idx = 4 * j + k - lead; if (idx >= 0 && idx < rb) srow[idx] = (uint8_t)(w >> (8 * k)); }
        }
        if (gup) {
            const int lead2 = (int)((uintptr_t)gup & 3), nw2 = (lead2 + rb + 3) / 4;
            const uint32_t *gw2 = reinterpret_cast<const uint32_t *>(gup - lead2);
            for (int j = threadIdx.x; j < nw2; j += blockDim.x) {
                const uint32_t w = gw2[j];
#pragma unroll
                for (int k = 0; k < 4; k++) { const int idx = 4 * j + k - lead2; if (idx >= 0 && idx < rb) sup[idx] = (uint8_t)(w >> (8 * k)); }
            }
        } else for (int i = threadIdx.x; i < rb; i += blockDim.x) sup[i] = 0;
    }
    __syncthreads();
    uint8_t *out = filt + (size_t)y * (rb + 1);
    int f = strategy;
    if (strategy >= 5) {
        if (threadIdx.x < 5) score[threadIdx.x] = 0;
        const int words = strategy == PNGF_MINSUM ? 0 : (strategy == PNGF_BIGRAMS ? 5 * 2048 : (strategy == PNGF_BIGENT ? 5 * 4096 : 5 * 256));
        for (int i = threadIdx.x; i < words / 4; i += blockDim.x) reinterpret_cast<uint4 *>(sm)[i] = make_uint4(0, 0, 0, 0);      // sm is 16-byte aligned, words % 4 == 0
        __syncthreads();
        if (strategy == PNGF_MINSUM) {
            unsigned long long s5[5] = {0, 0, 0, 0, 0};
            for (int x = threadIdx.x; x < rb; x += blockDim.x) { uint8_t v[5]; five_filters_sm(srow, sup, x, bpp, v); for (int k = 0; k < 5; k++) s5[k] += (unsigned)abs((int)(int8_t)v[k]); }
            for (int k = 0; k < 5; k++) atomicAdd(&score[k], s5[k]);
        } else if (strategy == PNGF_ENTROPY || strategy == PNGF_BRUTE) {
            for (int x = threadIdx.x; x < rb; x += blockDim.x) { uint8_t v[5]; five_filters_sm(srow, sup, x, bpp, v); for (int k = 0; k < 5; k++) atomicAdd(&sm[k * 256 + v[k]], 1u); }
            __syncthreads();
            for (int i = threadIdx.x; i < 5 * 256; i += blockDim.x) if (sm[i]) atomicAdd(&score[i >> 8], (unsigned long long)tlog[sm[i]]);
        } else {
            for (int x = threadIdx.x; x + 1 < rb; x += blockDim.x) {
                uint8_t v[5], w[5]; five_filters_sm(srow, sup, x, bpp, v); five_filters_sm(srow, sup, x + 1, bpp, w);
                for (int k = 0; k < 5; k++) {
                    const unsigned bg = ((unsigned)v[k] << 8) | w[k];
                    if (strategy == PNGF_BIGRAMS) atomicOr(&sm[k * 2048 + (bg >> 5)], 1u << (bg & 31));
                    else atomicAdd(&sm[k * 4096 + (((bg * 2654435761u) >> 20) & 4095u)], 1u);
                }
            }
            __syncthreads();
            if (strategy == PNGF_BIGRAMS) { for (int i = threadIdx.x; i < 5 * 2048; i += blockDim.x) if (sm[i]) atomicAdd(&score[i >> 11], (unsigned long long)__popc(sm[i])); }
            else for (int i = threadIdx.x; i < 5 * 4096; i += blockDim.x) if (sm[i]) atomicAdd(&score[i >> 12], (unsigned long long)tlog[min(sm[i], (uint32_t)rb)]);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            const bool want_max = strategy == PNGF_ENTROPY || strategy == PNGF_BRUTE || strategy == PNGF_BIGENT;   // sum c*log2(c): larger = lower entropy
            int best = 0;
            for (int k = 1; k < 5; k++) if (want_max ? score[k] > score[best] : score[k] < score[best]) best = k;
            chosen = best;
        }
        __syncthreads();
        f = chosen;
    }
    if (threadIdx.x == 0) out[0] = (uint8_t)f;
    for (int x = threadIdx.x; x < rb; x += blockDim.x) { uint8_t v[5]; five_filters_sm(srow, sup, x, bpp, v); out[1 + x] = v[f]; }
}

// the same from global memory, for rows too long to stage (more than ~58 KB)
__global__ void __launch_bounds__(256) k_png_filter_wide(const uint8_t *__restrict__ raw, uint8_t *__restrict__ filt, int h, int rb, int bpp, int strategy, const uint32_t *__restrict__ tlog)
{
    extern __shared__ uint32_t sm[];
    __shared__ unsigned long long score[5];
    __shared__ int chosen;
    const int y = blockIdx.x;
    const uint8_t *row = raw + (size_t)y * rb, *up = y ? row - rb : nullptr;
    uint8_t *out = filt + (size_t)y * (rb + 1);
    int f = strategy;
    if (strategy >= 5) {
        if (threadIdx.x < 5) score[threadIdx.x] = 0;
        const int words = strategy == PNGF_MINSUM ? 0 : (strategy == PNGF_BIGRAMS ? 5 * 2048 : (strategy == PNGF_BIGENT ? 5 * 4096 : 5 * 256));
        for (int i = threadIdx.x; i < words; i += blockDim.x) sm[i] = 0;
        __syncthreads();
        if (strategy == PNGF_MINSUM) {
            unsigned long long s[5] = {0, 0, 0, 0, 0};
            for (int x = threadIdx.x; x < rb; x += blockDim.x) { uint8_t v[5]; five_filters(row, up, x, bpp, v); for (int k = 0; k < 5; k++) s[k] += (unsigned)abs((int)(int8_t)v[k]); }
            for (int k = 0; k < 5; k++) atomicAdd(&score[k], s[k]);
        } else if (strategy == PNGF_ENTROPY || strategy == PNGF_BRUTE) {
            for (int x = threadIdx.x; x < rb; x += blockDim.x) { uint8_t v[5]; five_filters(row, up, x, bpp, v); for (int k = 0; k < 5; k++) atomicAdd(&sm[k * 256 + v[k]], 1u); }
            __syncthreads();
            for (int i = threadIdx.x; i < 5 * 256; i += blockDim.x) if (sm[i]) atomicAdd(&score[i >> 8], (unsigned long long)tlog[sm[i]]);
        } else {
            for (int x = threadIdx.x; x + 1 < rb; x += blockDim.x) {
                uint8_t v[5], w[5]; five_filters(row, up, x, bpp, v); five_filters(row, up, x + 1, bpp, w);
                for (int k = 0; k < 5; k++) {
                    const unsigned bg = ((unsigned)v[k] << 8) | w[k];
                    if (strategy == PNGF_BIGRAMS) atomicOr(&sm[k * 2048 + (bg >> 5)], 1u << (bg & 31));
                    else atomicAdd(&sm[k * 4096 + (((bg * 2654435761u) >> 20) & 4095u)], 1u);
                }
            }
            __syncthreads();
            if (strategy == PNGF_BIGRAMS) { for (int i = threadIdx.x; i < 5 * 2048; i += blockDim.x) if (sm[i]) atomicAdd(&score[i >> 11], (unsigned long long)__popc(sm[i])); }
            else for (int i = threadIdx.x; i < 5 * 4096; i += blockDim.x) if (sm[i]) atomicAdd(&score[i >> 12], (unsigned long long)tlog[min(sm[i], (uint32_t)rb)]);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            const bool want_max = strategy == PNGF_ENTROPY || strategy == PNGF_BRUTE || strategy == PNGF_BIGENT;   // sum c*log2(c): larger = lower entropy
            int best = 0;
            for (int k = 1; k < 5; k++) if (want_max ? score[k] > score[best] : score[k] < score[best]) best = k;
            chosen = best;
        }
        __syncthreads();
        f = chosen;
    }
    if (threadIdx.x == 0) out[0] = (uint8_t)f;
    for (int x = threadIdx.x; x < rb; x += blockDim.x) { uint8_t v[5]; five_filters(row, up, x, bpp, v); out[1 + x] = v[f]; }
}

// ---- K7 ---------------------------------------------------------------------------------------------------------------------
constexpr int PARSE_CHUNK_MAX = 4096;

__device__ __forceinline__ uint32_t load32u(const uint8_t *__restrict__ p)
{   // unaligned 32-bit little-endian load from two aligned words
    const uintptr_t a = (uintptr_t)p; const uint32_t *w = reinterpret_cast<const uint32_t *>(a & ~(uintptr_t)3);
    const int sh = (int)(a & 3) * 8;
    return sh ? __funnelshift_r(w[0], w[1], sh) : w[0];
}

__device__ __forceinline__ int match_len(const uint8_t *__restrict__ s, size_t i, int d, int maxlen)
{
    int l = 0;
    while (l + 4 <= maxlen) {
        const uint32_t x = load32u(s + i + l) ^ load32u(s + i + l - d);
        if (x) return l + ((__ffs((int)x) - 1) >> 3);
        l += 4;
    }
    while (l < maxlen && s[i + l] == s[i + l - d]) l++;
    return l;
}

// One thread per position, 256 positions per CTA (png_match_core.h).  Everything a CTA compares lies in three short windows of the
// stream -- the stretch itself (+ the 24 bytes before it: distances up to three pixels), the same stretch one row up (+- one pixel)
// and two rows up -- staged in shared memory once.  Per candidate distance the byte comparisons of the whole stretch are then made
// once (one ballot per 32 bytes) and kept as a bit array; a position's match length is the run of ones that starts at its bit.
// (The first version compared bytes per position and candidate: ~1,040 instructions per position, issue-bound at 2.2 ms per
// 4096 x 4096 RGBA stream.)
// All three windows live in one shared array of 32-bit words (byte offsets OFF0 / OFF1 / OFF2; one spare word behind each for the
// funnel shift of an unaligned read), addressed by integer offsets so that every access is a plain shared-memory load.
namespace pmk {
using namespace pm;
constexpr int OFF0 = 0, OFF1 = OFF0 + WIN0 + 4, OFF2 = OFF1 + WIN1 + 4, WIN_BYTES = OFF2 + WIN2 + 4;
static_assert(WIN0 % 4 == 0 && WIN1 % 4 == 0 && WIN2 % 4 == 0, "windows are whole words");
// stream bytes [b, b + nbytes) -> win[off / 4 ...], zero outside [0, n): aligned 32-bit loads + one funnel shift per word where the
// word and the aligned pair it is cut from lie inside the stream, bytes elsewhere (the two ends of the stream only)
__device__ __forceinline__ void stage(uint32_t *__restrict__ win, int off, int nbytes, const uint8_t *__restrict__ s, long long b, long long n)
{
    const int lo = b < 0 ? (int)min(-b, (long long)nbytes) : 0;                      // first window byte inside the stream
    const int hi = (int)max(0ll, min((long long)nbytes, n - b));                      // one past the last
    const uint8_t *base = s + b;                                                     // (may point before s: only dereferenced inside [lo, hi))
    const int mis = (int)((uintptr_t)base & 3);
    const uint32_t *ab = reinterpret_cast<const uint32_t *>(base - mis);
    const int sh = 8 * mis;
    for (int j = threadIdx.x; j < nbytes / 4; j += MATCH_T) {
        uint32_t v;
        if (4 * j >= lo + 4 && 4 * j + 8 <= hi) v = __funnelshift_r(ab[j], ab[j + 1], sh);       // (the pair ab[j], ab[j + 1] spans bytes 4j - mis .. 4j + 7 - mis)
        else {
            v = 0;
#pragma unroll
            for (int k = 0; k < 4; k++) { const int q = 4 * j + k; if (q >= lo && q < hi) v |= (uint32_t)base[q] << (8 * k); }
        }
        win[(off >> 2) + j] = v;
    }
    if (threadIdx.x == 0) win[(off + nbytes) >> 2] = 0;
}
// the same for a window that lies wholly inside the stream with eight bytes to spare on either side (every CTA but the first and last few)
__device__ __forceinline__ void stage_inside(uint32_t *__restrict__ win, int off, int nbytes, const uint8_t *__restrict__ base)
{
    const int mis = (int)((uintptr_t)base & 3);
    const uint32_t *ab = reinterpret_cast<const uint32_t *>(base - mis);
    const int sh = 8 * mis;
    for (int j = threadIdx.x; j <= nbytes / 4; j += MATCH_T) win[(off >> 2) + j] = __funnelshift_r(ab[j], ab[j + 1], sh);     // (<=: the spare word too)
}
__device__ __forceinline__ uint32_t word_at(const uint32_t *__restrict__ win, int byte_off)
{
    const int k = byte_off >> 2;
    return __funnelshift_r(win[k], win[k + 1], 8 * (byte_off & 3));
}
} // namespace pmk

__global__ void __launch_bounds__(pm::MATCH_T) k_png_match(const uint8_t *__restrict__ s, uint32_t *__restrict__ best, size_t n, int bpp, int stride, int chunk)
{
    using namespace pm;
    using namespace pmk;
    __shared__ __align__(16) uint32_t win[WIN_BYTES / 4];
    __shared__ uint32_t eq[NCAND][MATCH_WORDS];
    __shared__ int s_src[NCAND];                                                   // byte offset of "stretch byte 0 minus the distance" per candidate, -1: unusable
    const long long i0 = (long long)blockIdx.x * MATCH_T;
    const long long b0 = i0 - NEAR_BACK, b1 = i0 - stride - ROW_SLACK, b2 = i0 - 2ll * stride;
    if (min(b1, b2) >= 8 && i0 + WIN0 + 16 <= (long long)n) {                       // block-uniform
        stage_inside(win, OFF0, WIN0, s + b0); stage_inside(win, OFF1, WIN1, s + b1); stage_inside(win, OFF2, WIN2, s + b2);
    } else {
        stage(win, OFF0, WIN0, s, b0, (long long)n); stage(win, OFF1, WIN1, s, b1, (long long)n); stage(win, OFF2, WIN2, s, b2, (long long)n);
    }
    int cand[NCAND];
    candidates(bpp, stride, cand);
    if (threadIdx.x == 0) {
#pragma unroll
        for (int c = 0; c < NCAND; c++) {
            const int d = cand[c];
            s_src[c] = (d >= 1 && d <= 32768) ? (window_of(c) == 1 ? OFF1 : window_of(c) == 2 ? OFF2 : OFF0) + window_base(c, d, stride) : -1;
        }
    }
    __syncthreads();
    // comparison bit arrays: task (c, st) = candidate c, bytes 512 st .. 512 st + 511 of the stretch; a lane compares sixteen bytes
    // (four eq_nibble), two lanes make one 32-bit word
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int STEPS = (MATCH_BITS + 511) / 512;
    for (int task = warp; task < NCAND * STEPS; task += MATCH_T / 32) {
        const int c = task / STEPS, st = task - c * STEPS;
        const int so = s_src[c];
        const int q = 512 * st + 16 * lane;
        uint32_t v = 0;
        if (q < MATCH_BITS && so >= 0) {
            const int cw = (OFF0 + NEAR_BACK + q) >> 2, sw = (so + q) >> 2, sh = 8 * ((so + q) & 3);
            uint32_t a = win[sw];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const uint32_t b = win[sw + k + 1];
                v |= eq_nibble(win[cw + k], __funnelshift_r(a, b, sh)) << (4 * k);
                a = b;
            }
            v <<= 16 * (lane & 1);
        }
        v |= __shfl_xor_sync(0xFFFFFFFFu, v, 1);
        const int k = 16 * st + (lane >> 1);
        if ((lane & 1) == 0 && k < MATCH_WORDS) eq[c][k] = v;
    }
    __syncthreads();
    const size_t i = (size_t)i0 + threadIdx.x;
    if (i >= n) return;
    const size_t chunk_end = ((size_t)i0 / chunk + 1) * (size_t)chunk;            // MATCH_T divides the chunk size: one value per CTA
    const int maxlen = (int)min((size_t)MATCH_MAX, min(n, chunk_end) - i);
    best[i] = best_of(eq, cand, (int)threadIdx.x, (unsigned long long)i, maxlen);
}

// ---- K7, hash part: matches at ARBITRARY distances (north_star: "LZ77 match-find over a device hash table") ---------------------
// The fixed candidate set above finds what filtering leaves in photographs (pixel- and row-periodic repeats).  Flat art, text,
// dithering and UI screenshots repeat at arbitrary distances: for those every position is hashed by its next three bytes and looks
// at the nearest earlier positions with the same hash -- zlib's hash chains, built without a sequential insert loop: one CTA owns a
// segment of 16,384 positions, sorts (hash, position) with a stable block radix sort in shared memory, and the chain of a position
// is then simply the run of equal hashes in front of it (nearest first).  Chains do not cross segment starts; the fixed candidates
// (which reach back a whole row or two) do.  A hash candidate replaces the current best only if it is strictly longer, so the
// result is deterministic: the oracle twin walks ordinary head / prev chains and arrives at the same matches.
constexpr int HM_SEG = 16384, HM_THREADS = 512, HM_ITEMS = HM_SEG / HM_THREADS, HM_DEPTH = 4;
// A match at an arbitrary distance has to pay for its distance code, and what it saves depends on how cheap the literals it
// replaces are: in photographic residuals (3 - 4 bits per byte after Huffman coding) a 5-byte repeat 10,000 bytes back costs more
// than its literals and flattens the distance statistics of the matches that matter; in text or flat art the bytes a repeat covers
// are the rare, expensive ones.  So the stream is measured first -- a byte histogram, from it the order-0 cost of every byte value
// in 1024ths of a bit (pz_log2_q10: integer arithmetic, the same on the device and in the oracle) -- and a hash candidate is accepted when the
// literals it would replace cost at least 1.25 x (7 bits of length code + 5 of distance code + the distance's extra bits).
// (zlib's TOO_FAR rule, made proportional.)  The fixed pixel / row candidates are not subject to it.
// cost[0..255] = literal costs, cost[256..285] = match cost per distance code
__host__ __device__ inline void hash_cost_tables(const uint32_t *hist256, unsigned long long n, uint32_t *cost /*286*/)
{
    const uint32_t ln = pz_log2_q10(n ? n : 1);
    for (int v = 0; v < 256; v++) { const uint32_t c = hist256[v] ? ln - pz_log2_q10(hist256[v]) : 16u * 1024u; cost[v] = c < 256u ? 256u : c; }
    for (int ds = 0; ds < 30; ds++) cost[256 + ds] = (uint32_t)(7 + 5 + (ds < 4 ? 0 : (ds >> 1) - 1)) * 1280u;
}
__global__ void __launch_bounds__(256) k_png_bytehist(const uint8_t *__restrict__ s, size_t n, uint32_t *__restrict__ hist)
{
    __shared__ uint32_t h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    for (size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < n; i += (size_t)gridDim.x * blockDim.x * 4) {
        if (i + 4 <= n) { const uint32_t w = *reinterpret_cast<const uint32_t *>(s + i); atomicAdd(&h[w & 0xFF], 1u); atomicAdd(&h[(w >> 8) & 0xFF], 1u); atomicAdd(&h[(w >> 16) & 0xFF], 1u); atomicAdd(&h[w >> 24], 1u); }
        else for (size_t k = i; k < n; k++) atomicAdd(&h[s[k]], 1u);
    }
    __syncthreads();
    if (h[threadIdx.x]) atomicAdd(&hist[threadIdx.x], h[threadIdx.x]);
}
__global__ void k_png_costs(const uint32_t *__restrict__ hist, size_t n, uint32_t *__restrict__ cost)
{
    if (blockIdx.x == 0 && threadIdx.x == 0) hash_cost_tables(hist, n, cost);
}
__device__ __forceinline__ int dist_symbol_early(int d) { if (d <= 4) return d - 1; const int v = d - 1, hb = 31 - __clz(v); return hb * 2 + ((v >> (hb - 1)) & 1); }
__device__ __forceinline__ uint32_t hash3(const uint8_t *__restrict__ p) { return (((uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16)) * 2654435761u) >> 16; }

__global__ void __launch_bounds__(HM_THREADS) k_png_hashmatch(const uint8_t *__restrict__ s, uint32_t *__restrict__ best, size_t n, int chunk, const uint32_t *__restrict__ cost_tab)
{
    __shared__ uint32_t cost[286];
    if (threadIdx.x < 286) cost[threadIdx.x] = cost_tab[threadIdx.x];
    using Sort = cub::BlockRadixSort<uint16_t, HM_THREADS, HM_ITEMS, uint16_t>;
    extern __shared__ __align__(16) unsigned char hm_smem[];
    typename Sort::TempStorage &temp = *reinterpret_cast<typename Sort::TempStorage *>(hm_smem);
    uint16_t *sh_key = reinterpret_cast<uint16_t *>(hm_smem + ((sizeof(typename Sort::TempStorage) + 15) / 16) * 16), *sh_pos = sh_key + HM_SEG;
    const size_t seg0 = (size_t)blockIdx.x * HM_SEG;
    uint16_t keys[HM_ITEMS], vals[HM_ITEMS];
#pragma unroll
    for (int j = 0; j < HM_ITEMS; j++) {
        const int local = threadIdx.x * HM_ITEMS + j;
        const size_t p = seg0 + local;
        const bool ok = p + 3 <= n;
        keys[j] = ok ? (uint16_t)hash3(s + p) : (uint16_t)0xFFFF;
        vals[j] = ok ? (uint16_t)local : (uint16_t)0xFFFF;
    }
    Sort(temp).SortBlockedToStriped(keys, vals);       // stable LSD radix sort on the 16 hash bits: equal hashes stay in position order
    __syncthreads();
    // striped from here on (item j of thread t = rank j * HM_THREADS + t): consecutive lanes touch consecutive shared-memory entries
#pragma unroll
    for (int j = 0; j < HM_ITEMS; j++) { sh_key[j * HM_THREADS + threadIdx.x] = keys[j]; sh_pos[j * HM_THREADS + threadIdx.x] = vals[j]; }
    __syncthreads();
    for (int j = 0; j < HM_ITEMS; j++) {
        const int k = j * HM_THREADS + threadIdx.x;
        const uint32_t local = sh_pos[k];
        if (local == 0xFFFFu) continue;
        const size_t i = seg0 + local;
        const size_t chunk_end = (i / chunk + 1) * (size_t)chunk;
        const int maxlen = (int)min((size_t)258, min(n, chunk_end) - i);
        if (maxlen < 3) continue;
        const uint32_t cur = best[i];
        int bl = (int)(cur >> 16), bd = (int)(cur & 0xFFFF);
        if (bl == maxlen) continue;
        const uint16_t key = sh_key[k];
        for (int c = 1; c <= HM_DEPTH && k - c >= 0; c++) {
            if (sh_key[k - c] != key) break;
            const int d = (int)local - (int)sh_pos[k - c];
            if (bl > 0 && s[i + bl] != s[i + bl - d]) continue;      // cannot beat the current best
            const int l = match_len(s, i, d, maxlen);
            if (l > bl && l >= 4) {        // the literals it replaces must cost at least what the match costs
                const uint32_t need = cost[256 + dist_symbol_early(d)]; uint32_t worth = 0;
                for (int k2 = 0; k2 < l && worth < need; k2++) worth += cost[s[i + k2]];
                if (worth >= need) { bl = l; bd = d; }
            }
            if (bl == maxlen) break;
        }
        best[i] = bl >= 3 ? ((uint32_t)bl << 16) | (uint32_t)bd : 0u;
    }
}

__device__ __forceinline__ int len_symbol(int len)
{   // RFC 1951 3.2.5 length code 257..285 (index 0..28)
    if (len == 258) return 28;
    if (len < 11) return len - 3;
    const int l = len - 3, hb = 31 - __clz(l);              // l >= 8
    return (hb - 1) * 4 + ((l >> (hb - 2)) & 3);
}
__device__ __forceinline__ int dist_symbol(int d)
{
    if (d <= 4) return d - 1;
    const int v = d - 1, hb = 31 - __clz(v);
    return hb * 2 + ((v >> (hb - 1)) & 1);
}

// Greedy parse with one-step lazy matching (zlib's rule) of one chunk, in parallel: the step every position WOULD take if the
// parse arrived there (its match length after the TOO_FAR and lazy rules, else 1) depends only on best[i] and best[i + 1], so all
// steps are computed at once; the positions the sequential parse actually visits are those reachable from the chunk's first
// position, found by pointer doubling in shared memory (12 rounds for 4,096 positions); a block scan over the visited flags gives
// every token its slot.  Same tokens, same order, same histogram as the sequential walk (the oracle's orc_png_lz77 loop).
constexpr int PARSE_THREADS = 256, PARSE_PER = PARSE_CHUNK_MAX / PARSE_THREADS;
__global__ void __launch_bounds__(PARSE_THREADS) k_png_parse(const uint32_t *__restrict__ best, const uint8_t *__restrict__ s, size_t n, int chunk,
                                                             uint32_t *__restrict__ tokens, uint32_t *__restrict__ counts, uint32_t *__restrict__ hist)
{
    __shared__ uint16_t jump[PARSE_CHUNK_MAX + 1];
    __shared__ uint8_t visited[PARSE_CHUNK_MAX + 1];
    __shared__ uint32_t h[316];
    __shared__ uint32_t part[PARSE_THREADS];
    const size_t begin = (size_t)blockIdx.x * (size_t)chunk;
    if (begin >= n) return;
    const int len_chunk = (int)min((size_t)chunk, n - begin);
    for (int k = threadIdx.x; k < 316; k += PARSE_THREADS) h[k] = 0;
    // steps
    for (int j = threadIdx.x; j <= chunk; j += PARSE_THREADS) {
        int nx = len_chunk;
        if (j < len_chunk) {
            const uint32_t b = best[begin + j];
            int len = (int)(b >> 16); const int d = (int)(b & 0xFFFF);
            if (len == 3 && d > 4096) len = 0;                                                      // zlib's TOO_FAR rule
            if (len >= 3 && j + 1 < len_chunk && (int)(best[begin + j + 1] >> 16) > len) len = 0;   // one-step lazy matching
            nx = min(len_chunk, j + (len >= 3 ? len : 1));
        }
        jump[j] = (uint16_t)nx; visited[j] = j == 0;
    }
    __syncthreads();
    // reachability from position 0 by pointer doubling: after round r every visited position has marked its 2^r-th successor
    // (a round reads everything first and writes after the barrier: the visited positions form one chain, so their 2^r-th successors are
    // distinct and no two threads mark the same byte; the end-of-chunk sentinel, where all long jumps land, is never marked)
    for (int r = 0; (1 << r) < len_chunk; r++) {
        uint16_t nj[PARSE_PER + 1]; uint32_t marks = 0; int cnt = 0;     // (nj lives in local memory: at 30 registers eight CTAs fit an SM, which this latency-bound kernel needs more than it needs the array in registers -- measured 1.09 ms vs 1.87 ms)
        for (int j = threadIdx.x; j <= chunk; j += PARSE_THREADS, cnt++) {
            const uint16_t t = jump[j];
            if (j < len_chunk && visited[j] && t < len_chunk) marks |= 1u << cnt;
            nj[cnt] = jump[t];
        }
        __syncthreads();
        cnt = 0;
        for (int j = threadIdx.x; j <= chunk; j += PARSE_THREADS, cnt++) {
            if ((marks >> cnt) & 1u) visited[jump[j]] = 1;                // jump[j] is this thread's own entry: still the value read above
            jump[j] = nj[cnt];
        }
        __syncthreads();
    }
    // slots: thread t owns positions [t * PARSE_PER, (t + 1) * PARSE_PER)
    const int p0 = threadIdx.x * PARSE_PER;
    uint32_t mine = 0;
    for (int j = p0; j < p0 + PARSE_PER && j < len_chunk; j++) mine += visited[j];
    part[threadIdx.x] = mine;
    __syncthreads();
    uint32_t v = mine;
    for (int dd = 1; dd < PARSE_THREADS; dd <<= 1) {
        const uint32_t add = threadIdx.x >= (unsigned)dd ? part[threadIdx.x - dd] : 0u;
        __syncthreads();
        v += add; part[threadIdx.x] = v;
        __syncthreads();
    }
    uint32_t slot = v - mine;
    uint32_t *out = tokens + begin;
    for (int j = p0; j < p0 + PARSE_PER && j < len_chunk; j++) {
        if (!visited[j]) continue;
        const uint32_t b = best[begin + j];
        int len = (int)(b >> 16); const int d = (int)(b & 0xFFFF);
        if (len == 3 && d > 4096) len = 0;
        if (len >= 3 && j + 1 < len_chunk && (int)(best[begin + j + 1] >> 16) > len) len = 0;
        if (len >= 3) { out[slot++] = 0x80000000u | ((uint32_t)(len - 3) << 16) | (uint32_t)(d - 1); atomicAdd(&h[257 + len_symbol(len)], 1u); atomicAdd(&h[286 + dist_symbol(d)], 1u); }
        else { const uint32_t lit = s[begin + j]; out[slot++] = lit; atomicAdd(&h[lit], 1u); }
    }
    if (threadIdx.x == PARSE_THREADS - 1) counts[blockIdx.x] = v;
    __syncthreads();
    for (int k = threadIdx.x; k < 316; k += PARSE_THREADS) if (h[k]) atomicAdd(&hist[k], h[k]);
}

__global__ void k_png_compact(const uint32_t *__restrict__ tokens, const uint32_t *__restrict__ counts, const uint32_t *__restrict__ offsets, int chunk, uint32_t *__restrict__ out)
{
    const size_t c = blockIdx.x;
    const uint32_t n = counts[c], o = offsets[c];
    const uint32_t *src = tokens + c * (size_t)chunk;
    for (uint32_t t = threadIdx.x; t < n; t += blockDim.x) out[o + t] = src[t];
}

__global__ void k_png_adler(const uint8_t *__restrict__ s, size_t n, unsigned long long *__restrict__ sums)
{
    const size_t piece = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t begin = piece * 4096;
    if (begin >= n) return;
    const size_t len = min((size_t)4096, n - begin);
    unsigned long long a = 0, b = 0;
    for (size_t k = 0; k < len; k++) { const unsigned v = s[begin + k]; a += v; b += (unsigned long long)(len - k) * v; }
    sums[2 * piece] = a; sums[2 * piece + 1] = b;
}

__global__ void k_png_probe(const uint8_t *__restrict__ raw, size_t npix, int channels, uint32_t *__restrict__ flags)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    const uint8_t *p = raw + i * channels;
    if ((channels == 4 || channels == 2) && p[channels - 1] != 255) flags[0] = 1;
    if (channels >= 3 && (p[0] != p[1] || p[1] != p[2])) flags[1] = 1;
}
__global__ void k_png_repack(const uint8_t *__restrict__ raw, uint8_t *__restrict__ out, size_t npix, int channels, int keep_mask, int kept)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    const uint8_t *p = raw + i * channels; uint8_t *q = out + i * kept;
    int o = 0;
    for (int c = 0; c < channels; c++) if (keep_mask & (1 << c)) q[o++] = p[c];
}

// ---- un-filtering (PNG 9.2 reconstruction) on the device ------------------------------------------------------------------------
// Reconstruction is the one sequential piece of PNG: Sub / Average / Paeth need the reconstructed pixel to the left, Up / Average /
// Paeth the reconstructed row above.  Swept as a wavefront: one warp owns 32 consecutive rows, lane l works on row 32 g + l, and
// at step t it reconstructs pixel t - l of its row -- one pixel behind the lane above, so what it needs from the row above (pixel
// x and pixel x - 1) are that lane's results of the previous two steps and arrive by shuffle.  Lane 0's "row above" is the last
// row of the previous group, read back from HBM behind that group's progress counter; groups are handed out by an atomic ticket,
// so a waiting warp only ever waits for a warp that is already running (the K8 pattern).  BPP = filter distance in bytes (1..8).
// One group g of an image of h rows of rb bytes; progress[g - 1] is the previous group's counter.
template <int BPP>
__device__ __forceinline__ void unfilter_group(const uint8_t *__restrict__ filt, uint8_t *raw, int h, int rb, int g, volatile uint32_t *__restrict__ progress,
                                               uint32_t *__restrict__ bad)
{
    __shared__ uint8_t sh_up[2][32 * BPP];               // the row above lane 0, 32 pixels at a time, double buffered
    const int lane = threadIdx.x;
    const int y = g * 32 + lane;
    const bool live = y < h;
    const int npix = (rb + BPP - 1) / BPP;
    const uint8_t *f = filt + (size_t)(live ? y : 0) * (rb + 1);
    uint8_t *r = raw + (size_t)(live ? y : 0) * rb;
    const uint8_t *above = g > 0 ? raw + (size_t)(g * 32 - 1) * rb : nullptr;       // last row of the previous group
    const int ft = live ? f[0] : 0;
    if (live && ft > 4) atomicOr(bad, 1u);
    f++;
    int a[BPP], b[BPP], c[BPP];
#pragma unroll
    for (int k = 0; k < BPP; k++) a[k] = b[k] = c[k] = 0;
    const int steps = npix + 31;
    for (int t = 0; t < steps; t++) {
        if ((t & 31) == 0 && above && t < npix) {
            // the next 32 pixels of the row above the group: one poll of the previous group's progress per 32 steps (not per
            // step -- a poll is an L2 round trip and a fence, and the whole warp would wait for lane 0 on every pixel), then a
            // coalesced read through L2 (this SM's L1 may hold the lines from before they were written)
            const uint32_t need = (uint32_t)min(t + 32, npix);
            if (lane == 0) { while (progress[g - 1] < need) __nanosleep(100); }
            __syncwarp();
            __threadfence();
            const int px = t + lane;
#pragma unroll
            for (int k = 0; k < BPP; k++) sh_up[(t >> 5) & 1][lane * BPP + k] = (px < npix && px * BPP + k < rb) ? __ldcg(above + px * BPP + k) : (uint8_t)0;
            __syncwarp();
        }
        const int x = t - lane;
        const bool on = live && x >= 0 && x < npix;
        // the row above: lane l - 1's pixel of the previous step; lane 0 takes it from the staged copy of the previous group's last row
        int up[BPP];
#pragma unroll
        for (int k = 0; k < BPP; k++) up[k] = __shfl_up_sync(0xFFFFFFFFu, a[k], 1);
        if (lane == 0) {
#pragma unroll
            for (int k = 0; k < BPP; k++) up[k] = (above && t < npix) ? sh_up[(t >> 5) & 1][(t & 31) * BPP + k] : 0;
        }
        if (on) {
#pragma unroll
            for (int k = 0; k < BPP; k++) { c[k] = b[k]; b[k] = up[k]; }
            const int o = x * BPP;
#pragma unroll
            for (int k = 0; k < BPP; k++) if (o + k < rb) {
                const int p = ft == 0 ? 0 : ft == 1 ? a[k] : ft == 2 ? b[k] : ft == 3 ? ((a[k] + b[k]) >> 1) : paeth_pred(a[k], b[k], c[k]);
                a[k] = (f[o + k] + p) & 0xFF;
                r[o + k] = (uint8_t)a[k];
            }
        }
        // the last lane publishes its progress for the next group, 32 pixels at a time
        if (lane == 31 && on && ((x & 31) == 31 || x == npix - 1)) { __threadfence(); progress[g] = (uint32_t)(x + 1); }
    }
}

template <int BPP>
__global__ void __launch_bounds__(32) k_png_unfilter(const uint8_t *__restrict__ filt, uint8_t *raw, int h, int rb, uint32_t *__restrict__ ticket,
                                                     volatile uint32_t *__restrict__ progress, uint32_t *__restrict__ bad)
{
    int g = 0;
    if (threadIdx.x == 0) g = (int)atomicAdd(ticket, 1u);
    g = __shfl_sync(0xFFFFFFFFu, g, 0);
    unfilter_group<BPP>(filt, raw, h, rb, g, progress, bad);
}

// ---- Adam7: the seven passes in one wavefront launch ---------------------------------------------------------------------------
// Each pass is a PNG image of its own.  Groups take their tickets across all passes (pass p owns tickets first[p] .. first[p + 1] - 1);
// a pass's group 0 has no row above, and a group waits only for its predecessor in the same pass, which holds a lower ticket -- so,
// as in k_png_unfilter, a waiting warp only ever waits for one already running.  The passes run side by side: the launch takes about
// as long as the tallest pass's wavefront, not the sum of the seven.
struct Adam7Groups {
    int h[7], rb[7];
    unsigned long long filt_off[7], raw_off[7];
    int first[8];
};

template <int BPP>
__global__ void __launch_bounds__(32) k_png_adam7_unfilter(const uint8_t *__restrict__ filt, uint8_t *packed, const Adam7Groups d, uint32_t *__restrict__ ticket,
                                                           volatile uint32_t *__restrict__ progress, uint32_t *__restrict__ bad)
{
    int g = 0;
    if (threadIdx.x == 0) g = (int)atomicAdd(ticket, 1u);
    g = __shfl_sync(0xFFFFFFFFu, g, 0);
    int p = 0;
    while (p < 6 && g >= d.first[p + 1]) p++;          // empty passes own no tickets and are stepped over
    unfilter_group<BPP>(filt + d.filt_off[p], packed + d.raw_off[p], d.h[p], d.rb[p], g - d.first[p], progress + d.first[p], bad);
}

// the full image's rows from the pass-packed rows: one thread per output byte (so no two threads write one byte); blockIdx.y strides rows
__global__ void k_png_adam7_gather(const uint8_t *__restrict__ packed, uint8_t *__restrict__ raw, const Adam7Layout L, int bits, uint32_t w, uint32_t h, uint32_t rb)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rb) return;
    for (uint32_t y = blockIdx.y; y < h; y += gridDim.y) raw[(size_t)y * rb + i] = adam7_gather_byte(packed, L, bits, w, y, i);
}

// ---- palette probe: does the image have at most 256 distinct pixel values?  (8-bit RGB / RGBA; oxipng reduction::palette) -----------
// Open-addressing set of 1024 slots in global memory; the kernel gives up as soon as the 257th value appears, which for a
// photograph is within the first few hundred pixels of every CTA.  flags[2] = distinct values found (saturates above 256).
__global__ void k_png_colours(const uint8_t *__restrict__ raw, size_t npix, int channels, unsigned long long *__restrict__ set /*1024 slots, zeroed*/, uint32_t *__restrict__ flags)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (size_t)gridDim.x * blockDim.x) {
        if (*(volatile uint32_t *)&flags[2] > 256u) return;
        const uint8_t *p = raw + i * channels;
        const uint32_t v = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)(channels == 4 ? p[3] : 255) << 24);
        const unsigned long long key = (1ull << 32) | v;                            // never zero: zero marks an empty slot
        uint32_t hslot = (v * 2654435761u) >> 22;
        for (int probe = 0; probe < 1024; probe++, hslot = (hslot + 1) & 1023u) {
            unsigned long long cur = *(volatile unsigned long long *)&set[hslot];
            if (cur == 0ull) { cur = atomicCAS(&set[hslot], 0ull, key); if (cur == 0ull) { atomicAdd(&flags[2], 1u); break; } }
            if (cur == key) break;
        }
    }
}

static inline unsigned cdivu(size_t a, size_t b) { return (unsigned)((a + b - 1) / b); }

int launch_png_filter(const uint8_t *d_raw, uint8_t *d_filt, int h, int rb, int bpp, int strategy, const uint32_t *d_tlog, void *stream)
{
    const size_t hist = strategy == PNGF_BIGRAMS ? 5 * 2048 * 4 : (strategy == PNGF_BIGENT ? 5 * 4096 * 4 : (strategy >= 5 && strategy != PNGF_MINSUM ? 5 * 256 * 4 : 0));
    const int row_pitch = ((rb + 16 + 15) / 16) * 16;                       // 16 zero bytes + the row, 16-byte multiple
    const size_t smem = (size_t)2 * row_pitch + hist + 16;
    if (smem > 200 * 1024) {                                               // very long rows: the unstaged kernel
        if (hist > 48 * 1024) cudaFuncSetAttribute(k_png_filter_wide, cudaFuncAttributeMaxDynamicSharedMemorySize, 5 * 4096 * 4);
        k_png_filter_wide<<<h, 256, hist, (cudaStream_t)stream>>>(d_raw, d_filt, h, rb, bpp, strategy, d_tlog);
        LT_MARK("k_png_filter");
        return (int)cudaGetLastError();
    }
    cudaFuncSetAttribute(k_png_filter, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);   // per device, cheap
    const int threads = 256;            // (1,024-thread CTAs for the bigram strategies were measured 20 % slower: four times the contention on the shared counters)
    k_png_filter<<<h, threads, smem, (cudaStream_t)stream>>>(d_raw, d_filt, h, rb, bpp, strategy, d_tlog, row_pitch);
    LT_MARK("k_png_filter");
    return (int)cudaGetLastError();
}
int launch_png_match(const uint8_t *d_filt, uint32_t *d_best, size_t n, int bpp, int stride, void *stream)
{
    k_png_match<<<cdivu(n, 256), 256, 0, (cudaStream_t)stream>>>(d_filt, d_best, n, bpp, stride, PARSE_CHUNK_MAX);
    LT_MARK("k_png_match");
    return (int)cudaGetLastError();
}
int launch_png_hashmatch(const uint8_t *d_filt, uint32_t *d_best, size_t n, uint32_t *d_work /*256 + 286 words*/, void *stream)
{
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(d_work, 0, 256 * 4, st);
    k_png_bytehist<<<264, 256, 0, st>>>(d_filt, n, d_work);          // two CTAs on each of the H100's 132 SMs
    k_png_costs<<<1, 32, 0, st>>>(d_work, n, d_work + 256);
    LT_MARK("k_png_bytehist");
    using Sort = cub::BlockRadixSort<uint16_t, HM_THREADS, HM_ITEMS, uint16_t>;
    const size_t smem = ((sizeof(typename Sort::TempStorage) + 15) / 16) * 16 + (size_t)HM_SEG * 4;
    cudaFuncSetAttribute(k_png_hashmatch, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);      // per device; cheap to repeat
    k_png_hashmatch<<<cdivu(n, HM_SEG), HM_THREADS, smem, st>>>(d_filt, d_best, n, PARSE_CHUNK_MAX, d_work + 256);
    LT_MARK("k_png_hashmatch");
    return (int)cudaGetLastError();
}
int launch_png_parse(const uint32_t *d_best, const uint8_t *d_filt, size_t n, int chunk, uint32_t *d_tokens, uint32_t *d_counts, uint32_t *d_hist, void *stream)
{
    const size_t nchunks = (n + chunk - 1) / chunk;
    if (chunk > PARSE_CHUNK_MAX || chunk % PARSE_THREADS) return (int)cudaErrorInvalidValue;
    k_png_parse<<<(unsigned)nchunks, PARSE_THREADS, 0, (cudaStream_t)stream>>>(d_best, d_filt, n, chunk, d_tokens, d_counts, d_hist);
    LT_MARK("k_png_parse");
    return (int)cudaGetLastError();
}
int launch_png_compact(const uint32_t *d_tokens, const uint32_t *d_counts, const uint32_t *d_offsets, size_t nchunks, int chunk, uint32_t *d_out, void *stream)
{
    k_png_compact<<<(unsigned)nchunks, 128, 0, (cudaStream_t)stream>>>(d_tokens, d_counts, d_offsets, chunk, d_out);
    LT_MARK("k_png_compact");
    return (int)cudaGetLastError();
}
int launch_png_adler(const uint8_t *d_filt, size_t n, unsigned long long *d_sums, void *stream)
{
    k_png_adler<<<cdivu((n + 4095) / 4096, 64), 64, 0, (cudaStream_t)stream>>>(d_filt, n, d_sums);
    LT_MARK("k_png_adler");
    return (int)cudaGetLastError();
}
int launch_png_probe(const uint8_t *d_raw, size_t npixels, int channels, uint32_t *d_flags, void *stream)
{
    k_png_probe<<<cdivu(npixels, 256), 256, 0, (cudaStream_t)stream>>>(d_raw, npixels, channels, d_flags);
    LT_MARK("k_png_probe");
    return (int)cudaGetLastError();
}
int launch_png_unfilter(const uint8_t *d_filt, uint8_t *d_raw, int h, int rb, int bpp, uint32_t *d_sync /*2 + ceil(h/32) words*/, void *stream)
{
    cudaStream_t st = (cudaStream_t)stream;
    const int groups = (h + 31) / 32;
    cudaMemsetAsync(d_sync, 0, (size_t)(groups + 2) * 4, st);
    uint32_t *ticket = d_sync, *bad = d_sync + 1, *progress = d_sync + 2;
    switch (bpp) {
        case 1: k_png_unfilter<1><<<groups, 32, 0, st>>>(d_filt, d_raw, h, rb, ticket, progress, bad); break;
        case 2: k_png_unfilter<2><<<groups, 32, 0, st>>>(d_filt, d_raw, h, rb, ticket, progress, bad); break;
        case 3: k_png_unfilter<3><<<groups, 32, 0, st>>>(d_filt, d_raw, h, rb, ticket, progress, bad); break;
        case 4: k_png_unfilter<4><<<groups, 32, 0, st>>>(d_filt, d_raw, h, rb, ticket, progress, bad); break;
        case 6: k_png_unfilter<6><<<groups, 32, 0, st>>>(d_filt, d_raw, h, rb, ticket, progress, bad); break;
        case 8: k_png_unfilter<8><<<groups, 32, 0, st>>>(d_filt, d_raw, h, rb, ticket, progress, bad); break;
        default: return (int)cudaErrorInvalidValue;
    }
    LT_MARK("k_png_unfilter");
    return (int)cudaGetLastError();
}
int launch_png_adam7_unfilter(const uint8_t *d_filt, uint8_t *d_packed, uint8_t *d_raw, const Adam7Layout &L, uint32_t w, uint32_t h, int bits, int bpp,
                              uint32_t *d_sync, void *stream)
{
    cudaStream_t st = (cudaStream_t)stream;
    Adam7Groups d;
    d.first[0] = 0;
    for (int p = 0; p < 7; p++) {
        const Adam7Pass &P = L.pass[p];
        d.h[p] = (int)P.h; d.rb[p] = (int)P.rb; d.filt_off[p] = P.filt_off; d.raw_off[p] = P.raw_off;
        d.first[p + 1] = d.first[p] + (int)((P.h + 31) / 32);
    }
    const int groups = d.first[7];
    cudaMemsetAsync(d_sync, 0, (size_t)(groups + 2) * 4, st);
    uint32_t *ticket = d_sync, *bad = d_sync + 1, *progress = d_sync + 2;
    switch (bpp) {
        case 1: k_png_adam7_unfilter<1><<<groups, 32, 0, st>>>(d_filt, d_packed, d, ticket, progress, bad); break;
        case 2: k_png_adam7_unfilter<2><<<groups, 32, 0, st>>>(d_filt, d_packed, d, ticket, progress, bad); break;
        case 3: k_png_adam7_unfilter<3><<<groups, 32, 0, st>>>(d_filt, d_packed, d, ticket, progress, bad); break;
        case 4: k_png_adam7_unfilter<4><<<groups, 32, 0, st>>>(d_filt, d_packed, d, ticket, progress, bad); break;
        case 6: k_png_adam7_unfilter<6><<<groups, 32, 0, st>>>(d_filt, d_packed, d, ticket, progress, bad); break;
        case 8: k_png_adam7_unfilter<8><<<groups, 32, 0, st>>>(d_filt, d_packed, d, ticket, progress, bad); break;
        default: return (int)cudaErrorInvalidValue;
    }
    LT_MARK("k_png_adam7_unfilter");
    const uint32_t rb = (uint32_t)(((size_t)w * bits + 7) / 8);
    k_png_adam7_gather<<<dim3(cdivu(rb, 256), std::min<uint32_t>(h, 65535)), 256, 0, st>>>(d_packed, d_raw, L, bits, w, h, rb);
    LT_MARK("k_png_adam7_gather");
    return (int)cudaGetLastError();
}
int launch_png_colours(const uint8_t *d_raw, size_t npixels, int channels, uint32_t *d_set /*2048 words, 8-byte aligned*/, uint32_t *d_flags, void *stream)
{
    cudaMemsetAsync(d_set, 0, 2048 * 4, (cudaStream_t)stream);
    k_png_colours<<<64, 256, 0, (cudaStream_t)stream>>>(d_raw, npixels, channels, reinterpret_cast<unsigned long long *>(d_set), d_flags);
    LT_MARK("k_png_colours");
    return (int)cudaGetLastError();
}
int launch_png_repack(const uint8_t *d_raw, uint8_t *d_out, size_t npixels, int channels, int keep_mask, void *stream)
{
    int kept = 0; for (int c = 0; c < channels; c++) if (keep_mask & (1 << c)) kept++;
    k_png_repack<<<cdivu(npixels, 256), 256, 0, (cudaStream_t)stream>>>(d_raw, d_out, npixels, channels, keep_mask, kept);
    LT_MARK("k_png_repack");
    return (int)cudaGetLastError();
}

} // namespace b200
