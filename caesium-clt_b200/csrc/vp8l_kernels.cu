// vp8l_kernels.cu -- the per-pixel work of the lossless WebP (VP8L) encoder; the rules are vp8l_enc_core.h's, the host side is
// vp8l_encode.cpp.
//   k_vp8l_pack         R, G, B (+ alpha) planes anywhere on the device -> ARGB with subtract-green applied; flags an alpha below 255
//   k_vp8l_predict      CTA per 16x16 tile: the 14 modes scored in shared-memory histograms -> mode image, residual image
//   k_vp8l_cache_last   CTA per (parse chunk, cache candidate): last position of every cache key inside the chunk
//   k_vp8l_cache_carry  thread per (key, candidate): the last position before each chunk (a running scan over the chunks)
//   k_vp8l_cache_hits   warp per (chunk, candidate): the chunk in pixel order, 32 at a time, against a shared-memory cache
//   k_vp8l_match        CTA per chunk: per candidate distance an equality bit array, runs by the next zero bit
//   k_vp8l_parse        CTA per chunk: greedy / one-step lazy parse, visited positions by pointer doubling -> tokens
//   k_vp8l_hist         per cache candidate: the five alphabets' histograms of the tokens
//   k_vp8l_len          per chunk: bits of every thread's tokens under the chosen codes -> offsets inside the chunk
//   k_vp8l_scan         chunk sizes -> start bit of every chunk after the header (one CTA)
//   k_vp8l_emit         LSB-first emission of the tokens with atomic ORs into zeroed words
// The palette variant (vp8l_palette.cu) writes its packed index image into the residual image and runs everything after
// k_vp8l_predict over it.
#include <cuda_runtime.h>
#include <cstdint>
#include "vp8l_enc_core.h"
#include "vp8l_kernels.h"
#include "dev_bits.h"
#include "launch_timer.h"

namespace b200 {

constexpr int V_THREADS = 256, V_PER = VP8L_CHUNK / V_THREADS, V_WORDS = VP8L_CHUNK / 32;

__host__ __device__ __forceinline__ int cache_table_offset(int cand) { return cand <= 1 ? 0 : cand == 2 ? 64 : 320; }   // keys of candidates 1..3: 64, 256, 1024
constexpr int CACHE_TABLE_KEYS = 64 + 256 + 1024;

// a: nullptr for an opaque image; a grey source passes one plane as r, g and b
__global__ void __launch_bounds__(V_THREADS) k_vp8l_pack(const uint8_t *__restrict__ r_, const uint8_t *__restrict__ g_, const uint8_t *__restrict__ b_,
                                                          const uint8_t *__restrict__ a_, uint32_t n, uint32_t *__restrict__ argb, uint32_t *__restrict__ flags)
{
    const uint32_t i = blockIdx.x * V_THREADS + threadIdx.x;
    bool translucent = false;
    if (i < n) {
        const uint32_t r = r_[i], g = g_[i], b = b_[i], a = a_ ? a_[i] : 255u;
        translucent = a != 255u;
        argb[i] = vp8l_sub_green((a << 24) | (r << 16) | (g << 8) | b);
    }
    if (__any_sync(0xFFFFFFFFu, translucent) && (threadIdx.x & 31) == 0) atomicOr(flags, 1u);
}

__global__ void __launch_bounds__(V_THREADS) k_vp8l_predict(const uint32_t *__restrict__ argb, int w, int h, int tiles_x, uint32_t *__restrict__ res, uint8_t *__restrict__ modes)
{
    __shared__ uint32_t hist[4 * 256];
    __shared__ unsigned long long nlog[V_THREADS + 1];
    __shared__ unsigned long long part[V_THREADS / 32];
    __shared__ int npix_s;
    const int tx = blockIdx.x % tiles_x, ty = blockIdx.x / tiles_x;
    const int x = tx * VP8L_TILE + (threadIdx.x & (VP8L_TILE - 1)), y = ty * VP8L_TILE + (threadIdx.x >> VP8L_TILE_BITS);
    const bool valid = x < w && y < h;
    nlog[threadIdx.x] = vp8l_nlog2_q10(threadIdx.x);
    if (threadIdx.x == 0) { nlog[V_THREADS] = vp8l_nlog2_q10(V_THREADS); npix_s = 0; }
    uint32_t P = 0, L = 0, T = 0, TR = 0, TL = 0;
    const size_t idx = (size_t)y * w + x;
    if (valid) {
        P = argb[idx];
        if (x) L = argb[idx - 1];
        if (y) { T = argb[idx - w]; TR = argb[idx - w + 1]; if (x) TL = argb[idx - w - 1]; }
    }
    __syncthreads();
    if (valid) atomicAdd(&npix_s, 1);
    int best = 0; unsigned long long best_cost = 0;
    for (int m = 0; m < VP8L_NMODES; m++) {
        for (int k = threadIdx.x; k < 4 * 256; k += V_THREADS) hist[k] = 0;
        __syncthreads();
        uint32_t r = 0;
        if (valid) {
            const uint32_t pred = y == 0 ? (x ? L : 0xFF000000u) : x == 0 ? T : vp8l_predict(m, L, T, TR, TL);
            r = vp8l_sub_px(P, pred);
            atomicAdd(&hist[r & 0xFF], 1u); atomicAdd(&hist[256 + ((r >> 8) & 0xFF)], 1u);
            atomicAdd(&hist[512 + ((r >> 16) & 0xFF)], 1u); atomicAdd(&hist[768 + (r >> 24)], 1u);
        }
        __syncthreads();
        unsigned long long s = nlog[hist[threadIdx.x]] + nlog[hist[256 + threadIdx.x]] + nlog[hist[512 + threadIdx.x]] + nlog[hist[768 + threadIdx.x]];
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, o);
        if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long tot = 0;
            for (int k = 0; k < V_THREADS / 32; k++) tot += part[k];
            const unsigned long long cost = 4 * nlog[npix_s] - tot;
            if (m == 0 || cost < best_cost) { best_cost = cost; best = m; }
            part[0] = (unsigned long long)best;
        }
        __syncthreads();
        if (m == VP8L_NMODES - 1) best = (int)part[0];
        __syncthreads();
    }
    if (valid) res[idx] = vp8l_sub_px(P, y == 0 ? (x ? L : 0xFF000000u) : x == 0 ? T : vp8l_predict(best, L, T, TR, TL));
    if (threadIdx.x == 0) modes[blockIdx.x] = (uint8_t)best;
}

// last[cand table][chunk][key]: the last position of the key inside the chunk, -1 when absent
__global__ void __launch_bounds__(V_THREADS) k_vp8l_cache_last(const uint32_t *__restrict__ res, uint32_t n, int nchunks, int *__restrict__ last)
{
    __shared__ int t[1 << VP8L_MAX_CACHE_BITS];
    const int cand = blockIdx.y + 1, bits = vp8l_cache_bits(cand), nk = 1 << bits;
    const uint32_t begin = blockIdx.x * VP8L_CHUNK, end = min(n, begin + VP8L_CHUNK);
    for (int k = threadIdx.x; k < nk; k += V_THREADS) t[k] = -1;
    __syncthreads();
    for (uint32_t i = begin + threadIdx.x; i < end; i += V_THREADS) atomicMax(&t[vp8l_cache_key(res[i], bits)], (int)i);
    __syncthreads();
    int *out = last + (size_t)nchunks * cache_table_offset(cand) + (size_t)blockIdx.x * nk;
    for (int k = threadIdx.x; k < nk; k += V_THREADS) out[k] = t[k];
}

// in place: last -> the last position of the key before each chunk (-1: none yet)
__global__ void __launch_bounds__(V_THREADS) k_vp8l_cache_carry(int nchunks, int *__restrict__ last)
{
    const int cand = blockIdx.y + 1, nk = 1 << vp8l_cache_bits(cand), k = blockIdx.x * V_THREADS + threadIdx.x;
    if (k >= nk) return;
    int *t = last + (size_t)nchunks * cache_table_offset(cand) + k;
    int run = -1;
    for (int c = 0; c < nchunks; c++) { const int v = t[(size_t)c * nk]; t[(size_t)c * nk] = run; if (v >= 0) run = v; }
}

// hits[cand - 1][i] = 1 when pixel i finds its value in a cache of that candidate's size
__global__ void __launch_bounds__(32) k_vp8l_cache_hits(const uint32_t *__restrict__ res, uint32_t n, int nchunks, const int *__restrict__ carry, uint8_t *__restrict__ hits)
{
    __shared__ uint32_t cache[1 << VP8L_MAX_CACHE_BITS];
    const int cand = blockIdx.y + 1, bits = vp8l_cache_bits(cand), nk = 1 << bits, lane = threadIdx.x;
    const uint32_t begin = blockIdx.x * VP8L_CHUNK, end = min(n, begin + VP8L_CHUNK);
    const int *c0 = carry + (size_t)nchunks * cache_table_offset(cand) + (size_t)blockIdx.x * nk;
    for (int k = lane; k < nk; k += 32) { const int p = c0[k]; cache[k] = p >= 0 ? res[p] : 0u; }
    __syncwarp();
    uint8_t *out = hits + (size_t)(cand - 1) * n;
    const unsigned lt = (1u << lane) - 1u;
    for (uint32_t base = begin; base < end; base += 32) {
        const uint32_t i = base + lane;
        const bool in = i < end;
        const uint32_t v = in ? res[i] : 0u, key = in ? vp8l_cache_key(v, bits) : 0xFFFFFFFFu;
        const unsigned peers = __match_any_sync(0xFFFFFFFFu, key);
        const unsigned before = peers & lt;
        const int src = before ? 31 - __clz((int)before) : lane;
        const uint32_t prev_v = __shfl_sync(0xFFFFFFFFu, v, src);
        const uint32_t have = before ? prev_v : (in ? cache[key] : 0u);
        if (in) out[i] = have == v;
        __syncwarp();
        if (in && !(peers >> lane >> 1)) cache[key] = v;          // the key's last pixel of this step goes into the cache
        __syncwarp();
    }
}

// best[i] = (run << 8) | code of the longest copy at i (vp8l_best_copy), 0 when none reaches VP8L_MIN_COPY
__global__ void __launch_bounds__(V_THREADS) k_vp8l_match(const uint32_t *__restrict__ res, uint32_t n, int width, uint32_t *__restrict__ best)
{
    __shared__ uint32_t eq[VP8L_NCAND][V_WORDS];
    __shared__ uint32_t full[VP8L_NCAND][V_WORDS / 32];
    __shared__ uint32_t dist[VP8L_NCAND];
    const uint32_t begin = blockIdx.x * VP8L_CHUNK, len = min((uint32_t)VP8L_CHUNK, n - begin);
    if (threadIdx.x < VP8L_NCAND) dist[threadIdx.x] = vp8l_code_dist(threadIdx.x + 1, width);
    if (threadIdx.x < VP8L_NCAND * (V_WORDS / 32)) full[threadIdx.x / (V_WORDS / 32)][threadIdx.x % (V_WORDS / 32)] = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int wd = warp; wd < V_WORDS; wd += V_THREADS / 32) {
        const uint32_t j = (uint32_t)wd * 32 + lane, i = begin + j;
        const uint32_t v = j < len ? res[i] : 0u;
        for (int c = 0; c < VP8L_NCAND; c++) {
            const uint32_t d = dist[c];
            const bool e = j < len && i >= d && res[i - d] == v;
            const uint32_t word = __ballot_sync(0xFFFFFFFFu, e);
            if (lane == 0) { eq[c][wd] = word; if (word == 0xFFFFFFFFu) atomicOr(&full[c][wd >> 5], 1u << (wd & 31)); }
        }
    }
    __syncthreads();
    for (int k = 0; k < V_PER; k++) {
        const uint32_t j = (uint32_t)k * V_THREADS + threadIdx.x;
        if (j >= len) break;
        uint32_t bl = 0, bc = 0;
        for (int c = 0; c < VP8L_NCAND; c++) {
            const int w0 = (int)(j >> 5);
            uint32_t m = ~eq[c][w0] & (0xFFFFFFFFu << (j & 31));
            uint32_t stop = VP8L_CHUNK;                 // no unequal pixel up to the chunk end: only a full chunk gets here
            if (m) stop = (uint32_t)w0 * 32 + (uint32_t)(__ffs((int)m) - 1);
            else
                for (int wd = w0 + 1; wd < V_WORDS;) {          // the next word that is not all ones, through the summary bits
                    const int s = wd >> 5;
                    const uint32_t nf = ~full[c][s] & (0xFFFFFFFFu << (wd & 31));
                    if (nf) { wd = s * 32 + __ffs((int)nf) - 1; stop = (uint32_t)wd * 32 + (uint32_t)(__ffs((int)~eq[c][wd]) - 1); break; }
                    wd = (s + 1) * 32;
                }
            const uint32_t run = stop - j;
            if (run > bl) { bl = run; bc = (uint32_t)c + 1; }
        }
        best[begin + j] = bl >= VP8L_MIN_COPY ? (bl << 8) | bc : 0u;
    }
}

// tokens of chunk b at tok[b * VP8L_CHUNK ...]: (position, copy = (len << 8) | code, 0 for a literal); cnt[b] of them
__global__ void __launch_bounds__(V_THREADS) k_vp8l_parse(const uint32_t *__restrict__ best, uint32_t n, uint2 *__restrict__ tok, uint32_t *__restrict__ cnt)
{
    __shared__ uint16_t jump[VP8L_CHUNK + 1];
    __shared__ uint8_t visited[VP8L_CHUNK + 1];
    __shared__ uint32_t part[V_THREADS];
    const uint32_t begin = blockIdx.x * VP8L_CHUNK;
    const int len = (int)min((uint32_t)VP8L_CHUNK, n - begin);
    for (int j = threadIdx.x; j <= VP8L_CHUNK; j += V_THREADS) {
        int nx = len;
        if (j < len) nx = min(len, j + (int)vp8l_parse_step(best[begin + j], j + 1 < len ? best[begin + j + 1] : 0u));
        jump[j] = (uint16_t)nx; visited[j] = j == 0;
    }
    __syncthreads();
    // reachability from position 0 by pointer doubling (as k_png_parse): after round r every visited position has marked its 2^r-th
    // successor; a round reads everything before the barrier and writes after it
    for (int r = 0; (1 << r) < len; r++) {
        uint16_t nj[V_PER + 1]; uint32_t marks = 0; int c = 0;
        for (int j = threadIdx.x; j <= VP8L_CHUNK; j += V_THREADS, c++) {
            const uint16_t t = jump[j];
            if (j < len && visited[j] && t < len) marks |= 1u << c;
            nj[c] = jump[t];
        }
        __syncthreads();
        c = 0;
        for (int j = threadIdx.x; j <= VP8L_CHUNK; j += V_THREADS, c++) {
            if ((marks >> c) & 1u) visited[jump[j]] = 1;
            jump[j] = nj[c];
        }
        __syncthreads();
    }
    const int p0 = threadIdx.x * V_PER;
    uint32_t mine = 0;
    for (int j = p0; j < p0 + V_PER && j < len; j++) mine += visited[j];
    part[threadIdx.x] = mine;
    __syncthreads();
    uint32_t v = mine;
    for (int d = 1; d < V_THREADS; d <<= 1) {
        const uint32_t add = threadIdx.x >= (unsigned)d ? part[threadIdx.x - d] : 0u;
        __syncthreads();
        v += add; part[threadIdx.x] = v;
        __syncthreads();
    }
    uint32_t slot = v - mine;
    for (int j = p0; j < p0 + V_PER && j < len; j++) {
        if (!visited[j]) continue;
        tok[begin + slot++] = make_uint2(begin + (uint32_t)j, vp8l_token_copy(best[begin + j], j + 1 < len ? best[begin + j + 1] : 0u));
    }
    if (threadIdx.x == V_THREADS - 1) cnt[blockIdx.x] = v;
}

// hist[cand][VP8L_HIST]: the tokens' symbols as a coder with that cache size writes them
__global__ void __launch_bounds__(V_THREADS) k_vp8l_hist(const uint2 *__restrict__ tok, const uint32_t *__restrict__ cnt, const uint32_t *__restrict__ res, const uint8_t *__restrict__ hits,
                                                          uint32_t n, int nchunks, uint32_t *__restrict__ hist)
{
    __shared__ uint32_t h[VP8L_HIST];
    const int cand = blockIdx.y, bits = vp8l_cache_bits(cand);
    const uint8_t *hit = cand ? hits + (size_t)(cand - 1) * n : nullptr;
    for (int k = threadIdx.x; k < VP8L_HIST; k += V_THREADS) h[k] = 0;
    __syncthreads();
    for (int b = blockIdx.x; b < nchunks; b += gridDim.x) {
        const uint32_t nt = cnt[b];
        for (uint32_t k = threadIdx.x; k < nt; k += V_THREADS) {
            const uint2 t = tok[(size_t)b * VP8L_CHUNK + k];
            int s, nx; uint32_t xv;
            if (t.y) {
                vp8l_prefix_of(t.y >> 8, &s, &nx, &xv); atomicAdd(&h[256 + s], 1u);
                vp8l_prefix_of(t.y & 0xFF, &s, &nx, &xv); atomicAdd(&h[VP8L_HIST_DIST + s], 1u);
                continue;
            }
            const uint32_t p = res[t.x];
            if (hit && hit[t.x]) { atomicAdd(&h[280 + vp8l_cache_key(p, bits)], 1u); continue; }
            atomicAdd(&h[(p >> 8) & 0xFF], 1u); atomicAdd(&h[VP8L_HIST_RED + ((p >> 16) & 0xFF)], 1u);
            atomicAdd(&h[VP8L_HIST_BLUE + (p & 0xFF)], 1u); atomicAdd(&h[VP8L_HIST_ALPHA + (p >> 24)], 1u);
        }
    }
    __syncthreads();
    for (int k = threadIdx.x; k < VP8L_HIST; k += V_THREADS) if (h[k]) atomicAdd(&hist[(size_t)cand * VP8L_HIST + k], h[k]);
}

struct Vp8lSmemCodes { uint16_t code[VP8L_HIST]; uint8_t len[VP8L_HIST]; };

__device__ __forceinline__ void load_codes(const Vp8lCodes *__restrict__ g, Vp8lSmemCodes &s)
{
    for (int k = threadIdx.x; k < VP8L_HIST; k += blockDim.x) { s.code[k] = g->code[k]; s.len[k] = g->len[k]; }
}

// bits of one token, and its pieces through put(value, nbits)
template <class Put>
__device__ __forceinline__ uint32_t token_code(const Vp8lSmemCodes &C, uint2 t, const uint32_t *__restrict__ res, const uint8_t *__restrict__ hit, int bits, Put put)
{
    int s, nx; uint32_t xv;
    if (t.y) {
        vp8l_prefix_of(t.y >> 8, &s, &nx, &xv);
        uint32_t nb = C.len[256 + s] + nx; put(C.code[256 + s], C.len[256 + s]); put(xv, nx);
        vp8l_prefix_of(t.y & 0xFF, &s, &nx, &xv);
        nb += C.len[VP8L_HIST_DIST + s] + nx; put(C.code[VP8L_HIST_DIST + s], C.len[VP8L_HIST_DIST + s]); put(xv, nx);
        return nb;
    }
    const uint32_t p = res[t.x];
    if (hit && hit[t.x]) { const int k = 280 + (int)vp8l_cache_key(p, bits); put(C.code[k], C.len[k]); return C.len[k]; }
    const int g = (p >> 8) & 0xFF, r = VP8L_HIST_RED + ((p >> 16) & 0xFF), b = VP8L_HIST_BLUE + (p & 0xFF), a = VP8L_HIST_ALPHA + (p >> 24);
    put(C.code[g], C.len[g]); put(C.code[r], C.len[r]); put(C.code[b], C.len[b]); put(C.code[a], C.len[a]);
    return (uint32_t)C.len[g] + C.len[r] + C.len[b] + C.len[a];
}

__global__ void __launch_bounds__(V_THREADS) k_vp8l_len(const uint2 *__restrict__ tok, const uint32_t *__restrict__ cnt, const uint32_t *__restrict__ res, const uint8_t *__restrict__ hit, int bits,
                                                         const Vp8lCodes *__restrict__ codes, uint32_t *__restrict__ thread_off, unsigned long long *__restrict__ chunk_bits)
{
    __shared__ Vp8lSmemCodes C;
    __shared__ uint32_t part[V_THREADS];
    load_codes(codes, C);
    __syncthreads();
    const uint32_t nt = cnt[blockIdx.x], k0 = threadIdx.x * V_PER, k1 = min(nt, k0 + V_PER);
    uint32_t sum = 0;
    for (uint32_t k = k0; k < k1; k++) sum += token_code(C, tok[(size_t)blockIdx.x * VP8L_CHUNK + k], res, hit, bits, [](uint32_t, int) {});
    part[threadIdx.x] = sum;
    __syncthreads();
    uint32_t v = sum;
    for (int d = 1; d < V_THREADS; d <<= 1) {
        const uint32_t add = threadIdx.x >= (unsigned)d ? part[threadIdx.x - d] : 0u;
        __syncthreads();
        v += add; part[threadIdx.x] = v;
        __syncthreads();
    }
    thread_off[(size_t)blockIdx.x * V_THREADS + threadIdx.x] = v - sum;
    if (threadIdx.x == V_THREADS - 1) chunk_bits[blockIdx.x] = v;
}

// start bit of every chunk (the first after bit_base, the header's length) and the total; one CTA, chunks in steps of its size
__global__ void __launch_bounds__(1024) k_vp8l_scan(const unsigned long long *__restrict__ chunk_bits, int nchunks, unsigned long long bit_base,
                                                     unsigned long long *__restrict__ chunk_start, unsigned long long *__restrict__ total)
{
    __shared__ unsigned long long part[1024];
    __shared__ unsigned long long carry;
    if (threadIdx.x == 0) carry = bit_base;
    __syncthreads();
    for (int base = 0; base < nchunks; base += 1024) {
        const int i = base + threadIdx.x;
        const unsigned long long mine = i < nchunks ? chunk_bits[i] : 0ull;
        unsigned long long v = mine;
        part[threadIdx.x] = v;
        __syncthreads();
        for (int d = 1; d < 1024; d <<= 1) {
            const unsigned long long add = threadIdx.x >= (unsigned)d ? part[threadIdx.x - d] : 0ull;
            __syncthreads();
            v += add; part[threadIdx.x] = v;
            __syncthreads();
        }
        if (i < nchunks) chunk_start[i] = carry + v - mine;
        __syncthreads();
        if (threadIdx.x == 1023) carry += v;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry;
}

__global__ void __launch_bounds__(V_THREADS) k_vp8l_emit(const uint2 *__restrict__ tok, const uint32_t *__restrict__ cnt, const uint32_t *__restrict__ res, const uint8_t *__restrict__ hit, int bits,
                                                          const Vp8lCodes *__restrict__ codes, const uint32_t *__restrict__ thread_off, const unsigned long long *__restrict__ chunk_start,
                                                          uint32_t *__restrict__ words)
{
    __shared__ Vp8lSmemCodes C;
    load_codes(codes, C);
    __syncthreads();
    const uint32_t nt = cnt[blockIdx.x], k0 = threadIdx.x * V_PER, k1 = min(nt, k0 + V_PER);
    if (k0 >= k1) return;
    DevBits w(words, chunk_start[blockIdx.x] + thread_off[(size_t)blockIdx.x * V_THREADS + threadIdx.x]);
    for (uint32_t k = k0; k < k1; k++) token_code(C, tok[(size_t)blockIdx.x * VP8L_CHUNK + k], res, hit, bits, [&](uint32_t v, int nb) { w.put32(v, nb); });
    w.finish();
}

static inline unsigned cdiv(size_t a, size_t b) { return (unsigned)((a + b - 1) / b); }

int launch_vp8l_pack(const uint8_t *r, const uint8_t *g, const uint8_t *b, const uint8_t *a, const Vp8lBuffers &B, int w, int h, void *stream_)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const uint32_t n = (uint32_t)w * (uint32_t)h;
    cudaMemsetAsync(B.flags, 0, 4, st); LT_MARK("upload+memset");
    k_vp8l_pack<<<cdiv(n, V_THREADS), V_THREADS, 0, st>>>(r, g, b, a, n, B.argb, B.flags); LT_MARK("k_vp8l_pack");
    return (int)cudaGetLastError();
}

int launch_vp8l_analyse(const Vp8lBuffers &B, int w, int h, void *stream_)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const int tiles_x =(w + VP8L_TILE - 1) >> VP8L_TILE_BITS, tiles = tiles_x * ((h + VP8L_TILE - 1) >> VP8L_TILE_BITS);
    k_vp8l_predict<<<tiles, V_THREADS, 0, st>>>(B.argb, w, h, tiles_x, B.res, B.modes); LT_MARK("k_vp8l_predict");
    return launch_vp8l_analyse_res(B, w, h, stream_);
}

int launch_vp8l_analyse_res(const Vp8lBuffers &B, int w, int h, void *stream_)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const uint32_t n = (uint32_t)w * (uint32_t)h;
    const int nchunks = (int)cdiv(n, VP8L_CHUNK);
    cudaMemsetAsync(B.hist, 0, sizeof(uint32_t) * VP8L_NCACHE * VP8L_HIST, st); LT_MARK("memset");
    k_vp8l_cache_last<<<dim3(nchunks, VP8L_NCACHE - 1), V_THREADS, 0, st>>>(B.res, n, nchunks, B.cache_tab); LT_MARK("k_vp8l_cache_last");
    k_vp8l_cache_carry<<<dim3(cdiv(1 << VP8L_MAX_CACHE_BITS, V_THREADS), VP8L_NCACHE - 1), V_THREADS, 0, st>>>(nchunks, B.cache_tab); LT_MARK("k_vp8l_cache_carry");
    k_vp8l_cache_hits<<<dim3(nchunks, VP8L_NCACHE - 1), 32, 0, st>>>(B.res, n, nchunks, B.cache_tab, B.hits); LT_MARK("k_vp8l_cache_hits");
    k_vp8l_match<<<nchunks, V_THREADS, 0, st>>>(B.res, n, w, B.best); LT_MARK("k_vp8l_match");
    k_vp8l_parse<<<nchunks, V_THREADS, 0, st>>>(B.best, n, B.tok, B.cnt); LT_MARK("k_vp8l_parse");
    k_vp8l_hist<<<dim3(nchunks < 264 ? nchunks : 264, VP8L_NCACHE), V_THREADS, 0, st>>>(B.tok, B.cnt, B.res, B.hits, n, nchunks, B.hist); LT_MARK("k_vp8l_hist");
    return (int)cudaGetLastError();
}

int launch_vp8l_size(const Vp8lBuffers &B, int w, int h, int cand, unsigned long long bit_base, void *stream_)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const uint32_t n = (uint32_t)w * (uint32_t)h;
    const int nchunks = (int)cdiv(n, VP8L_CHUNK);
    const uint8_t *hit = cand ? B.hits + (size_t)(cand - 1) * n : nullptr;
    k_vp8l_len<<<nchunks, V_THREADS, 0, st>>>(B.tok, B.cnt, B.res, hit, vp8l_cache_bits(cand), B.codes, B.thread_off, B.chunk_bits); LT_MARK("k_vp8l_len");
    k_vp8l_scan<<<1, 1024, 0, st>>>(B.chunk_bits, nchunks, bit_base, B.chunk_start, B.total); LT_MARK("k_vp8l_scan");
    return (int)cudaGetLastError();
}

int launch_vp8l_emit(const Vp8lBuffers &B, int w, int h, int cand, size_t words, void *stream_)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const uint32_t n = (uint32_t)w * (uint32_t)h;
    const int nchunks = (int)cdiv(n, VP8L_CHUNK);
    const uint8_t *hit = cand ? B.hits + (size_t)(cand - 1) * n : nullptr;
    cudaMemsetAsync(B.words, 0, words * 4, st); LT_MARK("memset");
    k_vp8l_emit<<<nchunks, V_THREADS, 0, st>>>(B.tok, B.cnt, B.res, hit, vp8l_cache_bits(cand), B.codes, B.thread_off, B.chunk_start, B.words); LT_MARK("k_vp8l_emit");
    return (int)cudaGetLastError();
}

size_t vp8l_cache_table_ints(int nchunks) { return (size_t)nchunks * CACHE_TABLE_KEYS; }

} // namespace b200
