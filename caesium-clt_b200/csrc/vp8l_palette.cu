// vp8l_palette.cu -- the colour-indexing (palette) variant of the lossless WebP (VP8L) encoder; the rules are vp8l_palette_core.h's,
// the host side is vp8l_encode.cpp.
//   k_vp8l_palette_collect  CTA per VP8L_PAL_CTA_PIXELS pixels: the colours in a shared-memory set, merged into one global set; stops
//                           at entry and before each step once some CTA has seen more than VP8L_PAL_MAX colours
//   k_vp8l_palette_sort     one CTA: the global set compacted and bitonic-sorted -> count, overflow flag, ascending palette
//   k_vp8l_palette_pack     thread per packed pixel: the bundle of palette indices, written as the residual image the coder reads
#include <cuda_runtime.h>
#include <cstdint>
#include "vp8l_palette_core.h"
#include "vp8l_kernels.h"
#include "launch_timer.h"

namespace b200 {

constexpr unsigned long long PAL_USED = 1ull << 32;   // a set slot holds PAL_USED | colour; 0 is empty

__global__ void __launch_bounds__(VP8L_PAL_THREADS) k_vp8l_palette_collect(const uint32_t *__restrict__ argb, uint32_t n, unsigned long long *__restrict__ gset, uint32_t *__restrict__ info)
{
    __shared__ unsigned long long set[VP8L_PAL_SET];
    __shared__ int count, stop;
    volatile uint32_t *overflow = info + 1;
    for (int k = threadIdx.x; k < VP8L_PAL_SET; k += VP8L_PAL_THREADS) set[k] = 0;
    if (threadIdx.x == 0) { count = 0; stop = *overflow != 0; }
    __syncthreads();
    const uint32_t base = blockIdx.x * (uint32_t)VP8L_PAL_CTA_PIXELS;
    const int lane = threadIdx.x & 31;
    for (int s = 0; s < VP8L_PAL_STEPS; s++) {
        if (stop) return;
        const uint32_t i = base + (uint32_t)s * VP8L_PAL_THREADS + threadIdx.x;
        const unsigned long long key = i < n ? PAL_USED | vp8l_add_green(argb[i]) : 0ull;
        // one insertion per distinct colour of the warp: the lowest lane holding it
        const unsigned peers = __match_any_sync(0xFFFFFFFFu, key);
        if (key && (__ffs((int)peers) - 1) == lane)
            for (uint32_t h = vp8l_pal_hash((uint32_t)key);; h = (h + 1) & (VP8L_PAL_SET - 1)) {
                const unsigned long long old = atomicCAS(&set[h], 0ull, key);
                if (old == 0ull) { atomicAdd(&count, 1); break; }
                if (old == key) break;
            }
        __syncthreads();
        if (threadIdx.x == 0) {
            if (count > VP8L_PAL_MAX) atomicExch(info + 1, 1u);
            stop = count > VP8L_PAL_MAX || *overflow != 0;
        }
        __syncthreads();
    }
    if (stop) return;
    // at most VP8L_PAL_MAX colours per CTA; a global set holding VP8L_PAL_MAX of 1024 slots always has room, so a probe that finds
    // none means more colours than that have been merged
    for (int k = threadIdx.x; k < VP8L_PAL_SET; k += VP8L_PAL_THREADS) {
        const unsigned long long key = set[k];
        if (!key) continue;
        bool placed = false;
        uint32_t h = vp8l_pal_hash((uint32_t)key);
        for (int p = 0; p < VP8L_PAL_SET && !placed; p++, h = (h + 1) & (VP8L_PAL_SET - 1)) {
            const unsigned long long old = atomicCAS(&gset[h], 0ull, key);
            if (old == 0ull) { if (atomicAdd(info, 1u) >= (uint32_t)VP8L_PAL_MAX) atomicExch(info + 1, 1u); placed = true; }
            else placed = old == key;
        }
        if (!placed) atomicExch(info + 1, 1u);
    }
}

__global__ void __launch_bounds__(VP8L_PAL_MAX) k_vp8l_palette_sort(const unsigned long long *__restrict__ gset, uint32_t *__restrict__ info)
{
    __shared__ unsigned long long v[VP8L_PAL_MAX];
    __shared__ int m;
    const int t = threadIdx.x;
    if (info[1]) return;                                     // over VP8L_PAL_MAX colours: no palette
    v[t] = ~0ull;
    if (t == 0) m = 0;
    __syncthreads();
    for (int k = t; k < VP8L_PAL_SET; k += VP8L_PAL_MAX) { const unsigned long long key = gset[k]; if (key) v[atomicAdd(&m, 1)] = key; }
    __syncthreads();
    for (int k = 2; k <= VP8L_PAL_MAX; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            const int o = t ^ j;
            if (o > t) {
                const unsigned long long a = v[t], b = v[o];
                if ((a > b) == ((t & k) == 0)) { v[t] = b; v[o] = a; }
            }
            __syncthreads();
        }
    info[2 + t] = t < m ? (uint32_t)v[t] : 0u;
}

__global__ void __launch_bounds__(256) k_vp8l_palette_pack(const uint32_t *__restrict__ argb, int w, int wp, uint32_t np, const uint32_t *__restrict__ info, int count, int xbits,
                                                            uint32_t *__restrict__ res)
{
    __shared__ uint32_t pal[VP8L_PAL_MAX];
    pal[threadIdx.x] = info[2 + threadIdx.x];
    __syncthreads();
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    if (i >= np) return;
    const uint32_t y = i / (uint32_t)wp, xp = i - y * (uint32_t)wp;
    res[i] = vp8l_pal_pack(argb + (size_t)y * w, w, (int)xp, pal, count, xbits);
}

int launch_vp8l_palette(const Vp8lBuffers &B, int w, int h, void *stream_)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const uint32_t n = (uint32_t)w * (uint32_t)h;
    cudaMemsetAsync(B.pal_set, 0, sizeof(unsigned long long) * VP8L_PAL_SET, st);
    cudaMemsetAsync(B.pal_info, 0, 8, st); LT_MARK("memset");
    k_vp8l_palette_collect<<<(n + VP8L_PAL_CTA_PIXELS - 1) / VP8L_PAL_CTA_PIXELS, VP8L_PAL_THREADS, 0, st>>>(B.argb, n, B.pal_set, B.pal_info); LT_MARK("k_vp8l_palette_collect");
    k_vp8l_palette_sort<<<1, VP8L_PAL_MAX, 0, st>>>(B.pal_set, B.pal_info); LT_MARK("k_vp8l_palette_sort");
    return (int)cudaGetLastError();
}

int launch_vp8l_palette_pack(const Vp8lBuffers &B, int w, int h, int count, void *stream_)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const int xbits = vp8l_pal_xbits(count), wp = vp8l_pal_width(w, xbits);
    const uint32_t np = (uint32_t)wp * (uint32_t)h;
    k_vp8l_palette_pack<<<(np + 255) / 256, 256, 0, st>>>(B.argb, w, wp, np, B.pal_info, count, xbits, B.res); LT_MARK("k_vp8l_palette_pack");
    return (int)cudaGetLastError();
}

} // namespace b200
