// png_webp.cu -- see png_webp.h.  One thread per pixel, HBM-bound: each reads its pixel's bytes of the row and writes one ARGB word
// (k_png_rows_argb) or three / four plane bytes (k_png_rows_planes).  The palette goes to shared memory first.
#include <cuda_runtime.h>
#include "png_webp.h"
#include "vp8l_enc_core.h"
#include "launch_timer.h"

namespace b200 {

PngPixRule png_pix_rule(const PngInfo &info) { return png_pix_rule(info.color_type, info.bit_depth, info.trns.data(), info.trns.size()); }
PngPixLut png_pix_lut(const PngInfo &info) { return png_pix_lut(info.plte.data(), info.plte.size(), info.trns.data(), info.trns.size()); }
bool png_may_be_translucent(const PngInfo &info) { return info.color_type == 4 || info.color_type == 6 || !info.trns.empty(); }

constexpr int P_THREADS = 256;

__device__ __forceinline__ void load_lut(const PngPixRule &R, const PngPixLut &lut, uint32_t *s)
{
    if (R.ct == 3) s[threadIdx.x] = lut.v[threadIdx.x];
    __syncthreads();
}

__device__ __forceinline__ void flag_translucent(bool translucent, uint32_t *flags)
{
    if (__any_sync(0xFFFFFFFFu, translucent) && (threadIdx.x & 31) == 0) atomicOr(flags, 1u);
}

__global__ void __launch_bounds__(P_THREADS) k_png_rows_argb(const uint8_t *__restrict__ raw, size_t rb, uint32_t w, size_t n, const PngPixRule R, const PngPixLut lut,
                                                              uint32_t *__restrict__ argb, uint32_t *__restrict__ flags)
{
    __shared__ uint32_t s_lut[256];
    load_lut(R, lut, s_lut);
    const size_t i = (size_t)blockIdx.x * P_THREADS + threadIdx.x;
    bool translucent = false;
    if (i < n) {
        const size_t y = i / w;
        const uint32_t x = (uint32_t)(i - y * w);
        const uint32_t p = png_pix_argb(raw + (size_t)y * rb, x, R, s_lut);
        translucent = p < 0xFF000000u;
        argb[i] = vp8l_sub_green(p);
    }
    flag_translucent(translucent, flags);
}

__global__ void __launch_bounds__(P_THREADS) k_png_rows_planes(const uint8_t *__restrict__ raw, size_t rb, uint32_t w, size_t n, const PngPixRule R, const PngPixLut lut,
                                                                uint8_t *__restrict__ r, uint8_t *__restrict__ g, uint8_t *__restrict__ b, uint8_t *__restrict__ a,
                                                                uint32_t *__restrict__ flags)
{
    __shared__ uint32_t s_lut[256];
    load_lut(R, lut, s_lut);
    const size_t i = (size_t)blockIdx.x * P_THREADS + threadIdx.x;
    bool translucent = false;
    if (i < n) {
        const size_t y = i / w;
        const uint32_t x = (uint32_t)(i - y * w);
        const uint32_t p = png_pix_argb(raw + (size_t)y * rb, x, R, s_lut);
        translucent = p < 0xFF000000u;
        r[i] = (uint8_t)(p >> 16); g[i] = (uint8_t)(p >> 8); b[i] = (uint8_t)p;
        if (a) a[i] = (uint8_t)(p >> 24);
    }
    flag_translucent(translucent, flags);
}

static unsigned blocks_of(size_t n) { return (unsigned)((n + P_THREADS - 1) / P_THREADS); }

int launch_png_rows_argb(const uint8_t *d_raw, const PngInfo &info, uint32_t *argb, uint32_t *flags, void *stream)
{
    cudaStream_t st = (cudaStream_t)stream;
    const size_t n = (size_t)info.width * info.height;
    cudaMemsetAsync(flags, 0, 4, st);
    k_png_rows_argb<<<blocks_of(n), P_THREADS, 0, st>>>(d_raw, info.row_bytes, info.width, n, png_pix_rule(info), png_pix_lut(info), argb, flags);
    LT_MARK("k_png_rows_argb");
    return (int)cudaGetLastError();
}

int launch_png_rows_planes(const uint8_t *d_raw, const PngInfo &info, uint8_t *r, uint8_t *g, uint8_t *b, uint8_t *a, uint32_t *flags, void *stream)
{
    cudaStream_t st = (cudaStream_t)stream;
    const size_t n = (size_t)info.width * info.height;
    cudaMemsetAsync(flags, 0, 4, st);
    k_png_rows_planes<<<blocks_of(n), P_THREADS, 0, st>>>(d_raw, info.row_bytes, info.width, n, png_pix_rule(info), png_pix_lut(info), r, g, b, a, flags);
    LT_MARK("k_png_rows_planes");
    return (int)cudaGetLastError();
}

} // namespace b200
