// webp_anim_kernels.cu -- the animated WebP leg's kernels: compositing one frame onto a resident canvas, and cropping the output
// rectangle into either encoder's input.  The changed box comes from the GIF leg's k_gif_diff, which compares whole words too.
#include <cuda_runtime.h>
#include <algorithm>
#include "webp_anim_kernels.h"
#include "vp8l_enc_core.h"

namespace b200 {

static unsigned grid_for(size_t n, int threads) { return (unsigned)std::max<size_t>(1, std::min<size_t>((n + threads - 1) / threads, 132 * 16)); }

__global__ void __launch_bounds__(256) k_webp_anim_compose(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, int W, int H,
                                                           const uint32_t *__restrict__ frame, WaStep s)
{
    const size_t n = (size_t)W * H;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int y = (int)(i / W), x = (int)(i % W);
        const uint32_t src = wa_in_rect(s.rect, x, y) ? frame[(size_t)(y - s.rect.y) * s.rect.w + (x - s.rect.x)] : 0u;
        out[i] = webp_anim_pixel(&s, x, y, in[i], src);
    }
}

__global__ void __launch_bounds__(256) k_webp_anim_crop_planes(const uint32_t *__restrict__ canvas, int W, WaRect r, uint8_t *__restrict__ planes)
{
    const size_t n = (size_t)r.w * r.h;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t v = canvas[(size_t)(r.y + (int)(i / r.w)) * W + r.x + (int)(i % r.w)];
        planes[i] = (uint8_t)v; planes[n + i] = (uint8_t)(v >> 8); planes[2 * n + i] = (uint8_t)(v >> 16); planes[3 * n + i] = (uint8_t)(v >> 24);
    }
}

__global__ void __launch_bounds__(256) k_webp_anim_crop_argb(const uint32_t *__restrict__ canvas, int W, WaRect r, uint32_t *__restrict__ argb,
                                                             uint32_t *__restrict__ flags)
{
    const size_t n = (size_t)r.w * r.h;
    bool translucent = false;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t v = canvas[(size_t)(r.y + (int)(i / r.w)) * W + r.x + (int)(i % r.w)];
        translucent |= (v >> 24) != 255u;
        argb[i] = vp8l_sub_green((v & 0xFF00FF00u) | (v & 255u) << 16 | ((v >> 16) & 255u));      // RGBA word -> ARGB
    }
    if (__any_sync(0xFFFFFFFFu, translucent) && (threadIdx.x & 31) == 0) atomicOr(flags, 1u);
}

int launch_webp_anim_compose(const uint32_t *in, uint32_t *out, int W, int H, const uint32_t *frame, WaStep s, void *stream)
{
    k_webp_anim_compose<<<grid_for((size_t)W * H, 256), 256, 0, (cudaStream_t)stream>>>(in, out, W, H, frame, s);
    return (int)cudaGetLastError();
}

int launch_webp_anim_crop_planes(const uint32_t *canvas, int W, WaRect r, uint8_t *planes, void *stream)
{
    k_webp_anim_crop_planes<<<grid_for((size_t)r.w * r.h, 256), 256, 0, (cudaStream_t)stream>>>(canvas, W, r, planes);
    return (int)cudaGetLastError();
}

int launch_webp_anim_crop_argb(const uint32_t *canvas, int W, WaRect r, uint32_t *argb, uint32_t *flags, void *stream)
{
    k_webp_anim_crop_argb<<<grid_for((size_t)r.w * r.h, 256), 256, 0, (cudaStream_t)stream>>>(canvas, W, r, argb, flags);
    return (int)cudaGetLastError();
}

} // namespace b200
