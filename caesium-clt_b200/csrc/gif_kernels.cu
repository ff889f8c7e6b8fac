// gif_kernels.cu -- the GIF leg's kernels: canvas difference, crop and mask, the canvases of converted sources, and the segmented
// LZW coder (one walker per segment, a prefix sum of the segments' bit lengths, placement with DevBits, sub-blocking).
#include <cuda_runtime.h>
#include <algorithm>
#include "gif_kernels.h"
#include "dev_bits.h"

namespace b200 {

static unsigned grid_for(size_t n, int threads) { return (unsigned)std::max<size_t>(1, std::min<size_t>((n + threads - 1) / threads, 132 * 16)); }

__global__ void __launch_bounds__(256) k_gif_diff(const uint32_t *__restrict__ a, const uint32_t *__restrict__ b, int w, int h, uint32_t *__restrict__ box)
{
    uint32_t m[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const size_t npix = (size_t)w * h;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t pa = a[i], pb = b[i];
        if (pa == pb) continue;
        const uint32_t y = (uint32_t)(i / w), x = (uint32_t)(i % w);
        m[0] = max(m[0], (uint32_t)w - x); m[1] = max(m[1], (uint32_t)h - y); m[2] = max(m[2], x + 1); m[3] = max(m[3], y + 1);
        if ((pa >> 24) && !(pb >> 24)) { m[4] = max(m[4], (uint32_t)w - x); m[5] = max(m[5], (uint32_t)h - y); m[6] = max(m[6], x + 1); m[7] = max(m[7], y + 1); }
    }
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const uint32_t v = __reduce_max_sync(0xFFFFFFFFu, m[k]);
        if ((threadIdx.x & 31) == 0 && v) atomicMax(&box[k], v);
    }
}

__global__ void k_gif_crop(const uint32_t *__restrict__ prev, const uint32_t *__restrict__ cur, int w, GifRect r, GifRect redraw, uint32_t *__restrict__ out)
{
    const int rw = r.x1 - r.x0;
    const size_t n = (size_t)rw * (r.y1 - r.y0);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int x = r.x0 + (int)(i % rw), y = r.y0 + (int)(i / rw);
        const size_t at = (size_t)y * w + x;
        out[i] = gif_out_pixel(prev[at], cur[at], gif_in_rect(redraw, x, y));
    }
}

// converted sources: 8-bit planes (a grey source passes its one plane as r, g and b; a == null: opaque) -> canvas words
__global__ void k_gif_canvas(const uint8_t *__restrict__ r, const uint8_t *__restrict__ g, const uint8_t *__restrict__ b, const uint8_t *__restrict__ a,
                             size_t n, uint32_t *__restrict__ out)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        out[i] = gif_canvas_pixel(r[i], g[i], b[i], a ? a[i] : 255u);
}

// RGBA8 words (R in the low byte) -> canvas words, in place
__global__ void k_gif_canvas_rgba(uint32_t *__restrict__ px, size_t n)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t v = px[i];
        px[i] = gif_canvas_pixel(v & 255u, (v >> 8) & 255u, (v >> 16) & 255u, v >> 24);
    }
}

// one thread per segment, its dictionary hashed in shared memory
__global__ void __launch_bounds__(1) k_gif_walk(const uint8_t *__restrict__ idx, size_t n, int m, int nseg, uint16_t *__restrict__ codes,
                                                uint32_t *__restrict__ ncodes, unsigned long long *__restrict__ bits)
{
    __shared__ uint32_t table[GIF_HASH];
    const int s = blockIdx.x;
    const size_t at = (size_t)s * GIF_SEG;
    const int len = n - at < (size_t)GIF_SEG ? (int)(n - at) : (int)GIF_SEG;
    unsigned b = 0;
    ncodes[s] = (uint32_t)gif_lzw_segment(idx + at, len, m, s == 0, s == nseg - 1, table, codes + (size_t)s * GIF_SEG_CODES, &b);
    bits[s] = b;
}

__global__ void k_gif_emit(const uint16_t *__restrict__ codes, const uint32_t *__restrict__ ncodes, const unsigned long long *__restrict__ off, int nseg,
                           uint32_t *words)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= nseg) return;
    DevBits bw(words, off[s]);
    const uint16_t *c = codes + (size_t)s * GIF_SEG_CODES;
    const int nc = (int)ncodes[s];
    for (int k = 0; k < nc; k++) bw.put32(c[k] & 4095u, c[k] >> 12);
    bw.finish();
}

__global__ void k_gif_blocks(const uint8_t *__restrict__ data, const unsigned long long *__restrict__ off, int nseg, size_t cap, uint8_t *__restrict__ out)
{
    const size_t nbytes = (size_t)((off[nseg] + 7) >> 3), total = gif_blocks_size(nbytes);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total && i < cap; i += (size_t)gridDim.x * blockDim.x)
        out[i] = gif_blocks_byte(data, nbytes, i);
}

int launch_gif_diff(const uint32_t *a, const uint32_t *b, int w, int h, uint32_t *box, void *stream)
{
    k_gif_diff<<<grid_for((size_t)w * h, 256), 256, 0, (cudaStream_t)stream>>>(a, b, w, h, box);
    return (int)cudaGetLastError();
}

int launch_gif_crop(const uint32_t *prev, const uint32_t *cur, int w, GifRect r, GifRect redraw, uint32_t *out, void *stream)
{
    k_gif_crop<<<grid_for((size_t)(r.x1 - r.x0) * (r.y1 - r.y0), 256), 256, 0, (cudaStream_t)stream>>>(prev, cur, w, r, redraw, out);
    return (int)cudaGetLastError();
}

int launch_gif_canvas(const uint8_t *r, const uint8_t *g, const uint8_t *b, const uint8_t *a, size_t n, uint32_t *out, void *stream)
{
    k_gif_canvas<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(r, g, b, a, n, out);
    return (int)cudaGetLastError();
}

int launch_gif_canvas_rgba(uint32_t *px, size_t n, void *stream)
{
    k_gif_canvas_rgba<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(px, n);
    return (int)cudaGetLastError();
}

int launch_gif_walk(const uint8_t *idx, size_t n, int m, int nseg, uint16_t *codes, uint32_t *ncodes, unsigned long long *bits, void *stream)
{
    k_gif_walk<<<nseg, 1, 0, (cudaStream_t)stream>>>(idx, n, m, nseg, codes, ncodes, bits);
    return (int)cudaGetLastError();
}

int launch_gif_emit(const uint16_t *codes, const uint32_t *ncodes, const unsigned long long *off, int nseg, uint32_t *words, void *stream)
{
    k_gif_emit<<<(nseg + 31) / 32, 32, 0, (cudaStream_t)stream>>>(codes, ncodes, off, nseg, words);
    return (int)cudaGetLastError();
}

int launch_gif_blocks(const uint8_t *data, const unsigned long long *off, int nseg, size_t cap, uint8_t *out, void *stream)
{
    k_gif_blocks<<<grid_for(cap, 256), 256, 0, (cudaStream_t)stream>>>(data, off, nseg, cap, out);
    return (int)cudaGetLastError();
}

} // namespace b200
