// resize_kernels.cu -- K3 (separable Lanczos3 resize) and the colour halves of K2/K4 (YCbCr<->RGB), SURVEY.md §8a
// rows a6/a9: what libcaesium's resize::resize_image does through image 0.25.9 `resize_exact(.., Lanczos3)` between
// decode and encode when CSParameters.width/height are set (caesium-clt's src/compressor.rs:439-443, :503-536).
// Bit-exact with oracle/resize_oracle.c: tap windows and normalised f32 weights are computed on the host with the
// same libm calls (resize_host.cpp); the kernels accumulate taps in the same order with separately rounded multiply
// and add (__fmul_rn/__fadd_rn: no FMA contraction), clamp and round half away from zero.  Vertical pass first into
// an f32 plane, then horizontal, as imageops::resize does.  Planar u8 or u16 channels; HBM-bound streaming kernels.
#include <cuda_runtime.h>
#include <cstdint>
#include "resize_kernels.h"

namespace b200 {

// One launch resamples every plane of an image: blockIdx.z selects the plane, `in_pitch` / `out_pitch` are the planes' sizes in
// samples.  T = uint8_t or uint16_t; the horizontal pass clamps to T's range before rounding.
template <class T>
__global__ void k_resize_v(const T *__restrict__ in, int w, int stride, size_t in_pitch, float *__restrict__ out, int nh, size_t out_pitch,
                           const int *__restrict__ left, const int *__restrict__ count, const float *__restrict__ weights, int cap)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y;
    if (x >= w || oy >= nh) return;
    in += blockIdx.z * in_pitch; out += blockIdx.z * out_pitch;
    const int l = left[oy], n = count[oy];
    const float *ws = weights + (size_t)oy * cap;
    float t = 0.0f;
    for (int i = 0; i < n; i++) t = __fadd_rn(t, __fmul_rn((float)in[(size_t)(l + i) * stride + x], __ldg(ws + i)));
    out[(size_t)oy * w + x] = t;
}

template <class T>
__global__ void k_resize_h(const float *__restrict__ in, int w, size_t in_pitch, T *__restrict__ out, int nw, int nh, int ostride, size_t out_pitch,
                           const int *__restrict__ left, const int *__restrict__ count, const float *__restrict__ weights, int cap)
{
    const int ox = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (ox >= nw || y >= nh) return;
    in += blockIdx.z * in_pitch; out += blockIdx.z * out_pitch;
    const int l = left[ox], n = count[ox];
    const float *ws = weights + (size_t)ox * cap;
    const float *row = in + (size_t)y * w + l;
    float t = 0.0f;
    for (int i = 0; i < n; i++) t = __fadd_rn(t, __fmul_rn(row[i], __ldg(ws + i)));
    t = fminf(fmaxf(t, 0.0f), sizeof(T) == 1 ? 255.0f : 65535.0f);
    out[(size_t)y * ostride + ox] = (T)roundf(t);
}

#define FIXC(x) ((int)((x) * 65536.0 + 0.5))
__device__ __forceinline__ int clamp8(int v) { return min(255, max(0, v)); }

// jdcolor.c ycc_rgb_convert, in place on three planes
__global__ void k_ycc_to_rgb(uint8_t *__restrict__ p0, uint8_t *__restrict__ p1, uint8_t *__restrict__ p2, size_t n)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int Y = p0[i], xb = (int)p1[i] - 128, xr = (int)p2[i] - 128;
    const int cr_r = (FIXC(1.40200) * xr + 32768) >> 16;
    const int cb_b = (FIXC(1.77200) * xb + 32768) >> 16;
    const int g_off = ((-FIXC(0.34414)) * xb + 32768 + (-FIXC(0.71414)) * xr) >> 16;
    p0[i] = (uint8_t)clamp8(Y + cr_r); p1[i] = (uint8_t)clamp8(Y + g_off); p2[i] = (uint8_t)clamp8(Y + cb_b);
}

// jccolor.c rgb_ycc_convert, in place on three planes
__global__ void k_rgb_to_ycc(uint8_t *__restrict__ p0, uint8_t *__restrict__ p1, uint8_t *__restrict__ p2, size_t n)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int R = p0[i], G = p1[i], B = p2[i];
    p0[i] = (uint8_t)((FIXC(0.29900) * R + FIXC(0.58700) * G + FIXC(0.11400) * B + 32768) >> 16);
    p1[i] = (uint8_t)(((-FIXC(0.16874)) * R + (-FIXC(0.33126)) * G + FIXC(0.50000) * B + (128 << 16) + 32767) >> 16);
    p2[i] = (uint8_t)((FIXC(0.50000) * R + (-FIXC(0.41869)) * G + (-FIXC(0.08131)) * B + (128 << 16) + 32767) >> 16);
}

static inline int cdiv(size_t a, size_t b) { return (int)((a + b - 1) / b); }

int launch_resize_v(const uint8_t *in, int w, int h, int stride, float *out, int nh, const int *left, const int *count, const float *weights, int cap, void *stream)
{
    return launch_resize_v_planes(in, w, h, stride, 0, out, nh, 0, 1, left, count, weights, cap, stream);
}
int launch_resize_h(const float *in, int w, uint8_t *out, int nw, int nh, int ostride, const int *left, const int *count, const float *weights, int cap, void *stream)
{
    return launch_resize_h_planes(in, w, 0, out, nw, nh, ostride, 0, 1, left, count, weights, cap, stream);
}
template <class T>
int launch_resize_v_planes(const T *in, int w, int h, int stride, size_t in_pitch, float *out, int nh, size_t out_pitch, int planes,
                           const int *left, const int *count, const float *weights, int cap, void *stream)
{
    (void)h;
    dim3 grid(cdiv((size_t)w, 256), nh, planes);
    k_resize_v<T><<<grid, 256, 0, (cudaStream_t)stream>>>(in, w, stride, in_pitch, out, nh, out_pitch, left, count, weights, cap);
    return (int)cudaGetLastError();
}
template <class T>
int launch_resize_h_planes(const float *in, int w, size_t in_pitch, T *out, int nw, int nh, int ostride, size_t out_pitch, int planes,
                           const int *left, const int *count, const float *weights, int cap, void *stream)
{
    dim3 grid(cdiv((size_t)nw, 128), nh, planes);
    k_resize_h<T><<<grid, 128, 0, (cudaStream_t)stream>>>(in, w, in_pitch, out, nw, nh, ostride, out_pitch, left, count, weights, cap);
    return (int)cudaGetLastError();
}
template int launch_resize_v_planes<uint8_t>(const uint8_t *, int, int, int, size_t, float *, int, size_t, int, const int *, const int *, const float *, int, void *);
template int launch_resize_v_planes<uint16_t>(const uint16_t *, int, int, int, size_t, float *, int, size_t, int, const int *, const int *, const float *, int, void *);
template int launch_resize_h_planes<uint8_t>(const float *, int, size_t, uint8_t *, int, int, int, size_t, int, const int *, const int *, const float *, int, void *);
template int launch_resize_h_planes<uint16_t>(const float *, int, size_t, uint16_t *, int, int, int, size_t, int, const int *, const int *, const float *, int, void *);
int launch_ycc_to_rgb(uint8_t *p0, uint8_t *p1, uint8_t *p2, size_t n, void *stream)
{
    k_ycc_to_rgb<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(p0, p1, p2, n);
    return (int)cudaGetLastError();
}
int launch_rgb_to_ycc(uint8_t *p0, uint8_t *p1, uint8_t *p2, size_t n, void *stream)
{
    k_rgb_to_ycc<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(p0, p1, p2, n);
    return (int)cudaGetLastError();
}

} // namespace b200
