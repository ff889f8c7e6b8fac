// resize_kernels.cu -- K3 (separable Lanczos3 resize) and the colour halves of K2/K4 (YCbCr<->RGB), SURVEY.md §8a
// rows a6/a9: what libcaesium's resize::resize_image does through image 0.25.9 `resize_exact(.., Lanczos3)` between
// decode and encode when CSParameters.width/height are set (caesium-clt's src/compressor.rs:439-443, :503-536).
// Bit-exact with oracle/resize_oracle.c: tap windows and normalised f32 weights are computed on the host with the
// same libm calls (resize_host.cpp); the kernels accumulate taps in the same order with separately rounded multiply
// and add (__fmul_rn/__fadd_rn: no FMA contraction), clamp and round half away from zero.  Vertical pass first into
// an f32 plane, then horizontal, as imageops::resize does.  Planar u8 or u16 channels; HBM-bound streaming kernels.
#include <cuda_runtime.h>
#include <cstdint>
#include <cstring>
#include "resize_kernels.h"

namespace b200 {

// T = uint8_t or uint16_t; the horizontal pass clamps to T's range before rounding.
template <class T>
__global__ void k_resize_v(const T *__restrict__ in, int w, float *__restrict__ out, int nh,
                           const int *__restrict__ left, const int *__restrict__ count, const float *__restrict__ weights, int cap)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y;
    if (x >= w || oy >= nh) return;
    const int l = left[oy], n = count[oy];
    const float *ws = weights + (size_t)oy * cap;
    float t = 0.0f;
    for (int i = 0; i < n; i++) t = __fadd_rn(t, __fmul_rn((float)in[(size_t)(l + i) * w + x], __ldg(ws + i)));
    out[(size_t)oy * w + x] = t;
}

template <class T>
__global__ void k_resize_h(const float *__restrict__ in, int w, T *__restrict__ out, int nw, int nh,
                           const int *__restrict__ left, const int *__restrict__ count, const float *__restrict__ weights, int cap)
{
    const int ox = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (ox >= nw || y >= nh) return;
    const int l = left[ox], n = count[ox];
    const float *ws = weights + (size_t)ox * cap;
    const float *row = in + (size_t)y * w + l;
    float t = 0.0f;
    for (int i = 0; i < n; i++) t = __fadd_rn(t, __fmul_rn(row[i], __ldg(ws + i)));
    t = fminf(fmaxf(t, 0.0f), sizeof(T) == 1 ? 255.0f : 65535.0f);
    out[(size_t)y * nw + ox] = (T)roundf(t);
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

template <class T>
bool Resampler::run(const T *const *in, int w, int h, T *const *out, int nw, int nh, int planes, void *stream, std::string &err)
{
    if (nw == w && nh == h) return true;
    cudaStream_t st = (cudaStream_t)stream;
    ResizeAxis av, ah;
    make_resize_axis(h, nh, av);
    make_resize_axis(w, nw, ah);
    auto al = [](size_t b) { return (b + 255) / 256 * 256; };
    const size_t cv = al(4 * (size_t)nh), wv = cv + al(4 * (size_t)nh), lh = wv + al(4 * av.weights.size());
    const size_t chh = lh + al(4 * (size_t)nw), wh = chh + al(4 * (size_t)nw), end = wh + al(4 * ah.weights.size());
    if (!h_tab.reserve(end, rule, err) || !d_tab.reserve(end, rule, err) || !d_tmp.reserve((size_t)nh * w * sizeof(float), rule, err)) return false;
    memcpy(h_tab, av.left.data(), 4 * (size_t)nh); memcpy(h_tab + cv, av.count.data(), 4 * (size_t)nh);
    memcpy(h_tab + wv, av.weights.data(), 4 * av.weights.size());
    memcpy(h_tab + lh, ah.left.data(), 4 * (size_t)nw); memcpy(h_tab + chh, ah.count.data(), 4 * (size_t)nw);
    memcpy(h_tab + wh, ah.weights.data(), 4 * ah.weights.size());
    CU(cudaMemcpyAsync(d_tab, h_tab, end, cudaMemcpyHostToDevice, st));
    const int *ax = reinterpret_cast<const int *>(d_tab.get());
    const float *axf = reinterpret_cast<const float *>(d_tab.get());
    for (int p = 0; p < planes; p++) {
        k_resize_v<T><<<dim3(cdiv((size_t)w, 256), nh), 256, 0, st>>>(in[p], w, d_tmp, nh, ax, ax + cv / 4, axf + wv / 4, av.cap);
        k_resize_h<T><<<dim3(cdiv((size_t)nw, 128), nh), 128, 0, st>>>(d_tmp, w, out[p], nw, nh, ax + lh / 4, ax + chh / 4, axf + wh / 4, ah.cap);
        if (!launch_ok((int)cudaGetLastError(), "resize", err)) return false;
    }
    return true;
}
template bool Resampler::run<uint8_t>(const uint8_t *const *, int, int, uint8_t *const *, int, int, int, void *, std::string &);
template bool Resampler::run<uint16_t>(const uint16_t *const *, int, int, uint16_t *const *, int, int, int, void *, std::string &);

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
