// webp_device.cu -- see webp_device.h.  caesium::convert_in_memory(.., WebP) (caesium-clt's src/compressor.rs:288-292).
#include <cuda_runtime.h>
#include <cstring>
#include <chrono>
#include "webp_device.h"
#include "vp8_kernels.h"
#include "vp8_host.h"
#include "stream_wait.h"
#include "vp8_tokens_core.h"
#include <algorithm>
#include <atomic>
#include <cstdlib>

namespace b200 {

static std::atomic<unsigned long long> g_d2h_bytes{0};
unsigned long long webp_d2h_bytes_total() { return g_d2h_bytes.load(); }

#define CUW(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) { err = std::string(#expr) + ": " + cudaGetErrorString(e_); return false; } } while (0)

template <typename T> static bool groww(T *&p, size_t &cap, size_t need, bool host, std::string &err)
{
    if (need <= cap) return true;
    if (p) { if (host) cudaFreeHost(p); else cudaFree(p); }
    p = nullptr; cap = 0;
    size_t want = 1 << 16; while (want < need) want <<= 1;
    void *q = nullptr;
    cudaError_t e = host ? cudaHostAlloc(&q, want, cudaHostAllocDefault) : cudaMalloc(&q, want);
    if (e != cudaSuccess) { err = std::string(host ? "cudaHostAlloc: " : "cudaMalloc: ") + cudaGetErrorString(e); return false; }
    p = (T *)q; cap = want; return true;
}

WebpDevice::~WebpDevice()
{
    cudaFree(d_planes); cudaFree(d_rgb); cudaFree(d_levels); cudaFree(d_modes); cudaFree(d_progress); cudaFreeHost(h_out); cudaFreeHost(h_rgb);
    cudaFree(d_tokwork); cudaFree(d_toktemp); cudaFree(d_tokens); cudaFreeHost(h_tokens);
}

bool WebpDevice::encode_planes(const uint8_t *d_r, const uint8_t *d_g, const uint8_t *d_b, int w, int h, int quality, void *stream_,
                               std::vector<uint8_t> &out, std::string &err, int16_t *levels_out, uint8_t *modes_out)
{
    cudaStream_t st = (cudaStream_t)stream_;
    if (w < 1 || h < 1 || w > 16383 || h > 16383) { err = "WebP dimensions out of range"; return false; }
    if (quality < 0) quality = 0; if (quality > 100) quality = 100;
    Vp8Frame f; f.w = w; f.h = h; f.mbw = (w + 15) >> 4; f.mbh = (h + 15) >> 4;
    const size_t nmb = (size_t)f.mbw * f.mbh, ny = nmb * 256, nc = nmb * 64;
    const size_t lv_bytes = nmb * VP8_MB_COEFS * sizeof(int16_t), md_bytes = nmb * 4;
    if (!groww(d_planes, cap_planes, 2 * (ny + 2 * nc) + 256, false, err) || !groww(d_levels, cap_levels, lv_bytes, false, err) ||
        !groww(d_modes, cap_modes, md_bytes, false, err) || !groww(d_progress, cap_progress, sizeof(int) * (size_t)(f.mbh + 1), false, err) ||
        !groww(h_out, cap_hout, lv_bytes + md_bytes, true, err)) return false;
    uint8_t *Y = d_planes, *U = Y + ny, *V = U + nc;
    f.Y = Y; f.U = U; f.V = V; f.RY = V + nc; f.RU = f.RY + ny; f.RV = f.RU + nc;
    f.levels = d_levels; f.modes = d_modes; f.progress = d_progress;
    const int qi = vp8_qindex(quality);
    vp8_quant_factors(qi, f.q);
    int rc = launch_vp8_rgb_to_yuv(d_r, d_g, d_b, w, h, Y, U, V, st);
    if (!rc) rc = launch_vp8_encode(f, st);
    if (rc) { err = std::string("vp8 kernels: ") + cudaGetErrorString((cudaError_t)rc); return false; }
    // The residual token pass runs on the device too (one thread per macroblock): what comes back is the frame's decision list and the
    // tallies per probability slot, a third of the bytes of the levels; B200_WEBP_TOKENS=host walks the levels on the calling thread instead.
    static const bool host_tokens = [] { const char *e = getenv("B200_WEBP_TOKENS"); return e && !strcmp(e, "host"); }();
    struct Lap { WebpDevice *d; std::chrono::steady_clock::time_point a, b; ~Lap() { d->last_wait_ms = std::chrono::duration<double, std::milli>(b - a).count(); d->last_code_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - b).count(); } };
    if (host_tokens) {
        CUW(cudaMemcpyAsync(h_out, d_levels, lv_bytes, cudaMemcpyDeviceToHost, st));
        CUW(cudaMemcpyAsync(h_out + lv_bytes, d_modes, md_bytes, cudaMemcpyDeviceToHost, st));
        const auto t0 = std::chrono::steady_clock::now();
        CUW(stream_wait(st));
        Lap lap{this, t0, std::chrono::steady_clock::now()};
        g_d2h_bytes += lv_bytes + md_bytes;
        if (levels_out) memcpy(levels_out, h_out, lv_bytes);
        if (modes_out) memcpy(modes_out, h_out + lv_bytes, md_bytes);
        if (!vp8_write_file(w, h, qi, reinterpret_cast<const int16_t *>(h_out), h_out + lv_bytes, out)) { err = "VP8 frame cannot be framed (first partition too large)"; return false; }
        return true;
    }
    const size_t hist_words = (size_t)vt::kNumProbs * 2, work_words = 3 * (nmb + 1) + hist_words;
    const size_t temp_bytes = vp8_tokens_temp_bytes((int)nmb);
    if (!groww(d_tokwork, cap_tokwork, work_words * 4, false, err) || !groww(d_tokens, cap_tokens, nmb * 640 * 2, false, err) || !groww(h_tokens, cap_htokens, nmb * 640 * 2, true, err)) return false;
    if (temp_bytes > cap_toktemp) { uint8_t *p = (uint8_t *)d_toktemp; size_t c = cap_toktemp; if (!groww(p, c, temp_bytes, false, err)) return false; d_toktemp = p; cap_toktemp = c; }
    uint32_t *d_mask = d_tokwork, *d_counts = d_mask + (nmb + 1), *d_offsets = d_counts + (nmb + 1), *d_hist = d_offsets + (nmb + 1);
    rc = launch_vp8_token_count(f, d_mask, d_counts, d_offsets, d_hist, d_toktemp, cap_toktemp, st);
    if (rc) { err = std::string("vp8 token pass: ") + cudaGetErrorString((cudaError_t)rc); return false; }
    // first trip: modes, tallies and the length of the list (+ the levels when a caller wants the stage output)
    uint8_t *h_modes = h_out, *h_hist = h_out + ((md_bytes + 15) / 16) * 16, *h_total = h_hist + hist_words * 4, *h_levels = h_total + 16;
    if (!groww(h_out, cap_hout, (size_t)(h_levels - h_out) + lv_bytes, true, err)) return false;
    h_modes = h_out; h_hist = h_out + ((md_bytes + 15) / 16) * 16; h_total = h_hist + hist_words * 4; h_levels = h_total + 16;
    CUW(cudaMemcpyAsync(h_modes, d_modes, md_bytes, cudaMemcpyDeviceToHost, st));
    CUW(cudaMemcpyAsync(h_hist, d_hist, hist_words * 4, cudaMemcpyDeviceToHost, st));
    CUW(cudaMemcpyAsync(h_total, d_offsets + nmb, 4, cudaMemcpyDeviceToHost, st));
    if (levels_out) CUW(cudaMemcpyAsync(h_levels, d_levels, lv_bytes, cudaMemcpyDeviceToHost, st));
    const auto t0 = std::chrono::steady_clock::now();
    CUW(stream_wait(st));
    const size_t total = *reinterpret_cast<const uint32_t *>(h_total);
    if (total > nmb * (size_t)vt::kMaxDecisionsPerMb) { err = "vp8 token pass: decision count out of range"; return false; }
    if (!groww(d_tokens, cap_tokens, total * 2 + 64, false, err) || !groww(h_tokens, cap_htokens, total * 2 + 64, true, err)) return false;
    rc = launch_vp8_token_write(f, d_mask, d_offsets, d_tokens, (uint32_t)std::min<size_t>(cap_tokens / 2, 0xFFFFFFFFu), st);
    if (rc) { err = std::string("vp8 token pass: ") + cudaGetErrorString((cudaError_t)rc); return false; }
    if (total) CUW(cudaMemcpyAsync(h_tokens, d_tokens, total * 2, cudaMemcpyDeviceToHost, st));
    CUW(stream_wait(st));
    Lap lap{this, t0, std::chrono::steady_clock::now()};
    g_d2h_bytes += md_bytes + hist_words * 4 + 4 + total * 2 + (levels_out ? lv_bytes : 0);
    if (levels_out) memcpy(levels_out, h_levels, lv_bytes);
    if (modes_out) memcpy(modes_out, h_modes, md_bytes);
    if (!vp8_write_file_tokens(w, h, qi, h_modes, reinterpret_cast<const uint32_t *>(h_hist), reinterpret_cast<const uint16_t *>(h_tokens), total, out)) { err = "VP8 frame cannot be framed (first partition too large)"; return false; }
    return true;
}

bool WebpDevice::encode_host_rgb(const uint8_t *rgb, int w, int h, int quality, void *stream_, std::vector<uint8_t> &out, std::string &err,
                                 int16_t *levels_out, uint8_t *modes_out)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const size_t n = (size_t)w * h;
    if (!groww(h_rgb, cap_hrgb, 3 * n, true, err) || !groww(d_rgb, cap_rgb, 3 * n, false, err)) return false;
    memcpy(h_rgb, rgb, 3 * n);
    CUW(cudaMemcpyAsync(d_rgb, h_rgb, 3 * n, cudaMemcpyHostToDevice, st));
    return encode_planes(d_rgb, d_rgb + n, d_rgb + 2 * n, w, h, quality, st, out, err, levels_out, modes_out);
}

} // namespace b200
