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

// the smallest power of two >= 64 KiB and >= need
template <class B> static bool grow(B &buf, size_t need, std::string &err) { return buf.reserve(need, Grow::Pow2, err); }

bool WebpDevice::encode_planes(const uint8_t *d_r, const uint8_t *d_g, const uint8_t *d_b, int w, int h, int quality, void *stream_,
                               std::vector<uint8_t> &out, std::string &err, int16_t *levels_out, uint8_t *modes_out, uint8_t *bmodes_out, bool force_bpred)
{
    if (w < 1 || h < 1 || w > 16383 || h > 16383) { err = "WebP dimensions out of range"; return false; }
    if (quality < 0) quality = 0; if (quality > 100) quality = 100;
    if (force_bpred || webp_bpred()) {
        bool overflow = false;
        if (encode_frame(d_r, d_g, d_b, w, h, quality, stream_, out, err, levels_out, modes_out, bmodes_out, true, overflow)) return true;
        if (!overflow) return false;
        // B_PRED's sub-block modes can push the first partition past its 19-bit size field on large detailed frames: such a frame is
        // coded 16x16-only, byte for byte what the switch-off encoder writes
        err.clear();
    }
    bool overflow = false;
    const size_t nmb = (size_t)((w + 15) >> 4) * ((h + 15) >> 4);
    std::vector<uint8_t> own_modes(bmodes_out && !modes_out ? nmb * 4 : 0);      // a 16x16 frame's sub-block modes come from its modes
    uint8_t *md = modes_out ? modes_out : bmodes_out ? own_modes.data() : nullptr;
    if (!encode_frame(d_r, d_g, d_b, w, h, quality, stream_, out, err, levels_out, md, nullptr, false, overflow)) return false;
    if (bmodes_out) for (size_t i = 0; i < nmb; i++) memset(bmodes_out + 16 * i, md[4 * i], 16);
    return true;
}

bool WebpDevice::encode_frame(const uint8_t *d_r, const uint8_t *d_g, const uint8_t *d_b, int w, int h, int quality, void *stream_,
                              std::vector<uint8_t> &out, std::string &err, int16_t *levels_out, uint8_t *modes_out, uint8_t *bmodes_out, bool bpred, bool &overflow)
{
    cudaStream_t st = (cudaStream_t)stream_;
    Vp8Frame f; f.w = w; f.h = h; f.mbw = (w + 15) >> 4; f.mbh = (h + 15) >> 4;
    const size_t nmb = (size_t)f.mbw * f.mbh, ny = nmb * 256, nc = nmb * 64;
    const size_t lv_bytes = nmb * VP8_MB_COEFS * sizeof(int16_t), md_bytes = nmb * 4, bm_bytes = bpred ? nmb * 16 : 0;
    if (!grow(d_planes, 2 * (ny + 2 * nc) + 256, err) || !grow(d_levels, lv_bytes, err) ||
        !grow(d_modes, md_bytes + bm_bytes, err) || !grow(d_progress, sizeof(int) * (size_t)(f.mbh + 1), err) ||
        !grow(h_out, lv_bytes + md_bytes + bm_bytes, err)) return false;
    uint8_t *Y = d_planes, *U = Y + ny, *V = U + nc;
    f.Y = Y; f.U = U; f.V = V; f.RY = V + nc; f.RU = f.RY + ny; f.RV = f.RU + nc;
    f.levels = d_levels; f.modes = d_modes; f.progress = d_progress;
    f.bmodes = bpred ? d_modes + md_bytes : nullptr;                    // modes | sub-block modes, brought back in one copy
    const int qi = vp8_qindex(quality);
    vp8_quant_factors(qi, f.q);
    int rc = launch_vp8_rgb_to_yuv(d_r, d_g, d_b, w, h, Y, U, V, st);
    if (!rc) rc = bpred ? launch_vp8_encode_bpred(f, st) : launch_vp8_encode(f, st);
    if (!launch_ok(rc, "vp8 kernels", err)) return false;
    // The residual token pass runs on the device too (one thread per macroblock): what comes back is the frame's decision list and the
    // tallies per probability slot, a third of the bytes of the levels; B200_WEBP_TOKENS=host walks the levels on the calling thread instead.
    static const bool host_tokens = [] { const char *e = getenv("B200_WEBP_TOKENS"); return e && !strcmp(e, "host"); }();
    struct Lap { WebpDevice *d; std::chrono::steady_clock::time_point a, b; ~Lap() { d->last_wait_ms = std::chrono::duration<double, std::milli>(b - a).count(); d->last_code_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - b).count(); } };
    if (host_tokens) {
        CU(cudaMemcpyAsync(h_out, d_levels, lv_bytes, cudaMemcpyDeviceToHost, st));
        CU(cudaMemcpyAsync(h_out + lv_bytes, d_modes, md_bytes + bm_bytes, cudaMemcpyDeviceToHost, st));
        const auto t0 = std::chrono::steady_clock::now();
        CU(stream_wait(st));
        Lap lap{this, t0, std::chrono::steady_clock::now()};
        g_d2h_bytes += lv_bytes + md_bytes + bm_bytes;
        if (levels_out) memcpy(levels_out, h_out, lv_bytes);
        if (modes_out) memcpy(modes_out, h_out + lv_bytes, md_bytes);
        if (bmodes_out && bpred) memcpy(bmodes_out, h_out + lv_bytes + md_bytes, bm_bytes);
        if (!vp8_write_file(w, h, qi, reinterpret_cast<const int16_t *>(h_out.get()), h_out + lv_bytes, out, bpred ? h_out + lv_bytes + md_bytes : nullptr)) {
            err = "VP8 frame cannot be framed (first partition too large)"; overflow = true; return false;
        }
        return true;
    }
    // work: mask | counts | offsets | tallies | carried Y2 contexts (2 bytes per macroblock)
    const size_t hist_words = (size_t)vt::kNumProbs * 2, work_words = 3 * (nmb + 1) + hist_words + (2 * nmb + 3) / 4;
    const size_t temp_bytes = vp8_tokens_temp_bytes((int)nmb);
    if (!grow(d_tokwork, work_words * 4, err) || !grow(d_tokens, nmb * 640 * 2, err) || !grow(h_tokens, nmb * 640 * 2, err)) return false;
    if (!grow(d_toktemp, temp_bytes, err)) return false;
    uint32_t *d_mask = d_tokwork, *d_counts = d_mask + (nmb + 1), *d_offsets = d_counts + (nmb + 1), *d_hist = d_offsets + (nmb + 1);
    uint8_t *d_y2 = reinterpret_cast<uint8_t *>(d_hist + hist_words);
    rc = launch_vp8_token_count(f, d_mask, d_y2, d_counts, d_offsets, d_hist, d_toktemp, d_toktemp.capacity(), st);
    if (!launch_ok(rc, "vp8 token pass", err)) return false;
    // first trip: modes, tallies and the length of the list (+ the levels when a caller wants the stage output)
    // (+ the sub-block modes, which follow the modes on the device and on the host)
    const size_t mdb = ((md_bytes + bm_bytes + 15) / 16) * 16;
    uint8_t *h_modes = h_out, *h_hist = h_out + mdb, *h_total = h_hist + hist_words * 4, *h_levels = h_total + 16;
    if (!grow(h_out, (size_t)(h_levels - h_out) + lv_bytes, err)) return false;
    h_modes = h_out; h_hist = h_out + mdb; h_total = h_hist + hist_words * 4; h_levels = h_total + 16;
    CU(cudaMemcpyAsync(h_modes, d_modes, md_bytes + bm_bytes, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(h_hist, d_hist, hist_words * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(h_total, d_offsets + nmb, 4, cudaMemcpyDeviceToHost, st));
    if (levels_out) CU(cudaMemcpyAsync(h_levels, d_levels, lv_bytes, cudaMemcpyDeviceToHost, st));
    const auto t0 = std::chrono::steady_clock::now();
    CU(stream_wait(st));
    const size_t total = *reinterpret_cast<const uint32_t *>(h_total);
    if (total > nmb * (size_t)vt::kMaxDecisionsPerMb) { err = "vp8 token pass: decision count out of range"; return false; }
    if (!grow(d_tokens, total * 2 + 64, err) || !grow(h_tokens, total * 2 + 64, err)) return false;
    rc = launch_vp8_token_write(f, d_mask, d_y2, d_offsets, d_tokens, (uint32_t)std::min<size_t>(d_tokens.capacity() / 2, 0xFFFFFFFFu), st);
    if (!launch_ok(rc, "vp8 token pass", err)) return false;
    if (total) CU(cudaMemcpyAsync(h_tokens, d_tokens, total * 2, cudaMemcpyDeviceToHost, st));
    CU(stream_wait(st));
    Lap lap{this, t0, std::chrono::steady_clock::now()};
    g_d2h_bytes += md_bytes + bm_bytes + hist_words * 4 + 4 + total * 2 + (levels_out ? lv_bytes : 0);
    if (levels_out) memcpy(levels_out, h_levels, lv_bytes);
    if (modes_out) memcpy(modes_out, h_modes, md_bytes);
    if (bmodes_out && bpred) memcpy(bmodes_out, h_modes + md_bytes, bm_bytes);
    if (!vp8_write_file_tokens(w, h, qi, h_modes, reinterpret_cast<const uint32_t *>(h_hist), reinterpret_cast<const uint16_t *>(h_tokens.get()), total, out,
                               bpred ? h_modes + md_bytes : nullptr)) {
        err = "VP8 frame cannot be framed (first partition too large)"; overflow = true; return false;
    }
    return true;
}

bool WebpDevice::encode_host_rgb(const uint8_t *rgb, int w, int h, int quality, void *stream_, std::vector<uint8_t> &out, std::string &err,
                                 int16_t *levels_out, uint8_t *modes_out, uint8_t *bmodes_out, bool force_bpred)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const size_t n = (size_t)w * h;
    if (!grow(h_rgb, 3 * n, err) || !grow(d_rgb, 3 * n, err)) return false;
    memcpy(h_rgb, rgb, 3 * n);
    CU(cudaMemcpyAsync(d_rgb, h_rgb, 3 * n, cudaMemcpyHostToDevice, st));
    return encode_planes(d_rgb, d_rgb + n, d_rgb + 2 * n, w, h, quality, st, out, err, levels_out, modes_out, bmodes_out, force_bpred);
}

} // namespace b200
