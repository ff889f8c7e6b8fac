// webp_anim_device.cu -- host driver of the animated WebP leg (webp_anim_device.h): frame rectangles up, the changed box back,
// the output rectangle cropped into K8 or the VP8L encoder, and only coded frames (plus a lossy frame's alpha plane) back to the
// host, which writes the container.
#include <cuda_runtime.h>
#include <algorithm>
#include <chrono>
#include <cstring>
#include "webp_anim_device.h"
#include "webp_anim_host.h"
#include "webp_anim_kernels.h"
#include "gif_kernels.h"
#include "webp_device.h"
#include "vp8l_device.h"
#include "png_device.h"
#include "vp8l_alpha.h"
#include "stream_wait.h"

namespace b200 {

namespace {
template <class B> bool grow(B &buf, size_t need, std::string &err) { return buf.reserve(need, Grow::Pow2, err); }
template <class B> bool fixed(B &buf, size_t bytes, std::string &err) { return buf.reserve(bytes, Grow::Exact, err); }

using Clock = std::chrono::steady_clock;
double ms_since(Clock::time_point t) { return std::chrono::duration<double, std::milli>(Clock::now() - t).count(); }

// the chunks after the 12-byte RIFF / WEBP header of a file the still encoders wrote (one 'VP8 ' or one VP8L chunk), appended
void append_chunks(const std::vector<uint8_t> &file, std::vector<uint8_t> &out) { out.insert(out.end(), file.begin() + 12, file.end()); }
} // namespace

bool WebpAnimDevice::code_rect(const uint32_t *c, int W, WaRect r, WebpDevice &webp, Vp8lDevice &vp8l, PngDevice &png, bool lossless, int quality,
                               void *stream_, std::vector<uint8_t> &out, bool &alpha, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const size_t n = (size_t)r.w * r.h;
    std::vector<uint8_t> file;
    const auto t0 = Clock::now();
    if (lossless) {
        uint32_t *argb, *flags;
        if (!vp8l.reserve(r.w, r.h, argb, flags, err)) return false;
        CU(cudaMemsetAsync(flags, 0, 4, st));
        if (!launch_ok(launch_webp_anim_crop_argb(c, W, r, argb, flags, st), "k_webp_anim_crop_argb", err) ||
            !vp8l.encode_packed(r.w, r.h, st, file, err)) return false;
        encode_ms += ms_since(t0);
        code_ms += vp8l.last_code_ms;
        alpha |= (file[24] >> 4) & 1;                 // the VP8L header's alpha bit (bit 28 after the signature byte at 20)
        append_chunks(file, out);
        return true;
    }
    if (!grow(d_planes, 4 * n, err) || !grow(h_alpha, n, err)) return false;
    if (!launch_ok(launch_webp_anim_crop_planes(c, W, r, d_planes, st), "k_webp_anim_crop_planes", err)) return false;
    CU(cudaMemcpyAsync(h_alpha, d_planes + 3 * n, n, cudaMemcpyDeviceToHost, st));
    if (!webp.encode_planes(d_planes, d_planes + n, d_planes + 2 * n, r.w, r.h, quality, st, file, err)) return false;   // waits for the stream
    encode_ms += ms_since(t0);
    code_ms += webp.last_code_ms;
    const uint8_t *ap = h_alpha;
    if (!std::all_of(ap, ap + n, [](uint8_t v) { return v == 0xFF; })) {
        // the ALPH chunk rgb_to_webp writes: the filter chosen on the host, LZ77 tokens from K7, the VP8L-coded plane
        alpha = true;
        std::vector<uint32_t> tokens; std::vector<uint8_t> alph, residual;
        const int filter = webp_alpha_choose_filter(ap, r.w, r.h, residual);
        if (!png.plane_tokens(filter ? residual.data() : ap, n, r.w, st, tokens, err)) return false;
        if (!vp8l_alpha_from_tokens(tokens.data(), tokens.size(), r.w, r.h, alph, filter)) { err = "alpha plane could not be coded"; return false; }
        const uint8_t head[8] = {'A', 'L', 'P', 'H', (uint8_t)alph.size(), (uint8_t)(alph.size() >> 8), (uint8_t)(alph.size() >> 16), (uint8_t)(alph.size() >> 24)};
        out.insert(out.end(), head, head + 8);
        out.insert(out.end(), alph.begin(), alph.end());
        if (alph.size() & 1) out.push_back(0);
    }
    append_chunks(file, out);
    return true;
}

bool WebpAnimDevice::encode(WebpAnimReader &rd, WebpDevice &webp, Vp8lDevice &vp8l, PngDevice &png, bool lossless, int quality, void *stream_,
                            std::vector<uint8_t> &out, bool &corrupt, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    corrupt = false;
    decode_ms = compose_ms = encode_ms = code_ms = 0;
    frames_out = 0;
    const int W = rd.width, H = rd.height;
    const size_t np = (size_t)W * H;
    for (auto &c : d_canvas) if (!grow(c, np * 4, err)) return false;
    if (!fixed(d_box, 64, err) || !fixed(h_box, 64, err)) return false;
    out.resize(64);
    out.resize((size_t)webp_anim_put_header(out.data(), W, H, 0, rd.bg, rd.loop));
    const WaRect whole = {0, 0, W, H};
    WaRect prev = {0, 0, 0, 0};
    int prev_flags = 0, prev_key = 0, a = 0;         // d_canvas[a]: the last kept canvas
    size_t dur_at = 0;                               // where the last written frame's duration sits in out
    uint32_t dur = 0;
    bool alpha = false;
    WebpAnimFrame f;
    for (int k = 0;; k++) {
        auto t = Clock::now();
        const bool more = rd.next(f, err);
        decode_ms += ms_since(t);
        if (!more) {
            if (!err.empty()) { corrupt = true; return false; }
            break;
        }
        t = Clock::now();
        const size_t fn = f.rgba.size();
        if (!grow(h_frame, fn * 4, err) || !grow(d_frame, fn * 4, err)) return false;
        memcpy(h_frame, f.rgba.data(), fn * 4);
        CU(cudaMemcpyAsync(d_frame, h_frame, fn * 4, cudaMemcpyHostToDevice, st));
        const WaStep s = webp_anim_step(k, f.rect, f.has_alpha, f.flags, prev, prev_flags, prev_key, W, H);
        prev = f.rect; prev_flags = f.flags; prev_key = s.keyframe;
        const int b = 1 - a;
        if (!launch_ok(launch_webp_anim_compose(d_canvas[a], d_canvas[b], W, H, d_frame, s, st), "k_webp_anim_compose", err)) return false;
        WaRect r = whole;
        if (k > 0) {
            CU(cudaMemsetAsync(d_box, 0, 16, st));
            if (!launch_ok(launch_gif_diff(d_canvas[a], d_canvas[b], W, H, d_box, st), "k_gif_diff", err)) return false;
            CU(cudaMemcpyAsync(h_box, d_box, 16, cudaMemcpyDeviceToHost, st));
            CU(stream_wait(st));
            const uint32_t *bx = h_box;
            if (!bx[2]) {                            // nothing changed: the previous frame lasts longer
                compose_ms += ms_since(t);
                dur = webp_anim_add_duration(dur, f.duration);
                uint8_t *o = out.data() + dur_at;
                o[0] = (uint8_t)dur; o[1] = (uint8_t)(dur >> 8); o[2] = (uint8_t)(dur >> 16);
                continue;
            }
            r = webp_anim_out_rect(W - (int)bx[0], H - (int)bx[1], (int)bx[2], (int)bx[3]);
        }
        compose_ms += ms_since(t);
        const size_t head = out.size();
        out.resize(head + 24);
        if (!code_rect(d_canvas[b], W, r, webp, vp8l, png, lossless, quality, st, out, alpha, err)) return false;
        dur = std::min<uint32_t>(f.duration, WA_MAX_DURATION);
        webp_anim_put_frame_head(out.data() + head, r, dur, out.size() - head - 24);
        dur_at = head + 20;
        frames_out++;
        a = b;
    }
    if (alpha) out[20] |= 0x10;
    webp_anim_finish(out.data(), out.size());
    return true;
}

} // namespace b200
