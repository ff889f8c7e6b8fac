// webp_anim_device.h -- per-slot device state of the animated WebP leg (webp_anim_device.cu; rules in webp_anim_core.h).
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>
#include "dev_buffer.h"
#include "webp_anim_core.h"

namespace b200 {

class WebpAnimReader;
struct WebpDevice;
struct Vp8lDevice;
struct PngDevice;

// Re-encodes one animated WebP: every decoded frame rectangle goes up through pinned staging, k_webp_anim_compose draws it onto
// the resident canvas, k_gif_diff finds what changed since the last kept canvas, and k_webp_anim_crop hands the output rectangle
// to the lossy (K8) or the lossless (VP8L) encoder.  Two canvases suffice: a dropped canvas equals the kept one before it, so the
// canvas the next frame is drawn on is always the last kept canvas.  Only coded frames and, for a lossy frame, its alpha plane come
// back to the host, which writes the container.  Buffers are high-water allocations kept between calls.
struct WebpAnimDevice {
    DeviceBuffer<uint32_t> d_canvas[2], d_frame, d_box;
    DeviceBuffer<uint8_t> d_planes;
    PinnedBuffer<uint32_t> h_frame, h_box;
    PinnedBuffer<uint8_t> h_alpha;
    // tracing of the last encode(): host decode, compose and difference, the encoders (K8 or VP8L), and within those the host
    // coder (VP8's boolean coder, or VP8L's header and emission)
    double decode_ms = 0, compose_ms = 0, encode_ms = 0, code_ms = 0;
    int frames_out = 0;

    // the file behind rd (open() done): lossless frames through vp8l, else lossy frames at `quality` through webp, their alpha
    // planes through png's LZ77 kernels; corrupt says whether a failure was the input's
    bool encode(WebpAnimReader &rd, WebpDevice &webp, Vp8lDevice &vp8l, PngDevice &png, bool lossless, int quality, void *stream,
                std::vector<uint8_t> &out, bool &corrupt, std::string &err);

private:
    // the rectangle r of canvas c as the sub-chunks of one ANMF, appended to out; alpha |= some alpha in it is below 255
    bool code_rect(const uint32_t *c, int W, WaRect r, WebpDevice &webp, Vp8lDevice &vp8l, PngDevice &png, bool lossless, int quality, void *stream,
                   std::vector<uint8_t> &out, bool &alpha, std::string &err);
};

} // namespace b200
