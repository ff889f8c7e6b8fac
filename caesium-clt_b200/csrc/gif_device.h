// gif_device.h -- per-slot device state of the GIF leg (gif_device.cu; rules in gif_core.h).
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>
#include "dev_buffer.h"
#include "gif_core.h"

namespace b200 {

class GifReader;
struct PngQuant;

// Re-encodes one GIF: every decoded canvas goes up through pinned staging into one of three resident canvases (the canvas before
// the pending frame, the pending frame's and the incoming one), k_gif_diff decides what changed, and a pending frame is written
// once the next differing canvas shows whether it must be disposed to background.  Buffers are high-water allocations kept
// between calls.
struct GifDevice {
    DeviceBuffer<uint32_t> d_canvas[3], d_box, d_ncodes, d_words;
    DeviceBuffer<uint16_t> d_codes;
    DeviceBuffer<unsigned long long> d_bits, d_off;
    DeviceBuffer<uint8_t> d_temp, d_blocks, d_planes;
    PinnedBuffer<uint32_t> h_canvas, h_box;
    PinnedBuffer<uint8_t> h_out;
    double decode_ms = 0;        // host decoding of the last encode() (tracing)

    // the file behind rd (open() done) at `quality` through the quantiser q; corrupt says whether a failure was the input's
    bool encode(GifReader &rd, PngQuant &q, int quality, void *stream, std::vector<uint8_t> &out, bool &corrupt, std::string &err);
    // A converted source: the W x H canvas already in q.d_rgba (gif_canvas_pixel words) -> a whole one-frame GIF, the file encode()
    // writes for a one-frame GIF of that canvas without a loop count
    bool encode_canvas(PngQuant &q, int W, int H, int quality, void *stream, std::vector<uint8_t> &out, std::string &err);
    // the canvas of a converted source into q: 8-bit device planes r, g, b and an optional alpha plane a (null: opaque) ...
    bool canvas_from_planes(PngQuant &q, const uint8_t *r, const uint8_t *g, const uint8_t *b, const uint8_t *a, int W, int H, void *stream, std::string &err);
    // ... host planes rgb [3][H][W] and an optional alpha plane, uploaded once ...
    bool canvas_from_host(PngQuant &q, const uint8_t *rgb, const uint8_t *a, int W, int H, void *stream, std::string &err);
    // ... or the RGBA8 image q already holds (PngQuant::expand), in place
    bool canvas_from_rgba(PngQuant &q, void *stream, std::string &err);
    // the segmented LZW coder alone: n indices at d_idx (each below 2^m) -> sub-blocked image data with its terminator, appended
    bool lzw(const uint8_t *d_idx, size_t n, int m, void *stream, std::vector<uint8_t> &out, std::string &err);

private:
    // the frame whose pixels q holds (rgba_for / expand done), quantised at `quality`: frame head and image data, appended
    bool code_frame(PngQuant &q, int quality, int delay, int disposal, GifRect r, void *stream, std::vector<uint8_t> &out, std::string &err);
};

} // namespace b200
