// gif_device.h -- per-slot device state of the GIF leg (gif_device.cu; rules in gif_core.h).
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>
#include "dev_buffer.h"

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
    DeviceBuffer<uint8_t> d_temp, d_blocks;
    PinnedBuffer<uint32_t> h_canvas, h_box;
    PinnedBuffer<uint8_t> h_out;
    double decode_ms = 0;        // host decoding of the last encode() (tracing)

    // the file behind rd (open() done) at `quality` through the quantiser q; corrupt says whether a failure was the input's
    bool encode(GifReader &rd, PngQuant &q, int quality, void *stream, std::vector<uint8_t> &out, bool &corrupt, std::string &err);
    // the segmented LZW coder alone: n indices at d_idx (each below 2^m) -> sub-blocked image data with its terminator, appended
    bool lzw(const uint8_t *d_idx, size_t n, int m, void *stream, std::vector<uint8_t> &out, std::string &err);
};

} // namespace b200
