// vp8l_device.h -- per-slot device state of the lossless WebP (VP8L) encoder: planar RGB (+ alpha) on the host -> the kernels of
// vp8l_kernels.cu -> a RIFF file holding one VP8L chunk.  Every buffer is a high-water buffer allocated on the first lossless call.
#pragma once
#include <cstdint>
#include <cstddef>
#include <string>
#include <vector>
#include "dev_buffer.h"

namespace b200 {

struct Vp8lDevice {
    DeviceBuffer<uint8_t> d_arena;          // every per-pixel buffer of Vp8lBuffers
    DeviceBuffer<uint32_t> d_words;         // the coded pixels
    PinnedBuffer<uint8_t> h_in;             // R | G | B | A planes
    PinnedBuffer<uint8_t> h_small;          // histograms | flags | total | modes
    PinnedBuffer<uint8_t> h_codes;          // Vp8lCodes
    PinnedBuffer<uint8_t> h_words;          // the coded pixels coming back
    double last_analyse_ms = 0, last_code_ms = 0;              // tracing: wait for the analysis kernels, header + emission of the last encode
    int last_cache_bits = 0;
    // rgb: host, planar [3][h][w]; alpha: host [h][w] or nullptr (opaque).  out: the .webp file.
    bool encode(const uint8_t *rgb, const uint8_t *alpha, int w, int h, void *stream, std::vector<uint8_t> &out, std::string &err);
};

} // namespace b200
