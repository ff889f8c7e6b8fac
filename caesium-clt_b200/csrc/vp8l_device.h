// vp8l_device.h -- per-slot device state of the lossless WebP (VP8L) encoder: planar RGB (+ alpha) on the host -> the kernels of
// vp8l_kernels.cu -> a RIFF file holding one VP8L chunk.  Every buffer is a high-water buffer allocated on the first lossless call.
#pragma once
#include <cstdint>
#include <cstddef>
#include <string>
#include <vector>

namespace b200 {

struct Vp8lDevice {
    uint8_t *d_arena = nullptr; size_t cap_arena = 0;          // every per-pixel buffer of Vp8lBuffers
    uint32_t *d_words = nullptr; size_t cap_words = 0;         // the coded pixels
    uint8_t *h_in = nullptr; size_t cap_hin = 0;               // pinned: R | G | B | A planes
    uint8_t *h_small = nullptr; size_t cap_hsmall = 0;         // pinned: histograms | flags | total | modes
    uint8_t *h_codes = nullptr; size_t cap_hcodes = 0;         // pinned: Vp8lCodes
    uint8_t *h_words = nullptr; size_t cap_hwords = 0;         // pinned: the coded pixels coming back
    double last_analyse_ms = 0, last_code_ms = 0;              // tracing: wait for the analysis kernels, header + emission of the last encode
    int last_cache_bits = 0;
    ~Vp8lDevice();
    // rgb: host, planar [3][h][w]; alpha: host [h][w] or nullptr (opaque).  out: the .webp file.
    bool encode(const uint8_t *rgb, const uint8_t *alpha, int w, int h, void *stream, std::vector<uint8_t> &out, std::string &err);
};

} // namespace b200
