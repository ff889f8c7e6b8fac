// png_quant.h -- the lossy PNG leg's palette quantiser on the device (png_quant.cu; rules in png_quant_core.h).
#pragma once
#include <cstdint>
#include <cstddef>
#include <string>
#include <vector>
#include "dev_buffer.h"
#include "png_host.h"

namespace b200 {

// One image at a time: load (host RGBA8 or the un-filtered samples of a PNG already on the device), prepare (histogram, occupied
// cells, distinct-value count: independent of the quality), then quantize at any number of qualities.  Buffers are high-water
// allocations kept between calls.
struct PngQuant {
    // growable, image-sized
    DeviceBuffer<uint32_t> d_rgba, d_sync;
    DeviceBuffer<unsigned long long> d_edge;     // dithering: the last row of each 32-row group, four int16 errors per pixel
    DeviceBuffer<uint8_t> d_idx, d_planes, d_temp;
    // fixed-size
    DeviceBuffer<uint32_t> d_cells, d_coords, d_set, d_flags, d_lut;
    DeviceBuffer<unsigned long long> d_count, d_sums, d_box, d_acc, d_keys;
    DeviceBuffer<uint8_t> d_label, d_cand;
    DeviceBuffer<uint16_t> d_ncand;
    PinnedBuffer<uint8_t> h_small;
    int w = 0, h = 0, ncells = 0, distinct = 0, clear = 0;     // clear: some pixel is fully transparent (palette entry 0 reserved)
    double last_cut_ms = 0;                   // host-driven median cut of the last quantize() (tracing)

    bool load_host(const uint8_t *rgba, int width, int height, void *stream, std::string &err);
    // host planes [nc][h][w] (nc = 1 grey or 3 RGB) and an optional alpha plane, interleaved to RGBA8 on the device
    bool load_planes(const uint8_t *planes, int nc, const uint8_t *alpha, int width, int height, void *stream, std::string &err);
    // d_raw: height * row_bytes un-filtered samples of any PNG colour type / depth (16 bits: high byte; tRNS / palette expanded)
    bool expand(const uint8_t *d_raw, const PngInfo &info, void *stream, std::string &err);
    // room for a width x height RGBA8 image written in place by the caller's kernels (d_rgba), or null with err
    uint32_t *rgba_for(int width, int height, std::string &err);
    bool prepare(void *stream, std::string &err);
    bool exact() const { return distinct <= 256; }
    // palette (RGBA words, R in the low byte) and the indices (left in d_idx).  allow_exact = false quantises an image with at most
    // 256 distinct values too, so that the quality still applies to it.
    bool quantize(int quality, void *stream, std::vector<uint32_t> &palette, std::string &err, bool allow_exact = true);
    bool fetch_indices(uint8_t *idx, void *stream, std::string &err);
    bool fetch_rgba(std::vector<uint8_t> &rgba, void *stream, std::string &err);
    // indices -> rows of `depth`-bit samples (MSB first, padded to bytes) at d_dst
    bool pack(uint8_t *d_dst, int depth, void *stream, std::string &err);
};

// bits per index of a palette of n entries (PNG allows 1, 2, 4, 8)
inline int png_index_depth(int n) { return n <= 2 ? 1 : n <= 4 ? 2 : n <= 16 ? 4 : 8; }

} // namespace b200
