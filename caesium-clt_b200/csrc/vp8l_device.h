// vp8l_device.h -- per-slot device state of the lossless WebP (VP8L) encoder: RGB (+ alpha) planes, from the host or already on the
// device, or ARGB pixels a caller's own kernel wrote -> the kernels of vp8l_kernels.cu -> a RIFF file holding one VP8L chunk.  Every
// buffer is a high-water buffer allocated on the first lossless call.
#pragma once
#include <cstdint>
#include <cstddef>
#include <string>
#include <vector>
#include "dev_buffer.h"
#include "vp8l_kernels.h"

namespace b200 {

struct BitsLsb;
// the colour-indexing switch (api.cpp): the encoder also codes images of at most VP8L_PAL_MAX colours through a palette
bool webp_palette();

struct Vp8lDevice {
    DeviceBuffer<uint8_t> d_arena;          // every per-pixel buffer of Vp8lBuffers
    DeviceBuffer<uint32_t> d_words;         // the coded pixels
    PinnedBuffer<uint8_t> h_in;             // R | G | B | A planes of the host entry
    PinnedBuffer<uint8_t> h_small;          // histograms | flags | total | modes
    PinnedBuffer<uint8_t> h_codes;          // Vp8lCodes
    PinnedBuffer<uint8_t> h_words;          // the coded pixels coming back
    double last_analyse_ms = 0, last_code_ms = 0;              // tracing: wait for the analysis kernels, header + emission of the last encode
    int last_cache_bits = 0;
    size_t last_d2h_bytes = 0;              // what the last encode fetched: the analysis results, the coded size and the coded words
    int last_palette = -1;                  // the last encode's colour count with the palette switch on; -1: over VP8L_PAL_MAX or off
    bool last_palette_kept = false;         // the palette variant was the smaller file
    size_t last_bytes[2] = {0, 0};          // file sizes without / with the palette (0: not coded)
    double last_palette_ms = 0;             // the palette kernels' event times (B200_TRACE=2 only)
    std::string palette_trace() const;      // the trace line's palette part ("" with the switch off)
    // rgb: host, planar [3][h][w]; alpha: host [h][w] or nullptr (opaque).  out: the .webp file.  Staged and uploaded, then encode_planes.
    bool encode(const uint8_t *rgb, const uint8_t *alpha, int w, int h, void *stream, std::vector<uint8_t> &out, std::string &err);
    // r, g, b, a: device planes of w x h bytes, ordered on `stream` (a grey source passes one plane three times; a == nullptr: opaque)
    bool encode_planes(const uint8_t *r, const uint8_t *g, const uint8_t *b, const uint8_t *a, int w, int h, void *stream, std::vector<uint8_t> &out, std::string &err);
    // For a caller that writes the pixels itself: reserve() sizes every buffer for w x h (idempotent) and names where the pixels go --
    // argb: n words, subtract-green applied; flags: bit 0 set when some alpha is below 255 (the caller zeroes it first).  encode_packed()
    // then runs everything from the analysis on.
    bool reserve(int w, int h, uint32_t *&argb, uint32_t *&flags, std::string &err);
    bool encode_packed(int w, int h, void *stream, std::vector<uint8_t> &out, std::string &err);
private:
    Vp8lBuffers B{};                        // carved out of d_arena by reserve()
    // one variant after its analysis over cw x h: cache choice, codes and the header's tail after the transforms bw holds, the coded
    // size (file_bytes); then, unless the file would be `below` bytes or more, emission and the RIFF file in out
    bool code_image(int cw, int h, BitsLsb &bw, size_t below, std::vector<uint8_t> &out, size_t &file_bytes, void *stream, std::string &err);
};

} // namespace b200
