// png_adam7_core.h -- the geometry of an Adam7-interlaced PNG (PNG 8.2), shared by the device kernels (png_kernels.cu
// k_png_adam7_unfilter / k_png_adam7_gather), the host decoder (png_host.cpp png_decode) and the CPU emulation
// (tests/emul/adam7_emul.cpp).  An interlaced image is seven reduced images ("passes"), each a PNG image of its own: rows of
// filter byte + filtered bytes, one pass after another in the inflated stream.  A pass with zero width or zero height has no
// rows and no filter bytes.  Once un-filtered, the passes' rows sit pass after pass in a "pass-packed" buffer (the stream less
// its filter bytes), and adam7_gather_byte rebuilds the full image's rows from it.
#pragma once
#include <cstddef>
#include <cstdint>

#if defined(__CUDACC__)
#define ADAM7_HD __host__ __device__ __forceinline__
#else
#define ADAM7_HD inline
#endif

namespace b200 {

struct Adam7Pass {
    uint32_t w, h;              // pixels per row, rows (either may be 0: the pass is empty)
    size_t rb;                  // bytes per row without the filter byte
    size_t filt_off, raw_off;   // first byte of the pass in the inflated stream / in the pass-packed buffer
};
struct Adam7Layout {
    Adam7Pass pass[7];
    size_t filt_bytes, raw_bytes;   // the whole inflated stream / the whole pass-packed buffer
};

// pass p (0..6): first column / row and step between columns / rows
ADAM7_HD uint32_t adam7_x0(int p) { return p == 1 ? 4u : p == 3 ? 2u : p == 5 ? 1u : 0u; }
ADAM7_HD uint32_t adam7_y0(int p) { return p == 2 ? 4u : p == 4 ? 2u : p == 6 ? 1u : 0u; }
ADAM7_HD uint32_t adam7_dx(int p) { return p <= 1 ? 8u : p <= 3 ? 4u : p <= 5 ? 2u : 1u; }
ADAM7_HD uint32_t adam7_dy(int p) { return p <= 2 ? 8u : p <= 4 ? 4u : 2u; }

// the pass that holds pixel (x, y): the 8 x 8 pattern of PNG 8.2
ADAM7_HD int adam7_pass_of(uint32_t x, uint32_t y)
{
    if (y & 1) return 6;
    if (x & 1) return 5;
    if (y & 2) return 4;
    if (x & 2) return 3;
    if (y & 4) return 2;
    return (x & 4) ? 1 : 0;
}

// W x H image of bits_per_pixel bits per pixel
ADAM7_HD void adam7_layout(uint32_t W, uint32_t H, int bits_per_pixel, Adam7Layout &L)
{
    size_t fo = 0, ro = 0;
    for (int p = 0; p < 7; p++) {
        Adam7Pass &P = L.pass[p];
        const uint32_t x0 = adam7_x0(p), y0 = adam7_y0(p), dx = adam7_dx(p), dy = adam7_dy(p);
        P.w = W > x0 ? (W - x0 + dx - 1) / dx : 0;
        P.h = H > y0 ? (H - y0 + dy - 1) / dy : 0;
        if (!P.w || !P.h) { P.w = P.h = 0; }
        P.rb = ((size_t)P.w * (size_t)bits_per_pixel + 7) / 8;
        P.filt_off = fo; P.raw_off = ro;
        fo += (size_t)P.h * (P.rb + (P.h ? 1 : 0));
        ro += (size_t)P.h * P.rb;
    }
    L.filt_bytes = fo; L.raw_bytes = ro;
}

// Byte i of full-image row y (row_bytes = (W * bits + 7) / 8 bytes) from the pass-packed rows.  Depths below 8 collect the
// pixels of one byte from several passes; bits after the row's last pixel are zero, as in a non-interlaced file's rows.
ADAM7_HD uint8_t adam7_gather_byte(const uint8_t *packed, const Adam7Layout &L, int bits_per_pixel, uint32_t W, uint32_t y, size_t i)
{
    if (bits_per_pixel >= 8) {
        const uint32_t B = (uint32_t)bits_per_pixel / 8, x = (uint32_t)(i / B), k = (uint32_t)(i % B);
        const int p = adam7_pass_of(x, y);
        const Adam7Pass &P = L.pass[p];
        const size_t px = (x - adam7_x0(p)) / adam7_dx(p), py = (y - adam7_y0(p)) / adam7_dy(p);
        return packed[P.raw_off + py * P.rb + px * B + k];
    }
    const uint32_t per = 8u / (uint32_t)bits_per_pixel, mask = (1u << bits_per_pixel) - 1;
    uint32_t v = 0;
    for (uint32_t j = 0; j < per; j++) {
        const uint32_t x = (uint32_t)i * per + j;
        if (x >= W) break;
        const int p = adam7_pass_of(x, y);
        const Adam7Pass &P = L.pass[p];
        const size_t px = (x - adam7_x0(p)) / adam7_dx(p), py = (y - adam7_y0(p)) / adam7_dy(p);
        const uint32_t s = packed[P.raw_off + py * P.rb + px / per];
        const uint32_t val = (s >> (8 - bits_per_pixel * (1 + (uint32_t)(px % per)))) & mask;
        v |= val << (8 - bits_per_pixel * (1 + j));
    }
    return (uint8_t)v;
}

} // namespace b200
