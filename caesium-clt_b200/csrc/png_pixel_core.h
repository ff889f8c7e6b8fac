// png_pixel_core.h -- one pixel of an un-filtered PNG row as the conversions to WebP see it, shared by the device kernels
// (png_webp.cu) and the CPU emulation (tests/emul/png_pixel_emul.cpp).  The rule is the lossy PNG -> WebP conversion's
// (api.cpp png_expand_planar without grey planes, png_extract_alpha):
//   - palette: the PLTE entry (an index past PLTE: 0, 0, 0), alpha from tRNS (an index past tRNS: 255);
//   - grey: one value for R, G and B; sub-byte samples scaled v * 255 / (2^bd - 1);
//   - 16-bit samples and 16-bit alpha: the high byte;
//   - a tRNS colour key (grey, RGB) compares against the full-precision sample and makes the pixel's alpha 0, else 255.
#pragma once
#include <cstddef>
#include <cstdint>

#if defined(__CUDACC__)
#define PNGPX_HD __host__ __device__ __forceinline__
#else
#define PNGPX_HD inline
#endif

namespace b200 {

struct PngPixRule {
    int ct, bd;                 // colour type, bit depth
    int key;                    // 1: a tRNS colour key applies (grey: k[0]; RGB: k[0..2])
    uint32_t k[3];
};
// the palette as A << 24 | R << 16 | G << 8 | B, 256 entries (passed by value to the kernels)
struct PngPixLut { uint32_t v[256]; };

inline PngPixRule png_pix_rule(int ct, int bd, const uint8_t *trns, size_t ntrns)
{
    PngPixRule r{ct, bd, 0, {0, 0, 0}};
    if (ct == 0 && ntrns >= 2) { r.key = 1; r.k[0] = (uint32_t)trns[0] << 8 | trns[1]; }
    if (ct == 2 && ntrns >= 6) { r.key = 1; for (int c = 0; c < 3; c++) r.k[c] = (uint32_t)trns[2 * c] << 8 | trns[2 * c + 1]; }
    return r;
}

inline PngPixLut png_pix_lut(const uint8_t *plte, size_t nplte, const uint8_t *trns, size_t ntrns)
{
    PngPixLut l;
    for (size_t i = 0; i < 256; i++) {
        const uint32_t a = i < ntrns ? trns[i] : 255u;
        const uint32_t rgb = 3 * i + 2 < nplte ? (uint32_t)plte[3 * i] << 16 | (uint32_t)plte[3 * i + 1] << 8 | plte[3 * i + 2] : 0u;
        l.v[i] = a << 24 | rgb;
    }
    return l;
}

// sample k of a row: 16 bits big-endian, 8 bits, or a sub-byte value (MSB first)
PNGPX_HD uint32_t png_pix_sample(const uint8_t *row, uint32_t k, int bd)
{
    if (bd == 16) return (uint32_t)row[2 * k] << 8 | row[2 * k + 1];
    if (bd == 8) return row[k];
    const uint32_t bit = k * (uint32_t)bd;
    return (uint32_t)(row[bit >> 3] >> (8 - bd - (int)(bit & 7))) & ((1u << bd) - 1);
}

// a full-precision sample as 8 bits: the high byte of 16, sub-byte greys scaled
PNGPX_HD uint32_t png_pix_eight(uint32_t v, int bd) { return bd == 16 ? v >> 8 : bd < 8 ? v * 255u / ((1u << bd) - 1) : v; }

// pixel x of an un-filtered row -> A << 24 | R << 16 | G << 8 | B
PNGPX_HD uint32_t png_pix_argb(const uint8_t *row, uint32_t x, const PngPixRule &R, const uint32_t *lut)
{
    const int bd = R.bd;
    switch (R.ct) {
        case 3: return lut[png_pix_sample(row, x, bd) & 255u];
        case 0: {
            const uint32_t v = png_pix_sample(row, x, bd), g = png_pix_eight(v, bd);
            return (R.key && v == R.k[0] ? 0u : 0xFF000000u) | g * 0x010101u;
        }
        case 4: {
            const uint32_t g = png_pix_eight(png_pix_sample(row, 2 * x, bd), bd), a = png_pix_eight(png_pix_sample(row, 2 * x + 1, bd), bd);
            return a << 24 | g * 0x010101u;
        }
        case 2: {
            const uint32_t r = png_pix_sample(row, 3 * x, bd), g = png_pix_sample(row, 3 * x + 1, bd), b = png_pix_sample(row, 3 * x + 2, bd);
            const bool keyed = R.key && r == R.k[0] && g == R.k[1] && b == R.k[2];
            return (keyed ? 0u : 0xFF000000u) | png_pix_eight(r, bd) << 16 | png_pix_eight(g, bd) << 8 | png_pix_eight(b, bd);
        }
        default: {
            const uint32_t r = png_pix_sample(row, 4 * x, bd), g = png_pix_sample(row, 4 * x + 1, bd), b = png_pix_sample(row, 4 * x + 2, bd),
                           a = png_pix_sample(row, 4 * x + 3, bd);
            return png_pix_eight(a, bd) << 24 | png_pix_eight(r, bd) << 16 | png_pix_eight(g, bd) << 8 | png_pix_eight(b, bd);
        }
    }
}

} // namespace b200
