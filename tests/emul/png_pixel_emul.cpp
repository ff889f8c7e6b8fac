// CPU run of the PNG-row -> ARGB rule the lossless WebP conversion's kernels apply (csrc/png_pixel_core.h, k_png_rows_argb /
// k_png_rows_planes in csrc/png_webp.cu): every pixel of every row through png_pix_argb with the rule and palette the product builds.
// The test compares the result with a numpy restatement.  Test infrastructure only.
#include <cstdint>
#include <cstddef>
#include "../../caesium-clt_b200/csrc/png_pixel_core.h"

using namespace b200;

// raw: h rows of rb bytes (no filter byte); out: h * w words A << 24 | R << 16 | G << 8 | B
extern "C" void emul_png_rows_argb(const uint8_t *raw, size_t rb, int w, int h, int ct, int bd, const uint8_t *plte, size_t nplte, const uint8_t *trns,
                                   size_t ntrns, uint32_t *out)
{
    const PngPixRule R = png_pix_rule(ct, bd, trns, ntrns);
    const PngPixLut lut = png_pix_lut(plte, nplte, trns, ntrns);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) out[(size_t)y * w + x] = png_pix_argb(raw + (size_t)y * rb, (uint32_t)x, R, lut.v);
}
