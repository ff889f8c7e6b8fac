// png_webp.h -- the PNG front end of the lossless WebP conversion (png_webp.cu): un-filtered rows of any colour type / depth / tRNS
// (PngDevice::d_raw) -> the pixels of png_pixel_core.h, either straight into the VP8L encoder's ARGB buffer or as 8-bit planes for K3.
#pragma once
#include <cstdint>
#include <cstddef>
#include "png_host.h"
#include "png_pixel_core.h"

namespace b200 {

PngPixRule png_pix_rule(const PngInfo &info);
PngPixLut png_pix_lut(const PngInfo &info);
// true when the header allows a pixel with alpha below 255 (an alpha channel or a tRNS chunk)
bool png_may_be_translucent(const PngInfo &info);

// d_raw [h][row_bytes] -> argb[h * w] with subtract-green applied (the encoder's input); *flags is zeroed, then bit 0 is set when some alpha is below 255
int launch_png_rows_argb(const uint8_t *d_raw, const PngInfo &info, uint32_t *argb, uint32_t *flags, void *stream);
// d_raw [h][row_bytes] -> 8-bit planes r, g, b and (a != nullptr) alpha of h * w bytes; *flags as above
int launch_png_rows_planes(const uint8_t *d_raw, const PngInfo &info, uint8_t *r, uint8_t *g, uint8_t *b, uint8_t *a, uint32_t *flags, void *stream);

} // namespace b200
