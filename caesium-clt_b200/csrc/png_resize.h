// png_resize.h -- the PNG resize leg's own kernels (png_resize.cu): un-filtered PNG rows of any colour type / depth / tRNS -> planar
// samples of the image crate's decoded type, and planes -> PNG rows.  K3 (resize_kernels.cu) resamples the planes in between.
#pragma once
#include <cstdint>
#include <cstddef>
#include "png_host.h"

namespace b200 {

// What libcaesium's resize path decodes a PNG to (image::load_from_memory, the png crate with EXPAND): every channel kept, 16 bits
// stay 16 bits.  Grey 1/2/4/8 -> L8 (sub-byte samples scaled v * 255 / (2^d - 1)), palette -> RGB8, a tRNS colour key or palette
// tRNS adds an alpha channel (LA / RGBA).
struct PngDecodedType { int color_type, channels, depth; };
PngDecodedType png_decoded_type(const PngInfo &info);

// The source's header rewritten for the resized image (nw x nh of the decoded type).  The image crate's round trip keeps no
// ancillary chunk, so the resized file carries none of the source's: PLTE, tRNS and every kept chunk are cleared here, whatever
// keep_metadata asked for.  PLTE / tRNS come back only from the back end's own reductions.
void png_resized_info(PngInfo &info, uint32_t nw, uint32_t nh);

// 256 palette entries as R | G << 8 | B << 16 | A << 24 (entries past PLTE opaque black, past tRNS opaque), passed by value
struct PngLut { uint32_t v[256]; };
PngLut png_palette_lut(const PngInfo &info);

// d_raw [h][row_bytes] (the source's layout) -> planes [channels][h][w] of png_decoded_type(info): uint8_t planes for depth 8,
// uint16_t planes for depth 16 (big-endian input)
int launch_png_expand_planes(const uint8_t *d_raw, const PngInfo &info, const PngLut &lut, void *planes, void *stream);
// planes [channels][h][w] (depth 8: uint8_t, 16: uint16_t) -> interleaved PNG rows [h][w * channels * depth / 8], 16 bits big-endian
int launch_png_pack_planes(const void *planes, int channels, int depth, int w, int h, uint8_t *d_raw, void *stream);

} // namespace b200
