// gif_kernels.h -- launchers of the GIF leg's kernels (gif_kernels.cu; rules in gif_core.h).  Each returns a cudaError_t (0 =
// launched).
#pragma once
#include <cstddef>
#include <cstdint>
#include "gif_core.h"

namespace b200 {

// box[0..7] (zeroed by the caller) of canvases a -> b, w pixels wide: the changed pixels' bounding box as (w - x0, h - y0, x1, y1)
// maxima in words 0..3, and the same for the pixels that go from opaque to clear in words 4..7 (x1 == 0: none)
int launch_gif_diff(const uint32_t *a, const uint32_t *b, int w, int h, uint32_t *box, void *stream);
// rectangle r of canvas cur, masked against prev as in gif_out_pixel (redraw: the positions drawn whatever they hold), into out
int launch_gif_crop(const uint32_t *prev, const uint32_t *cur, int w, GifRect r, GifRect redraw, uint32_t *out, void *stream);
// n pixels of 8-bit planes r, g, b (a grey source passes one plane three times) and an optional alpha plane a -> canvas words
// (gif_canvas_pixel) in out
int launch_gif_canvas(const uint8_t *r, const uint8_t *g, const uint8_t *b, const uint8_t *a, size_t n, uint32_t *out, void *stream);
// n RGBA8 words -> canvas words, in place
int launch_gif_canvas_rgba(uint32_t *px, size_t n, void *stream);
// segmented LZW: per segment its codes (GIF_SEG_CODES apart), their count and their bit total (bits[nseg] is left alone)
int launch_gif_walk(const uint8_t *idx, size_t n, int m, int nseg, uint16_t *codes, uint32_t *ncodes, unsigned long long *bits, void *stream);
// the codes at their scanned bit offsets into zeroed words
int launch_gif_emit(const uint16_t *codes, const uint32_t *ncodes, const unsigned long long *off, int nseg, uint32_t *words, void *stream);
// the (off[nseg] + 7) / 8 LZW bytes as sub-blocks and terminator; cap bounds the output size
int launch_gif_blocks(const uint8_t *data, const unsigned long long *off, int nseg, size_t cap, uint8_t *out, void *stream);

} // namespace b200
