// webp_anim_kernels.h -- launchers of the animated WebP leg's kernels (webp_anim_kernels.cu); rules in webp_anim_core.h.
#pragma once
#include <cstddef>
#include <cstdint>
#include "webp_anim_core.h"

namespace b200 {

// one frame onto the canvas: out = the step s applied to `in` (both W x H RGBA words), the frame's pixels at `frame`
// (s.rect.w * s.rect.h words); disposal of the previous rectangle, the keyframe zero-fill and blend or replace in one pass
int launch_webp_anim_compose(const uint32_t *in, uint32_t *out, int W, int H, const uint32_t *frame, WaStep s, void *stream);
// rectangle r of the canvas as R, G, B, A planes of r.w * r.h bytes each at planes (the lossy encoder's input) ...
int launch_webp_anim_crop_planes(const uint32_t *canvas, int W, WaRect r, uint8_t *planes, void *stream);
// ... or as subtract-green ARGB words at argb, bit 0 of *flags set when some alpha is below 255 (the lossless encoder's input;
// the caller zeroes *flags first)
int launch_webp_anim_crop_argb(const uint32_t *canvas, int W, WaRect r, uint32_t *argb, uint32_t *flags, void *stream);

} // namespace b200
