// vp8_host.h -- host half of the WebP (lossy VP8) leg: quality -> quantiser mapping, the boolean entropy coder, header / mode /
// token partitions (RFC 6386 sections 7, 9, 13, 19) and the RIFF container, around the levels and modes K8 leaves in HBM.
#pragma once
#include <cstdint>
#include <cstddef>
#include <vector>

namespace b200 {

// libwebp's quality (0..100) -> base quantiser index curve (one segment)
int vp8_qindex(int quality);
// strength of the decoder-side simple loop filter requested in the frame header: none at the finest quantisers, rising with
// the step size (+0.5..0.9 dB on photographic content at -q 10..75)
int vp8_filter_level(int qindex);
// dequantisation factors of an index: y1 dc, y1 ac, y2 dc, y2 ac, uv dc, uv ac (RFC 6386 9.6 / 14.1)
void vp8_quant_factors(int qindex, int f[6]);

// levels: [mbh*mbw][25][16] int16 in zigzag order (Y2, 16 Y, 4 U, 4 V); modes: [mbh*mbw][4] = ymode, uvmode, skip, 0
// (prediction modes 0 DC, 1 TM, 2 V, 3 H; ymode 4 = B_PRED, whose 16 sub-block modes are bmodes[mb][16] in raster order, numbered
// as in vp8_bpred_core.h, and whose Y2 levels are zero).  Writes a complete simple-format .webp file.  false if the frame cannot be
// framed: a mode out of range (ymode 4 without bmodes among them), or a first partition of 2^19 bytes or more.
bool vp8_write_file(int width, int height, int qindex, const int16_t *levels, const uint8_t *modes, std::vector<uint8_t> &out, const uint8_t *bmodes = nullptr);
// the same from the frame's decision list (vp8_tokens_core.h record format, macroblocks in raster order) and the tallies of its tree
// decisions cnt[slot][bit] -- what k_vp8_tokens leaves on the device: the host only picks the probabilities and runs the boolean coder
bool vp8_write_file_tokens(int width, int height, int qindex, const uint8_t *modes, const uint32_t *cnt, const uint16_t *tokens, size_t ntokens, std::vector<uint8_t> &out,
                           const uint8_t *bmodes = nullptr);
// mb_no_coeff_skip of the frame: does any macroblock carry the skip flag (modes[4 * mb + 2])
bool vp8_frame_uses_skip(int width, int height, const uint8_t *modes);

} // namespace b200
