// vp8_kernels.h -- K8: the device half of the WebP (lossy VP8 key frame) leg, SURVEY.md §8a row a10:
// caesium::convert_in_memory(.., WebP) (caesium-clt's src/compressor.rs:288-292 -> libcaesium webp::compress -> libwebp).
// RGB -> Y'CbCr 4:2:0, then per macroblock: intra mode choice, forward DCT/WHT, quantisation, and the decoder-exact
// reconstruction the next macroblocks predict from.  The boolean entropy coder stays on the host (vp8_host.cpp).
#pragma once
#include <cstdint>
#include <cstddef>

namespace b200 {

constexpr int VP8_MB_COEFS = 25 * 16;        // int16 levels per macroblock: Y2, 16 Y, 4 U, 4 V, each 16 in zigzag order

struct Vp8Frame {
    int w = 0, h = 0, mbw = 0, mbh = 0;
    int q[6] = {0, 0, 0, 0, 0, 0};           // y1 dc, y1 ac, y2 dc, y2 ac, uv dc, uv ac
    const uint8_t *Y = nullptr, *U = nullptr, *V = nullptr;     // source planes, macroblock-padded (pitch mbw*16 / mbw*8)
    uint8_t *RY = nullptr, *RU = nullptr, *RV = nullptr;        // reconstruction, same geometry
    int16_t *levels = nullptr;               // [mbh*mbw][VP8_MB_COEFS]
    uint8_t *modes = nullptr;                // [mbh*mbw][4]: ymode, uvmode, skip, 0   (modes: 0 DC, 1 TM, 2 V, 3 H; ymode 4 B_PRED)
    uint8_t *bmodes = nullptr;               // [mbh*mbw][16]: sub-block modes (vp8_bpred_core.h; a 16x16 macroblock's ymode x 16).  B_PRED encoder only.
    int *progress = nullptr;                 // [mbh + 1]: macroblocks finished per row; [mbh] = row ticket.  Zeroed by the launcher.
};

// planar RGB (pitch w) -> macroblock-padded Y, U, V (libwebp fixed-point weights, 2x2 box chroma, edges replicated)
int launch_vp8_rgb_to_yuv(const uint8_t *r, const uint8_t *g, const uint8_t *b, int w, int h, uint8_t *Y, uint8_t *U, uint8_t *V, void *stream);
// wavefront over macroblocks: one warp per macroblock row, rows released in ticket order
int launch_vp8_encode(const Vp8Frame &f, void *stream);
// the same with 4x4 intra prediction (B_PRED) chosen per macroblock by rate and distortion (vp8_bpred_core.h); also fills f.bmodes.
// Rows trail the row above by two macroblocks.
int launch_vp8_encode_bpred(const Vp8Frame &f, void *stream);
// The residual token pass (RFC 6386 section 13) on the device, one thread per macroblock (vp8_tokens_core.h): masks of the blocks with
// coded coefficients, the carried Y2 contexts (d_y2[2 * nmb]: from above, then from the left), a counting walk (decisions per macroblock -> d_counts[nmb + 1]; tallies per probability slot -> d_hist[kNumProbs * 2]),
// exclusive scan into d_offsets[nmb + 1] (the last entry = decisions in the frame) ...
size_t vp8_tokens_temp_bytes(int nmb);
int launch_vp8_token_count(const Vp8Frame &f, uint32_t *d_mask, uint8_t *d_y2, uint32_t *d_counts, uint32_t *d_offsets, uint32_t *d_hist, void *d_temp, size_t temp_bytes, void *stream);
// ... and the same walk writing the 16-bit decision records at every macroblock's offset (macroblocks whose records would pass `capacity` are left out:
// the caller sizes the buffer from d_offsets[nmb] first)
int launch_vp8_token_write(const Vp8Frame &f, const uint32_t *d_mask, const uint8_t *d_y2, const uint32_t *d_offsets, uint16_t *d_tokens, uint32_t capacity, void *stream);

} // namespace b200
