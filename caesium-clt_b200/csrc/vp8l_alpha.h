// vp8l_alpha.h -- the alpha plane of a lossy WebP: the ALPH chunk of a VP8X file (libcaesium webp::compress on an image with
// transparency -> libwebp WebPEncodeRGBA: lossy VP8 colour + losslessly coded alpha; caesium-clt's src/compressor.rs:288-292, :305).
// The plane is coded as a VP8L image stream (WebP lossless bitstream, alpha in the green channel, no transforms, no colour cache,
// one prefix-code group) from LZ77 tokens the device's K7 kernels produce over the plane.
#pragma once
#include <cstdint>
#include <cstddef>
#include <vector>

namespace b200 {

// Prediction filter of the ALPH chunk (0 none, 1 horizontal, 2 vertical, 3 gradient: the decoder adds the prediction back): the one
// whose residuals have the lowest order-0 entropy on every fourth row.  filtered receives the residual plane when the answer is not 0.
int webp_alpha_choose_filter(const uint8_t *alpha, int width, int height, std::vector<uint8_t> &filtered);

// tokens: K7 / dfl_core.h format (bit 31 clear: literal byte; set: (len - 3) << 16 | (dist - 1)), covering width * height bytes of the
// (filtered) plane.  alph = payload of the ALPH chunk (header byte + VP8L image stream).  false: the tokens do not cover the plane.
bool vp8l_alpha_from_tokens(const uint32_t *tok, size_t ntok, int width, int height, std::vector<uint8_t> &alph, int filter = 0);

// RIFF container of a lossy WebP with alpha: VP8X (alpha flag) + ALPH + the 'VP8 ' chunk taken out of `simple_file` (a RIFF file
// holding only a 'VP8 ' chunk, as vp8_write_file produces)
bool webp_wrap_alpha(const std::vector<uint8_t> &simple_file, const std::vector<uint8_t> &alph, int width, int height, std::vector<uint8_t> &out);

} // namespace b200
