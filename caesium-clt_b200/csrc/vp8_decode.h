// vp8_decode.h -- host VP8 key-frame DECODER (lossy WebP input): RIFF container, RFC 6386 bitstream, reconstruction, loop filters and
// libwebp's RGB output conversion.  libcaesium's webp::compress decodes its input before it re-encodes
// (caesium::compress_in_memory on a .webp, caesium-clt's src/compressor.rs:305; the reference's own tests require
// samples/w0.webp to succeed, :769-787): this is that decode, as format plumbing in front of the device encoder (K8) -- like the
// PNG inflate.  Bit-exact with libwebp's decoder (tests compare against Pillow).
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

namespace b200 {

struct WebpInfo { int width = 0, height = 0; bool has_alpha = false, lossless = false, animated = false; };
// container sniff: dimensions and which features the file uses (no pixel work)
bool webp_probe(const uint8_t *data, size_t len, WebpInfo &info, std::string &err);
// Decode a lossy (VP8) still image to planar 8-bit RGB [3][h][w] exactly as libwebp's WebPDecodeRGB would (fancy chroma
// upsampling, fixed-point BT.601); lossless (VP8L) files and the alpha plane of either kind go through vp8l_decode.cpp.  alpha
// (optional) receives the alpha plane [h][w] when some pixel is not opaque (info.has_alpha), else it is left empty; without it a
// file with transparency is refused.  Returns 0 ok, 1 unsupported feature (animation; alpha not asked for), 2 corrupt.
int webp_decode_rgb(const uint8_t *data, size_t len, WebpInfo &info, std::vector<uint8_t> &rgb_planar, std::string &err, std::vector<uint8_t> *alpha = nullptr);
// The same decode from one image's chunk payloads once the container is walked (a still file's, or one animation frame's): vp8 /
// vp8_len the 'VP8 ' payload and alph / alph_len its ALPH payload, or vp8l / vp8l_len a VP8L payload.  info.lossless and
// info.has_alpha say which of them the caller found; the rest of info is filled in.  Returns as webp_decode_rgb.
int webp_decode_chunks(const uint8_t *vp8, size_t vp8_len, const uint8_t *alph, size_t alph_len, const uint8_t *vp8l, size_t vp8l_len, WebpInfo &info,
                       std::vector<uint8_t> &rgb_planar, std::string &err, std::vector<uint8_t> *alpha = nullptr);

} // namespace b200
