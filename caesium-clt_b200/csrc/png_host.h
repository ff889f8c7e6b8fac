// png_host.h -- host half of the lossless PNG path (libcaesium png::lossless -> oxipng, reached with png.optimize == true,
// caesium-clt's src/compressor.rs:428,436-437): container parsing, inflate + unfilter of the source IDAT, and the
// DEFLATE bit-packer (dynamic Huffman blocks) + zlib/PNG framing around the LZ77 tokens the device produces.  Row-filter
// selection (K6) and LZ77 match finding (K7) are CUDA kernels (png_kernels.cu); entropy coding stays here.
#pragma once
#include <cstdint>
#include <cstddef>
#include <string>
#include <vector>

namespace b200 {

struct PngInfo {
    uint32_t width = 0, height = 0;
    int bit_depth = 8, color_type = 0, interlace = 0;
    int channels = 1, bits_per_pixel = 8, bpp = 1;        // bpp = filter distance in bytes (>= 1)
    size_t row_bytes = 0;                                  // without the filter byte
    std::vector<uint8_t> plte, trns;                       // chunk payloads
    std::vector<uint8_t> kept_before_idat, kept_after_idat;   // ancillary chunks carried over, serialised (len|type|data|crc)
};

// Whether Adam7-interlaced files are accepted (b200_set_png_interlaced, else B200_PNG_INTERLACED=gpu; off by default).  The switch
// belongs to the C ABI (api.cpp); png_parse_chunks asks it, so every leg that parses a PNG follows it.
bool png_interlaced();

// Container parse only (chunk CRCs checked, IHDR validated, PLTE / tRNS / kept chunks collected): where the zlib stream lies.
// Interlace method 1 (Adam7) is refused with "interlaced PNG is not supported on the GPU path" unless png_interlaced(); any other
// non-zero method always is.
struct PngIdat { const uint8_t *p = nullptr; size_t n = 0; std::vector<uint8_t> joined; };      // p points into the file (one IDAT) or into joined
bool png_parse_chunks(const uint8_t *data, size_t len, bool keep_all_metadata, PngInfo &info, PngIdat &idat, std::string &err);
// Bytes of the inflated image data: height * (row_bytes + 1), or for an Adam7 file the rows of its seven passes (png_adam7_core.h).
size_t png_inflated_size(const PngInfo &info);
// Container parse + inflate only: filt = png_inflated_size(info) bytes, every row led by its filter-type byte (the lossless path
// un-filters on the device, png_kernels.cu k_png_unfilter / k_png_adam7_unfilter).
bool png_parse_inflate(const uint8_t *data, size_t len, bool keep_all_metadata, PngInfo &info, std::vector<uint8_t> &filt, std::string &err);
// Parse + inflate + unfilter (+ de-interlace).  raw = height * row_bytes bytes of packed samples (no filter bytes); info.interlace
// is 0 afterwards.
bool png_decode(const uint8_t *data, size_t len, bool keep_all_metadata, PngInfo &info, std::vector<uint8_t> &raw, std::string &err);

// oxipng reduction::palette (lossless): an 8-bit RGB / RGBA image with at most 256 distinct pixel values becomes an 8-bit
// indexed image (PLTE, plus tRNS when some entry is not opaque; entries with alpha < 255 first so that tRNS stays short), packed
// to 4 / 2 / 1 bits per index when the palette has at most 16 / 4 / 2 entries (oxipng reduction::bit_depth).
// Grey images (r == g == b everywhere) are left alone -- the grey / opaque-alpha reductions that follow serve them better --
// and so are files whose kept chunks depend on the colour type (sBIT, bKGD, hIST) or carry animation frames (acTL).
// Returns true when info / raw were rewritten.
bool png_reduce_palette(PngInfo &info, std::vector<uint8_t> &raw);
// the header-level conditions of that reduction (8-bit RGB / RGBA, no tRNS / PLTE, no colour-type dependent kept chunks)
bool png_palette_candidate(const PngInfo &info);

// RFC 1951 inflate of a complete zlib stream (RFC 1950 wrapper checked, Adler-32 verified)
bool zlib_inflate(const uint8_t *in, size_t n, std::vector<uint8_t> &out, size_t size_hint, std::string &err);

// The same into a caller's buffer of cap >= size_limit + 4096 bytes (pinned staging memory): no allocation, no zero fill.  The
// stream's Adler-32 is NOT verified here -- *stored_adler receives it and the caller checks it where the bytes end up (the
// lossless PNG path sums them on the device).
bool zlib_inflate_to(const uint8_t *in, size_t n, uint8_t *buf, size_t cap, size_t size_limit, size_t *out_len, uint32_t *stored_adler, std::string &err);

// LZ77 token: literal = byte value (0..255); match = 0x80000000 | (length - 3) << 16 | (distance - 1)
static inline uint32_t tok_match(int len, int dist) { return 0x80000000u | ((uint32_t)(len - 3) << 16) | (uint32_t)(dist - 1); }

// DEFLATE-encode a token stream (dynamic Huffman, one block per `block_tokens` tokens) into a zlib stream.
// adler = Adler-32 of the uncompressed bytes the tokens expand to.
void deflate_tokens(const uint32_t *tokens, size_t ntokens, uint32_t adler, std::vector<uint8_t> &out, size_t block_tokens = 1 << 16);

// Assemble the PNG file around one zlib stream.
void png_write(const PngInfo &info, const std::vector<uint8_t> &zlib_stream, std::vector<uint8_t> &out);

uint32_t crc32_update(uint32_t crc, const uint8_t *p, size_t n);
uint32_t adler32(const uint8_t *p, size_t n);

} // namespace b200
