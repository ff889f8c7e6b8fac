// png_kernels.h -- launchers for K6 (PNG row-filter selection) and K7 (LZ77 match finding), SURVEY.md §8a row a8:
// the device work of libcaesium png::lossless -> oxipng (caesium-clt's src/compressor.rs:428,436-437).
#pragma once
#include <cstdint>
#include <cstddef>
#include "png_adam7_core.h"

namespace b200 {

// Row-filter strategies (oxipng RowFilter): the five PNG filters plus the per-row heuristics.
enum PngStrategy { PNGF_NONE = 0, PNGF_SUB = 1, PNGF_UP = 2, PNGF_AVERAGE = 3, PNGF_PAETH = 4,
                   PNGF_MINSUM = 5, PNGF_ENTROPY = 6, PNGF_BIGRAMS = 7, PNGF_BIGENT = 8, PNGF_BRUTE = 9 };

// tlog[c] = round(c * log2(c) * 1024), c = 0..n (shared by the product and the oracle so scores are identical integers)
void png_make_tlog(uint32_t *tlog, size_t n);

// K6: raw [h][rb] -> filtered [h][rb + 1] (filter byte first) using `strategy`; d_tlog has rb + 2 entries.
int launch_png_filter(const uint8_t *d_raw, uint8_t *d_filt, int h, int rb, int bpp, int strategy, const uint32_t *d_tlog, void *stream);
// K7 phase 1: best (length << 16 | distance) per position of the filtered stream (0 = no match of length >= 3).
int launch_png_match(const uint8_t *d_filt, uint32_t *d_best, size_t n, int bpp, int stride, void *stream);
// K7 phase 1b: hash-chain candidates at arbitrary distances (nearest 4 earlier positions with the same 3-byte hash inside a
// 16,384-position segment) improve d_best where they are strictly longer AND long enough to pay for their distance code given
// how cheap the stream's literals are (order-0 entropy of the stream, measured first)
int launch_png_hashmatch(const uint8_t *d_filt, uint32_t *d_best, size_t n, uint32_t *d_work /*544 words: byte histogram + cost tables*/, void *stream);
// K7 phase 2: greedy/lazy parse per chunk of `chunk` positions into tokens (chunk-local slots) + per-chunk counts,
// plus the litlen/dist symbol histogram (316 counters) used to estimate the DEFLATE size of the strategy.
int launch_png_parse(const uint32_t *d_best, const uint8_t *d_filt, size_t n, int chunk, uint32_t *d_tokens, uint32_t *d_counts, uint32_t *d_hist, void *stream);
// compact chunk-local token slots into one stream given the exclusive prefix sum of the counts
int launch_png_compact(const uint32_t *d_tokens, const uint32_t *d_counts, const uint32_t *d_offsets, size_t nchunks, int chunk, uint32_t *d_out, void *stream);
// Adler-32 partial sums per 4096-byte piece: sums[2*i] = sum of bytes, sums[2*i+1] = sum of (len - k) * byte_k
int launch_png_adler(const uint8_t *d_filt, size_t n, unsigned long long *d_sums, void *stream);
// alpha / grey reduction probes: flags[0] |= 1 if some alpha != 255 (8-bit RGBA / GA), flags[1] |= 1 if some pixel has r != g or g != b
int launch_png_probe(const uint8_t *d_raw, size_t npixels, int channels, uint32_t *d_flags, void *stream);
// wavefront un-filtering: filtered [h][rb + 1] -> raw [h][rb]; d_sync[1] != 0 afterwards = a row had a filter type > 4
int launch_png_unfilter(const uint8_t *d_filt, uint8_t *d_raw, int h, int rb, int bpp, uint32_t *d_sync /*2 + ceil(h/32) words*/, void *stream);
// Adam7: the seven passes of the inflated stream d_filt (layout L of a w x h image, bits per pixel, filter distance bpp) un-filtered in
// one wavefront launch into d_packed (L.raw_bytes), then the full rows gathered into d_raw [h][row_bytes]; d_sync[1] != 0 afterwards =
// a row had a filter type > 4.  d_sync: 2 + sum over the passes of ceil(pass height / 32) words.
int launch_png_adam7_unfilter(const uint8_t *d_filt, uint8_t *d_packed, uint8_t *d_raw, const Adam7Layout &L, uint32_t w, uint32_t h, int bits, int bpp,
                              uint32_t *d_sync, void *stream);
// palette probe (8-bit RGB / RGBA): flags[2] = number of distinct pixel values, saturating above 256
int launch_png_colours(const uint8_t *d_raw, size_t npixels, int channels, uint32_t *d_set /*2048 words*/, uint32_t *d_flags, void *stream);
// repack pixels keeping `keep_mask` channels (bit c = keep channel c) : 8-bit samples only
int launch_png_repack(const uint8_t *d_raw, uint8_t *d_out, size_t npixels, int channels, int keep_mask, void *stream);

} // namespace b200
