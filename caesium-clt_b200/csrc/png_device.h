// png_device.h -- per-worker device state of the lossless PNG path (see png_device.cu).
#pragma once
#include <cstdint>
#include <cstddef>
#include <cmath>
#include <memory>
#include <string>
#include <vector>
#include "dev_buffer.h"
#include "png_host.h"
#include "resize_kernels.h"

namespace b200 {

struct PngQuant;

// strategies tried per oxipng optimisation level 0..6 (PngStrategy values)
std::vector<int> png_level_strategies(int level);

struct PngDevice {
    DeviceBuffer<uint8_t> d_raw, d_raw2, d_filt, d_temp;
    DeviceBuffer<uint32_t> d_best, d_tok, d_out, d_counts, d_offsets, d_hist, d_tlog;
    DeviceBuffer<unsigned long long> d_sums;
    PinnedBuffer<uint8_t> h_small, h_raw;
    PinnedBuffer<uint32_t> h_tok;
    DeviceBuffer<uint8_t> d_fin, d_dfl, d_z; PinnedBuffer<uint8_t> h_z; DeviceBuffer<uint32_t> d_sync; DeviceBuffer<unsigned long long> d_sums_in;
    size_t z_cap = 0;
    bool corrupt = false;                                // the last failure was the INPUT's fault (bad filter byte, Adler-32 mismatch)
    size_t tlog_n = 0;
    double last_deflate_ms = 0;                          // host Huffman/bit-packing time of the last compress() (tracing)
    PngDevice();
    ~PngDevice();

    // The lossless path: the caller inflates the IDAT stream into input_buffer() (pinned, `bytes` = height * (row_bytes + 1); the
    // buffer has 4096 bytes of slack for the inflate) and hands over its length and the stream's stored Adler-32; un-filtering,
    // checksum verification, reductions, K6 / K7 and the DEFLATE coding run on the device.
    uint8_t *input_buffer(size_t bytes, size_t &cap, std::string &err);
    // nw, nh > 0: the image is first expanded to the image crate's decoded type and resized to nw x nh (Lanczos3), and info is rewritten
    // to the resized image (png_resized_info: no source chunks survive); the back end then codes that image.
    bool compress_filtered(PngInfo &info, size_t nfilt, uint32_t stored_adler, int level, void *stream, std::vector<uint8_t> &zlib_stream, int *chosen_strategy, std::string &err,
                           uint32_t nw = 0, uint32_t nh = 0);
    // The lossy leg's front end: the same upload, un-filter and checks as compress_filtered, then the samples are expanded to RGBA8
    // and the quantiser's histogram is built (quantiser(); independent of the quality, so compress_to_size does it once).  nw, nh > 0:
    // resized first, as in compress_filtered, and info describes the resized image afterwards.
    bool load_filtered_lossy(PngInfo &info, size_t nfilt, uint32_t stored_adler, void *stream, std::string &err, uint32_t nw = 0, uint32_t nh = 0);
    // The resize alone (b200_png_resize_samples): the same upload, un-filter, checks and resize, then the rows of the resized image
    // (info rewritten) come back to the host.
    bool resize_filtered(PngInfo &info, size_t nfilt, uint32_t stored_adler, uint32_t nw, uint32_t nh, void *stream, std::vector<uint8_t> &raw, std::string &err);
    // The lossy leg's back end over whatever quantiser() holds: palette + dithered indices at `quality`, packed into d_raw as an
    // indexed image (info becomes colour type 3 with PLTE / tRNS), then the lossless leg's filter trials, LZ77 and DEFLATE.  An
    // image with at most 256 distinct values is not quantised: it takes the lossless leg's exact palette reduction.
    bool code_quantized(PngInfo &info, int quality, int level, void *stream, std::vector<uint8_t> &zlib_stream, std::string &err);
    PngQuant *quantiser();
    std::unique_ptr<PngQuant> quant;
    enum class Tail { Code, Quantise, Samples };       // what follows the checks: the lossless back end, the quantiser, nothing
    bool from_filtered(PngInfo &info, size_t nfilt, uint32_t stored_adler, int level, void *stream, std::vector<uint8_t> &zlib_stream, int *chosen_strategy, std::string &err,
                       Tail tail, uint32_t nw, uint32_t nh);
    // d_raw (the source's un-filtered rows, `src`) -> expansion -> K3 -> packed rows of `out` (png_resized_info) in d_raw
    bool resize_raw(const PngInfo &src, const PngInfo &out, void *stream, std::string &err);
    bool ensure_buffers(size_t nraw, size_t nmax, size_t rb, void *stream, std::string &err);
    bool reduce_and_code(PngInfo &info, bool probed, const uint32_t *h_flags, int level, void *stream, std::vector<uint8_t> &zlib_stream, int *chosen_strategy, std::string &err);
    // info/raw from png_decode; may rewrite info (colour-type reductions).  Produces the zlib stream of the re-filtered image.
    bool compress(PngInfo &info, const std::vector<uint8_t> &raw, int level, void *stream, std::vector<uint8_t> &zlib_stream, int *chosen_strategy, std::string &err);
    // filter + match + parse of d_raw with one strategy (results in d_filt / d_tok / d_counts / d_hist)
    bool run_strategy(int strategy, int h, int rb, int bpp, void *stream, std::string &err, uint8_t *filt = nullptr, bool do_filter = true, bool with_hash = true);
    // K7 over a byte plane on the host (bpp 1, stride = width) -> compacted LZ77 tokens on the host
    bool plane_tokens(const uint8_t *plane, size_t n, int stride, void *stream, std::vector<uint32_t> &tokens, std::string &err);
    DeviceBuffer<uint8_t> d_filt_all;                   // the trials' filtered streams, one after another
    // the resize: source planes, resized planes, and K3's tables and intermediate
    DeviceBuffer<uint8_t> d_planes, d_rplanes;
    Resampler resampler{Grow::Pow2Quarter};
};

// allocate-run-free stage helpers behind b200_png_filter / b200_png_lz77 (current device)
bool png_stage_filter(const uint8_t *raw, int h, int rb, int bpp, int strategy, uint8_t *filtered, std::string &err);
bool png_stage_lz77(const uint8_t *filtered, size_t n, int bpp, int stride, std::vector<uint32_t> &tokens, uint32_t *hist, std::string &err);

} // namespace b200
