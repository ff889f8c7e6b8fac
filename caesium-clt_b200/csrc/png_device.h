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
struct PngZopfli;

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
    // --zopfli (png_force_zopfli with the switch on, decided by the caller): reduce_and_code also codes the winner's filtered stream
    // from the iterated optimal parse (png_zopfli.cu) and keeps the smaller zlib payload, the greedy / lazy one on a tie
    bool zopfli = false;
    std::unique_ptr<PngZopfli> zop;
    double last_deflate_ms = 0;                          // host Huffman/bit-packing time of the last compress() (tracing)
    PngDevice();
    ~PngDevice();

    // The front end of every leg that starts from a PNG's IDAT: the caller inflates the stream into input_buffer() (pinned, `bytes` =
    // png_inflated_size; the buffer has 4096 bytes of slack for the inflate) and hands over its length and the stream's stored
    // Adler-32.  unfilter() uploads it, un-filters it into d_raw (Adam7: passes gathered into full rows), waits for the device once
    // and checks the filter bytes and the Adler-32 (corrupt = true when they fail).  nw, nh > 0: the image is first expanded to the
    // image crate's decoded type and resized to nw x nh (Lanczos3) before that wait, and info is rewritten to the resized image
    // (png_resized_info: no source chunks survive).  probes: code_unfiltered() follows, and its alpha / grey and palette probes are
    // enqueued before the wait.  The caller then runs its own tail over d_raw.
    uint8_t *input_buffer(size_t bytes, size_t &cap, std::string &err);
    bool unfilter(PngInfo &info, size_t nfilt, uint32_t stored_adler, void *stream, std::string &err, uint32_t nw = 0, uint32_t nh = 0, bool probes = false);
    // The lossless back end after unfilter(..., probes = true): the palette reduction when the probe found at most 256 colours,
    // else the alpha / grey reductions, the filter trials, LZ77 and DEFLATE over d_raw.
    bool code_unfiltered(PngInfo &info, int level, void *stream, std::vector<uint8_t> &zlib_stream, int *chosen_strategy, std::string &err);
    // the rows in d_raw (info's image) back to the host
    bool fetch_rows(const PngInfo &info, std::vector<uint8_t> &raw, void *stream, std::string &err);
    // The lossy leg's back end over whatever quantiser() holds: palette + dithered indices at `quality`, packed into d_raw as an
    // indexed image (info becomes colour type 3 with PLTE / tRNS), then the lossless leg's filter trials, LZ77 and DEFLATE.  An
    // image with at most 256 distinct values is not quantised: it takes the lossless leg's exact palette reduction.
    bool code_quantized(PngInfo &info, int quality, int level, void *stream, std::vector<uint8_t> &zlib_stream, std::string &err);
    PngQuant *quantiser();
    std::unique_ptr<PngQuant> quant;
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
    // the same over a filtered stream with filter distance bpp; optimal: the --zopfli parse instead of the greedy / lazy one
    bool lz77_tokens(const uint8_t *s, size_t n, int bpp, int stride, bool optimal, void *stream, std::vector<uint32_t> &tokens, std::string &err);
    DeviceBuffer<uint8_t> d_filt_all;                   // the trials' filtered streams, one after another
    // the resize: source planes, resized planes, and K3's tables and intermediate
    DeviceBuffer<uint8_t> d_planes, d_rplanes;
    Resampler resampler{Grow::Pow2Quarter};
};

// allocate-run-free stage helpers behind b200_png_filter / b200_png_lz77 (current device)
bool png_stage_filter(const uint8_t *raw, int h, int rb, int bpp, int strategy, uint8_t *filtered, std::string &err);
bool png_stage_lz77(const uint8_t *filtered, size_t n, int bpp, int stride, std::vector<uint32_t> &tokens, uint32_t *hist, std::string &err);

} // namespace b200
