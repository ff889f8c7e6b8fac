// png_device.cu -- device orchestration of the lossless PNG path (libcaesium png::lossless -> oxipng::optimize_from_memory,
// caesium-clt's src/compressor.rs:428,436-437): upload the decoded samples, apply the cheap lossless reductions
// (opaque alpha, grey RGB), then for every row-filter strategy of the optimisation preset run K6 (filter) + K7 (match,
// parse) and estimate the DEFLATE size from the token histogram; the winning strategy's tokens come back to the host,
// which Huffman-codes and frames them (png_host.cpp).
#include <cuda_runtime.h>
#include <cub/device/device_scan.cuh>
#include <algorithm>
#include <cstring>
#include "png_device.h"
#include "png_kernels.h"
#include "png_deflate.h"
#include "png_quant.h"
#include "png_zopfli.h"
#include "png_resize.h"
#include "resize_kernels.h"
#include <chrono>
#include <cstdlib>
#include "stream_wait.h"
#include "launch_timer.h"

namespace b200 {

static const int kChunk = 4096;
static const int kBlockTokens = 1 << 16;            // tokens per DEFLATE block (deflate_tokens' default)

// growable buffers: the smallest power of two >= 64 KiB and >= need + need / 4
template <class B> static bool grow(B &buf, size_t need, std::string &err) { return buf.reserve(need, Grow::Pow2Quarter, err); }

PngDevice::PngDevice() = default;
PngDevice::~PngDevice() = default;

PngQuant *PngDevice::quantiser() { if (!quant) quant.reset(new PngQuant()); return quant.get(); }

// oxipng presets (SURVEY.md §3.4-iii): which row-filter strategies each optimisation level tries
std::vector<int> png_level_strategies(int level)
{
    switch (level) {
        case 0: return {PNGF_NONE};
        case 1: return {PNGF_NONE, PNGF_BIGRAMS};
        case 2: return {PNGF_NONE, PNGF_SUB, PNGF_ENTROPY, PNGF_BIGRAMS};
        case 3: case 4: return {PNGF_NONE, PNGF_BIGRAMS, PNGF_BIGENT, PNGF_BRUTE};
        case 5: return {PNGF_NONE, PNGF_BIGRAMS, PNGF_BIGENT, PNGF_BRUTE, PNGF_UP, PNGF_MINSUM};
        default: return {PNGF_NONE, PNGF_BIGRAMS, PNGF_BIGENT, PNGF_BRUTE, PNGF_UP, PNGF_MINSUM, PNGF_AVERAGE, PNGF_PAETH};
    }
}

// estimated DEFLATE payload bits of a token histogram under its own optimal (unlimited) code: sum f * (log2(total/f)) + extra
static double estimate_bits(const uint32_t *h)
{
    static const uint8_t lx[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
    static const uint8_t dx[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
    double tl = 0, td = 0, bits = 0;
    for (int i = 0; i < 286; i++) tl += h[i];
    for (int i = 0; i < 30; i++) td += h[286 + i];
    for (int i = 0; i < 286; i++) if (h[i]) bits += h[i] * (std::log2(tl / h[i]) + (i >= 257 ? lx[i - 257] : 0));
    for (int i = 0; i < 30; i++) if (h[286 + i]) bits += h[286 + i] * (std::log2(td / h[286 + i]) + dx[i]);
    return bits;
}

// One strategy: K6 into `filt` (skipped when the stream is already there), K7 over it.  Trials run the fixed-distance candidates only
// (enough to rank the strategies by their token statistics); the winner's stream then gets the hash candidates as well.
bool PngDevice::run_strategy(int strategy, int h, int rb, int bpp, void *stream_, std::string &err, uint8_t *filt, bool do_filter, bool with_hash)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const size_t n = (size_t)h * (rb + 1);
    if (!filt) filt = d_filt;
    int rc = do_filter ? launch_png_filter(d_raw, filt, h, rb, bpp, strategy, d_tlog, st) : 0;
    if (!rc) rc = launch_png_match(filt, d_best, n, bpp, rb + 1, st);
    if (!rc && with_hash) rc = launch_png_hashmatch(filt, d_best, n, d_hist + 2048, st);
    if (!launch_ok(rc, "png kernels", err)) return false;
    CU(cudaMemsetAsync(d_hist, 0, 316 * 4, st));
    rc = launch_png_parse(d_best, filt, n, kChunk, d_tok, d_counts, d_hist, st);
    if (!launch_ok(rc, "png parse", err)) return false;
    return true;
}

// number of tokens of the compacted stream = last offset + last count (both still on the device)
__global__ void k_png_ntok(const uint32_t *__restrict__ counts, const uint32_t *__restrict__ offsets, size_t nchunks, uint32_t *__restrict__ ntok)
{
    if (blockIdx.x == 0 && threadIdx.x == 0) *ntok = offsets[nchunks - 1] + counts[nchunks - 1];
}

bool PngDevice::ensure_buffers(size_t nraw, size_t nmax, size_t rb, void *stream_, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const size_t nchunks_max = (nmax + kChunk - 1) / kChunk;
    z_cap = nmax + nmax / 32 + ((nmax >> 16) + 2) * 512 + 4096;                 // the zlib payload: Huffman-coded literals cannot exceed ~8.1 bits each
    z_cap = (z_cap + 255) / 256 * 256;
    if (!grow(d_raw, nraw + 64, err) || !grow(d_raw2, nraw + 64, err) ||
        !grow(d_filt, nmax + 64, err) || !grow(d_best, nmax * 4, err) || !grow(d_tok, nmax * 4, err) ||
        !grow(d_out, nmax * 4, err) || !grow(d_counts, nchunks_max * 4 + 4, err) || !grow(d_offsets, nchunks_max * 4 + 4, err) ||
        !grow(d_hist, 316 * 4 * 16, err) || !grow(d_sums, ((nmax + 4095) / 4096) * 16 + 16, err) ||
        !grow(d_sums_in, ((nmax + 4095) / 4096) * 16 + 16, err) ||
        !grow(d_tlog, (rb + 8) * 4, err) || !grow(h_small, 1 << 16, err) ||
        !grow(d_sync, ((nraw / std::max<size_t>(rb, 1) + 31) / 32 + 16) * 4 + 2048 * 4 + 64, err) ||
        !grow(d_dfl, png_deflate_scratch_bytes(nmax, kBlockTokens), err) || !grow(d_z, z_cap + 64, err) ||
        !grow(h_z, z_cap + ((nmax + 4095) / 4096) * 32 + 256, err)) return false;
    size_t tb = 0; cub::DeviceScan::ExclusiveSum((void *)nullptr, tb, d_counts.get(), d_offsets.get(), (int)nchunks_max, st);
    if (!grow(d_temp, tb + 256, err)) return false;
    if (tlog_n < rb + 2) { std::vector<uint32_t> t(rb + 2); png_make_tlog(t.data(), rb + 1); CU(cudaMemcpyAsync(d_tlog, t.data(), (rb + 2) * 4, cudaMemcpyHostToDevice, st)); CU(stream_wait(st)); tlog_n = rb + 2; }
    return true;
}

static uint32_t combine_adler(const unsigned long long *sums, size_t n)
{   // Adler-32 of n bytes from per-4096-byte pieces (S = sum of bytes, T = sum of (len - k) * byte_k): a' = a + S, b' = b + len * a + T  (mod 65521)
    unsigned long long a = 1, b = 0;
    const size_t npieces = (n + 4095) / 4096;
    for (size_t p = 0; p < npieces; p++) {
        const unsigned long long len = std::min<size_t>(4096, n - p * 4096);
        b = (b + len * a + sums[2 * p + 1]) % 65521; a = (a + sums[2 * p]) % 65521;
    }
    return (uint32_t)((b << 16) | a);
}

uint8_t *PngDevice::input_buffer(size_t bytes, size_t &cap, std::string &err)
{
    if (!grow(h_raw, bytes + 4096 + 64, err)) return nullptr;
    cap = h_raw.capacity();
    return h_raw;
}

// K3 of the ch planes of T at `in` (W x H each, one after another) into `out` (NW x NH each)
template <class T> static bool resample_planes(Resampler &rs, const uint8_t *in, int W, int H, uint8_t *out, int NW, int NH, int ch, void *stream, std::string &err)
{
    const T *src[4]; T *dst[4];
    for (int c = 0; c < ch; c++) { src[c] = reinterpret_cast<const T *>(in) + (size_t)c * W * H; dst[c] = reinterpret_cast<T *>(out) + (size_t)c * NW * NH; }
    return rs.run(src, W, H, dst, NW, NH, ch, stream, err);
}

// Expansion, K3 (skipped at the same size: imageops::resize copies) and packing, all enqueued behind the un-filter: d_raw holds the
// source's rows on entry and the resized image's rows on exit.
bool PngDevice::resize_raw(const PngInfo &src, const PngInfo &out, void *stream_, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const PngDecodedType t = png_decoded_type(src);
    const int W = (int)src.width, H = (int)src.height, NW = (int)out.width, NH = (int)out.height, ch = t.channels;
    const size_t bps = (size_t)t.depth / 8;
    if (!grow(d_planes, ch * (size_t)W * H * bps + 64, err)) return false;
    if (!launch_ok(launch_png_expand_planes(d_raw, src, png_palette_lut(src), d_planes, st), "png expand", err)) return false;
    const uint8_t *planes = d_planes;
    if (NW != W || NH != H) {
        if (!grow(d_rplanes, ch * (size_t)NW * NH * bps + 64, err)) return false;
        if (!(t.depth == 16 ? resample_planes<uint16_t>(resampler, d_planes, W, H, d_rplanes, NW, NH, ch, st, err)
                            : resample_planes<uint8_t>(resampler, d_planes, W, H, d_rplanes, NW, NH, ch, st, err))) return false;
        planes = d_rplanes;
    }
    if (!launch_ok(launch_png_pack_planes(planes, ch, t.depth, NW, NH, d_raw, st), "png pack", err)) return false;
    LT_MARK("png_resize");
    return true;
}

// the inputs of the alpha / grey probe: 8-bit samples without tRNS that have colour or alpha to drop
static bool alpha_grey_candidate(const PngInfo &info)
{
    return info.bit_depth == 8 && info.trns.empty() && (info.color_type == 2 || info.color_type == 4 || info.color_type == 6);
}

// nw, nh > 0: the resize runs between the un-filter and the checks' host wait (a corrupt input's resized samples are discarded)
// and info describes the resized image from there on
bool PngDevice::unfilter(PngInfo &info, size_t nfilt, uint32_t stored_adler, void *stream_, std::string &err, uint32_t nw, uint32_t nh, bool probes)
{
    cudaStream_t st = (cudaStream_t)stream_;
    corrupt = false;
    const int h = (int)info.height; const size_t rb = info.row_bytes; const int bpp = info.bpp;
    // Adam7: the seven passes are un-filtered into d_raw2 (pass-packed) and gathered into d_raw; from there on the image is the
    // non-interlaced one and every tail sees full-image rows
    const bool adam7 = info.interlace == 1;
    const uint32_t w = info.width; const int bits = info.bits_per_pixel;      // the source's (a resize rewrites info below)
    Adam7Layout L;
    if (adam7) adam7_layout(w, info.height, bits, L);
    info.interlace = 0;
    const size_t nraw = (size_t)h * rb, nin = adam7 ? L.filt_bytes : (size_t)h * (rb + 1);
    if (nfilt < nin) { err = "IDAT too short"; corrupt = true; return false; }
    size_t ngroups = ((size_t)h + 31) / 32;
    if (adam7) { ngroups = 0; for (const Adam7Pass &P : L.pass) ngroups += (P.h + 31) / 32; }
    const size_t nmax = nin + 64;
    if (!ensure_buffers(nraw, nmax, rb, st, err) || !grow(d_fin, nmax + 64, err)) return false;
    if (adam7 && (!grow(d_raw2, L.raw_bytes + 64, err) || !grow(d_sync, (ngroups + 16) * 4 + 2048 * 4 + 64, err))) return false;
    const bool resize = nw && nh;
    const PngInfo src = resize ? info : PngInfo();
    if (resize) {   // every buffer of the back end for the larger of the two images
        png_resized_info(info, nw, nh);
        if (!ensure_buffers(info.row_bytes * info.height, (info.row_bytes + 1) * info.height + 64, info.row_bytes, st, err)) return false;
    }
    CU(cudaMemcpyAsync(d_fin, h_raw, nin, cudaMemcpyHostToDevice, st)); LT_MARK("h2d");
    int rc = launch_png_adler(d_fin, nin, d_sums_in, st);
    uint32_t *d_un = d_sync, *d_flags = d_hist;
    uint32_t *d_set = reinterpret_cast<uint32_t *>(((uintptr_t)(d_sync + (ngroups + 8)) + 7) & ~(uintptr_t)7);
    if (!rc) rc = adam7 ? launch_png_adam7_unfilter(d_fin, d_raw2, d_raw, L, w, (uint32_t)h, bits, bpp, d_un, st)
                        : launch_png_unfilter(d_fin, d_raw, h, (int)rb, bpp, d_un, st);
    if (!launch_ok(rc, "png unfilter", err)) return false;
    LT_MARK("png_unfilter");
    if (resize && !resize_raw(src, info, st, err)) return false;
    CU(cudaMemsetAsync(d_flags, 0, 16, st));
    const size_t npix = (size_t)info.width * info.height;
    if (probes && alpha_grey_candidate(info) && launch_png_probe(d_raw, npix, info.channels, d_flags, st)) { err = "png probe launch failed"; return false; }
    if (probes && png_palette_candidate(info) && launch_png_colours(d_raw, npix, info.channels, d_set, d_flags, st)) { err = "png palette probe launch failed"; return false; }
    uint32_t *h_flags = reinterpret_cast<uint32_t *>(h_small.get());
    unsigned long long *h_sums_in = reinterpret_cast<unsigned long long *>(h_z.get());
    const size_t npieces_in = (nin + 4095) / 4096;
    CU(cudaMemcpyAsync(h_flags, d_flags, 16, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(h_flags + 4, d_un, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(h_sums_in, d_sums_in, npieces_in * 16, cudaMemcpyDeviceToHost, st));
    CU(stream_wait(st)); LT_MARK("host_wait");
    if (h_flags[5]) { err = "bad filter type"; corrupt = true; return false; }
    if (combine_adler(h_sums_in, nin) != stored_adler) { err = "Adler-32 mismatch"; corrupt = true; return false; }
    return true;
}

bool PngDevice::code_unfiltered(PngInfo &info, int level, void *stream_, std::vector<uint8_t> &zlib_stream, int *chosen, std::string &err)
{
    const uint32_t *h_flags = reinterpret_cast<const uint32_t *>(h_small.get());
    const bool probed = alpha_grey_candidate(info);
    if (png_palette_candidate(info) && h_flags[2] <= 256) {
        // few colours: oxipng's palette reduction (first-appearance order, tRNS layout, bit packing) runs on the host over the
        // reconstructed samples, and the indexed image takes the raw-sample entry point
        std::vector<uint8_t> raw(info.row_bytes * info.height);
        CU(cudaMemcpy(raw.data(), d_raw, raw.size(), cudaMemcpyDeviceToHost));
        if (png_reduce_palette(info, raw)) return compress(info, raw, level, stream_, zlib_stream, chosen, err);
    }
    return reduce_and_code(info, probed, h_flags, level, stream_, zlib_stream, chosen, err);
}

bool PngDevice::fetch_rows(const PngInfo &info, std::vector<uint8_t> &raw, void *stream_, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    raw.resize(info.row_bytes * info.height);
    CU(cudaMemcpyAsync(raw.data(), d_raw, raw.size(), cudaMemcpyDeviceToHost, st));
    CU(stream_wait(st));
    return true;
}

bool PngDevice::compress(PngInfo &info, const std::vector<uint8_t> &raw_in, int level, void *stream_, std::vector<uint8_t> &zlib_stream, int *chosen, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    corrupt = false;
    const int h = (int)info.height; const size_t rb = info.row_bytes;
    const size_t nraw = raw_in.size();
    const size_t nmax = (size_t)h * (rb + 1) + 64;
    size_t cap = 0;
    if (!ensure_buffers(nraw, nmax, rb, st, err) || !input_buffer(nraw, cap, err)) return false;
    memcpy(h_raw, raw_in.data(), nraw);
    CU(cudaMemcpyAsync(d_raw, h_raw, nraw, cudaMemcpyHostToDevice, st));
    uint32_t *h_flags = reinterpret_cast<uint32_t *>(h_small.get());
    const bool probe_ag = alpha_grey_candidate(info);
    if (probe_ag) {
        uint32_t *d_flags = d_hist;
        CU(cudaMemsetAsync(d_flags, 0, 16, st));
        if (launch_png_probe(d_raw, (size_t)info.width * info.height, info.channels, d_flags, st)) { err = "png probe launch failed"; return false; }
        CU(cudaMemcpyAsync(h_flags, d_flags, 16, cudaMemcpyDeviceToHost, st));
        CU(stream_wait(st)); LT_MARK("host_wait");
    }
    return reduce_and_code(info, probe_ag, h_flags, level, stream_, zlib_stream, chosen, err);
}

bool PngDevice::code_quantized(PngInfo &info, int quality, int level, void *stream_, std::vector<uint8_t> &zlib_stream, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    PngQuant *q = quantiser();
    info.plte.clear(); info.trns.clear();
    if (q->exact()) {
        std::vector<uint8_t> raw;
        if (!q->fetch_rgba(raw, st, err)) return false;
        info.color_type = 6; info.bit_depth = 8; info.channels = 4; info.bits_per_pixel = 32; info.bpp = 4; info.row_bytes = (size_t)info.width * 4;
        png_reduce_palette(info, raw);
        return compress(info, raw, level, stream_, zlib_stream, nullptr, err);
    }
    std::vector<uint32_t> pal;
    if (!q->quantize(quality, st, pal, err)) return false;
    const int n = (int)pal.size(), depth = png_index_depth(n);
    info.color_type = 3; info.bit_depth = depth; info.channels = 1; info.bits_per_pixel = depth; info.bpp = 1;
    info.row_bytes = ((size_t)info.width * depth + 7) / 8;
    info.plte.resize((size_t)n * 3);
    int ntrans = 0;
    for (int k = 0; k < n; k++) {
        for (int c = 0; c < 3; c++) info.plte[3 * k + c] = (uint8_t)(pal[k] >> (8 * c));
        if ((pal[k] >> 24) != 255) ntrans = k + 1;
    }
    for (int k = 0; k < ntrans; k++) info.trns.push_back((uint8_t)(pal[k] >> 24));
    const size_t rb = info.row_bytes, nraw = rb * info.height;
    if (!ensure_buffers(nraw, (size_t)info.height * (rb + 1) + 64, rb, st, err) || !q->pack(d_raw, depth, st, err)) return false;
    return reduce_and_code(info, false, nullptr, level, stream_, zlib_stream, nullptr, err);
}

// d_raw holds the reconstructed samples; h_flags the probe results.  Lossless reductions (oxipng reduction::*: opaque alpha, grey
// RGB -- 8-bit samples without tRNS only), then every strategy of the preset, then the winner is DEFLATE-coded on the device.
bool PngDevice::reduce_and_code(PngInfo &info, bool probed, const uint32_t *h_flags, int level, void *stream_, std::vector<uint8_t> &zlib_stream, int *chosen, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    int h = (int)info.height; size_t rb = info.row_bytes; int bpp = info.bpp;
    if (probed) {
        const size_t npix = (size_t)info.width * info.height;
        const bool has_alpha = info.color_type == 4 || info.color_type == 6, is_rgb = info.color_type == 2 || info.color_type == 6;
        const bool drop_alpha = has_alpha && h_flags[0] == 0, to_grey = is_rgb && h_flags[1] == 0;
        if (drop_alpha || to_grey) {
            int mask = 0, ch = info.channels;
            const int ncolor = is_rgb ? 3 : 1;
            for (int c = 0; c < ncolor; c++) if (!to_grey || c == 0) mask |= 1 << c;
            if (has_alpha && !drop_alpha) mask |= 1 << (ch - 1);
            if (launch_png_repack(d_raw, d_raw2, npix, ch, mask, st)) { err = "png repack launch failed"; return false; }
            d_raw.swap(d_raw2);
            const bool grey = to_grey || !is_rgb, alpha = has_alpha && !drop_alpha;
            info.color_type = grey ? (alpha ? 4 : 0) : (alpha ? 6 : 2);
            info.channels = (grey ? 1 : 3) + (alpha ? 1 : 0);
            info.bits_per_pixel = 8 * info.channels; info.bpp = info.channels; info.row_bytes = (size_t)info.width * info.channels;
            rb = info.row_bytes; bpp = info.bpp;
        }
    }
    const size_t n = (size_t)h * (rb + 1);
    const size_t nchunks = (n + kChunk - 1) / kChunk;
    // ---- try every strategy of the preset; keep the one whose token histogram promises the smallest stream
    const std::vector<int> strategies = png_level_strategies(level);
    int best_s = strategies[0]; double best_bits = -1; size_t best_k = 0;
    const size_t fstride = (n + 64 + 255) / 256 * 256;
    if (strategies.size() > 1) {
        // every trial keeps its filtered stream (K6 is not repeated for the winner)
        if (!grow(d_filt_all, fstride * strategies.size() + 64, err)) return false;
        for (size_t k = 0; k < strategies.size(); k++) {
            if (!run_strategy(strategies[k], h, (int)rb, bpp, st, err, d_filt_all + k * fstride, true, false)) return false;
            CU(cudaMemcpyAsync(h_small + 1024 + k * 316 * 4, d_hist, 316 * 4, cudaMemcpyDeviceToHost, st));
        }
        CU(stream_wait(st)); LT_MARK("host_wait");
        for (size_t k = 0; k < strategies.size(); k++) {
            const double bits = estimate_bits(reinterpret_cast<const uint32_t *>(h_small + 1024 + k * 316 * 4));
            if (best_bits < 0 || bits < best_bits) { best_bits = bits; best_s = strategies[k]; best_k = k; }
        }
    }
    if (chosen) *chosen = best_s;
    // ---- the winner, for real: full match search (fixed + hash candidates), tokens compacted, Adler-32 pieces of the filtered
    //      stream, DEFLATE coding -- all on the device
    uint8_t *const wfilt = strategies.size() > 1 ? d_filt_all + best_k * fstride : d_filt;
    if (!run_strategy(best_s, h, (int)rb, bpp, st, err, wfilt, strategies.size() <= 1, true)) return false;
    size_t tb = d_temp.capacity();
    cub::DeviceScan::ExclusiveSum(d_temp, tb, d_counts.get(), d_offsets.get(), (int)nchunks, st); LT_MARK("cub_scan");
    int rc = launch_png_compact(d_tok, d_counts, d_offsets, nchunks, kChunk, d_out, st);
    if (!rc) rc = launch_png_adler(wfilt, n, d_sums, st);
    if (!launch_ok(rc, "png compact/adler", err)) return false;
    unsigned long long *d_total = reinterpret_cast<unsigned long long *>(d_hist + 1024);          // [0] payload bits, [1] tokens
    uint32_t *d_ntok = d_hist + 1032;
    k_png_ntok<<<1, 32, 0, st>>>(d_counts, d_offsets, nchunks, d_ntok);
    const bool host_huffman = [] { const char *e = getenv("B200_PNG_HUFFMAN"); return e && !strcmp(e, "host"); }();
    unsigned long long *h_total = reinterpret_cast<unsigned long long *>(h_small + 64);
    const size_t npieces = (n + 4095) / 4096;
    unsigned long long *h_sums = reinterpret_cast<unsigned long long *>(h_z + z_cap + 64);
    if (!host_huffman) {
        rc = launch_png_deflate(d_out, d_ntok, n, kBlockTokens, d_dfl, reinterpret_cast<uint32_t *>(d_z.get()), z_cap, d_total, st);
        if (!launch_ok(rc, "png deflate", err)) return false;
        CU(cudaMemcpyAsync(h_total, d_total, 16, cudaMemcpyDeviceToHost, st));
        if (zopfli) {   // --zopfli: the optimal parse of the same stream, coded into its own buffer behind the greedy one
            if (!zop) zop.reset(new PngZopfli());
            unsigned long long *d_ztotal = reinterpret_cast<unsigned long long *>(d_hist + 1036);
            uint32_t *d_zntok = d_hist + 1034;
            if (!grow(zop->d_z, z_cap + 64, err) || !zop->tokens(wfilt, n, bpp, (int)rb + 1, d_tok, d_counts, kChunk, d_out, st, err)) return false;
            k_png_ntok<<<1, 32, 0, st>>>(zop->d_segn, zop->d_offsets, PngZopfli::nseg(n), d_zntok);
            rc = launch_png_deflate(d_out, d_zntok, n, kBlockTokens, d_dfl, reinterpret_cast<uint32_t *>(zop->d_z.get()), z_cap, d_ztotal, st);
            if (!launch_ok(rc, "png zopfli deflate", err)) return false;
            CU(cudaMemcpyAsync(h_total + 2, d_ztotal, 16, cudaMemcpyDeviceToHost, st));
        }
        CU(cudaMemcpyAsync(h_sums, d_sums, npieces * 16, cudaMemcpyDeviceToHost, st));
        CU(stream_wait(st)); LT_MARK("host_wait");
        size_t zbytes = (size_t)((h_total[0] + 7) / 8);
        const uint8_t *zsrc = d_z;
        if (zopfli) {   // the smaller payload; the greedy one on a tie
            const size_t zz = (size_t)((h_total[2] + 7) / 8);
            if (zz < zbytes && zz + 8 <= z_cap) { zbytes = zz; zsrc = zop->d_z; }
        }
        if (zbytes + 8 <= z_cap) {
            CU(cudaMemcpyAsync(h_z, zsrc, zbytes, cudaMemcpyDeviceToHost, st)); LT_MARK("d2h");
            CU(stream_wait(st)); LT_MARK("host_wait");
            const uint32_t adler = combine_adler(h_sums, n);
            zlib_stream.resize(zbytes + 4);
            memcpy(zlib_stream.data(), h_z, zbytes);
            zlib_stream[0] = 0x78; zlib_stream[1] = 0xDA;
            zlib_stream[zbytes] = adler >> 24; zlib_stream[zbytes + 1] = adler >> 16; zlib_stream[zbytes + 2] = adler >> 8; zlib_stream[zbytes + 3] = adler;
            last_deflate_ms = 0;
            return true;
        }
        // does not fit the device buffer (cannot happen for Huffman-coded literals; kept as a guard): the host codes the tokens
    } else {
        CU(cudaMemcpyAsync(h_total + 1, d_ntok, 4, cudaMemcpyDeviceToHost, st));
        CU(cudaMemcpyAsync(h_sums, d_sums, npieces * 16, cudaMemcpyDeviceToHost, st));
        CU(stream_wait(st)); LT_MARK("host_wait");
        h_total[1] &= 0xFFFFFFFFull;
    }
    const size_t ntok = (size_t)h_total[1];
    if (!grow(h_tok, (n + 64) * 4 + 64, err)) return false;
    CU(cudaMemcpyAsync(h_tok, d_out, ntok * 4, cudaMemcpyDeviceToHost, st));
    CU(stream_wait(st)); LT_MARK("host_wait");
    const auto td = std::chrono::steady_clock::now();
    deflate_tokens(h_tok, ntok, combine_adler(h_sums, n), zlib_stream);
    last_deflate_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - td).count();
    return true;
}

// LZ77 tokens of a byte plane that sits on the host (the alpha plane of a WebP with transparency: bpp 1, stride = width): K7 with
// its pixel / row candidates and the hash chains, parallel parse, compaction; the tokens come back to the host (vp8l_alpha.cpp codes them).
bool PngDevice::plane_tokens(const uint8_t *plane, size_t n, int stride, void *stream_, std::vector<uint32_t> &tokens, std::string &err)
{
    return lz77_tokens(plane, n, 1, stride, false, stream_, tokens, err);
}

bool PngDevice::lz77_tokens(const uint8_t *plane, size_t n, int bpp, int stride, bool optimal, void *stream_, std::vector<uint32_t> &tokens, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    if (!n || stride < 1) { err = "empty plane"; return false; }
    if (!ensure_buffers(n, n, (size_t)stride, st, err)) return false;
    if (!grow(h_raw, n + 4096 + 64, err) || !grow(h_tok, (n + 64) * 4 + 64, err)) return false;
    memcpy(h_raw, plane, n);
    CU(cudaMemcpyAsync(d_filt, h_raw, n, cudaMemcpyHostToDevice, st));
    const size_t nchunks = (n + kChunk - 1) / kChunk;
    int rc = launch_png_match(d_filt, d_best, n, bpp, stride, st);
    if (!rc) rc = launch_png_hashmatch(d_filt, d_best, n, d_hist + 2048, st);
    if (!launch_ok(rc, "png kernels", err)) return false;
    CU(cudaMemsetAsync(d_hist, 0, 316 * 4, st));
    rc = launch_png_parse(d_best, d_filt, n, kChunk, d_tok, d_counts, d_hist, st);
    if (!launch_ok(rc, "png parse", err)) return false;
    uint32_t *d_ntok = d_hist + 1032;
    if (optimal) {
        if (!zop) zop.reset(new PngZopfli());
        if (!zop->tokens(d_filt, n, bpp, stride, d_tok, d_counts, kChunk, d_out, st, err)) return false;
        k_png_ntok<<<1, 32, 0, st>>>(zop->d_segn, zop->d_offsets, PngZopfli::nseg(n), d_ntok);
    } else {
        size_t tb = d_temp.capacity();
        cub::DeviceScan::ExclusiveSum(d_temp, tb, d_counts.get(), d_offsets.get(), (int)nchunks, st);
        rc = launch_png_compact(d_tok, d_counts, d_offsets, nchunks, kChunk, d_out, st);
        if (!launch_ok(rc, "png compact", err)) return false;
        k_png_ntok<<<1, 32, 0, st>>>(d_counts, d_offsets, nchunks, d_ntok);
    }
    uint32_t *h_n = reinterpret_cast<uint32_t *>(h_small + 64);
    CU(cudaMemcpyAsync(h_n, d_ntok, 4, cudaMemcpyDeviceToHost, st));
    CU(stream_wait(st));
    const size_t ntok = *h_n;
    if (ntok > n) { err = "token count out of range"; return false; }
    CU(cudaMemcpyAsync(h_tok, d_out, ntok * 4, cudaMemcpyDeviceToHost, st));
    CU(stream_wait(st));
    tokens.assign(h_tok.get(), h_tok + ntok);
    return true;
}

// ---- stage entry points (b200_png_filter / b200_png_lz77): plain allocate-run-free, used by the parity tests ----------------
bool png_stage_filter(const uint8_t *raw, int h, int rb, int bpp, int strategy, uint8_t *filtered, std::string &err)
{
    DeviceBuffer<uint8_t> d_raw, d_filt; DeviceBuffer<uint32_t> d_tlog;
    const size_t nraw = (size_t)h * rb, n = (size_t)h * (rb + 1);
    if (!d_raw.reserve(nraw + 64, Grow::Exact, err) || !d_filt.reserve(n + 64, Grow::Exact, err) || !d_tlog.reserve(((size_t)rb + 8) * 4, Grow::Exact, err)) return false;
    std::vector<uint32_t> t(rb + 2); png_make_tlog(t.data(), rb + 1);
    cudaMemcpy(d_tlog, t.data(), t.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(d_raw, raw, nraw, cudaMemcpyHostToDevice);
    if (launch_png_filter(d_raw, d_filt, h, rb, bpp, strategy, d_tlog, nullptr)) { err = "png filter launch failed"; return false; }
    cudaError_t e = cudaMemcpy(filtered, d_filt, n, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) { err = std::string("png filter: ") + cudaGetErrorString(e); return false; }
    return true;
}

bool png_stage_lz77(const uint8_t *filtered, size_t n, int bpp, int stride, std::vector<uint32_t> &tokens, uint32_t *hist, std::string &err)
{
    DeviceBuffer<uint8_t> d_filt, d_temp; DeviceBuffer<uint32_t> d_best, d_tok, d_out, d_counts, d_offsets, d_hist;
    const size_t nchunks = (n + kChunk - 1) / kChunk;
    size_t tb = 0; cub::DeviceScan::ExclusiveSum((void *)nullptr, tb, d_counts.get(), d_offsets.get(), (int)nchunks);
    if (!d_filt.reserve(n + 64, Grow::Exact, err) || !d_best.reserve(n * 4 + 64, Grow::Exact, err) || !d_tok.reserve(n * 4 + 64, Grow::Exact, err) ||
        !d_out.reserve(n * 4 + 64, Grow::Exact, err) || !d_counts.reserve(nchunks * 4 + 4, Grow::Exact, err) || !d_offsets.reserve(nchunks * 4 + 4, Grow::Exact, err) ||
        !d_hist.reserve((320 + 544) * 4, Grow::Exact, err) || !d_temp.reserve(tb + 256, Grow::Exact, err)) return false;
    cudaMemset(d_filt + n, 0, 64);
    cudaMemcpy(d_filt, filtered, n, cudaMemcpyHostToDevice);
    cudaMemset(d_hist, 0, 316 * 4);
    if (launch_png_match(d_filt, d_best, n, bpp, stride, nullptr) || launch_png_hashmatch(d_filt, d_best, n, d_hist + 320, nullptr) || launch_png_parse(d_best, d_filt, n, kChunk, d_tok, d_counts, d_hist, nullptr)) { err = "png lz77 launch failed"; return false; }
    cub::DeviceScan::ExclusiveSum(d_temp, tb, d_counts.get(), d_offsets.get(), (int)nchunks);
    if (launch_png_compact(d_tok, d_counts, d_offsets, nchunks, kChunk, d_out, nullptr)) { err = "png compact launch failed"; return false; }
    uint32_t last[2];
    cudaMemcpy(&last[0], d_offsets + (nchunks - 1), 4, cudaMemcpyDeviceToHost);
    cudaError_t e = cudaMemcpy(&last[1], d_counts + (nchunks - 1), 4, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) { err = std::string("png lz77: ") + cudaGetErrorString(e); return false; }
    tokens.resize((size_t)last[0] + last[1]);
    cudaMemcpy(tokens.data(), d_out, tokens.size() * 4, cudaMemcpyDeviceToHost);
    e = cudaMemcpy(hist, d_hist, 316 * 4, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) { err = std::string("png lz77: ") + cudaGetErrorString(e); return false; }
    return true;
}

} // namespace b200
