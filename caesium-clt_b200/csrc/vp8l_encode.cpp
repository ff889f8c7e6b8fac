// vp8l_encode.cpp -- see vp8l_device.h.  The host side of the lossless WebP (VP8L) encoder: it runs the analysis kernels, picks the
// colour-cache size from their histograms, builds the five prefix codes (dfl_core.h, limit 15), writes the header, the transforms and
// the code descriptions (vp8l_writer.h, shared with the ALPH coder), and frames what the emission kernel wrote.  Every loop over
// pixels runs on the device; the host walks tiles (the predictor sub-image) and alphabets only.
#include <cuda_runtime.h>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include "vp8l_device.h"
#include "vp8l_kernels.h"
#include "vp8l_palette_core.h"
#include "vp8l_writer.h"
#include "stream_wait.h"
#include "launch_timer.h"

namespace b200 {

// the smallest power of two >= 64 KiB and >= need
template <class B> static bool grow(B &buf, size_t need, std::string &err) { return buf.reserve(need, Grow::Pow2, err); }

namespace {

// the per-pixel buffers of an n-pixel image carved out of one arena (nullptr base: just the size)
size_t carve(uint8_t *base, size_t n, int nchunks, int tiles, Vp8lBuffers &B)
{
    size_t off = 0;
    auto take = [&](size_t bytes) { uint8_t *q = base ? base + off : nullptr; off += (bytes + 255) / 256 * 256; return q; };
    B.planes = take(4 * n);
    B.argb = (uint32_t *)take(4 * n); B.res = (uint32_t *)take(4 * n); B.best = (uint32_t *)take(4 * n);
    B.modes = take((size_t)tiles);
    B.cache_tab = (int *)take(4 * vp8l_cache_table_ints(nchunks));
    B.hits = take((size_t)(VP8L_NCACHE - 1) * n);
    B.tok = (uint2 *)take(8 * n); B.cnt = (uint32_t *)take(4 * (size_t)nchunks);
    B.hist = (uint32_t *)take(sizeof(uint32_t) * VP8L_NCACHE * VP8L_HIST);
    B.flags = (uint32_t *)take(4);
    B.codes = (Vp8lCodes *)take(sizeof(Vp8lCodes));
    B.thread_off = (uint32_t *)take(4 * 256 * (size_t)nchunks);
    B.chunk_bits = (unsigned long long *)take(8 * (size_t)nchunks); B.chunk_start = (unsigned long long *)take(8 * (size_t)nchunks);
    B.total = (unsigned long long *)take(8);
    B.pal_set = (unsigned long long *)take(sizeof(unsigned long long) * VP8L_PAL_SET);
    B.pal_info = (uint32_t *)take(4 * VP8L_PAL_INFO);
    B.words = nullptr;
    return off;
}

Vp8lHuffScratch &scratch() { static thread_local Vp8lHuffScratch S; return S; }
void code_of(const std::vector<uint32_t> &freq, PrefixCode &pc, Vp8lHuffScratch &S) { vp8l_make_code(freq, pc, S); }
PrefixCode zero_code(int n) { PrefixCode pc; pc.len.assign(n, 0); pc.code.assign(n, 0); pc.used = 0; return pc; }

// where the palette info lies in h_small: after histograms | flags | total | modes
size_t small_pal_offset(int tiles) { return sizeof(uint32_t) * VP8L_NCACHE * VP8L_HIST + 16 + ((size_t)tiles + 15) / 16 * 16; }

// event times of the palette kernels (collect + sort, pack) of a traced call
struct PaletteTimes {
    cudaStream_t st; bool on; cudaEvent_t ev[4] = {}; bool rec[4] = {};
    PaletteTimes(cudaStream_t s, bool o) : st(s), on(o) { if (on) for (auto &e : ev) if (cudaEventCreate(&e) != cudaSuccess) on = false; }
    ~PaletteTimes() { for (auto &e : ev) if (e) cudaEventDestroy(e); }
    void mark(int k) { if (on) rec[k] = cudaEventRecord(ev[k], st) == cudaSuccess; }
    double ms()    // after the stream has been waited for
    {
        double t = 0; float m;
        for (int k = 0; k < 4 && on; k += 2) if (rec[k] && rec[k + 1] && cudaEventElapsedTime(&m, ev[k], ev[k + 1]) == cudaSuccess) t += m;
        return t;
    }
};

} // namespace

bool Vp8lDevice::reserve(int w, int h, uint32_t *&argb, uint32_t *&flags, std::string &err)
{
    if (w < 1 || h < 1 || w > 16384 || h > 16384) { err = "VP8L dimensions out of range"; return false; }
    const size_t n = (size_t)w * h;
    const int nchunks = (int)((n + VP8L_CHUNK - 1) / VP8L_CHUNK);
    const int tiles = ((w + VP8L_TILE - 1) >> VP8L_TILE_BITS) * ((h + VP8L_TILE - 1) >> VP8L_TILE_BITS);
    const size_t arena = carve(nullptr, n, nchunks, tiles, B);
    const size_t small = small_pal_offset(tiles) + 4 * VP8L_PAL_INFO;
    if (!grow(d_arena, arena, err) || !grow(h_small, small, err) || !grow(h_codes, sizeof(Vp8lCodes), err)) return false;
    carve(d_arena, n, nchunks, tiles, B);
    argb = B.argb; flags = B.flags;
    return true;
}

bool Vp8lDevice::encode(const uint8_t *rgb, const uint8_t *alpha, int w, int h, void *stream_, std::vector<uint8_t> &out, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    uint32_t *argb, *flags;
    if (!reserve(w, h, argb, flags, err)) return false;
    const size_t n = (size_t)w * h;
    if (!grow(h_in, 4 * n, err)) return false;
    memcpy(h_in, rgb, 3 * n);
    if (alpha) memcpy(h_in + 3 * n, alpha, n);
    CU(cudaMemcpyAsync(B.planes, h_in, (alpha ? 4 : 3) * n, cudaMemcpyHostToDevice, st));
    return encode_planes(B.planes, B.planes + n, B.planes + 2 * n, alpha ? B.planes + 3 * n : nullptr, w, h, stream_, out, err);
}

bool Vp8lDevice::encode_planes(const uint8_t *r, const uint8_t *g, const uint8_t *b, const uint8_t *a, int w, int h, void *stream, std::vector<uint8_t> &out, std::string &err)
{
    uint32_t *argb, *flags;
    if (!reserve(w, h, argb, flags, err)) return false;
    if (!launch_ok(launch_vp8l_pack(r, g, b, a, B, w, h, stream), "vp8l kernels", err)) return false;
    return encode_packed(w, h, stream, out, err);
}

// ---- analysis: everything that decides the bitstream, for every cache candidate at once.  With the palette switch on, the colours
// are collected first; an image of at most VP8L_PAL_MAX colours is then also coded through the colour-indexing transform, and the
// smaller file is kept (the one without the palette on a tie).
bool Vp8lDevice::encode_packed(int w, int h, void *stream_, std::vector<uint8_t> &out, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const int tiles_x = (w + VP8L_TILE - 1) >> VP8L_TILE_BITS, tiles_y = (h + VP8L_TILE - 1) >> VP8L_TILE_BITS, tiles = tiles_x * tiles_y;
    const size_t hist_bytes = sizeof(uint32_t) * VP8L_NCACHE * VP8L_HIST;
    const bool palette = webp_palette();
    PaletteTimes pt(st, palette && trace_level() >= 2);
    uint32_t *h_hist = (uint32_t *)h_small.get(), *h_flags = (uint32_t *)(h_small + hist_bytes);
    uint8_t *h_modes = h_small + hist_bytes + 16;
    const uint32_t *h_pal = (const uint32_t *)(h_small + small_pal_offset(tiles));
    last_palette = -1; last_palette_kept = false; last_bytes[0] = last_bytes[1] = 0;
    int rc = 0;
    if (palette) {
        pt.mark(0);
        if (!launch_ok(launch_vp8l_palette(B, w, h, st), "vp8l palette kernels", err)) return false;
        pt.mark(1);
        CU(cudaMemcpyAsync((void *)h_pal, B.pal_info, 4 * VP8L_PAL_INFO, cudaMemcpyDeviceToHost, st));
    }
    rc = launch_vp8l_analyse(B, w, h, st);
    if (!launch_ok(rc, "vp8l kernels", err)) return false;
    CU(cudaMemcpyAsync(h_hist, B.hist, hist_bytes, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(h_flags, B.flags, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(h_modes, B.modes, (size_t)tiles, cudaMemcpyDeviceToHost, st));
    const auto t0 = std::chrono::steady_clock::now();
    CU(stream_wait(st));
    const auto t1 = std::chrono::steady_clock::now();
    last_analyse_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
    last_d2h_bytes = hist_bytes + 4 + (size_t)tiles + (palette ? 4 * VP8L_PAL_INFO : 0);
    const uint32_t alpha_used = *h_flags & 1u;
    if (palette && !h_pal[1]) last_palette = (int)h_pal[0];
    const std::vector<uint32_t> pal(h_pal + 2, h_pal + 2 + (last_palette > 0 ? last_palette : 0));
    Vp8lHuffScratch &S = scratch();
    // ---- header, transforms, predictor sub-image
    std::vector<uint8_t> hdr;
    hdr.reserve(4096 + (size_t)tiles);
    BitsLsb bw(hdr);
    bw.put(0x2f, 8); bw.put((uint32_t)w - 1, 14); bw.put((uint32_t)h - 1, 14); bw.put(alpha_used, 1); bw.put(0, 3);
    bw.put(1, 1); bw.put(2, 2);                                             // subtract-green
    bw.put(1, 1); bw.put(0, 2); bw.put(VP8L_TILE_BITS - 2, 3);              // predictor, 16x16 tiles
    {   // the mode image: an entropy-coded image without a cache, the mode in the green channel, literals only
        std::vector<uint32_t> mf(280, 0);
        for (int t = 0; t < tiles; t++) mf[h_modes[t]]++;
        PrefixCode mc; code_of(mf, mc, S);
        const PrefixCode z256 = zero_code(256), z40 = zero_code(VP8L_NDIST);
        bw.put(0, 1);
        vp8l_write_code(bw, mc, S); vp8l_write_code(bw, z256, S); vp8l_write_code(bw, z256, S); vp8l_write_code(bw, z256, S); vp8l_write_code(bw, z40, S);
        for (int t = 0; t < tiles; t++) vp8l_put_sym(bw, mc, h_modes[t]);
    }
    bw.put(0, 1);                                                           // no further transform
    if (!code_image(w, h, bw, (size_t)-1, out, last_bytes[0], st, err)) return false;
    if (last_palette > 0) {
        // ---- the palette variant: the packed index image replaces the residuals, and the colour-indexing transform is the only one
        const int count = last_palette, xbits = vp8l_pal_xbits(count), wp = vp8l_pal_width(w, xbits);
        pt.mark(2);
        if (!launch_ok(launch_vp8l_palette_pack(B, w, h, count, st), "vp8l palette kernels", err)) return false;
        pt.mark(3);
        if (!launch_ok(launch_vp8l_analyse_res(B, wp, h, st), "vp8l kernels", err)) return false;
        CU(cudaMemcpyAsync(h_hist, B.hist, hist_bytes, cudaMemcpyDeviceToHost, st));
        CU(stream_wait(st));
        last_d2h_bytes += hist_bytes;
        std::vector<uint8_t> phdr;
        phdr.reserve(4096);
        BitsLsb pw(phdr);
        pw.put(0x2f, 8); pw.put((uint32_t)w - 1, 14); pw.put((uint32_t)h - 1, 14); pw.put(alpha_used, 1); pw.put(0, 3);
        pw.put(1, 1); pw.put(3, 2); pw.put((uint32_t)count - 1, 8);        // colour indexing
        {   // the palette image: count x 1, entropy-coded without a cache, entries as deltas, literals only
            std::vector<uint32_t> fg(280, 0), fr(256, 0), fb(256, 0), fa(256, 0);
            for (int i = 0; i < count; i++) {
                const uint32_t d = vp8l_pal_delta(pal.data(), i);
                fg[(d >> 8) & 0xFF]++; fr[(d >> 16) & 0xFF]++; fb[d & 0xFF]++; fa[d >> 24]++;
            }
            PrefixCode cg, cr, cb, ca; code_of(fg, cg, S); code_of(fr, cr, S); code_of(fb, cb, S); code_of(fa, ca, S);
            pw.put(0, 1);
            vp8l_write_code(pw, cg, S); vp8l_write_code(pw, cr, S); vp8l_write_code(pw, cb, S); vp8l_write_code(pw, ca, S); vp8l_write_code(pw, zero_code(VP8L_NDIST), S);
            for (int i = 0; i < count; i++) {
                const uint32_t d = vp8l_pal_delta(pal.data(), i);
                vp8l_put_sym(pw, cg, (d >> 8) & 0xFF); vp8l_put_sym(pw, cr, (d >> 16) & 0xFF); vp8l_put_sym(pw, cb, d & 0xFF); vp8l_put_sym(pw, ca, d >> 24);
            }
        }
        pw.put(0, 1);                                                       // no further transform
        std::vector<uint8_t> alt;
        if (!code_image(wp, h, pw, out.size(), alt, last_bytes[1], st, err)) return false;
        if (!alt.empty()) { out.swap(alt); last_palette_kept = true; }
    }
    last_palette_ms = pt.ms();
    last_code_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count();
    return true;
}

// ---- the rest of one variant after its analysis over cw x h (histograms in h_small): cache size and codes, the header's tail
bool Vp8lDevice::code_image(int cw, int h, BitsLsb &bw, size_t below, std::vector<uint8_t> &out, size_t &file_bytes, void *stream_, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const uint32_t *h_hist = (const uint32_t *)h_small.get();
    unsigned long long *h_total = (unsigned long long *)(h_small + sizeof(uint32_t) * VP8L_NCACHE * VP8L_HIST + 8);
    // ---- cache size and codes
    const int cand = vp8l_choose_cache(h_hist), bits = vp8l_cache_bits(cand);
    last_cache_bits = bits;
    const uint32_t *hc = h_hist + (size_t)cand * VP8L_HIST;
    Vp8lHuffScratch &S = scratch();
    PrefixCode pc[5];
    const int base[5] = {0, VP8L_HIST_RED, VP8L_HIST_BLUE, VP8L_HIST_ALPHA, VP8L_HIST_DIST};
    const int size[5] = {256 + 24 + (bits ? 1 << bits : 0), 256, 256, 256, VP8L_NDIST};
    for (int k = 0; k < 5; k++) code_of(std::vector<uint32_t>(hc + base[k], hc + base[k] + size[k]), pc[k], S);
    // ---- code descriptions
    if (bits) { bw.put(1, 1); bw.put((uint32_t)bits, 4); } else bw.put(0, 1);
    bw.put(0, 1);                                                           // no meta prefix image
    for (int k = 0; k < 5; k++) vp8l_write_code(bw, pc[k], S);
    const unsigned long long bit_base = bw.bits();
    bw.flush();
    const std::vector<uint8_t> &hdr = bw.o;
    // ---- the codes go up, the tokens are sized and emitted
    Vp8lCodes *C = (Vp8lCodes *)h_codes.get();
    memset(C, 0, sizeof(Vp8lCodes));
    for (int k = 0; k < 5; k++)
        if (pc[k].used > 1) for (int s = 0; s < size[k]; s++) { C->code[base[k] + s] = pc[k].code[s]; C->len[base[k] + s] = pc[k].len[s]; }
    CU(cudaMemcpyAsync(B.codes, C, sizeof(Vp8lCodes), cudaMemcpyHostToDevice, st));
    int rc = launch_vp8l_size(B, cw, h, cand, bit_base, st);
    if (!launch_ok(rc, "vp8l kernels", err)) return false;
    CU(cudaMemcpyAsync(h_total, B.total, 8, cudaMemcpyDeviceToHost, st));
    CU(stream_wait(st));
    const unsigned long long total = *h_total;
    const size_t words = (size_t)((total + 31) / 32), nbytes = (size_t)((total + 7) / 8);
    const size_t pad = nbytes & 1, riff = 4 + 8 + nbytes + pad;
    last_d2h_bytes += 8;
    file_bytes = 8 + riff;
    if (file_bytes >= below) return true;                                   // not kept: no emission
    if (!grow(d_words, words * 4, err) || !grow(h_words, words * 4, err)) return false;
    B.words = d_words;
    last_d2h_bytes += words * 4;
    rc = launch_vp8l_emit(B, cw, h, cand, words, st);
    if (!launch_ok(rc, "vp8l kernels", err)) return false;
    CU(cudaMemcpyAsync(h_words, d_words, words * 4, cudaMemcpyDeviceToHost, st));
    CU(stream_wait(st));
    // ---- the header bits go into the first bytes, then the RIFF framing
    uint8_t *payload = h_words;
    for (size_t i = 0; i < hdr.size(); i++) payload[i] |= hdr[i];
    out.resize(8 + riff);
    uint8_t *o = out.data();
    auto u32 = [](uint8_t *p, uint32_t v) { for (int i = 0; i < 4; i++) p[i] = (uint8_t)(v >> (8 * i)); };
    memcpy(o, "RIFF", 4); u32(o + 4, (uint32_t)riff); memcpy(o + 8, "WEBPVP8L", 8); u32(o + 16, (uint32_t)nbytes);
    memcpy(o + 20, payload, nbytes);
    if (pad) o[20 + nbytes] = 0;
    return true;
}

std::string Vp8lDevice::palette_trace() const
{
    if (!webp_palette()) return "";
    char b[160];
    if (last_palette < 0) snprintf(b, sizeof b, ", palette: over %d colours (collect %.4f ms)", VP8L_PAL_MAX, last_palette_ms);
    else snprintf(b, sizeof b, ", palette: %d colours, kept %s, %zu B without / %zu B with (palette kernels %.4f ms)", last_palette,
                  last_palette_kept ? "palette" : "no palette", last_bytes[0], last_bytes[1], last_palette_ms);
    return b;
}

} // namespace b200
