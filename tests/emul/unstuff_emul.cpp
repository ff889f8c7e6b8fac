// tests/emul/unstuff_emul.cpp -- TEST INFRASTRUCTURE.  Serial CPU run of the device decoder's un-stuff passes
// (k_gd_unstuff_count, the exclusive scan, k_gd_unstuff_scatter in jpeg_gpudec.cu) over one decode batch, laid out the way
// GpuDecoder::prepare / enqueue lay it out, with the kernels' per-thread bodies from jpeg_gpudec_core.h.  Not part of the product.
//
// Besides the output, the run reports what a serial run would otherwise hide: every output byte a CTA writes is recorded, so a
// byte written by two CTAs (a race on the device) or outside the image's stream region shows up even when the last writer
// happened to leave the right value.
#include <cstdint>
#include <cstring>
#include <vector>
#include "../../caesium-clt_b200/csrc/jpeg_gpudec_core.h"

using namespace b200;

namespace {
struct Image {                  // the fields of b200::DecImage the un-stuff passes read and write
    uint32_t raw_off, nraw, stream_off, grp_off, ngrp, verify;
    gd::Geometry g;
};
size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
uint32_t cdiv(uint32_t a, uint32_t b) { return (a + b - 1) / b; }
struct Rng {                    // garbage for the buffers the device never initialises
    uint64_t s;
    uint32_t next() { s ^= s << 13; s ^= s >> 7; s ^= s << 17; return (uint32_t)s; }
};
constexpr uint8_t CANARY_A = 0xA5, CANARY_B = 0x5A;
}

// Stats reported in stats[]:
//   CTAs run; CTAs by (first output byte mod 4) and by (end of their output range mod 4); bytes written more than once; bytes
//   written outside their image's stream region
enum { ST_CTAS, ST_FIRST_MOD4, ST_END_MOD4 = ST_FIRST_MOD4 + 4, ST_DOUBLE_WRITES = ST_END_MOD4 + 4, ST_STRAY_WRITES, ST_N };

// n images, segment n at segs + sum(lens[0..n-1]); verify[n] as the batch's DeviceScan::verified would give it (1 = the host did
// not walk the segment).  `threads` = threads per CTA of both kernels, subseq_bits = the decoder's subsequence size.  stream (stream_cap bytes) receives the batch's stream
// buffer; bytes no pass writes hold CANARY_A.  Per image: stream_off, the descriptor's nbits / nsub after the passes and the
// marker flag.  Returns 0, or 1 if stream_cap is too small / threads is out of range.
extern "C" int emul_unstuff_batch(int n, const uint8_t *segs, const uint32_t *lens, const int *verify, int threads, int subseq_bits, uint64_t seed,
                                  uint8_t *stream, size_t stream_cap, uint32_t *stream_off, uint32_t *nbits, uint32_t *nsub, uint32_t *marker,
                                  long long stats[ST_N])
{
    if (threads < 1 || threads > 1024 || subseq_bits < 32) return 1;
    for (int i = 0; i < ST_N; i++) stats[i] = 0;
    Rng rng{seed * 0x9E3779B97F4A7C15ull + 1};
    // ---- GpuDecoder::prepare: descriptors, raw buffer (16-aligned segments, 16 bytes of slack each), stream regions
    std::vector<Image> im((size_t)n);
    size_t raw_total = 0, stream_total = 0; uint32_t grp_total = 0, max_grp = 0;
    std::vector<size_t> seg_at((size_t)n);
    for (int k = 0, at = 0; k < n; at += (int)lens[k], k++) {
        Image &m = im[(size_t)k]; memset(&m, 0, sizeof(m));
        const uint8_t *s = segs + at; const uint32_t nraw = lens[k];
        seg_at[(size_t)k] = (size_t)at;
        uint32_t stuffed = 0;                                   // the host's walk (JpegReader::DeviceScan::stuffed)
        for (uint32_t j = 1; j < nraw; j++) stuffed += s[j] == 0 && s[j - 1] == 0xFF;
        const uint32_t nstream = verify[k] ? nraw : nraw - stuffed;
        m.verify = verify[k] ? 1u : 0u;
        m.g.subseq_bits = (uint32_t)subseq_bits; m.g.nbits = nstream * 8; m.g.nsub = cdiv(m.g.nbits, m.g.subseq_bits);
        m.raw_off = (uint32_t)raw_total; m.nraw = nraw; raw_total += align_up((size_t)nraw + 16, 16);
        m.stream_off = (uint32_t)stream_total; stream_total += align_up((size_t)nstream + 32, 16);
        m.grp_off = grp_total; m.ngrp = cdiv(nraw, 16); grp_total += m.ngrp;
        if (m.ngrp > max_grp) max_grp = m.ngrp;
    }
    if (stream_total > stream_cap) return 1;
    // high-water sizes as GpuDecoder keeps them: the count array and its scan run past this batch's groups into a stale tail
    const uint32_t hw_grp = grp_total + grp_total / 8 + 64, hw_mgrp = max_grp + max_grp / 8 + 64;
    std::vector<uint8_t> raw(raw_total + 64);
    for (auto &b : raw) { const uint32_t r = rng.next(); b = (r & 3) == 0 ? 0xFF : (r & 3) == 1 ? 0x00 : (uint8_t)(r >> 8); }   // slack: 0xFF / 0x00-rich garbage
    for (int k = 0; k < n; k++) memcpy(&raw[im[(size_t)k].raw_off], segs + seg_at[(size_t)k], lens[k]);
    std::vector<uint32_t> cnt(hw_grp + 1), off(hw_grp + 1), mark((size_t)n, 0);
    for (auto &c : cnt) c = rng.next();                     // stale counts of earlier batches
    memset(stream, CANARY_A, stream_cap);
    auto group = [&](const Image &m, uint32_t g) { gd::RawGroup q; memcpy(&q, &raw[m.raw_off + 16 * (size_t)g], 16); return q; };
    // ---- k_gd_unstuff_count: grid (cdiv(hw_mgrp, threads), n)
    const uint32_t gx = cdiv(hw_mgrp, (uint32_t)threads);
    for (int y = 0; y < n; y++) for (uint32_t bx = 0; bx < gx; bx++) for (int t = 0; t < threads; t++) {
        const Image &m = im[(size_t)y];
        const uint32_t g = bx * (uint32_t)threads + (uint32_t)t;
        if (g >= m.ngrp) continue;
        bool mk;
        cnt[m.grp_off + g] = gd::unstuff_count_group(&raw[m.raw_off], group(m, g), g, m.nraw, m.verify, &mk);
        if (mk) mark[(size_t)y] = 1;
    }
    // ---- cub::DeviceScan::ExclusiveSum over hw_grp counts (modulo 2^32, stale tail included)
    { uint32_t run = 0; for (uint32_t i = 0; i < hw_grp; i++) { off[i] = run; run += cnt[i]; } }
    // ---- k_gd_unstuff_scatter, one CTA at a time: every thread places its group, then (after the barrier) every thread stores
    std::vector<uint32_t> sbuf((size_t)threads * 4 + 1 + 64);       // the kernel's buffer, and slack that a wrong offset would run into
    const size_t span = stream_cap + 4096;                   // room for stray stores past the buffer
    std::vector<uint8_t> writes(span, 0), runA(span), runB(span);
    for (int y = 0; y < n; y++) for (uint32_t bx = 0; bx < gx; bx++) {
        Image &m = im[(size_t)y];
        const uint32_t g0 = bx * (uint32_t)threads;
        if (g0 >= m.ngrp) continue;
        stats[ST_CTAS]++;
        for (auto &w : sbuf) w = rng.next();                 // shared memory is not initialised
        uint8_t *sb = reinterpret_cast<uint8_t *>(sbuf.data());
        const uint32_t base = off[m.grp_off];
        const uint32_t first = g0 * 16 - (off[m.grp_off + g0] - base), aligned = first & ~3u;
        uint32_t range_end = rng.next();
        for (int t = 0; t < threads; t++) {
            const uint32_t g = g0 + (uint32_t)t;
            if (g >= m.ngrp) continue;
            const uint32_t o = gd::unstuff_place_group(&raw[m.raw_off], group(m, g), g, m.nraw, g * 16 - (off[m.grp_off + g] - base), aligned, sb);
            if (g == g0 + (uint32_t)threads - 1 || g == m.ngrp - 1) range_end = o;
        }
        stats[ST_FIRST_MOD4 + (first & 3)]++; stats[ST_END_MOD4 + (range_end & 3)]++;
        // the store phase runs twice, on buffers filled with two different canaries: a byte is written iff it changed in either
        const gd::Geometry g_in = m.g;
        gd::Geometry g_out = m.g;
        for (int pass = 0; pass < 2; pass++) {
            std::vector<uint8_t> &buf = pass ? runB : runA;
            memset(buf.data(), pass ? CANARY_B : CANARY_A, span);
            gd::Geometry gg = g_in;
            for (int t = 0; t < threads; t++) {
                const uint32_t g = g0 + (uint32_t)t;
                const bool last = g == m.ngrp - 1;
                gd::unstuff_store(sbuf.data(), aligned, first, range_end, (uint32_t)t, (uint32_t)threads, buf.data() + m.stream_off, last, m.verify, m.nraw,
                                  last ? &off[m.grp_off + g] : nullptr, last ? &cnt[m.grp_off + g] : nullptr, base, gg);
            }
            g_out = gg;
        }
        m.g = g_out;
        for (size_t j = 0; j < span; j++) {
            if (runA[j] == CANARY_A && runB[j] == CANARY_B) continue;
            const uint8_t v = runA[j] == CANARY_A ? runB[j] : runA[j];
            if (writes[j]++) stats[ST_DOUBLE_WRITES]++;
            const size_t lo = m.stream_off, hi = (size_t)m.stream_off + align_up((size_t)(m.verify ? m.nraw : g_in.nbits / 8) + 32, 16);
            if (j < lo || j >= hi) stats[ST_STRAY_WRITES]++;
            if (j < stream_cap) stream[j] = v;
        }
    }
    for (int k = 0; k < n; k++) { stream_off[k] = im[(size_t)k].stream_off; nbits[k] = im[(size_t)k].g.nbits; nsub[k] = im[(size_t)k].g.nsub; marker[k] = mark[(size_t)k]; }
    return 0;
}

// the stream buffer size emul_unstuff_batch needs for these segments
extern "C" size_t emul_unstuff_stream_bytes(int n, const uint32_t *lens)
{
    size_t t = 0;
    for (int k = 0; k < n; k++) t += align_up((size_t)lens[k] + 32, 16);
    return t;
}
