// tests/emul/stuff_emul.cpp -- TEST INFRASTRUCTURE.  Serial CPU run of the device encoder's stuffing passes (k_ge_ffcount,
// k_ge_layout, k_ge_scatter in jpeg_gpuenc.cu) over one megabatch, laid out the way k_ge_scanout / GpuEncoder lay it out, with
// the kernels' per-thread bodies from jpeg_gpuenc_stuff_core.h.  Not part of the product.
//
// The run records every output byte a CTA writes (each CTA's store phase runs twice, on buffers holding two different canaries),
// so a byte written by two CTAs (a race on the device) or outside its scan's output range shows up even when the last writer left
// the right value.  `fault` swaps one rule for a deliberately wrong one, so that a test can show the checks catch it.
#include <cstdint>
#include <cstring>
#include <utility>
#include <vector>
#include "../../caesium-clt_b200/csrc/jpeg_gpuenc_stuff_core.h"

using namespace b200;

namespace {
struct Rng {                    // garbage for the buffers the device never initialises
    uint64_t s;
    uint32_t next() { s ^= s << 13; s ^= s >> 7; s ^= s << 17; return (uint32_t)s; }
};
constexpr uint8_t CANARY_A = 0xA5, CANARY_B = 0x5A;
constexpr uint32_t SLACK = 64;  // bytes on either side of a tile's output range where a stray store would be seen (a multiple of 4)
}

// the wrong rules `fault` selects
enum { FAULT_NONE, FAULT_NO_PADDING, FAULT_NO_CLEAR, FAULT_WHOLE_EDGE_WORDS, FAULT_CHUNK_PREFIX, FAULT_NO_TILE_CARRY, FAULT_N };

// Stats reported in stats[]:
//   tiles stored; tiles by (first output byte mod 4) and by (end of their output range mod 4); bytes written more than once; bytes
//   written outside their scan's output range
enum { ST_TILES, ST_FIRST_MOD4, ST_END_MOD4 = ST_FIRST_MOD4 + 4, ST_DOUBLE_WRITES = ST_END_MOD4 + 4, ST_STRAY_WRITES, ST_N };

// nimages x spi scans; scan s has total_bits[s] bits in words (big-endian within a word; ceil(total_bits / 32) words per scan,
// back to back, bits and bytes past the scan's end arbitrary).  nchunks / tile = CTAs per scan and threads per CTA.  out
// (nimages x out_stride bytes) receives the stuffed scans at out_off / out_len within each image's region; bytes no pass writes hold
// CANARY_A.  flags[3] / flags[4] as k_ge_layout leaves them.  Returns 0, or 1 on bad arguments.
extern "C" int emul_stuff_batch(int nimages, int spi, const uint32_t *total_bits, const uint32_t *words, int nchunks, int tile, uint32_t out_stride,
                                int fault, uint64_t seed, uint8_t *out, uint32_t *out_off, uint32_t *out_len, uint32_t *flags, long long stats[ST_N])
{
    if (nimages < 1 || spi < 1 || nchunks < 1 || tile < 1 || tile > 1024 || nchunks > tile || out_stride % 4 || fault < 0 || fault >= FAULT_N) return 1;
    const int NS = nimages * spi;
    for (int i = 0; i < ST_N; i++) stats[i] = 0;
    Rng rng{seed * 0x9E3779B97F4A7C15ull + 1};
    // ---- k_ge_scanout: every scan's words start at a multiple of four; the bit buffer holds garbage where emit wrote nothing
    std::vector<uint32_t> nbytes((size_t)NS), word_base((size_t)NS);
    size_t wtotal = 0;
    for (int s = 0; s < NS; s++) {
        word_base[(size_t)s] = (uint32_t)wtotal; nbytes[(size_t)s] = (total_bits[s] + 7) / 8;
        wtotal += ((total_bits[s] + 31) / 32 + 1 + 3) & ~3u;
    }
    std::vector<uint32_t> buf(wtotal + 4);
    for (auto &w : buf) w = rng.next() | ((rng.next() & 1) ? 0xFF00FF00u : 0u);
    for (int s = 0, at = 0; s < NS; at += (int)((total_bits[s] + 31) / 32), s++) memcpy(&buf[word_base[(size_t)s]], words + at, (total_bits[s] + 31) / 32 * 4);
    auto group = [&](int s, uint32_t g) {
        ge::ScanGroup q; memcpy(q.w, &buf[word_base[(size_t)s] + 4 * (size_t)g], 16);
        if (fault == FAULT_NO_CLEAR) { return std::make_pair(q, nbytes[(size_t)s] - 16 * g < 16 ? nbytes[(size_t)s] - 16 * g : 16u); }
        const uint32_t n = ge::stuff_group(q, g, nbytes[(size_t)s], fault == FAULT_NO_PADDING ? total_bits[s] & ~7u : total_bits[s]);
        return std::make_pair(q, n);
    };
    // ---- k_ge_ffcount: grid (nchunks, NS); chunkff is not initialised
    std::vector<uint32_t> chunkff((size_t)NS * nchunks);
    for (auto &c : chunkff) c = rng.next();
    for (int y = 0; y < NS; y++) for (int x = 0; x < nchunks; x++) {
        uint32_t g0, g1, n = 0;
        ge::stuff_chunk(nbytes[(size_t)y], (uint32_t)x, (uint32_t)nchunks, (uint32_t)tile, g0, g1);
        for (int t = 0; t < tile; t++) for (uint32_t g = g0 + (uint32_t)t; g < g1; g += (uint32_t)tile) n += ge::stuff_ff_count(group(y, g).first);
        chunkff[(size_t)y * nchunks + x] = n;
    }
    // ---- k_ge_layout: one CTA per image; flags[3..4] were zeroed by k_ge_scanout
    flags[3] = 0; flags[4] = 0;
    for (int im = 0; im < nimages; im++) {
        uint32_t off = 0;
        for (int k = 0; k < spi; k++) {
            const int si = im * spi + k;
            uint32_t ff = 0;
            for (int x = 0; x < nchunks; x++) ff += chunkff[(size_t)si * nchunks + x];
            out_off[si] = off; out_len[si] = nbytes[(size_t)si] + ff; off += out_len[si];
        }
        if (off > flags[3]) flags[3] = off;
        if (off > out_stride) flags[4] = 1;
    }
    // ---- k_ge_scatter: grid (nchunks, NS), nothing at all once flags[4] is raised
    memset(out, CANARY_A, (size_t)nimages * out_stride);
    if (flags[4]) return 0;
    std::vector<uint8_t> writes((size_t)nimages * (out_stride + 2 * SLACK), 0), runA, runB;
    std::vector<uint32_t> sbuf((size_t)tile * 8 + 1 + 64);  // the kernel's buffer, and slack that a wrong offset would run into
    uint8_t *sb = reinterpret_cast<uint8_t *>(sbuf.data());
    std::vector<ge::ScanGroup> q((size_t)tile);
    std::vector<uint32_t> n((size_t)tile), len((size_t)tile);
    for (int y = 0; y < NS; y++) for (int x = 0; x < nchunks; x++) {
        uint32_t g0, g1;
        ge::stuff_chunk(nbytes[(size_t)y], (uint32_t)x, (uint32_t)nchunks, (uint32_t)tile, g0, g1);
        if (g0 >= g1) continue;
        const int im = y / spi;
        uint32_t ff_before = 0;
        for (int j = 0; j < x - (fault == FAULT_CHUNK_PREFIX && x > 1 ? 1 : 0); j++) ff_before += chunkff[(size_t)y * nchunks + j];
        uint32_t at = out_off[y] + g0 * 16 + ff_before;
        for (uint32_t t0 = g0; t0 < g1; t0 += (uint32_t)tile) {
            for (auto &w : sbuf) w = rng.next();            // shared memory is not initialised
            uint32_t L = 0;
            for (int t = 0; t < tile; t++) {
                const uint32_t g = t0 + (uint32_t)t;
                n[(size_t)t] = len[(size_t)t] = 0;
                if (g < g1) { auto qn = group(y, g); q[(size_t)t] = qn.first; n[(size_t)t] = qn.second; len[(size_t)t] = qn.second + ge::stuff_ff_count(qn.first); }
                L += len[(size_t)t];
            }
            const uint32_t aligned = at & ~3u;
            for (int t = 0, rel = 0; t < tile; rel += (int)len[(size_t)t], t++)
                if (n[(size_t)t]) ge::stuff_place_group(q[(size_t)t], n[(size_t)t], at - aligned + (uint32_t)rel, sb);
            stats[ST_TILES]++; stats[ST_FIRST_MOD4 + (at & 3)]++; stats[ST_END_MOD4 + ((at + L) & 3)]++;
            // the store phase, on a window of the tile's range and SLACK bytes on either side (positions shifted by `aligned`, a
            // multiple of four, so that the word alignment is the image region's)
            const size_t win = (size_t)(at - aligned) + L + 4 + 2 * SLACK;
            runA.assign(win, CANARY_A); runB.assign(win, CANARY_B);
            for (int pass = 0; pass < 2; pass++) {
                uint8_t *b = (pass ? runB : runA).data() + SLACK;
                for (int t = 0; t < tile; t++) {
                    if (fault == FAULT_WHOLE_EDGE_WORDS)
                        for (uint32_t a = 4 * (uint32_t)t; a < at - aligned + L; a += 4 * (uint32_t)tile) memcpy(b + a, &sbuf[a >> 2], 4);
                    else ge::stuff_store(sbuf.data(), 0, at - aligned, at - aligned + L, (uint32_t)t, (uint32_t)tile, b);
                }
            }
            for (size_t j = 0; j < win; j++) {
                if (runA[j] == CANARY_A && runB[j] == CANARY_B) continue;
                const uint8_t v = runA[j] == CANARY_A ? runB[j] : runA[j];
                const long long p = (long long)aligned - SLACK + (long long)j;          // position in the image's region
                if (p < -(long long)SLACK || p >= (long long)out_stride + SLACK) { stats[ST_STRAY_WRITES]++; continue; }
                if (writes[(size_t)im * (out_stride + 2 * SLACK) + (size_t)(p + SLACK)]++) stats[ST_DOUBLE_WRITES]++;
                if (p < (long long)out_off[y] || p >= (long long)out_off[y] + out_len[y] || p >= (long long)out_stride) { stats[ST_STRAY_WRITES]++; continue; }
                out[(size_t)im * out_stride + (size_t)p] = v;
            }
            at += fault == FAULT_NO_TILE_CARRY ? L - (L > 0) : L;
        }
    }
    return 0;
}
