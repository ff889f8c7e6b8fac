// CPU emulation of the lossless WebP (VP8L) analysis kernels (csrc/vp8l_kernels.cu) through the shared bodies of
// csrc/vp8l_enc_core.h, in the kernels' shapes: k_vp8l_predict's per-tile scoring with the 257-entry n log2 n table, the colour cache
// as per-chunk last-occurrence tables + a carry scan + 32-pixel steps against a cache table (k_vp8l_cache_last / _carry / _hits),
// the copy search on equality bit arrays with all-ones summary words (k_vp8l_match), and the parse by pointer doubling
// (k_vp8l_parse).  The test compares its modes, cache hits and tokens with the oracle's plain loops.  Test infrastructure only.
#include <cstdint>
#include <cstring>
#include <vector>
#include "../../caesium-clt_b200/csrc/vp8l_enc_core.h"

using namespace b200;

static int ffs32(uint32_t m) { return __builtin_ffs((int)m); }

// check_definition: also hold every pixel's copy against vp8l_best_copy (the definition, quadratic on flat images); returns the
// token count, or (size_t)-1 when the two differ somewhere
extern "C" size_t emul_vp8l_stages(const uint8_t *rgba, int w, int h, int check_definition, uint8_t *modes_out, uint8_t *hits_out, uint32_t *tok_out)
{
    const size_t n = (size_t)w * h;
    const int tiles_x = (w + VP8L_TILE - 1) >> VP8L_TILE_BITS, tiles_y = (h + VP8L_TILE - 1) >> VP8L_TILE_BITS;
    std::vector<uint32_t> argb(n), res(n), best(n);
    for (size_t i = 0; i < n; i++)
        argb[i] = vp8l_sub_green(((uint32_t)rgba[4 * i + 3] << 24) | ((uint32_t)rgba[4 * i] << 16) | ((uint32_t)rgba[4 * i + 1] << 8) | rgba[4 * i + 2]);
    // ---- k_vp8l_predict: one "CTA" per tile, 256 "threads" each holding its pixel and neighbours
    uint64_t nlog[257];
    for (int k = 0; k <= 256; k++) nlog[k] = vp8l_nlog2_q10((uint32_t)k);
    for (int t = 0; t < tiles_x * tiles_y; t++) {
        const int tx = t % tiles_x, ty = t / tiles_x;
        int best_m = 0; uint64_t best_cost = 0;
        for (int m = 0; m < VP8L_NMODES; m++) {
            uint32_t hist[1024] = {0}, npix = 0;
            for (int th = 0; th < 256; th++) {
                const int x = tx * VP8L_TILE + (th & 15), y = ty * VP8L_TILE + (th >> 4);
                if (x >= w || y >= h) continue;
                const size_t idx = (size_t)y * w + x;
                const uint32_t P = argb[idx], L = x ? argb[idx - 1] : 0, T = y ? argb[idx - w] : 0, TR = y ? argb[idx - w + 1] : 0, TL = x && y ? argb[idx - w - 1] : 0;
                const uint32_t r = vp8l_sub_px(P, y == 0 ? (x ? L : 0xFF000000u) : x == 0 ? T : vp8l_predict(m, L, T, TR, TL));
                hist[r & 0xFF]++; hist[256 + ((r >> 8) & 0xFF)]++; hist[512 + ((r >> 16) & 0xFF)]++; hist[768 + (r >> 24)]++; npix++;
            }
            uint64_t tot = 0;
            for (int th = 0; th < 256; th++) tot += nlog[hist[th]] + nlog[hist[256 + th]] + nlog[hist[512 + th]] + nlog[hist[768 + th]];
            const uint64_t cost = 4 * nlog[npix] - tot;
            if (m == 0 || cost < best_cost) { best_cost = cost; best_m = m; }
        }
        modes_out[t] = (uint8_t)best_m;
        for (int th = 0; th < 256; th++) {
            const int x = tx * VP8L_TILE + (th & 15), y = ty * VP8L_TILE + (th >> 4);
            if (x < w && y < h) res[(size_t)y * w + x] = vp8l_sub_px(argb[(size_t)y * w + x], vp8l_predict_at(best_m, argb.data(), w, x, y));
        }
    }
    // ---- colour cache: last position per (chunk, key), carried over the chunks, then each chunk in steps of 32
    const int nchunks = (int)((n + VP8L_CHUNK - 1) / VP8L_CHUNK);
    for (int c = 1; c < VP8L_NCACHE; c++) {
        const int bits = vp8l_cache_bits(c), nk = 1 << bits;
        std::vector<int> last((size_t)nchunks * nk, -1);
        for (int b = 0; b < nchunks; b++)
            for (size_t i = (size_t)b * VP8L_CHUNK; i < n && i < (size_t)(b + 1) * VP8L_CHUNK; i++) {
                int &slot = last[(size_t)b * nk + vp8l_cache_key(res[i], bits)];
                if ((int)i > slot) slot = (int)i;
            }
        for (int k = 0; k < nk; k++) { int run = -1; for (int b = 0; b < nchunks; b++) { const int v = last[(size_t)b * nk + k]; last[(size_t)b * nk + k] = run; if (v >= 0) run = v; } }
        for (int b = 0; b < nchunks; b++) {
            std::vector<uint32_t> cache(nk);
            for (int k = 0; k < nk; k++) { const int p = last[(size_t)b * nk + k]; cache[k] = p >= 0 ? res[p] : 0u; }
            const size_t begin = (size_t)b * VP8L_CHUNK, end = begin + VP8L_CHUNK < n ? begin + VP8L_CHUNK : n;
            for (size_t base = begin; base < end; base += 32) {
                const int lanes = (int)(end - base < 32 ? end - base : 32);
                uint32_t have[32];
                for (int l = 0; l < lanes; l++) {        // an earlier lane with the same key, else the cache table
                    const uint32_t key = vp8l_cache_key(res[base + l], bits);
                    int src = -1;
                    for (int e = 0; e < l; e++) if (vp8l_cache_key(res[base + e], bits) == key) src = e;
                    have[l] = src >= 0 ? res[base + src] : cache[key];
                }
                for (int l = 0; l < lanes; l++) {
                    hits_out[(size_t)(c - 1) * n + base + l] = have[l] == res[base + l];
                    cache[vp8l_cache_key(res[base + l], bits)] = res[base + l];        // lanes in order: the last one of a key stays
                }
            }
        }
    }
    // ---- k_vp8l_match: equality bit arrays per candidate and all-ones summary words, runs to the next zero bit
    const int NW = VP8L_CHUNK / 32;
    for (int b = 0; b < nchunks; b++) {
        const size_t begin = (size_t)b * VP8L_CHUNK;
        const uint32_t len = (uint32_t)(n - begin < (size_t)VP8L_CHUNK ? n - begin : (size_t)VP8L_CHUNK);
        uint32_t eq[VP8L_NCAND][NW], full[VP8L_NCAND][NW / 32];
        memset(eq, 0, sizeof(eq)); memset(full, 0, sizeof(full));
        for (int c = 0; c < VP8L_NCAND; c++) {
            const uint32_t d = vp8l_code_dist(c + 1, w);
            for (uint32_t j = 0; j < len; j++) if (begin + j >= d && res[begin + j - d] == res[begin + j]) eq[c][j >> 5] |= 1u << (j & 31);
            for (int wd = 0; wd < NW; wd++) if (eq[c][wd] == 0xFFFFFFFFu) full[c][wd >> 5] |= 1u << (wd & 31);
        }
        for (uint32_t j = 0; j < len; j++) {
            uint32_t bl = 0, bc = 0;
            for (int c = 0; c < VP8L_NCAND; c++) {
                const int w0 = (int)(j >> 5);
                const uint32_t m = ~eq[c][w0] & (0xFFFFFFFFu << (j & 31));
                uint32_t stop = VP8L_CHUNK;
                if (m) stop = (uint32_t)w0 * 32 + (uint32_t)(ffs32(m) - 1);
                else
                    for (int wd = w0 + 1; wd < NW;) {
                        const int s = wd >> 5;
                        const uint32_t nf = ~full[c][s] & (0xFFFFFFFFu << (wd & 31));
                        if (nf) { wd = s * 32 + ffs32(nf) - 1; stop = (uint32_t)wd * 32 + (uint32_t)(ffs32(~eq[c][wd]) - 1); break; }
                        wd = (s + 1) * 32;
                    }
                if (stop - j > bl) { bl = stop - j; bc = (uint32_t)c + 1; }
            }
            best[begin + j] = bl >= VP8L_MIN_COPY ? (bl << 8) | bc : 0u;
            if (check_definition && best[begin + j] != vp8l_best_copy(res.data(), (uint32_t)n, w, (uint32_t)(begin + j))) return (size_t)-1;
        }
    }
    // ---- k_vp8l_parse: reachability from each chunk's first pixel by pointer doubling
    size_t ntok = 0;
    for (int b = 0; b < nchunks; b++) {
        const size_t begin = (size_t)b * VP8L_CHUNK;
        const int len = (int)(n - begin < (size_t)VP8L_CHUNK ? n - begin : (size_t)VP8L_CHUNK);
        std::vector<int> jump(VP8L_CHUNK + 1), nj(VP8L_CHUNK + 1);
        std::vector<uint8_t> visited(VP8L_CHUNK + 1, 0), mark(VP8L_CHUNK + 1);
        for (int j = 0; j <= VP8L_CHUNK; j++) {
            int nx = len;
            if (j < len) { const int s = (int)vp8l_parse_step(best[begin + j], j + 1 < len ? best[begin + j + 1] : 0u); nx = j + s < len ? j + s : len; }
            jump[j] = nx;
        }
        visited[0] = 1;
        for (int r = 0; (1 << r) < len; r++) {
            for (int j = 0; j <= VP8L_CHUNK; j++) { mark[j] = j < len && visited[j] && jump[j] < len; nj[j] = jump[jump[j]]; }
            for (int j = 0; j <= VP8L_CHUNK; j++) { if (mark[j]) visited[jump[j]] = 1; }
            jump.swap(nj);
        }
        for (int j = 0; j < len; j++) {
            if (!visited[j]) continue;
            tok_out[2 * ntok] = (uint32_t)(begin + j);
            tok_out[2 * ntok + 1] = vp8l_token_copy(best[begin + j], j + 1 < len ? best[begin + j + 1] : 0u);
            ntok++;
        }
    }
    return ntok;
}
