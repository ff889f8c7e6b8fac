// CPU emulation of the lossless WebP (VP8L) encoder's palette kernels (csrc/vp8l_palette.cu) through the shared bodies of
// csrc/vp8l_palette_core.h, in the kernels' shapes: k_vp8l_palette_collect's CTAs one after another -- the overflow flag read at
// entry and after each step, a step's 256 pixels deduplicated per 32-lane warp and inserted into the CTA's 1024-slot set, the
// CTA's colours merged into the global set by bounded probing -- then k_vp8l_palette_sort's compaction and 256-wide bitonic
// network, then k_vp8l_palette_pack per packed pixel.  The test compares the result with a numpy restatement.  Test
// infrastructure only.
#include <cstdint>
#include <cstring>
#include <vector>
#include "../../caesium-clt_b200/csrc/vp8l_palette_core.h"

using namespace b200;

static const uint64_t USED = 1ull << 32;

// insert key into a set of VP8L_PAL_SET slots, probing at most `limit` slots: 1 when new, 0 when present, -1 when no slot was found
static int insert(uint64_t *set, uint64_t key, int limit)
{
    uint32_t h = vp8l_pal_hash((uint32_t)key);
    for (int p = 0; p < limit; p++, h = (h + 1) & (VP8L_PAL_SET - 1)) {
        if (set[h] == 0) { set[h] = key; return 1; }
        if (set[h] == key) return 0;
    }
    return -1;
}

// rgba [h][w][4] -> info (VP8L_PAL_INFO words: count, overflow flag, palette), packed [w x h] and *packed_w (only without overflow),
// stats[3]: CTAs that reached the merge, CTAs that stopped inside their steps, CTAs that stopped at entry
extern "C" void emul_vp8l_palette(const uint8_t *rgba, int w, int h, uint32_t *info, uint32_t *packed, int *packed_w, int *stats)
{
    const uint32_t n = (uint32_t)w * (uint32_t)h;
    std::vector<uint32_t> argb(n);
    for (uint32_t i = 0; i < n; i++)
        argb[i] = vp8l_sub_green(((uint32_t)rgba[4 * i + 3] << 24) | ((uint32_t)rgba[4 * i] << 16) | ((uint32_t)rgba[4 * i + 1] << 8) | rgba[4 * i + 2]);
    memset(info, 0, 4 * VP8L_PAL_INFO);
    stats[0] = stats[1] = stats[2] = 0;
    *packed_w = 0;
    std::vector<uint64_t> gset(VP8L_PAL_SET, 0);
    const uint32_t nctas = (n + VP8L_PAL_CTA_PIXELS - 1) / VP8L_PAL_CTA_PIXELS;
    for (uint32_t b = 0; b < nctas; b++) {
        if (info[1]) { stats[2]++; continue; }
        std::vector<uint64_t> set(VP8L_PAL_SET, 0);
        int count = 0; bool stop = false;
        for (int s = 0; s < VP8L_PAL_STEPS && !stop; s++) {
            for (int warp = 0; warp < VP8L_PAL_THREADS / 32; warp++) {
                uint64_t key[32];
                for (int lane = 0; lane < 32; lane++) {
                    const uint32_t i = b * VP8L_PAL_CTA_PIXELS + (uint32_t)s * VP8L_PAL_THREADS + (uint32_t)(warp * 32 + lane);
                    key[lane] = i < n ? USED | vp8l_add_green(argb[i]) : 0;
                }
                for (int lane = 0; lane < 32; lane++) {
                    bool leader = key[lane] != 0;
                    for (int o = 0; o < lane && leader; o++) leader = key[o] != key[lane];
                    if (leader && insert(set.data(), key[lane], VP8L_PAL_SET) == 1) count++;
                }
            }
            if (count > VP8L_PAL_MAX) info[1] = 1;
            stop = count > VP8L_PAL_MAX || info[1];
        }
        if (stop) { stats[1]++; continue; }
        stats[0]++;
        for (int k = 0; k < VP8L_PAL_SET; k++) {
            if (!set[k]) continue;
            const int r = insert(gset.data(), set[k], VP8L_PAL_SET);
            if (r == 1 && info[0]++ >= (uint32_t)VP8L_PAL_MAX) info[1] = 1;
            if (r < 0) info[1] = 1;
        }
    }
    if (info[1]) return;
    // ---- k_vp8l_palette_sort: compaction in slot order, then the bitonic network as 256 threads run it
    std::vector<uint64_t> v(VP8L_PAL_MAX, ~0ull);
    int m = 0;
    for (int t = 0; t < VP8L_PAL_MAX; t++)
        for (int k = t; k < VP8L_PAL_SET; k += VP8L_PAL_MAX) if (gset[k]) v[m++] = gset[k];
    for (int k = 2; k <= VP8L_PAL_MAX; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1)
            for (int t = 0; t < VP8L_PAL_MAX; t++) {
                const int o = t ^ j;
                if (o > t && ((v[t] > v[o]) == ((t & k) == 0))) { const uint64_t a = v[t]; v[t] = v[o]; v[o] = a; }
            }
    for (int t = 0; t < VP8L_PAL_MAX; t++) info[2 + t] = t < m ? (uint32_t)v[t] : 0u;
    // ---- k_vp8l_palette_pack
    const int count = (int)info[0], xbits = vp8l_pal_xbits(count), wp = vp8l_pal_width(w, xbits);
    *packed_w = wp;
    for (uint32_t i = 0; i < (uint32_t)wp * (uint32_t)h; i++) {
        const uint32_t y = i / (uint32_t)wp, xp = i - y * (uint32_t)wp;
        packed[i] = vp8l_pal_pack(argb.data() + (size_t)y * w, w, (int)xp, info + 2, count, xbits);
    }
}
