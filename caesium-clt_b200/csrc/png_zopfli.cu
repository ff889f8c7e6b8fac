// png_zopfli.cu -- the PNG `--zopfli` leg on the device: zopfli's method (a shortest-path parse over every match a position
// offers, re-run with costs from the previous parse's statistics) over the rules of png_zopfli_core.h, slice by slice:
//   k_pz_keys / CUB radix sort / k_pz_prev   the hash chains of the slice (and the window before it) as a "previous position with
//                                            the same hash" array: sorting (hash, position) stably puts each chain in order
//   k_pz_matches                             the kept match entries of every position (one thread per position)
//   per iteration: k_pz_costs (cost tables per region), k_pz_squeeze (one warp per segment: forward DP, back-trace, region
//   histograms), k_pz_score (the parse's score against the best so far), k_pz_keep (the best parse's tokens and counts)
// The iterations are enqueued back to back with no host wait; the tail (CUB scan, k_png_compact, launch_png_deflate) is the
// lossless leg's own.
#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <algorithm>
#include "png_zopfli.h"
#include "png_zopfli_core.h"
#include "png_kernels.h"
#include "launch_timer.h"

namespace b200 {

namespace {
constexpr int PZ_RING = 512;                // the squeeze's cost ring: a power of two above the 259 targets i .. i + 258
constexpr unsigned FULL = 0xFFFFFFFFu;
struct Cand { int d[10]; };

inline unsigned cdiv(size_t a, size_t b) { return (unsigned)((a + b - 1) / b); }
}

// iteration 1's statistics: the greedy parse's chunk-local tokens, counted into the region their chunk lies in (chunks divide regions)
__global__ void __launch_bounds__(256) k_pz_greedy_hist(const uint32_t *__restrict__ gtok, const uint32_t *__restrict__ gcounts, int gchunk, uint32_t *__restrict__ hist)
{
    __shared__ uint32_t h[PZ_NSYM];
    for (int x = threadIdx.x; x < PZ_NSYM; x += blockDim.x) h[x] = 0;
    __syncthreads();
    const size_t c = blockIdx.x;
    const uint32_t m = gcounts[c];
    const uint32_t *t = gtok + c * (size_t)gchunk;
    for (uint32_t k = threadIdx.x; k < m; k += blockDim.x) {
        const uint32_t v = t[k];
        if (v & 0x80000000u) { atomicAdd(&h[257 + pz_len_symbol(pz_elen(v & 0x7FFFFFFFu))], 1u); atomicAdd(&h[286 + pz_dist_symbol(pz_edist(v & 0x7FFFFFFFu))], 1u); }
        else atomicAdd(&h[v], 1u);
    }
    __syncthreads();
    uint32_t *dst = hist + (c * (size_t)gchunk / PZ_REGION) * PZ_NSYM;
    for (int x = threadIdx.x; x < PZ_NSYM; x += blockDim.x) if (h[x]) atomicAdd(&dst[x], h[x]);
}

__global__ void k_pz_keys(const uint8_t *__restrict__ s, size_t n, size_t ws, size_t cnt, uint32_t *__restrict__ key, uint32_t *__restrict__ val)
{
    const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= cnt) return;
    const size_t p = ws + k;
    key[k] = p + 3 <= n ? pz_hash3(s + p) : PZ_NOHASH;
    val[k] = (uint32_t)k;
}
// sorted stably by hash, each chain is a run in position order: a position's predecessor with the same hash is the entry before it
__global__ void k_pz_prev(const uint32_t *__restrict__ key, const uint32_t *__restrict__ val, size_t cnt, long long ws, int32_t *__restrict__ prev)
{
    const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= cnt) return;
    prev[val[k]] = k > 0 && key[k] == key[k - 1] && key[k] != PZ_NOHASH ? (int32_t)(ws + val[k - 1]) : -1;
}

__global__ void __launch_bounds__(256) k_pz_matches(const uint8_t *__restrict__ s, size_t n, size_t sl0, size_t sl1, Cand cand, const int32_t *__restrict__ prev, long long pbase,
                                                    uint32_t *__restrict__ ent)
{
    const size_t i = sl0 + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sl1) return;
    uint32_t e[PZ_K];
    const int m = pz_match_set(s, n, i, cand.d, prev, pbase, e);
    uint32_t *o = ent + (i - sl0) * PZ_K;
#pragma unroll
    for (int k = 0; k < PZ_K; k++) o[k] = k < m ? e[k] : PZ_NONE;
}

__global__ void k_pz_costs(const uint32_t *__restrict__ hist, uint32_t *__restrict__ cost, size_t r0, size_t r1)
{
    const size_t r = r0 + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r < r1) pz_costs(hist + r * PZ_NSYM, cost + r * PZ_NSYM);
}

// One warp per segment.  ring[t mod PZ_RING] holds the best cost found so far to reach segment position t; when the warp reaches i
// every source before i has been relaxed, so ring[i] is final.  The lanes then relax the match targets i + 3 .. i + top, 32 lengths
// a step (one target per lane: no two lanes write one target, so no atomics), lane 0 the literal target i + 1; bp[t - 1] keeps the
// token of the best edge into t.  A position's entries (PZ_K words) and byte are loaded one step ahead.
__global__ void __launch_bounds__(32) k_pz_squeeze(const uint8_t *__restrict__ s, size_t n, size_t sl0, const uint32_t *__restrict__ ent, const uint32_t *__restrict__ cost_all,
                                                   uint32_t *__restrict__ bp, uint32_t *__restrict__ tok, uint32_t *__restrict__ segc, uint32_t *__restrict__ hist_all)
{
    __shared__ uint32_t cost[PZ_NSYM], h[PZ_NSYM], ring[PZ_RING];
    const int lane = threadIdx.x;
    const size_t s0 = sl0 + (size_t)blockIdx.x * PZ_SEG, b0 = s0 - sl0;
    const int L = (int)min((size_t)PZ_SEG, n - s0);
    const size_t reg = s0 / PZ_REGION;
    for (int x = lane; x < PZ_NSYM; x += 32) { cost[x] = cost_all[reg * PZ_NSYM + x]; h[x] = 0; }
    for (int x = lane; x < PZ_RING; x += 32) ring[x] = x == 0 ? 0u : 0xFFFFFFFFu;
    __syncwarp();
    uint32_t nx = lane < PZ_K ? ent[b0 * PZ_K + lane] : PZ_NONE;
    uint32_t nb = lane == 0 ? s[s0] : 0;
    for (int i = 0; i < L; i++) {
        const uint32_t my = nx, byte = nb;
        if (i + 1 < L) { nx = lane < PZ_K ? ent[(b0 + i + 1) * PZ_K + lane] : PZ_NONE; if (lane == 0) nb = s[s0 + i + 1]; }
        const uint32_t ci = ring[i & (PZ_RING - 1)];
        const uint32_t mydc = my != PZ_NONE ? cost[286 + pz_dist_symbol(pz_edist(my))] : 0u;
        __syncwarp();
        if (lane == 0) {
            ring[i & (PZ_RING - 1)] = 0xFFFFFFFFu;                  // the slot becomes target i + PZ_RING, which no source has reached yet
            const uint32_t v = ci + cost[byte];
            if (v < ring[(i + 1) & (PZ_RING - 1)]) { ring[(i + 1) & (PZ_RING - 1)] = v; bp[b0 + i] = byte; }
        }
        const int cnt = __popc(__ballot_sync(FULL, my != PZ_NONE));
        if (cnt) {
            const int top = pz_elen(__shfl_sync(FULL, my, cnt - 1));
            for (int l0 = 3; l0 <= top; l0 += 32) {
                const int l = l0 + lane;
                uint32_t best = 0xFFFFFFFFu, be = 0;
                for (int k = 0; k < cnt; k++) {                     // pz_edge over the lanes' entries: farther entries win only when strictly cheaper
                    const uint32_t e = __shfl_sync(FULL, my, k), dc = __shfl_sync(FULL, mydc, k);
                    if (pz_elen(e) >= l && dc < best) { best = dc; be = e; }
                }
                if (l <= top) {
                    const uint32_t v = ci + best + cost[257 + pz_len_symbol(l)];
                    const int t = i + l;
                    if (v < ring[t & (PZ_RING - 1)]) { ring[t & (PZ_RING - 1)] = v; bp[b0 + t - 1] = 0x80000000u | ((uint32_t)(l - 3) << 16) | (be & 0xFFFFu); }
                }
            }
        }
        __syncwarp();
    }
    // back-trace (lane 0, tokens in reverse), then the warp puts them in order
    uint32_t m = 0;
    if (lane == 0) {
        for (int t = L; t > 0;) {
            const uint32_t v = bp[b0 + t - 1];
            tok[b0 + m++] = v;
            pz_count(h, v);
            t -= v & 0x80000000u ? pz_elen(v & 0x7FFFFFFFu) : 1;
        }
        segc[s0 / PZ_SEG] = m;
    }
    m = __shfl_sync(FULL, m, 0);
    __syncwarp();
    for (uint32_t a = lane; a < m / 2; a += 32) { const uint32_t x = tok[b0 + a]; tok[b0 + a] = tok[b0 + m - 1 - a]; tok[b0 + m - 1 - a] = x; }
    for (int x = lane; x < PZ_NSYM; x += 32) if (h[x]) atomicAdd(&hist_all[reg * PZ_NSYM + x], h[x]);
}

// the slice's score; state[0] = the best score so far, state[1] = 1 when this parse is strictly better (it is then kept)
__global__ void __launch_bounds__(256) k_pz_score(const uint32_t *__restrict__ hist, size_t r0, size_t r1, unsigned long long *__restrict__ state)
{
    __shared__ unsigned long long total;
    if (threadIdx.x == 0) total = 0;
    __syncthreads();
    unsigned long long sc = 0;
    for (size_t r = r0 + threadIdx.x; r < r1; r += blockDim.x) sc += pz_score(hist + r * PZ_NSYM);
    if (sc) atomicAdd(&total, sc);
    __syncthreads();
    if (threadIdx.x == 0) {
        const bool better = total < state[0];
        if (better) state[0] = total;
        state[1] = better;
    }
}
__global__ void __launch_bounds__(256) k_pz_keep(const uint32_t *__restrict__ tok, const uint32_t *__restrict__ segc, size_t g0, size_t sl0, const unsigned long long *__restrict__ state,
                                                 uint32_t *__restrict__ best, uint32_t *__restrict__ segn)
{
    if (!state[1]) return;
    const size_t g = g0 + blockIdx.x;
    const uint32_t m = segc[g];
    const uint32_t *src = tok + (g * PZ_SEG - sl0);
    uint32_t *dst = best + g * PZ_SEG;
    for (uint32_t k = threadIdx.x; k < m; k += blockDim.x) dst[k] = src[k];
    if (threadIdx.x == 0) segn[g] = m;
}

size_t PngZopfli::nseg(size_t n) { return (n + PZ_SEG - 1) / PZ_SEG; }

bool PngZopfli::tokens(const uint8_t *d_filt, size_t n, int bpp, int stride, const uint32_t *d_gtok, const uint32_t *d_gcounts, int gchunk, uint32_t *d_out,
                       void *stream_, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    if (!n || PZ_REGION % gchunk) { err = "png zopfli: bad arguments"; return false; }
    const size_t ns = nseg(n), nreg = (n + PZ_REGION - 1) / PZ_REGION, sl = std::min<size_t>(n, PZ_SLICE), win = sl + PZ_WINDOW;
    const Grow g = Grow::Pow2Quarter;
    size_t sort_tb = 0, scan_tb = 0;
    cub::DeviceRadixSort::SortPairs((void *)nullptr, sort_tb, d_key.get(), d_key2.get(), d_val.get(), d_val2.get(), (int)win, 0, 17, st);
    cub::DeviceScan::ExclusiveSum((void *)nullptr, scan_tb, d_segn.get(), d_offsets.get(), (int)ns, st);
    if (!d_key.reserve(win * 4, g, err) || !d_key2.reserve(win * 4, g, err) || !d_val.reserve(win * 4, g, err) || !d_val2.reserve(win * 4, g, err) ||
        !d_prev.reserve(win * 4, g, err) || !d_ent.reserve(sl * PZ_K * 4, g, err) || !d_bp.reserve(sl * 4, g, err) || !d_tok.reserve(sl * 4, g, err) ||
        !d_best.reserve(n * 4 + 64, g, err) || !d_segc.reserve(ns * 4 + 4, g, err) || !d_segn.reserve(ns * 4 + 4, g, err) || !d_offsets.reserve(ns * 4 + 4, g, err) ||
        !d_hg.reserve(nreg * PZ_NSYM * 4, g, err) || !d_ha.reserve(nreg * PZ_NSYM * 4, g, err) || !d_hb.reserve(nreg * PZ_NSYM * 4, g, err) ||
        !d_cost.reserve(nreg * PZ_NSYM * 4, g, err) || !d_state.reserve(16, g, err) || !d_temp.reserve(std::max(sort_tb, scan_tb) + 256, g, err)) return false;
    CU(cudaMemsetAsync(d_hg, 0, nreg * PZ_NSYM * 4, st));
    k_pz_greedy_hist<<<cdiv(n, gchunk), 256, 0, st>>>(d_gtok, d_gcounts, gchunk, d_hg);
    LT_MARK("k_pz_greedy_hist");
    Cand cand; pz_fixed_sorted(bpp, stride, cand.d);
    for (size_t sl0 = 0; sl0 < n; sl0 += PZ_SLICE) {
        const size_t sl1 = std::min(n, sl0 + PZ_SLICE), ws = sl0 >= PZ_WINDOW ? sl0 - PZ_WINDOW : 0, cnt = sl1 - ws;
        const size_t r0 = sl0 / PZ_REGION, r1 = (sl1 + PZ_REGION - 1) / PZ_REGION, g0 = sl0 / PZ_SEG, g1 = (sl1 + PZ_SEG - 1) / PZ_SEG;
        k_pz_keys<<<cdiv(cnt, 256), 256, 0, st>>>(d_filt, n, ws, cnt, d_key, d_val);
        size_t tb = d_temp.capacity();
        CU(cub::DeviceRadixSort::SortPairs(d_temp.get(), tb, d_key.get(), d_key2.get(), d_val.get(), d_val2.get(), (int)cnt, 0, 17, st));
        k_pz_prev<<<cdiv(cnt, 256), 256, 0, st>>>(d_key2, d_val2, cnt, (long long)ws, d_prev);
        LT_MARK("k_pz_chains");
        k_pz_matches<<<cdiv(sl1 - sl0, 256), 256, 0, st>>>(d_filt, n, sl0, sl1, cand, d_prev, (long long)ws, d_ent);
        LT_MARK("k_pz_matches");
        CU(cudaMemsetAsync(d_state, 0xFF, 8, st));
        uint32_t *hsrc = d_hg, *hdst = d_ha, *hnext = d_hb;
        for (int it = 0; it < PZ_ITERS; it++) {
            k_pz_costs<<<cdiv(r1 - r0, 64), 64, 0, st>>>(hsrc, d_cost, r0, r1);
            LT_MARK("k_pz_costs");
            CU(cudaMemsetAsync(hdst + r0 * PZ_NSYM, 0, (r1 - r0) * PZ_NSYM * 4, st));
            k_pz_squeeze<<<(unsigned)(g1 - g0), 32, 0, st>>>(d_filt, n, sl0, d_ent, d_cost, d_bp, d_tok, d_segc, hdst);
            LT_MARK("k_pz_squeeze");
            k_pz_score<<<1, 256, 0, st>>>(hdst, r0, r1, d_state);
            k_pz_keep<<<(unsigned)(g1 - g0), 256, 0, st>>>(d_tok, d_segc, g0, sl0, d_state, d_best, d_segn);
            LT_MARK("k_pz_score");
            hsrc = hdst; std::swap(hdst, hnext);          // iteration k + 1's costs come from iteration k's histograms
        }
    }
    size_t tb = d_temp.capacity();
    CU(cub::DeviceScan::ExclusiveSum(d_temp.get(), tb, d_segn.get(), d_offsets.get(), (int)ns, st));
    return launch_ok(launch_png_compact(d_best, d_segn, d_offsets, ns, PZ_SEG, d_out, st), "png zopfli compact", err);
}

} // namespace b200
