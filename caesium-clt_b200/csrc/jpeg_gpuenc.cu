// jpeg_gpuenc.cu -- the block-parallel JPEG entropy encoder on the device (SURVEY.md §8f rank 1).  Every pass is a thin
// CUDA wrapper around a body from jpeg_gpuenc_core.h (the same bodies tests/emul/ runs serially on the CPU); the
// cross-block dependencies of jchuff.c / jcphuff.c (DC prediction, EOB runs, buffered correction bits, bit positions,
// 0xFF stuffing) are resolved with prefix scans (CUB DeviceScan -- plumbing, not one of the path's named kernels).
//
// Passes (one launch each for ANY number of images x scans; blockIdx.y = scan):
//   classify + inline-symbol histogram + correction-bit counts -> [max-scan: previous event] [sum-scan: trailing correction bits] ->
//   groups + EOBn histogram -> tables + bits per table -> scan sizes / buffer layout (on the device) | D2H: sizes ->
//   lengths of the sequential interleaved scans' units -> [sum-scan: their bit offsets] -> zero -> emit (single-component scans: CTA
//   runs into a staging arena) -> DC-first interleaved scan (MCU runs into the arena) -> [sum-scan: run offsets] -> place runs -> 0xFF count per chunk of each scan -> layout -> scatter (byte stuffing
//   through shared memory) | D2H: stuffed scans + DHT payloads.  No host wait in between: see "host orchestration".
#include <cuda_runtime.h>
#include <cub/device/device_scan.cuh>
#include <cuda_pipeline.h>
#include <algorithm>
#include <chrono>
#include <cstring>
#include "jpeg_gpuenc.h"
#include "jpeg_gpuenc_stuff_core.h"
#include "stream_wait.h"
#include "launch_timer.h"

namespace b200 {

using namespace ge;

// ---- kernels ------------------------------------------------------------------------------------------------------
// EOB groups of the AC scans, and their EOBn symbols into the scan's AC table histogram: a group of c blocks is one symbol
// (nbits(c) - 1) << 4, so a CTA (one scan: blockIdx.y) counts into 15 shared bins and flushes them once.
__global__ void k_ge_groups(const Scan *__restrict__ scans, const uint32_t *__restrict__ meta, const int *__restrict__ evkey,
                            const int *__restrict__ prev, const uint32_t *__restrict__ tsum, uint32_t *__restrict__ gcount, uint32_t *__restrict__ hist)
{
    __shared__ uint32_t eob[16];
    const Scan s = scans[blockIdx.y];
    if (s.mode != MODE_AC_FIRST && s.mode != MODE_AC_REFINE) return;
    if ((int)(blockIdx.x * blockDim.x) > s.nblocks) return;
    if (threadIdx.x < 16) eob[threadIdx.x] = 0;
    __syncthreads();
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b <= s.nblocks && (b == s.nblocks || meta_event(meta[s.unit_base + b]))) {
        int pg;
        if (b < s.nblocks) pg = prev[s.unit_base + b];
        else { const long long last = s.unit_base + s.nblocks - 1; pg = max(prev[last], evkey[last]); }
        const int pl = pg >= s.unit_base ? (int)(pg - s.unit_base) : -1;
        assign_groups(meta + s.unit_base, tsum + s.unit_base, s.nblocks, pl, b, gcount + s.unit_base,
                      [&](uint32_t c) { atomicAdd(&eob[eob_symbol(c) >> 4], 1u); });
    }
    __syncthreads();
    if (threadIdx.x < 16 && eob[threadIdx.x]) atomicAdd(&hist[((size_t)s.tab_base + 2 + s.tbl[0]) * 256 + (threadIdx.x << 4)], eob[threadIdx.x]);
}

// jchuff.c jpeg_gen_optimal_table with the two minimum searches spread over a warp (ties resolve to the LARGEST index,
// exactly like the sequential `<=` scans); the chain merges and the canonical code assignment stay on lane 0.
// Also the table's share of its scan's size: sum(hist[symbol] * (code length + sym_extra_bits)) into tbits[t].
__global__ void k_ge_tables(const uint32_t *__restrict__ hist, Table *__restrict__ tabs, DhtOut *__restrict__ dht, unsigned long long *__restrict__ tbits)
{
    __shared__ long long freq[257];
    __shared__ int codesize[257], others[257];
    __shared__ uint8_t bits[33];
    const int t = blockIdx.x, lane = threadIdx.x;
    const uint32_t *f = hist + (size_t)t * 256;
    for (int i = lane; i < 257; i += 32) { freq[i] = i < 256 ? (long long)f[i] : 1; codesize[i] = 0; others[i] = -1; }
    if (lane == 0) for (int i = 0; i < 33; i++) bits[i] = 0;
    __syncwarp();
    // argmin over the live entries (freq > 0), ties to the LARGEST index, entries above 10^9 never chosen (jchuff.c's `v = 1000000000L`
    // start value): each lane scans its 9 entries in ascending order, then three warp reductions (REDUX) pick the winner --
    // high word, low word, index -- instead of a five-step shuffle butterfly on (value, index) pairs.
    auto warp_argmin = [&](int exclude) {
        unsigned long long v = 1000000000ULL; int c = -1;
        for (int i = lane; i < 257; i += 32) { const unsigned long long fi = (unsigned long long)freq[i]; if (fi && fi <= v && i != exclude) { v = fi; c = i; } }
        const unsigned hi = (unsigned)(v >> 32), lo = (unsigned)v;
        const unsigned mhi = __reduce_min_sync(0xFFFFFFFFu, hi);
        const unsigned mlo = __reduce_min_sync(0xFFFFFFFFu, hi == mhi ? lo : 0xFFFFFFFFu);
        return __reduce_max_sync(0xFFFFFFFFu, (hi == mhi && lo == mlo) ? c : -1);
    };
    for (;;) {
        const int c1 = warp_argmin(-1);
        const int c2 = c1 < 0 ? -1 : warp_argmin(c1);
        if (c2 < 0) break;
        if (lane == 0) {
            int a = c1, b = c2;
            freq[a] += freq[b]; freq[b] = 0;
            codesize[a]++; while (others[a] >= 0) { a = others[a]; codesize[a]++; }
            others[a] = b;
            codesize[b]++; while (others[b] >= 0) { b = others[b]; codesize[b]++; }
        }
        __syncwarp();
    }
    if (lane == 0) {
        Table &T = tabs[t];
        for (int i = 0; i <= 256; i++) if (codesize[i]) bits[codesize[i] > 32 ? 32 : codesize[i]]++;
        for (int i = 32; i > 16; i--) while (bits[i] > 0) {
            int j = i - 2; while (bits[j] == 0) j--;
            bits[i] -= 2; bits[i - 1]++; bits[j + 1] += 2; bits[j]--;
        }
        int i = 16; while (i > 0 && bits[i] == 0) i--;
        if (i > 0) bits[i]--;
        // symbols sorted by (code length, symbol value): counting sort on the UNLIMITED lengths, as the IJG loop orders them
        int start[34];
        for (int l = 0; l < 34; l++) start[l] = 0;
        for (int s = 0; s <= 255; s++) if (codesize[s]) start[min(codesize[s], 32) + 1]++;
        for (int l = 1; l < 34; l++) start[l] += start[l - 1];
        const int p = start[33];
        for (int s = 0; s <= 255; s++) if (codesize[s]) T.vals[start[min(codesize[s], 32)]++] = (uint8_t)s;
        T.nvals = p;
        for (int k = 0; k < 17; k++) T.bits[k] = bits[k];
        for (int s = 0; s < 256; s++) T.code_len[s] = 0;
        uint32_t code = 0; int k = 0;
        for (int l = 1; l <= 16; l++) { for (int n = 0; n < bits[l]; n++, k++) T.code_len[T.vals[k]] = (code++ << 8) | (uint32_t)l; code <<= 1; }
        DhtOut &D = dht[t];
        D.nvals = p;
        for (int k2 = 0; k2 < 17; k2++) D.bits[k2] = bits[k2];
        for (int k2 = 0; k2 < p; k2++) D.vals[k2] = T.vals[k2];
    }
    __syncwarp();                           // lane 0's code lengths are visible to the warp
    const int kind = (t & 3) >> 1;
    unsigned long long nb = 0;
    for (int i = lane; i < 256; i += 32) if (f[i]) nb += (unsigned long long)f[i] * ((tabs[t].code_len[i] & 0xFFu) + (unsigned)sym_extra_bits(kind, i));
    for (int d = 16; d; d >>= 1) nb += __shfl_xor_sync(0xFFFFFFFFu, nb, d);
    if (lane == 0) tbits[t] = nb;
}

// Sizes on the device: bits per scan (its four tables' bits + its correction bits), then every scan's place in the group's bit
// buffer (word_base) and, for a single-component scan, in the staging arena of its CTA runs (arena_base: a run takes whole words,
// so a scan takes at most its words plus one per run) and its byte count -- what the host
// used to compute between two halves of the pipeline (one stream wait per megabatch less).  The buffers are sized from an ESTIMATE of the output (the input's size for a re-encode);
// if the real sizes do not fit, flags[0] is raised, every scan is given zero length so the back half does nothing, and the host
// re-runs the back half with exact sizes (flags[1] = words needed).  A scan's words are rounded up to a multiple of four, so that
// every scan starts 16-byte aligned for the stuffing passes' group loads.  One warp; scans in chunks of 32.
__global__ void k_ge_scanout(const Scan *__restrict__ scans, int nscans, const unsigned long long *__restrict__ tbits, const uint32_t *__restrict__ corr,
                             uint32_t *__restrict__ total, ScanOut *__restrict__ so, uint32_t words_cap, uint32_t *__restrict__ flags)
{
    const int lane = threadIdx.x;
    uint32_t wbase = 0, abase = 0;
    for (int c0 = 0; c0 < nscans; c0 += 32) {
        const int i = c0 + lane;
        uint32_t tb = 0, na = 0;
        if (i < nscans) {
            tb = (uint32_t)(tbits[4 * i] + tbits[4 * i + 1] + tbits[4 * i + 2] + tbits[4 * i + 3] + corr[i]);
            na = scans[i].nruns ? (tb + 31) / 32 + scans[i].nruns : 0;
        }
        const uint32_t nbytes = (tb + 7) / 8, nw = i < nscans ? ((tb + 31) / 32 + 1 + 3) & ~3u : 0;
        uint32_t wi = nw, ai = na;          // inclusive warp scans
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t a = __shfl_up_sync(0xFFFFFFFFu, wi, d), c = __shfl_up_sync(0xFFFFFFFFu, ai, d);
            if (lane >= d) { wi += a; ai += c; }
        }
        if (i < nscans) {
            total[i] = tb;
            ScanOut o; o.total_bits = tb; o.nbytes = nbytes; o.word_base = wbase + wi - nw; o.arena_base = abase + ai - na;
            so[i] = o;
        }
        wbase += __shfl_sync(0xFFFFFFFFu, wi, 31); abase += __shfl_sync(0xFFFFFFFFu, ai, 31);
    }
    __syncwarp();
    const bool ovf = wbase > words_cap;     // the arena holds words_cap + total_runs words: it fits when the words do
    if (lane == 0) { flags[0] = ovf ? 1u : 0u; flags[1] = wbase; flags[3] = 0; flags[4] = 0; }
    if (ovf) for (int i = lane; i < nscans; i += 32) { so[i].total_bits = 0; so[i].nbytes = 0; so[i].word_base = 0; so[i].arena_base = 0; }
}

// a scan's bit buffer, and for a single-component scan its part of the staging arena (the runs' edge words are ORed)
__global__ void k_ge_zero(const Scan *__restrict__ scans, const ScanOut *__restrict__ so, uint32_t *__restrict__ words, uint32_t *__restrict__ arena)
{
    const ScanOut o = so[blockIdx.y];
    if (!o.total_bits) return;
    const uint32_t n = (o.total_bits + 31) / 32 + 1, nruns = (uint32_t)scans[blockIdx.y].nruns, na = nruns ? n - 1 + nruns : 0;
    uint32_t *w = words + o.word_base, *a = arena + o.arena_base;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < max(n, na); i += gridDim.x * blockDim.x) {
        if (i < n) w[i] = 0;
        if (i < na) a[i] = 0;
    }
}

// ---- block-major passes: one thread per block; the block is read (and its threshold masks built) once per pass and
// serves every scan that visits the block ------------------------------------------------------------------------------------
// A CTA of the block-major passes owns ENC_THREADS consecutive blocks i = row * bw + col of one component: 16 KB of contiguous
// coefficients, staged in shared memory with coalesced 16-byte loads so that the symbol loops read their scattered non-zero
// coefficients from the tile instead of with one dependent global load each.  Rows are 144 bytes apart: the 16-byte reads of a
// quarter warp (eight consecutive blocks at the same offset) then fall on distinct banks.
constexpr int TILE_PITCH = 72;                  // int16 per tile row
typedef int16_t Tile[ENC_THREADS][TILE_PITCH];

// asynchronous copies (cp.async): the 16-byte pieces go to shared memory without passing through registers
__device__ __forceinline__ void stage_tile(Tile &tile, const BlockComp &bc, int i0, int nblk)
{
    const uint4 *src = reinterpret_cast<const uint4 *>(bc.coef + bc.comp_off + (long long)i0 * 64);
    const int n = min(ENC_THREADS, nblk - i0) * 8;                  // 16-byte pieces, 8 per block
#pragma unroll
    for (int k = 0; k < 8; k++) { const int q = threadIdx.x + k * ENC_THREADS; if (q < n) __pipeline_memcpy_async(&tile[q >> 3][(q & 7) * 8], src + q, 16); }
    __pipeline_commit();
}
__device__ __forceinline__ void wait_tile()
{
    __pipeline_wait_prior(0);
    __syncthreads();
}

// The component's scan visits go to shared memory once per CTA: the symbol loops index them with the loop counter, which would
// put a register copy in local memory, and read their fields on every block, which from the descriptors in global memory would
// be one load each.
__device__ __forceinline__ void stage_visits(EncVisit *vis, const BlockComp &bc)
{
    if ((int)threadIdx.x < bc.nscan) vis[threadIdx.x] = bc.visit[threadIdx.x];
}
// block (row, col) in the scan of visit v: blk = the block in the CTA's shared tile; the DC predecessor of a DC-coding scan is
// read from the tile when it is one of the CTA's blocks, from global memory otherwise
__device__ __forceinline__ BlockRef ref_of(const EncVisit &v, const BlockComp &bc, const Tile &tile, int i0, int row, int col)
{
    BlockRef r;
    r.blk = tile[threadIdx.x]; r.prev = nullptr; r.slot = 0;
    if (v.mode == MODE_SEQ || v.mode == MODE_DC_FIRST) {
        const int p = enc_dc_prev(bc, v.ns, row, col);
        if (p >= i0 && p < i0 + ENC_THREADS) r.prev = tile[p - i0];
        else if (p >= 0) r.prev = bc.coef + bc.comp_off + (long long)p * 64;
    }
    return r;
}

// symbol counters / code words of the visit's two table kinds in the on-chip table layout
template <class T>
__device__ __forceinline__ KindTabs<T> kind_tabs(T *tab, const EncVisit &v) { return KindTabs<T>{tab + ENC_DC_ENTRY, tab + v.ac_entry}; }

// The classify pass builds each block's threshold masks once and leaves them in `masks` (24 bytes per block, indexed
// comp.mask_base + block); the length and emit passes read them back instead of re-deriving them from the 128-byte block (the
// mask construction was a quarter to a third of those passes' instructions).
__device__ __forceinline__ Masks3 load_masks(const Masks3 *__restrict__ masks, const BlockComp &bc, int i)
{
    const unsigned long long *q = reinterpret_cast<const unsigned long long *>(masks + bc.mask_base + i);   // 24-byte records
    Masks3 M;
    M.m[0] = __ldg(q); M.m[1] = __ldg(q + 1); M.m[2] = __ldg(q + 2);
    return M;
}

// Classify + the statistics of the inline symbols (DC differences, run/size symbols, ZRLs: they do not depend on the EOB
// groups; k_ge_groups adds the EOBn symbols), counted into the on-chip table slots of the CTA's visits and flushed once.
struct SmemHist {
    KindTabs<uint32_t> h;
    __device__ void sym(int kind, int, int symbol, int, unsigned) { atomicAdd((kind ? h.ac : h.dc) + symbol, 1u); }
    __device__ void raw64(int, unsigned long long) {}
};
// Also each refinement scan's correction bits (corr[scan]), the one part of a scan's size that is not in its histograms.
// And, for a script with a DC-first interleaved scan, each block's DC coefficient into the compact DC array (dc != nullptr; component
// at mask_base, entries in MCU order: enc_dc_index) that k_geb_dc_first codes from.
__global__ void __launch_bounds__(ENC_THREADS) k_geb_classify(const BlockComp *__restrict__ comps, uint32_t *__restrict__ meta, int *__restrict__ evkey,
                                                              uint32_t *__restrict__ tail, Masks3 *__restrict__ masks, uint32_t *__restrict__ hist, uint32_t *__restrict__ corr,
                                                              int16_t *__restrict__ dc)
{
    __shared__ __align__(16) Tile tile;
    __shared__ uint32_t h[ENC_TAB_ENTRIES];
    __shared__ EncVisit vis[ENC_MAX_VISITS];
    __shared__ uint32_t vcorr[ENC_MAX_VISITS];
    const BlockComp &bc = comps[blockIdx.y];
    const int nblk = bc.bw * bc.bh, i0 = blockIdx.x * ENC_THREADS, i = i0 + threadIdx.x;
    if (i0 >= nblk) return;
    stage_tile(tile, bc, i0, nblk);
    for (int k = threadIdx.x; k < ENC_TAB_ENTRIES; k += ENC_THREADS) h[k] = 0;
    if (threadIdx.x < ENC_MAX_VISITS) vcorr[threadIdx.x] = 0;
    stage_visits(vis, bc);
    wait_tile();
    if (i < nblk) {
        const int row = i / bc.bw, col = i - row * bc.bw;
        const Masks3 M = make_masks3(tile[threadIdx.x]);
        masks[bc.mask_base + i] = M;
        if (dc) dc[bc.mask_base + enc_dc_index(bc, row, col)] = tile[threadIdx.x][0];
        for (int j = 0; j < bc.nscan; j++) {
            const EncVisit &v = vis[j];
            const int u = enc_unit_of(bc, v.ns, row, col);
            if (u < 0) continue;
            const uint32_t m = classify_m(v, M);
            const int g = v.unit_base + u;
            meta[g] = m; evkey[g] = meta_event(m) ? g : -1; tail[g] = (uint32_t)meta_tail(m);
            SmemHist sk{kind_tabs(h, v)};
            gen_block_m(v, v.tbl, ref_of(v, bc, tile, i0, row, col), M, 0, sk);
            const int nc = corr_bits_m(v, M);
            if (nc) atomicAdd(&vcorr[j], (uint32_t)nc);
        }
    }
    __syncthreads();
    if ((int)threadIdx.x < bc.nscan && vcorr[threadIdx.x]) atomicAdd(&corr[vis[threadIdx.x].scan], vcorr[threadIdx.x]);
    for (int k = threadIdx.x; k < ENC_TAB_ENTRIES; k += ENC_THREADS) {
        int symbol; const int t = enc_entry_table(bc, k, symbol);
        if (h[k]) atomicAdd(&hist[(size_t)t * 256 + symbol], h[k]);     // an unused slot counts nothing
    }
}

// The length and emit passes load the tables of the CTA's visits once (k_ge_tables wrote them): the per-symbol lookup on the
// symbol's dependent chain is a shared-memory read.  len keeps the code lengths only.
// len runs over the visits of interleaved scans (ns > 1) only: the blocks of a CTA are not consecutive units there, so emit needs
// every unit's bit offset.
__global__ void __launch_bounds__(ENC_THREADS) k_geb_len(const BlockComp *__restrict__ comps, const uint32_t *__restrict__ gcount, const Table *__restrict__ tabs,
                                                         uint32_t *__restrict__ bitlen, const Masks3 *__restrict__ masks)
{
    __shared__ __align__(16) Tile tile;
    __shared__ uint8_t tl[ENC_TAB_ENTRIES];
    __shared__ EncVisit vis[ENC_MAX_VISITS];
    const BlockComp &bc = comps[blockIdx.y];
    const int nblk = bc.bw * bc.bh, i0 = blockIdx.x * ENC_THREADS, i = i0 + threadIdx.x;
    if (i0 >= nblk) return;
    stage_tile(tile, bc, i0, nblk);
    const Masks3 M = load_masks(masks, bc, min(i, nblk - 1));   // in flight with the tile
    stage_visits(vis, bc);
    for (int k = threadIdx.x; k < ENC_TAB_ENTRIES; k += ENC_THREADS) {
        int symbol; const int t = enc_entry_table(bc, k, symbol);
        if (t >= 0) tl[k] = (uint8_t)tabs[t].code_len[symbol];
    }
    wait_tile();
    if (i >= nblk) return;
    const int row = i / bc.bw, col = i - row * bc.bw;
    for (int j = 0; j < bc.nscan; j++) {
        const EncVisit &v = vis[j];
        if (v.ns == 1) continue;
        const int u = enc_unit_of(bc, v.ns, row, col);
        if (u < 0) continue;
        LenSinkT<KindTabs<const uint8_t>> sk{kind_tabs<const uint8_t>(tl, v)};
        gen_block_m(v, v.tbl, ref_of(v, bc, tile, i0, row, col), M, gcount[v.unit_base + u], sk);
        bitlen[v.lu_base + u] = (uint32_t)sk.bits;
    }
}
// exclusive prefix sum of x over the CTA, and the CTA's total; every thread calls it (it has a barrier)
__device__ __forceinline__ uint32_t cta_exclusive_sum(uint32_t x, uint32_t *wsum /*ENC_THREADS / 32*/, uint32_t &total)
{
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t inc = x;
    for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, inc, d); if (lane >= d) inc += y; }
    if (lane == 31) wsum[w] = inc;
    __syncthreads();
    uint32_t base = 0, tot = 0;
#pragma unroll
    for (int k = 0; k < ENC_THREADS / 32; k++) { const uint32_t sk = wsum[k]; if (k < w) base += sk; tot += sk; }
    total = tot;
    return base + inc - x;
}

// Emit.  A visit of a sequential interleaved scan writes each unit at the bit offset k_geb_len's lengths gave it (a DC-first
// interleaved scan is k_geb_dc_first's).  A visit of a single-component
// scan codes its units once for length and bits together: the CTA's units are consecutive units of the scan, so their offsets inside
// the CTA's run follow from the lengths, and the run's place in the scan from the other runs' lengths (k_ge_place):
//   - each thread codes its unit into its slot of ENC_SLOT_WORDS words in shared memory, counting bits past the slot's end;
//   - a CTA-wide prefix sum gives each unit's offset in the run and the run's length;
//   - the run takes its words in the scan's part of the staging arena (a per-scan counter: the order of the runs in the arena does
//     not matter, k_ge_place finds each through runpos), and each unit is copied there from its slot -- or, when it overflowed the
//     slot, coded a second time straight to its place.
constexpr int ENC_SLOT_WORDS = 8;
__global__ void __launch_bounds__(ENC_THREADS) k_geb_emit(const BlockComp *__restrict__ comps, const uint32_t *__restrict__ gcount, const Table *__restrict__ tabs,
                                                          const uint32_t *__restrict__ bitoff, uint32_t *__restrict__ words, const Masks3 *__restrict__ masks, const ScanOut *__restrict__ so,
                                                          const uint32_t *__restrict__ flags, uint32_t *__restrict__ arena, uint32_t *__restrict__ cursor,
                                                          uint32_t *__restrict__ runlen, uint32_t *__restrict__ runpos)
{
    __shared__ __align__(16) Tile tile;
    __shared__ uint32_t tc[ENC_TAB_ENTRIES];
    __shared__ EncVisit vis[ENC_MAX_VISITS];
    __shared__ uint32_t vword[ENC_MAX_VISITS], vbit0[ENC_MAX_VISITS];     // interleaved scan: first word, bit offset of unit 0; else arena base
    __shared__ uint32_t slot[ENC_SLOT_WORDS][ENC_THREADS];                // word-major: a warp's stores to its slots hit 32 banks
    __shared__ uint32_t wsum[ENC_THREADS / 32], run_word;
    if (flags[0]) return;                   // the bit buffer is too small for this batch: the host re-runs this half with exact sizes
    const BlockComp &bc = comps[blockIdx.y];
    const int nblk = bc.bw * bc.bh, i0 = blockIdx.x * ENC_THREADS, i = i0 + threadIdx.x;
    if (i0 >= nblk) return;
    const bool live = i < nblk;
    stage_tile(tile, bc, i0, nblk);
    const Masks3 M = load_masks(masks, bc, min(i, nblk - 1));   // in flight with the tile
    stage_visits(vis, bc);
    if ((int)threadIdx.x < bc.nscan) {
        const EncVisit &v = bc.visit[threadIdx.x];
        const ScanOut &o = so[v.scan];
        const bool unit = v.ns > 1 && v.mode != MODE_DC_FIRST;
        vword[threadIdx.x] = unit ? o.word_base : o.arena_base; vbit0[threadIdx.x] = unit ? bitoff[v.lu_base] : 0;
    }
    for (int k = threadIdx.x; k < ENC_TAB_ENTRIES; k += ENC_THREADS) {
        int symbol; const int t = enc_entry_table(bc, k, symbol);
        if (t >= 0) tc[k] = tabs[t].code_len[symbol];
    }
    wait_tile();
    const int row = i / bc.bw, col = i - row * bc.bw;
    auto orw = [&](long long w, uint32_t v) { if (v) atomicOr(&words[w], v); };
    auto stw = [&](long long w, uint32_t v) { words[w] = v; };
    auto ora = [&](long long w, uint32_t v) { if (v) atomicOr(&arena[w], v); };
    auto sta = [&](long long w, uint32_t v) { arena[w] = v; };
    auto sls = [&](long long w, uint32_t v) { if (w < ENC_SLOT_WORDS) slot[w][threadIdx.x] = v; };
    typedef KindTabs<const uint32_t> KT;
    for (int j = 0; j < bc.nscan; j++) {                        // v.ns is the same for the whole CTA: the barriers below are uniform
        const EncVisit &v = vis[j];
        const int u = live ? enc_unit_of(bc, v.ns, row, col) : -1;
        if (v.ns > 1) {
            if (u < 0 || v.mode == MODE_DC_FIRST) continue;
            EmitSink<decltype(orw), decltype(stw), KT> sk(kind_tabs<const uint32_t>(tc, v), orw, stw, (long long)vword[j], (unsigned long long)(bitoff[v.lu_base + u] - vbit0[j]));
            gen_block_m(v, v.tbl, ref_of(v, bc, tile, i0, row, col), M, gcount[v.unit_base + u], sk);
            sk.finish();
            continue;
        }
        uint32_t nb = 0;
        if (u >= 0) {
            EmitSink<decltype(sls), decltype(sls), KT> sk(kind_tabs<const uint32_t>(tc, v), sls, sls, 0, 0);
            gen_block_m(v, v.tbl, ref_of(v, bc, tile, i0, row, col), M, gcount[v.unit_base + u], sk);
            sk.finish();
            nb = (uint32_t)sk.bits_written(0);
        }
        uint32_t L;
        const uint32_t off = cta_exclusive_sum(nb, wsum, L);
        if (threadIdx.x == 0) {
            const uint32_t a = vword[j] + atomicAdd(&cursor[v.scan], (L + 31) / 32);
            run_word = a; runlen[v.run_base + blockIdx.x] = L; runpos[v.run_base + blockIdx.x] = a;
        }
        __syncthreads();
        const unsigned long long at = (unsigned long long)run_word * 32 + off;
        if (nb <= ENC_SLOT_WORDS * 32) place_bits([&](long long k) { return slot[k][threadIdx.x]; }, nb, at, ora, sta);
        else {                              // rare: the unit overflowed its slot
            EmitSink<decltype(ora), decltype(sta), KT> sk(kind_tabs<const uint32_t>(tc, v), ora, sta, 0, at);
            gen_block_m(v, v.tbl, ref_of(v, bc, tile, i0, row, col), M, gcount[v.unit_base + u], sk);
            sk.finish();
        }
    }
}

// The DC-first scan with ns > 1 (the progressive script's first scan): one thread per MCU, whose units are consecutive in the scan,
// coded from the compact DC array (gen_dc_mcu) into the thread's slot; then the CTA's run into the arena as k_geb_emit does for a
// single-component visit.  A 4:2:0 MCU is six units of ~6 bits; the largest (10 blocks of 16 + 11 bits) overflows the slot and is
// coded a second time straight to its place.  Grid (MCU runs, images): the scan is script entry `k` of every image.  The minimum of one
// CTA per SM in the launch bounds keeps ptxas from capping the kernel at 32 registers, where it spills.
__global__ void __launch_bounds__(ENC_DC_MCUS, 1) k_geb_dc_first(const Scan *__restrict__ scans, int spi, int k, const int16_t *__restrict__ dc,
                                                              const Table *__restrict__ tabs, const ScanOut *__restrict__ so, const uint32_t *__restrict__ flags,
                                                              uint32_t *__restrict__ arena, uint32_t *__restrict__ cursor, uint32_t *__restrict__ runlen,
                                                              uint32_t *__restrict__ runpos)
{
    static_assert(ENC_DC_MCUS == ENC_THREADS, "cta_exclusive_sum sums ENC_THREADS lanes");
    __shared__ uint32_t tc[2 * ENC_DC_SYMBOLS];                         // DC code words of table ids 0 and 1
    __shared__ uint32_t slot[ENC_SLOT_WORDS][ENC_DC_MCUS];
    __shared__ uint32_t wsum[ENC_DC_MCUS / 32], run_word;
    if (flags[0]) return;
    const int si = blockIdx.y * spi + k;
    const Scan &s = scans[si];
    const int nmcu = s.mcux * s.mcuy, m = blockIdx.x * ENC_DC_MCUS + threadIdx.x;
    if ((int)(blockIdx.x * ENC_DC_MCUS) >= nmcu) return;
    if (threadIdx.x < 2 * ENC_DC_SYMBOLS) tc[threadIdx.x] = tabs[s.tab_base + threadIdx.x / ENC_DC_SYMBOLS].code_len[threadIdx.x % ENC_DC_SYMBOLS];
    __syncthreads();
    struct DcTabs { const uint32_t *t; __device__ uint32_t operator()(int, int tbl, int symbol) const { return t[tbl * ENC_DC_SYMBOLS + symbol]; } };
    auto sls = [&](long long w, uint32_t v) { if (w < ENC_SLOT_WORDS) slot[w][threadIdx.x] = v; };
    auto ora = [&](long long w, uint32_t v) { if (v) atomicOr(&arena[w], v); };
    auto sta = [&](long long w, uint32_t v) { arena[w] = v; };
    uint32_t nb = 0;
    if (m < nmcu) {
        EmitSink<decltype(sls), decltype(sls), DcTabs> sk(DcTabs{tc}, sls, sls, 0, 0);
        gen_dc_mcu(s, dc, m, sk);
        sk.finish();
        nb = (uint32_t)sk.bits_written(0);
    }
    uint32_t L;
    const uint32_t off = cta_exclusive_sum(nb, wsum, L);
    if (threadIdx.x == 0) {
        const uint32_t a = so[si].arena_base + atomicAdd(&cursor[si], (L + 31) / 32);
        run_word = a; runlen[s.run_base + blockIdx.x] = L; runpos[s.run_base + blockIdx.x] = a;
    }
    __syncthreads();
    const unsigned long long at = (unsigned long long)run_word * 32 + off;
    if (nb <= ENC_SLOT_WORDS * 32) place_bits([&](long long w) { return slot[w][threadIdx.x]; }, nb, at, ora, sta);
    else {                                  // rare: the MCU overflowed its slot
        EmitSink<decltype(ora), decltype(sta), DcTabs> sk(DcTabs{tc}, ora, sta, 0, at);
        gen_dc_mcu(s, dc, m, sk);
        sk.finish();
    }
}

// Runs (of the single-component scans and of the DC-first interleaved scan) to their place in the scan's bit buffer: run r of scan y starts runoff[r] - runoff[first run]
// bits into the scan (an exclusive sum over the run lengths); one warp per run, funnel-shifting the run's whole arena words.
constexpr int PLACE_THREADS = 128;
__global__ void __launch_bounds__(PLACE_THREADS) k_ge_place(const Scan *__restrict__ scans, const ScanOut *__restrict__ so, const uint32_t *__restrict__ runlen,
                                                            const uint32_t *__restrict__ runoff, const uint32_t *__restrict__ runpos, const uint32_t *__restrict__ arena,
                                                            uint32_t *__restrict__ words, const uint32_t *__restrict__ flags)
{
    if (flags[0]) return;
    const int nruns = scans[blockIdx.y].nruns, x = blockIdx.x * (PLACE_THREADS / 32) + (threadIdx.x >> 5);
    if (x >= nruns) return;
    const int r0 = scans[blockIdx.y].run_base, r = r0 + x;
    const uint32_t *src = arena + runpos[r];
    uint32_t *dst = words + so[blockIdx.y].word_base;
    place_bits([&](long long k) { return src[k]; }, runlen[r], runoff[r] - runoff[r0],
               [&](long long w, uint32_t v) { atomicOr(&dst[w], v); }, [&](long long w, uint32_t v) { dst[w] = v; }, threadIdx.x & 31, 32);
}

// ---- 0xFF stuffing: the bodies are in jpeg_gpuenc_stuff_core.h --------------------------------------------------------------
// Grid (STUFF_CHUNKS, nscans) for both k_ge_ffcount and k_ge_scatter: CTA x of scan y owns chunk x of the scan's 16-byte groups
// (stuff_chunk: whole tiles of STUFF_THREADS groups) and walks it a tile at a time, one 16-byte load per thread and tile.
constexpr int STUFF_THREADS = ENC_THREADS;      // groups per tile (the CTA prefix sum is cta_exclusive_sum's)
constexpr int STUFF_CHUNKS = 32;                // CTAs per scan
static_assert(STUFF_CHUNKS <= STUFF_THREADS, "k_ge_scatter sums the chunks before its own with one thread each");
__device__ __forceinline__ ScanGroup load_scan_group(const uint32_t *w, uint32_t g) { const uint4 q = reinterpret_cast<const uint4 *>(w)[g]; return ScanGroup{{q.x, q.y, q.z, q.w}}; }

// 0xFF bytes per chunk: chunkff[y * STUFF_CHUNKS + x] (every CTA writes its entry, an empty chunk 0)
__global__ void __launch_bounds__(STUFF_THREADS) k_ge_ffcount(const ScanOut *__restrict__ so, const uint32_t *__restrict__ words, uint32_t *__restrict__ chunkff)
{
    __shared__ uint32_t wsum[STUFF_THREADS / 32];
    const ScanOut o = so[blockIdx.y];
    const uint32_t *w = words + o.word_base;
    uint32_t g0, g1;
    stuff_chunk(o.nbytes, blockIdx.x, STUFF_CHUNKS, STUFF_THREADS, g0, g1);
    uint32_t n = 0;
    for (uint32_t g = g0 + threadIdx.x; g < g1; g += STUFF_THREADS) {
        ScanGroup q = load_scan_group(w, g);
        stuff_group(q, g, o.nbytes, o.total_bits);
        n += stuff_ff_count(q);
    }
    uint32_t total;
    cta_exclusive_sum(n, wsum, total);
    if (threadIdx.x == 0) chunkff[blockIdx.y * STUFF_CHUNKS + blockIdx.x] = total;
}

// One CTA per image: lay its scans out back to back in the image's output region (a scan's stuffed length is its bytes plus its
// chunks' 0xFF counts; warp k sums scan k's); out_off / out_len per scan; an image that outgrows its region raises flags[4] (and
// flags[3] = the largest image size seen, so the host can size the retry)
constexpr int LAYOUT_THREADS = 256;
__global__ void __launch_bounds__(LAYOUT_THREADS) k_ge_layout(const ScanOut *__restrict__ so, int scans_per_image, const uint32_t *__restrict__ chunkff,
                                                              uint32_t *__restrict__ out_off, uint32_t *__restrict__ out_len, uint32_t out_image_stride, uint32_t *__restrict__ flags)
{
    extern __shared__ uint32_t slen[];      // scans_per_image
    const int lane = threadIdx.x & 31, s0 = blockIdx.x * scans_per_image;
    for (int k = threadIdx.x >> 5; k < scans_per_image; k += LAYOUT_THREADS / 32) {
        uint32_t ff = 0;
        for (int x = lane; x < STUFF_CHUNKS; x += 32) ff += chunkff[(s0 + k) * STUFF_CHUNKS + x];
        ff = __reduce_add_sync(0xFFFFFFFFu, ff);
        if (lane == 0) slen[k] = so[s0 + k].nbytes + ff;
    }
    __syncthreads();
    if (threadIdx.x) return;
    uint32_t off = 0;
    for (int k = 0; k < scans_per_image; k++) { out_off[s0 + k] = off; out_len[s0 + k] = slen[k]; off += slen[k]; }
    atomicMax(&flags[3], off);
    if (off > out_image_stride) atomicOr(&flags[4], 1u);
}

// The chunk's output starts after its groups' bytes before it and the 0xFF bytes of the chunks before it.  Per tile: each thread
// re-reads its group, a CTA prefix sum over the stuffed lengths gives its place, the bytes are stuffed into shared memory at the
// output's word alignment and leave as aligned 4-byte stores, coalesced across the CTA (stuff_store); the next tile starts where
// this one ended.
__global__ void __launch_bounds__(STUFF_THREADS) k_ge_scatter(const ScanOut *__restrict__ so, const uint32_t *__restrict__ words, const uint32_t *__restrict__ chunkff,
                                                              const uint32_t *__restrict__ out_off, uint8_t *__restrict__ out, int scans_per_image, size_t out_image_stride,
                                                              const uint32_t *__restrict__ flags)
{
    __shared__ uint32_t sbuf[STUFF_THREADS * 8 + 1];       // a tile of 0xFF bytes stuffs to 32 bytes a group, after up to 3 bytes of alignment
    __shared__ uint32_t wsum[STUFF_THREADS / 32];
    if (flags[4]) return;                   // some image does not fit its output region: nothing is written, the host retries
    const ScanOut o = so[blockIdx.y];
    uint32_t g0, g1;
    stuff_chunk(o.nbytes, blockIdx.x, STUFF_CHUNKS, STUFF_THREADS, g0, g1);
    if (g0 >= g1) return;
    const uint32_t *w = words + o.word_base;
    uint8_t *img = out + (size_t)(blockIdx.y / scans_per_image) * out_image_stride, *sb = reinterpret_cast<uint8_t *>(sbuf);
    uint32_t ff_before;
    cta_exclusive_sum(threadIdx.x < blockIdx.x ? chunkff[blockIdx.y * STUFF_CHUNKS + threadIdx.x] : 0u, wsum, ff_before);
    uint32_t at = out_off[blockIdx.y] + g0 * 16 + ff_before;
    for (uint32_t t0 = g0; t0 < g1; t0 += STUFF_THREADS) {
        const uint32_t g = t0 + threadIdx.x;
        ScanGroup q;
        uint32_t n = 0, len = 0;
        if (g < g1) { q = load_scan_group(w, g); n = stuff_group(q, g, o.nbytes, o.total_bits); len = n + stuff_ff_count(q); }
        __syncthreads();                    // the previous tile's wsum / sbuf reads are done
        uint32_t L;
        const uint32_t rel = cta_exclusive_sum(len, wsum, L), aligned = at & ~3u;
        if (n) stuff_place_group(q, n, at - aligned + rel, sb);
        __syncthreads();
        stuff_store(sbuf, aligned, at, at + L, threadIdx.x, STUFF_THREADS, img);
        at += L;
    }
}

// dummy blocks of partial MCUs (jccoefct.c / jctrans.c rule, jpeg_fill_dummy_blocks on the host): AC = 0, DC copied
__global__ void k_ge_fill_dummy(int16_t *__restrict__ coef, long long comp_off, int bw, int bh, int rbw, int rbh, int hs)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= bw * bh) return;
    const int row = i / bw, col = i - row * bw;
    if (row < rbh && col < rbw) return;
    int r = row, c = col;
    while (r >= rbh || c >= rbw) { if (r >= rbh) { c = (c / hs) * hs + hs - 1; r--; } else c = rbw - 1; }
    int16_t *base = coef + comp_off;
    int16_t *dst = base + ((long long)row * bw + col) * 64;
    const int16_t dc = base[((long long)r * bw + c) * 64];
    for (int k = 1; k < 64; k++) dst[k] = 0;
    dst[0] = dc;
}

// ---- host orchestration ---------------------------------------------------------------------------------------------
// Three steps so that a megabatch costs the host one wait that overlaps device work plus the final one, and so that a caller with
// everything resident in HBM (bench.py's device-only figure) can enqueue the whole pass sequence without any wait:
//   prepare()  plan + buffers (sized from an estimate of the output) + H2D of the descriptors
//   enqueue()  every kernel; D2H of the sizes right after the tables (event), D2H of DHT payloads / stuffed lengths at the end
//   finish()   wait for the sizes (the emit / stuffing kernels are still running), size and enqueue the D2H of the stuffed scans,
//              final wait; a batch that outgrew the estimate re-runs the back half with exact sizes
static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

GpuEncoder::~GpuEncoder()
{
    if (ev_sizes) cudaEventDestroy((cudaEvent_t)ev_sizes);
}

// Sizes here depend on image CONTENT (bytes of entropy-coded output): Grow::Pow2Half rounds up to a power of two with headroom so a
// slot stops reallocating after its first image of a given class (cudaFree / cudaHostAlloc stall every stream).
bool GpuEncoder::size_back_buffers(size_t image_bytes, std::string &err)
{   // everything whose size follows the OUTPUT: bit buffer, stuffed bytes
    const int NS = (int)plan.scans.size();
    // capacities only grow (per image count): they are kernel arguments of the launch sequence, and a sequence whose arguments do
    // not change from megabatch to megabatch can be replayed as a CUDA graph
    auto grow = [&](auto &buf, size_t need) { return buf.reserve(need, Grow::Pow2Half, err, &generation); };
    // the staging arena of the single-component scans' runs: at most the scans' words plus one per run (k_ge_scanout)
    auto grow_arena = [&]() { return grow(d_arena, ((size_t)words_cap + (size_t)plan.total_runs) * 4 + 64); };
    if (nimg != cap_nimg) { cap_nimg = nimg; est_image_bytes = 0; }
    if (image_bytes <= est_image_bytes && words_cap) return grow_arena();
    est_image_bytes = image_bytes + image_bytes / 8;
    image_bytes = est_image_bytes;
    // a scan takes its bits' words, one more, and up to three to round its words to a multiple of four (k_ge_scanout)
    words_cap = (uint32_t)std::min<size_t>((size_t)nimg * (image_bytes / 4 + 1) + 5 * (size_t)NS + 64, 0xFFFFFF00u);
    out_stride = align_up(image_bytes + image_bytes / 8 + 1024, 256);
    return grow_arena() && grow(d_words, (size_t)words_cap * 4 + 64) && grow(d_out, out_stride * nimg);
}

bool GpuEncoder::prepare(const JpegGeom &g, bool progressive, int16_t *const *d_coefs, int nimages, void *stream_, size_t out_bytes_hint, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    geom = g; prog = progressive;
    std::vector<const int16_t *> bases(d_coefs, d_coefs + nimages);
    coef_bases.assign(d_coefs, d_coefs + nimages);
    gpuenc_plan(g, progressive, bases.data(), nimages, plan);
    nimg = nimages;
    const int NS = (int)plan.scans.size();
    const long long U = plan.total_units, LU = plan.unit_coded ? std::max(plan.total_lunits, 1ll) : 1;
    const int R = std::max(plan.total_runs, 1);
    if (U >= (1ll << 31)) { err = "batch too large for the entropy encoder"; return false; }
    overflow = false;
    for (auto &sc_ : plan.scans) if (!masks_cover(sc_.mode, sc_.Al)) { err = "scan script outside the device encoder's mask range"; overflow = true; return false; }
    if (!plan.on_chip) { err = "scan script outside the device encoder's on-chip table slots"; overflow = true; return false; }
    if (!ev_sizes) { cudaEvent_t e; CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming | (stream_wait_mode() == 0 ? 0 : cudaEventBlockingSync))); ev_sizes = e; }
    // ---- buffers whose size follows the INPUT
    auto grow = [&](auto &buf, size_t need) { return buf.reserve(need, Grow::Pow2Half, err, &generation); };
    const int NC = (int)plan.comps.size();
    if (!grow(d_scans, NS * sizeof(Scan)) || !grow(d_comps, NC * sizeof(BlockComp)) ||
        !grow(d_meta, U * 4) || !grow(d_evkey, U * 4) || !grow(d_prev, U * 4) || !grow(d_tail, U * 4) || !grow(d_tsum, U * 4) ||
        !grow(d_gcount, U * 4) || !grow(d_bitlen, LU * 4) || !grow(d_bitoff, LU * 4) || !grow(d_corr, (size_t)NS * 4) || !grow(d_tbits, (size_t)NS * 4 * 8) ||
        !grow(d_cursor, (size_t)NS * 4) || !grow(d_runlen, (size_t)R * 4) || !grow(d_runoff, (size_t)R * 4) || !grow(d_runpos, (size_t)R * 4) ||
        !grow(d_hist, (size_t)NS * 4 * 256 * 4) || !grow(d_tabs, (size_t)NS * 4 * sizeof(Table)) || !grow(d_dht, (size_t)NS * 4 * sizeof(DhtOut)) ||
        !grow(d_total, (size_t)NS * 4) || !grow(d_so, (size_t)NS * sizeof(ScanOut)) || !grow(d_outoff, (size_t)NS * 4) || !grow(d_outlen, (size_t)NS * 4) ||
        !grow(d_flags, 64) || !grow(d_masks, (size_t)plan.total_comp_blocks * sizeof(Masks3)) || !grow(d_dc, (size_t)plan.total_comp_blocks * 2) || !grow(d_chunkff, (size_t)NS * STUFF_CHUNKS * 4)) return false;
    o_scans = 0; o_total = o_scans + align_up((size_t)NS * sizeof(Scan), 256); o_outlen = o_total + align_up((size_t)NS * 4, 256);
    o_dht = o_outlen + align_up((size_t)NS * 4, 256); o_comps = o_dht + align_up((size_t)NS * 4 * sizeof(DhtOut), 256);
    o_flags = o_comps + align_up((size_t)NC * sizeof(BlockComp), 256);
    const size_t small_bytes = o_flags + 256;
    if (!grow(h_small, small_bytes)) return false;
    size_t tb1 = 0, tb2 = 0, tb3 = 0, tb4 = 0;
    cub::DeviceScan::ExclusiveScan((void *)nullptr, tb1, d_evkey.get(), d_prev.get(), cub::Max(), -1, (int)U, st);
    cub::DeviceScan::ExclusiveSum((void *)nullptr, tb2, d_tail.get(), d_tsum.get(), (int)U, st);
    cub::DeviceScan::ExclusiveSum((void *)nullptr, tb3, d_bitlen.get(), d_bitoff.get(), (int)LU, st);
    cub::DeviceScan::ExclusiveSum((void *)nullptr, tb4, d_runlen.get(), d_runoff.get(), R, st);
    if (!grow(d_temp, std::max(std::max(tb1, tb2), std::max(tb3, tb4)) + 256)) return false;
    // ---- buffers whose size follows the OUTPUT: estimate now, exact on a retry.  A re-encode at lower quality does not grow, so
    // the caller's hint is the input's entropy-coded size; without a hint a third of the coefficient bytes (~ 1 byte / pixel).
    const size_t coef_bytes = (size_t)g.total_coefs * 2;
    if (coef_bytes != learned_for) { learned_for = coef_bytes; learned_image_bytes = 0; }
    size_t est = out_bytes_hint ? out_bytes_hint / nimages + out_bytes_hint / nimages / 4 : coef_bytes / 3;
    est = std::max(est, learned_image_bytes + learned_image_bytes / 8) + 8192;
    est = std::min(est, coef_bytes * 2 + (size_t)plan.scans_per_image * 64 + 8192);      // worst case: 128 B per block and scan... bounded by the retry anyway
    if (!size_back_buffers(est, err)) return false;
    memcpy(h_small + o_scans, plan.scans.data(), NS * sizeof(Scan));
    memcpy(h_small + o_comps, plan.comps.data(), NC * sizeof(BlockComp));
    (void)st;
    return true;
}

bool GpuEncoder::upload(void *stream_, std::string &err)
{   // H2D of the scan / component descriptors prepare() wrote into pinned memory
    cudaStream_t st = (cudaStream_t)stream_;
    const int NS = (int)plan.scans.size(), NC = (int)plan.comps.size();
    CU(cudaMemcpyAsync(d_scans, h_small + o_scans, NS * sizeof(Scan), cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_comps, h_small + o_comps, NC * sizeof(BlockComp), cudaMemcpyHostToDevice, st));
    return true;
}

unsigned long long GpuEncoder::signature() const
{   // everything upload() + enqueue_front() + enqueue_sizes() + enqueue_back() bake into their driver calls
    unsigned long long h = 1469598103934665603ull;
    auto mix = [&](unsigned long long v) { h = (h ^ v) * 1099511628211ull; };
    mix((unsigned long long)nimg); mix((unsigned long long)plan.scans.size()); mix((unsigned long long)plan.comps.size()); mix((unsigned long long)plan.total_units);
    mix((unsigned long long)plan.max_comp_blocks); mix((unsigned long long)plan.scans_per_image); mix(words_cap); mix(out_stride); mix(generation);
    mix((unsigned long long)geom.width); mix((unsigned long long)geom.height); mix(prog ? 1 : 0);
    for (int c = 0; c < geom.ncomp; c++) { mix((unsigned long long)geom.bw[c]); mix((unsigned long long)geom.bh[c]); mix((unsigned long long)geom.rbw[c]); mix((unsigned long long)geom.rbh[c]); mix((unsigned long long)geom.hs[c]); }
    for (auto pb : coef_bases) mix((unsigned long long)(uintptr_t)pb);
    int max_units = 0; for (auto &sc : plan.scans) max_units = std::max(max_units, sc.nblocks);
    mix((unsigned long long)max_units);
    mix((unsigned long long)plan.total_lunits); mix((unsigned long long)plan.total_runs); mix((unsigned long long)plan.max_runs);
    mix((unsigned long long)(plan.dc_first_scan + 1)); mix(plan.unit_coded ? 1 : 0);
    return h;
}

// scan sizes / buffer layout on the device, and their way back to the host
bool GpuEncoder::enqueue_sizes(void *stream_, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const int NS = (int)plan.scans.size();
    uint32_t *h_total = reinterpret_cast<uint32_t *>(h_small + o_total), *h_flags = reinterpret_cast<uint32_t *>(h_small + o_flags);
    k_ge_scanout<<<1, 32, 0, st>>>(d_scans, NS, d_tbits, d_corr, d_total, d_so, words_cap, d_flags);
    LT_MARK("k_ge_scanout");
    CU(cudaMemcpyAsync(h_total, d_total, (size_t)NS * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(h_flags, d_flags, 8, cudaMemcpyDeviceToHost, st));
    LT_MARK("copy");
    return true;
}
bool GpuEncoder::mark_sizes(void *stream_, std::string &err)
{   // the event finish() waits for before it sizes the D2H of the scans (kept out of captured graphs: a plain stream operation)
    CU(cudaEventRecord((cudaEvent_t)ev_sizes, (cudaStream_t)stream_));
    return true;
}

bool GpuEncoder::enqueue_back(void *stream_, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const int NS = (int)plan.scans.size(), NC = (int)plan.comps.size();
    uint32_t *h_flags = reinterpret_cast<uint32_t *>(h_small + o_flags);
    const dim3 gb(cdiv(plan.max_comp_blocks, ENC_THREADS), NC);
    int n = 5;
    if (plan.unit_coded) {                  // units of the sequential interleaved scans: lengths, then bit offsets
        k_geb_len<<<gb, ENC_THREADS, 0, st>>>(d_comps, d_gcount, d_tabs, d_bitlen, d_masks);
        LT_MARK("k_geb_len");
        size_t tb = d_temp.capacity();
        cub::DeviceScan::ExclusiveSum(d_temp, tb, d_bitlen.get(), d_bitoff.get(), (int)plan.total_lunits, st);
        LT_MARK("cub_scan");
        n += 2;
    }
    CU(cudaMemsetAsync(d_cursor, 0, (size_t)NS * 4, st));
    LT_MARK("memset");
    k_ge_zero<<<dim3(64, NS), 256, 0, st>>>(d_scans, d_so, d_words, d_arena);
    LT_MARK("k_ge_zero");
    k_geb_emit<<<gb, ENC_THREADS, 0, st>>>(d_comps, d_gcount, d_tabs, d_bitoff, d_words, d_masks, d_so, d_flags, d_arena, d_cursor, d_runlen, d_runpos);
    LT_MARK("k_geb_emit");
    if (plan.dc_first_scan >= 0) {
        k_geb_dc_first<<<dim3(cdiv((long long)geom.mcux * geom.mcuy, ENC_DC_MCUS), nimg), ENC_DC_MCUS, 0, st>>>(d_scans, plan.scans_per_image, plan.dc_first_scan, d_dc,
                                                                                                         d_tabs, d_so, d_flags, d_arena, d_cursor, d_runlen, d_runpos);
        LT_MARK("k_geb_dc_first");
        n++;
    }
    if (plan.total_runs) {                  // runs of the single-component scans: offsets, then placement
        size_t tb = d_temp.capacity();
        cub::DeviceScan::ExclusiveSum(d_temp, tb, d_runlen.get(), d_runoff.get(), plan.total_runs, st);
        LT_MARK("cub_scan");
        k_ge_place<<<dim3(cdiv(plan.max_runs, PLACE_THREADS / 32), NS), PLACE_THREADS, 0, st>>>(d_scans, d_so, d_runlen, d_runoff, d_runpos, d_arena, d_words, d_flags);
        LT_MARK("k_ge_place");
        n += 2;
    }
    k_ge_ffcount<<<dim3(STUFF_CHUNKS, NS), STUFF_THREADS, 0, st>>>(d_so, d_words, d_chunkff);
    LT_MARK("k_ge_ffcount");
    k_ge_layout<<<nimg, LAYOUT_THREADS, plan.scans_per_image * 4, st>>>(d_so, plan.scans_per_image, d_chunkff, d_outoff, d_outlen, (uint32_t)out_stride, d_flags);
    LT_MARK("k_ge_layout");
    k_ge_scatter<<<dim3(STUFF_CHUNKS, NS), STUFF_THREADS, 0, st>>>(d_so, d_words, d_chunkff, d_outoff, d_out, plan.scans_per_image, out_stride, d_flags);
    LT_MARK("k_ge_scatter");
    CU(cudaMemcpyAsync(h_small + o_outlen, d_outlen, (size_t)NS * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(h_small + o_dht, d_dht, (size_t)NS * 4 * sizeof(DhtOut), cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(h_flags + 4, d_flags, 32, cudaMemcpyDeviceToHost, st));         // second snapshot: image-level overflow (flags[3..4])
    CU(cudaGetLastError());
    launches += n;
    return true;
}

bool GpuEncoder::enqueue(void *stream_, bool fill_dummy, std::string &err)
{
    return enqueue_front(stream_, fill_dummy, err) && enqueue_sizes(stream_, err) && mark_sizes(stream_, err) && enqueue_back(stream_, err);
}

bool GpuEncoder::enqueue_front(void *stream_, bool fill_dummy, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const JpegGeom &g = geom;
    const int NS = (int)plan.scans.size(), NC = (int)plan.comps.size();
    const long long U = plan.total_units;
    int max_units = 0; for (auto &s : plan.scans) max_units = std::max(max_units, s.nblocks);
    launches = 0;
    const dim3 gb(cdiv(plan.max_comp_blocks, ENC_THREADS), NC);
    if (fill_dummy) {
        for (int im = 0; im < nimg; im++) for (int cc = 0; cc < g.ncomp; cc++) {
            if (g.rbw[cc] == g.bw[cc] && g.rbh[cc] == g.bh[cc]) continue;
            k_ge_fill_dummy<<<cdiv((long long)g.bw[cc] * g.bh[cc], 256), 256, 0, st>>>(coef_bases[im], g.comp_offset[cc], g.bw[cc], g.bh[cc], g.rbw[cc], g.rbh[cc], g.hs[cc]);
            LT_MARK("k_ge_fill_dummy");
            launches++;
        }
    }
    const dim3 gu1(cdiv(max_units + 1, 128), NS);
    CU(cudaMemsetAsync(d_hist, 0, (size_t)NS * 4 * 256 * 4, st));
    LT_MARK("memset");
    CU(cudaMemsetAsync(d_corr, 0, (size_t)NS * 4, st));
    LT_MARK("memset");
    k_geb_classify<<<gb, ENC_THREADS, 0, st>>>(d_comps, d_meta, d_evkey, d_tail, d_masks, d_hist, d_corr, plan.dc_first_scan >= 0 ? d_dc.get() : nullptr);
    LT_MARK("k_geb_classify");
    size_t tb = d_temp.capacity();
    cub::DeviceScan::ExclusiveScan(d_temp, tb, d_evkey.get(), d_prev.get(), cub::Max(), -1, (int)U, st);
    LT_MARK("cub_scan");
    tb = d_temp.capacity();
    cub::DeviceScan::ExclusiveSum(d_temp, tb, d_tail.get(), d_tsum.get(), (int)U, st);
    LT_MARK("cub_scan");
    CU(cudaMemsetAsync(d_gcount, 0, U * 4, st));
    LT_MARK("memset");
    k_ge_groups<<<gu1, 128, 0, st>>>(d_scans, d_meta, d_evkey, d_prev, d_tsum, d_gcount, d_hist);
    LT_MARK("k_ge_groups");
    k_ge_tables<<<NS * 4, 32, 0, st>>>(d_hist, d_tabs, d_dht, d_tbits);
    LT_MARK("k_ge_tables");
    launches += 5;
    CU(cudaGetLastError());
    return true;
}

bool GpuEncoder::finish(void *stream_, bool fetch, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const int NS = (int)plan.scans.size(), spi = plan.scans_per_image;
    uint32_t *h_total = reinterpret_cast<uint32_t *>(h_small + o_total), *h_flags = reinterpret_cast<uint32_t *>(h_small + o_flags);
    uint32_t *h_outlen = reinterpret_cast<uint32_t *>(h_small + o_outlen);
    const DhtOut *h_dht = reinterpret_cast<const DhtOut *>(h_small + o_dht);
    for (int attempt = 0;; attempt++) {
        // sizes are on the host while the emit / stuffing kernels still run
        const auto tw0 = std::chrono::steady_clock::now();
        if (fetch) { CU(event_wait((cudaEvent_t)ev_sizes)); } else { CU(stream_wait(st)); }
        wait_sizes_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tw0).count();
        size_t img_max = 0, img = 0;
        for (int si = 0; si < NS; si++) { img += (h_total[si] + 7) / 8; if ((si + 1) % spi == 0) { img_max = std::max(img_max, img); img = 0; } }
        if (h_flags[0]) {                                       // the estimate was too small for the bit buffer: exact sizes, back half again
            if (attempt >= 3) { err = "entropy encoder could not size its buffers"; return false; }
            CU(stream_wait(st));
            if (!size_back_buffers(img_max + img_max / 16 + 4096, err)) return false;
            retries++;
            if (!enqueue_sizes(st, err) || !mark_sizes(st, err) || !enqueue_back(st, err)) return false;
            continue;
        }
        if (fetch) {
            copy_bytes = std::min(out_stride, align_up(img_max + img_max / 8 + 256, 256));
            if (!h_out.reserve(copy_bytes * nimg, Grow::Pow2Half, err, &generation)) return false;
            for (int im = 0; im < nimg; im++) CU(cudaMemcpyAsync(h_out + (size_t)im * copy_bytes, d_out + (size_t)im * out_stride, copy_bytes, cudaMemcpyDeviceToHost, st));
            CU(cudaGetLastError());
            const auto tw1 = std::chrono::steady_clock::now();
            CU(stream_wait(st));
            wait_final_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tw1).count();
        }
        if (h_flags[4 + 4]) {                                   // an image stuffed past its output region (more 0xFF bytes than one in eight)
            if (attempt >= 3) { err = "entropy encoder could not size its output"; return false; }
            if (!size_back_buffers((size_t)h_flags[4 + 3] + 4096, err)) return false;
            retries++;
            if (!enqueue_sizes(st, err) || !mark_sizes(st, err) || !enqueue_back(st, err)) return false;
            continue;
        }
        learned_image_bytes = std::max<size_t>(learned_image_bytes, h_flags[4 + 3]);
        if (fetch) {   // rare: an image stuffed more than the copied margin -> fetch everything at full stride
            bool shortc = false;
            for (int im = 0; im < nimg && !shortc; im++) { size_t tot = 0; for (int k = 0; k < spi; k++) tot += h_outlen[im * spi + k]; shortc = tot > copy_bytes; }
            if (shortc) {
                if (!h_out.reserve(out_stride * nimg, Grow::Pow2Half, err, &generation)) return false;
                copy_bytes = out_stride;
                for (int j = 0; j < nimg; j++) CU(cudaMemcpyAsync(h_out + (size_t)j * copy_bytes, d_out + (size_t)j * out_stride, copy_bytes, cudaMemcpyDeviceToHost, st));
                CU(stream_wait(st));
            }
        }
        break;
    }
    // ---- describe the result
    results.assign((size_t)NS, EncodedScan());
    for (int si = 0; si < NS; si++) {
        EncodedScan &e = results[si];
        const int im = si / spi, k = si % spi;
        e.def = plan.defs[k];
        size_t off = 0; for (int j = 0; j < k; j++) off += h_outlen[im * spi + j];
        e.data = fetch ? h_out + (size_t)im * copy_bytes + off : nullptr; e.len = h_outlen[si];
        bool need[2][2]; jpeg_scan_tables_needed(geom, prog, e.def, need);
        for (int kind = 0; kind < 2; kind++) for (int t = 0; t < 2; t++) {
            e.has_tab[kind][t] = need[kind][t];
            const DhtOut &D = h_dht[(size_t)si * 4 + kind * 2 + t];
            memcpy(e.bits[kind][t], D.bits, 17); memcpy(e.vals[kind][t], D.vals, 256); e.nvals[kind][t] = D.nvals;
        }
    }
    return true;
}

bool GpuEncoder::encode(const JpegGeom &g, bool progressive, int16_t *const *d_coefs, int nimages, void *stream_, bool fill_dummy, std::string &err, size_t out_bytes_hint)
{
    return prepare(g, progressive, d_coefs, nimages, stream_, out_bytes_hint, err) && upload(stream_, err) && enqueue(stream_, fill_dummy, err) && finish(stream_, true, err);
}

} // namespace b200
