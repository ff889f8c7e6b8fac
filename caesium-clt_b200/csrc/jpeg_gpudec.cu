// jpeg_gpudec.cu -- device entropy DECODER for baseline single-scan JPEG files: CUDA wrappers around the bodies in
// jpeg_gpudec_core.h (self-synchronising parallel Huffman decoding) plus byte un-stuffing and the DC prefix sums.
// Batched: every pass is one launch for all images of the batch (blockIdx.y = image), which is what keeps the launch
// count per image low when b200_compress_batch packs images into megabatches.
// Pass order: unstuff (count, scan, scatter) -> round 0 -> rounds (in groups, one host check per group) -> block-count
// scan -> write (coefficients and DC differences) -> DC scan / scatter (no scatter when the batch defers the DC to the transform).  Coefficients land directly in the transform kernels' input buffers, so the
// host never sees them.
#include <cuda_runtime.h>
#include <cub/device/device_scan.cuh>
#include <algorithm>
#include <cstring>
#include "jpeg_gpudec.h"
#include "jpeg_gpuenc_plan.h"
#include "stream_wait.h"
#include "launch_timer.h"
#include "host_copy.h"

namespace b200 {

using namespace gd;

// ---- un-stuffing: drop the 0x00 that follows every 0xFF -----------------------------------------------------------------
// One thread per 16-byte group of the entropy-coded segment, read with one 16-byte load (the raw buffer of every image starts
// 16-byte aligned and has at least 16 bytes of slack behind it, so the last group's load stays inside the buffer).  The
// per-thread bodies are gd::unstuff_count_group / unstuff_place_group / unstuff_store (jpeg_gpudec_core.h).
constexpr int UNSTUFF_THREADS = 128;
__device__ __forceinline__ RawGroup load_group(const uint8_t *raw, uint32_t g) { const uint4 q = reinterpret_cast<const uint4 *>(raw)[g]; return RawGroup{q.x, q.y, q.z, q.w}; }

__global__ void __launch_bounds__(UNSTUFF_THREADS) k_gd_unstuff_count(const DecImage *__restrict__ imgs, const uint8_t *__restrict__ raw_all, uint32_t *__restrict__ cnt, uint32_t *__restrict__ marker)
{
    const DecImage &im = imgs[blockIdx.y];
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= im.ngrp) return;
    const uint8_t *raw = raw_all + im.raw_off;
    bool mark;
    cnt[im.grp_off + g] = unstuff_count_group(raw, load_group(raw, g), g, im.nraw, im.verify, &mark);
    if (mark) marker[blockIdx.y] = 1;
}
// A CTA's groups un-stuff into one contiguous range of the output: the bytes are compacted in shared memory, at the output's
// word alignment, and leave as aligned 4-byte stores, coalesced across the CTA; only the up to three bytes at either end of the
// range, whose words the neighbouring CTAs share, leave one by one.
// (for images the host did not walk, the thread of the last group also publishes the true stream length: g.nbits and g.nsub in
// the device copy of the descriptor were upper bounds taken from the raw length)
__global__ void __launch_bounds__(UNSTUFF_THREADS) k_gd_unstuff_scatter(DecImage *imgs, const uint8_t *__restrict__ raw_all, const uint32_t *__restrict__ off, const uint32_t *__restrict__ cnt, uint8_t *__restrict__ stream_all)
{
    __shared__ uint32_t sbuf[UNSTUFF_THREADS * 4 + 1];
    __shared__ uint32_t range_end;
    DecImage &im = imgs[blockIdx.y];
    const uint32_t g0 = blockIdx.x * blockDim.x, g = g0 + threadIdx.x;
    if (g0 >= im.ngrp) return;
    const uint8_t *raw = raw_all + im.raw_off;
    uint8_t *out = stream_all + im.stream_off;
    uint8_t *sb = reinterpret_cast<uint8_t *>(sbuf);
    const uint32_t base = off[im.grp_off];
    const uint32_t first = g0 * 16 - (off[im.grp_off + g0] - base), aligned = first & ~3u;     // the CTA's first output byte
    if (g < im.ngrp) {
        const uint32_t o = unstuff_place_group(raw, load_group(raw, g), g, im.nraw, g * 16 - (off[im.grp_off + g] - base), aligned, sb);
        if (g == g0 + blockDim.x - 1 || g == im.ngrp - 1) range_end = o;
    }
    __syncthreads();
    const uint32_t end = range_end;
    unstuff_store(sbuf, aligned, first, end, threadIdx.x, blockDim.x, out, g == im.ngrp - 1, im.verify, im.nraw, off + (im.grp_off + g), cnt + (im.grp_off + g), base, im.g);
}

// ---- synchronisation rounds ------------------------------------------------------------------------------------------------
// Geometry and the Huffman tables are staged in shared memory: the decode loop indexes both dynamically.
struct DecShared { Geometry g; DecTables T; };
__device__ __forceinline__ void stage_shared(DecShared &sh, const DecImage &im, const DecTables *__restrict__ tabs)
{
    const uint32_t *src = reinterpret_cast<const uint32_t *>(&im.g);
    uint32_t *dst = reinterpret_cast<uint32_t *>(&sh.g);
    for (int i = threadIdx.x; i < (int)(sizeof(Geometry) / 4); i += blockDim.x) dst[i] = src[i];
    // only what the image uses: its first-level tables, the used part of the second-level pool, the selector / header words
    const int nlook = tabs->nlook * (LOOK_N / 2), next = (tabs->next + 1) / 2;
    src = reinterpret_cast<const uint32_t *>(tabs->look); dst = reinterpret_cast<uint32_t *>(sh.T.look);
    for (int i = threadIdx.x; i < nlook; i += blockDim.x) dst[i] = src[i];
    src = reinterpret_cast<const uint32_t *>(tabs->ext); dst = reinterpret_cast<uint32_t *>(sh.T.ext);
    for (int i = threadIdx.x; i < next; i += blockDim.x) dst[i] = src[i];
    src = reinterpret_cast<const uint32_t *>(tabs->sel); dst = reinterpret_cast<uint32_t *>(sh.T.sel);
    for (int i = threadIdx.x; i < 12; i += blockDim.x) dst[i] = src[i];          // sel[20] + nlook, next, ok, pad
    __syncthreads();
}

__global__ void __launch_bounds__(64) k_gd_round0(const DecImage *__restrict__ imgs, const uint8_t *__restrict__ stream_all, const DecTables *__restrict__ tabs_all,
                                                  DecState *__restrict__ A, uint8_t *__restrict__ chg, uint32_t *__restrict__ nblk)
{
    __shared__ DecShared sh;
    const DecImage &im = imgs[blockIdx.y];
    if (blockIdx.x * blockDim.x >= im.g.nsub) return;
    stage_shared(sh, im, tabs_all + blockIdx.y);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sh.g.nsub) return;
    NullSink sk; DecState st; st.p = i * sh.g.subseq_bits; st.k = 0; st.b = 0;
    A[im.sub_off + i] = decode_subsequence(stream_all + im.stream_off, sh.g, sh.T, i, st, sk);
    nblk[im.sub_off + i] = sk.nblk; chg[im.sub_off + i] = 0;       // epoch 0: "changed in round 0"
}

__device__ __forceinline__ DecState load_state(const DecState *p) { const unsigned long long v = *reinterpret_cast<const volatile unsigned long long *>(p); DecState s; memcpy(&s, &v, 8); return s; }
__device__ __forceinline__ void store_state(DecState *p, const DecState &s) { unsigned long long v; memcpy(&v, &s, 8); *reinterpret_cast<volatile unsigned long long *>(p) = v; }

// Round r (1, 2, ...): subsequence i is decoded again iff the exit state of i-1 changed in round r-1 (epoch[i-1] == r-1).
// States are updated in place with single 64-bit accesses: a reader sees the old or the new exit of its predecessor, and
// if it was the old one the predecessor's epoch makes it run again next round.  A CTA whose 64 predecessors all kept their
// exits is "clean": it leaves after one byte read (dirty flags double-buffered by round parity), and an image whose
// previous round changed nothing leaves at once, so the tail rounds of a launch group cost almost nothing.
__global__ void __launch_bounds__(64) k_gd_round(const DecImage *__restrict__ imgs, const uint8_t *__restrict__ stream_all, const DecTables *__restrict__ tabs_all,
                                                 DecState *__restrict__ S, uint8_t *__restrict__ epoch, uint8_t *__restrict__ dirty_in, uint8_t *__restrict__ dirty_out,
                                                 uint32_t *__restrict__ nblk, uint32_t *__restrict__ any_changed /*[image]*/,
                                                 const uint32_t *__restrict__ prev_changed /*[image] of the round before, or null*/, int r)
{
    __shared__ DecShared sh;
    __shared__ int go;
    if (prev_changed && prev_changed[blockIdx.y] == 0) return;
    const DecImage &im = imgs[blockIdx.y];
    const uint32_t nsub = im.g.nsub;
    if (blockIdx.x * blockDim.x >= nsub) return;
    const size_t cta = (size_t)blockIdx.y * gridDim.x + blockIdx.x;
    if (threadIdx.x == 0) { go = r == 1 || dirty_in[cta]; if (r > 1 && go) dirty_in[cta] = 0; }
    __syncthreads();
    if (!go) return;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, gi = im.sub_off + i;
    const bool mine = i > 0 && i < nsub && epoch[gi - 1] == (uint8_t)(r - 1);
    if (!__syncthreads_or(mine)) return;             // nobody in this CTA has to re-decode: skip the table staging too
    stage_shared(sh, im, tabs_all + blockIdx.y);
    if (!mine) return;
    NullSink sk;
    const DecState st = load_state(S + gi - 1), old = load_state(S + gi);
    const DecState o = decode_subsequence(stream_all + im.stream_off, sh.g, sh.T, i, st, sk);
    nblk[gi] = sk.nblk;
    if (!same_state(o, old)) {
        store_state(S + gi, o); epoch[gi] = (uint8_t)r;
        if (i + 1 < nsub) dirty_out[threadIdx.x == blockDim.x - 1 ? cta + 1 : cta] = 1;
        atomicOr(&any_changed[blockIdx.y], 1u);
    }
}

// Write pass sink: whole-sector stores.  A block of this layout (int16, zigzag, 128 bytes) is one cache line of four 32-byte
// sectors, a block's non-zero coefficients arrive in ascending zigzag index, and in gd::decode_owned_blocks every block has one
// writer.  So the sink holds the block's current sector (16 coefficients) in shared memory, stores it with two 16-byte writes
// when a coefficient of a later sector arrives, and stores zeros for the sectors in between and behind: every owned block
// receives exactly eight 16-byte stores whatever its content, and nothing has to be zeroed beforehand.  The staging area is
// word-major, stage[word][thread]: a thread's eight words live in its own bank, so neither the 2-byte placement nor the flush
// can conflict.  The lanes of a warp reach their sector changes at unrelated symbols, and a flush run by one lane costs the
// warp as much as one run by all, so there is ONE flush site in the loop: the end of a block only marks the held block as
// ended, and its last sectors leave when the next block's DC coefficient arrives (or in finish()), together with the other
// lanes' mid-block sector changes of that iteration.  With a second flush site at the end of the block the kernel took
// 0.436 ms per 8-image 4K megabatch, H100 SXM 700 W; see DESIGN.md 4.2 for the figures of the sink this one replaced.
// The sector that holds the DC coefficient also delivers the block's DC difference to the component-major array the DC prefix
// sum runs over.  The block address moves with a gd::Cursor: no divisions inside the decode loop.  Every subsequence starts
// from its true state here, so a stream anomaly met inside a real block (cur < total) is in the stream itself: it is collected
// and the image goes to the host decoder.
constexpr int WRITE_THREADS = 64;
struct SectorWriteSink {
    const Walk *walk; int16_t *coefs; int32_t *dc; uint32_t *stage;
    uint32_t cur, total; Cursor c;      // the block the decoder is in (cur >= total: padding after the last real block)
    int16_t *ptr; int32_t *dcp;         // the held block and where its DC difference goes; null before the first DC and in the padding
    int sec; bool ended; uint32_t anom; // sector held; the held block is complete (the cursor has moved on)
    __device__ __forceinline__ void seek() { c.seek(*walk, cur); ptr = nullptr; dcp = nullptr; sec = 0; ended = true; for (int w = 0; w < 8; w++) stage[w * WRITE_THREADS] = 0; }
    __device__ __forceinline__ void flush_to(int target)
    {   // sectors sec .. target - 1 leave: the held one from the staging words, the others as zeros
        uint4 lo = make_uint4(stage[0], stage[WRITE_THREADS], stage[2 * WRITE_THREADS], stage[3 * WRITE_THREADS]);
        uint4 hi = make_uint4(stage[4 * WRITE_THREADS], stage[5 * WRITE_THREADS], stage[6 * WRITE_THREADS], stage[7 * WRITE_THREADS]);
        if (sec == 0) *dcp = (int16_t)(lo.x & 0xFFFFu);
        for (int w = 0; w < 8; w++) stage[w * WRITE_THREADS] = 0;
        uint4 *out = reinterpret_cast<uint4 *>(ptr) + 2 * sec;
        for (int s = sec; s < target; s++, out += 2) { out[0] = lo; out[1] = hi; lo = hi = make_uint4(0, 0, 0, 0); }
    }
    __device__ __forceinline__ void coef(int k, int v)
    {
        const int s = k >> 4;
        if (ended || s != sec) {
            if (ptr) flush_to(ended ? 4 : s);
            if (ended) { ended = false; ptr = cur < total ? coefs + c.offset(*walk) : nullptr; dcp = dc + c.dc_slot(*walk); }
            sec = s;
        }
        if (ptr) reinterpret_cast<int16_t *>(stage + ((k & 15) >> 1) * WRITE_THREADS)[k & 1] = (int16_t)v;
    }
    __device__ __forceinline__ void anomaly(uint32_t m) { if (cur < total) anom |= m; }
    __device__ __forceinline__ void block_done() { cur++; c.next(*walk); ended = true; }
    __device__ __forceinline__ void finish() { if (ptr) flush_to(4); }      // the last block (cut short only if the stream was: flagged)
};

// marker word per image: bit 0 = a marker inside the segment (un-stuff pass), ANOM_* << 1 = the write pass's stream anomalies
__global__ void __launch_bounds__(WRITE_THREADS) k_gd_write(const DecImage *__restrict__ imgs, const uint8_t *__restrict__ stream_all, const DecTables *__restrict__ tabs_all,
                                                            const DecState *__restrict__ A, const uint32_t *__restrict__ first, int32_t *__restrict__ dc, uint32_t *__restrict__ marker)
{
    __shared__ DecShared sh;
    __shared__ Walk walk;
    __shared__ uint32_t stage[8][WRITE_THREADS];
    static_assert(sizeof(Walk) / 4 <= WRITE_THREADS, "one thread per word stages the Walk");
    const DecImage &im = imgs[blockIdx.y];
    if (blockIdx.x * blockDim.x >= im.g.nsub) return;
    if (threadIdx.x < sizeof(Walk) / 4) reinterpret_cast<uint32_t *>(&walk)[threadIdx.x] = reinterpret_cast<const uint32_t *>(&im.walk)[threadIdx.x];
    stage_shared(sh, im, tabs_all + blockIdx.y);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sh.g.nsub) return;
    DecState st;
    if (i == 0) { st.p = 0; st.k = 0; st.b = 0; } else st = A[im.sub_off + i - 1];
    SectorWriteSink sk;
    sk.walk = &walk; sk.coefs = const_cast<int16_t *>(im.scan.coef); sk.dc = dc + im.blk_off; sk.stage = &stage[0][threadIdx.x];
    sk.cur = first_owned_block(first[im.sub_off + i] - first[im.sub_off], st); sk.total = sh.g.total_blocks; sk.anom = 0;
    sk.seek();
    decode_owned_blocks(stream_all + im.stream_off, sh.g, sh.T, i, st, sk);
    sk.finish();
    if (sk.anom) atomicOr(&marker[blockIdx.y], sk.anom << 1);
}

// ---- DC: the write pass left the differences component-major; inclusive scan, subtract the component's base, scatter ------------------
// (a stream that ends before its last block is flagged by the write pass and decoded on the host: nothing to finish here)
__global__ void k_gd_dc_scatter(const DecImage *__restrict__ imgs, const int32_t *__restrict__ sum)
{
    const DecImage &im = imgs[blockIdx.y];
    const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= im.g.total_blocks) return;
    uint32_t cs;
    const uint32_t idx = dc_slot_index(im.scan, u, &cs);
    const uint32_t b = im.blk_off + cs;
    const int32_t base = b ? sum[b - 1] : 0;
    const_cast<int16_t *>(ge::locate(im.scan, (int)u).blk)[0] = (int16_t)(sum[im.blk_off + idx] - base);
}

// ---- host ---------------------------------------------------------------------------------------------------------------------
static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }
// prepare(): per-image descriptors, buffers, Huffman tables; entropy-coded bytes and parameters staged in pinned memory and
// their H2D copies enqueued.  enqueue(): every pass, no host wait -- a fixed number of synchronisation rounds (rounds whose image
// has already settled leave at once), the per-round "something changed" flags copied back at the end.  finish(): after the
// caller's wait, says per image whether it settled.  decode() = the three in a row with a wait.
bool GpuDecoder::prepare(std::vector<Item> &items, void *stream_, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const int N = (int)items.size();
    nitems = N;
    if (N == 0) return true;
    // ---- per-image descriptors
    imgs.assign((size_t)N, DecImage());
    coef_ptrs.resize((size_t)N); coef_bytes.resize((size_t)N);
    defer_dc = items[0].defer_dc;
    for (const Item &it : items) if (it.defer_dc != defer_dc) { err = "a decode batch takes one DC setting"; return false; }
    raw_total = 0; size_t stream_total = 0; grp_total = 0; sub_total = 0; blk_total = 0; max_grp = 0; max_sub = 0; max_blk = 0;
    for (int n = 0; n < N; n++) {
        const JpegReader &rd = *items[n].rd; const JpegReader::DeviceScan &ds = *items[n].ds; const JpegGeom &g = rd.geom();
        items[n].result = FAILED;
        DecImage &im = imgs[n]; memset(&im, 0, sizeof(im));
        const size_t nraw = ds.ecs_end - ds.ecs_begin;
        if (nraw >= (1ull << 28)) { err = "entropy-coded segment too large for the device decoder"; return false; }
        const uint32_t nstream = (uint32_t)(ds.verified ? nraw - ds.stuffed : nraw);      // unverified: upper bound, the device finds the real length
        im.verify = ds.verified ? 0u : 1u;
        Geometry &G = im.g;
        int q = 0;
        for (int c = 0; c < g.ncomp; c++) for (int k = 0; k < (g.ncomp == 1 ? 1 : g.hs[c] * g.vs[c]); k++) { if (q >= 10) { err = "MCU too large"; return false; } G.dc_tbl[q] = ds.td[c]; G.ac_tbl[q] = ds.ta[c]; q++; }
        G.blocks_per_mcu = q;
        G.total_blocks = g.ncomp == 1 ? (uint32_t)(g.rbw[0] * g.rbh[0]) : (uint32_t)(g.mcux * g.mcuy * q);
        static const int subseq_bits = [] { const char *e = getenv("B200_DEC_SUBSEQ"); const int v = e ? atoi(e) : 0; return v >= 128 && v <= 8192 && v % 32 == 0 ? v : (int)SUBSEQ_BITS; }();
        G.nbits = nstream * 8; G.subseq_bits = subseq_bits; G.nsub = (G.nbits + G.subseq_bits - 1) / G.subseq_bits;
        if (G.nsub == 0) { err = "empty scan"; return false; }
        GpuEncPlan plan; const int16_t *base = items[n].d_coefs;
        gpuenc_plan(g, false, &base, 1, plan);
        im.scan = plan.scans[0];
        im.walk = make_walk(im.scan);
        im.raw_off = (uint32_t)raw_total; im.nraw = (uint32_t)nraw; raw_total += align_up(nraw + 16, 16);
        im.stream_off = (uint32_t)stream_total; stream_total += align_up((size_t)nstream + 32, 16);
        im.grp_off = grp_total; im.ngrp = (uint32_t)((nraw + 15) / 16); grp_total += im.ngrp;
        im.sub_off = sub_total; sub_total += G.nsub;
        im.blk_off = blk_total; blk_total += G.total_blocks;
        max_grp = std::max(max_grp, im.ngrp); max_sub = std::max(max_sub, G.nsub); max_blk = std::max(max_blk, G.total_blocks);
        // The write pass stores every block of the scan whole, so the buffer needs no clearing -- unless the layout has blocks the
        // scan does not code: a single-component scan codes rbw x rbh blocks into a plane pitched bw, and those padding blocks
        // would have to read as zero.  JpegReader lays a single-component file out at one block per MCU whatever sampling
        // factors it declares (bw == rbw), so no file it accepts has them today; the layout is still checked, not assumed.
        coef_ptrs[n] = items[n].d_coefs; coef_bytes[n] = (long long)G.total_blocks * 64 != g.total_coefs ? (size_t)g.total_coefs * 2 : 0;
    }
    if (raw_total >= (1ull << 31) || stream_total >= (1ull << 31)) { err = "decode batch too large"; return false; }
    // ---- launch-side sizes are HIGH-WATER marks, not this batch's exact sizes: grids, scan lengths and the H2D size of the pass
    //      sequence then stay the same from batch to batch (kernels test against the per-image sizes in the descriptors), which is
    //      what lets the caller replay the sequence as a CUDA graph instead of ~70 driver calls per megabatch
    auto hw = [](size_t &mark, size_t need) { if (need > mark) mark = need + need / 8 + 64; };
    if (N != hw_n) { hw_n = N; hw_raw = hw_stream = hw_grp = hw_sub = hw_blk = hw_mgrp = hw_msub = hw_mblk = 0; }
    hw(hw_raw, raw_total); hw(hw_stream, stream_total); hw(hw_grp, grp_total); hw(hw_sub, sub_total); hw(hw_blk, blk_total);
    hw(hw_mgrp, max_grp); hw(hw_msub, max_sub); hw(hw_mblk, max_blk);
    // ---- buffers
    o_img = 0; o_tab = align_up(sizeof(DecImage) * N, 256); o_flag = o_tab + align_up(sizeof(DecTables) * N, 256);
    o_mark = o_flag + align_up((size_t)4 * N * (MAX_ROUNDS + 2), 256);
    par_bytes = o_mark + align_up((size_t)4 * N, 256);
    // sizes here depend on image CONTENT (bytes of entropy-coded data): Grow::Pow2Half rounds up to a power of two with headroom so a
    // slot stops reallocating after its first image of a given class (cudaFree / cudaHostAlloc stall every stream)
    auto grow = [&](auto &buf, size_t need) { return buf.reserve(need, Grow::Pow2Half, err, &generation); };
    if (!grow(h_raw, hw_raw + 64) || !grow(d_raw, hw_raw + 64) || !grow(d_stream, hw_stream + 64) ||
        !grow(d_cnt, hw_grp * 4 + 4) || !grow(d_off, hw_grp * 4 + 4) || !grow(d_A, hw_sub * sizeof(DecState)) ||
        !grow(d_chgA, hw_sub) || !grow(d_chgB, (size_t)2 * N * cdiv((long long)hw_msub, 64) + 64) ||
        !grow(d_nblk, hw_sub * 4) || !grow(d_first, hw_sub * 4) || !grow(d_dc, hw_blk * 4) || !grow(d_dcs, hw_blk * 4) ||
        !grow(d_par, par_bytes) || !grow(h_par, par_bytes)) return false;
    size_t t1 = 0, t2 = 0, t3 = 0;
    cub::DeviceScan::ExclusiveSum((void *)nullptr, t1, d_cnt.get(), d_off.get(), (int)hw_grp, st);
    cub::DeviceScan::ExclusiveSum((void *)nullptr, t2, d_nblk.get(), d_first.get(), (int)hw_sub, st);
    cub::DeviceScan::InclusiveSum((void *)nullptr, t3, d_dc.get(), d_dcs.get(), (int)hw_blk, st);
    if (!grow(d_temp, std::max(t1, std::max(t2, t3)) + 256)) return false;
    // ---- parameters + raw bytes
    DecTables *ht = reinterpret_cast<DecTables *>(h_par + o_tab);
    tables_ok.assign((size_t)N, 1);
    for (int n = 0; n < N; n++) {
        const JpegReader &rd = *items[n].rd;
        const uint8_t *db[8], *dv[8];
        for (int id = 0; id < 4; id++) for (int kind = 0; kind < 2; kind++) { const bool pr = rd.dht_present(kind, id); db[kind * 4 + id] = pr ? rd.dht_bits(kind, id) : nullptr; dv[kind * 4 + id] = pr ? rd.dht_vals(kind, id) : nullptr; }
        // tables that do not fit the second-level pool: the kernels run on an all-invalid table set and the image is reported
        // NOT_CONVERGED, which sends it to the host decoder
        tables_ok[n] = build_dec_tables(db, dv, imgs[n].g, ht[n]) ? 1 : 0;
        stream_copy(h_raw + imgs[n].raw_off, rd.data() + items[n].ds->ecs_begin, imgs[n].nraw);      // pinned staging: read next by the DMA engine only
    }
    memcpy(h_par + o_img, imgs.data(), sizeof(DecImage) * N);
    memset(h_par + o_flag, 0, (size_t)4 * N * (MAX_ROUNDS + 2));
    return true;
}

// H2D of what prepare() staged: descriptors + tables, and the entropy-coded bytes (high-water size: the tail past this batch's
// bytes is stale and unused)
bool GpuDecoder::upload(void *stream_, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    if (nitems == 0) return true;
    CU(cudaMemcpyAsync(d_par, h_par, o_flag, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_raw, h_raw, hw_raw, cudaMemcpyHostToDevice, st));
    return true;
}

unsigned long long GpuDecoder::signature() const
{   // everything a captured launch sequence bakes in: counts, high-water sizes, buffer identities
    unsigned long long h = 1469598103934665603ull;
    auto mix = [&](unsigned long long v) { h = (h ^ v) * 1099511628211ull; };
    mix((unsigned long long)nitems); mix(hw_raw); mix(hw_grp); mix(hw_sub); mix(hw_blk); mix(hw_mgrp); mix(hw_msub); mix(hw_mblk); mix(generation);
    mix(o_flag); mix(o_mark); mix(defer_dc);
    for (size_t n = 0; n < coef_ptrs.size(); n++) { mix((unsigned long long)(uintptr_t)coef_ptrs[n]); mix(coef_bytes[n]); }
    return h;
}

bool GpuDecoder::enqueue(void *stream_, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const int N = nitems;
    if (N == 0) return true;
    static const int nrounds = [] { const char *e = getenv("B200_DEC_ROUNDS"); const int v = e ? atoi(e) : 0; return v >= 1 && v <= MAX_ROUNDS ? v : (int)ROUNDS; }();
    DecImage *dIw = reinterpret_cast<DecImage *>(d_par + o_img);
    const DecImage *dI = dIw;
    const DecTables *dT = reinterpret_cast<const DecTables *>(d_par + o_tab);
    uint32_t *dF = reinterpret_cast<uint32_t *>(d_par + o_flag), *dM = reinterpret_cast<uint32_t *>(d_par + o_mark);
    uint32_t *hF = reinterpret_cast<uint32_t *>(h_par + o_flag);
    CU(cudaMemsetAsync(dF, 0, (o_mark - o_flag) + (size_t)4 * N, st));                 // round flags + marker flags
    LT_MARK("memset");
    // ---- unstuff
    const dim3 gg(cdiv((long long)hw_mgrp, UNSTUFF_THREADS), N);
    k_gd_unstuff_count<<<gg, UNSTUFF_THREADS, 0, st>>>(dI, d_raw, d_cnt, dM);
    LT_MARK("k_gd_unstuff_count");
    size_t tb = d_temp.capacity();
    cub::DeviceScan::ExclusiveSum(d_temp, tb, d_cnt.get(), d_off.get(), (int)hw_grp, st);
    LT_MARK("cub_scan");
    k_gd_unstuff_scatter<<<gg, UNSTUFF_THREADS, 0, st>>>(dIw, d_raw, d_off, d_cnt, d_stream);
    LT_MARK("k_gd_unstuff_scatter");
    for (int n = 0; n < N; n++) if (coef_bytes[n]) CU(cudaMemsetAsync(coef_ptrs[n], 0, coef_bytes[n], st));      // padding blocks only
    // ---- rounds
    const dim3 gs(cdiv((long long)hw_msub, 64), N);
    const size_t ncta = (size_t)N * gs.x;                    // dirty flags: two buffers of one byte per CTA, by round parity
    CU(cudaMemsetAsync(d_chgB, 0, 2 * ncta, st));
    LT_MARK("memset");
    k_gd_round0<<<gs, 64, 0, st>>>(dI, d_stream, dT, d_A, d_chgA, d_nblk);
    LT_MARK("k_gd_round0");
    for (int rounds = 0; rounds < nrounds; rounds++) {
        const int rn = rounds + 1;                            // round number: reads dirty[rn & 1], writes dirty[(rn + 1) & 1]
        k_gd_round<<<gs, 64, 0, st>>>(dI, d_stream, dT, d_A, d_chgA, d_chgB + (size_t)(rn & 1) * ncta, d_chgB + (size_t)((rn + 1) & 1) * ncta, d_nblk,
                                      dF + (size_t)rounds * N, rounds ? dF + (size_t)(rounds - 1) * N : nullptr, rn);
        LT_MARK("k_gd_round");
    }
    rounds_used = nrounds;
    CU(cudaMemcpyAsync(hF, dF, (size_t)4 * N * nrounds, cudaMemcpyDeviceToHost, st));
    // ---- block counts -> first block of each subsequence -> write -> DC (images that did not converge, or whose stream the
    //      write pass flagged, produce garbage that their caller discards)
    tb = d_temp.capacity();
    cub::DeviceScan::ExclusiveSum(d_temp, tb, d_nblk.get(), d_first.get(), (int)hw_sub, st);
    LT_MARK("cub_scan");
    k_gd_write<<<gs, WRITE_THREADS, 0, st>>>(dI, d_stream, dT, d_A, d_first, d_dc, dM);
    LT_MARK("k_gd_write");
    CU(cudaMemcpyAsync(h_par + o_mark, dM, (size_t)4 * N, cudaMemcpyDeviceToHost, st));
    const dim3 gb(cdiv((long long)hw_mblk, 128), N);
    tb = d_temp.capacity();
    cub::DeviceScan::InclusiveSum(d_temp, tb, d_dc.get(), d_dcs.get(), (int)hw_blk, st);
    LT_MARK("cub_scan");
    if (!defer_dc) {
        k_gd_dc_scatter<<<gb, 128, 0, st>>>(dI, d_dcs);
        LT_MARK("k_gd_dc_scatter");
    }
    CU(cudaGetLastError());
    launches = (defer_dc ? 8 : 9) + nrounds;
    return true;
}

GpuDecoder::DcSums GpuDecoder::dc_sums(int n, int c) const
{   // the component-major layout of dc_slot_index: a component's blocks in MCU order, hs * vs of them per MCU
    DcSums d{nullptr, nullptr, 1, 1, 1};
    if (!defer_dc || n < 0 || n >= nitems) return d;
    const DecImage &im = imgs[(size_t)n];
    const ge::Scan &s = im.scan;
    uint32_t start = 0;
    for (int i = 0; i < s.ns; i++) {
        const int hs = s.ns == 1 ? 1 : s.hs[i], vs = s.ns == 1 ? 1 : s.vs[i];
        if (s.comp[i] == c) {
            const uint32_t b = im.blk_off + start;
            d.sum = d_dcs.get() + b; d.prev = b ? d_dcs.get() + b - 1 : nullptr;
            d.hs = hs; d.vs = vs; d.mcux = s.ns == 1 ? s.rbw : s.mcux;
            return d;
        }
        start += (uint32_t)s.mcux * (uint32_t)s.mcuy * (uint32_t)(hs * vs);
    }
    return d;
}

void GpuDecoder::finish(std::vector<Item> &items)
{   // the caller has waited for the stream: an image settled iff some round changed nothing in it
    const int N = nitems;
    const uint32_t *hF = reinterpret_cast<const uint32_t *>(h_par + o_flag), *hM = reinterpret_cast<const uint32_t *>(h_par + o_mark);
    for (int n = 0; n < N && n < (int)items.size(); n++) {
        bool conv = false;
        for (int r = 0; r < rounds_used && !conv; r++) conv = hF[(size_t)r * N + n] == 0;
        // a marker inside the segment, or a stream anomaly inside a real block: the host decoder's business
        items[n].result = conv && tables_ok[n] && !hM[n] ? OK : NOT_CONVERGED;
    }
}

bool GpuDecoder::decode(std::vector<Item> &items, void *stream_, std::string &err)
{
    if (items.empty()) return true;
    if (!prepare(items, stream_, err) || !upload(stream_, err) || !enqueue(stream_, err)) return false;
    CU(stream_wait((cudaStream_t)stream_));
    finish(items);
    return true;
}

} // namespace b200
