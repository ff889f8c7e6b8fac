// jpeg_kernels.cu -- hand-written sm_90a kernels for the JPEG transform stages of
// caesium::compress_in_memory (call site caesium-clt's src/compressor.rs:305; SURVEY.md §8a row a6):
//   K1 dequantise + 8x8 inverse DCT          K2 chroma upsample ("fancy" triangle filter)
//   K4 chroma box downsample                 K5 forward DCT + quantise + zigzag
// and the fusions the no-resize path uses (K1->K5 for full-resolution components, K2->K4->K5 for 4:2:0 chroma).
//
// Arithmetic contract (bit-exact with oracle/jpeg_oracle.c): 13-bit fixed-point "ISLOW" butterflies with the
// IJG constants, round-half-away quantisation, IJG range-limit wrap.  All work is integer ALU + HBM streaming,
// so there is deliberately no tensor-core path; the design rules are: one thread owns one 8x8 block in 64
// registers (no shuffles, no transposes -- de-zigzag and zigzag are register renames), 128-bit coalesced
// global accesses staged through conflict-free padded shared memory, tables broadcast from shared memory.
#include <cuda_runtime.h>
#include <cstdint>
#include "jpeg_kernels.h"
#include "jpeg_trellis_core.h"

namespace b200 {

#define FIX_0_298631336 2446
#define FIX_0_390180644 3196
#define FIX_0_541196100 4433
#define FIX_0_765366865 6270
#define FIX_0_899976223 7373
#define FIX_1_175875602 9633
#define FIX_1_501321110 12299
#define FIX_1_847759065 15137
#define FIX_1_961570560 16069
#define FIX_2_053119869 16819
#define FIX_2_562915447 20995
#define FIX_3_072711026 25172

// X(k, n): zigzag index k <-> natural (row-major) position n
#define ZZ_LIST(X) \
    X(0,0) X(1,1) X(2,8) X(3,16) X(4,9) X(5,2) X(6,3) X(7,10) \
    X(8,17) X(9,24) X(10,32) X(11,25) X(12,18) X(13,11) X(14,4) X(15,5) \
    X(16,12) X(17,19) X(18,26) X(19,33) X(20,40) X(21,48) X(22,41) X(23,34) \
    X(24,27) X(25,20) X(26,13) X(27,6) X(28,7) X(29,14) X(30,21) X(31,28) \
    X(32,35) X(33,42) X(34,49) X(35,56) X(36,57) X(37,50) X(38,43) X(39,36) \
    X(40,29) X(41,22) X(42,15) X(43,23) X(44,30) X(45,37) X(46,44) X(47,51) \
    X(48,58) X(49,59) X(50,52) X(51,45) X(52,38) X(53,31) X(54,39) X(55,46) \
    X(56,53) X(57,60) X(58,61) X(59,54) X(60,47) X(61,55) X(62,62) X(63,63)

constexpr int WARPS_PER_CTA = 8;
constexpr int THREADS = WARPS_PER_CTA * 32;
constexpr int BLOCKS_PER_CTA = THREADS;       // one 8x8 block per thread
constexpr int STAGE_INT4_PER_WARP = 32 * 9;   // 32 blocks x (8 + 1 pad) int4 -> 144 B pitch, conflict-free

template <int N> __device__ __forceinline__ int descale(int x) { return (x + (1 << (N - 1))) >> N; }

// 1-D inverse butterfly of jidctint.c; SHIFT = CONST_BITS - PASS1_BITS (11) in pass 1, CONST_BITS + PASS1_BITS + 3 (18) in pass 2
// IDCT_range_limit[(x >> SHIFT) & 1023] as an UNCENTRED sample 0..255; x already carries the rounding constant
template <int SHIFT> __device__ __forceinline__ int sample_of(int x)
{
    const int w = (int)((unsigned)x << (22 - SHIFT)) >> 22;          // the descaled value, wrapped to 10 signed bits
    return __viaddmin_s32_relu(w, 128, 255);                         // max(min(w + 128, 255), 0)
}

template <int SHIFT, bool SAMPLES = false>
__device__ __forceinline__ void idct8(int &d0, int &d1, int &d2, int &d3, int &d4, int &d5, int &d6, int &d7)
{
    constexpr int R = 1 << (SHIFT - 1);         // the descale's rounding constant rides in on the even part (one multiply-add)
    int z1 = (d2 + d6) * FIX_0_541196100;
    int t2 = z1 + d6 * (-FIX_1_847759065);
    int t3 = z1 + d2 * FIX_0_765366865;
    int t0 = (d0 + d4) * 8192 + R, t1 = (d0 - d4) * 8192 + R;
    int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    int o0 = d7, o1 = d5, o2 = d3, o3 = d1;
    z1 = o0 + o3; int z2 = o1 + o2, z3 = o0 + o2, z4 = o1 + o3;
    int z5 = (z3 + z4) * FIX_1_175875602;
    o0 *= FIX_0_298631336; o1 *= FIX_2_053119869; o2 *= FIX_3_072711026; o3 *= FIX_1_501321110;
    z1 *= -FIX_0_899976223; z2 *= -FIX_2_562915447; z3 *= -FIX_1_961570560; z4 *= -FIX_0_390180644;
    z3 += z5; z4 += z5;
    o0 += z1 + z3; o1 += z2 + z4; o2 += z2 + z3; o3 += z1 + z4;
    if (!SAMPLES) {
        d0 = (t10 + o3) >> SHIFT; d7 = (t10 - o3) >> SHIFT;
        d1 = (t11 + o2) >> SHIFT; d6 = (t11 - o2) >> SHIFT;
        d2 = (t12 + o1) >> SHIFT; d5 = (t12 - o1) >> SHIFT;
        d3 = (t13 + o0) >> SHIFT; d4 = (t13 - o0) >> SHIFT;
    } else {
        // pass 2 ends in IDCT_range_limit[(x >> SHIFT) & RANGE_MASK]: the descale, the 10-bit wrap and the clamp as
        // (x + round) << (22 - SHIFT) >> 22 (sign-extends bit 9 of the descaled value) and one add-min-relu to [0, 255]
        d0 = sample_of<SHIFT>(t10 + o3); d7 = sample_of<SHIFT>(t10 - o3);
        d1 = sample_of<SHIFT>(t11 + o2); d6 = sample_of<SHIFT>(t11 - o2);
        d2 = sample_of<SHIFT>(t12 + o1); d5 = sample_of<SHIFT>(t12 - o1);
        d3 = sample_of<SHIFT>(t13 + o0); d4 = sample_of<SHIFT>(t13 - o0);
    }
}

// 1-D forward butterfly of jfdctint.c.  PASS 1: outputs scaled up by PASS1_BITS; PASS 2: scaled back down.
template <int PASS>
__device__ __forceinline__ void fdct8(int &d0, int &d1, int &d2, int &d3, int &d4, int &d5, int &d6, int &d7)
{
    constexpr int SH = PASS == 1 ? 11 : 15, R = 1 << (SH - 1);       // rounding constants folded into the multiply-adds
    int t0 = d0 + d7, t7 = d0 - d7, t1 = d1 + d6, t6 = d1 - d6;
    int t2 = d2 + d5, t5 = d2 - d5, t3 = d3 + d4, t4 = d3 - d4;
    int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    if (PASS == 1) { d0 = (t10 + t11) * 4; d4 = (t10 - t11) * 4; }
    else           { d0 = (t10 + t11 + 2) >> 2; d4 = (t10 - t11 + 2) >> 2; }
    int z1 = (t12 + t13) * FIX_0_541196100 + R;
    d2 = (z1 + t13 * FIX_0_765366865) >> SH;
    d6 = (z1 + t12 * (-FIX_1_847759065)) >> SH;
    z1 = t4 + t7; int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
    int z5 = (z3 + z4) * FIX_1_175875602 + R;
    t4 *= FIX_0_298631336; t5 *= FIX_2_053119869; t6 *= FIX_3_072711026; t7 *= FIX_1_501321110;
    z1 *= -FIX_0_899976223; z2 *= -FIX_2_562915447; z3 *= -FIX_1_961570560; z4 *= -FIX_0_390180644;
    z3 += z5; z4 += z5;
    d7 = (t4 + z1 + z3) >> SH; d5 = (t5 + z2 + z4) >> SH;
    d3 = (t6 + z2 + z3) >> SH; d1 = (t7 + z1 + z4) >> SH;
}

struct Tables {
    uint16_t dq[64];
    uint2 mc[64];           // (m, c) of QuantDev, one 8-byte shared-memory read per coefficient
    uint32_t kpair[32];
    uint8_t sh[64];
    uint32_t any_shift;
};

__device__ __forceinline__ void load_tables(Tables &t, const CompWork &w, bool need_dq, bool need_q)
{
    int i = threadIdx.x;
    if (i < 64) {
        if (need_dq) t.dq[i] = w.dq[i];
        if (need_q) { t.mc[i] = make_uint2(w.q->m[i], w.q->c[i]); t.sh[i] = w.q->sh[i]; if (i < 32) t.kpair[i] = w.q->kpair[i]; if (i == 0) t.any_shift = w.q->any_shift; }
    }
    __syncthreads();
}

// Row-aligned tiling: a warp owns up to 32 consecutive blocks of ONE block row, a CTA owns 8 consecutive tiles.
struct Tile { int by, bx0, nvalid; bool active, cta_idle; };
__device__ __forceinline__ Tile tile_of(int rbw, int rbh)
{
    Tile t;
    const int tpr = (rbw + 31) >> 5, ntiles = tpr * rbh;
    const int tile = blockIdx.x * WARPS_PER_CTA + (threadIdx.x >> 5);
    t.cta_idle = (int)blockIdx.x * WARPS_PER_CTA >= ntiles;
    t.active = tile < ntiles;
    t.by = tile / tpr;
    t.bx0 = (tile - t.by * tpr) * 32;
    t.nvalid = min(32, rbw - t.bx0);
    return t;
}

// Warp-cooperative load of up to 32 consecutive blocks (128 B each) with coalesced 16 B accesses; lane L ends up
// holding block L in r[0..7].  `g` points at the first block of the warp's tile.
__device__ __forceinline__ void warp_load_blocks(const int4 *__restrict__ g, int nvalid, int4 *stage, int lane, int4 (&r)[8])
{
    int4 tmp[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        int chunk = i * 32 + lane;
        tmp[i] = (chunk >> 3) < nvalid ? __ldg(g + chunk) : make_int4(0, 0, 0, 0);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) {
        int chunk = i * 32 + lane;
        stage[(chunk >> 3) * 9 + (chunk & 7)] = tmp[i];
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 8; j++) r[j] = stage[lane * 9 + j];
    __syncwarp();
}

__device__ __forceinline__ void warp_store_blocks(int4 *__restrict__ g, int nvalid, int4 *stage, int lane, const int4 (&r)[8])
{
#pragma unroll
    for (int j = 0; j < 8; j++) stage[lane * 9 + j] = r[j];
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 8; i++) {
        int chunk = i * 32 + lane;
        if ((chunk >> 3) < nvalid) g[chunk] = stage[(chunk >> 3) * 9 + (chunk & 7)];
    }
    __syncwarp();
}

// A block read from a deferred-DC decode (w.dc_sum set) carries its DC difference: put the DC from the decoder's prefix sums in its
// place (the low half of the first word, truncated to int16 as the DC scatter would store it).  bx, by: the block in the component.
__device__ __forceinline__ void put_dc(const CompWork &w, int bx, int by, int4 (&r)[8])
{
    const int mx = bx / w.dc_hs, my = by / w.dc_vs;
    const int slot = (my * w.dc_mcux + mx) * (w.dc_hs * w.dc_vs) + (by - my * w.dc_vs) * w.dc_hs + (bx - mx * w.dc_hs);
    const int dc = __ldg(w.dc_sum + slot) - (w.dc_prev ? __ldg(w.dc_prev) : 0);
    r[0].x = (int)(((uint32_t)r[0].x & 0xFFFF0000u) | ((uint32_t)dc & 0xFFFFu));
}

// zigzag quantised int16 block (8 x int4) -> dequantised natural-order ints
__device__ __forceinline__ void dequant_dezigzag(const int4 (&r)[8], const Tables &t, int (&v)[64])
{
    int cw[32];
#pragma unroll
    for (int j = 0; j < 8; j++) { cw[4 * j] = r[j].x; cw[4 * j + 1] = r[j].y; cw[4 * j + 2] = r[j].z; cw[4 * j + 3] = r[j].w; }
#define X(k, n) v[n] = (((k) & 1) ? (cw[(k) >> 1] >> 16) : (int)(short)(cw[(k) >> 1] & 0xFFFF)) * (int)t.dq[k];
    ZZ_LIST(X)
#undef X
}

// v: dequantised coefficients (natural order) -> samples 0..255 in place
__device__ __forceinline__ void idct_block(int (&v)[64])
{
#pragma unroll
    for (int c = 0; c < 8; c++) idct8<11>(v[c], v[8 + c], v[16 + c], v[24 + c], v[32 + c], v[40 + c], v[48 + c], v[56 + c]);
#pragma unroll
    for (int r = 0; r < 8; r++) idct8<18, true>(v[8 * r], v[8 * r + 1], v[8 * r + 2], v[8 * r + 3], v[8 * r + 4], v[8 * r + 5], v[8 * r + 6], v[8 * r + 7]);
}

// v: samples 0..255 -> forward DCT (scaled by 8) of the CENTRED samples, in place.  jcdctmgr.c subtracts CENTERJSAMPLE first;
// the butterflies are linear and every output but DC is built from differences, so running them on the uncentred samples adds
// exactly 8 * 128 * 8 = 8192 to v[0] (row pass: +4096 in column 0 only; column pass: (x + 32768 + 2) >> 2) and nothing else.
__device__ __forceinline__ void fdct_block(int (&v)[64])
{
#pragma unroll
    for (int r = 0; r < 8; r++) fdct8<1>(v[8 * r], v[8 * r + 1], v[8 * r + 2], v[8 * r + 3], v[8 * r + 4], v[8 * r + 5], v[8 * r + 6], v[8 * r + 7]);
#pragma unroll
    for (int c = 0; c < 8; c++) fdct8<2>(v[c], v[8 + c], v[16 + c], v[24 + c], v[32 + c], v[40 + c], v[48 + c], v[56 + c]);
    v[0] -= 8192;
}

// DCT output (natural order) -> quantised zigzag int16 block packed into 8 x int4 (QuantDev: biased sign-free division)
template <bool SHIFT>
__device__ __forceinline__ void quant_zigzag_t(const int (&v)[64], const Tables &t, int4 (&r)[8])
{
    uint32_t ow[32];
#define X(k, n) { const uint2 mc = t.mc[k]; const uint32_t qb = quant_biased(v[n], mc.x, mc.y, SHIFT ? (uint32_t)t.sh[k] : 0u); \
                  if ((k) & 1) ow[(k) >> 1] = quant_pack(ow[(k) >> 1], qb, t.kpair[(k) >> 1]); else ow[(k) >> 1] = qb; }
    ZZ_LIST(X)
#undef X
#pragma unroll
    for (int j = 0; j < 8; j++) r[j] = make_int4((int)ow[4 * j], (int)ow[4 * j + 1], (int)ow[4 * j + 2], (int)ow[4 * j + 3]);
}
__device__ __forceinline__ void quant_zigzag(const int (&v)[64], const Tables &t, int4 (&r)[8])
{
    if (t.any_shift) quant_zigzag_t<true>(v, t, r); else quant_zigzag_t<false>(v, t, r);     // block-uniform branch
}
// RAW: the unquantised DCT output (|v| <= 2^13 for 8-bit samples) as zigzag int16, for k_jpeg_trellis to quantise in place
template <bool RAW>
__device__ __forceinline__ void store_zigzag(const int (&v)[64], const Tables &t, int4 (&r)[8])
{
    if (!RAW) { quant_zigzag(v, t, r); return; }
    uint32_t ow[32];
#define X(k, n) if ((k) & 1) ow[(k) >> 1] |= (uint32_t)v[n] << 16; else ow[(k) >> 1] = (uint32_t)v[n] & 0xFFFFu;
    ZZ_LIST(X)
#undef X
#pragma unroll
    for (int j = 0; j < 8; j++) r[j] = make_int4((int)ow[4 * j], (int)ow[4 * j + 1], (int)ow[4 * j + 2], (int)ow[4 * j + 3]);
}

// ------------------------------------------------------------------------------------------------------------
// K1->K5 fused: components whose sample grid is unchanged between decode and encode (luma always; chroma too when
// neither side subsamples).  coefficients in -> coefficients out, 6 algorithmic bytes... per sample 4 B.
// ------------------------------------------------------------------------------------------------------------
template <bool RAW>
__global__ void __launch_bounds__(THREADS, 2) k_fused_same(const CompWork *__restrict__ work)
{
    __shared__ Tables tab;
    __shared__ int4 stage[WARPS_PER_CTA * STAGE_INT4_PER_WARP];
    const CompWork w = work[blockIdx.y];
    const Tile t = tile_of(w.rbw_out, w.rbh_out);
    if (t.cta_idle) return;
    load_tables(tab, w, true, true);
    if (!t.active) return;
    const int lane = threadIdx.x & 31;
    int4 *st = stage + (threadIdx.x >> 5) * STAGE_INT4_PER_WARP;
    int4 r[8];
    warp_load_blocks(reinterpret_cast<const int4 *>(w.cin) + ((size_t)t.by * w.bw_in + t.bx0) * 8, t.nvalid, st, lane, r);
    if (w.dc_sum && lane < t.nvalid) put_dc(w, t.bx0 + lane, t.by, r);
    int v[64];
    dequant_dezigzag(r, tab, v);
    idct_block(v);
    // The decoder crops to W x H and the encoder re-pads by edge replication (jcsample.c expand_right_edge,
    // jcprepct.c expand_bottom_edge): blocks straddling the right / bottom image edge lose their decoded padding.
    const int vc = w.cw - (t.bx0 + lane) * 8, vr = w.ch - t.by * 8;
    if (vc < 8 || vr < 8) {
#pragma unroll
        for (int y = 0; y < 8; y++)
#pragma unroll
            for (int x = 1; x < 8; x++) if (x >= vc) v[8 * y + x] = v[8 * y + x - 1];
#pragma unroll
        for (int y = 1; y < 8; y++)
#pragma unroll
            for (int x = 0; x < 8; x++) if (y >= vr) v[8 * y + x] = v[8 * (y - 1) + x];
    }
    fdct_block(v);
    store_zigzag<RAW>(v, tab, r);
    warp_store_blocks(reinterpret_cast<int4 *>(w.cout) + ((size_t)t.by * w.bw_out + t.bx0) * 8, t.nvalid, st, lane, r);
}

// ------------------------------------------------------------------------------------------------------------
// K1: dequant + IDCT -> u8 component plane (row pitch pstride = bw_in * 8)
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(THREADS) k_idct_plane(const CompWork *__restrict__ work)
{
    __shared__ Tables tab;
    __shared__ int4 stage[WARPS_PER_CTA * STAGE_INT4_PER_WARP];
    const CompWork w = work[blockIdx.y];
    const Tile t = tile_of(w.rbw_in, w.rbh_in);
    if (t.cta_idle) return;
    load_tables(tab, w, true, false);
    if (!t.active) return;
    const int lane = threadIdx.x & 31;
    int4 r[8];
    warp_load_blocks(reinterpret_cast<const int4 *>(w.cin) + ((size_t)t.by * w.bw_in + t.bx0) * 8, t.nvalid, stage + (threadIdx.x >> 5) * STAGE_INT4_PER_WARP, lane, r);
    if (lane >= t.nvalid) return;
    if (w.dc_sum) put_dc(w, t.bx0 + lane, t.by, r);
    int v[64];
    dequant_dezigzag(r, tab, v);
    idct_block(v);
    uint8_t *p = w.plane + (size_t)(t.by * 8) * w.pstride + (t.bx0 + lane) * 8;
#pragma unroll
    for (int y = 0; y < 8; y++) {
        uint32_t lo = (uint32_t)v[8 * y] | ((uint32_t)v[8 * y + 1] << 8) | ((uint32_t)v[8 * y + 2] << 16) | ((uint32_t)v[8 * y + 3] << 24);
        uint32_t hi = (uint32_t)v[8 * y + 4] | ((uint32_t)v[8 * y + 5] << 8) | ((uint32_t)v[8 * y + 6] << 16) | ((uint32_t)v[8 * y + 7] << 24);
        *reinterpret_cast<uint2 *>(p + (size_t)y * w.pstride) = make_uint2(lo, hi);   // lanes -> consecutive 8 B: coalesced
    }
}

// ------------------------------------------------------------------------------------------------------------
// K2 o K4 o K5 for 4:2:0 -> 4:2:0 chroma: the decoder's h2v2 "fancy" upsample (jdsample.c) followed by the
// encoder's h2v2 box downsample (jcsample.c) collapses to a 3x3 stencil on the decoded chroma plane, evaluated
// here on the fly in front of the forward DCT.  Interior blocks take the register/shuffle fast path; blocks that
// touch an image edge evaluate the generic clamped formulas.
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int up_h2v2(const uint8_t *__restrict__ P, int pstride, int cw, int ch, int y, int x)
{   // one full-resolution sample of h2v2_fancy_upsample (box replication when cw <= 2, as jinit_upsampler decides)
    int r = y >> 1, c = x >> 1;
    r = min(r, ch - 1); c = min(c, cw - 1);
    if (cw <= 2) return P[(size_t)r * pstride + c];
    int rn = (y & 1) ? min(r + 1, ch - 1) : max(r - 1, 0);
    int cn = (x & 1) ? min(c + 1, cw - 1) : max(c - 1, 0);
    int a = 3 * P[(size_t)r * pstride + c] + P[(size_t)rn * pstride + c];
    int b = 3 * P[(size_t)r * pstride + cn] + P[(size_t)rn * pstride + cn];
    return (3 * a + b + ((x & 1) ? 7 : 8)) >> 4;
}

// generic clamped evaluation of one 8x8 output block (image edges, odd dimensions, tiny planes) following the
// jcprepct/jcsample padding rules (oracle orc_downsample); results are written as bytes to `mine` (64 B)
__device__ __noinline__ void chroma420_edge_block(const CompWork &w, int bx, int by, uint8_t *mine)
{
    const uint8_t *__restrict__ P = w.plane;
    const int ps = w.pstride, nreal = (w.H + 1) >> 1;
    for (int i = 0; i < 64; i++) {
        int Y = i >> 3, X = i & 7;
        int yy = min(by * 8 + Y, nreal - 1);
        int y0 = min(2 * yy, w.H - 1), y1 = min(2 * yy + 1, w.H - 1);
        int xo = bx * 8 + X;
        int x0 = min(2 * xo, w.W - 1), x1 = min(2 * xo + 1, w.W - 1);
        int s = up_h2v2(P, ps, w.cw, w.ch, y0, x0) + up_h2v2(P, ps, w.cw, w.ch, y0, x1)
              + up_h2v2(P, ps, w.cw, w.ch, y1, x0) + up_h2v2(P, ps, w.cw, w.ch, y1, x1);
        mine[i] = (uint8_t)((s + 1 + (xo & 1)) >> 2);
    }
}

template <bool RAW>
__global__ void __launch_bounds__(THREADS, 2) k_chroma420_refdct(const CompWork *__restrict__ work)
{
    __shared__ Tables tab;
    __shared__ int4 stage[WARPS_PER_CTA * STAGE_INT4_PER_WARP];
    const CompWork w = work[blockIdx.y];
    const Tile t = tile_of(w.rbw_out, w.rbh_out);
    if (t.cta_idle) return;
    load_tables(tab, w, false, true);
    if (!t.active) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int by = t.by, bx = min(t.bx0 + lane, w.rbw_out - 1);
    const uint8_t *__restrict__ P = w.plane;
    const int ps = w.pstride;
    // The register fast path is exact whenever every clamp of the generic formulas degenerates to "replicate the
    // nearest decoded sample": the block lies wholly inside the decoded plane and, if it is the last block column /
    // row, the image width / height is even (then x1 = 2X+1 and y1 = 2Y+1 never clamp).  Left and top edges always
    // replicate.  Everything else (partial edge blocks, odd sizes, planes <= 2 samples wide) takes the generic path.
    const bool fast = w.cw > 2 && bx * 8 + 8 <= w.cw && by * 8 + 8 <= w.ch &&
                      (bx * 8 + 8 < w.cw || 2 * w.cw == w.W) && (by * 8 + 8 < w.ch || 2 * w.ch == w.H);
    int v[64];
    int pL = 0, pM0 = 0, pM1 = 0, pR = 0, cL = 0, cM0 = 0, cM1 = 0, cR = 0;
    const bool edge_r = lane == 31 || lane == t.nvalid - 1;
#pragma unroll
    for (int rr = 0; rr < 10; rr++) {
        const int gy = min(max(by * 8 + rr - 1, 0), w.ch - 1);
        const uint8_t *row = P + (size_t)gy * ps;
        const uint2 m = __ldg(reinterpret_cast<const uint2 *>(row + bx * 8));
        int nL = __shfl_up_sync(0xFFFFFFFFu, (int)(m.y >> 24), 1);
        int nR = __shfl_down_sync(0xFFFFFFFFu, (int)(m.x & 0xFF), 1);
        if (lane == 0) nL = row[max(bx * 8 - 1, 0)];
        if (edge_r) nR = row[min(bx * 8 + 8, w.cw - 1)];
        const int nM0 = (int)m.x, nM1 = (int)m.y;
        if (rr >= 2) {
            // output row Y = rr - 2 uses plane rows (p, c, n) = (Y-1, Y, Y+1) of the block; su/sl are the column sums of
            // the upper (y = 2Y: rows Y, Y-1) and lower (y = 2Y+1: rows Y, Y+1) full-resolution rows, columns -1..8
            const int Y = rr - 2;
            int su[10], sl[10];
            su[0] = 3 * cL + pL; sl[0] = 3 * cL + nL;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const int c0 = (cM0 >> (8 * k)) & 0xFF, c1 = (cM1 >> (8 * k)) & 0xFF;
                su[1 + k] = 3 * c0 + ((pM0 >> (8 * k)) & 0xFF); sl[1 + k] = 3 * c0 + ((nM0 >> (8 * k)) & 0xFF);
                su[5 + k] = 3 * c1 + ((pM1 >> (8 * k)) & 0xFF); sl[5 + k] = 3 * c1 + ((nM1 >> (8 * k)) & 0xFF);
            }
            su[9] = 3 * cR + pR; sl[9] = 3 * cR + nR;
#pragma unroll
            for (int X = 0; X < 8; X++) {
                // full-res x0 = 2X (even: neighbour column X-1, bias 8), x1 = 2X+1 (odd: neighbour X+1, bias 7)
                const int tu = 3 * su[X + 1], tl = 3 * sl[X + 1];
                const int u00 = (tu + su[X] + 8) >> 4, u01 = (tu + su[X + 2] + 7) >> 4;
                const int u10 = (tl + sl[X] + 8) >> 4, u11 = (tl + sl[X + 2] + 7) >> 4;
                v[8 * Y + X] = (u00 + u01 + u10 + u11 + 1 + (X & 1)) >> 2;   // bias 1,2,1,2 across output columns
            }
        }
        pL = cL; pM0 = cM0; pM1 = cM1; pR = cR;
        cL = nL; cM0 = nM0; cM1 = nM1; cR = nR;
    }
    if (!fast) {
        uint8_t *mine = reinterpret_cast<uint8_t *>(stage + warp * STAGE_INT4_PER_WARP) + lane * 68;
        chroma420_edge_block(w, bx, by, mine);
#pragma unroll
        for (int j = 0; j < 16; j++) {
            uint32_t m4 = *reinterpret_cast<const uint32_t *>(mine + 4 * j);
#pragma unroll
            for (int k = 0; k < 4; k++) v[4 * j + k] = (int)((m4 >> (8 * k)) & 0xFF);
        }
    }
    __syncwarp();
    fdct_block(v);
    int4 r[8];
    store_zigzag<RAW>(v, tab, r);
    warp_store_blocks(reinterpret_cast<int4 *>(w.cout) + ((size_t)t.by * w.bw_out + t.bx0) * 8, t.nvalid, stage + warp * STAGE_INT4_PER_WARP, lane, r);
}

// ------------------------------------------------------------------------------------------------------------
// Generic path pieces (any supported sampling combination; also the front/back ends of the resize path)
// ------------------------------------------------------------------------------------------------------------
__global__ void k_upsample(const CompWork *__restrict__ work)
{   // K2: component plane -> full-resolution plane (jdsample.c method selection of jinit_upsampler)
    const CompWork w = work[blockIdx.z];
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w.W || y >= w.H) return;
    const uint8_t *__restrict__ P = w.plane; const int ps = w.pstride, cw = w.cw, ch = w.ch;
    int out;
    if (w.up_hx == 1 && w.up_vx == 1) out = P[(size_t)y * ps + x];
    else if (w.up_hx == 2 && w.up_vx == 2) out = up_h2v2(P, ps, cw, ch, y, x);
    else if (w.up_hx == 2 && w.up_vx == 1 && cw > 2) {
        int c = x >> 1, r = min(y, ch - 1), cn = (x & 1) ? min(c + 1, cw - 1) : max(c - 1, 0);
        out = (3 * P[(size_t)r * ps + c] + P[(size_t)r * ps + cn] + ((x & 1) ? 2 : 1)) >> 2;
    } else if (w.up_hx == 1 && w.up_vx == 2) {
        int r = y >> 1, rn = (y & 1) ? min(r + 1, ch - 1) : max(r - 1, 0), c = min(x, cw - 1);
        out = (3 * P[(size_t)r * ps + c] + P[(size_t)rn * ps + c] + ((y & 1) ? 2 : 1)) >> 2;
    } else out = P[(size_t)min(y / w.up_vx, ch - 1) * ps + min(x / w.up_hx, cw - 1)];
    w.full[(size_t)y * w.fstride + x] = (uint8_t)out;
}

__global__ void k_downsample(const CompWork *__restrict__ work)
{   // K4: full-resolution plane -> padded component plane (jcsample.c + jcprepct.c edge rules)
    const CompWork w = work[blockIdx.z];
    const int pw = w.rbw_out * 8, ph = w.rbh_out * 8;
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= pw || y >= ph) return;
    const int hx = w.dn_hx, vx = w.dn_vx;
    const int nreal = (w.H + vx - 1) / vx;
    const int yy = min(y, nreal - 1);
    int sum = 0;
    for (int dy = 0; dy < vx; dy++) {
        const uint8_t *row = w.full + (size_t)min(yy * vx + dy, w.H - 1) * w.fstride;
        for (int dx = 0; dx < hx; dx++) sum += row[min(x * hx + dx, w.W - 1)];
    }
    int v;
    if (hx == 1 && vx == 1) v = sum;
    else if (hx == 2 && vx == 1) v = (sum + (x & 1)) >> 1;
    else if (hx == 2 && vx == 2) v = (sum + 1 + (x & 1)) >> 2;
    else { int n = hx * vx; v = (sum + n / 2) / n; }
    w.dplane[(size_t)y * pw + x] = (uint8_t)v;
}

template <bool RAW>
__global__ void __launch_bounds__(THREADS) k_fdct_plane(const CompWork *__restrict__ work)
{   // K5: padded component plane -> quantised zigzag coefficients
    __shared__ Tables tab;
    __shared__ int4 stage[WARPS_PER_CTA * STAGE_INT4_PER_WARP];
    const CompWork w = work[blockIdx.y];
    const Tile t = tile_of(w.rbw_out, w.rbh_out);
    if (t.cta_idle) return;
    load_tables(tab, w, false, true);
    if (!t.active) return;
    const int lane = threadIdx.x & 31;
    const int by = t.by, bx = min(t.bx0 + lane, w.rbw_out - 1);
    const int pw = w.rbw_out * 8;
    int v[64];
#pragma unroll
    for (int y = 0; y < 8; y++) {
        uint2 m = __ldg(reinterpret_cast<const uint2 *>(w.dplane + (size_t)(by * 8 + y) * pw + bx * 8));
#pragma unroll
        for (int k = 0; k < 4; k++) { v[8 * y + k] = (int)((m.x >> (8 * k)) & 0xFF); v[8 * y + 4 + k] = (int)((m.y >> (8 * k)) & 0xFF); }
    }
    fdct_block(v);
    int4 r[8];
    store_zigzag<RAW>(v, tab, r);
    warp_store_blocks(reinterpret_cast<int4 *>(w.cout) + ((size_t)t.by * w.bw_out + t.bx0) * 8, t.nvalid, stage + (threadIdx.x >> 5) * STAGE_INT4_PER_WARP, lane, r);
}

// ------------------------------------------------------------------------------------------------------------
// Trellis quantisation (jpeg_trellis_core.h) of the raw DCT output the RAW transform kernels left in cout, in place, real blocks
// only.  One thread per block.  The programme's per-position arrays live in shared memory as [position][thread], so the 64
// threads of a CTA touch one 8-byte word (G) or one byte (pos, pred, size) each at whatever position they have reached: G stays
// conflict-free (bank = thread), and registers stay free of dynamically indexed arrays that would spill to local memory.
// 64 x (8 + 3) B x 64 threads = 44 KB + the table: under the 48 KB static limit.  The block is read from and written back to
// global memory in place (each thread owns its 128 B; the reads of one position across a warp hit L1).
// ------------------------------------------------------------------------------------------------------------
constexpr int TRELLIS_THREADS = 64;
__global__ void __launch_bounds__(TRELLIS_THREADS) k_jpeg_trellis(const CompWork *__restrict__ work, const QuantDev *qbase, const JtTable *__restrict__ tables)
{
    __shared__ long long G[64 * TRELLIS_THREADS];
    __shared__ uint8_t pos[64 * TRELLIS_THREADS], pred[64 * TRELLIS_THREADS], size[64 * TRELLIS_THREADS];
    __shared__ JtTable tab;
    const CompWork w = work[blockIdx.y];
    const int nblk = w.rbw_out * w.rbh_out;
    if ((int)blockIdx.x * TRELLIS_THREADS >= nblk) return;
    {
        const JtTable *src = tables + (w.q - qbase);
        const uint32_t *s4 = reinterpret_cast<const uint32_t *>(src);
        uint32_t *d4 = reinterpret_cast<uint32_t *>(&tab);
        for (int i = threadIdx.x; i < (int)(sizeof(JtTable) / 4); i += TRELLIS_THREADS) d4[i] = s4[i];
    }
    __syncthreads();
    const int i = blockIdx.x * TRELLIS_THREADS + threadIdx.x;
    if (i >= nblk) return;
    const int by = i / w.rbw_out, bx = i - by * w.rbw_out;
    int16_t *blk = w.cout + ((size_t)by * w.bw_out + bx) * 64;
    const int t = threadIdx.x;
    jt_trellis_block(blk, &tab, blk, G + t, pos + t, pred + t, size + t, TRELLIS_THREADS);
}

// ------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------
static inline int cdiv(int a, int b) { return (a + b - 1) / b; }

int launch_fused_same(const CompWork *work, int n, int max_tiles, void *stream, bool raw)
{
    if (n <= 0 || max_tiles <= 0) return 0;
    dim3 grid(cdiv(max_tiles, WARPS_PER_CTA), n);
    if (raw) k_fused_same<true><<<grid, THREADS, 0, (cudaStream_t)stream>>>(work);
    else k_fused_same<false><<<grid, THREADS, 0, (cudaStream_t)stream>>>(work);
    return (int)cudaGetLastError();
}
int launch_idct_plane(const CompWork *work, int n, int max_tiles, void *stream)
{
    if (n <= 0 || max_tiles <= 0) return 0;
    dim3 grid(cdiv(max_tiles, WARPS_PER_CTA), n);
    k_idct_plane<<<grid, THREADS, 0, (cudaStream_t)stream>>>(work);
    return (int)cudaGetLastError();
}
int launch_chroma420_refdct(const CompWork *work, int n, int max_tiles, void *stream, bool raw)
{
    if (n <= 0 || max_tiles <= 0) return 0;
    dim3 grid(cdiv(max_tiles, WARPS_PER_CTA), n);
    if (raw) k_chroma420_refdct<true><<<grid, THREADS, 0, (cudaStream_t)stream>>>(work);
    else k_chroma420_refdct<false><<<grid, THREADS, 0, (cudaStream_t)stream>>>(work);
    return (int)cudaGetLastError();
}
int launch_upsample(const CompWork *work, int n, int max_w, int max_h, void *stream)
{
    if (n <= 0 || max_w <= 0 || max_h <= 0) return 0;
    dim3 blk(64, 4), grid(cdiv(max_w, 64), cdiv(max_h, 4), n);
    k_upsample<<<grid, blk, 0, (cudaStream_t)stream>>>(work);
    return (int)cudaGetLastError();
}
int launch_downsample(const CompWork *work, int n, int max_w, int max_h, void *stream)
{
    if (n <= 0 || max_w <= 0 || max_h <= 0) return 0;
    dim3 blk(64, 4), grid(cdiv(max_w, 64), cdiv(max_h, 4), n);
    k_downsample<<<grid, blk, 0, (cudaStream_t)stream>>>(work);
    return (int)cudaGetLastError();
}
int launch_fdct_plane(const CompWork *work, int n, int max_tiles, void *stream, bool raw)
{
    if (n <= 0 || max_tiles <= 0) return 0;
    dim3 grid(cdiv(max_tiles, WARPS_PER_CTA), n);
    if (raw) k_fdct_plane<true><<<grid, THREADS, 0, (cudaStream_t)stream>>>(work);
    else k_fdct_plane<false><<<grid, THREADS, 0, (cudaStream_t)stream>>>(work);
    return (int)cudaGetLastError();
}
int launch_jpeg_trellis(const CompWork *work, int n, int max_blocks, const QuantDev *qbase, const JtTable *tables, void *stream)
{
    if (n <= 0 || max_blocks <= 0) return 0;
    dim3 grid(cdiv(max_blocks, TRELLIS_THREADS), n);
    k_jpeg_trellis<<<grid, TRELLIS_THREADS, 0, (cudaStream_t)stream>>>(work, qbase, tables);
    return (int)cudaGetLastError();
}
int launch_memset_warm(void *p, size_t n, void *stream)
{
    return (int)cudaMemsetAsync(p, 0, n, (cudaStream_t)stream);
}

} // namespace b200
