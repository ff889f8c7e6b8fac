// vp8_kernels.cu -- K8, see vp8_kernels.h.  Intra prediction makes a macroblock depend on its left, top and top-left
// neighbours' RECONSTRUCTION, so the frame is swept as a wavefront: one warp owns one macroblock row and trails the row above
// by one macroblock (progress counters in global memory, rows handed out by ticket so a waiting warp only ever waits on a
// warp that is already running).  Inside a macroblock nothing is sequential with 16x16 prediction: lane k < 16 owns luma
// 4x4 block k, lanes 16..19 / 20..23 own the U / V blocks, lane 24 does the 16-point Walsh-Hadamard of the luma DCs.
// Integer arithmetic only; every inverse step is the normative RFC 6386 one, so a decoder reproduces RY/RU/RV exactly.
#include <cuda_runtime.h>
#include <cub/device/device_scan.cuh>
#include <cstdint>
#include "vp8_kernels.h"
#include "vp8_tokens_core.h"
#include "vp8_bpred_core.h"

namespace b200 {

namespace {

constexpr unsigned FULL = 0xffffffffu;
__device__ __forceinline__ int clip8(int v) { return v < 0 ? 0 : v > 255 ? 255 : v; }

__global__ void k_vp8_rgb_to_yuv(const uint8_t *__restrict__ r, const uint8_t *__restrict__ g, const uint8_t *__restrict__ b, int w, int h,
                                 uint8_t *__restrict__ Y, uint8_t *__restrict__ U, uint8_t *__restrict__ V, int cw, int chh)
{
    const int cx = blockIdx.x * blockDim.x + threadIdx.x, cy = blockIdx.y * blockDim.y + threadIdx.y;
    if (cx >= cw || cy >= chh) return;
    int R = 0, G = 0, B = 0;
#pragma unroll
    for (int dy = 0; dy < 2; dy++)
#pragma unroll
        for (int dx = 0; dx < 2; dx++) {
            const int x = 2 * cx + dx, y = 2 * cy + dy;
            const size_t i = (size_t)min(y, h - 1) * w + min(x, w - 1);
            const int rr = r[i], gg = g[i], bb = b[i];
            Y[(size_t)y * (2 * cw) + x] = (uint8_t)((16839 * rr + 33059 * gg + 6420 * bb + (1 << 15) + (16 << 16)) >> 16);
            R += rr; G += gg; B += bb;
        }
    U[(size_t)cy * cw + cx] = (uint8_t)clip8((-9719 * R - 19081 * G + 28800 * B + (128 << 18) + (1 << 17)) >> 18);
    V[(size_t)cy * cw + cx] = (uint8_t)clip8((28800 * R - 24116 * G - 4684 * B + (128 << 18) + (1 << 17)) >> 18);
}

// forward 4x4 DCT of a residual block (libwebp FTransform); d and out are raster 4x4
__device__ __forceinline__ void fdct4(const int d[16], int out[16])
{
    int tmp[16];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int a0 = d[4 * i] + d[4 * i + 3], a1 = d[4 * i + 1] + d[4 * i + 2], a2 = d[4 * i + 1] - d[4 * i + 2], a3 = d[4 * i] - d[4 * i + 3];
        tmp[0 + i * 4] = (a0 + a1) * 8;
        tmp[1 + i * 4] = (a2 * 2217 + a3 * 5352 + 1812) >> 9;
        tmp[2 + i * 4] = (a0 - a1) * 8;
        tmp[3 + i * 4] = (a3 * 2217 - a2 * 5352 + 937) >> 9;
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int a0 = tmp[0 + i] + tmp[12 + i], a1 = tmp[4 + i] + tmp[8 + i], a2 = tmp[4 + i] - tmp[8 + i], a3 = tmp[0 + i] - tmp[12 + i];
        out[0 + i] = (a0 + a1 + 7) >> 4;
        out[4 + i] = ((a2 * 2217 + a3 * 5352 + 12000) >> 16) + (a3 != 0);
        out[8 + i] = (a0 - a1 + 7) >> 4;
        out[12 + i] = (a3 * 2217 - a2 * 5352 + 51000) >> 16;
    }
}
#define VP8_MUL1(a) ((((a) * 20091) >> 16) + (a))
#define VP8_MUL2(a) (((a) * 35468) >> 16)
// RFC 6386 14.4 inverse DCT; res = residual to add to the prediction (before the >> 3)
__device__ __forceinline__ void idct4(const int in[16], int res[16])
{
    int tmp[16];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int a = in[i] + in[8 + i], b = in[i] - in[8 + i];
        const int c = VP8_MUL2(in[4 + i]) - VP8_MUL1(in[12 + i]), d = VP8_MUL1(in[4 + i]) + VP8_MUL2(in[12 + i]);
        tmp[4 * i + 0] = a + d; tmp[4 * i + 1] = b + c; tmp[4 * i + 2] = b - c; tmp[4 * i + 3] = a - d;
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int dc = tmp[i] + 4, a = dc + tmp[8 + i], b = dc - tmp[8 + i];
        const int c = VP8_MUL2(tmp[4 + i]) - VP8_MUL1(tmp[12 + i]), d = VP8_MUL1(tmp[4 + i]) + VP8_MUL2(tmp[12 + i]);
        res[4 * i + 0] = (a + d) >> 3; res[4 * i + 1] = (b + c) >> 3; res[4 * i + 2] = (b - c) >> 3; res[4 * i + 3] = (a - d) >> 3;
    }
}
__device__ __forceinline__ int quant1(int c, int q)
{
    const int a = abs(c), l = min(2047, (a + ((q * 3) >> 3)) / q);
    return c < 0 ? -l : l;
}

__global__ void __launch_bounds__(32) k_vp8_encode(const Vp8Frame f)
{
    __shared__ uint8_t sTop[3][16], sLeft[3][16];
    __shared__ int sTl[3], sDc[16], sDcRec[16], sY2nz;
    const int lane = threadIdx.x;
    int row = 0;
    if (lane == 0) row = atomicAdd(&f.progress[f.mbh], 1);
    row = __shfl_sync(FULL, row, 0);
    if (row >= f.mbh) return;
    const int ys = f.mbw * 16, cs = f.mbw * 8;
    const int plane = lane < 16 ? 0 : lane < 20 ? 1 : lane < 24 ? 2 : 3;              // 3: no block of its own
    const int k = plane == 0 ? lane : plane == 1 ? lane - 16 : lane - 20;
    const int n = plane == 0 ? 16 : 8, bx = plane == 0 ? (k & 3) : (k & 1), by = plane == 0 ? (k >> 2) : (k >> 1);
    const int st = plane == 0 ? ys : cs;
    const uint8_t *S = plane == 0 ? f.Y : plane == 1 ? f.U : f.V;
    uint8_t *R = plane == 0 ? f.RY : plane == 1 ? f.RU : f.RV;
    const int pl = plane < 3 ? plane : 0;
    const int qdc = plane == 0 ? f.q[0] : f.q[4], qac = plane == 0 ? f.q[1] : f.q[5];
    const int blk = plane == 0 ? 1 + k : plane == 1 ? 17 + k : 21 + k;                // position in the macroblock's level array
    constexpr int zig[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};
    volatile int *prog = f.progress;

    for (int mbx = 0; mbx < f.mbw; mbx++) {
        if (row > 0) {
            if (lane == 0) while (prog[row - 1] < mbx + 1) { }
            __syncwarp();
            __threadfence();
        }
        // ---- neighbours: top-left first (it is the previous macroblock's last top sample), then the new top row
        if (lane < 3) sTl[lane] = row == 0 ? 127 : (mbx == 0 ? 129 : sTop[lane][lane == 0 ? 15 : 7]);
        if (mbx == 0) { if (lane < 16) sLeft[0][lane] = 129; else if (lane < 24) sLeft[1][lane - 16] = 129; else sLeft[2][lane - 24] = 129; }
        __syncwarp();
        if (lane < 16) sTop[0][lane] = row ? __ldcg(f.RY + (size_t)(row * 16 - 1) * ys + mbx * 16 + lane) : 127;
        else if (lane < 24) sTop[1][lane - 16] = row ? __ldcg(f.RU + (size_t)(row * 8 - 1) * cs + mbx * 8 + lane - 16) : 127;
        else sTop[2][lane - 24] = row ? __ldcg(f.RV + (size_t)(row * 8 - 1) * cs + mbx * 8 + lane - 24) : 127;
        __syncwarp();
        // ---- this lane's source block and the DC predictor of its plane
        int src[16];
        {
            const uint8_t *sp = S + (size_t)(row * n + by * 4) * st + mbx * n + bx * 4;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const uint32_t v = plane < 3 ? *reinterpret_cast<const uint32_t *>(sp + (size_t)j * st) : 0u;
                src[4 * j] = v & 255; src[4 * j + 1] = (v >> 8) & 255; src[4 * j + 2] = (v >> 16) & 255; src[4 * j + 3] = v >> 24;
            }
        }
        int sumT = 0, sumL = 0;
        for (int i = 0; i < n; i++) { sumT += sTop[pl][i]; sumL += sLeft[pl][i]; }
        const int sh = n == 16 ? 4 : 3;
        const int dcv = (row && mbx) ? (sumT + sumL + n) >> (sh + 1) : row ? (sumT + (n >> 1)) >> sh : mbx ? (sumL + (n >> 1)) >> sh : 128;
        const int tl = sTl[pl];
        int tp[4], lf[4];
#pragma unroll
        for (int i = 0; i < 4; i++) { tp[i] = sTop[pl][bx * 4 + i]; lf[i] = sLeft[pl][by * 4 + i]; }
        // ---- mode decision: squared error of the four predictors, summed over the plane(s)
        unsigned e[4] = {0, 0, 0, 0};
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int s = src[4 * j + i];
                int d = s - dcv; e[0] += d * d;
                d = s - clip8(lf[j] + tp[i] - tl); e[1] += d * d;
                d = s - tp[i]; e[2] += d * d;
                d = s - lf[j]; e[3] += d * d;
            }
        int ymode = 0, uvmode = 0; unsigned by_ = 0, bc_ = 0;
#pragma unroll
        for (int m = 0; m < 4; m++) {
            const unsigned ey = __reduce_add_sync(FULL, plane == 0 ? e[m] : 0u), ec = __reduce_add_sync(FULL, (plane == 1 || plane == 2) ? e[m] : 0u);
            if (m == 0 || ey < by_) { by_ = ey; ymode = m; }
            if (m == 0 || ec < bc_) { bc_ = ec; uvmode = m; }
        }
        const int mode = plane == 0 ? ymode : uvmode;
        // ---- residual -> forward DCT
        int pred[16], d[16], coef[16];
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int p = mode == 0 ? dcv : mode == 1 ? clip8(lf[j] + tp[i] - tl) : mode == 2 ? tp[i] : lf[j];
                pred[4 * j + i] = p; d[4 * j + i] = src[4 * j + i] - p;
            }
        fdct4(d, coef);
        if (plane == 0) sDc[k] = coef[0];
        __syncwarp();
        int16_t *mbl = f.levels + ((size_t)row * f.mbw + mbx) * VP8_MB_COEFS;
        if (lane == 24) {   // Y2: forward WHT of the 16 luma DCs, quantise, and the decoder's inverse WHT of the dequantised levels
            int t[16], w2[16], dq[16];
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int a0 = sDc[4 * i] + sDc[4 * i + 2], a1 = sDc[4 * i + 1] + sDc[4 * i + 3], a2 = sDc[4 * i + 1] - sDc[4 * i + 3], a3 = sDc[4 * i] - sDc[4 * i + 2];
                t[0 + i * 4] = a0 + a1; t[1 + i * 4] = a3 + a2; t[2 + i * 4] = a3 - a2; t[3 + i * 4] = a0 - a1;
            }
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int a0 = t[0 + i] + t[8 + i], a1 = t[4 + i] + t[12 + i], a2 = t[4 + i] - t[12 + i], a3 = t[0 + i] - t[8 + i];
                w2[0 + i] = (a0 + a1) >> 1; w2[4 + i] = (a3 + a2) >> 1; w2[8 + i] = (a3 - a2) >> 1; w2[12 + i] = (a0 - a1) >> 1;
            }
            int nz = 0;
            uint32_t pk[8];
#pragma unroll
            for (int s = 0; s < 16; s++) {
                const int q = s == 0 ? f.q[2] : f.q[3], l = quant1(w2[zig[s]], q);
                dq[zig[s]] = l * q; nz |= l;
                if (s & 1) pk[s >> 1] |= (uint32_t)(uint16_t)l << 16; else pk[s >> 1] = (uint16_t)l;
            }
            reinterpret_cast<uint4 *>(mbl)[0] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
            reinterpret_cast<uint4 *>(mbl)[1] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
            sY2nz = nz;
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int a0 = dq[0 + i] + dq[12 + i], a1 = dq[4 + i] + dq[8 + i], a2 = dq[4 + i] - dq[8 + i], a3 = dq[0 + i] - dq[12 + i];
                t[0 + i] = a0 + a1; t[8 + i] = a0 - a1; t[4 + i] = a3 + a2; t[12 + i] = a3 - a2;
            }
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int dd = t[0 + i * 4] + 3, a0 = dd + t[3 + i * 4], a1 = t[1 + i * 4] + t[2 + i * 4], a2 = t[1 + i * 4] - t[2 + i * 4], a3 = dd - t[3 + i * 4];
                sDcRec[4 * i + 0] = (a0 + a1) >> 3; sDcRec[4 * i + 1] = (a3 + a2) >> 3; sDcRec[4 * i + 2] = (a0 - a1) >> 3; sDcRec[4 * i + 3] = (a3 - a2) >> 3;
            }
        }
        __syncwarp();
        // ---- quantise (zigzag order), dequantise, inverse DCT, reconstruct
        int nz = 0;
        if (plane < 3) {
            int dq[16], res[16];
            uint32_t pk[8];
#pragma unroll
            for (int s = 0; s < 16; s++) {
                const int q = s == 0 ? qdc : qac;
                const int l = (plane == 0 && s == 0) ? 0 : quant1(coef[zig[s]], q);
                dq[zig[s]] = l * q; nz |= l;
                if (s & 1) pk[s >> 1] |= (uint32_t)(uint16_t)l << 16; else pk[s >> 1] = (uint16_t)l;
            }
            if (plane == 0) dq[0] = sDcRec[k];
            reinterpret_cast<uint4 *>(mbl + blk * 16)[0] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
            reinterpret_cast<uint4 *>(mbl + blk * 16)[1] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
            idct4(dq, res);
            uint8_t *rp = R + (size_t)(row * n + by * 4) * st + mbx * n + bx * 4;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int p0 = clip8(pred[4 * j] + res[4 * j]), p1 = clip8(pred[4 * j + 1] + res[4 * j + 1]), p2 = clip8(pred[4 * j + 2] + res[4 * j + 2]), p3 = clip8(pred[4 * j + 3] + res[4 * j + 3]);
                *reinterpret_cast<uint32_t *>(rp + (size_t)j * st) = (uint32_t)p0 | ((uint32_t)p1 << 8) | ((uint32_t)p2 << 16) | ((uint32_t)p3 << 24);
                if (bx == (n >> 2) - 1) sLeft[pl][by * 4 + j] = (uint8_t)p3;          // right column = the next macroblock's left edge
            }
        }
        const bool any = __any_sync(FULL, nz != 0) || sY2nz != 0;
        if (lane == 0) *reinterpret_cast<uint32_t *>(f.modes + ((size_t)row * f.mbw + mbx) * 4) = (uint32_t)ymode | ((uint32_t)uvmode << 8) | ((any ? 0u : 1u) << 16);
        __threadfence();
        __syncwarp();
        if (lane == 0) prog[row] = mbx + 1;
    }
}


// K8 with 4x4 intra prediction (vp8_bpred_core.h): every macroblock is coded both ways -- the 16x16 arm exactly as k_vp8_encode codes
// it, and the B_PRED arm, whose sub-blocks are decided in 10 anti-diagonal steps (sub-block (x, y) needs (x-1, y), (x, y-1), (x-1, y-1)
// and (x+1, y-1), so the at most two blocks of x + 2y = t are independent): lane 10 s + m tries mode m on the step's block s.  Both
// reconstructions and level sets stay in shared memory until the rate-distortion rule picks one.  The above-right samples of a
// macroblock's top-right sub-block belong to the macroblock above and to the right, so a row trails the row above by TWO macroblocks.
__global__ void __launch_bounds__(32) k_vp8_encode_bpred(const Vp8Frame f)
{
    __shared__ __align__(16) uint8_t sSrc[256], sRec16[256], sRec4[256];
    __shared__ __align__(16) int16_t sLv16[17][16], sLv4[16][16];
    __shared__ uint8_t sTop[21], sLeft[16], sCTop[2][8], sCLeft[2][8];
    __shared__ int sCTl[2], sDc[16], sDcRec[16], sY2nz;
    __shared__ uint8_t sMode4[16], sNz4[16], sAboveModes[4], sLeftModes[4];
    __shared__ unsigned long long sScore[20], sBlockScore[16];
    const int lane = threadIdx.x;
    int row = 0;
    if (lane == 0) row = atomicAdd(&f.progress[f.mbh], 1);
    row = __shfl_sync(FULL, row, 0);
    if (row >= f.mbh) return;
    const int ys = f.mbw * 16, cs = f.mbw * 8;
    // phase A (the 16x16 arm and chroma) keeps k_vp8_encode's layout: lanes 0..15 luma blocks, 16..19 U, 20..23 V, 24 the Y2
    const int plane = lane < 16 ? 0 : lane < 20 ? 1 : lane < 24 ? 2 : 3;
    const int k = plane == 0 ? lane : plane == 1 ? lane - 16 : lane - 20;
    const int n = plane == 0 ? 16 : 8, bx = plane == 0 ? (k & 3) : (k & 1), by = plane == 0 ? (k >> 2) : (k >> 1);
    const int st = plane == 0 ? ys : cs;
    const uint8_t *S = plane == 0 ? f.Y : plane == 1 ? f.U : f.V;
    const int qdc = plane == 0 ? f.q[0] : f.q[4], qac = plane == 0 ? f.q[1] : f.q[5];
    const int lam = vp8bp_lambda(f.q[1]);
    constexpr int zig[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};
    volatile int *prog = f.progress;

    for (int mbx = 0; mbx < f.mbw; mbx++) {
        if (row > 0) {
            if (lane == 0) while (prog[row - 1] < min(mbx + 2, f.mbw)) { }
            __syncwarp();
            __threadfence();
        }
        const size_t mb = (size_t)row * f.mbw + mbx;
        // ---- borders (vp8bp_mb_border's rules, read past L1: the rows above were written by other warps)
        if (lane < 21) {
            uint8_t v = 127;
            if (row > 0) {
                const uint8_t *a = f.RY + (size_t)(row * 16 - 1) * ys + mbx * 16;
                v = lane == 0 ? (mbx ? __ldcg(a - 1) : 129) : (lane > 16 && mbx == f.mbw - 1) ? __ldcg(a + 15) : __ldcg(a + lane - 1);
            }
            sTop[lane] = v;
        } else if (lane < 23) {
            const int c = lane - 21;
            sCTl[c] = row == 0 ? 127 : mbx == 0 ? 129 : __ldcg((c ? f.RV : f.RU) + (size_t)(row * 8 - 1) * cs + mbx * 8 - 1);
        } else if (lane < 27) {
            const int x = lane - 23;
            sAboveModes[x] = row ? __ldcg(f.bmodes + (mb - f.mbw) * 16 + 12 + x) : 0;
        }
        if (lane < 16) {
            if (mbx == 0) sLeft[lane] = 129;
            const int c = lane >> 3, i = lane & 7;
            sCTop[c][i] = row ? __ldcg((c ? f.RV : f.RU) + (size_t)(row * 8 - 1) * cs + mbx * 8 + i) : 127;
            if (mbx == 0) sCLeft[c][i] = 129;
        }
        if (mbx == 0 && lane < 4) sLeftModes[lane] = 0;
        __syncwarp();
        const uint8_t *T = plane == 0 ? sTop + 1 : sCTop[plane == 2];
        const uint8_t *Lf = plane == 0 ? sLeft : sCLeft[plane == 2];
        const int tl = plane == 0 ? sTop[0] : sCTl[plane == 2];
        const int ex = plane < 3 ? bx : 0, ey = plane < 3 ? by : 0;      // lanes without a block read in-bounds edges they then ignore
        int src[16];
        {
            const uint8_t *sp = S + (size_t)(row * n + by * 4) * st + mbx * n + bx * 4;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const uint32_t v = plane < 3 ? *reinterpret_cast<const uint32_t *>(sp + (size_t)j * st) : 0u;
                src[4 * j] = v & 255; src[4 * j + 1] = (v >> 8) & 255; src[4 * j + 2] = (v >> 16) & 255; src[4 * j + 3] = v >> 24;
                if (plane == 0) *reinterpret_cast<uint32_t *>(sSrc + (by * 4 + j) * 16 + bx * 4) = v;
            }
        }
        int sumT = 0, sumL = 0;
        for (int i = 0; i < n; i++) { sumT += T[i]; sumL += Lf[i]; }
        const int sh = n == 16 ? 4 : 3;
        const int dcv = (row && mbx) ? (sumT + sumL + n) >> (sh + 1) : row ? (sumT + (n >> 1)) >> sh : mbx ? (sumL + (n >> 1)) >> sh : 128;
        int tp[4], lf[4];
#pragma unroll
        for (int i = 0; i < 4; i++) { tp[i] = T[ex * 4 + i]; lf[i] = Lf[ey * 4 + i]; }
        unsigned e[4] = {0, 0, 0, 0};
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int s = src[4 * j + i];
                int d = s - dcv; e[0] += d * d;
                d = s - clip8(lf[j] + tp[i] - tl); e[1] += d * d;
                d = s - tp[i]; e[2] += d * d;
                d = s - lf[j]; e[3] += d * d;
            }
        int ymode = 0, uvmode = 0; unsigned by_ = 0, bc_ = 0;
#pragma unroll
        for (int m = 0; m < 4; m++) {
            const unsigned ey = __reduce_add_sync(FULL, plane == 0 ? e[m] : 0u), ec = __reduce_add_sync(FULL, (plane == 1 || plane == 2) ? e[m] : 0u);
            if (m == 0 || ey < by_) { by_ = ey; ymode = m; }
            if (m == 0 || ec < bc_) { bc_ = ec; uvmode = m; }
        }
        const int mode = plane == 0 ? ymode : uvmode;
        int pred[16], coef[16];
        {
            int d[16];
#pragma unroll
            for (int j = 0; j < 4; j++)
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const int p = mode == 0 ? dcv : mode == 1 ? clip8(lf[j] + tp[i] - tl) : mode == 2 ? tp[i] : lf[j];
                    pred[4 * j + i] = p; d[4 * j + i] = src[4 * j + i] - p;
                }
            fdct4(d, coef);
        }
        if (plane == 0) sDc[k] = coef[0];
        __syncwarp();
        int16_t *mbl = f.levels + mb * VP8_MB_COEFS;
        uint32_t rate = 0;
        if (lane == 24) {   // Y2, as in k_vp8_encode, kept in shared memory with its rate (context 0)
            int t[16], w2[16], dq[16];
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int a0 = sDc[4 * i] + sDc[4 * i + 2], a1 = sDc[4 * i + 1] + sDc[4 * i + 3], a2 = sDc[4 * i + 1] - sDc[4 * i + 3], a3 = sDc[4 * i] - sDc[4 * i + 2];
                t[0 + i * 4] = a0 + a1; t[1 + i * 4] = a3 + a2; t[2 + i * 4] = a3 - a2; t[3 + i * 4] = a0 - a1;
            }
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int a0 = t[0 + i] + t[8 + i], a1 = t[4 + i] + t[12 + i], a2 = t[4 + i] - t[12 + i], a3 = t[0 + i] - t[8 + i];
                w2[0 + i] = (a0 + a1) >> 1; w2[4 + i] = (a3 + a2) >> 1; w2[8 + i] = (a3 - a2) >> 1; w2[12 + i] = (a0 - a1) >> 1;
            }
            int nz = 0;
#pragma unroll
            for (int s = 0; s < 16; s++) {
                const int q = s == 0 ? f.q[2] : f.q[3], l = quant1(w2[zig[s]], q);
                dq[zig[s]] = l * q; nz |= l; sLv16[0][s] = (int16_t)l;
            }
            sY2nz = nz;
            int dummy;
            rate = vp8bp_block_rate(sLv16[0], 1, 0, 0, &dummy);
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int a0 = dq[0 + i] + dq[12 + i], a1 = dq[4 + i] + dq[8 + i], a2 = dq[4 + i] - dq[8 + i], a3 = dq[0 + i] - dq[12 + i];
                t[0 + i] = a0 + a1; t[8 + i] = a0 - a1; t[4 + i] = a3 + a2; t[12 + i] = a3 - a2;
            }
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int dd = t[0 + i * 4] + 3, a0 = dd + t[3 + i * 4], a1 = t[1 + i * 4] + t[2 + i * 4], a2 = t[1 + i * 4] - t[2 + i * 4], a3 = dd - t[3 + i * 4];
                sDcRec[4 * i + 0] = (a0 + a1) >> 3; sDcRec[4 * i + 1] = (a3 + a2) >> 3; sDcRec[4 * i + 2] = (a0 - a1) >> 3; sDcRec[4 * i + 3] = (a3 - a2) >> 3;
            }
        }
        __syncwarp();
        int nz = 0;
        uint32_t sse = 0;
        if (plane < 3) {
            int dq[16], res[16];
            uint32_t pk[8];
#pragma unroll
            for (int s = 0; s < 16; s++) {
                const int q = s == 0 ? qdc : qac;
                const int l = (plane == 0 && s == 0) ? 0 : quant1(coef[zig[s]], q);
                dq[zig[s]] = l * q; nz |= l;
                if (s & 1) pk[s >> 1] |= (uint32_t)(uint16_t)l << 16; else pk[s >> 1] = (uint16_t)l;
            }
            if (plane == 0) dq[0] = sDcRec[k];
            idct4(dq, res);
            if (plane == 0) {   // luma of the 16x16 arm: levels and reconstruction stay in shared memory
                reinterpret_cast<uint4 *>(sLv16[1 + k])[0] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
                reinterpret_cast<uint4 *>(sLv16[1 + k])[1] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
#pragma unroll
                for (int j = 0; j < 4; j++)
#pragma unroll
                    for (int i = 0; i < 4; i++) {
                        const int r = clip8(pred[4 * j + i] + res[4 * j + i]), d = src[4 * j + i] - r;
                        sRec16[(by * 4 + j) * 16 + bx * 4 + i] = (uint8_t)r; sse += d * d;
                    }
            } else {            // chroma is the same in both arms: straight out
                uint8_t *R = plane == 1 ? f.RU : f.RV;
                const int blk = plane == 1 ? 17 + k : 21 + k;
                reinterpret_cast<uint4 *>(mbl + blk * 16)[0] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
                reinterpret_cast<uint4 *>(mbl + blk * 16)[1] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
                uint8_t *rp = R + (size_t)(row * 8 + by * 4) * cs + mbx * 8 + bx * 4;
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int p0 = clip8(pred[4 * j] + res[4 * j]), p1 = clip8(pred[4 * j + 1] + res[4 * j + 1]), p2 = clip8(pred[4 * j + 2] + res[4 * j + 2]), p3 = clip8(pred[4 * j + 3] + res[4 * j + 3]);
                    *reinterpret_cast<uint32_t *>(rp + (size_t)j * cs) = (uint32_t)p0 | ((uint32_t)p1 << 8) | ((uint32_t)p2 << 16) | ((uint32_t)p3 << 24);
                    if (bx == 1) sCLeft[plane - 1][by * 4 + j] = (uint8_t)p3;
                }
            }
        }
        // ---- the 16x16 arm's score: AC blocks with their contexts inside the macroblock (0 across its edges)
        const unsigned acnz = __ballot_sync(FULL, plane == 0 && nz != 0);
        const bool chroma_nz = __any_sync(FULL, (plane == 1 || plane == 2) && nz != 0);
        __syncwarp();
        if (plane == 0) {
            int dummy;
            const int ctx = (by ? (acnz >> (k - 4)) & 1 : 0) + (bx ? (acnz >> (k - 1)) & 1 : 0);
            rate = vp8bp_block_rate(sLv16[1 + k], 0, 1, ctx, &dummy);
        }
        const uint32_t sse16 = __reduce_add_sync(FULL, sse), rate16 = __reduce_add_sync(FULL, rate);
        const unsigned long long score16 = vp8bp_score(sse16, rate16 + vp8bp_i16_cost(ymode), lam);
        // ---- the B_PRED arm: 10 anti-diagonal steps, lane 10 s + m = mode m on the step's s-th block
        for (int t = 0; t < 10; t++) {
            const int slot = lane / 10, m = lane - 10 * slot;
            const int y = (t <= 3 ? 0 : (t - 2) >> 1) + slot, x = t - 2 * y;
            const bool active = lane < 20 && y <= min(3, t >> 1) && x >= 0;
            const int kb = 4 * y + x;
            int16_t lv[16];
            uint8_t rec[16];
            int bnz = 0;
            if (active) {
                uint8_t eg[13], p[16];
                vp8bp_edges(sTop, sLeft, sRec4, 16, x, y, eg);
                vp8bp_pred4(m, eg, p);
                int d[16], c[16], dq[16], res[16];
#pragma unroll
                for (int i = 0; i < 16; i++) d[i] = sSrc[(4 * y + (i >> 2)) * 16 + 4 * x + (i & 3)] - p[i];
                fdct4(d, c);
#pragma unroll
                for (int s = 0; s < 16; s++) {
                    const int q = s == 0 ? f.q[0] : f.q[1], l = quant1(c[zig[s]], q);
                    lv[s] = (int16_t)l; dq[zig[s]] = l * q;
                }
                idct4(dq, res);
                uint32_t e2 = 0;
#pragma unroll
                for (int i = 0; i < 16; i++) {
                    const int r = clip8(p[i] + res[i]), dd = sSrc[(4 * y + (i >> 2)) * 16 + 4 * x + (i & 3)] - r;
                    rec[i] = (uint8_t)r; e2 += dd * dd;
                }
                const int ctx = (y ? sNz4[kb - 4] : 0) + (x ? sNz4[kb - 1] : 0);
                const uint32_t r = vp8bp_block_rate(lv, 3, 0, ctx, &bnz) + vp8bp_bmode_cost(y ? sMode4[kb - 4] : sAboveModes[x], x ? sMode4[kb - 1] : sLeftModes[y], m);
                sScore[lane] = vp8bp_score(e2, r, lam);
            }
            __syncwarp();
            if (active) {
                int best = 0;
                for (int i = 1; i < 10; i++) if (sScore[10 * slot + i] < sScore[10 * slot + best]) best = i;
                if (best == m) {
#pragma unroll
                    for (int i = 0; i < 16; i++) { sRec4[(4 * y + (i >> 2)) * 16 + 4 * x + (i & 3)] = rec[i]; sLv4[kb][i] = lv[i]; }
                    sNz4[kb] = (uint8_t)bnz; sMode4[kb] = (uint8_t)m; sBlockScore[kb] = sScore[lane];
                }
            }
            __syncwarp();
        }
        // ---- the decision, then the winner's luma out: reconstruction, levels, sub-block modes
        unsigned long long sum4 = lane < 16 ? sBlockScore[lane] : 0ull;
#pragma unroll
        for (int o = 16; o; o >>= 1) sum4 += __shfl_xor_sync(FULL, sum4, o);
        const bool bp = sum4 + (unsigned long long)lam * vp8bp_bit(0, VP8BP_FLAG_PROB) < score16;
        const uint8_t *rec = bp ? sRec4 : sRec16;
        if (lane < 16) {
            const uint4 v = reinterpret_cast<const uint4 *>(rec)[lane];
            *reinterpret_cast<uint4 *>(f.RY + (size_t)(row * 16 + lane) * ys + mbx * 16) = v;
            f.bmodes[mb * 16 + lane] = bp ? sMode4[lane] : (uint8_t)ymode;
        }
        bool lnz = false;
        for (int i = lane; i < 17 * 8; i += 32) {      // 17 blocks of 16 levels, two per 32-bit word
            const int b = i >> 3, w = i & 7;
            const uint32_t v = bp ? (b ? reinterpret_cast<const uint32_t *>(sLv4[b - 1])[w] : 0u) : reinterpret_cast<const uint32_t *>(sLv16[b])[w];
            reinterpret_cast<uint32_t *>(mbl)[i] = v;
            lnz |= bp && v != 0;
        }
        const bool any = bp ? (__any_sync(FULL, lnz) || chroma_nz) : (acnz != 0 || sY2nz != 0 || chroma_nz);
        __syncwarp();
        if (lane < 16) sLeft[lane] = rec[lane * 16 + 15];
        if (lane < 4) sLeftModes[lane] = bp ? sMode4[4 * lane + 3] : (uint8_t)ymode;
        if (lane == 0) *reinterpret_cast<uint32_t *>(f.modes + mb * 4) = (uint32_t)(bp ? 4 : ymode) | ((uint32_t)uvmode << 8) | ((any ? 0u : 1u) << 16);
        __threadfence();
        __syncwarp();
        if (lane == 0) prog[row] = mbx + 1;
    }
}
} // namespace

// ---- token pass on the device (vp8_tokens_core.h): one thread per macroblock -------------------------------------------------------
// A block's context is whether the blocks above / to its left have coded coefficients -- a property of the levels alone -- so with a
// 25-bit mask per macroblock every macroblock's decision list is independent: masks, then a counting walk (list length per
// macroblock + the frame's tallies per probability slot), an exclusive scan, and the same walk again writing 16-bit decision records
// at the macroblock's offset.  The host is left with choosing the probabilities and the (sequential) boolean coder.
namespace {
struct TokenCountSink {
    uint32_t n; uint32_t *hist;                          // hist: shared memory, [slot][bit]
    __device__ __forceinline__ void node(int s, bool bit) { n++; atomicAdd(&hist[2 * s + (bit ? 1 : 0)], 1u); }
    __device__ __forceinline__ void fixed(bool, int) { n++; }
};
struct TokenWriteSink {
    uint16_t *q;
    __device__ __forceinline__ void node(int s, bool bit) { *q++ = vt::rec_node(s, bit); }
    __device__ __forceinline__ void fixed(bool bit, int prob) { *q++ = vt::rec_fixed(bit, prob); }
};

__global__ void k_vp8_mbmask(const int16_t *__restrict__ levels, const uint8_t *__restrict__ modes, int nmb, uint32_t *__restrict__ mask)
{
    const int mb = blockIdx.x * blockDim.x + threadIdx.x;
    if (mb < nmb) mask[mb] = modes[4 * mb + 2] ? 0u : vt::mb_mask(levels + (size_t)mb * VP8_MB_COEFS, modes[4 * mb] == 4);      // a skipped macroblock has no coefficients
}

// the carried Y2 contexts (vt::y2_carry_col / _row): threads 0..mbw-1 walk the columns, mbw..mbw+mbh-1 the rows
__global__ void k_vp8_y2carry(const uint32_t *__restrict__ mask, const uint8_t *__restrict__ modes, int mbw, int mbh, uint8_t *__restrict__ y2top, uint8_t *__restrict__ y2left)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < mbw) vt::y2_carry_col(mask, modes, mbw, mbh, i, y2top);
    else if (i < mbw + mbh) vt::y2_carry_row(mask, modes, mbw, i - mbw, y2left);
}

__global__ void __launch_bounds__(64) k_vp8_token_count(const int16_t *__restrict__ levels, const uint8_t *__restrict__ modes, const uint32_t *__restrict__ mask,
                                                        const uint8_t *__restrict__ y2top, const uint8_t *__restrict__ y2left, int mbw, int nmb,
                                                        uint32_t *__restrict__ counts /*[nmb + 1], the last one 0*/, uint32_t *__restrict__ hist /*[kNumProbs][2]*/)
{
    __shared__ uint32_t h[vt::kNumProbs * 2];
    for (int i = threadIdx.x; i < vt::kNumProbs * 2; i += blockDim.x) h[i] = 0;
    __syncthreads();
    const int mb = blockIdx.x * blockDim.x + threadIdx.x;
    if (mb < nmb) {
        uint32_t n = 0;
        if (!modes[4 * mb + 2]) {
            const int my = mb / mbw, mx = mb - my * mbw;
            TokenCountSink sk{0u, h};
            vt::walk_mb(sk, levels + (size_t)mb * VP8_MB_COEFS, vt::with_y2(my ? mask[mb - mbw] : 0u, y2top[mb]), vt::with_y2(mx ? mask[mb - 1] : 0u, y2left[mb]), modes[4 * mb] == 4);
            n = sk.n;
        }
        counts[mb] = n;
        if (mb == nmb - 1) counts[nmb] = 0;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < vt::kNumProbs * 2; i += blockDim.x) if (h[i]) atomicAdd(&hist[i], h[i]);
}

__global__ void __launch_bounds__(64) k_vp8_token_write(const int16_t *__restrict__ levels, const uint8_t *__restrict__ modes, const uint32_t *__restrict__ mask,
                                                        const uint8_t *__restrict__ y2top, const uint8_t *__restrict__ y2left, int mbw, int nmb,
                                                        const uint32_t *__restrict__ offsets /*[nmb + 1]*/, uint16_t *__restrict__ tokens, uint32_t capacity)
{
    const int mb = blockIdx.x * blockDim.x + threadIdx.x;
    if (mb >= nmb || modes[4 * mb + 2] || offsets[mb + 1] > capacity) return;
    const int my = mb / mbw, mx = mb - my * mbw;
    TokenWriteSink sk{tokens + offsets[mb]};
    vt::walk_mb(sk, levels + (size_t)mb * VP8_MB_COEFS, vt::with_y2(my ? mask[mb - mbw] : 0u, y2top[mb]), vt::with_y2(mx ? mask[mb - 1] : 0u, y2left[mb]), modes[4 * mb] == 4);
}
} // namespace

size_t vp8_tokens_temp_bytes(int nmb)
{
    size_t tb = 0;
    cub::DeviceScan::ExclusiveSum((void *)nullptr, tb, (const uint32_t *)nullptr, (uint32_t *)nullptr, nmb + 1, (cudaStream_t)0);
    return tb;
}
int launch_vp8_token_count(const Vp8Frame &f, uint32_t *d_mask, uint8_t *d_y2, uint32_t *d_counts, uint32_t *d_offsets, uint32_t *d_hist, void *d_temp, size_t temp_bytes, void *stream)
{
    cudaStream_t st = (cudaStream_t)stream;
    const int nmb = f.mbw * f.mbh;
    cudaError_t e = cudaMemsetAsync(d_hist, 0, sizeof(uint32_t) * vt::kNumProbs * 2, st);
    if (e != cudaSuccess) return (int)e;
    k_vp8_mbmask<<<(nmb + 127) / 128, 128, 0, st>>>(f.levels, f.modes, nmb, d_mask);
    k_vp8_y2carry<<<(f.mbw + f.mbh + 127) / 128, 128, 0, st>>>(d_mask, f.modes, f.mbw, f.mbh, d_y2, d_y2 + nmb);
    k_vp8_token_count<<<(nmb + 63) / 64, 64, 0, st>>>(f.levels, f.modes, d_mask, d_y2, d_y2 + nmb, f.mbw, nmb, d_counts, d_hist);
    e = cub::DeviceScan::ExclusiveSum(d_temp, temp_bytes, d_counts, d_offsets, nmb + 1, st);
    if (e != cudaSuccess) return (int)e;
    return (int)cudaGetLastError();
}
int launch_vp8_token_write(const Vp8Frame &f, const uint32_t *d_mask, const uint8_t *d_y2, const uint32_t *d_offsets, uint16_t *d_tokens, uint32_t capacity, void *stream)
{
    const int nmb = f.mbw * f.mbh;
    k_vp8_token_write<<<(nmb + 63) / 64, 64, 0, (cudaStream_t)stream>>>(f.levels, f.modes, d_mask, d_y2, d_y2 + nmb, f.mbw, nmb, d_offsets, d_tokens, capacity);
    return (int)cudaGetLastError();
}

int launch_vp8_rgb_to_yuv(const uint8_t *r, const uint8_t *g, const uint8_t *b, int w, int h, uint8_t *Y, uint8_t *U, uint8_t *V, void *stream)
{
    const int cw = ((w + 15) >> 4) * 8, chh = ((h + 15) >> 4) * 8;
    const dim3 blk(32, 8), grid((cw + 31) / 32, (chh + 7) / 8);
    k_vp8_rgb_to_yuv<<<grid, blk, 0, (cudaStream_t)stream>>>(r, g, b, w, h, Y, U, V, cw, chh);
    return (int)cudaGetLastError();
}

int launch_vp8_encode(const Vp8Frame &f, void *stream)
{
    cudaError_t e = cudaMemsetAsync(f.progress, 0, sizeof(int) * (size_t)(f.mbh + 1), (cudaStream_t)stream);
    if (e != cudaSuccess) return (int)e;
    k_vp8_encode<<<f.mbh, 32, 0, (cudaStream_t)stream>>>(f);
    return (int)cudaGetLastError();
}

int launch_vp8_encode_bpred(const Vp8Frame &f, void *stream)
{
    cudaError_t e = cudaMemsetAsync(f.progress, 0, sizeof(int) * (size_t)(f.mbh + 1), (cudaStream_t)stream);
    if (e != cudaSuccess) return (int)e;
    k_vp8_encode_bpred<<<f.mbh, 32, 0, (cudaStream_t)stream>>>(f);
    return (int)cudaGetLastError();
}

} // namespace b200
