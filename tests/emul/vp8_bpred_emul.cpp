// CPU emulation of k_vp8_encode_bpred (csrc/vp8_kernels.cu) through the shared rules of csrc/vp8_bpred_core.h, in the kernel's
// shapes: macroblocks in the order the trail-by-two wavefront allows at its tightest (macroblock (x, y) at step x + 2y), every read of
// the frame's reconstruction or sub-block modes checked against the macroblocks already finished; inside a macroblock the warp's
// lanes one after another -- phase A's layout (lanes 0..15 luma, 16..23 chroma, 24 the Y2) with its reductions, then phase B's 10
// anti-diagonal steps with lane 10 s + m trying mode m on the step's s-th block, the scan of the 10 scores (ties to the lower mode),
// and the winner's write-back -- then the rate-distortion choice and the write-out.  The test compares the result with the scalar
// twin (oracle/webp_bpred_oracle.c), which codes the sub-blocks in raster order.  Test infrastructure only.
#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../caesium-clt_b200/csrc/vp8_bpred_core.h"

using namespace b200;

namespace {

int clip8(int v) { return v < 0 ? 0 : v > 255 ? 255 : v; }
const int zig[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};

// the kernel's fdct4 / idct4 / quant1
void fdct4(const int d[16], int out[16])
{
    int tmp[16];
    for (int i = 0; i < 4; i++) {
        const int a0 = d[4 * i] + d[4 * i + 3], a1 = d[4 * i + 1] + d[4 * i + 2], a2 = d[4 * i + 1] - d[4 * i + 2], a3 = d[4 * i] - d[4 * i + 3];
        tmp[0 + i * 4] = (a0 + a1) * 8;
        tmp[1 + i * 4] = (a2 * 2217 + a3 * 5352 + 1812) >> 9;
        tmp[2 + i * 4] = (a0 - a1) * 8;
        tmp[3 + i * 4] = (a3 * 2217 - a2 * 5352 + 937) >> 9;
    }
    for (int i = 0; i < 4; i++) {
        const int a0 = tmp[0 + i] + tmp[12 + i], a1 = tmp[4 + i] + tmp[8 + i], a2 = tmp[4 + i] - tmp[8 + i], a3 = tmp[0 + i] - tmp[12 + i];
        out[0 + i] = (a0 + a1 + 7) >> 4;
        out[4 + i] = ((a2 * 2217 + a3 * 5352 + 12000) >> 16) + (a3 != 0);
        out[8 + i] = (a0 - a1 + 7) >> 4;
        out[12 + i] = (a3 * 2217 - a2 * 5352 + 51000) >> 16;
    }
}
#define MUL1(a) ((((a) * 20091) >> 16) + (a))
#define MUL2(a) (((a) * 35468) >> 16)
void idct4(const int in[16], int res[16])
{
    int tmp[16];
    for (int i = 0; i < 4; i++) {
        const int a = in[i] + in[8 + i], b = in[i] - in[8 + i];
        const int c = MUL2(in[4 + i]) - MUL1(in[12 + i]), d = MUL1(in[4 + i]) + MUL2(in[12 + i]);
        tmp[4 * i + 0] = a + d; tmp[4 * i + 1] = b + c; tmp[4 * i + 2] = b - c; tmp[4 * i + 3] = a - d;
    }
    for (int i = 0; i < 4; i++) {
        const int dc = tmp[i] + 4, a = dc + tmp[8 + i], b = dc - tmp[8 + i];
        const int c = MUL2(tmp[4 + i]) - MUL1(tmp[12 + i]), d = MUL1(tmp[4 + i]) + MUL2(tmp[12 + i]);
        res[4 * i + 0] = (a + d) >> 3; res[4 * i + 1] = (b + c) >> 3; res[4 * i + 2] = (b - c) >> 3; res[4 * i + 3] = (a - d) >> 3;
    }
}
int quant1(int c, int q)
{
    const int a = abs(c), l = std::min(2047, (a + ((q * 3) >> 3)) / q);
    return c < 0 ? -l : l;
}

struct Frame {
    int mbw, mbh, q[6];
    const uint8_t *Y, *U, *V;
    uint8_t *RY, *RU, *RV, *modes, *bmodes;
    int16_t *levels;
    std::vector<uint8_t> done;           // macroblocks finished
    int *violations;
    // a read of macroblock (x, y)'s output: it must be finished
    void need(int x, int y) { if (!done[(size_t)y * mbw + x]) ++*violations; }
};

void encode_mb(Frame &f, int row, int mbx, uint8_t sLeft[16], uint8_t sCLeft[2][8], uint8_t sLeftModes[4])
{
    const int ys = f.mbw * 16, cs = f.mbw * 8, lam = vp8bp_lambda(f.q[1]);
    const size_t mb = (size_t)row * f.mbw + mbx;
    uint8_t sTop[21], sCTop[2][8], sAboveModes[4], sSrc[256], sRec16[256], sRec4[256], sMode4[16], sNz4[16];
    int16_t sLv16[17][16], sLv4[16][16];
    int sCTl[2], sDc[16], sDcRec[16], sY2nz = 0;
    uint64_t sScore[20], sBlockScore[16];
    // ---- borders, lane by lane as the kernel loads them
    if (mbx == 0) { memset(sLeft, 129, 16); memset(sCLeft, 129, 16); memset(sLeftModes, 0, 4); }
    for (int lane = 0; lane < 32; lane++) {
        if (lane < 21) {
            uint8_t v = 127;
            if (row > 0) {
                const uint8_t *a = f.RY + (size_t)(row * 16 - 1) * ys + mbx * 16;
                const int col = lane == 0 ? (mbx ? -1 : 0) : (lane > 16 && mbx == f.mbw - 1) ? 15 : lane - 1;
                if (lane == 0 && !mbx) v = 129;
                else { f.need((mbx * 16 + col) >> 4, row - 1); v = a[col]; }
            }
            sTop[lane] = v;
        } else if (lane < 23) {
            const int c = lane - 21;
            if (row && mbx) f.need(mbx - 1, row - 1);
            sCTl[c] = row == 0 ? 127 : mbx == 0 ? 129 : (c ? f.RV : f.RU)[(size_t)(row * 8 - 1) * cs + mbx * 8 - 1];
        } else if (lane < 27) {
            const int x = lane - 23;
            if (row) f.need(mbx, row - 1);
            sAboveModes[x] = row ? f.bmodes[(mb - f.mbw) * 16 + 12 + x] : 0;
        }
        if (lane < 16) {
            const int c = lane >> 3, i = lane & 7;
            if (row) f.need(mbx, row - 1);
            sCTop[c][i] = row ? (c ? f.RV : f.RU)[(size_t)(row * 8 - 1) * cs + mbx * 8 + i] : 127;
        }
    }
    // ---- phase A: per lane state
    int ymodeL = 0, uvmodeL = 0;
    int src[32][16], pred[32][16], coef[32][16], nzL[32] = {0};
    uint32_t rate[32] = {0}, sse[32] = {0};
    unsigned eL[32][4] = {};
    int dcvL[32], tlL[32], tpL[32][4], lfL[32][4];
    for (int lane = 0; lane < 32; lane++) {
        const int plane = lane < 16 ? 0 : lane < 20 ? 1 : lane < 24 ? 2 : 3;
        const int k = plane == 0 ? lane : plane == 1 ? lane - 16 : lane - 20;
        const int n = plane == 0 ? 16 : 8, bx = plane == 0 ? (k & 3) : (k & 1), by = plane == 0 ? (k >> 2) : (k >> 1);
        const int st = plane == 0 ? ys : cs;
        const uint8_t *S = plane == 0 ? f.Y : plane == 1 ? f.U : f.V;
        const uint8_t *T = plane == 0 ? sTop + 1 : sCTop[plane == 2];
        const uint8_t *Lf = plane == 0 ? sLeft : sCLeft[plane == 2];
        const int tl = plane == 0 ? sTop[0] : sCTl[plane == 2];
        const int ex = plane < 3 ? bx : 0, ey = plane < 3 ? by : 0;
        for (int j = 0; j < 4; j++)
            for (int i = 0; i < 4; i++) {
                src[lane][4 * j + i] = plane < 3 ? S[(size_t)(row * n + by * 4 + j) * st + mbx * n + bx * 4 + i] : 0;
                if (plane == 0) sSrc[(by * 4 + j) * 16 + bx * 4 + i] = (uint8_t)src[lane][4 * j + i];
            }
        int sumT = 0, sumL = 0;
        for (int i = 0; i < n; i++) { sumT += T[i]; sumL += Lf[i]; }
        const int sh = n == 16 ? 4 : 3;
        dcvL[lane] = (row && mbx) ? (sumT + sumL + n) >> (sh + 1) : row ? (sumT + (n >> 1)) >> sh : mbx ? (sumL + (n >> 1)) >> sh : 128;
        tlL[lane] = tl;
        for (int i = 0; i < 4; i++) { tpL[lane][i] = T[ex * 4 + i]; lfL[lane][i] = Lf[ey * 4 + i]; }
        for (int j = 0; j < 4; j++)
            for (int i = 0; i < 4; i++) {
                const int s = src[lane][4 * j + i];
                int d = s - dcvL[lane]; eL[lane][0] += d * d;
                d = s - clip8(lfL[lane][j] + tpL[lane][i] - tl); eL[lane][1] += d * d;
                d = s - tpL[lane][i]; eL[lane][2] += d * d;
                d = s - lfL[lane][j]; eL[lane][3] += d * d;
            }
    }
    {   // the warp reductions
        unsigned by_ = 0, bc_ = 0;
        for (int m = 0; m < 4; m++) {
            unsigned ey = 0, ec = 0;
            for (int lane = 0; lane < 24; lane++) (lane < 16 ? ey : ec) += eL[lane][m];
            if (m == 0 || ey < by_) { by_ = ey; ymodeL = m; }
            if (m == 0 || ec < bc_) { bc_ = ec; uvmodeL = m; }
        }
    }
    int16_t *mbl = f.levels + mb * 400;
    for (int lane = 0; lane < 32; lane++) {
        const int plane = lane < 16 ? 0 : lane < 20 ? 1 : lane < 24 ? 2 : 3;
        const int mode = plane == 0 ? ymodeL : uvmodeL, dcv = dcvL[lane], tl = tlL[lane];
        int d[16];
        for (int j = 0; j < 4; j++)
            for (int i = 0; i < 4; i++) {
                const int p = mode == 0 ? dcv : mode == 1 ? clip8(lfL[lane][j] + tpL[lane][i] - tl) : mode == 2 ? tpL[lane][i] : lfL[lane][j];
                pred[lane][4 * j + i] = p; d[4 * j + i] = src[lane][4 * j + i] - p;
            }
        fdct4(d, coef[lane]);
        if (plane == 0) sDc[lane] = coef[lane][0];
    }
    {   // lane 24: the Y2
        int t[16], w2[16], dq[16];
        for (int i = 0; i < 4; i++) {
            const int a0 = sDc[4 * i] + sDc[4 * i + 2], a1 = sDc[4 * i + 1] + sDc[4 * i + 3], a2 = sDc[4 * i + 1] - sDc[4 * i + 3], a3 = sDc[4 * i] - sDc[4 * i + 2];
            t[0 + i * 4] = a0 + a1; t[1 + i * 4] = a3 + a2; t[2 + i * 4] = a3 - a2; t[3 + i * 4] = a0 - a1;
        }
        for (int i = 0; i < 4; i++) {
            const int a0 = t[0 + i] + t[8 + i], a1 = t[4 + i] + t[12 + i], a2 = t[4 + i] - t[12 + i], a3 = t[0 + i] - t[8 + i];
            w2[0 + i] = (a0 + a1) >> 1; w2[4 + i] = (a3 + a2) >> 1; w2[8 + i] = (a3 - a2) >> 1; w2[12 + i] = (a0 - a1) >> 1;
        }
        int nz = 0;
        for (int s = 0; s < 16; s++) {
            const int q = s == 0 ? f.q[2] : f.q[3], l = quant1(w2[zig[s]], q);
            dq[zig[s]] = l * q; nz |= l; sLv16[0][s] = (int16_t)l;
        }
        sY2nz = nz;
        int dummy;
        rate[24] = vp8bp_block_rate(sLv16[0], 1, 0, 0, &dummy);
        for (int i = 0; i < 4; i++) {
            const int a0 = dq[0 + i] + dq[12 + i], a1 = dq[4 + i] + dq[8 + i], a2 = dq[4 + i] - dq[8 + i], a3 = dq[0 + i] - dq[12 + i];
            t[0 + i] = a0 + a1; t[8 + i] = a0 - a1; t[4 + i] = a3 + a2; t[12 + i] = a3 - a2;
        }
        for (int i = 0; i < 4; i++) {
            const int dd = t[0 + i * 4] + 3, a0 = dd + t[3 + i * 4], a1 = t[1 + i * 4] + t[2 + i * 4], a2 = t[1 + i * 4] - t[2 + i * 4], a3 = dd - t[3 + i * 4];
            sDcRec[4 * i + 0] = (a0 + a1) >> 3; sDcRec[4 * i + 1] = (a3 + a2) >> 3; sDcRec[4 * i + 2] = (a0 - a1) >> 3; sDcRec[4 * i + 3] = (a3 - a2) >> 3;
        }
    }
    for (int lane = 0; lane < 24; lane++) {
        const int plane = lane < 16 ? 0 : lane < 20 ? 1 : 2;
        const int k = plane == 0 ? lane : plane == 1 ? lane - 16 : lane - 20;
        const int bx = plane == 0 ? (k & 3) : (k & 1), by = plane == 0 ? (k >> 2) : (k >> 1);
        const int qdc = plane == 0 ? f.q[0] : f.q[4], qac = plane == 0 ? f.q[1] : f.q[5];
        int dq[16], res[16], nz = 0;
        int16_t lv[16];
        for (int s = 0; s < 16; s++) {
            const int q = s == 0 ? qdc : qac;
            const int l = (plane == 0 && s == 0) ? 0 : quant1(coef[lane][zig[s]], q);
            dq[zig[s]] = l * q; nz |= l; lv[s] = (int16_t)l;
        }
        if (plane == 0) dq[0] = sDcRec[k];
        idct4(dq, res);
        nzL[lane] = nz;
        if (plane == 0) {
            memcpy(sLv16[1 + k], lv, 32);
            for (int j = 0; j < 4; j++)
                for (int i = 0; i < 4; i++) {
                    const int r = clip8(pred[lane][4 * j + i] + res[4 * j + i]), d = src[lane][4 * j + i] - r;
                    sRec16[(by * 4 + j) * 16 + bx * 4 + i] = (uint8_t)r; sse[lane] += d * d;
                }
        } else {
            uint8_t *R = plane == 1 ? f.RU : f.RV;
            memcpy(mbl + (plane == 1 ? 17 + k : 21 + k) * 16, lv, 32);
            for (int j = 0; j < 4; j++)
                for (int i = 0; i < 4; i++) {
                    const int r = clip8(pred[lane][4 * j + i] + res[4 * j + i]);
                    R[(size_t)(row * 8 + by * 4 + j) * cs + mbx * 8 + bx * 4 + i] = (uint8_t)r;
                    if (bx == 1 && i == 3) sCLeft[plane - 1][by * 4 + j] = (uint8_t)r;
                }
        }
    }
    unsigned acnz = 0; bool chroma_nz = false;
    for (int lane = 0; lane < 24; lane++) { if (lane < 16 && nzL[lane]) acnz |= 1u << lane; if (lane >= 16 && nzL[lane]) chroma_nz = true; }
    for (int k = 0; k < 16; k++) {
        int dummy;
        const int bx = k & 3, by = k >> 2, ctx = (by ? (acnz >> (k - 4)) & 1 : 0) + (bx ? (acnz >> (k - 1)) & 1 : 0);
        rate[k] = vp8bp_block_rate(sLv16[1 + k], 0, 1, ctx, &dummy);
    }
    uint32_t sse16 = 0, rate16 = 0;
    for (int lane = 0; lane < 32; lane++) { sse16 += sse[lane]; rate16 += rate[lane]; }
    const uint64_t score16 = vp8bp_score(sse16, rate16 + vp8bp_i16_cost(ymodeL), lam);
    // ---- phase B: 10 anti-diagonal steps over 20 lanes
    for (int t = 0; t < 10; t++) {
        int16_t lv[20][16]; uint8_t rec[20][16]; int bnz[20] = {0}; bool active[20]; int xs[20], ysb[20];
        for (int lane = 0; lane < 20; lane++) {
            const int slot = lane / 10, m = lane - 10 * slot;
            const int y = (t <= 3 ? 0 : (t - 2) >> 1) + slot, x = t - 2 * y;
            active[lane] = y <= std::min(3, t >> 1) && x >= 0; xs[lane] = x; ysb[lane] = y;
            if (!active[lane]) continue;
            const int kb = 4 * y + x;
            uint8_t eg[13], p[16];
            vp8bp_edges(sTop, sLeft, sRec4, 16, x, y, eg);
            vp8bp_pred4(m, eg, p);
            int d[16], c[16], dq[16], res[16];
            for (int i = 0; i < 16; i++) d[i] = sSrc[(4 * y + (i >> 2)) * 16 + 4 * x + (i & 3)] - p[i];
            fdct4(d, c);
            for (int s = 0; s < 16; s++) {
                const int q = s == 0 ? f.q[0] : f.q[1], l = quant1(c[zig[s]], q);
                lv[lane][s] = (int16_t)l; dq[zig[s]] = l * q;
            }
            idct4(dq, res);
            uint32_t e2 = 0;
            for (int i = 0; i < 16; i++) {
                const int r = clip8(p[i] + res[i]), dd = sSrc[(4 * y + (i >> 2)) * 16 + 4 * x + (i & 3)] - r;
                rec[lane][i] = (uint8_t)r; e2 += dd * dd;
            }
            const int ctx = (y ? sNz4[kb - 4] : 0) + (x ? sNz4[kb - 1] : 0);
            const uint32_t r = vp8bp_block_rate(lv[lane], 3, 0, ctx, &bnz[lane]) + vp8bp_bmode_cost(y ? sMode4[kb - 4] : sAboveModes[x], x ? sMode4[kb - 1] : sLeftModes[y], m);
            sScore[lane] = vp8bp_score(e2, r, lam);
        }
        for (int lane = 0; lane < 20; lane++) {
            if (!active[lane]) continue;
            const int slot = lane / 10, m = lane - 10 * slot, x = xs[lane], y = ysb[lane], kb = 4 * y + x;
            int best = 0;
            for (int i = 1; i < 10; i++) if (sScore[10 * slot + i] < sScore[10 * slot + best]) best = i;
            if (best != m) continue;
            for (int i = 0; i < 16; i++) { sRec4[(4 * y + (i >> 2)) * 16 + 4 * x + (i & 3)] = rec[lane][i]; sLv4[kb][i] = lv[lane][i]; }
            sNz4[kb] = (uint8_t)bnz[lane]; sMode4[kb] = (uint8_t)m; sBlockScore[kb] = sScore[lane];
        }
    }
    // ---- the decision and the write-out
    uint64_t sum4 = 0;
    for (int k = 0; k < 16; k++) sum4 += sBlockScore[k];
    const bool bp = sum4 + (uint64_t)lam * vp8bp_bit(0, VP8BP_FLAG_PROB) < score16;
    const uint8_t *rec = bp ? sRec4 : sRec16;
    bool lnz = false;
    for (int j = 0; j < 16; j++) memcpy(f.RY + (size_t)(row * 16 + j) * ys + mbx * 16, rec + 16 * j, 16);
    for (int k = 0; k < 16; k++) f.bmodes[mb * 16 + k] = bp ? sMode4[k] : (uint8_t)ymodeL;
    for (int b = 0; b < 17; b++)
        for (int i = 0; i < 16; i++) {
            const int16_t v = bp ? (b ? sLv4[b - 1][i] : 0) : sLv16[b][i];
            mbl[b * 16 + i] = v; lnz |= bp && v != 0;
        }
    const bool any = bp ? (lnz || chroma_nz) : (acnz != 0 || sY2nz != 0 || chroma_nz);
    for (int j = 0; j < 16; j++) sLeft[j] = rec[j * 16 + 15];
    for (int j = 0; j < 4; j++) sLeftModes[j] = bp ? sMode4[4 * j + 3] : (uint8_t)ymodeL;
    f.modes[mb * 4] = (uint8_t)(bp ? 4 : ymodeL); f.modes[mb * 4 + 1] = (uint8_t)uvmodeL; f.modes[mb * 4 + 2] = any ? 0 : 1; f.modes[mb * 4 + 3] = 0;
}

} // namespace

// Y, U, V: source planes, macroblock-padded (pitch mbw*16 / mbw*8); q[6]: dequantisation factors.  Fills levels [nmb][400],
// modes [nmb][4], bmodes [nmb][16] and the unfiltered reconstruction RY, RU, RV.  Returns the number of reads of a macroblock the
// trail-by-two wavefront would not have finished (0 when the schedule is sound).
extern "C" int emul_vp8_bpred(const uint8_t *Y, const uint8_t *U, const uint8_t *V, int mbw, int mbh, const int *q, int16_t *levels,
                              uint8_t *modes, uint8_t *bmodes, uint8_t *RY, uint8_t *RU, uint8_t *RV)
{
    int violations = 0;
    Frame f{mbw, mbh, {q[0], q[1], q[2], q[3], q[4], q[5]}, Y, U, V, RY, RU, RV, modes, bmodes, levels, std::vector<uint8_t>((size_t)mbw * mbh, 0), &violations};
    // each row's warp carries its left edge and left sub-block modes from one macroblock to the next
    std::vector<uint8_t> left((size_t)mbh * 16), cleft((size_t)mbh * 16), lmodes((size_t)mbh * 4);
    // macroblock (x, y) may run once (x + 1, y - 1) is done (or the row above is finished): at its earliest, step x + 2y.  Within a
    // step the rows go bottom-up, so a read of a macroblock of the same step would be caught.
    for (int t = 0; t <= mbw - 1 + 2 * (mbh - 1); t++)
        for (int y = std::min(mbh - 1, t / 2); y >= 0; y--) {
            const int x = t - 2 * y;
            if (x < 0 || x >= mbw) continue;
            encode_mb(f, y, x, &left[(size_t)y * 16], reinterpret_cast<uint8_t (*)[8]>(&cleft[(size_t)y * 16]), &lmodes[(size_t)y * 4]);
            f.done[(size_t)y * mbw + x] = 1;
        }
    return violations;
}
