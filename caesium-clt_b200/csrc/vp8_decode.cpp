// vp8_decode.cpp -- see vp8_decode.h.  RFC 6386 key-frame decoding: frame header, segment / filter / quantiser headers, per-macroblock
// intra modes (16x16, and 4x4 "B_PRED" with its 10 sub-block modes and contextual mode probabilities), DCT token partitions, inverse
// WHT / DCT, intra prediction with libwebp's frame-border conventions, simple and normal loop filters, then libwebp's output stage.
#include "vp8_decode.h"
#include "vp8l_decode.h"
#include <algorithm>
#include <cstring>
#include "vp8_tables.h"
#include "vp8_bpred_core.h"

namespace b200 {
namespace {

enum { B_DC = 0 };
enum { DC_PRED = 0, TM_PRED = 1, V_PRED = 2, H_PRED = 3 };
const uint8_t kZigzag4[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};
const uint8_t kBands4[17] = {0, 1, 2, 3, 6, 4, 5, 6, 6, 6, 6, 6, 6, 6, 6, 7, 0};
const uint8_t kCat3[] = {173, 148, 140, 0}, kCat4[] = {176, 155, 140, 135, 0}, kCat5[] = {180, 157, 141, 134, 130, 0},
              kCat6[] = {254, 254, 243, 230, 196, 177, 153, 140, 133, 130, 129, 0};
const uint8_t *const kCat3456[] = {kCat3, kCat4, kCat5, kCat6};

struct BoolDec {                 // RFC 6386 section 7
    const uint8_t *p, *end; uint32_t value = 0, range = 255; int bit_count = 0;
    void init(const uint8_t *b, const uint8_t *e) { p = b; end = e; value = 0; for (int i = 0; i < 2; i++) value = (value << 8) | (p < end ? *p++ : 0); range = 255; bit_count = 0; }
    inline int bit(int prob)
    {
        const uint32_t split = 1 + (((range - 1) * (uint32_t)prob) >> 8), big = split << 8;
        int r;
        if (value >= big) { r = 1; range -= split; value -= big; } else { r = 0; range = split; }
        while (range < 128) { value <<= 1; range <<= 1; if (++bit_count == 8) { bit_count = 0; value |= (p < end ? *p++ : 0); } }
        return r;
    }
    uint32_t lit(int n) { uint32_t v = 0; while (n-- > 0) v = (v << 1) | (uint32_t)bit(128); return v; }
    int slit(int n) { const int v = (int)lit(n); return bit(128) ? -v : v; }
};

inline uint8_t clip8(int v) { return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v); }
inline int clipq(int v, int m) { return v < 0 ? 0 : v > m ? m : v; }

struct Quant { int y1[2], y2[2], uv[2]; };
struct FInfo { uint8_t limit, ilevel, inner, hev; };

// ---- inverse transforms (libwebp TransformOne / TransformWHT: the RFC's exact integer arithmetic) --------------------------------
// (64-bit products: corrupt streams can carry coefficients whose 32-bit product overflows; valid ones never get near)
inline int mul1(int a) { return (int)(((long long)a * 20091) >> 16) + a; }
inline int mul2(int a) { return (int)(((long long)a * 35468) >> 16); }
void idct_add(const int16_t *in, uint8_t *dst, int stride)
{
    int C[16], *tmp = C;
    for (int i = 0; i < 4; i++) {
        const int a = in[0] + in[8], b = in[0] - in[8], c = mul2(in[4]) - mul1(in[12]), d = mul1(in[4]) + mul2(in[12]);
        tmp[0] = a + d; tmp[1] = b + c; tmp[2] = b - c; tmp[3] = a - d;
        tmp += 4; in++;
    }
    tmp = C;
    for (int i = 0; i < 4; i++) {
        const int dc = tmp[0] + 4, a = dc + tmp[8], b = dc - tmp[8], c = mul2(tmp[4]) - mul1(tmp[12]), d = mul1(tmp[4]) + mul2(tmp[12]);
        dst[0] = clip8(dst[0] + ((a + d) >> 3)); dst[1] = clip8(dst[1] + ((b + c) >> 3)); dst[2] = clip8(dst[2] + ((b - c) >> 3)); dst[3] = clip8(dst[3] + ((a - d) >> 3));
        tmp++; dst += stride;
    }
}
void iwht(const int16_t *in, int16_t *out /* 16 blocks x 16 coefficients: DC slots */)
{
    int tmp[16];
    for (int i = 0; i < 4; i++) {
        const int a0 = in[0 + i] + in[12 + i], a1 = in[4 + i] + in[8 + i], a2 = in[4 + i] - in[8 + i], a3 = in[0 + i] - in[12 + i];
        tmp[0 + i] = a0 + a1; tmp[8 + i] = a0 - a1; tmp[4 + i] = a3 + a2; tmp[12 + i] = a3 - a2;
    }
    for (int i = 0; i < 4; i++) {
        const int dc = tmp[0 + i * 4] + 3, a0 = dc + tmp[3 + i * 4], a1 = tmp[1 + i * 4] + tmp[2 + i * 4], a2 = tmp[1 + i * 4] - tmp[2 + i * 4], a3 = dc - tmp[3 + i * 4];
        out[0] = (int16_t)((a0 + a1) >> 3); out[16] = (int16_t)((a3 + a2) >> 3); out[32] = (int16_t)((a0 - a1) >> 3); out[48] = (int16_t)((a3 - a2) >> 3);
        out += 64;
    }
}

// ---- intra prediction on a bordered work area (row -1 / column -1 hold the neighbours) ---------------------------------------------
// whole-block predictors (16x16 luma / 8x8 chroma); have_top / have_left only matter for DC (the other modes read the 127 / 129 borders)
void pred_block(int mode, uint8_t *d, int s, int n, bool have_top, bool have_left)
{
    const uint8_t *top = d - s;
    switch (mode) {
        case DC_PRED: {
            int dc; const int sh = n == 16 ? 4 : 3;
            if (have_top && have_left) { dc = n; for (int i = 0; i < n; i++) dc += top[i] + d[-1 + i * s]; dc >>= sh + 1; }
            else if (have_left) { dc = n / 2; for (int i = 0; i < n; i++) dc += d[-1 + i * s]; dc >>= sh; }
            else if (have_top) { dc = n / 2; for (int i = 0; i < n; i++) dc += top[i]; dc >>= sh; }
            else dc = 0x80;
            for (int y = 0; y < n; y++) memset(d + y * s, dc, (size_t)n);
            break;
        }
        case TM_PRED: { const int X = top[-1]; for (int y = 0; y < n; y++) { const int l = d[-1 + y * s]; for (int x = 0; x < n; x++) d[x + y * s] = clip8(top[x] + l - X); } break; }
        case V_PRED: for (int y = 0; y < n; y++) memcpy(d + y * s, top, (size_t)n); break;
        default: for (int y = 0; y < n; y++) memset(d + y * s, d[-1 + y * s], (size_t)n); break;
    }
}

// ---- loop filters (RFC 6386 section 15; libwebp's formulation) ----------------------------------------------------------------------
inline int sclip1(int v) { return v < -128 ? -128 : v > 127 ? 127 : v; }       // [-1020, 1020] -> [-128, 127]
inline int sclip2(int v) { return v < -16 ? -16 : v > 15 ? 15 : v; }           // [-112, 112] -> [-16, 15]
inline int iabs(int v) { return v < 0 ? -v : v; }
inline void filter2(uint8_t *p, int step)
{
    const int p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step];
    const int a = 3 * (q0 - p0) + sclip1(p1 - q1), a1 = sclip2((a + 4) >> 3), a2 = sclip2((a + 3) >> 3);
    p[-step] = clip8(p0 + a2); p[0] = clip8(q0 - a1);
}
inline void filter4(uint8_t *p, int step)
{
    const int p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step];
    const int a = 3 * (q0 - p0), a1 = sclip2((a + 4) >> 3), a2 = sclip2((a + 3) >> 3), a3 = (a1 + 1) >> 1;
    p[-2 * step] = clip8(p1 + a3); p[-step] = clip8(p0 + a2); p[0] = clip8(q0 - a1); p[step] = clip8(q1 - a3);
}
inline void filter6(uint8_t *p, int step)
{
    const int p2 = p[-3 * step], p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step], q2 = p[2 * step];
    const int a = sclip1(3 * (q0 - p0) + sclip1(p1 - q1));
    const int a1 = (27 * a + 63) >> 7, a2 = (18 * a + 63) >> 7, a3 = (9 * a + 63) >> 7;
    p[-3 * step] = clip8(p2 + a3); p[-2 * step] = clip8(p1 + a2); p[-step] = clip8(p0 + a1);
    p[0] = clip8(q0 - a1); p[step] = clip8(q1 - a2); p[2 * step] = clip8(q2 - a3);
}
inline bool hev(const uint8_t *p, int step, int t) { return iabs(p[-2 * step] - p[-step]) > t || iabs(p[step] - p[0]) > t; }
inline bool needs1(const uint8_t *p, int step, int t) { return 4 * iabs(p[-step] - p[0]) + iabs(p[-2 * step] - p[step]) <= t; }
inline bool needs2(const uint8_t *p, int step, int t, int it)
{
    const int p3 = p[-4 * step], p2 = p[-3 * step], p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step], q2 = p[2 * step], q3 = p[3 * step];
    if (4 * iabs(p0 - q0) + iabs(p1 - q1) > t) return false;
    return iabs(p3 - p2) <= it && iabs(p2 - p1) <= it && iabs(p1 - p0) <= it && iabs(q3 - q2) <= it && iabs(q2 - q1) <= it && iabs(q1 - q0) <= it;
}
void simple_edge(uint8_t *p, int hstride, int vstride, int n, int thresh)
{
    const int t2 = 2 * thresh + 1;
    for (int i = 0; i < n; i++, p += vstride) if (needs1(p, hstride, t2)) filter2(p, hstride);
}
void loop26(uint8_t *p, int hstride, int vstride, int n, int thresh, int ithresh, int hevt)
{
    const int t2 = 2 * thresh + 1;
    for (int i = 0; i < n; i++, p += vstride) if (needs2(p, hstride, t2, ithresh)) { if (hev(p, hstride, hevt)) filter2(p, hstride); else filter6(p, hstride); }
}
void loop24(uint8_t *p, int hstride, int vstride, int n, int thresh, int ithresh, int hevt)
{
    const int t2 = 2 * thresh + 1;
    for (int i = 0; i < n; i++, p += vstride) if (needs2(p, hstride, t2, ithresh)) { if (hev(p, hstride, hevt)) filter2(p, hstride); else filter4(p, hstride); }
}

inline uint32_t rd24(const uint8_t *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16); }
inline uint32_t rd32(const uint8_t *p) { return rd24(p) | ((uint32_t)p[3] << 24); }

// the VP8 payload of a RIFF/WEBP file; flags what else is in there
struct OtherChunks { const uint8_t *alph = nullptr, *vp8l = nullptr; size_t alph_len = 0, vp8l_len = 0; };
bool find_vp8(const uint8_t *d, size_t n, const uint8_t **vp8, size_t *vp8_len, WebpInfo &info, std::string &err, OtherChunks *oc = nullptr)
{
    if (n < 20 || memcmp(d, "RIFF", 4) || memcmp(d + 8, "WEBP", 4)) { err = "not a WebP file"; return false; }
    size_t i = 12; *vp8 = nullptr;
    while (i + 8 <= n) {
        const uint8_t *tag = d + i; const size_t sz = rd32(d + i + 4);
        if (sz > n - i - 8) { err = "truncated WebP chunk"; return false; }
        if (!memcmp(tag, "VP8 ", 4) && !*vp8) { *vp8 = d + i + 8; *vp8_len = sz; }
        else if (!memcmp(tag, "VP8L", 4)) { info.lossless = true; if (oc && !oc->vp8l) { oc->vp8l = d + i + 8; oc->vp8l_len = sz; } }
        else if (!memcmp(tag, "ALPH", 4)) { info.has_alpha = true; if (oc && !oc->alph) { oc->alph = d + i + 8; oc->alph_len = sz; } }
        else if (!memcmp(tag, "ANIM", 4) || !memcmp(tag, "ANMF", 4)) info.animated = true;
        else if (!memcmp(tag, "VP8X", 4) && sz >= 10) { info.width = 1 + (int)rd24(d + i + 12); info.height = 1 + (int)rd24(d + i + 15); }
        i += 8 + sz + (sz & 1);
    }
    if (*vp8 && *vp8_len >= 10) {
        const uint8_t *f = *vp8;
        if (f[3] == 0x9d && f[4] == 0x01 && f[5] == 0x2a) { info.width = (f[6] | (f[7] << 8)) & 0x3fff; info.height = (f[8] | (f[9] << 8)) & 0x3fff; }
    }
    return true;
}

} // namespace

bool webp_probe(const uint8_t *data, size_t len, WebpInfo &info, std::string &err)
{
    const uint8_t *v; size_t vl = 0;
    info = WebpInfo();
    return find_vp8(data, len, &v, &vl, info, err);
}

int webp_decode_rgb(const uint8_t *data, size_t len, WebpInfo &info, std::vector<uint8_t> &rgb, std::string &err, std::vector<uint8_t> *alpha)
{
    const uint8_t *f; size_t flen = 0;
    OtherChunks oc;
    info = WebpInfo();
    if (alpha) alpha->clear();
    if (!find_vp8(data, len, &f, &flen, info, err, &oc)) return 2;
    if (info.animated) { err = "animated WebP is outside the GPU path (route to caesium::compress_in_memory)"; return 1; }
    return webp_decode_chunks(f, flen, oc.alph, oc.alph_len, oc.vp8l, oc.vp8l_len, info, rgb, err, alpha);
}

int webp_decode_chunks(const uint8_t *f, size_t flen, const uint8_t *alph, size_t alph_len, const uint8_t *vp8l, size_t vp8l_len, WebpInfo &info,
                       std::vector<uint8_t> &rgb, std::string &err, std::vector<uint8_t> *alpha)
{
    if (alpha) alpha->clear();
    if (info.lossless && !f) {
        // lossless file: the VP8L decoder gives ARGB; the alpha plane is reported only if some pixel is not opaque
        std::vector<uint32_t> argb; int W = 0, H = 0; bool hint = false;
        if (!vp8l_decode_file_chunk(vp8l, vp8l_len, W, H, hint, argb, err)) return 2;
        info.width = W; info.height = H;
        const size_t n = (size_t)W * H;
        rgb.resize(3 * n);
        bool any = false;
        for (size_t i = 0; i < n; i++) { const uint32_t p = argb[i]; rgb[i] = (uint8_t)(p >> 16); rgb[n + i] = (uint8_t)(p >> 8); rgb[2 * n + i] = (uint8_t)p; any |= (p >> 24) != 0xFFu; }
        info.has_alpha = any;
        if (any) {
            if (!alpha) { err = "WebP with an alpha plane: the caller did not ask for it"; return 1; }
            alpha->resize(n);
            for (size_t i = 0; i < n; i++) (*alpha)[i] = (uint8_t)(argb[i] >> 24);
        }
        return 0;
    }
    if (info.has_alpha && !alpha) { err = "WebP with an alpha plane: the caller did not ask for it"; return 1; }
    if (!f || flen < 10) { err = "no VP8 bitstream in the WebP file"; return 2; }
    // ---- frame tag + key-frame header (RFC 6386 9.1)
    const uint32_t tag = rd24(f);
    if (tag & 1) { err = "WebP still image is not a key frame"; return 2; }
    const size_t part0 = tag >> 5;
    if (f[3] != 0x9d || f[4] != 0x01 || f[5] != 0x2a) { err = "bad VP8 start code"; return 2; }
    const int W = (f[6] | (f[7] << 8)) & 0x3fff, H = (f[8] | (f[9] << 8)) & 0x3fff;
    if (!W || !H) { err = "empty VP8 frame"; return 2; }
    if (10 + part0 > flen) { err = "truncated VP8 first partition"; return 2; }
    info.width = W; info.height = H;
    const int mbw = (W + 15) >> 4, mbh = (H + 15) >> 4;
    BoolDec br; br.init(f + 10, f + 10 + part0);
    br.bit(128); br.bit(128);                                  // colour space, clamping type (libwebp ignores both on output)
    // ---- segmentation (9.3)
    bool use_segment = br.bit(128) != 0, update_map = false, absolute_delta = true;
    int seg_q[4] = {0, 0, 0, 0}, seg_f[4] = {0, 0, 0, 0}; uint8_t seg_p[3] = {255, 255, 255};
    if (use_segment) {
        update_map = br.bit(128) != 0;
        if (br.bit(128)) {
            absolute_delta = br.bit(128) != 0;
            for (int s = 0; s < 4; s++) seg_q[s] = br.bit(128) ? br.slit(7) : 0;
            for (int s = 0; s < 4; s++) seg_f[s] = br.bit(128) ? br.slit(6) : 0;
        }
        if (update_map) for (int s = 0; s < 3; s++) seg_p[s] = br.bit(128) ? (uint8_t)br.lit(8) : 255;
    }
    // ---- loop filter header (9.6)
    const bool simple = br.bit(128) != 0;
    const int level = (int)br.lit(6), sharpness = (int)br.lit(3);
    bool use_lf_delta = br.bit(128) != 0; int ref_lf_delta[4] = {0, 0, 0, 0}, mode_lf_delta[4] = {0, 0, 0, 0};
    if (use_lf_delta && br.bit(128)) {
        for (int i = 0; i < 4; i++) if (br.bit(128)) ref_lf_delta[i] = br.slit(6);
        for (int i = 0; i < 4; i++) if (br.bit(128)) mode_lf_delta[i] = br.slit(6);
    }
    const int filter_type = level == 0 ? 0 : simple ? 1 : 2;
    // ---- token partitions (9.5)
    const int nparts = 1 << br.lit(2);
    const uint8_t *pbase = f + 10 + part0, *fend = f + flen;
    if ((size_t)(fend - pbase) < (size_t)3 * (nparts - 1)) { err = "truncated VP8 partition table"; return 2; }
    std::vector<BoolDec> parts((size_t)nparts);
    {
        const uint8_t *sz = pbase, *start = pbase + 3 * (nparts - 1);
        for (int p = 0; p < nparts; p++) {
            size_t psz = p + 1 < nparts ? rd24(sz + 3 * p) : (size_t)(fend - start);
            if (psz > (size_t)(fend - start)) psz = (size_t)(fend - start);
            parts[(size_t)p].init(start, start + psz); start += psz;
        }
    }
    // ---- quantiser (9.6)
    const int base_q = (int)br.lit(7);
    const int dqy1_dc = br.bit(128) ? br.slit(4) : 0, dqy2_dc = br.bit(128) ? br.slit(4) : 0, dqy2_ac = br.bit(128) ? br.slit(4) : 0;
    const int dquv_dc = br.bit(128) ? br.slit(4) : 0, dquv_ac = br.bit(128) ? br.slit(4) : 0;
    Quant qm[4];
    for (int s = 0; s < 4; s++) {
        int q = use_segment ? (absolute_delta ? seg_q[s] : base_q + seg_q[s]) : base_q;
        if (!use_segment && s > 0) { qm[s] = qm[0]; continue; }
        qm[s].y1[0] = VP8_DC_Q[clipq(q + dqy1_dc, 127)]; qm[s].y1[1] = VP8_AC_Q[clipq(q, 127)];
        qm[s].y2[0] = VP8_DC_Q[clipq(q + dqy2_dc, 127)] * 2;
        qm[s].y2[1] = (VP8_AC_Q[clipq(q + dqy2_ac, 127)] * 101581) >> 16; if (qm[s].y2[1] < 8) qm[s].y2[1] = 8;
        qm[s].uv[0] = VP8_DC_Q[clipq(q + dquv_dc, 117)]; qm[s].uv[1] = VP8_AC_Q[clipq(q + dquv_ac, 127)];
    }
    // ---- filter strengths per (segment, 4x4 or not) (libwebp PrecomputeFilterStrengths)
    FInfo fst[4][2];
    for (int s = 0; s < 4; s++) for (int i4 = 0; i4 < 2; i4++) {
        int base_level = use_segment ? (absolute_delta ? seg_f[s] : seg_f[s] + level) : level;
        int lv = base_level;
        if (use_lf_delta) { lv += ref_lf_delta[0]; if (i4) lv += mode_lf_delta[0]; }
        lv = lv < 0 ? 0 : lv > 63 ? 63 : lv;
        FInfo fi{0, 0, (uint8_t)i4, 0};
        if (lv > 0) {
            int il = lv;
            if (sharpness > 0) { il >>= sharpness > 4 ? 2 : 1; if (il > 9 - sharpness) il = 9 - sharpness; }
            if (il < 1) il = 1;
            fi.ilevel = (uint8_t)il; fi.limit = (uint8_t)(2 * lv + il); fi.hev = (uint8_t)(lv >= 40 ? 2 : lv >= 15 ? 1 : 0);
        }
        fst[s][i4] = fi;
    }
    br.bit(128);                                               // refresh_entropy_probs: irrelevant for a single key frame
    // ---- token probabilities (13.4)
    uint8_t coef[4][8][3][11];
    memcpy(coef, VP8_COEF_PROBS, sizeof(coef));
    for (int t = 0; t < 4; t++) for (int b = 0; b < 8; b++) for (int c = 0; c < 3; c++) for (int p = 0; p < 11; p++)
        if (br.bit(VP8_COEF_UPDATE_PROBS[((t * 8 + b) * 3 + c) * 11 + p])) coef[t][b][c][p] = (uint8_t)br.lit(8);
    const bool use_skip = br.bit(128) != 0;
    const int skip_p = use_skip ? (int)br.lit(8) : 0;

    // ---- frame buffers (whole macroblocks), unfiltered reconstruction first
    const int ys = mbw * 16, cs = mbw * 8;
    std::vector<uint8_t> Y((size_t)ys * mbh * 16), U((size_t)cs * mbh * 8), V((size_t)cs * mbh * 8);
    std::vector<FInfo> finfo((size_t)mbw * mbh);
    std::vector<uint8_t> top_modes((size_t)mbw * 4, B_DC), top_nz((size_t)mbw, 0), top_nzdc((size_t)mbw, 0);
    for (int my = 0; my < mbh; my++) {
        BoolDec &tb = parts[(size_t)(my & (nparts - 1))];
        uint8_t left_modes[4] = {B_DC, B_DC, B_DC, B_DC}; unsigned left_nz = 0, left_nzdc = 0;
        for (int mx = 0; mx < mbw; mx++) {
            // -- modes (first partition)
            int segment = 0;
            if (update_map) segment = !br.bit(seg_p[0]) ? br.bit(seg_p[1]) : br.bit(seg_p[2]) + 2;
            bool skip = use_skip ? br.bit(skip_p) != 0 : false;
            const bool i4 = !br.bit(145);
            uint8_t imodes[16]; int ymode = DC_PRED;
            uint8_t *tm = &top_modes[(size_t)mx * 4];
            if (!i4) {
                ymode = br.bit(156) ? (br.bit(128) ? TM_PRED : H_PRED) : (br.bit(163) ? V_PRED : DC_PRED);
                memset(tm, ymode, 4); memset(left_modes, ymode, 4);
            } else {
                for (int y = 0; y < 4; y++) {
                    int ym = left_modes[y];
                    for (int x = 0; x < 4; x++) {
                        const uint8_t *prob = VP8_BMODES_PROBA[tm[x]][ym];
                        int i = VP8_YMODES_INTRA4[br.bit(prob[0])];
                        while (i > 0) i = VP8_YMODES_INTRA4[2 * i + br.bit(prob[i])];
                        ym = -i; tm[x] = (uint8_t)ym; imodes[y * 4 + x] = (uint8_t)ym;
                    }
                    left_modes[y] = (uint8_t)ym;
                }
            }
            const int uvmode = !br.bit(142) ? DC_PRED : !br.bit(114) ? V_PRED : br.bit(183) ? TM_PRED : H_PRED;
            // -- residuals (token partition of this macroblock row)
            int16_t coeffs[25 * 16]; memset(coeffs, 0, sizeof(coeffs));       // 16 Y, 4 U, 4 V blocks (raster positions inside a block); [24] = Y2
            bool any_nz = false;
            const Quant &q = qm[segment];
            auto get_coeffs = [&](int type, int ctx, const int *dq, int n, int16_t *out) -> int {
                const uint8_t *p = coef[type][kBands4[n]][ctx];
                for (; n < 16; ++n) {
                    if (!tb.bit(p[0])) return n;
                    while (!tb.bit(p[1])) { p = coef[type][kBands4[++n]][0]; if (n == 16) return 16; }
                    int v;
                    if (!tb.bit(p[2])) { v = 1; p = coef[type][kBands4[n + 1]][1]; }
                    else {
                        if (!tb.bit(p[3])) { v = !tb.bit(p[4]) ? 2 : 3 + tb.bit(p[5]); }
                        else if (!tb.bit(p[6])) { if (!tb.bit(p[7])) v = 5 + tb.bit(159); else { v = 7 + 2 * tb.bit(165); v += tb.bit(145); } }
                        else {
                            const int bit1 = tb.bit(p[8]), bit0 = tb.bit(p[9 + bit1]), cat = 2 * bit1 + bit0;
                            v = 0; for (const uint8_t *tab = kCat3456[cat]; *tab; ++tab) v += v + tb.bit(*tab);
                            v += 3 + (8 << cat);
                        }
                        p = coef[type][kBands4[n + 1]][2];
                    }
                    out[kZigzag4[n]] = (int16_t)((tb.bit(128) ? -v : v) * dq[n > 0]);
                }
                return 16;
            };
            unsigned tnz_all = top_nz[(size_t)mx], lnz_all = left_nz;
            if (!skip) {
                int first = 0, actype = 3;
                if (!i4) {
                    int16_t dc[16]; memset(dc, 0, sizeof(dc));
                    const int ctx = top_nzdc[(size_t)mx] + (int)left_nzdc;
                    const int nz = get_coeffs(1, ctx, q.y2, 0, dc);
                    top_nzdc[(size_t)mx] = (uint8_t)(nz > 0); left_nzdc = nz > 0;
                    if (nz > 1) iwht(dc, coeffs);
                    else { const int dc0 = (dc[0] + 3) >> 3; for (int i = 0; i < 16; i++) coeffs[i * 16] = (int16_t)dc0; }
                    first = 1; actype = 0;
                }
                unsigned tnz = tnz_all & 0x0f, lnz = lnz_all & 0x0f;
                for (int y = 0; y < 4; y++) {
                    int l = lnz & 1;
                    for (int x = 0; x < 4; x++) {
                        int16_t *dst = coeffs + (y * 4 + x) * 16;
                        const int ctx = l + (int)(tnz & 1), nz = get_coeffs(actype, ctx, q.y1, first, dst);
                        l = nz > first; tnz = (tnz >> 1) | ((unsigned)l << 7);
                        any_nz |= nz > 1 || dst[0] != 0;
                    }
                    tnz >>= 4; lnz = (lnz >> 1) | ((unsigned)l << 7);
                }
                unsigned out_t = tnz, out_l = lnz >> 4;
                for (int ch = 0; ch < 4; ch += 2) {
                    tnz = tnz_all >> (4 + ch); lnz = lnz_all >> (4 + ch);
                    for (int y = 0; y < 2; y++) {
                        int l = lnz & 1;
                        for (int x = 0; x < 2; x++) {
                            int16_t *dst = coeffs + (16 + ch * 2 + y * 2 + x) * 16;
                            const int ctx = l + (int)(tnz & 1), nz = get_coeffs(2, ctx, q.uv, 0, dst);
                            l = nz > 0; tnz = (tnz >> 1) | ((unsigned)l << 3);
                            any_nz |= nz > 1 || dst[0] != 0;
                        }
                        tnz >>= 2; lnz = (lnz >> 1) | ((unsigned)l << 5);
                    }
                    out_t |= (tnz << 4) << ch; out_l |= (lnz & 0xf0) << ch;
                }
                top_nz[(size_t)mx] = (uint8_t)out_t; left_nz = out_l;
            } else {
                top_nz[(size_t)mx] = 0; left_nz = 0;
                if (!i4) { top_nzdc[(size_t)mx] = 0; left_nzdc = 0; }
            }
            if (filter_type) { FInfo fi = fst[segment][i4 ? 1 : 0]; fi.inner |= any_nz ? 1 : 0; finfo[(size_t)my * mbw + mx] = fi; }
            // -- reconstruction on a bordered work area: [1 + 16 rows][1 + 16 + 4 columns]
            {
                enum { WS = 32 };
                uint8_t wa[17 * WS];
                uint8_t *yd = wa + WS + 1;                       // pixel (0, 0)
                // top row incl. top-left and top-right
                if (my > 0) {
                    const uint8_t *above = &Y[(size_t)(my * 16 - 1) * ys + (size_t)mx * 16];
                    memcpy(yd - WS, above, 16);
                    if (mx < mbw - 1) memcpy(yd - WS + 16, above + 16, 4); else memset(yd - WS + 16, above[15], 4);
                    yd[-WS - 1] = mx > 0 ? above[-1] : 129;
                } else memset(yd - WS - 1, 127, 21);
                for (int j = 0; j < 16; j++) yd[j * WS - 1] = mx > 0 ? Y[(size_t)(my * 16 + j) * ys + (size_t)mx * 16 - 1] : 129;
                if (i4) {
                    uint8_t top[21], left[16], e[13], p[16];
                    memcpy(top, yd - WS - 1, 21);
                    for (int j = 0; j < 16; j++) left[j] = yd[j * WS - 1];
                    for (int n = 0; n < 16; n++) {
                        uint8_t *d = yd + (n >> 2) * 4 * WS + (n & 3) * 4;
                        vp8bp_edges(top, left, yd, WS, n & 3, n >> 2, e);
                        vp8bp_pred4(imodes[n], e, p);
                        for (int y = 0; y < 4; y++) memcpy(d + y * WS, p + 4 * y, 4);
                        idct_add(coeffs + n * 16, d, WS);
                    }
                } else {
                    pred_block(ymode, yd, WS, 16, my > 0, mx > 0);
                    for (int n = 0; n < 16; n++) idct_add(coeffs + n * 16, yd + (n >> 2) * 4 * WS + (n & 3) * 4, WS);
                }
                for (int j = 0; j < 16; j++) memcpy(&Y[(size_t)(my * 16 + j) * ys + (size_t)mx * 16], yd + j * WS, 16);
                for (int pl = 0; pl < 2; pl++) {
                    std::vector<uint8_t> &P = pl ? V : U;
                    uint8_t *cd = wa + WS + 1;
                    if (my > 0) { const uint8_t *above = &P[(size_t)(my * 8 - 1) * cs + (size_t)mx * 8]; memcpy(cd - WS, above, 8); cd[-WS - 1] = mx > 0 ? above[-1] : 129; }
                    else memset(cd - WS - 1, 127, 9);
                    for (int j = 0; j < 8; j++) cd[j * WS - 1] = mx > 0 ? P[(size_t)(my * 8 + j) * cs + (size_t)mx * 8 - 1] : 129;
                    pred_block(uvmode, cd, WS, 8, my > 0, mx > 0);
                    for (int n = 0; n < 4; n++) idct_add(coeffs + (16 + pl * 4 + n) * 16, cd + (n >> 1) * 4 * WS + (n & 1) * 4, WS);
                    for (int j = 0; j < 8; j++) memcpy(&P[(size_t)(my * 8 + j) * cs + (size_t)mx * 8], cd + j * WS, 8);
                }
            }
        }
    }
    // ---- loop filter, in place, macroblocks in raster order (the prediction above used unfiltered neighbours)
    if (filter_type) for (int my = 0; my < mbh; my++) for (int mx = 0; mx < mbw; mx++) {
        const FInfo fi = finfo[(size_t)my * mbw + mx];
        if (!fi.limit) continue;
        uint8_t *y = &Y[(size_t)my * 16 * ys + (size_t)mx * 16], *u = &U[(size_t)my * 8 * cs + (size_t)mx * 8], *v = &V[(size_t)my * 8 * cs + (size_t)mx * 8];
        const int limit = fi.limit, il = fi.ilevel, hv = fi.hev;
        if (filter_type == 1) {
            if (mx > 0) simple_edge(y, 1, ys, 16, limit + 4);
            if (fi.inner) for (int k = 1; k < 4; k++) simple_edge(y + 4 * k, 1, ys, 16, limit);
            if (my > 0) simple_edge(y, ys, 1, 16, limit + 4);
            if (fi.inner) for (int k = 1; k < 4; k++) simple_edge(y + 4 * k * ys, ys, 1, 16, limit);
        } else {
            if (mx > 0) { loop26(y, 1, ys, 16, limit + 4, il, hv); loop26(u, 1, cs, 8, limit + 4, il, hv); loop26(v, 1, cs, 8, limit + 4, il, hv); }
            if (fi.inner) { for (int k = 1; k < 4; k++) loop24(y + 4 * k, 1, ys, 16, limit, il, hv); loop24(u + 4, 1, cs, 8, limit, il, hv); loop24(v + 4, 1, cs, 8, limit, il, hv); }
            if (my > 0) { loop26(y, ys, 1, 16, limit + 4, il, hv); loop26(u, cs, 1, 8, limit + 4, il, hv); loop26(v, cs, 1, 8, limit + 4, il, hv); }
            if (fi.inner) { for (int k = 1; k < 4; k++) loop24(y + 4 * k * ys, ys, 1, 16, limit, il, hv); loop24(u + 4 * cs, cs, 1, 8, limit, il, hv); loop24(v + 4 * cs, cs, 1, 8, limit, il, hv); }
        }
    }
    // ---- output: fancy (9-3-3-1) chroma upsampling + libwebp's 14-bit fixed-point YUV -> RGB
    rgb.resize((size_t)3 * W * H);
    const int cw = (W + 1) >> 1, chh = (H + 1) >> 1;
    std::vector<int> cu((size_t)W), cv((size_t)W);
    auto up_row = [&](const uint8_t *a, const uint8_t *b, std::vector<int> &out) {          // a = nearer chroma row, b = farther one
        out[0] = (3 * a[0] + b[0] + 2) >> 2;
        const int n = (W - 1) >> 1;
        for (int x = 1; x <= n; x++) {
            const int tl = a[x - 1], t = a[x], l = b[x - 1], c = b[x];
            const int avg = tl + t + l + c + 8, d12 = (avg + 2 * (t + l)) >> 3, d03 = (avg + 2 * (tl + c)) >> 3;
            out[2 * x - 1] = (d12 + tl) >> 1; out[2 * x] = (d03 + t) >> 1;
        }
        if (!(W & 1)) out[W - 1] = (3 * a[(W - 1) >> 1] + b[(W - 1) >> 1] + 2) >> 2;
    };
    auto c8 = [](int v) -> uint8_t { return (v & ~16383) == 0 ? (uint8_t)(v >> 6) : v < 0 ? 0 : 255; };
    (void)cw;
    for (int yy = 0; yy < H; yy++) {
        const int near = yy >> 1; int far = (yy & 1) == 0 ? near - 1 : near + 1;
        far = far < 0 ? 0 : far > chh - 1 ? chh - 1 : far;
        up_row(&U[(size_t)near * cs], &U[(size_t)far * cs], cu); up_row(&V[(size_t)near * cs], &V[(size_t)far * cs], cv);
        const uint8_t *yr = &Y[(size_t)yy * ys];
        uint8_t *R = &rgb[(size_t)yy * W], *G = &rgb[(size_t)W * H + (size_t)yy * W], *B = &rgb[(size_t)2 * W * H + (size_t)yy * W];
        for (int x = 0; x < W; x++) {
            const int y1 = (yr[x] * 19077) >> 8, u = cu[(size_t)x], v = cv[(size_t)x];
            R[x] = c8(y1 + ((v * 26149) >> 8) - 14234);
            G[x] = c8(y1 - ((u * 6419) >> 8) - ((v * 13320) >> 8) + 8708);
            B[x] = c8(y1 + ((u * 33050) >> 8) - 17685);
        }
    }
    if (info.has_alpha) {
        // the ALPH chunk has the frame's size (for a still image, the canvas's)
        if (!webp_alpha_decode(alph, alph_len, W, H, *alpha, err)) return 2;
        bool any = false;
        for (uint8_t a : *alpha) if (a != 0xFF) { any = true; break; }
        if (!any) { alpha->clear(); info.has_alpha = false; }
    }
    return 0;
}

} // namespace b200
