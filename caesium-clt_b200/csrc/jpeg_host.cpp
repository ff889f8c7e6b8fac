// jpeg_host.cpp -- see jpeg_host.h.  Upstream behaviour restated (mozjpeg 4.x via mozjpeg-sys 2.2.1,
// caesium-clt's Cargo.lock:1035; reached from caesium-clt's src/compressor.rs:305): jdmarker.c (markers),
// jdhuff.c / jdphuff.c (entropy decode), jchuff.c / jcphuff.c (entropy encode, optimised tables),
// jcmarker.c (file layout), jccoefct.c / jctrans.c (dummy blocks), jcparam.c (quality scaling, sampling).
#include "jpeg_host.h"
#include "host_copy.h"
#include <cstring>
#include <cstdlib>
#include <emmintrin.h>

namespace b200 {

const uint8_t kZigzag[64] = {
     0,  1,  8, 16,  9,  2,  3, 10, 17, 24, 32, 25, 18, 11,  4,  5,
    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,  6,  7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63 };

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }

void JpegGeom::finalize()
{
    hmax = vmax = 1;
    for (int c = 0; c < ncomp; c++) { if (hs[c] > hmax) hmax = hs[c]; if (vs[c] > vmax) vmax = vs[c]; }
    mcux = cdiv(width, 8 * hmax); mcuy = cdiv(height, 8 * vmax);
    int64_t off = 0;
    for (int c = 0; c < 4; c++) {
        if (c < ncomp) {
            cw[c] = cdiv(width * hs[c], hmax); ch[c] = cdiv(height * vs[c], vmax);
            rbw[c] = cdiv(cw[c], 8); rbh[c] = cdiv(ch[c], 8);
            bw[c] = mcux * hs[c]; bh[c] = mcuy * vs[c];
        } else { cw[c] = ch[c] = rbw[c] = rbh[c] = bw[c] = bh[c] = 0; }
        comp_offset[c] = off;
        off += (int64_t)bw[c] * bh[c] * 64;
    }
    total_coefs = off;
}

// ---- quality -> tables (jcparam.c; Robidoux base table, SURVEY.md KAT-1) -------------------------------------
static const uint16_t kBaseTable[64] = {
    16, 16, 16, 18, 25, 37, 56, 85,   16, 17, 20, 27, 34, 40, 53, 75,
    16, 20, 24, 31, 43, 62, 91, 135,  18, 27, 31, 40, 53, 74, 106, 156,
    25, 34, 43, 53, 69, 94, 131, 189, 37, 40, 62, 74, 94, 124, 169, 238,
    56, 53, 91, 106, 131, 169, 226, 311, 85, 75, 135, 156, 189, 238, 311, 418 };

void jpeg_quant_table(int quality, int /*which: luma and chroma share base table 3*/, uint16_t out[64])
{
    int q = quality <= 0 ? 1 : (quality > 100 ? 100 : quality);
    int scale = q < 50 ? 5000 / q : 200 - 2 * q;
    for (int i = 0; i < 64; i++) {
        long t = ((long)kBaseTable[i] * scale + 50) / 100;
        out[i] = (uint16_t)(t < 1 ? 1 : (t > 32767 ? 32767 : t));
    }
}

bool jpeg_output_geom(const JpegGeom &in, int quality, int subsampling, JpegGeom &out, std::string &err)
{
    out = JpegGeom();
    out.width = in.width; out.height = in.height; out.ncomp = in.ncomp;
    int lh = 1, lv = 1;
    if (in.ncomp == 3) {
        switch (subsampling) {   // libcaesium set_chroma_subsampling; Auto keeps jpeg_set_defaults' 2x2
            case 444: lh = 1; lv = 1; break;
            case 422: lh = 2; lv = 1; break;
            case 411: lh = 4; lv = 1; break;
            case 420: case 0: lh = 2; lv = 2; break;
            default: err = "invalid chroma subsampling"; return false;
        }
    } else if (in.ncomp != 1) { err = "unsupported component count"; return false; }
    uint16_t nat[64];
    for (int c = 0; c < in.ncomp; c++) { out.cid[c] = c + 1; out.hs[c] = c ? 1 : lh; out.vs[c] = c ? 1 : lv; out.tq[c] = c ? 1 : 0; }
    for (int t = 0; t < (in.ncomp == 3 ? 2 : 1); t++) {
        jpeg_quant_table(quality, t, nat);
        for (int k = 0; k < 64; k++) out.qt[t][k] = nat[kZigzag[k]];
        out.qt_present[t] = true;
    }
    out.finalize();
    return true;
}

// ================================================================================================================
// Reader
// ================================================================================================================
void JpegReader::Huff::build()
{
    memset(look, 0, sizeof(look));
    int code = 0, p = 0;
    for (int l = 1; l <= 16; l++) {
        valoff[l] = p - code;
        for (int i = 0; i < bits[l]; i++, p++, code++) {
            if (l <= 10) {
                int first = code << (10 - l), cnt = 1 << (10 - l);
                if (first + cnt <= 1024) for (int k = 0; k < cnt; k++) look[first + k] = (uint16_t)((l << 8) | vals[p]);
            }
        }
        maxcode[l] = bits[l] ? code - 1 : -1;
        code <<= 1;
    }
    maxcode[17] = 0x7FFFFFFF;
}

namespace {

struct BitReader {
    const uint8_t *p, *end;
    uint64_t acc = 0; int n = 0; bool marker = false;
    inline void refill()
    {
        if (n > 56) return;
        if (!marker && p + 8 <= end) {
            uint64_t w; memcpy(&w, p, 8); w = __builtin_bswap64(w);
            uint64_t v = ~w;
            if (!((v - 0x0101010101010101ull) & ~v & 0x8080808080808080ull)) {   // no 0xFF among the 8 bytes
                acc |= w >> n;
                int take = (64 - n) >> 3;
                p += take; n += take * 8;
                return;
            }
        }
        while (n <= 56) {
            unsigned c = 0;
            if (!marker && p < end) {
                c = *p++;
                if (c == 0xFF) {
                    unsigned c2 = p < end ? *p : 0xD9;
                    if (c2 == 0) p++;
                    else { p--; marker = true; c = 0; }
                }
            }
            acc |= (uint64_t)c << (56 - n);
            n += 8;
        }
    }
    inline unsigned peek(int k) const { return (unsigned)(acc >> (64 - k)); }
    inline void drop(int k) { acc <<= k; n -= k; }
    inline int get(int k) { unsigned v = peek(k); drop(k); return (int)v; }   // 1 <= k <= 16, caller refilled
    inline int bit() { int v = (int)(acc >> 63); acc <<= 1; n--; return v; }
};

inline int extend(int v, int s) { return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v; }

inline int decode_sym(BitReader &b, const JpegReader::Huff &h)
{
    unsigned e = h.look[b.peek(10)];
    if (e) { b.drop(e >> 8); return e & 0xFF; }
    int code = (int)b.peek(16);
    for (int l = 11; l <= 16; l++) {
        int c = code >> (16 - l);
        if (c <= h.maxcode[l]) { b.drop(l); return h.vals[(h.valoff[l] + c) & 0xFF]; }
    }
    return -1;
}

} // namespace

static unsigned rd16(const uint8_t *p) { return ((unsigned)p[0] << 8) | p[1]; }

bool JpegReader::parse_segment(unsigned m, const uint8_t *seg, size_t sl, std::string &err)
{
    if (m == 0xDB) {
        size_t k = 0;
        while (k < sl) {
            int pq = seg[k] >> 4, tq = seg[k] & 15; k++;
            if (tq > 3 || pq > 1) { err = "bad DQT"; return false; }
            if (k + (pq ? 128u : 64u) > sl) { err = "truncated DQT"; return false; }
            for (int z = 0; z < 64; z++) { g_.qt[tq][z] = (uint16_t)(pq ? rd16(seg + k) : seg[k]); k += pq ? 2 : 1; }
            g_.qt_present[tq] = true;
        }
    } else if (m == 0xC4) {
        size_t k = 0;
        while (k + 17 <= sl) {
            int tc = seg[k] >> 4, th = seg[k] & 15; k++;
            if (tc > 1 || th > 3) { err = "bad DHT"; return false; }
            Huff &h = tc ? ac_[th] : dc_[th];
            int n = 0; h.bits[0] = 0;
            for (int l = 1; l <= 16; l++) { h.bits[l] = seg[k++]; n += h.bits[l]; }
            if (n > 256 || k + n > sl) { err = "bad DHT counts"; return false; }
            memset(h.vals, 0, sizeof(h.vals)); memcpy(h.vals, seg + k, n); k += n;
            h.present = true; h.build();
        }
    } else if (m == 0xC0 || m == 0xC1 || m == 0xC2) {
        if (have_sof_) { err = "duplicate SOF"; return false; }
        if (sl < 6) { err = "short SOF"; return false; }
        if (seg[0] != 8) { err = "unsupported sample precision"; return false; }
        g_.progressive = m == 0xC2;
        g_.height = (int)rd16(seg + 1); g_.width = (int)rd16(seg + 3); g_.ncomp = seg[5];
        if (g_.width <= 0 || g_.height <= 0) { err = "empty image"; return false; }
        if ((uint32_t)g_.width > kJpegMaxDimension || (uint32_t)g_.height > kJpegMaxDimension) {      // jdinput.c initial_setup
            err = "Maximum supported image dimension is " + std::to_string(kJpegMaxDimension) + " pixels"; return false;
        }
        if (g_.ncomp != 1 && g_.ncomp != 3) { err = "unsupported component count " + std::to_string(g_.ncomp); return false; }
        if (sl < (size_t)(6 + 3 * g_.ncomp)) { err = "short SOF"; return false; }
        for (int c = 0; c < g_.ncomp; c++) {
            g_.cid[c] = seg[6 + 3 * c]; g_.hs[c] = seg[7 + 3 * c] >> 4; g_.vs[c] = seg[7 + 3 * c] & 15; g_.tq[c] = seg[8 + 3 * c];
            if (g_.hs[c] < 1 || g_.hs[c] > 4 || g_.vs[c] < 1 || g_.vs[c] > 4 || g_.tq[c] > 3) { err = "bad sampling factors"; return false; }
        }
        if (g_.ncomp == 1) g_.hs[0] = g_.vs[0] = 1;
        g_.finalize();
        have_sof_ = true;
    } else if (m == 0xDD) {
        if (sl >= 2) restart_interval_ = (int)rd16(seg);
    } else if ((m >= 0xE0 && m <= 0xEF) || m == 0xFE) {
        const uint8_t *whole = seg - 4; size_t wl = sl + 4;
        if (m == 0xE0 && sl >= 14 && !memcmp(seg, "JFIF\0", 5) && !m_.jfif) { m_.jfif = true; memcpy(m_.jfif_body, seg + 5, 9); m_.jfif_body[7] = m_.jfif_body[8] = 0; }
        else if (m == 0xE0 && m_.jfif) { /* JFXX / duplicate JFIF: dropped */ }
        else if (m == 0xEE && sl >= 12 && !memcmp(seg, "Adobe", 5)) { m_.adobe = true; m_.adobe_transform = seg[11]; }     // not re-emitted: see read_header
        else if (m == 0xE2 && sl >= 12 && !memcmp(seg, "ICC_PROFILE\0", 12)) m_.icc_markers.insert(m_.icc_markers.end(), whole, whole + wl);
        else {
            m_.app_markers.insert(m_.app_markers.end(), whole, whole + wl);
        }
    } else if (m >= 0xC3 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {
        err = "unsupported JPEG process (SOF" + std::to_string(m - 0xC0) + ")"; return false;
    }
    return true;
}

bool JpegReader::read_header(std::string &err)
{
    if (n_ < 4 || d_[0] != 0xFF || d_[1] != 0xD8) { err = "not a JPEG (no SOI)"; return false; }
    pos_ = 2;
    while (pos_ + 3 < n_) {
        if (d_[pos_] != 0xFF) { pos_++; continue; }
        unsigned m = d_[pos_ + 1];
        if (m == 0xFF) { pos_++; continue; }
        if (m == 0x00 || m == 0x01 || (m >= 0xD0 && m <= 0xD8)) { pos_ += 2; continue; }
        if (m == 0xD9) break;
        if (m == 0xDA) {
            if (!have_sof_) { err = "SOS before SOF"; return false; }
            // Colour space, libjpeg's jdapimin.c default_decompress_parms rule: a 3-component file is YCbCr unless an Adobe
            // marker says transform 0, or (no JFIF, no Adobe) its component ids spell "RGB".  Every output of this path is
            // written as JFIF / YCbCr, so RGB-coded sources are handed back (the caller routes them to libcaesium) instead of
            // being re-tagged with the wrong colour space.
            if (g_.ncomp == 3 && ((m_.adobe && m_.adobe_transform == 0) || (!m_.adobe && !m_.jfif && g_.cid[0] == 'R' && g_.cid[1] == 'G' && g_.cid[2] == 'B'))) {
                err = "RGB-coded JPEG (Adobe transform 0) is outside the GPU path (route to caesium::compress_in_memory)"; return false;
            }
            return true;
        }
        size_t L = rd16(d_ + pos_ + 2);
        if (L < 2 || pos_ + 2 + L > n_) { err = "truncated marker segment"; return false; }
        if (!parse_segment(m, d_ + pos_ + 4, L - 2, err)) return false;
        pos_ += 2 + L;
    }
    err = "no image data"; return false;
}

bool JpegReader::decode_scan(const uint8_t *seg, size_t sl, const uint8_t *ecs, const uint8_t **next, int16_t *coefs, std::string &err)
{
    const JpegGeom &g = g_;
    int ns = seg[0];
    if (ns < 1 || ns > g.ncomp || sl < (size_t)(4 + 2 * ns)) { err = "bad SOS"; return false; }
    int ci[4], td[4], ta[4];
    for (int k = 0; k < ns; k++) {
        int id = seg[1 + 2 * k]; ci[k] = -1;
        for (int c = 0; c < g.ncomp; c++) if (g.cid[c] == id) ci[k] = c;
        if (ci[k] < 0) { err = "SOS names unknown component"; return false; }
        td[k] = seg[2 + 2 * k] >> 4; ta[k] = seg[2 + 2 * k] & 15;
        if (td[k] > 3 || ta[k] > 3) { err = "bad table selector"; return false; }
    }
    if (mcu_blocks(ns, ci) > 10) { err = "corrupt JPEG data: more than 10 blocks in an interleaved MCU"; return false; }
    int Ss = seg[1 + 2 * ns], Se = seg[2 + 2 * ns], Ah = seg[3 + 2 * ns] >> 4, Al = seg[3 + 2 * ns] & 15;
    const bool prog = g.progressive;
    if (!prog) { Ss = 0; Se = 63; Ah = Al = 0; }
    else if (Ss > Se || Se > 63 || (Ss == 0 && Se != 0) || (Ss > 0 && ns != 1) || Al > 13) { err = "bad progressive scan parameters"; return false; }
    for (int k = 0; k < ns; k++) {
        if (Ss == 0 && (!prog || Ah == 0) && !dc_[td[k]].present) { err = "missing DC Huffman table"; return false; }
        if (Se > 0 && !ac_[ta[k]].present) { err = "missing AC Huffman table"; return false; }
    }
    const bool inter = ns > 1;
    const int mcus_x = inter ? g.mcux : g.rbw[ci[0]], mcus_y = inter ? g.mcuy : g.rbh[ci[0]];
    // Baseline interleaved scans overwrite every allocated block, so the blocks are zeroed one at a time as they
    // are decoded (cache-hot); anything else needs the whole buffer cleared once up front.
    // Only a scan that carries EVERY component does that: a baseline file may spread its components over several scans
    // (2 + 1, or one each), and then the whole buffer is cleared once, before the first of them -- later scans must not wipe
    // what earlier ones decoded, and a component no scan ever codes stays zero instead of holding a previous image's data.
    const bool zero_per_block = !prog && inter && ns == g.ncomp && !zeroed_;
    if (!zero_per_block && !zeroed_) memset(coefs, 0, (size_t)g.total_coefs * sizeof(int16_t));
    zeroed_ = true;

    BitReader b; b.p = ecs; b.end = d_ + n_;
    int pred[4] = {0, 0, 0, 0}, eobrun = 0, rst = 0;
    const int ri = restart_interval_;
    for (int my = 0; my < mcus_y; my++) for (int mx = 0; mx < mcus_x; mx++) {
        if (ri && rst == ri) {   // jdhuff.c process_restart
            b.n = 0; b.acc = 0;
            const uint8_t *q = b.p, *e = d_ + n_;
            while (q + 1 < e && !(q[0] == 0xFF && q[1] >= 0xD0 && q[1] <= 0xD7)) {
                if (q[0] == 0xFF && q[1] != 0 && q[1] != 0xFF) break;
                q++;
            }
            if (q + 1 < e && q[0] == 0xFF && q[1] >= 0xD0 && q[1] <= 0xD7) q += 2;
            b.p = q; b.marker = false;
            pred[0] = pred[1] = pred[2] = pred[3] = 0; eobrun = 0; rst = 0;
        }
        rst++;
        for (int i = 0; i < ns; i++) {
            const int c = ci[i];
            const int nbx = inter ? g.hs[c] : 1, nby = inter ? g.vs[c] : 1;
            int16_t *cbase = coefs + g.comp_offset[c];
            for (int by = 0; by < nby; by++) for (int bx = 0; bx < nbx; bx++) {
                const int row = inter ? my * g.vs[c] + by : my, col = inter ? mx * g.hs[c] + bx : mx;
                int16_t *blk = cbase + ((size_t)row * g.bw[c] + col) * 64;
                if (!prog) {
                    if (zero_per_block) {
                        __m128i z = _mm_setzero_si128();
                        for (int k = 0; k < 8; k++) _mm_storeu_si128(reinterpret_cast<__m128i *>(blk) + k, z);
                    }
                    const Huff &hd = dc_[td[i]], &ha = ac_[ta[i]];
                    b.refill();
                    int s = decode_sym(b, hd);
                    if (s < 0 || s > 16) { err = "corrupt JPEG data: bad DC code"; return false; }
                    if (s) { b.refill(); pred[i] += extend(b.get(s), s); }
                    blk[0] = (int16_t)pred[i];
                    for (int k = 1; k < 64;) {
                        b.refill();
                        int rs = decode_sym(b, ha);
                        if (rs < 0) { err = "corrupt JPEG data: bad AC code"; return false; }
                        int r = rs >> 4; s = rs & 15;
                        if (s) {
                            k += r; if (k > 63) break;
                            blk[k] = (int16_t)extend(b.get(s), s);   // <= 16 + 16 bits since the refill: still buffered
                            k++;
                        } else { if (r != 15) break; k += 16; }
                    }
                } else if (Ss == 0) {
                    b.refill();
                    if (Ah == 0) {
                        int s = decode_sym(b, dc_[td[i]]);
                        if (s < 0 || s > 16) { err = "corrupt JPEG data: bad DC code"; return false; }
                        if (s) { b.refill(); pred[i] += extend(b.get(s), s); }
                        blk[0] = (int16_t)(pred[i] * (1 << Al));
                    } else if (b.bit()) blk[0] |= (int16_t)(1 << Al);
                } else if (Ah == 0) {
                    if (eobrun > 0) { eobrun--; continue; }
                    const Huff &ha = ac_[ta[i]];
                    for (int k = Ss; k <= Se; k++) {
                        b.refill();
                        int rs = decode_sym(b, ha);
                        if (rs < 0) { err = "corrupt JPEG data: bad AC code"; return false; }
                        int r = rs >> 4, s = rs & 15;
                        if (s) { k += r; if (k > 63) break; blk[k] = (int16_t)(extend(b.get(s), s) * (1 << Al)); }
                        else if (r == 15) k += 15;
                        else { eobrun = 1 << r; if (r) { b.refill(); eobrun += b.get(r); } eobrun--; break; }
                    }
                } else {
                    const Huff &ha = ac_[ta[i]];
                    const int p1 = 1 << Al, m1 = -(1 << Al);
                    int k = Ss;
                    if (eobrun == 0) {
                        for (; k <= Se; k++) {
                            b.refill();
                            int rs = decode_sym(b, ha);
                            if (rs < 0) { err = "corrupt JPEG data: bad AC code"; return false; }
                            int r = rs >> 4, s = rs & 15, val = 0;
                            if (s) val = b.bit() ? p1 : m1;
                            else if (r != 15) { eobrun = 1 << r; if (r) { b.refill(); eobrun += b.get(r); } break; }
                            do {
                                int16_t *cf = blk + k;
                                if (*cf != 0) {
                                    b.refill();
                                    if (b.bit() && (*cf & p1) == 0) *cf = (int16_t)(*cf >= 0 ? *cf + p1 : *cf + m1);
                                } else if (--r < 0) break;
                                k++;
                            } while (k <= Se);
                            if (val && k <= 63) blk[k] = (int16_t)val;
                        }
                    }
                    if (eobrun > 0) {
                        for (; k <= Se; k++) {
                            int16_t *cf = blk + k;
                            if (*cf != 0) { b.refill(); if (b.bit() && (*cf & p1) == 0) *cf = (int16_t)(*cf >= 0 ? *cf + p1 : *cf + m1); }
                        }
                        eobrun--;
                    }
                }
            }
        }
    }
    const uint8_t *q = b.p, *e = d_ + n_;
    if (!b.marker) {
        // the bit buffer may have read ahead of the scan's end: rescan from a safe point for the next marker
        q = ecs;
        // fast forward: markers cannot precede the bytes already consumed minus the buffered ones
        size_t back = (size_t)((b.n + 7) / 8) + 1;
        q = (size_t)(b.p - ecs) > back ? b.p - back : ecs;
    }
    while (q + 1 < e && !(q[0] == 0xFF && q[1] != 0 && q[1] != 0xFF && !(q[1] >= 0xD0 && q[1] <= 0xD7))) q++;
    *next = q;
    return true;
}

bool JpegReader::device_decodable(DeviceScan &ds, bool scan_on_device)
{
    if (!have_sof_ || g_.progressive || restart_interval_ != 0) return false;
    if (pos_ + 4 > n_ || d_[pos_] != 0xFF || d_[pos_ + 1] != 0xDA) return false;
    const size_t L = rd16(d_ + pos_ + 2);
    if (L < 2 || pos_ + 2 + L > n_) return false;
    const uint8_t *seg = d_ + pos_ + 4;
    ds.ns = seg[0];
    if (ds.ns != g_.ncomp || L - 2 < (size_t)(4 + 2 * ds.ns)) return false;
    for (int k = 0; k < ds.ns; k++) {
        ds.ci[k] = -1;
        for (int c = 0; c < g_.ncomp; c++) if (g_.cid[c] == seg[1 + 2 * k]) ds.ci[k] = c;
        if (ds.ci[k] != k) return false;                       // components must appear in frame order
        ds.td[k] = seg[2 + 2 * k] >> 4; ds.ta[k] = seg[2 + 2 * k] & 15;
        if (ds.td[k] > 3 || ds.ta[k] > 3 || !dc_[ds.td[k]].present || !ac_[ds.ta[k]].present) return false;
    }
    if (mcu_blocks(ds.ns, ds.ci) > 10) return false;           // corrupt: decode_scan refuses it with the reason
    for (int c = 0; c < g_.ncomp; c++) if (!g_.qt_present[g_.tq[c]]) return false;
    ds.ecs_begin = pos_ + 2 + L;
    ds.stuffed = 0; ds.verified = !scan_on_device;
    if (scan_on_device) {
        // the last EOI of the file, searched from the end (trailing garbage after it is tolerated, like the forward walk does)
        size_t e = n_;
        while (e >= ds.ecs_begin + 2 && !(d_[e - 2] == 0xFF && d_[e - 1] == 0xD9)) e--;
        if (e < ds.ecs_begin + 2) return false;
        ds.ecs_end = e - 2;
        return ds.ecs_end > ds.ecs_begin;
    }
    // the segment ends at the first marker that is not a stuffed zero; anything but EOI right there disqualifies the file
    size_t q = ds.ecs_begin;
    {   // 16 bytes at a time: find 0xFF bytes, count the stuffed zeros behind them, stop at the first real marker
        const __m128i ff = _mm_set1_epi8((char)0xFF);
        bool found = false;
        while (!found) {
            if (q + 17 <= n_) {
                unsigned m = (unsigned)_mm_movemask_epi8(_mm_cmpeq_epi8(_mm_loadu_si128(reinterpret_cast<const __m128i *>(d_ + q)), ff));
                if (!m) { q += 16; continue; }
                size_t adv = 16;
                while (m) {
                    const int b = __builtin_ctz(m); m &= m - 1;
                    const uint8_t nx = d_[q + b + 1];
                    if (nx == 0x00) { ds.stuffed++; if (b == 15) adv = 17; continue; }
                    if (nx == 0xFF) return false;           // fill bytes: rare, host path
                    q += (size_t)b; found = true; break;
                }
                if (!found) q += adv;
            } else {
                if (q + 1 >= n_) return false;
                if (d_[q] != 0xFF) { q++; continue; }
                if (d_[q + 1] == 0x00) { ds.stuffed++; q += 2; continue; }
                if (d_[q + 1] == 0xFF) return false;
                found = true;
            }
        }
    }
    if (d_[q + 1] != 0xD9) return false;                      // RSTn, DNL or another scan: leave it to the host decoder
    ds.ecs_end = q;
    return ds.ecs_end > ds.ecs_begin;
}

bool JpegReader::decode(int16_t *coefs, std::string &err)
{
    if (!have_sof_) { err = "no frame header"; return false; }
    for (int c = 0; c < g_.ncomp; c++) if (!g_.qt_present[g_.tq[c]]) { err = "missing quantisation table"; return false; }
    int nscans = 0;
    zeroed_ = false;
    while (pos_ + 3 < n_) {
        if (d_[pos_] != 0xFF) { pos_++; continue; }
        unsigned m = d_[pos_ + 1];
        if (m == 0xFF) { pos_++; continue; }
        if (m == 0x00 || m == 0x01 || (m >= 0xD0 && m <= 0xD8)) { pos_ += 2; continue; }
        if (m == 0xD9) break;
        size_t L = rd16(d_ + pos_ + 2);
        if (L < 2 || pos_ + 2 + L > n_) { err = "truncated marker segment"; return false; }
        if (m == 0xDA) {
            const uint8_t *next = nullptr;
            if (!decode_scan(d_ + pos_ + 4, L - 2, d_ + pos_ + 2 + L, &next, coefs, err)) return false;
            nscans++;
            pos_ = (size_t)(next - d_);
            continue;
        }
        if (m == 0xC0 || m == 0xC1 || m == 0xC2) { err = "duplicate SOF"; return false; }
        if (!parse_segment(m, d_ + pos_ + 4, L - 2, err)) return false;
        pos_ += 2 + L;
    }
    if (!nscans) { err = "no image data"; return false; }
    return true;
}

// ================================================================================================================
// Writer
// ================================================================================================================
void jpeg_fill_dummy_blocks(const JpegGeom &g, int16_t *coefs)
{
    for (int c = 0; c < g.ncomp; c++) {
        const int bw = g.bw[c], hsf = g.hs[c];
        if (g.rbw[c] == bw && g.rbh[c] == g.bh[c]) continue;
        int16_t *base = coefs + g.comp_offset[c];
        for (int r = 0; r < g.bh[c]; r++) {
            int16_t *row = base + (size_t)r * bw * 64;
            if (r < g.rbh[c]) {
                for (int x = g.rbw[c]; x < bw; x++) { memset(row + (size_t)x * 64, 0, 128); row[(size_t)x * 64] = row[(size_t)(x - 1) * 64]; }
            } else {
                const int16_t *prev = row - (size_t)bw * 64;
                for (int m = 0; m < bw / hsf; m++) {
                    int16_t dc = prev[(size_t)(m * hsf + hsf - 1) * 64];
                    for (int b = 0; b < hsf; b++) { memset(row + (size_t)(m * hsf + b) * 64, 0, 128); row[(size_t)(m * hsf + b) * 64] = dc; }
                }
            }
        }
    }
}

namespace {

struct EncTab { uint8_t bits[17]; uint8_t vals[256]; int nvals; uint32_t code[256]; uint8_t size[256]; };

// jchuff.c jpeg_gen_optimal_table + jpeg_make_c_derived_tbl
void gen_optimal_table(EncTab &t, const uint32_t *freq_in)
{
    uint8_t bits[33]; int codesize[257], others[257]; long freq[257];
    memset(bits, 0, sizeof(bits)); memset(codesize, 0, sizeof(codesize));
    for (int i = 0; i < 256; i++) { freq[i] = freq_in[i]; others[i] = -1; }
    others[256] = -1; freq[256] = 1;
    for (;;) {
        int c1 = -1, c2 = -1; long v = 1000000000L;
        for (int i = 0; i <= 256; i++) if (freq[i] && freq[i] <= v) { v = freq[i]; c1 = i; }
        v = 1000000000L;
        for (int i = 0; i <= 256; i++) if (freq[i] && freq[i] <= v && i != c1) { v = freq[i]; c2 = i; }
        if (c2 < 0) break;
        freq[c1] += freq[c2]; freq[c2] = 0;
        codesize[c1]++; while (others[c1] >= 0) { c1 = others[c1]; codesize[c1]++; }
        others[c1] = c2;
        codesize[c2]++; while (others[c2] >= 0) { c2 = others[c2]; codesize[c2]++; }
    }
    for (int i = 0; i <= 256; i++) if (codesize[i]) bits[codesize[i] > 32 ? 32 : codesize[i]]++;
    for (int i = 32; i > 16; i--) while (bits[i] > 0) {
        int j = i - 2; while (bits[j] == 0) j--;
        bits[i] -= 2; bits[i - 1]++; bits[j + 1] += 2; bits[j]--;
    }
    int i = 16; while (bits[i] == 0) i--; bits[i]--;
    memset(&t, 0, sizeof(t));
    memcpy(t.bits, bits, 17);
    int p = 0;
    for (int l = 1; l <= 32; l++) for (int s = 0; s <= 255; s++) if (codesize[s] == l) t.vals[p++] = (uint8_t)s;
    t.nvals = p;
    uint32_t code = 0; int k = 0;
    for (int l = 1; l <= 16; l++) { for (int n = 0; n < t.bits[l]; n++, k++) { t.code[t.vals[k]] = code++; t.size[t.vals[k]] = (uint8_t)l; } code <<= 1; }
}

// Token: [31:30] kind (0 DC symbol, 1 AC symbol, 2 raw bits) [29] table [28:24] nbits [23:16] symbol [15:0] extra bits
inline uint32_t tok_sym(int kind, int tbl, int sym, int nbits, unsigned extra)
{
    return ((uint32_t)kind << 30) | ((uint32_t)tbl << 29) | ((uint32_t)nbits << 24) | ((uint32_t)sym << 16) | (extra & ((1u << nbits) - 1) & 0xFFFFu);
}

struct TokenBuf {
    std::vector<uint32_t> v; size_t n = 0;
    uint32_t freq[2][2][256];     // [kind][tbl][sym]
    void reset(size_t reserve) { if (v.size() < reserve) v.resize(reserve); n = 0; memset(freq, 0, sizeof(freq)); }
    inline void room(size_t k) { if (n + k > v.size()) v.resize(v.size() * 2 + k); }
    inline void sym(int kind, int tbl, int s, int nbits, unsigned extra) { v[n++] = tok_sym(kind, tbl, s, nbits, extra); freq[kind][tbl][s]++; }
    inline void raw(int nbits, unsigned bitsv) { v[n++] = (2u << 30) | ((uint32_t)nbits << 24) | (bitsv & 0xFFFFu); }
};

inline int nbits_of(unsigned v) { return v ? 32 - __builtin_clz(v) : 0; }

// 64-bit mask of the non-zero coefficients of a zigzag block (bit k = coefficient k)
inline uint64_t nonzero_mask(const int16_t *blk)
{
    const __m128i z = _mm_setzero_si128();
    uint64_t m = 0;
    for (int i = 0; i < 4; i++) {
        __m128i a = _mm_cmpeq_epi16(_mm_loadu_si128(reinterpret_cast<const __m128i *>(blk + 16 * i)), z);
        __m128i b = _mm_cmpeq_epi16(_mm_loadu_si128(reinterpret_cast<const __m128i *>(blk + 16 * i + 8)), z);
        m |= (uint64_t)(uint16_t)_mm_movemask_epi8(_mm_packs_epi16(a, b)) << (16 * i);
    }
    return ~m;
}


struct ProgState { unsigned eobrun = 0, BE = 0; int tbl = 0; uint8_t corr[1000 + 64]; };

inline void flush_eobrun(TokenBuf &t, ProgState &s)
{   // jcphuff.c emit_eobrun
    if (!s.eobrun) return;
    int nb = nbits_of(s.eobrun) - 1;
    t.room(4 + s.BE);
    t.sym(1, s.tbl, nb << 4, nb, s.eobrun);
    s.eobrun = 0;
    unsigned i = 0;
    while (i < s.BE) {   // buffered correction bits, packed 16 per raw token
        unsigned n = s.BE - i > 16 ? 16 : s.BE - i, v = 0;
        for (unsigned k = 0; k < n; k++) v = (v << 1) | s.corr[i + k];
        t.raw((int)n, v); i += n;
    }
    s.BE = 0;
}

inline void emit_corr(TokenBuf &t, const uint8_t *b, unsigned n)
{
    unsigned i = 0;
    t.room(n / 16 + 2);
    while (i < n) { unsigned m = n - i > 16 ? 16 : n - i, v = 0; for (unsigned k = 0; k < m; k++) v = (v << 1) | b[i + k]; t.raw((int)m, v); i += m; }
}

// tokenise one scan (jchuff.c encode_one_block, jcphuff.c encode_mcu_*)
void tokenize_scan(const JpegGeom &g, const int16_t *coefs, bool prog, const ScanDef &s, TokenBuf &t)
{
    int last_dc[4] = {0, 0, 0, 0};
    ProgState ps;
    const bool inter = s.ns > 1;
    const int c0 = s.ci[0];
    const int mx_n = inter ? g.mcux : g.rbw[c0], my_n = inter ? g.mcuy : g.rbh[c0];
    for (int my = 0; my < my_n; my++) for (int mx = 0; mx < mx_n; mx++) for (int i = 0; i < s.ns; i++) {
        const int c = s.ci[i], nbx = inter ? g.hs[c] : 1, nby = inter ? g.vs[c] : 1, tbl = c ? 1 : 0;
        const int16_t *cbase = coefs + g.comp_offset[c];
        for (int by = 0; by < nby; by++) for (int bx = 0; bx < nbx; bx++) {
            const int row = inter ? my * g.vs[c] + by : my, col = inter ? mx * g.hs[c] + bx : mx;
            const int16_t *blk = cbase + ((size_t)row * g.bw[c] + col) * 64;
            t.room(160);
            if (!prog) {
                int temp = blk[0] - last_dc[c], temp2 = temp; last_dc[c] = blk[0];
                if (temp < 0) { temp = -temp; temp2--; }
                int nb = nbits_of((unsigned)temp);
                t.sym(0, tbl, nb, nb, (unsigned)temp2);
                uint64_t m = nonzero_mask(blk) & ~1ull;
                int prev = 0;
                while (m) {
                    int k = __builtin_ctzll(m); m &= m - 1;
                    int r = k - prev - 1; prev = k;
                    while (r > 15) { t.sym(1, tbl, 0xF0, 0, 0); r -= 16; }
                    temp = blk[k]; temp2 = temp; if (temp < 0) { temp = -temp; temp2--; }
                    nb = nbits_of((unsigned)temp);
                    t.sym(1, tbl, (r << 4) + nb, nb, (unsigned)temp2);
                }
                if (prev != 63) t.sym(1, tbl, 0, 0, 0);
            } else if (s.Ss == 0) {
                if (s.Ah == 0) {
                    int t2 = blk[0] >> s.Al, temp = t2 - last_dc[c]; last_dc[c] = t2;
                    t2 = temp; if (temp < 0) { temp = -temp; t2--; }
                    int nb = nbits_of((unsigned)temp);
                    t.sym(0, tbl, nb, nb, (unsigned)t2);
                } else t.raw(1, (unsigned)(blk[0] >> s.Al) & 1);
            } else if (s.Ah == 0) {
                ps.tbl = tbl;
                int r = 0;
                for (int k = s.Ss; k <= s.Se; k++) {
                    int temp = blk[k], temp2;
                    if (temp == 0) { r++; continue; }
                    if (temp < 0) { temp = -temp; temp >>= s.Al; temp2 = ~temp; } else { temp >>= s.Al; temp2 = temp; }
                    if (temp == 0) { r++; continue; }
                    if (ps.eobrun) flush_eobrun(t, ps);
                    while (r > 15) { t.sym(1, tbl, 0xF0, 0, 0); r -= 16; }
                    int nb = nbits_of((unsigned)temp);
                    t.sym(1, tbl, (r << 4) + nb, nb, (unsigned)temp2);
                    r = 0;
                }
                if (r > 0) { ps.eobrun++; if (ps.eobrun == 0x7FFF) flush_eobrun(t, ps); }
            } else {
                ps.tbl = tbl;
                int absv[64], EOB = 0;
                for (int k = s.Ss; k <= s.Se; k++) { int a = blk[k]; if (a < 0) a = -a; a >>= s.Al; absv[k] = a; if (a == 1) EOB = k; }
                int r = 0; unsigned BR = 0; uint8_t *BRbuf = ps.corr + ps.BE;
                for (int k = s.Ss; k <= s.Se; k++) {
                    int a = absv[k];
                    if (a == 0) { r++; continue; }
                    while (r > 15 && k <= EOB) {
                        flush_eobrun(t, ps);
                        t.room(8); t.sym(1, tbl, 0xF0, 0, 0); r -= 16;
                        emit_corr(t, BRbuf, BR); BRbuf = ps.corr; BR = 0;
                    }
                    if (a > 1) { BRbuf[BR++] = (uint8_t)(a & 1); continue; }
                    flush_eobrun(t, ps);
                    t.room(8); t.sym(1, tbl, (r << 4) + 1, 1, blk[k] < 0 ? 0u : 1u);
                    emit_corr(t, BRbuf, BR); BRbuf = ps.corr; BR = 0;
                    r = 0;
                }
                if (r > 0 || BR > 0) {
                    ps.eobrun++; ps.BE += BR;
                    if (ps.eobrun == 0x7FFF || ps.BE > (1000 - 64 + 1)) flush_eobrun(t, ps);
                }
            }
        }
    }
    if (prog && s.Ss > 0) flush_eobrun(t, ps);
}

struct ByteSink {
    std::vector<uint8_t> &o;
    explicit ByteSink(std::vector<uint8_t> &out) : o(out) {}
    void u8(unsigned v) { o.push_back((uint8_t)v); }
    void u16(unsigned v) { o.push_back((uint8_t)(v >> 8)); o.push_back((uint8_t)v); }
    void raw(const void *p, size_t n) { const uint8_t *s = (const uint8_t *)p; o.insert(o.end(), s, s + n); }
};

void write_dht(ByteSink &w, int tc, int th, const EncTab &t)
{
    w.u16(0xFFC4); w.u16(2 + 1 + 16 + t.nvals); w.u8((tc << 4) | th);
    for (int l = 1; l <= 16; l++) w.u8(t.bits[l]);
    w.raw(t.vals, t.nvals);
}

// emit the token stream with the given tables: MSB-first bit packing, 0xFF -> 0xFF00 stuffing, pad with ones
void emit_tokens(std::vector<uint8_t> &out, const TokenBuf &t, const EncTab tabs[2][2])
{
    size_t pos = out.size();
    out.resize(pos + t.n * 8 + 16);
    uint8_t *p = out.data() + pos;
    uint64_t acc = 0; int n = 0;
    for (size_t i = 0; i < t.n; i++) {
        uint32_t tk = t.v[i];
        int kind = tk >> 30, nb = (tk >> 24) & 31;
        uint32_t code; int size;
        if (kind == 2) { code = tk & 0xFFFF; size = nb; }
        else {
            const EncTab &tab = tabs[kind][(tk >> 29) & 1];
            int s = (tk >> 16) & 0xFF;
            code = (tab.code[s] << nb) | (tk & 0xFFFF & ((1u << nb) - 1)); size = tab.size[s] + nb;
        }
        acc = (acc << size) | code; n += size;
        if (n >= 32) {
            uint32_t w = (uint32_t)(acc >> (n - 32)); n -= 32;
            uint32_t v = ~w;
            if (!((v - 0x01010101u) & ~v & 0x80808080u)) { uint32_t be = __builtin_bswap32(w); memcpy(p, &be, 4); p += 4; }
            else for (int k = 3; k >= 0; k--) { uint8_t c = (uint8_t)(w >> (8 * k)); *p++ = c; if (c == 0xFF) *p++ = 0; }
        }
    }
    while (n >= 8) { uint8_t c = (uint8_t)(acc >> (n - 8)); n -= 8; *p++ = c; if (c == 0xFF) *p++ = 0; }
    if (n > 0) { uint8_t c = (uint8_t)(((acc << (8 - n)) | ((1u << (8 - n)) - 1)) & 0xFF); *p++ = c; if (c == 0xFF) *p++ = 0; }
    out.resize((size_t)(p - out.data()));
}

} // namespace

int jpeg_scan_script(const JpegGeom &g, bool progressive, ScanDef sc[16])
{
    int ns = 0;
    if (!progressive) { sc[0].ns = g.ncomp; for (int c = 0; c < 3; c++) sc[0].ci[c] = c < g.ncomp ? c : 0; sc[0].Ss = 0; sc[0].Se = 63; sc[0].Ah = sc[0].Al = 0; return 1; }
    sc[ns].ns = g.ncomp; for (int c = 0; c < 3; c++) sc[ns].ci[c] = c < g.ncomp ? c : 0; sc[ns].Ss = 0; sc[ns].Se = 0; sc[ns].Ah = 0; sc[ns].Al = 0; ns++;
    sc[ns++] = ScanDef{1, {0, 0, 0}, 1, 2, 0, 1};
    sc[ns++] = ScanDef{1, {0, 0, 0}, 3, 63, 0, 1};
    for (int c = 1; c < g.ncomp; c++) sc[ns++] = ScanDef{1, {c, 0, 0}, 1, 63, 0, 1};
    for (int c = 0; c < g.ncomp; c++) sc[ns++] = ScanDef{1, {c, 0, 0}, 1, 63, 1, 0};
    return ns;
}

void jpeg_scan_tables_needed(const JpegGeom &, bool progressive, const ScanDef &s, bool need[2][2])
{   // jcmarker.c write_scan_header: progressive scans define the DC table (Ss == 0, Ah == 0) or the AC table (Ss > 0)
    need[0][0] = need[0][1] = need[1][0] = need[1][1] = false;
    if (progressive && s.Ss == 0 && s.Ah != 0) return;     // DC refinement: no table
    for (int i = 0; i < s.ns; i++) {
        int t = s.ci[i] ? 1 : 0;
        if (!progressive || s.Ss == 0) need[0][t] = true;
        if (!progressive || s.Ss > 0) need[1][t] = true;
    }
}

static void write_file_header(ByteSink &w, const JpegGeom &g, const JpegWriteOptions &opt, const JpegMeta *meta)
{
    w.u16(0xFFD8);
    {   // jcmarker.c emit_jfif_app0
        uint8_t body[9] = {1, 1, 0, 0, 1, 0, 1, 0, 0};
        if (opt.copy_jfif && meta && meta->jfif) memcpy(body, meta->jfif_body, 9);
        w.u16(0xFFE0); w.u16(16); w.raw("JFIF", 5); w.raw(body, 9);
    }
    if (meta) {
        if (opt.keep_metadata && !meta->app_markers.empty()) w.raw(meta->app_markers.data(), meta->app_markers.size());
        if ((opt.keep_metadata || opt.preserve_icc) && !meta->icc_markers.empty()) w.raw(meta->icc_markers.data(), meta->icc_markers.size());
    }
    {   // all tables in one DQT segment (mozjpeg emit_multi_dqt), 16-bit precision only where needed
        bool used[4] = {false, false, false, false}; int prec[4] = {0, 0, 0, 0}, seglen = 2;
        for (int c = 0; c < g.ncomp; c++) used[g.tq[c]] = true;
        for (int t = 0; t < 4; t++) if (used[t]) { for (int i = 0; i < 64; i++) if (g.qt[t][i] > 255) prec[t] = 1; seglen += 1 + (prec[t] ? 128 : 64); }
        w.u16(0xFFDB); w.u16(seglen);
        for (int t = 0; t < 4; t++) if (used[t]) {
            w.u8((prec[t] << 4) | t);
            for (int z = 0; z < 64; z++) { if (prec[t]) w.u8(g.qt[t][z] >> 8); w.u8(g.qt[t][z] & 0xFF); }
        }
    }
    w.u16(opt.progressive ? 0xFFC2 : 0xFFC0); w.u16(8 + 3 * g.ncomp); w.u8(8);
    w.u16(g.height); w.u16(g.width); w.u8(g.ncomp);
    for (int c = 0; c < g.ncomp; c++) { w.u8(g.cid[c]); w.u8((g.hs[c] << 4) | g.vs[c]); w.u8(g.tq[c]); }
}

static void write_sos(ByteSink &w, const JpegGeom &g, bool progressive, const ScanDef &s)
{   // jcmarker.c emit_sos
    w.u16(0xFFDA); w.u16(6 + 2 * s.ns); w.u8(s.ns);
    for (int i = 0; i < s.ns; i++) {
        int c = s.ci[i], td = c ? 1 : 0, ta = c ? 1 : 0;
        if (progressive) { if (s.Ss == 0) { ta = 0; if (s.Ah != 0) td = 0; } else td = 0; }
        w.u8(g.cid[c]); w.u8((td << 4) | ta);
    }
    w.u8(s.Ss); w.u8(s.Se); w.u8((s.Ah << 4) | s.Al);
}

bool jpeg_write(const JpegGeom &g, const int16_t *coefs, const JpegWriteOptions &opt, const JpegMeta *meta,
                std::vector<uint8_t> &out, std::string &err)
{
    if (g.ncomp != 1 && g.ncomp != 3) { err = "unsupported component count"; return false; }
    out.clear();
    out.reserve((size_t)g.total_coefs / 6 + 4096);
    ByteSink w(out);
    write_file_header(w, g, opt, meta);
    ScanDef sc[16];
    const int ns = jpeg_scan_script(g, opt.progressive, sc);
    static thread_local TokenBuf tb;
    int64_t nblocks = 0; for (int c = 0; c < g.ncomp; c++) nblocks += g.blocks(c);
    for (int si = 0; si < ns; si++) {
        const ScanDef &s = sc[si];
        tb.reset((size_t)nblocks * 12 + 4096);
        tokenize_scan(g, coefs, opt.progressive, s, tb);
        EncTab tabs[2][2];
        bool need[2][2];
        jpeg_scan_tables_needed(g, opt.progressive, s, need);
        for (int t = 0; t < 2; t++) for (int kind = 0; kind < 2; kind++) if (need[kind][t]) {
            gen_optimal_table(tabs[kind][t], tb.freq[kind][t]);
            write_dht(w, kind, t, tabs[kind][t]);
        }
        write_sos(w, g, opt.progressive, s);
        emit_tokens(out, tb, tabs);
    }
    w.u16(0xFFD9);
    return true;
}

bool jpeg_assemble_malloc(const JpegGeom &g, const JpegWriteOptions &opt, const JpegMeta *meta, const EncodedScan *scans, int nscans,
                          uint8_t **out, size_t *out_len, std::string &err)
{   // same bytes as jpeg_assemble, written once into an exactly-sized malloc'd buffer (the C-ABI's ownership convention)
    if (g.ncomp != 1 && g.ncomp != 3) { err = "unsupported component count"; return false; }
    std::vector<uint8_t> head; head.reserve(4096 + (meta ? meta->app_markers.size() + meta->icc_markers.size() : 0));
    { ByteSink w(head); write_file_header(w, g, opt, meta); }
    std::vector<std::vector<uint8_t>> pre((size_t)nscans);
    size_t total = head.size() + 2;
    for (int si = 0; si < nscans; si++) {
        const EncodedScan &e = scans[si];
        pre[si].reserve(1400);
        ByteSink w(pre[si]);
        for (int t = 0; t < 2; t++) for (int kind = 0; kind < 2; kind++) if (e.has_tab[kind][t]) {
            w.u16(0xFFC4); w.u16(2 + 1 + 16 + e.nvals[kind][t]); w.u8((kind << 4) | t);
            for (int l = 1; l <= 16; l++) w.u8(e.bits[kind][t][l]);
            w.raw(e.vals[kind][t], e.nvals[kind][t]);
        }
        write_sos(w, g, opt.progressive, e.def);
        total += pre[si].size() + e.len;
    }
    uint8_t *p = (uint8_t *)malloc(total);
    if (!p) { err = "out of memory"; return false; }
    uint8_t *q = p;
    memcpy(q, head.data(), head.size()); q += head.size();
    for (int si = 0; si < nscans; si++) { memcpy(q, pre[si].data(), pre[si].size()); q += pre[si].size(); stream_copy(q, scans[si].data, scans[si].len); q += scans[si].len; }
    *q++ = 0xFF; *q++ = 0xD9;
    *out = p; *out_len = total;
    return true;
}

size_t jpeg_assembled_size(const JpegGeom &g, const JpegWriteOptions &opt, const JpegMeta *meta, const EncodedScan *scans, int nscans)
{   // the length jpeg_assemble would produce, without touching the scans' bytes (compress_to_size only needs sizes for most tries)
    std::vector<uint8_t> head; head.reserve(4096 + (meta ? meta->app_markers.size() + meta->icc_markers.size() : 0));
    { ByteSink w(head); write_file_header(w, g, opt, meta); }
    size_t total = head.size() + 2;
    std::vector<uint8_t> pre;
    for (int si = 0; si < nscans; si++) {
        const EncodedScan &e = scans[si];
        for (int t = 0; t < 2; t++) for (int kind = 0; kind < 2; kind++) if (e.has_tab[kind][t]) total += 2 + 2 + 1 + 16 + (size_t)e.nvals[kind][t];
        pre.clear(); { ByteSink w(pre); write_sos(w, g, opt.progressive, e.def); }
        total += pre.size() + e.len;
    }
    return total;
}

bool jpeg_assemble(const JpegGeom &g, const JpegWriteOptions &opt, const JpegMeta *meta, const EncodedScan *scans, int nscans,
                   std::vector<uint8_t> &out, std::string &err)
{
    if (g.ncomp != 1 && g.ncomp != 3) { err = "unsupported component count"; return false; }
    out.clear();
    size_t total = 4096;
    for (int i = 0; i < nscans; i++) total += scans[i].len + 1200;
    if (meta) total += meta->app_markers.size() + meta->icc_markers.size();
    out.reserve(total);
    ByteSink w(out);
    write_file_header(w, g, opt, meta);
    for (int si = 0; si < nscans; si++) {
        const EncodedScan &e = scans[si];
        for (int t = 0; t < 2; t++) for (int kind = 0; kind < 2; kind++) if (e.has_tab[kind][t]) {
            w.u16(0xFFC4); w.u16(2 + 1 + 16 + e.nvals[kind][t]); w.u8((kind << 4) | t);
            for (int l = 1; l <= 16; l++) w.u8(e.bits[kind][t][l]);
            w.raw(e.vals[kind][t], e.nvals[kind][t]);
        }
        write_sos(w, g, opt.progressive, e.def);
        w.raw(e.data, e.len);
    }
    w.u16(0xFFD9);
    return true;
}

} // namespace b200
