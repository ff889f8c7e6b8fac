// vp8l_decode.cpp -- host decoder of the WebP lossless bitstream ("VP8L"): lossless WebP inputs and the alpha plane (ALPH chunk) of
// lossy ones.  libcaesium's webp::compress decodes its input before it re-encodes (caesium::compress_in_memory on a .webp,
// caesium-clt's src/compressor.rs:305); this is that decode for the files the VP8 key-frame decoder (vp8_decode.cpp) does not
// cover -- format plumbing in front of the device encoder, like the PNG inflate.  Written from the format specification (LSB-first
// bit reader, canonical prefix codes, LZ77 with the 120 neighbourhood distance codes, colour cache, meta prefix image, the four
// transforms); the tests pin it against libwebp (Pillow) on lossless files and alpha planes of every flavour libwebp writes.
#include "vp8l_decode.h"
#include "vp8l_enc_core.h"
#include <cstring>

namespace b200 {
namespace {

struct BitReader {
    const uint8_t *p, *end; uint64_t acc = 0; int have = 0; bool eos = false;     // past the end zeros are served and eos is raised
    BitReader(const uint8_t *d, size_t len) : p(d), end(d + len) {}
    inline void refill() { while (have <= 56 && p < end) { acc |= (uint64_t)*p++ << have; have += 8; } }
    inline uint32_t peek(int nb) { refill(); return (uint32_t)(acc & ((1ull << nb) - 1ull)); }
    inline void skip(int nb) { if (nb > have) { eos = true; acc = 0; have = 0; return; } acc >>= nb; have -= nb; }
    inline uint32_t bits(int nb) { if (!nb) return 0; const uint32_t v = peek(nb); skip(nb); return v; }
};

constexpr int kMaxLen = 15, kFast = 9;

// canonical prefix code, decoded LSB-first: a 2^kFast table for the short codes, the canonical walk for the rest
struct Code {
    std::vector<uint16_t> fast;         // (len << 12 is too small for 280 + 2048 symbols) -> two arrays
    std::vector<uint8_t> fast_len;
    uint16_t count[kMaxLen + 1];        // codes per length
    uint32_t first[kMaxLen + 2];        // first canonical code of each length
    uint16_t offs[kMaxLen + 2];         // index into sorted[] of each length's first symbol
    std::vector<uint16_t> sorted;       // symbols by (length, value)
    int single = -1;                    // >= 0: the code has one symbol and takes no bits
    bool build(const uint8_t *len, int n)
    {
        memset(count, 0, sizeof(count));
        int used = 0, last = -1;
        for (int i = 0; i < n; i++) { if (len[i] > kMaxLen) return false; if (len[i]) { count[len[i]]++; used++; last = i; } }
        if (used == 0) return false;
        if (used == 1) { single = last; return true; }
        single = -1;
        // the code must be complete
        uint32_t code = 0; int left = 1;
        for (int l = 1; l <= kMaxLen; l++) { left = left * 2 - count[l]; if (left < 0) return false; }
        if (left != 0) return false;
        offs[1] = 0; first[1] = 0;
        for (int l = 1; l <= kMaxLen; l++) { offs[l + 1] = (uint16_t)(offs[l] + count[l]); code = (code + count[l]) << 1; first[l + 1] = code; }
        sorted.assign(used, 0);
        { uint16_t o[kMaxLen + 2]; memcpy(o, offs, sizeof(o)); for (int i = 0; i < n; i++) if (len[i]) sorted[o[len[i]]++] = (uint16_t)i; }
        fast.assign(1u << kFast, 0); fast_len.assign(1u << kFast, 0);
        for (int l = 1; l <= kFast; l++)
            for (int k = 0; k < count[l]; k++) {
                const uint32_t c = first[l] + (uint32_t)k;      // MSB-first canonical code of length l
                uint32_t r = 0; for (int b = 0; b < l; b++) r |= ((c >> (l - 1 - b)) & 1u) << b;
                for (uint32_t x = r; x < (1u << kFast); x += 1u << l) { fast[x] = sorted[offs[l] + k]; fast_len[x] = (uint8_t)l; }
            }
        return true;
    }
    inline int read(BitReader &br) const
    {
        if (single >= 0) return single;
        const uint32_t w = br.peek(kMaxLen);
        const uint32_t f = w & ((1u << kFast) - 1u);
        if (fast_len[f]) { br.skip(fast_len[f]); return fast[f]; }
        uint32_t code = 0;
        for (int l = 1; l <= kMaxLen; l++) {
            code = (code << 1) | ((w >> (l - 1)) & 1u);
            if (code - first[l] < count[l]) { br.skip(l); return sorted[offs[l] + (code - first[l])]; }
        }
        br.eos = true; return 0;
    }
};

struct Group { Code c[5]; };

const uint8_t kCodeToPlane[120] = {
    0x18, 0x07, 0x17, 0x19, 0x28, 0x06, 0x27, 0x29, 0x16, 0x1a, 0x26, 0x2a, 0x38, 0x05, 0x37, 0x39, 0x15, 0x1b, 0x36, 0x3a,
    0x25, 0x2b, 0x48, 0x04, 0x47, 0x49, 0x14, 0x1c, 0x35, 0x3b, 0x46, 0x4a, 0x24, 0x2c, 0x58, 0x45, 0x4b, 0x34, 0x3c, 0x03,
    0x57, 0x59, 0x13, 0x1d, 0x56, 0x5a, 0x23, 0x2d, 0x44, 0x4c, 0x55, 0x5b, 0x33, 0x3d, 0x68, 0x02, 0x67, 0x69, 0x12, 0x1e,
    0x66, 0x6a, 0x22, 0x2e, 0x54, 0x5c, 0x43, 0x4d, 0x65, 0x6b, 0x32, 0x3e, 0x78, 0x01, 0x77, 0x79, 0x53, 0x5d, 0x11, 0x1f,
    0x64, 0x6c, 0x42, 0x4e, 0x76, 0x7a, 0x21, 0x2f, 0x75, 0x7b, 0x31, 0x3f, 0x63, 0x6d, 0x52, 0x5e, 0x00, 0x74, 0x7c, 0x41,
    0x4f, 0x10, 0x20, 0x62, 0x6e, 0x30, 0x73, 0x7d, 0x51, 0x5f, 0x40, 0x72, 0x7e, 0x61, 0x6f, 0x50, 0x71, 0x7f, 0x60, 0x70};

struct Decoder {
    BitReader br;
    std::string &err;
    Decoder(const uint8_t *d, size_t n, std::string &e) : br(d, n), err(e) {}
    bool fail(const char *m) { if (err.empty()) err = m; return false; }

    bool read_code(int alphabet, Code &c)
    {
        std::vector<uint8_t> len(alphabet, 0);
        if (br.bits(1)) {                                   // simple code: one or two symbols
            const int nsym = (int)br.bits(1) + 1;
            const int s0 = (int)br.bits(br.bits(1) ? 8 : 1);
            if (s0 >= alphabet) return fail("VP8L: simple code symbol out of range");
            len[s0] = 1;
            if (nsym == 2) { const int s1 = (int)br.bits(8); if (s1 >= alphabet) return fail("VP8L: simple code symbol out of range"); len[s1] = 1; }
        } else {
            static const uint8_t order[19] = {17, 18, 0, 1, 2, 3, 4, 5, 16, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15};
            uint8_t cl[19] = {0};
            const int ncl = (int)br.bits(4) + 4;
            for (int i = 0; i < ncl; i++) cl[order[i]] = (uint8_t)br.bits(3);
            Code clc;
            if (!clc.build(cl, 19)) return fail("VP8L: bad code-length code");
            int max_symbol = alphabet;
            if (br.bits(1)) { const int nb = 2 + 2 * (int)br.bits(3); max_symbol = 2 + (int)br.bits(nb); if (max_symbol > alphabet) return fail("VP8L: max_symbol out of range"); }
            int sym = 0, prev = 8;
            while (sym < alphabet) {
                if (max_symbol-- == 0) break;
                const int l = clc.read(br);
                if (br.eos) return fail("VP8L: truncated prefix code");
                if (l < 16) { len[sym++] = (uint8_t)l; if (l) prev = l; }
                else {
                    static const int xb[3] = {2, 3, 7}, ro[3] = {3, 3, 11};
                    const int rep = (int)br.bits(xb[l - 16]) + ro[l - 16];
                    if (sym + rep > alphabet) return fail("VP8L: code-length run past the alphabet");
                    const uint8_t v = l == 16 ? (uint8_t)prev : 0;
                    for (int k = 0; k < rep; k++) len[sym++] = v;
                }
            }
        }
        if (br.eos) return fail("VP8L: truncated prefix code");
        if (!c.build(len.data(), alphabet)) return fail("VP8L: incomplete prefix code");
        return true;
    }

    inline uint32_t prefix_value(int sym)
    {
        if (sym < 4) return (uint32_t)sym + 1u;
        const int xb = (sym - 2) >> 1;
        const uint32_t off = (2u + ((uint32_t)sym & 1u)) << xb;
        return off + br.bits(xb) + 1u;
    }

    // one entropy-coded image (xs x ys ARGB pixels); level0: the main image (may carry a meta prefix image)
    bool image(int xs, int ys, bool level0, std::vector<uint32_t> &pix)
    {
        int cache_bits = 0;
        if (br.bits(1)) { cache_bits = (int)br.bits(4); if (cache_bits < 1 || cache_bits > 11) return fail("VP8L: bad colour-cache size"); }
        std::vector<uint32_t> meta; int meta_bits = 0, meta_w = 0, ngroups = 1;
        if (level0 && br.bits(1)) {
            meta_bits = (int)br.bits(3) + 2;
            meta_w = (xs + (1 << meta_bits) - 1) >> meta_bits;
            const int meta_h = (ys + (1 << meta_bits) - 1) >> meta_bits;
            if (!image(meta_w, meta_h, false, meta)) return false;
            for (uint32_t &m : meta) { m = (m >> 8) & 0xFFFFu; if ((int)m + 1 > ngroups) ngroups = (int)m + 1; }
        }
        if (br.eos) return fail("VP8L: truncated image header");
        std::vector<Group> groups(ngroups);
        const int alpha_sizes[5] = {256 + 24 + (cache_bits ? 1 << cache_bits : 0), 256, 256, 256, 40};
        for (Group &g : groups) for (int k = 0; k < 5; k++) if (!read_code(alpha_sizes[k], g.c[k])) return false;
        std::vector<uint32_t> cache(cache_bits ? (size_t)1 << cache_bits : 0, 0);
        const size_t n = (size_t)xs * ys;
        pix.assign(n, 0);
        size_t pos = 0, cached = 0;         // pixels [cached, pos) still have to enter the colour cache
        int x = 0, y = 0;
        const Group *g = &groups[0];
        auto flush_cache = [&]() { if (cache_bits) while (cached < pos) { const uint32_t v = pix[cached++]; cache[(0x1e35a7bdu * v) >> (32 - cache_bits)] = v; } };
        while (pos < n) {
            if (meta_bits) g = &groups[meta[(size_t)(y >> meta_bits) * meta_w + (x >> meta_bits)]];
            const int s = g->c[0].read(br);
            if (s < 256) {
                const uint32_t r = (uint32_t)g->c[1].read(br), b = (uint32_t)g->c[2].read(br), a = (uint32_t)g->c[3].read(br);
                pix[pos++] = (a << 24) | (r << 16) | ((uint32_t)s << 8) | b;
                if (++x >= xs) { x = 0; y++; }
            } else if (s < 256 + 24) {
                const uint32_t len = prefix_value(s - 256);
                const uint32_t dcode = prefix_value(g->c[4].read(br));
                uint32_t dist;
                if (dcode > 120) dist = dcode - 120;
                else { const int c = kCodeToPlane[dcode - 1]; const long long d = (long long)(c >> 4) * xs + (8 - (c & 15)); dist = d >= 1 ? (uint32_t)d : 1u; }
                if (br.eos) return fail("VP8L: truncated pixel data");
                if (dist > pos || len > n - pos) return fail("VP8L: copy outside the image");
                for (uint32_t k = 0; k < len; k++, pos++) pix[pos] = pix[pos - dist];
                x += (int)len; while (x >= xs) { x -= xs; y++; }
            } else {
                const int key = s - (256 + 24);
                if (!cache_bits || key >= (1 << cache_bits)) return fail("VP8L: colour-cache index out of range");
                flush_cache();
                pix[pos++] = cache[key];
                if (++x >= xs) { x = 0; y++; }
            }
            if (br.eos) return fail("VP8L: truncated pixel data");
            if (cache_bits && pos - cached >= 4096) flush_cache();
        }
        return true;
    }
};

struct Transform { int type, bits, xs; std::vector<uint32_t> data; };

} // namespace

bool vp8l_decode_stream(const uint8_t *data, size_t len, int width, int height, std::vector<uint32_t> &argb, std::string &err)
{
    if (width < 1 || height < 1 || width > 16384 || height > 16384) { err = "VP8L: bad dimensions"; return false; }
    Decoder d(data, len, err);
    std::vector<Transform> tf;
    int xs = width;
    unsigned seen = 0;
    while (d.br.bits(1)) {
        Transform t; t.type = (int)d.br.bits(2); t.bits = 0; t.xs = xs;
        if (seen & (1u << t.type)) { err = "VP8L: a transform is used twice"; return false; }
        seen |= 1u << t.type;
        if (t.type == 0 || t.type == 1) {
            t.bits = (int)d.br.bits(3) + 2;
            const int bw = (xs + (1 << t.bits) - 1) >> t.bits, bh = (height + (1 << t.bits) - 1) >> t.bits;
            if (!d.image(bw, bh, false, t.data)) return false;
        } else if (t.type == 3) {
            const int ncol = (int)d.br.bits(8) + 1;
            if (!d.image(ncol, 1, false, t.data)) return false;
            for (int i = 1; i < ncol; i++) t.data[i] = vp8l_add_px(t.data[i], t.data[i - 1]);
            t.bits = ncol <= 2 ? 3 : ncol <= 4 ? 2 : ncol <= 16 ? 1 : 0;
            t.data.resize(256, 0u);                                   // indices past the table read transparent black
            xs = (xs + (1 << t.bits) - 1) >> t.bits;
        }
        if (d.br.eos) { err = "VP8L: truncated transform"; return false; }
        tf.push_back(std::move(t));
    }
    std::vector<uint32_t> pix;
    if (!d.image(xs, height, true, pix)) return false;
    // ---- inverse transforms, last one first
    for (size_t k = tf.size(); k-- > 0;) {
        const Transform &t = tf[k];
        const int w = t.xs;
        if (t.type == 2) { for (uint32_t &p : pix) { const uint32_t g = (p >> 8) & 0xFFu; p = (p & 0xFF00FF00u) | ((((p & 0x00FF00FFu) + ((g << 16) | g))) & 0x00FF00FFu); } }
        else if (t.type == 1) {
            const int bw = (w + (1 << t.bits) - 1) >> t.bits;
            for (int y = 0; y < height; y++) for (int x = 0; x < w; x++) {
                const uint32_t m = t.data[(size_t)(y >> t.bits) * bw + (x >> t.bits)];
                uint32_t &p = pix[(size_t)y * w + x];
                const int8_t g2r = (int8_t)(m & 0xFF), g2b = (int8_t)((m >> 8) & 0xFF), r2b = (int8_t)((m >> 16) & 0xFF);
                const int8_t green = (int8_t)((p >> 8) & 0xFF);
                int red = (int)((p >> 16) & 0xFF), blue = (int)(p & 0xFF);
                red = (red + (((int)g2r * green) >> 5)) & 0xFF;
                blue = (blue + (((int)g2b * green) >> 5) + (((int)r2b * (int8_t)red) >> 5)) & 0xFF;
                p = (p & 0xFF00FF00u) | ((uint32_t)red << 16) | (uint32_t)blue;
            }
        } else if (t.type == 0) {
            const int bw = (w + (1 << t.bits) - 1) >> t.bits;
            pix[0] = vp8l_add_px(pix[0], 0xFF000000u);
            for (int x = 1; x < w; x++) pix[x] = vp8l_add_px(pix[x], pix[x - 1]);
            for (int y = 1; y < height; y++) {
                uint32_t *row = pix.data() + (size_t)y * w;
                row[0] = vp8l_add_px(row[0], row[-w]);
                for (int x = 1; x < w; x++) {
                    const int mode = (int)((t.data[(size_t)(y >> t.bits) * bw + (x >> t.bits)] >> 8) & 0xF);
                    row[x] = vp8l_add_px(row[x], vp8l_predict(mode, row[x - 1], row[x - w], row[x - w + 1], row[x - w - 1]));
                }
            }
        } else {
            // colour indexing: w = the width before the transform packed the indices; pix holds ceil(w / 2^bits) words per row
            const int pw = (w + (1 << t.bits) - 1) >> t.bits, bpp = 8 >> t.bits, per = 1 << t.bits;
            std::vector<uint32_t> out((size_t)w * height);
            for (int y = 0; y < height; y++) for (int x = 0; x < w; x++) {
                const uint32_t packed = (pix[(size_t)y * pw + (x >> t.bits)] >> 8) & 0xFFu;
                const uint32_t idx = t.bits ? (packed >> ((x & (per - 1)) * bpp)) & ((1u << bpp) - 1u) : packed;
                out[(size_t)y * w + x] = t.data[idx];
            }
            pix.swap(out);
        }
    }
    if (pix.size() != (size_t)width * height) { err = "VP8L: size mismatch after the transforms"; return false; }
    argb.swap(pix);
    return true;
}

bool vp8l_decode_file_chunk(const uint8_t *chunk, size_t len, int &width, int &height, bool &has_alpha, std::vector<uint32_t> &argb, std::string &err)
{
    if (len < 5 || chunk[0] != 0x2f) { err = "VP8L: bad signature"; return false; }
    const uint32_t h = (uint32_t)chunk[1] | ((uint32_t)chunk[2] << 8) | ((uint32_t)chunk[3] << 16) | ((uint32_t)chunk[4] << 24);
    width = (int)(h & 0x3FFF) + 1; height = (int)((h >> 14) & 0x3FFF) + 1; has_alpha = (h >> 28) & 1;
    if ((h >> 29) != 0) { err = "VP8L: unknown version"; return false; }
    return vp8l_decode_stream(chunk + 5, len - 5, width, height, argb, err);
}

bool webp_alpha_decode(const uint8_t *alph, size_t len, int width, int height, std::vector<uint8_t> &alpha, std::string &err)
{
    if (len < 1) { err = "ALPH: empty chunk"; return false; }
    const int method = alph[0] & 3, filter = (alph[0] >> 2) & 3;
    const size_t n = (size_t)width * height;
    alpha.assign(n, 0);
    if (method == 0) { if (len - 1 < n) { err = "ALPH: truncated raw plane"; return false; } memcpy(alpha.data(), alph + 1, n); }
    else if (method == 1) {
        std::vector<uint32_t> argb;
        if (!vp8l_decode_stream(alph + 1, len - 1, width, height, argb, err)) return false;
        for (size_t i = 0; i < n; i++) alpha[i] = (uint8_t)(argb[i] >> 8);
    } else { err = "ALPH: unknown compression method"; return false; }
    if (filter) {
        for (int y = 0; y < height; y++) {
            uint8_t *row = alpha.data() + (size_t)y * width;
            const uint8_t *prev = y ? row - width : nullptr;
            if (filter == 1 || !prev) { uint8_t pred = prev ? prev[0] : 0; for (int x = 0; x < width; x++) { row[x] = (uint8_t)(pred + row[x]); pred = row[x]; } }
            else if (filter == 2) { for (int x = 0; x < width; x++) row[x] = (uint8_t)(prev[x] + row[x]); }
            else {
                uint8_t top = prev[0], tl = top, left = top;
                for (int x = 0; x < width; x++) { top = prev[x]; left = (uint8_t)(row[x] + vp8l_clip255((int)left + top - tl)); tl = top; row[x] = left; }
            }
        }
    }
    return true;
}

} // namespace b200
