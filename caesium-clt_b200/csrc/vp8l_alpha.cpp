// vp8l_alpha.cpp -- see vp8l_alpha.h.  WebP lossless bitstream (the "VP8L" specification: LSB-first bits, canonical prefix codes
// of at most 15 bits, five codes per group: green + length prefixes, red, blue, alpha, distance prefixes), restricted to what an
// alpha plane needs: no transforms, no colour cache, no meta prefix image; red / blue / alpha are single-symbol codes (zero bits).
// The prefix-code writer here (vp8l_writer.h) also serves the lossless WebP encoder (vp8l_encode.cpp).
#include "vp8l_alpha.h"
#include "vp8l_writer.h"
#include <cstring>

namespace b200 {

void vp8l_make_code(const std::vector<uint32_t> &freq, PrefixCode &pc, Vp8lHuffScratch &S)
{
    const int n = (int)freq.size();
    if (n < 1 || n > VP8L_NGREEN) return;
    pc.len.assign(n, 0); pc.code.assign(n, 0); pc.used = 0;
    for (int i = 0; i < n; i++) pc.used += freq[i] != 0;
    dfl::huff_lengths(freq.data(), n, 15, pc.len.data(), S);
    dfl::canon_codes(pc.len.data(), n, pc.code.data());
}

// one prefix code in the bitstream (section 6.2.1 / 6.2.2 of the specification)
void vp8l_write_code(BitsLsb &bw, const PrefixCode &pc, Vp8lHuffScratch &S)
{
    const int n = (int)pc.len.size();
    int s0 = -1, s1 = -1;
    for (int i = 0; i < n; i++) if (pc.len[i]) { if (s0 < 0) s0 = i; else if (s1 < 0) s1 = i; }
    if (pc.used == 0) { bw.put(1, 1); bw.put(0, 1); bw.put(0, 1); bw.put(0, 1); return; }                // simple code, one symbol: 0
    if (pc.used <= 2 && s0 < 256 && (pc.used == 1 || s1 < 256)) {
        bw.put(1, 1); bw.put((uint32_t)pc.used - 1u, 1);
        if (s0 < 2) { bw.put(0, 1); bw.put((uint32_t)s0, 1); } else { bw.put(1, 1); bw.put((uint32_t)s0, 8); }
        if (pc.used == 2) bw.put((uint32_t)s1, 8);
        return;
    }
    // normal code: the lengths, run-length coded with zero runs (17: 3..10, 18: 11..138), themselves prefix coded (limit 7)
    struct Tk { uint8_t sym, extra; };
    std::vector<Tk> tk;
    for (int i = 0; i < n;) {
        if (pc.len[i]) { tk.push_back({pc.len[i], 0}); i++; continue; }
        int run = 1; while (i + run < n && !pc.len[i + run]) run++;
        i += run;
        while (run >= 11) { const int r = run > 138 ? 138 : run; tk.push_back({18, (uint8_t)(r - 11)}); run -= r; }
        if (run >= 3) { tk.push_back({17, (uint8_t)(run - 3)}); run = 0; }
        while (run-- > 0) tk.push_back({0, 0});
    }
    std::vector<uint32_t> cf(19, 0);
    for (const Tk &t : tk) cf[t.sym]++;
    PrefixCode cl; cl.len.assign(19, 0); cl.code.assign(19, 0);
    for (int i = 0; i < 19; i++) cl.used += cf[i] != 0;
    dfl::huff_lengths(cf.data(), 19, 7, cl.len.data(), S);
    dfl::canon_codes(cl.len.data(), 19, cl.code.data());
    static const uint8_t order[19] = {17, 18, 0, 1, 2, 3, 4, 5, 16, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15};
    int ncodes = 19; while (ncodes > 4 && !cl.len[order[ncodes - 1]]) ncodes--;
    bw.put(0, 1);
    bw.put((uint32_t)ncodes - 4u, 4);
    for (int i = 0; i < ncodes; i++) bw.put(cl.len[order[i]], 3);
    bw.put(0, 1);                                   // every symbol's length follows (no max_symbol)
    for (const Tk &t : tk) {
        vp8l_put_sym(bw, cl, t.sym);
        if (t.sym == 17) bw.put(t.extra, 3); else if (t.sym == 18) bw.put(t.extra, 7);
    }
}

bool vp8l_alpha_from_tokens(const uint32_t *tok, size_t ntok, int width, int height, std::vector<uint8_t> &alph, int filter)
{
    const size_t npix = (size_t)width * height;
    // ---- tokens -> operations: consecutive copies at the same distance continue each other (K7 cuts matches at 258 and at its
    //      parse-chunk ends; this format allows 4096 pixels per copy)
    struct Op { uint32_t len, dist; };              // len 0: literal `dist`
    std::vector<Op> ops; ops.reserve(ntok);
    size_t pos = 0;
    for (size_t i = 0; i < ntok; i++) {
        const uint32_t t = tok[i];
        if (!(t & 0x80000000u)) { ops.push_back({0u, t & 0xFFu}); pos++; continue; }
        const uint32_t len = ((t >> 16) & 0xFFu) + 3u, dist = (t & 0xFFFFu) + 1u;
        if (dist > pos) return false;
        if (!ops.empty() && ops.back().len && ops.back().dist == dist && ops.back().len + len <= 4096u) ops.back().len += len;
        else ops.push_back({len, dist});
        pos += len;
    }
    if (pos != npix) return false;
    // ---- statistics and codes
    Vp8lPlaneCodes planes; vp8l_plane_codes_init(&planes, width);
    std::vector<uint32_t> gf(256 + 24, 0), df(40, 0);
    for (Op &o : ops) {
        if (!o.len) { gf[o.dist]++; continue; }
        int s, nx; uint32_t xv;
        vp8l_prefix_of(o.len, &s, &nx, &xv); gf[256 + s]++;
        vp8l_prefix_of(vp8l_plane_code_of(&planes, o.dist), &s, &nx, &xv); df[s]++;
    }
    static thread_local Vp8lHuffScratch S;
    PrefixCode green, dist, zero;
    vp8l_make_code(gf, green, S); vp8l_make_code(df, dist, S);
    zero.len.assign(256, 0); zero.code.assign(256, 0); zero.used = 0;
    // ---- the chunk: header byte (no pre-processing, the caller's prediction filter, lossless compression) + image stream
    alph.clear(); alph.reserve(npix / 8 + 64);
    alph.push_back((uint8_t)(0x01 | ((filter & 3) << 2)));
    BitsLsb bw(alph);
    bw.put(0, 1);                       // no transform
    bw.put(0, 1);                       // no colour cache
    bw.put(0, 1);                       // one prefix-code group
    vp8l_write_code(bw, green, S);
    vp8l_write_code(bw, zero, S); vp8l_write_code(bw, zero, S); vp8l_write_code(bw, zero, S);      // red, blue, alpha: always 0
    vp8l_write_code(bw, dist, S);
    for (const Op &o : ops) {
        if (!o.len) { vp8l_put_sym(bw, green, (int)o.dist); continue; }
        int s, nx; uint32_t xv;
        vp8l_prefix_of(o.len, &s, &nx, &xv); vp8l_put_sym(bw, green, 256 + s); bw.put(xv, nx);
        vp8l_prefix_of(vp8l_plane_code_of(&planes, o.dist), &s, &nx, &xv); vp8l_put_sym(bw, dist, s); bw.put(xv, nx);
    }
    bw.flush();
    return true;
}

// residual of one row under filter f (1 horizontal, 2 vertical, 3 gradient); prev = the row above (unfiltered), nullptr for row 0.
// The first row is always predicted from the left, the first column of later rows from above (the conventions the decoder undoes).
static void alpha_filter_row(int f, const uint8_t *row, const uint8_t *prev, int w, uint8_t *out)
{
    if (!prev) { out[0] = row[0]; for (int x = 1; x < w; x++) out[x] = (uint8_t)(row[x] - row[x - 1]); return; }
    out[0] = (uint8_t)(row[0] - prev[0]);
    if (f == 1) for (int x = 1; x < w; x++) out[x] = (uint8_t)(row[x] - row[x - 1]);
    else if (f == 2) for (int x = 1; x < w; x++) out[x] = (uint8_t)(row[x] - prev[x]);
    else for (int x = 1; x < w; x++) { const int g = (int)row[x - 1] + prev[x] - prev[x - 1]; out[x] = (uint8_t)(row[x] - (g < 0 ? 0 : g > 255 ? 255 : g)); }
}

int webp_alpha_choose_filter(const uint8_t *alpha, int width, int height, std::vector<uint8_t> &filtered)
{
    // order-0 cost of the residuals of every fourth row, per filter, in 1/1024 bit (integer log2 as the PNG leg's literal costs)
    uint32_t hist[4][256];
    memset(hist, 0, sizeof(hist));
    std::vector<uint8_t> tmp((size_t)width);
    size_t rows = 0;
    for (int y = 0; y < height; y += 4, rows++) {
        const uint8_t *row = alpha + (size_t)y * width, *prev = y ? row - width : nullptr;
        for (int x = 0; x < width; x++) hist[0][row[x]]++;
        for (int f = 1; f < 4; f++) { alpha_filter_row(f, row, prev, width, tmp.data()); for (int x = 0; x < width; x++) hist[f][tmp[x]]++; }
    }
    const unsigned long long total = (unsigned long long)rows * width;
    auto log2q = [](unsigned long long v) { int e = 63; while (!((v >> e) & 1ull)) e--; const unsigned long long fr = e >= 10 ? (v >> (e - 10)) & 1023ull : (v << (10 - e)) & 1023ull; return (unsigned long long)e * 1024ull + fr; };
    int best = 0; unsigned long long best_cost = ~0ull;
    for (int f = 0; f < 4; f++) {
        unsigned long long cost = 0;
        for (int v = 0; v < 256; v++) if (hist[f][v]) cost += hist[f][v] * (log2q(total) - log2q(hist[f][v]));
        if (cost < best_cost) { best_cost = cost; best = f; }            // ties: the simpler filter
    }
    if (best) {
        filtered.resize((size_t)width * height);
        for (int y = 0; y < height; y++) alpha_filter_row(best, alpha + (size_t)y * width, y ? alpha + (size_t)(y - 1) * width : nullptr, width, filtered.data() + (size_t)y * width);
    }
    return best;
}

bool webp_wrap_alpha(const std::vector<uint8_t> &f, const std::vector<uint8_t> &alph, int width, int height, std::vector<uint8_t> &out)
{
    if (f.size() < 20 || memcmp(f.data(), "RIFF", 4) || memcmp(f.data() + 8, "WEBPVP8 ", 8)) return false;
    const uint32_t vsz = (uint32_t)f[16] | ((uint32_t)f[17] << 8) | ((uint32_t)f[18] << 16) | ((uint32_t)f[19] << 24);
    if ((size_t)vsz + 20 > f.size()) return false;
    auto u32 = [&](uint32_t v) { for (int i = 0; i < 4; i++) out.push_back((uint8_t)(v >> (8 * i))); };
    auto u24 = [&](uint32_t v) { for (int i = 0; i < 3; i++) out.push_back((uint8_t)(v >> (8 * i))); };
    auto tag = [&](const char *t) { out.insert(out.end(), t, t + 4); };
    const size_t asz = alph.size();
    const size_t total = 4 + (8 + 10) + (8 + asz + (asz & 1)) + (8 + vsz + (vsz & 1));
    out.clear(); out.reserve(total + 8);
    tag("RIFF"); u32((uint32_t)total); tag("WEBP");
    tag("VP8X"); u32(10); out.push_back(0x10); u24(0); u24((uint32_t)width - 1); u24((uint32_t)height - 1);
    tag("ALPH"); u32((uint32_t)asz); out.insert(out.end(), alph.begin(), alph.end()); if (asz & 1) out.push_back(0);
    tag("VP8 "); u32(vsz); out.insert(out.end(), f.begin() + 20, f.begin() + 20 + vsz); if (vsz & 1) out.push_back(0);
    return true;
}

} // namespace b200
