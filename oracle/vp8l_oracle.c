/* vp8l_oracle.c -- scalar twin of the lossless WebP (VP8L) encoder (caesium-clt_b200/csrc/vp8l_kernels.cu + vp8l_encode.cpp):
 * every rule comes from the shared definitions of csrc/vp8l_enc_core.h, applied the plain way -- the 14 modes scored per tile, the
 * colour cache simulated in pixel order, the copy runs by a backward recurrence, the parse walked chunk by chunk -- and the bitstream is
 * written by a restatement of the host writer (length-limited Huffman codes as dfl_core.h builds them, the code serialisation of
 * vp8l_alpha.cpp).  TEST INFRASTRUCTURE, NOT PRODUCT CODE. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "../caesium-clt_b200/csrc/vp8l_enc_core.h"

/* ---- LSB-first bit writer -------------------------------------------------------------------------------------------------- */
typedef struct { uint8_t *p; size_t cap, n; uint64_t acc; int nb; int overflow; } OBits;
static void ob_put(OBits *b, uint32_t v, int nb)
{
    if (!nb) return;
    b->acc |= (uint64_t)(v & (nb >= 32 ? 0xFFFFFFFFu : ((1u << nb) - 1u))) << b->nb; b->nb += nb;
    while (b->nb >= 8) { if (b->n < b->cap) b->p[b->n] = (uint8_t)b->acc; else b->overflow = 1; b->n++; b->acc >>= 8; b->nb -= 8; }
}
static void ob_flush(OBits *b) { if (b->nb > 0) { if (b->n < b->cap) b->p[b->n] = (uint8_t)b->acc; else b->overflow = 1; b->n++; b->acc = 0; b->nb = 0; } }

/* ---- length-limited Huffman code lengths (the construction of dfl_core.h) and canonical codes ------------------------------ */
enum { OMAX = VP8L_NGREEN };
static void huff_lengths(const uint32_t *freq, int n, int limit, uint8_t *len)
{
    static uint16_t order[OMAX]; static uint64_t w[2 * OMAX]; static int16_t parent[2 * OMAX]; static uint8_t depth[2 * OMAX];
    int m = 0, i, bl[64];
    for (i = 0; i < n; i++) len[i] = 0;
    for (i = 0; i < n; i++) if (freq[i]) order[m++] = (uint16_t)i;
    for (i = 1; i < m; i++) {
        const uint16_t s = order[i]; const uint32_t f = freq[s]; int j = i - 1;
        while (j >= 0 && freq[order[j]] > f) { order[j + 1] = order[j]; j--; }
        order[j + 1] = s;
    }
    if (m == 0) return;
    if (m == 1) { len[order[0]] = 1; return; }
    for (i = 0; i < m; i++) w[i] = freq[order[i]];
    {
        int lq = 0, iq = m, next = m, k, t;
        for (k = 0; k < m - 1; k++) {
            int pick[2];
            for (t = 0; t < 2; t++) { if (lq < m && (iq >= next || w[lq] <= w[iq])) pick[t] = lq++; else pick[t] = iq++; }
            w[next] = w[pick[0]] + w[pick[1]];
            parent[pick[0]] = (int16_t)next; parent[pick[1]] = (int16_t)next;
            next++;
        }
        {
            const int root = next - 1;
            depth[root] = 0;
            for (i = 0; i < 64; i++) bl[i] = 0;
            for (i = root - 1; i >= 0; i--) { const int d = depth[parent[i]] + 1; depth[i] = (uint8_t)(d > 63 ? 63 : d); if (i < m) bl[depth[i]]++; }
        }
    }
    for (i = 63; i > limit; i--) while (bl[i] > 0) { int j = i - 2; while (bl[j] == 0) j--; bl[i] -= 2; bl[i - 1]++; bl[j + 1] += 2; bl[j]--; }
    {
        int k = m - 1, l = 1, left = bl[1];
        while (k >= 0) {
            int lo = k; const uint32_t f = freq[order[k]];
            while (lo > 0 && freq[order[lo - 1]] == f) lo--;
            for (i = lo; i <= k; i++) { while (left == 0 && l < limit) { l++; left = bl[l]; } len[order[i]] = (uint8_t)l; left--; }
            k = lo - 1;
        }
    }
}
static void canon_codes(const uint8_t *len, int n, uint16_t *code)
{
    int cnt[16], next[16], c = 0, i, l, b;
    for (i = 0; i < 16; i++) cnt[i] = 0;
    for (i = 0; i < n; i++) cnt[len[i]]++;
    cnt[0] = 0; next[0] = 0;
    for (l = 1; l <= 15; l++) { c = (c + cnt[l - 1]) << 1; next[l] = c; }
    for (i = 0; i < n; i++) {
        code[i] = 0;
        if (len[i]) { const int v = next[len[i]]++; int r = 0; for (b = 0; b < len[i]; b++) if (v & (1 << b)) r |= 1 << (len[i] - 1 - b); code[i] = (uint16_t)r; }
    }
}

typedef struct { int n, used; uint8_t len[OMAX]; uint16_t code[OMAX]; } OCode;
static void make_code(const uint32_t *freq, int n, OCode *pc)
{
    int i;
    pc->n = n; pc->used = 0;
    for (i = 0; i < n; i++) pc->used += freq[i] != 0;
    huff_lengths(freq, n, 15, pc->len);
    canon_codes(pc->len, n, pc->code);
}
static void zero_code(int n, OCode *pc) { pc->n = n; pc->used = 0; memset(pc->len, 0, (size_t)n); memset(pc->code, 0, 2 * (size_t)n); }
static void put_sym(OBits *b, const OCode *pc, int s) { if (pc->used > 1) ob_put(b, pc->code[s], pc->len[s]); }

static void write_code(OBits *bw, const OCode *pc)
{
    static const uint8_t order[19] = {17, 18, 0, 1, 2, 3, 4, 5, 16, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15};
    static uint8_t tks[OMAX], tkx[OMAX];
    const int n = pc->n;
    int s0 = -1, s1 = -1, i, ntk = 0, ncodes;
    uint32_t cf[19];
    OCode cl;
    for (i = 0; i < n; i++) if (pc->len[i]) { if (s0 < 0) s0 = i; else if (s1 < 0) s1 = i; }
    if (pc->used == 0) { ob_put(bw, 1, 1); ob_put(bw, 0, 1); ob_put(bw, 0, 1); ob_put(bw, 0, 1); return; }
    if (pc->used <= 2 && s0 < 256 && (pc->used == 1 || s1 < 256)) {
        ob_put(bw, 1, 1); ob_put(bw, (uint32_t)pc->used - 1u, 1);
        if (s0 < 2) { ob_put(bw, 0, 1); ob_put(bw, (uint32_t)s0, 1); } else { ob_put(bw, 1, 1); ob_put(bw, (uint32_t)s0, 8); }
        if (pc->used == 2) ob_put(bw, (uint32_t)s1, 8);
        return;
    }
    for (i = 0; i < n;) {
        int run = 1;
        if (pc->len[i]) { tks[ntk] = pc->len[i]; tkx[ntk++] = 0; i++; continue; }
        while (i + run < n && !pc->len[i + run]) run++;
        i += run;
        while (run >= 11) { const int r = run > 138 ? 138 : run; tks[ntk] = 18; tkx[ntk++] = (uint8_t)(r - 11); run -= r; }
        if (run >= 3) { tks[ntk] = 17; tkx[ntk++] = (uint8_t)(run - 3); run = 0; }
        while (run-- > 0) { tks[ntk] = 0; tkx[ntk++] = 0; }
    }
    for (i = 0; i < 19; i++) cf[i] = 0;
    for (i = 0; i < ntk; i++) cf[tks[i]]++;
    make_code(cf, 19, &cl);
    huff_lengths(cf, 19, 7, cl.len);
    canon_codes(cl.len, 19, cl.code);
    ncodes = 19; while (ncodes > 4 && !cl.len[order[ncodes - 1]]) ncodes--;
    ob_put(bw, 0, 1);
    ob_put(bw, (uint32_t)ncodes - 4u, 4);
    for (i = 0; i < ncodes; i++) ob_put(bw, cl.len[order[i]], 3);
    ob_put(bw, 0, 1);
    for (i = 0; i < ntk; i++) {
        put_sym(bw, &cl, tks[i]);
        if (tks[i] == 17) ob_put(bw, tkx[i], 3); else if (tks[i] == 18) ob_put(bw, tkx[i], 7);
    }
}

/* rgba: [h][w][4].  force_mode >= 0: every tile takes that predictor; force_cache >= 0: that cache candidate (0..VP8L_NCACHE-1).
 * Stage outputs (any may be NULL): modes [tiles], hits [(VP8L_NCACHE - 1) x n], tokens [2 x n] as (position, copy) pairs with
 * *ntok of them, *cache_bits.  Returns the file size, or -1 (bad arguments, out > cap). */
long long orc_vp8l_encode(const uint8_t *rgba, int w, int h, int force_mode, int force_cache, uint8_t *out, size_t cap,
                          uint8_t *modes_out, uint8_t *hits_out, uint32_t *tok_out, size_t *ntok_out, int *cache_bits_out)
{
    const size_t n = (size_t)w * h;
    const int tiles_x = (w + VP8L_TILE - 1) >> VP8L_TILE_BITS, tiles_y = (h + VP8L_TILE - 1) >> VP8L_TILE_BITS, tiles = tiles_x * tiles_y;
    uint32_t *argb, *res, *best, *tok, *hist;
    uint8_t *modes, *hits;
    size_t i, ntok = 0;
    int alpha_used = 0, c, t, cand, bits, k;
    long long ret = -1;
    OCode pc[5], mc, z256, z40;
    OBits bw;
    if (w < 1 || h < 1 || w > 16384 || h > 16384 || cap < 32) return -1;
    argb = (uint32_t *)malloc(4 * n); res = (uint32_t *)malloc(4 * n); best = (uint32_t *)malloc(4 * n); tok = (uint32_t *)malloc(8 * n);
    hist = (uint32_t *)calloc((size_t)VP8L_NCACHE * VP8L_HIST, 4); modes = (uint8_t *)malloc((size_t)tiles); hits = (uint8_t *)calloc((size_t)(VP8L_NCACHE - 1) * n, 1);
    if (!argb || !res || !best || !tok || !hist || !modes || !hits) goto done;
    for (i = 0; i < n; i++) {
        const uint32_t r = rgba[4 * i], g = rgba[4 * i + 1], b = rgba[4 * i + 2], a = rgba[4 * i + 3];
        alpha_used |= a != 255;
        argb[i] = vp8l_sub_green((a << 24) | (r << 16) | (g << 8) | b);
    }
    /* predictor per tile */
    for (t = 0; t < tiles; t++) {
        const int tx = t % tiles_x, ty = t / tiles_x;
        int m, bm = 0, x, y; uint64_t bc = 0;
        for (m = 0; m < VP8L_NMODES; m++) {
            uint32_t hh[4 * 256], npix = 0; uint64_t cost;
            if (force_mode >= 0 && m != force_mode) continue;
            memset(hh, 0, sizeof(hh));
            for (y = ty * VP8L_TILE; y < h && y < (ty + 1) * VP8L_TILE; y++)
                for (x = tx * VP8L_TILE; x < w && x < (tx + 1) * VP8L_TILE; x++) {
                    const uint32_t r = vp8l_sub_px(argb[(size_t)y * w + x], vp8l_predict_at(m, argb, w, x, y));
                    hh[r & 0xFF]++; hh[256 + ((r >> 8) & 0xFF)]++; hh[512 + ((r >> 16) & 0xFF)]++; hh[768 + (r >> 24)]++; npix++;
                }
            cost = vp8l_tile_cost(hh, npix);     /* (a 257-entry table of vp8l_nlog2_q10 on the device) */
            if (force_mode >= 0 || m == 0 || cost < bc) { bc = cost; bm = m; }
        }
        modes[t] = (uint8_t)bm;
    }
    for (i = 0; i < n; i++) {
        const int x = (int)(i % (size_t)w), y = (int)(i / (size_t)w);
        res[i] = vp8l_sub_px(argb[i], vp8l_predict_at(modes[(y >> VP8L_TILE_BITS) * tiles_x + (x >> VP8L_TILE_BITS)], argb, w, x, y));
    }
    /* colour-cache hits, simulated in pixel order */
    for (c = 1; c < VP8L_NCACHE; c++) {
        const int b = vp8l_cache_bits(c);
        uint32_t cache[1 << VP8L_MAX_CACHE_BITS];
        memset(cache, 0, sizeof(cache));
        for (i = 0; i < n; i++) { const uint32_t key = vp8l_cache_key(res[i], b); hits[(size_t)(c - 1) * n + i] = cache[key] == res[i]; cache[key] = res[i]; }
    }
    /* copies and the parse */
    /* vp8l_best_copy at every pixel, its runs by the backward recurrence run(i) = equal(i) ? run(i + 1) + 1 : 0 inside each chunk (a
     * chunk is no longer than VP8L_MAX_COPY, so the cap never binds); the tests pin the recurrence to the definition */
    for (i = 0; i < n; i += VP8L_CHUNK) {
        const size_t end = i + VP8L_CHUNK < n ? i + VP8L_CHUNK : n;
        uint32_t run[VP8L_NCAND + 1];
        size_t j = end;
        memset(run, 0, sizeof(run));
        while (j-- > i) {
            uint32_t bl = 0, bb = 0;
            for (c = 1; c <= VP8L_NCAND; c++) {
                const uint32_t d = vp8l_code_dist(c, w);
                run[c] = (d <= j && res[j] == res[j - d]) ? run[c] + 1 : 0;
                if (run[c] > bl) { bl = run[c]; bb = (run[c] << 8) | (uint32_t)c; }
            }
            best[j] = bl >= VP8L_MIN_COPY ? bb : 0u;
        }
    }
    for (i = 0; i < n; i += VP8L_CHUNK) {
        const size_t end = i + VP8L_CHUNK < n ? i + VP8L_CHUNK : n;
        size_t j = i;
        while (j < end) {
            const uint32_t next = j + 1 < end ? best[j + 1] : 0u, step = vp8l_parse_step(best[j], next);
            tok[2 * ntok] = (uint32_t)j; tok[2 * ntok + 1] = vp8l_token_copy(best[j], next); ntok++;
            j += step;
        }
    }
    /* histograms per cache candidate and the choice */
    for (c = 0; c < VP8L_NCACHE; c++) {
        uint32_t *hc = hist + (size_t)c * VP8L_HIST;
        const int b = vp8l_cache_bits(c);
        for (i = 0; i < ntok; i++) {
            const uint32_t pos = tok[2 * i], cp = tok[2 * i + 1];
            int s, nx; uint32_t xv;
            if (cp) { vp8l_prefix_of(cp >> 8, &s, &nx, &xv); hc[256 + s]++; vp8l_prefix_of(cp & 0xFF, &s, &nx, &xv); hc[VP8L_HIST_DIST + s]++; continue; }
            if (c && hits[(size_t)(c - 1) * n + pos]) { hc[280 + vp8l_cache_key(res[pos], b)]++; continue; }
            hc[(res[pos] >> 8) & 0xFF]++; hc[VP8L_HIST_RED + ((res[pos] >> 16) & 0xFF)]++; hc[VP8L_HIST_BLUE + (res[pos] & 0xFF)]++; hc[VP8L_HIST_ALPHA + (res[pos] >> 24)]++;
        }
    }
    cand = force_cache >= 0 ? force_cache : vp8l_choose_cache(hist);
    bits = vp8l_cache_bits(cand);
    {
        const uint32_t *hc = hist + (size_t)cand * VP8L_HIST;
        const int base[5] = {0, VP8L_HIST_RED, VP8L_HIST_BLUE, VP8L_HIST_ALPHA, VP8L_HIST_DIST};
        const int size[5] = {256 + 24 + (bits ? 1 << bits : 0), 256, 256, 256, VP8L_NDIST};
        for (k = 0; k < 5; k++) make_code(hc + base[k], size[k], &pc[k]);
    }
    /* the file: RIFF header (sizes patched at the end), then the VP8L chunk */
    memset(&bw, 0, sizeof(bw)); bw.p = out + 20; bw.cap = cap - 21;
    ob_put(&bw, 0x2f, 8); ob_put(&bw, (uint32_t)w - 1, 14); ob_put(&bw, (uint32_t)h - 1, 14); ob_put(&bw, (uint32_t)alpha_used, 1); ob_put(&bw, 0, 3);
    ob_put(&bw, 1, 1); ob_put(&bw, 2, 2);
    ob_put(&bw, 1, 1); ob_put(&bw, 0, 2); ob_put(&bw, VP8L_TILE_BITS - 2, 3);
    {
        uint32_t mf[280];
        memset(mf, 0, sizeof(mf));
        for (t = 0; t < tiles; t++) mf[modes[t]]++;
        make_code(mf, 280, &mc); zero_code(256, &z256); zero_code(VP8L_NDIST, &z40);
        ob_put(&bw, 0, 1);
        write_code(&bw, &mc); write_code(&bw, &z256); write_code(&bw, &z256); write_code(&bw, &z256); write_code(&bw, &z40);
        for (t = 0; t < tiles; t++) put_sym(&bw, &mc, modes[t]);
    }
    ob_put(&bw, 0, 1);
    if (bits) { ob_put(&bw, 1, 1); ob_put(&bw, (uint32_t)bits, 4); } else ob_put(&bw, 0, 1);
    ob_put(&bw, 0, 1);
    for (k = 0; k < 5; k++) write_code(&bw, &pc[k]);
    for (i = 0; i < ntok; i++) {
        const uint32_t pos = tok[2 * i], cp = tok[2 * i + 1], p = res[pos];
        int s, nx; uint32_t xv;
        if (cp) {
            vp8l_prefix_of(cp >> 8, &s, &nx, &xv); put_sym(&bw, &pc[0], 256 + s); ob_put(&bw, xv, nx);
            vp8l_prefix_of(cp & 0xFF, &s, &nx, &xv); put_sym(&bw, &pc[4], s); ob_put(&bw, xv, nx);
        } else if (cand && hits[(size_t)(cand - 1) * n + pos]) put_sym(&bw, &pc[0], 280 + (int)vp8l_cache_key(p, bits));
        else { put_sym(&bw, &pc[0], (p >> 8) & 0xFF); put_sym(&bw, &pc[1], (p >> 16) & 0xFF); put_sym(&bw, &pc[2], p & 0xFF); put_sym(&bw, &pc[3], p >> 24); }
    }
    ob_flush(&bw);
    if (bw.overflow) goto done;
    {
        const size_t nb = bw.n, pad = nb & 1, riff = 4 + 8 + nb + pad;
        memcpy(out, "RIFF", 4); for (k = 0; k < 4; k++) out[4 + k] = (uint8_t)(riff >> (8 * k));
        memcpy(out + 8, "WEBPVP8L", 8); for (k = 0; k < 4; k++) out[16 + k] = (uint8_t)(nb >> (8 * k));
        if (pad) out[20 + nb] = 0;
        ret = (long long)(8 + riff);
    }
    if (modes_out) memcpy(modes_out, modes, (size_t)tiles);
    if (hits_out) memcpy(hits_out, hits, (size_t)(VP8L_NCACHE - 1) * n);
    if (tok_out) memcpy(tok_out, tok, 8 * ntok);
    if (ntok_out) *ntok_out = ntok;
    if (cache_bits_out) *cache_bits_out = bits;
done:
    free(argb); free(res); free(best); free(tok); free(hist); free(modes); free(hits);
    return ret;
}
