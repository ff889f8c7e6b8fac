/* vp8l_palette_oracle.c -- scalar twin of the lossless WebP (VP8L) encoder's colour-indexing (palette) variant
 * (caesium-clt_b200/csrc/vp8l_palette.cu + vp8l_encode.cpp): the rules of csrc/vp8l_palette_core.h applied the plain way -- the
 * colours by sorting the image, the indices by search -- and the packed index image coded by a plain restatement of the encoder's
 * entropy stage (colour cache in pixel order, copies by a backward recurrence, the chunked greedy parse, the Huffman codes of
 * dfl_core.h).  The variant without the palette is orc_vp8l_encode's file.  TEST INFRASTRUCTURE, NOT PRODUCT CODE. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "../caesium-clt_b200/csrc/vp8l_palette_core.h"

long long orc_vp8l_encode(const uint8_t *rgba, int w, int h, int force_mode, int force_cache, uint8_t *out, size_t cap,
                          uint8_t *modes_out, uint8_t *hits_out, uint32_t *tok_out, size_t *ntok_out, int *cache_bits_out);

/* ---- LSB-first bit writer ---------------------------------------------------------------------------------------------------- */
typedef struct { uint8_t *p; size_t cap, n; uint64_t acc; int nb; int overflow; } PBits;
static void pb_put(PBits *b, uint32_t v, int nb)
{
    if (!nb) return;
    b->acc |= (uint64_t)(v & (nb >= 32 ? 0xFFFFFFFFu : ((1u << nb) - 1u))) << b->nb; b->nb += nb;
    while (b->nb >= 8) { if (b->n < b->cap) b->p[b->n] = (uint8_t)b->acc; else b->overflow = 1; b->n++; b->acc >>= 8; b->nb -= 8; }
}
static void pb_flush(PBits *b) { if (b->nb > 0) pb_put(b, 0, 8 - b->nb); }

/* ---- length-limited Huffman codes (dfl_core.h's construction: a two-queue merge of the sorted weights, the overflow of depths
 * past the limit moved up a level, lengths handed out longest-first over equal-frequency groups) ------------------------------ */
enum { PMAX = VP8L_NGREEN };
typedef struct { int n, used; uint8_t len[PMAX]; uint16_t code[PMAX]; } PCode;
static void p_lengths(const uint32_t *freq, int n, int limit, uint8_t *len)
{
    static uint16_t order[PMAX]; static uint64_t wt[2 * PMAX]; static int16_t parent[2 * PMAX]; static uint8_t depth[2 * PMAX];
    int m = 0, i, bl[64];
    for (i = 0; i < n; i++) len[i] = 0;
    for (i = 0; i < n; i++) if (freq[i]) order[m++] = (uint16_t)i;
    for (i = 1; i < m; i++) {
        const uint16_t s = order[i]; int j = i - 1;
        while (j >= 0 && freq[order[j]] > freq[s]) { order[j + 1] = order[j]; j--; }
        order[j + 1] = s;
    }
    if (m == 0) return;
    if (m == 1) { len[order[0]] = 1; return; }
    for (i = 0; i < m; i++) wt[i] = freq[order[i]];
    {
        int lq = 0, iq = m, next = m, k, t;
        for (k = 0; k < m - 1; k++) {
            int pick[2];
            for (t = 0; t < 2; t++) { if (lq < m && (iq >= next || wt[lq] <= wt[iq])) pick[t] = lq++; else pick[t] = iq++; }
            wt[next] = wt[pick[0]] + wt[pick[1]];
            parent[pick[0]] = (int16_t)next; parent[pick[1]] = (int16_t)next;
            next++;
        }
        depth[next - 1] = 0;
        for (i = 0; i < 64; i++) bl[i] = 0;
        for (i = next - 2; i >= 0; i--) { const int d = depth[parent[i]] + 1; depth[i] = (uint8_t)(d > 63 ? 63 : d); if (i < m) bl[depth[i]]++; }
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
static void p_make(const uint32_t *freq, int n, int limit, PCode *pc)
{
    int cnt[16], next[16], c = 0, i, l, b;
    pc->n = n; pc->used = 0;
    for (i = 0; i < n; i++) pc->used += freq[i] != 0;
    p_lengths(freq, n, limit, pc->len);
    for (i = 0; i < 16; i++) cnt[i] = 0;
    for (i = 0; i < n; i++) cnt[pc->len[i]]++;
    cnt[0] = 0; next[0] = 0;
    for (l = 1; l <= 15; l++) { c = (c + cnt[l - 1]) << 1; next[l] = c; }
    for (i = 0; i < n; i++) {
        pc->code[i] = 0;
        if (pc->len[i]) { const int v = next[pc->len[i]]++; int r = 0; for (b = 0; b < pc->len[i]; b++) if (v & (1 << b)) r |= 1 << (pc->len[i] - 1 - b); pc->code[i] = (uint16_t)r; }
    }
}
static void p_sym(PBits *b, const PCode *pc, int s) { if (pc->used > 1) pb_put(b, pc->code[s], pc->len[s]); }
/* the code's description (specification section 6.2.1 / 6.2.2): simple codes for up to two symbols below 256, else the code
 * lengths run-length coded (17 / 18 for zero runs) under a code-length code of limit 7 */
static void p_write(PBits *bw, const PCode *pc)
{
    static const uint8_t order[19] = {17, 18, 0, 1, 2, 3, 4, 5, 16, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15};
    static uint8_t tks[PMAX], tkx[PMAX];
    int s0 = -1, s1 = -1, i, ntk = 0, ncodes;
    uint32_t cf[19];
    PCode cl;
    for (i = 0; i < pc->n; i++) if (pc->len[i]) { if (s0 < 0) s0 = i; else if (s1 < 0) s1 = i; }
    if (pc->used == 0) { pb_put(bw, 1, 1); pb_put(bw, 0, 1); pb_put(bw, 0, 1); pb_put(bw, 0, 1); return; }
    if (pc->used <= 2 && s0 < 256 && (pc->used == 1 || s1 < 256)) {
        pb_put(bw, 1, 1); pb_put(bw, (uint32_t)pc->used - 1u, 1);
        if (s0 < 2) { pb_put(bw, 0, 1); pb_put(bw, (uint32_t)s0, 1); } else { pb_put(bw, 1, 1); pb_put(bw, (uint32_t)s0, 8); }
        if (pc->used == 2) pb_put(bw, (uint32_t)s1, 8);
        return;
    }
    for (i = 0; i < pc->n;) {
        int run = 1;
        if (pc->len[i]) { tks[ntk] = pc->len[i]; tkx[ntk++] = 0; i++; continue; }
        while (i + run < pc->n && !pc->len[i + run]) run++;
        i += run;
        while (run >= 11) { const int r = run > 138 ? 138 : run; tks[ntk] = 18; tkx[ntk++] = (uint8_t)(r - 11); run -= r; }
        if (run >= 3) { tks[ntk] = 17; tkx[ntk++] = (uint8_t)(run - 3); run = 0; }
        while (run-- > 0) { tks[ntk] = 0; tkx[ntk++] = 0; }
    }
    for (i = 0; i < 19; i++) cf[i] = 0;
    for (i = 0; i < ntk; i++) cf[tks[i]]++;
    p_make(cf, 19, 7, &cl);
    ncodes = 19; while (ncodes > 4 && !cl.len[order[ncodes - 1]]) ncodes--;
    pb_put(bw, 0, 1);
    pb_put(bw, (uint32_t)ncodes - 4u, 4);
    for (i = 0; i < ncodes; i++) pb_put(bw, cl.len[order[i]], 3);
    pb_put(bw, 0, 1);
    for (i = 0; i < ntk; i++) {
        p_sym(bw, &cl, tks[i]);
        if (tks[i] == 17) pb_put(bw, tkx[i], 3); else if (tks[i] == 18) pb_put(bw, tkx[i], 7);
    }
}

/* ---- the entropy-coded main image of res (cw x h, no predictor): cache bits, no meta image, five codes, the pixels ------------ */
static int code_main(PBits *bw, const uint32_t *res, int cw, int h)
{
    const size_t n = (size_t)cw * h;
    uint32_t *best = (uint32_t *)malloc(4 * n), *tok = (uint32_t *)malloc(8 * n), *hist = (uint32_t *)calloc((size_t)VP8L_NCACHE * VP8L_HIST, 4);
    uint8_t *hits = (uint8_t *)calloc((size_t)(VP8L_NCACHE - 1) * n, 1);
    size_t i, ntok = 0;
    int c, k, cand, bits, ok = 0;
    static PCode pc[5];
    if (!best || !tok || !hist || !hits) goto done;
    for (c = 1; c < VP8L_NCACHE; c++) {                     /* the colour cache, simulated in pixel order */
        const int b = vp8l_cache_bits(c);
        uint32_t cache[1 << VP8L_MAX_CACHE_BITS];
        memset(cache, 0, sizeof(cache));
        for (i = 0; i < n; i++) { const uint32_t key = vp8l_cache_key(res[i], b); hits[(size_t)(c - 1) * n + i] = cache[key] == res[i]; cache[key] = res[i]; }
    }
    for (i = 0; i < n; i += VP8L_CHUNK) {                   /* copies: run(j) = equal(j) ? run(j + 1) + 1 : 0 inside each chunk */
        const size_t end = i + VP8L_CHUNK < n ? i + VP8L_CHUNK : n;
        uint32_t run[VP8L_NCAND + 1];
        size_t j = end;
        memset(run, 0, sizeof(run));
        while (j-- > i) {
            uint32_t bl = 0, bb = 0;
            for (c = 1; c <= VP8L_NCAND; c++) {
                const uint32_t d = vp8l_code_dist(c, cw);
                run[c] = (d <= j && res[j] == res[j - d]) ? run[c] + 1 : 0;
                if (run[c] > bl) { bl = run[c]; bb = (run[c] << 8) | (uint32_t)c; }
            }
            best[j] = bl >= VP8L_MIN_COPY ? bb : 0u;
        }
    }
    for (i = 0; i < n; i += VP8L_CHUNK) {                   /* the parse, chunk by chunk */
        const size_t end = i + VP8L_CHUNK < n ? i + VP8L_CHUNK : n;
        size_t j = i;
        while (j < end) {
            const uint32_t next = j + 1 < end ? best[j + 1] : 0u;
            tok[2 * ntok] = (uint32_t)j; tok[2 * ntok + 1] = vp8l_token_copy(best[j], next); ntok++;
            j += vp8l_parse_step(best[j], next);
        }
    }
    for (c = 0; c < VP8L_NCACHE; c++) {
        uint32_t *hc = hist + (size_t)c * VP8L_HIST;
        const int b = vp8l_cache_bits(c);
        for (i = 0; i < ntok; i++) {
            const uint32_t pos = tok[2 * i], cp = tok[2 * i + 1], p = res[pos];
            int s, nx; uint32_t xv;
            if (cp) { vp8l_prefix_of(cp >> 8, &s, &nx, &xv); hc[256 + s]++; vp8l_prefix_of(cp & 0xFF, &s, &nx, &xv); hc[VP8L_HIST_DIST + s]++; continue; }
            if (c && hits[(size_t)(c - 1) * n + pos]) { hc[280 + vp8l_cache_key(p, b)]++; continue; }
            hc[(p >> 8) & 0xFF]++; hc[VP8L_HIST_RED + ((p >> 16) & 0xFF)]++; hc[VP8L_HIST_BLUE + (p & 0xFF)]++; hc[VP8L_HIST_ALPHA + (p >> 24)]++;
        }
    }
    cand = vp8l_choose_cache(hist);
    bits = vp8l_cache_bits(cand);
    {
        const uint32_t *hc = hist + (size_t)cand * VP8L_HIST;
        const int base[5] = {0, VP8L_HIST_RED, VP8L_HIST_BLUE, VP8L_HIST_ALPHA, VP8L_HIST_DIST};
        const int size[5] = {256 + 24 + (bits ? 1 << bits : 0), 256, 256, 256, VP8L_NDIST};
        for (k = 0; k < 5; k++) p_make(hc + base[k], size[k], 15, &pc[k]);
    }
    if (bits) { pb_put(bw, 1, 1); pb_put(bw, (uint32_t)bits, 4); } else pb_put(bw, 0, 1);
    pb_put(bw, 0, 1);
    for (k = 0; k < 5; k++) p_write(bw, &pc[k]);
    for (i = 0; i < ntok; i++) {
        const uint32_t pos = tok[2 * i], cp = tok[2 * i + 1], p = res[pos];
        int s, nx; uint32_t xv;
        if (cp) {
            vp8l_prefix_of(cp >> 8, &s, &nx, &xv); p_sym(bw, &pc[0], 256 + s); pb_put(bw, xv, nx);
            vp8l_prefix_of(cp & 0xFF, &s, &nx, &xv); p_sym(bw, &pc[4], s); pb_put(bw, xv, nx);
        } else if (cand && hits[(size_t)(cand - 1) * n + pos]) p_sym(bw, &pc[0], 280 + (int)vp8l_cache_key(p, bits));
        else { p_sym(bw, &pc[0], (p >> 8) & 0xFF); p_sym(bw, &pc[1], (p >> 16) & 0xFF); p_sym(bw, &pc[2], p & 0xFF); p_sym(bw, &pc[3], p >> 24); }
    }
    ok = 1;
done:
    free(best); free(tok); free(hist); free(hits);
    return ok;
}

static int cmp_u32(const void *a, const void *b) { const uint32_t x = *(const uint32_t *)a, y = *(const uint32_t *)b; return x < y ? -1 : x > y; }

/* rgba: [h][w][4].  out: the file the encoder keeps with the palette switch on; sizes[2]: the file sizes without / with the palette
 * (sizes[1] = 0 when there are more than 256 colours); pal [256] and *count: the palette (*count = -1 over 256 colours); packed
 * [w x h] and *packed_w: the packed index image; pal_file (cap bytes, or NULL): the palette variant's file, kept or not.  Returns
 * the kept file's size, or -1 (bad arguments, out > cap). */
long long orc_vp8l_encode_palette(const uint8_t *rgba, int w, int h, uint8_t *out, size_t cap, long long *sizes, uint32_t *pal, int *count,
                                  uint32_t *packed, int *packed_w, uint8_t *pal_file)
{
    const size_t n = (size_t)w * h;
    uint32_t *argb, *sorted;
    uint8_t *alt = NULL;
    size_t i;
    int m = 0, alpha_used = 0, k;
    long long ret = -1, s0;
    if (w < 1 || h < 1 || w > 16384 || h > 16384 || cap < 32) return -1;
    sizes[0] = sizes[1] = 0; *count = -1; *packed_w = 0;
    s0 = orc_vp8l_encode(rgba, w, h, -1, -1, out, cap, NULL, NULL, NULL, NULL, NULL);
    if (s0 < 0) return -1;
    sizes[0] = s0;
    argb = (uint32_t *)malloc(4 * n); sorted = (uint32_t *)malloc(4 * n);
    if (!argb || !sorted) goto done;
    for (i = 0; i < n; i++) {
        const uint32_t r = rgba[4 * i], g = rgba[4 * i + 1], b = rgba[4 * i + 2], a = rgba[4 * i + 3];
        alpha_used |= a != 255;
        argb[i] = vp8l_sub_green((a << 24) | (r << 16) | (g << 8) | b);   /* as the encoder's buffer holds them */
        sorted[i] = (a << 24) | (r << 16) | (g << 8) | b;
    }
    qsort(sorted, n, 4, cmp_u32);
    for (i = 0; i < n && m <= VP8L_PAL_MAX; i++) if (i == 0 || sorted[i] != sorted[i - 1]) { if (m < VP8L_PAL_MAX) pal[m] = sorted[i]; m++; }
    ret = s0;
    if (m > VP8L_PAL_MAX) goto done;
    *count = m;
    {
        const int xbits = vp8l_pal_xbits(m), wp = vp8l_pal_width(w, xbits);
        int x, y;
        PBits bw;
        *packed_w = wp;
        for (y = 0; y < h; y++)
            for (x = 0; x < wp; x++) {                       /* plain: each index by a linear search of the palette */
                uint32_t bundle = 0; int j;
                for (j = 0; j < (1 << xbits) && (x << xbits) + j < w; j++) {
                    const uint32_t c = vp8l_add_green(argb[(size_t)y * w + (x << xbits) + j]);
                    int idx = 0;
                    while (pal[idx] != c) idx++;
                    bundle |= (uint32_t)idx << (j * (8 >> xbits));
                }
                packed[(size_t)y * wp + x] = 0xFF000000u | (bundle << 8);
            }
        alt = (uint8_t *)malloc(cap);
        if (!alt) { ret = -1; goto done; }
        memset(&bw, 0, sizeof(bw)); bw.p = alt + 20; bw.cap = cap - 21;
        pb_put(&bw, 0x2f, 8); pb_put(&bw, (uint32_t)w - 1, 14); pb_put(&bw, (uint32_t)h - 1, 14); pb_put(&bw, (uint32_t)alpha_used, 1); pb_put(&bw, 0, 3);
        pb_put(&bw, 1, 1); pb_put(&bw, 3, 2); pb_put(&bw, (uint32_t)m - 1, 8);
        {   /* the palette image: m x 1, no cache, entries minus the previous entry, literals only */
            static uint32_t f[5][280];
            static PCode c[5];
            memset(f, 0, sizeof(f));
            for (k = 0; k < m; k++) {
                const uint32_t d = vp8l_pal_delta(pal, k);
                f[0][(d >> 8) & 0xFF]++; f[1][(d >> 16) & 0xFF]++; f[2][d & 0xFF]++; f[3][d >> 24]++;
            }
            p_make(f[0], 280, 15, &c[0]); p_make(f[1], 256, 15, &c[1]); p_make(f[2], 256, 15, &c[2]); p_make(f[3], 256, 15, &c[3]);
            p_make(f[4], VP8L_NDIST, 15, &c[4]);
            pb_put(&bw, 0, 1);
            for (k = 0; k < 5; k++) p_write(&bw, &c[k]);
            for (k = 0; k < m; k++) {
                const uint32_t d = vp8l_pal_delta(pal, k);
                p_sym(&bw, &c[0], (d >> 8) & 0xFF); p_sym(&bw, &c[1], (d >> 16) & 0xFF); p_sym(&bw, &c[2], d & 0xFF); p_sym(&bw, &c[3], d >> 24);
            }
        }
        pb_put(&bw, 0, 1);
        if (!code_main(&bw, packed, wp, h)) { ret = -1; goto done; }
        pb_flush(&bw);
        if (bw.overflow) { ret = -1; goto done; }
        {
            const size_t nb = bw.n, pad = nb & 1, riff = 4 + 8 + nb + pad;
            memcpy(alt, "RIFF", 4); for (k = 0; k < 4; k++) alt[4 + k] = (uint8_t)(riff >> (8 * k));
            memcpy(alt + 8, "WEBPVP8L", 8); for (k = 0; k < 4; k++) alt[16 + k] = (uint8_t)(nb >> (8 * k));
            if (pad) alt[20 + nb] = 0;
            sizes[1] = (long long)(8 + riff);
        }
        if (pal_file) memcpy(pal_file, alt, (size_t)sizes[1]);
        if (sizes[1] < s0) { memcpy(out, alt, (size_t)sizes[1]); ret = sizes[1]; }
    }
done:
    free(argb); free(sorted); free(alt);
    return ret;
}
