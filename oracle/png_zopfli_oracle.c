/* png_zopfli_oracle.c -- scalar twin of the PNG `--zopfli` leg (caesium-clt_b200/csrc/png_zopfli.cu) over the same rules
 * (png_zopfli_core.h): match sets, cost tables, the per-segment shortest path, iterations, scoring and slices, run one position at a
 * time.  TEST INFRASTRUCTURE, NOT PRODUCT CODE. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "../caesium-clt_b200/csrc/png_zopfli_core.h"

size_t orc_png_lz77(const uint8_t *s, size_t n, int bpp, int stride, uint32_t *tokens, uint32_t *hist);

/* prev[j] = the nearest earlier position with j's hash, -1 if none (a plain head table over the whole stream) */
static int32_t *hash_prev(const uint8_t *s, size_t n)
{
    int32_t *prev = (int32_t *)malloc((n + 1) * sizeof(int32_t)), *head = (int32_t *)malloc(65536 * sizeof(int32_t));
    memset(head, 0xFF, 65536 * sizeof(int32_t));
    for (size_t j = 0; j < n; j++) {
        if (j + 3 > n) { prev[j] = -1; continue; }
        const uint32_t h = pz_hash3(s + j);
        prev[j] = head[h]; head[h] = (int32_t)j;
    }
    free(head);
    return prev;
}

/* the shortest path of segment [s0, s0 + L) under `cost`; tokens to out, their number returned, counted into hist */
static size_t squeeze(const uint8_t *s, size_t s0, size_t L, const uint32_t *ent, const int *cnt, const uint32_t *cost, uint32_t *out, uint32_t *hist)
{
    uint32_t *c = (uint32_t *)malloc((L + 1) * 4), *bp = (uint32_t *)malloc((L + 1) * 4);
    c[0] = 0;
    for (size_t t = 1; t <= L; t++) c[t] = 0xFFFFFFFFu;
    for (size_t i = 0; i < L; i++) {
        const uint32_t ci = c[i];
        const uint32_t lit = ci + cost[s[s0 + i]];
        if (lit < c[i + 1]) { c[i + 1] = lit; bp[i + 1] = s[s0 + i]; }
        const uint32_t *e = ent + i * PZ_K;
        const int k = cnt[i];
        if (!k) continue;
        const int top = pz_elen(e[k - 1]);
        for (int l = 3; l <= top; l++) {
            uint32_t tok; const uint32_t v = ci + pz_edge(e, k, l, cost, &tok);
            if (v < c[i + l]) { c[i + l] = v; bp[i + l] = tok; }
        }
    }
    size_t m = 0;
    for (size_t t = L; t > 0;) { const uint32_t tok = bp[t]; out[m++] = tok; t -= tok & 0x80000000u ? (size_t)pz_elen(tok & 0x7FFFFFFFu) : 1; }
    for (size_t a = 0, b = m ? m - 1 : 0; a < b; a++, b--) { const uint32_t x = out[a]; out[a] = out[b]; out[b] = x; }
    for (size_t q = 0; q < m; q++) pz_count(hist, out[q]);
    free(c); free(bp);
    return m;
}

/* the kept entries of every position of [p0, p1) */
static void match_sets(const uint8_t *s, size_t n, int bpp, int stride, const int32_t *prev, size_t p0, size_t p1, uint32_t *ent, int *cnt)
{
    int cand[10]; pz_fixed_sorted(bpp, stride, cand);
    for (size_t i = p0; i < p1; i++) cnt[i - p0] = pz_match_set(s, n, i, cand, prev, 0, ent + (i - p0) * PZ_K);
}

/* tokens must hold n entries; returns the token count */
size_t orc_png_lz77_zopfli(const uint8_t *s, size_t n, int bpp, int stride, uint32_t *tokens)
{
    if (!n) return 0;
    const size_t nreg = (n + PZ_REGION - 1) / PZ_REGION, nseg = (n + PZ_SEG - 1) / PZ_SEG;
    uint32_t *hg = (uint32_t *)calloc(nreg * PZ_NSYM, 4), *hprev = (uint32_t *)calloc(nreg * PZ_NSYM, 4), *hcur = (uint32_t *)calloc(nreg * PZ_NSYM, 4), *cost = (uint32_t *)malloc(nreg * PZ_NSYM * 4);
    {   /* iteration 1's statistics: the greedy / lazy parse, token by token into the region where the token starts */
        uint32_t *g = (uint32_t *)malloc((n + 1) * 4), gh[PZ_NSYM];
        const size_t ng = orc_png_lz77(s, n, bpp, stride, g, gh);
        size_t p = 0;
        for (size_t t = 0; t < ng; t++) { pz_count(hg + (p / PZ_REGION) * PZ_NSYM, g[t]); p += g[t] & 0x80000000u ? (size_t)pz_elen(g[t] & 0x7FFFFFFFu) : 1; }
        free(g);
    }
    int32_t *prev = hash_prev(s, n);
    const size_t slice_cap = n < PZ_SLICE ? n : PZ_SLICE;
    uint32_t *ent = (uint32_t *)malloc(slice_cap * PZ_K * 4), *tok = (uint32_t *)malloc((slice_cap + 1) * 4), *best = (uint32_t *)malloc((n + 1) * 4);
    int *cnt = (int *)malloc(slice_cap * sizeof(int));
    size_t *segn = (size_t *)calloc(nseg, sizeof(size_t)), *segc = (size_t *)calloc(nseg, sizeof(size_t));
    for (size_t sl0 = 0; sl0 < n; sl0 += PZ_SLICE) {
        const size_t sl1 = sl0 + PZ_SLICE < n ? sl0 + PZ_SLICE : n;
        const size_t r0 = sl0 / PZ_REGION, r1 = (sl1 + PZ_REGION - 1) / PZ_REGION, g0 = sl0 / PZ_SEG, g1 = (sl1 + PZ_SEG - 1) / PZ_SEG;
        match_sets(s, n, bpp, stride, prev, sl0, sl1, ent, cnt);
        unsigned long long best_score = ~0ull;
        for (int it = 0; it < PZ_ITERS; it++) {
            for (size_t r = r0; r < r1; r++) pz_costs((it ? hprev : hg) + r * PZ_NSYM, cost + r * PZ_NSYM);
            memset(hcur + r0 * PZ_NSYM, 0, (r1 - r0) * PZ_NSYM * 4);
            for (size_t g = g0; g < g1; g++) {
                const size_t s0 = g * PZ_SEG, L = (s0 + PZ_SEG < n ? PZ_SEG : n - s0);
                segc[g] = squeeze(s, s0, L, ent + (s0 - sl0) * PZ_K, cnt + (s0 - sl0), cost + (s0 / PZ_REGION) * PZ_NSYM, tok + (s0 - sl0), hcur + (s0 / PZ_REGION) * PZ_NSYM);
            }
            unsigned long long sc = 0;
            for (size_t r = r0; r < r1; r++) sc += pz_score(hcur + r * PZ_NSYM);
            if (sc < best_score) {
                best_score = sc;
                for (size_t g = g0; g < g1; g++) { segn[g] = segc[g]; memcpy(best + g * PZ_SEG, tok + (g * PZ_SEG - sl0), segc[g] * 4); }
            }
            uint32_t *t = hprev; hprev = hcur; hcur = t;
        }
    }
    size_t nt = 0;
    for (size_t g = 0; g < nseg; g++) { memmove(tokens + nt, best + g * PZ_SEG, segn[g] * 4); nt += segn[g]; }
    free(hg); free(hprev); free(hcur); free(cost); free(prev); free(ent); free(tok); free(best); free(cnt); free(segn); free(segc);
    return nt;
}

/* ---- the pieces on their own, for the tests ---- */
/* one parse of the whole stream with one cost table for every segment (no iterations) */
size_t orc_pz_squeeze(const uint8_t *s, size_t n, int bpp, int stride, const uint32_t *cost, uint32_t *tokens)
{
    if (!n) return 0;
    int32_t *prev = hash_prev(s, n);
    uint32_t *ent = (uint32_t *)malloc(n * PZ_K * 4), h[PZ_NSYM];
    int *cnt = (int *)malloc(n * sizeof(int));
    match_sets(s, n, bpp, stride, prev, 0, n, ent, cnt);
    size_t nt = 0;
    for (size_t s0 = 0; s0 < n; s0 += PZ_SEG) nt += squeeze(s, s0, s0 + PZ_SEG < n ? PZ_SEG : n - s0, ent + s0 * PZ_K, cnt + s0, cost, tokens + nt, h);
    free(prev); free(ent); free(cnt);
    return nt;
}
/* the kept entries of every position: out[i * PZ_K ...], counts in cnt */
void orc_pz_match_sets(const uint8_t *s, size_t n, int bpp, int stride, uint32_t *out, int *cnt)
{
    int32_t *prev = hash_prev(s, n);
    match_sets(s, n, bpp, stride, prev, 0, n, out, cnt);
    free(prev);
}
/* the front rule on a candidate list given in increasing distance */
int orc_pz_front(const int *len, const int *dist, int m, uint32_t *out)
{
    PzFront f; pz_front_init(&f);
    for (int k = 0; k < m; k++) pz_front_add(&f, len[k], dist[k]);
    for (int k = 0; k < f.cnt; k++) out[k] = f.e[k];
    return f.cnt;
}
void orc_pz_costs(const uint32_t *h, uint32_t *cost) { pz_costs(h, cost); }
int orc_pz_constants(int *out)
{
    out[0] = PZ_SEG; out[1] = PZ_CHAIN; out[2] = PZ_K; out[3] = PZ_REGION; out[4] = PZ_ITERS; out[5] = PZ_SLICE;
    return 6;
}
