/* png_zopfli_core.h -- the rules of the PNG `--zopfli` leg (png_force_zopfli with the switch on), written once for every party that has
 * to agree on them: the device kernels and their host driver (png_zopfli.cu) and the scalar twin (oracle/png_zopfli_oracle.c, plain C
 * -- hence no namespace and no C++ in this file).  Everything that decides a token is integer arithmetic, so the parties agree bit for
 * bit and no thread order can change a result.
 *
 *   stream       the filtered PNG stream s[0, n); positions are cut into segments of PZ_SEG, segments into cost regions of PZ_REGION
 *                and regions into slices of PZ_SLICE (each a multiple of the one before, so no segment or region spans a slice)
 *   match set    of position i: every (length, distance) pair with length >= 3 among the candidates, where a length is the run of
 *                equal bytes s[i + k] == s[i + k - d], at most pz_maxlen(i) (258, and never past i's segment end), and a distance
 *                at most min(i, PZ_WINDOW) (a match may reach back into earlier segments and slices).  Candidates: the ten fixed
 *                pixel / row distances of png_match_core.h, then -- unless a fixed candidate already reaches pz_maxlen(i) -- the
 *                nearest PZ_CHAIN earlier positions j with pz_hash3(j) == pz_hash3(i) and i - j <= PZ_WINDOW (hash collisions count
 *                toward PZ_CHAIN).  The set kept is the Pareto front: no kept pair has another candidate with a length at least as
 *                long and a distance at most as short (so, by increasing distance, strictly increasing lengths).  A front of more
 *                than PZ_K pairs keeps its PZ_K - 1 smallest distances and its longest pair: every length up to the longest stays
 *                reachable.  An entry is packed as (length - 3) << 16 | (distance - 1).
 *   costs        in 1024ths of a bit, per cost region, from a token histogram h (316 counters: 286 literal / length symbols, 30
 *                distance symbols, the end of block not counted).  With T the total of h's side (literal / length or distance),
 *                symbol x costs log2q(T) - log2q(h[x]), or log2q(T) + 1024 when h[x] = 0, clamped to [1024, 15 * 1024], plus 1024
 *                per extra bit of x; log2q = pz_log2_q10 (log2q(0) is taken as log2q(1)).  A literal costs its symbol; a match of
 *                length l at distance d costs its length symbol plus its distance symbol.  Iteration 1 takes h from the region's
 *                tokens of the greedy / lazy parse of the same stream (png_kernels.cu k_png_parse); iteration k + 1 from iteration
 *                k's parse.
 *   parse        of one segment: the cheapest path from its start to its end over literal edges (i -> i + 1) and match edges
 *                (i -> i + l for l = 3 .. the longest kept length of i; the edge costs the minimum over the kept entries at least
 *                l long, ties to the smaller distance).  Sources are relaxed in increasing order and a target's cost changes only
 *                on a strictly smaller value, so among equal paths the one whose last token starts earliest wins.
 *   score        of a parse: the sum over its regions of sum_x h[x] * cost_h[x], each region's histogram under its own cost table.
 *                Of the PZ_ITERS parses of a slice the lowest score wins, ties to the earlier iteration.
 *   tokens       the format of b200_png_lz77: a literal is its byte, a match 0x80000000 | entry. */
#ifndef PNG_ZOPFLI_CORE_H
#define PNG_ZOPFLI_CORE_H
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define PZ_HD static __host__ __device__ __forceinline__
#else
#define PZ_HD static inline
#endif

/* one warp parses one segment; 32 KiB keeps a segment's back-pointers and tokens in one 128 KiB stretch and gives a 4096 x 4096 RGBA
 * stream 2,049 independent warps, while its paths are long enough that the cut at its end costs under a token */
#define PZ_SEG 32768
/* hash-chain depth: far enough down the chain to find the repeats of text and flat art (zlib 9 walks 4096, but its greedy parse
 * needs the single longest match; the optimal parse gains most from the near ones); each step is one byte compare loop */
#define PZ_CHAIN 32
/* entries kept per position: the match-set storage is PZ_K words per position (PZ_K * 4 bytes per position of a slice) */
#define PZ_K 8
/* cost-region length: symbol statistics drift across an image; 256 KiB is four DEFLATE blocks of 65,536 tokens at ~1 byte per token */
#define PZ_REGION 262144
/* iterations of cost re-estimation and parsing: oxipng's zopfli setting */
#define PZ_ITERS 15
/* slice length: the match sets, back-pointers and hash-chain sort of one slice are resident at a time, so device memory is
 * O(PZ_SLICE), not O(n) (about 60 bytes per position) */
#define PZ_SLICE 8388608
/* DEFLATE's window: the largest distance */
#define PZ_WINDOW 32768
#define PZ_MAXLEN 258
#define PZ_NSYM 316
#define PZ_NONE 0xFFFFFFFFu                 /* an empty entry slot (no packed entry reaches it: length - 3 <= 255) */
#define PZ_NOHASH 0x10000u                  /* the hash key of a position with fewer than three bytes left */

/* 1024 * log2(x), piecewise linear between powers of two (exact at them, at most 0.09 low in between); x >= 1.  Also behind the
 * greedy parse's hash_cost_tables (png_kernels.cu). */
PZ_HD uint32_t pz_log2_q10(unsigned long long x)
{
    int e = 63; while (!((x >> e) & 1ull)) e--;
    const unsigned long long frac = e >= 10 ? (x >> (e - 10)) & 1023ull : (x << (10 - e)) & 1023ull;
    return (uint32_t)e * 1024u + (uint32_t)frac;
}

PZ_HD uint32_t pz_hash3(const uint8_t *p) { return (((uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16)) * 2654435761u) >> 16; }

PZ_HD int pz_hibit(uint32_t v) { int b = 31; while (!((v >> b) & 1u)) b--; return b; }
/* RFC 1951 3.2.5: length code 257 + pz_len_symbol(len), distance code pz_dist_symbol(d) */
PZ_HD int pz_len_symbol(int len)
{
    if (len == 258) return 28;
    if (len < 11) return len - 3;
    { const int l = len - 3, hb = pz_hibit((uint32_t)l); return (hb - 1) * 4 + ((l >> (hb - 2)) & 3); }
}
PZ_HD int pz_dist_symbol(int d)
{
    if (d <= 4) return d - 1;
    { const int v = d - 1, hb = pz_hibit((uint32_t)v); return hb * 2 + ((v >> (hb - 1)) & 1); }
}
PZ_HD int pz_len_extra(int ls) { return ls < 8 || ls == 28 ? 0 : (ls >> 2) - 1; }
PZ_HD int pz_dist_extra(int ds) { return ds < 4 ? 0 : (ds >> 1) - 1; }

PZ_HD uint32_t pz_pack(int len, int d) { return ((uint32_t)(len - 3) << 16) | (uint32_t)(d - 1); }
PZ_HD int pz_elen(uint32_t e) { return (int)(e >> 16) + 3; }
PZ_HD int pz_edist(uint32_t e) { return (int)(e & 0xFFFFu) + 1; }

/* the longest match position i may take: 258, never past its segment's end */
PZ_HD int pz_maxlen(size_t i, size_t n)
{
    size_t end = (i / PZ_SEG + 1) * (size_t)PZ_SEG;
    if (end > n) end = n;
    return end - i > PZ_MAXLEN ? PZ_MAXLEN : (int)(end - i);
}

PZ_HD int pz_match_len(const uint8_t *s, size_t i, int d, int maxlen)
{
    int l = 0;
    while (l < maxlen && s[i + l] == s[i + l - d]) l++;
    return l;
}

/* png_match_core.h's ten candidate distances, sorted ascending (insertion sort; duplicates and unusable ones stay) */
PZ_HD void pz_fixed_sorted(int bpp, int stride, int cand[10])
{
    const int c0[10] = {bpp, 1, 2 * bpp, stride, stride - bpp, stride + bpp, 3 * bpp, 2, 3, 2 * stride};
    for (int a = 0; a < 10; a++) {
        int b = a; const int v = c0[a];
        while (b > 0 && cand[b - 1] > v) { cand[b] = cand[b - 1]; b--; }
        cand[b] = v;
    }
}

/* The front under construction: candidates arrive in increasing distance, so a candidate is on the front iff it is longer than
 * every one before it; the first PZ_K - 1 such records stay, and the last slot holds the latest (the longest). */
typedef struct { uint32_t e[PZ_K]; int n, cnt, top; } PzFront;
PZ_HD void pz_front_init(PzFront *f) { f->n = 0; f->cnt = 0; f->top = 2; }
PZ_HD void pz_front_add(PzFront *f, int len, int d)
{
    if (len <= f->top) return;
    f->top = len;
    if (f->n < PZ_K - 1) { f->e[f->n++] = pz_pack(len, d); f->cnt = f->n; }
    else { f->e[PZ_K - 1] = pz_pack(len, d); f->cnt = PZ_K; }
}

/* The kept entries of position i (returns their number, entries by increasing distance).  prev[j - pbase] is the nearest earlier
 * position with j's hash (or -1) for every j the chain may visit; cand: pz_fixed_sorted. */
PZ_HD int pz_match_set(const uint8_t *s, size_t n, size_t i, const int cand[10], const int32_t *prev, long long pbase, uint32_t out[PZ_K])
{
    const int maxlen = pz_maxlen(i, n);
    if (maxlen < 3) return 0;
    const int reach = i > PZ_WINDOW ? PZ_WINDOW : (int)i;
    int flen[10], full = 0;
    for (int c = 0; c < 10; c++) {
        const int d = cand[c];
        flen[c] = d >= 1 && d <= reach ? pz_match_len(s, i, d, maxlen) : 0;
        full |= flen[c] == maxlen;
    }
    PzFront f; pz_front_init(&f);
    long long j = full ? -1 : prev[(long long)i - pbase];
    int c = 0, depth = 0;
    while (f.top < maxlen) {                 /* (a candidate after the front reached maxlen cannot be strictly longer) */
        const int dh = j >= 0 && depth < PZ_CHAIN && (long long)i - j <= PZ_WINDOW ? (int)((long long)i - j) : 0x7FFFFFFF;
        const int df = c < 10 ? cand[c] : 0x7FFFFFFF;
        if (dh == 0x7FFFFFFF && df == 0x7FFFFFFF) break;
        if (df <= dh) { if (flen[c] >= 3) pz_front_add(&f, flen[c], df); c++; }
        else { pz_front_add(&f, pz_match_len(s, i, dh, maxlen), dh); depth++; j = prev[j - pbase]; }
    }
    for (int k = 0; k < f.cnt; k++) out[k] = f.e[k];
    return f.cnt;
}

/* the cost table (316 entries, 1024ths of a bit, extra bits included) of histogram h */
PZ_HD void pz_costs(const uint32_t *h, uint32_t *cost)
{
    unsigned long long tl = 0, td = 0;
    for (int x = 0; x < 286; x++) tl += h[x];
    for (int x = 286; x < PZ_NSYM; x++) td += h[x];
    const uint32_t ll = pz_log2_q10(tl ? tl : 1), ld = pz_log2_q10(td ? td : 1);
    for (int x = 0; x < PZ_NSYM; x++) {
        const uint32_t lt = x < 286 ? ll : ld;
        uint32_t c = h[x] ? lt - pz_log2_q10(h[x]) : lt + 1024u;
        c = c < 1024u ? 1024u : c > 15u * 1024u ? 15u * 1024u : c;
        const int extra = x >= 286 ? pz_dist_extra(x - 286) : x >= 257 && x < 286 ? pz_len_extra(x - 257) : 0;
        cost[x] = c + 1024u * (uint32_t)extra;
    }
}
PZ_HD unsigned long long pz_score(const uint32_t *h)
{
    uint32_t cost[PZ_NSYM];
    pz_costs(h, cost);
    unsigned long long sc = 0;
    for (int x = 0; x < PZ_NSYM; x++) sc += (unsigned long long)h[x] * cost[x];
    return sc;
}

/* the cheapest match edge of length l from a position with entries e[0, cnt) (by increasing distance): its cost (length and
 * distance symbols) and token; the entries at least l long are a suffix, and a later (farther) one wins only when strictly cheaper */
PZ_HD uint32_t pz_edge(const uint32_t *e, int cnt, int l, const uint32_t *cost, uint32_t *tok)
{
    uint32_t best = 0xFFFFFFFFu; int bd = 0;
    for (int k = 0; k < cnt; k++) {
        if (pz_elen(e[k]) < l) continue;
        const int d = pz_edist(e[k]);
        const uint32_t c = cost[286 + pz_dist_symbol(d)];
        if (c < best) { best = c; bd = d; }
    }
    *tok = 0x80000000u | pz_pack(l, bd);
    return best + cost[257 + pz_len_symbol(l)];
}

/* the histogram of one token */
PZ_HD void pz_count(uint32_t *h, uint32_t tok)
{
    if (tok & 0x80000000u) { h[257 + pz_len_symbol(pz_elen(tok & 0x7FFFFFFFu))]++; h[286 + pz_dist_symbol(pz_edist(tok & 0x7FFFFFFFu))]++; }
    else h[tok]++;
}
#endif /* PNG_ZOPFLI_CORE_H */
