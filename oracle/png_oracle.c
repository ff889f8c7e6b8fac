/* png_oracle.c -- TEST INFRASTRUCTURE ONLY (never linked into or called by the product).
 *
 * CPU restatement of the lossless PNG leg of the hot path: libcaesium png::lossless -> oxipng::optimize_from_memory
 * (caesium-clt's src/compressor.rs:428 `parameters.png.optimize`, :436 `optimization_level`, :437 `force_zopfli`).
 * oxipng 9.x and libdeflate are Cargo dependencies that are NOT vendored under the caesium-clt sources, so this file restates
 * their published algorithms: the PNG filters (PNG spec 9.2), oxipng's per-row filter heuristics (RowFilter::MinSum,
 * Entropy, Bigrams, BigEnt; Brute is scored like Entropy -- documented deviation in DESIGN.md), and an LZ77 parse over a
 * fixed candidate set with zlib's one-step lazy evaluation.  Parity status: "pinned by losslessness" -- the product's
 * files must decode (Pillow/libpng, zlib) to exactly the source pixels, and the product's row-filter choices and tokens
 * must equal this file's; byte-identity with oxipng's own output is NOT claimed (libdeflate's optimal parser is not
 * restated).  Plain scalar C, one row / one position at a time, nothing shared with the CUDA sources.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { F_NONE, F_SUB, F_UP, F_AVG, F_PAETH, F_MINSUM, F_ENTROPY, F_BIGRAMS, F_BIGENT, F_BRUTE };

static int paeth(int a, int b, int c)
{
    int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    if (pa <= pb && pa <= pc) return a;
    return pb <= pc ? b : c;
}

/* PNG 9.2: filter one row with filter type f (0..4); prev == NULL for the first row (treated as zeros) */
static void filter_row(const uint8_t *row, const uint8_t *prev, int rb, int bpp, int f, uint8_t *out)
{
    for (int x = 0; x < rb; x++) {
        int a = x >= bpp ? row[x - bpp] : 0, b = prev ? prev[x] : 0, c = (prev && x >= bpp) ? prev[x - bpp] : 0, pred;
        switch (f) {
            case F_SUB: pred = a; break;
            case F_UP: pred = b; break;
            case F_AVG: pred = (a + b) / 2; break;
            case F_PAETH: pred = paeth(a, b, c); break;
            default: pred = 0;
        }
        out[x] = (uint8_t)(row[x] - pred);
    }
}

/* c * log2(c) in 1/1024 units, the integer table both sides score entropy with */
static uint64_t tlog(uint32_t c) { return c ? (uint64_t)llround((double)c * log2((double)c) * 1024.0) : 0; }

/* score of one filtered row under a heuristic; *larger_is_better tells the caller which way to compare */
static uint64_t row_score(const uint8_t *f, int rb, int strategy, int *larger_is_better)
{
    uint64_t s = 0;
    *larger_is_better = 0;
    if (strategy == F_MINSUM) {                       /* oxipng RowFilter::MinSum: sum |signed byte| */
        for (int x = 0; x < rb; x++) s += (uint64_t)abs((int)(int8_t)f[x]);
    } else if (strategy == F_ENTROPY || strategy == F_BRUTE) {   /* Shannon entropy of the bytes: max sum c log c */
        uint32_t cnt[256] = {0};
        for (int x = 0; x < rb; x++) cnt[f[x]]++;
        for (int v = 0; v < 256; v++) s += tlog(cnt[v]);
        *larger_is_better = 1;
    } else if (strategy == F_BIGRAMS) {               /* number of distinct byte pairs */
        uint8_t *seen = (uint8_t *)calloc(65536, 1);
        for (int x = 0; x + 1 < rb; x++) { unsigned bg = ((unsigned)f[x] << 8) | f[x + 1]; if (!seen[bg]) { seen[bg] = 1; s++; } }
        free(seen);
    } else {                                          /* BigEnt: entropy of byte pairs, pairs hashed into 4096 buckets */
        uint32_t *cnt = (uint32_t *)calloc(4096, 4);
        for (int x = 0; x + 1 < rb; x++) { uint32_t bg = ((uint32_t)f[x] << 8) | f[x + 1]; cnt[((bg * 2654435761u) >> 20) & 4095u]++; }
        for (int v = 0; v < 4096; v++) s += tlog(cnt[v] < (uint32_t)rb ? cnt[v] : (uint32_t)rb);
        free(cnt);
        *larger_is_better = 1;
    }
    return s;
}

/* raw [h][rb] -> out [h][rb + 1]; returns 0 */
int orc_png_filter(const uint8_t *raw, int h, int rb, int bpp, int strategy, uint8_t *out)
{
    uint8_t *cand = (uint8_t *)malloc((size_t)rb * 5 + 8);
    for (int y = 0; y < h; y++) {
        const uint8_t *row = raw + (size_t)y * rb, *prev = y ? row - rb : NULL;
        uint8_t *o = out + (size_t)y * (rb + 1);
        int f = strategy;
        if (strategy >= F_MINSUM) {
            uint64_t best = 0; int lib = 0; f = 0;
            for (int k = 0; k < 5; k++) {
                filter_row(row, prev, rb, bpp, k, cand + (size_t)k * rb);
                uint64_t sc = row_score(cand + (size_t)k * rb, rb, strategy, &lib);
                if (k == 0 || (lib ? sc > best : sc < best)) { best = sc; f = k; }      /* first of equals wins */
            }
        }
        o[0] = (uint8_t)f;
        filter_row(row, prev, rb, bpp, f, o + 1);
    }
    free(cand);
    return 0;
}

/* inverse (PNG 9.2 reconstruction), for the round-trip property tests */
int orc_png_unfilter(const uint8_t *filt, int h, int rb, int bpp, uint8_t *raw)
{
    for (int y = 0; y < h; y++) {
        const uint8_t *f = filt + (size_t)y * (rb + 1);
        uint8_t *row = raw + (size_t)y * rb, *prev = y ? row - rb : NULL;
        if (f[0] > 4) return -1;
        for (int x = 0; x < rb; x++) {
            int a = x >= bpp ? row[x - bpp] : 0, b = prev ? prev[x] : 0, c = (prev && x >= bpp) ? prev[x - bpp] : 0, pred = 0;
            switch (f[0]) { case 1: pred = a; break; case 2: pred = b; break; case 3: pred = (a + b) / 2; break; case 4: pred = paeth(a, b, c); break; default: break; }
            row[x] = (uint8_t)(f[1 + x] + pred);
        }
    }
    return 0;
}

/* ---- LZ77 ------------------------------------------------------------------------------------------------------- */
#define CHUNK 4096

static int len_symbol(int len)
{   /* RFC 1951 3.2.5 table, by search */
    static const int base[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
    int s = 28; while (base[s] > len) s--;
    return s;
}
static int dist_symbol(int d)
{
    static const int base[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
    int s = 29; while (base[s] > d) s--;
    return s;
}

/* longest match at position i among the candidate distances, confined to i's 4 KiB chunk; candidates are visited in a
 * fixed order and a later one must be strictly longer to replace an earlier one */
static uint32_t best_match(const uint8_t *s, size_t n, size_t i, int bpp, int stride)
{
    size_t chunk_end = (i / CHUNK + 1) * (size_t)CHUNK; if (chunk_end > n) chunk_end = n;
    int maxlen = chunk_end - i > 258 ? 258 : (int)(chunk_end - i);
    int bl = 0, bd = 0;
    if (maxlen < 3) return 0;
    const int cand[10] = {bpp, 1, 2 * bpp, stride, stride - bpp, stride + bpp, 3 * bpp, 2, 3, 2 * stride};
    for (int c = 0; c < 10; c++) {
        int d = cand[c], l = 0;
        if (d < 1 || d > 32768 || (size_t)d > i) continue;
        while (l < maxlen && s[i + l] == s[i + l - d]) l++;
        if (l > bl) { bl = l; bd = d; }
        if (bl == maxlen) break;
    }
    return bl >= 3 ? ((uint32_t)bl << 16) | (uint32_t)bd : 0;
}

/* Matches at arbitrary distances: zlib-style hash chains over the next three bytes, confined to segments of 16,384 positions
 * (a chain never crosses a segment start), at most the 4 nearest earlier positions with the same hash; a chain candidate replaces
 * the fixed-candidate result only when it is strictly longer.  (The device builds the same chains by sorting (hash, position)
 * pairs per segment -- caesium-clt_b200/csrc/png_kernels.cu k_png_hashmatch.) */
#define HM_SEG 16384
#define HM_DEPTH 4
#define COSTF 1280u          /* 1.25 x 1024 */
/* 1024 * log2(x), piecewise linear between powers of two; x >= 1 (the product's log2_q10) */
static uint32_t log2_q10(unsigned long long x)
{
    int e = 63; while (!((x >> e) & 1ull)) e--;
    unsigned long long frac = e >= 10 ? (x >> (e - 10)) & 1023ull : (x << (10 - e)) & 1023ull;
    return (uint32_t)e * 1024u + (uint32_t)frac;
}
/* What a hash match must be worth: the order-0 cost (1024ths of a bit) of every byte value of this stream, and the cost of a match
 * per distance code (7 bits of length code + 5 of distance code + the extra bits, x 1.25).  A candidate is accepted when the
 * literals it replaces would cost at least that much. */
static void hash_cost_tables(const uint8_t *s, size_t n, uint32_t *litcost /*256*/, uint32_t *matchcost /*30*/)
{
    uint32_t hist[256]; memset(hist, 0, sizeof hist);
    for (size_t i = 0; i < n; i++) hist[s[i]]++;
    uint32_t ln = log2_q10(n ? n : 1);
    for (int v = 0; v < 256; v++) { uint32_t c = hist[v] ? ln - log2_q10(hist[v]) : 16 * 1024; litcost[v] = c < 256 ? 256 : c; }
    for (int ds = 0; ds < 30; ds++) matchcost[ds] = (uint32_t)(7 + 5 + (ds < 4 ? 0 : (ds >> 1) - 1)) * COSTF;
}

static void hash_chain_matches(const uint8_t *s, size_t n, uint32_t *best)
{
    uint32_t litcost[256], matchcost[30]; hash_cost_tables(s, n, litcost, matchcost);
    int32_t *head = (int32_t *)malloc(65536 * 4), *prev = (int32_t *)malloc(HM_SEG * 4);
    for (size_t seg0 = 0; seg0 < n; seg0 += HM_SEG) {
        memset(head, 0xFF, 65536 * 4);
        size_t seg_end = seg0 + HM_SEG < n ? seg0 + HM_SEG : n;
        for (size_t i = seg0; i < seg_end; i++) {
            if (i + 3 > n) break;
            uint32_t h = (((uint32_t)s[i] | ((uint32_t)s[i + 1] << 8) | ((uint32_t)s[i + 2] << 16)) * 2654435761u) >> 16;
            size_t chunk_end = (i / CHUNK + 1) * (size_t)CHUNK; if (chunk_end > n) chunk_end = n;
            int maxlen = chunk_end - i > 258 ? 258 : (int)(chunk_end - i);
            if (maxlen >= 3) {
                int bl = (int)(best[i] >> 16), bd = (int)(best[i] & 0xFFFF);
                int32_t q = head[h];
                for (int c = 0; c < HM_DEPTH && q >= 0 && bl < maxlen; c++, q = prev[q]) {
                    int d = (int)(i - seg0) - q, l = 0;
                    while (l < maxlen && s[i + l] == s[i + l - d]) l++;
                    if (l > bl && l >= 4) {      /* the literals it replaces must cost at least what the match costs */
                        uint32_t worth = 0, need = matchcost[dist_symbol(d)];
                        for (int k = 0; k < l && worth < need; k++) worth += litcost[s[i + k]];
                        if (worth >= need) { bl = l; bd = d; }
                    }      /* far matches must be long enough to pay for their distance code */
                }
                best[i] = bl >= 3 ? ((uint32_t)bl << 16) | (uint32_t)bd : 0;
            }
            prev[i - seg0] = head[h]; head[h] = (int32_t)(i - seg0);
        }
    }
    free(head); free(prev);
}

/* tokens must hold n entries; hist 316 counters (286 litlen + 30 dist; end-of-block not counted); returns token count */
size_t orc_png_lz77(const uint8_t *s, size_t n, int bpp, int stride, uint32_t *tokens, uint32_t *hist)
{
    size_t nt = 0;
    memset(hist, 0, 316 * 4);
    uint32_t *best = (uint32_t *)malloc((n + 1) * 4);
    for (size_t i = 0; i < n; i++) best[i] = best_match(s, n, i, bpp, stride);
    hash_chain_matches(s, n, best);
    for (size_t begin = 0; begin < n; begin += CHUNK) {
        size_t end = begin + CHUNK < n ? begin + CHUNK : n, i = begin;
        while (i < end) {
            int len = (int)(best[i] >> 16), d = (int)(best[i] & 0xFFFF);
            if (len == 3 && d > 4096) len = 0;                                  /* zlib TOO_FAR */
            if (len >= 3 && i + 1 < end && (int)(best[i + 1] >> 16) > len) len = 0;   /* lazy: defer to a longer match one byte on */
            if (len >= 3) { tokens[nt++] = 0x80000000u | ((uint32_t)(len - 3) << 16) | (uint32_t)(d - 1); hist[257 + len_symbol(len)]++; hist[286 + dist_symbol(d)]++; i += (size_t)len; }
            else { tokens[nt++] = s[i]; hist[s[i]]++; i++; }
        }
    }
    free(best);
    return nt;
}

/* expand tokens back to bytes (validates distances); returns produced length or (size_t)-1 */
size_t orc_png_expand(const uint32_t *tokens, size_t nt, uint8_t *out, size_t cap)
{
    size_t o = 0;
    for (size_t t = 0; t < nt; t++) {
        uint32_t v = tokens[t];
        if (v & 0x80000000u) {
            size_t len = ((v >> 16) & 0x7FFF) + 3, d = (v & 0xFFFF) + 1;
            if (d > o || o + len > cap || len > 258) return (size_t)-1;
            for (size_t k = 0; k < len; k++, o++) out[o] = out[o - d];
        } else { if (o >= cap || v > 255) return (size_t)-1; out[o++] = (uint8_t)v; }
    }
    return o;
}
