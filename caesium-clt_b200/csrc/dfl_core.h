// dfl_core.h -- the DEFLATE block coder of the lossless PNG path (libcaesium png::lossless -> oxipng -> deflate,
// caesium-clt's src/compressor.rs:428,436-437) written ONCE as __host__ __device__ code: png_host.cpp's deflate_tokens()
// (the CPU writer, and the twin the GPU tests compare against) and png_deflate.cu's kernels (the device writer) run the same
// bodies, so their output is identical bit for bit.  Per block of tokens: symbol statistics -> length-limited Huffman code
// lengths (limit 15, code-length code limit 7) -> canonical codes (stored bit-reversed for LSB-first output) -> the dynamic
// block header (RFC 1951 3.2.7, code lengths run-length coded) -> tokens.
//
// Code lengths: plain Huffman by the two-queue construction over the leaves sorted by (frequency, symbol) -- which pops exactly
// the nodes a binary heap ordered by (weight, creation index) would pop: leaves were created in symbol order, internal nodes
// in the order they are produced, and produced weights never decrease -- then the IJG / zlib overflow repair on the
// per-length counts, then the lengths are handed out by rank (most frequent first, ties to the lower symbol).
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define DFL_HD __host__ __device__ __forceinline__
#else
#define DFL_HD inline
#endif

namespace b200 {
namespace dfl {

constexpr int NLIT = 286, NDIST = 30, NCL = 19, MAXSYM = 288;

DFL_HD int len_base(int s)
{   // RFC 1951 3.2.5: base length of code 257 + s
    return s < 8 ? 3 + s : s == 28 ? 258 : 3 + ((4 + (s & 3)) << ((s >> 2) - 1));
}
DFL_HD int len_extra(int s) { return s < 8 || s == 28 ? 0 : (s >> 2) - 1; }
DFL_HD int dist_base(int s) { return s < 4 ? 1 + s : 1 + ((2 + (s & 1)) << ((s >> 1) - 1)); }
DFL_HD int dist_extra(int s) { return s < 4 ? 0 : (s >> 1) - 1; }
DFL_HD int hibit(unsigned v)
{
#if defined(__CUDA_ARCH__)
    return 31 - __clz((int)v);
#else
    return 31 - __builtin_clz(v);
#endif
}
DFL_HD int len_sym(int len)
{   // 3..258 -> 0..28
    if (len == 258) return 28;
    if (len < 11) return len - 3;
    const int l = len - 3, hb = hibit((unsigned)l);
    return (hb - 1) * 4 + ((l >> (hb - 2)) & 3);
}
DFL_HD int dist_sym(int d)
{   // 1..32768 -> 0..29
    const unsigned x = (unsigned)d - 1u;
    if (x < 4u) return (int)x;
    const int nb = hibit(x);
    return 2 * nb + (int)((x >> (nb - 1)) & 1u);
}

// ---- code lengths -------------------------------------------------------------------------------------------------------------
// scratch: order[n] (symbols), w[2n] (node weights), parent[2n]; all <= MAXSYM
struct HuffScratch { uint16_t order[MAXSYM]; uint64_t w[2 * MAXSYM]; int16_t parent[2 * MAXSYM]; uint8_t depth[2 * MAXSYM]; };

// the same for alphabets of up to N symbols (VP8L's green alphabet with a colour cache has up to 1304)
template <int N> struct HuffScratchN { uint16_t order[N]; uint64_t w[2 * N]; int16_t parent[2 * N]; uint8_t depth[2 * N]; };

// leaves (symbols with a non-zero count) sorted by (frequency, symbol) ascending into S.order; returns their number.  Insertion
// sort: m <= 286.  (The device sorts the litlen alphabet with the whole warp instead -- png_deflate.cu -- into the same order.)
template <class Scratch>
DFL_HD int huff_sort_leaves(const uint32_t *freq, int n, Scratch &S)
{
    int m = 0;
    for (int i = 0; i < n; i++) if (freq[i]) S.order[m++] = (uint16_t)i;
    for (int i = 1; i < m; i++) {
        const uint16_t s = S.order[i]; const uint32_t f = freq[s];
        int j = i - 1;
        while (j >= 0 && freq[S.order[j]] > f) { S.order[j + 1] = S.order[j]; j--; }       // stable: equal frequencies keep symbol order
        S.order[j + 1] = s;
    }
    return m;
}

// code lengths from the sorted leaves S.order[0 .. m)
template <class Scratch>
DFL_HD void huff_lengths_sorted(const uint32_t *freq, int n, int m, int limit, uint8_t *len, Scratch &S)
{
    for (int i = 0; i < n; i++) len[i] = 0;
    if (m == 0) return;
    if (m == 1) { len[S.order[0]] = 1; return; }
    for (int i = 0; i < m; i++) S.w[i] = freq[S.order[i]];
    // two queues: leaves [lq, m) and internal nodes [iq, next); on equal weight the leaf goes first (lower creation index)
    int lq = 0, iq = m, next = m;
    for (int k = 0; k < m - 1; k++) {
        int pick[2];
        for (int t = 0; t < 2; t++) {
            if (lq < m && (iq >= next || S.w[lq] <= S.w[iq])) pick[t] = lq++; else pick[t] = iq++;
        }
        S.w[next] = S.w[pick[0]] + S.w[pick[1]];
        S.parent[pick[0]] = (int16_t)next; S.parent[pick[1]] = (int16_t)next;
        next++;
    }
    const int root = next - 1;
    S.depth[root] = 0;
    int bl[64];
    for (int i = 0; i < 64; i++) bl[i] = 0;
    for (int i = root - 1; i >= 0; i--) {                 // parents have larger indices than their children
        const int d = S.depth[S.parent[i]] + 1;
        S.depth[i] = (uint8_t)(d > 63 ? 63 : d);
        if (i < m) bl[S.depth[i]]++;
    }
    for (int i = 63; i > limit; i--) while (bl[i] > 0) {
        int j = i - 2; while (bl[j] == 0) j--;
        bl[i] -= 2; bl[i - 1]++; bl[j + 1] += 2; bl[j]--;
    }
    // most frequent symbols get the shortest lengths; ties to the lower symbol: walk the (frequency, symbol)-ascending order from
    // the top, but inside a run of equal frequencies from its low-symbol end
    int k = m - 1, l = 1, left = bl[1];
    while (k >= 0) {
        int lo = k; const uint32_t f = freq[S.order[k]];
        while (lo > 0 && freq[S.order[lo - 1]] == f) lo--;
        for (int i = lo; i <= k; i++) {
            while (left == 0 && l < limit) { l++; left = bl[l]; }
            len[S.order[i]] = (uint8_t)l; left--;
        }
        k = lo - 1;
    }
}

template <class Scratch>
DFL_HD void huff_lengths(const uint32_t *freq, int n, int limit, uint8_t *len, Scratch &S)
{
    const int m = huff_sort_leaves(freq, n, S);
    huff_lengths_sorted(freq, n, m, limit, len, S);
}

DFL_HD void canon_codes(const uint8_t *len, int n, uint16_t *code)
{   // RFC 1951 3.2.2, stored bit-reversed for LSB-first output
    int cnt[16], next[16];
    for (int i = 0; i < 16; i++) cnt[i] = 0;
    for (int i = 0; i < n; i++) cnt[len[i]]++;
    cnt[0] = 0; int c = 0; next[0] = 0;
    for (int l = 1; l <= 15; l++) { c = (c + cnt[l - 1]) << 1; next[l] = c; }
    for (int i = 0; i < n; i++) {
        code[i] = 0;
        if (len[i]) {
            const int v = next[len[i]]++; int r = 0;
            for (int b = 0; b < len[i]; b++) if (v & (1 << b)) r |= 1 << (len[i] - 1 - b);
            code[i] = (uint16_t)r;
        }
    }
}

// ---- one block's tables ------------------------------------------------------------------------------------------------------
struct BlockTables {
    uint8_t ll[NLIT], dl[NDIST], cll[NCL];
    uint16_t lc[NLIT], dc[NDIST], clc[NCL];
    uint16_t hlit, hdist, hclen, ncl;
    uint8_t cls_sym[320], cls_extra[320];          // the run-length coded code-length sequence
    uint32_t header_bits;                           // 3 + 14 + 3 * hclen + the coded sequence
};

// lf[286] / df[30]: symbol counts of the block (lf[256], the end-of-block symbol, is counted here)
// litlen_sorted >= 0: S.order already holds the litlen leaves in sorted order (that many of them)
DFL_HD void build_block_tables(uint32_t *lf, const uint32_t *df, BlockTables &T, HuffScratch &S, int litlen_sorted = -1)
{
    const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    lf[256] = 1;
    if (litlen_sorted >= 0) huff_lengths_sorted(lf, NLIT, litlen_sorted, 15, T.ll, S); else huff_lengths(lf, NLIT, 15, T.ll, S);
    huff_lengths(df, NDIST, 15, T.dl, S);
    int ndist = 0; for (int i = 0; i < NDIST; i++) if (T.dl[i]) ndist++;
    if (ndist == 0) T.dl[0] = 1;                    // at least one distance code must be described
    canon_codes(T.ll, NLIT, T.lc); canon_codes(T.dl, NDIST, T.dc);
    int hlit = NLIT; while (hlit > 257 && !T.ll[hlit - 1]) hlit--;
    int hdist = NDIST; while (hdist > 1 && !T.dl[hdist - 1]) hdist--;
    // run-length code the two length arrays as one sequence (RFC 1951 3.2.7)
    uint32_t cf[NCL]; for (int i = 0; i < NCL; i++) cf[i] = 0;
    const int ns = hlit + hdist; int ncl = 0;
    auto at = [&](int i) -> int { return i < hlit ? T.ll[i] : T.dl[i - hlit]; };
    for (int i = 0; i < ns;) {
        const int v = at(i); int run = 1; while (i + run < ns && at(i + run) == v) run++;
        int left = run;
        if (v == 0) {
            while (left >= 11) { const int r = left < 138 ? left : 138; T.cls_sym[ncl] = 18; T.cls_extra[ncl++] = (uint8_t)(r - 11); cf[18]++; left -= r; }
            if (left >= 3) { T.cls_sym[ncl] = 17; T.cls_extra[ncl++] = (uint8_t)(left - 3); cf[17]++; left = 0; }
            while (left-- > 0) { T.cls_sym[ncl] = 0; T.cls_extra[ncl++] = 0; cf[0]++; }
        } else {
            T.cls_sym[ncl] = (uint8_t)v; T.cls_extra[ncl++] = 0; cf[v]++; left--;
            while (left >= 3) { const int r = left < 6 ? left : 6; T.cls_sym[ncl] = 16; T.cls_extra[ncl++] = (uint8_t)(r - 3); cf[16]++; left -= r; }
            while (left-- > 0) { T.cls_sym[ncl] = (uint8_t)v; T.cls_extra[ncl++] = 0; cf[v]++; }
        }
        i += run;
    }
    huff_lengths(cf, NCL, 7, T.cll, S); canon_codes(T.cll, NCL, T.clc);
    int hclen = NCL; while (hclen > 4 && !T.cll[order[hclen - 1]]) hclen--;
    T.hlit = (uint16_t)hlit; T.hdist = (uint16_t)hdist; T.hclen = (uint16_t)hclen; T.ncl = (uint16_t)ncl;
    uint32_t bits = 3 + 5 + 5 + 4 + 3 * (uint32_t)hclen;
    for (int i = 0; i < ncl; i++) { const int s = T.cls_sym[i]; bits += T.cll[s] + (s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0); }
    T.header_bits = bits;
}

// put(value, nbits): LSB-first, nbits <= 32
template <class Put>
DFL_HD void write_block_header(const BlockTables &T, bool final_block, Put &put)
{
    const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    put(final_block ? 1u : 0u, 1); put(2u, 2);
    put((uint32_t)(T.hlit - 257), 5); put((uint32_t)(T.hdist - 1), 5); put((uint32_t)(T.hclen - 4), 4);
    for (int i = 0; i < T.hclen; i++) put((uint32_t)T.cll[order[i]], 3);
    for (int i = 0; i < T.ncl; i++) {
        const int s = T.cls_sym[i];
        put((uint32_t)T.clc[s], T.cll[s]);
        if (s == 16) put((uint32_t)T.cls_extra[i], 2); else if (s == 17) put((uint32_t)T.cls_extra[i], 3); else if (s == 18) put((uint32_t)T.cls_extra[i], 7);
    }
}

// per-block emit tables: literal -> (code, bits); match length 3..258 -> code and extra bits as one piece (<= 20 bits);
// distance symbol -> code (extra bits are added per token)
struct EmitTables { uint32_t lit_cb[256], len_cb[256]; uint8_t lit_nb[256], len_nb[256]; uint16_t dc[NDIST]; uint8_t dl[NDIST]; uint16_t eob_code; uint8_t eob_len; };
DFL_HD void fill_emit_entry(const BlockTables &T, EmitTables &E, int i)
{   // i = 0..255: literal i and match length 3 + i
    E.lit_cb[i] = T.lc[i]; E.lit_nb[i] = T.ll[i];
    const int l = 3 + i, ls = len_sym(l), sym = 257 + ls;
    E.len_cb[i] = (uint32_t)T.lc[sym] | ((uint32_t)(l - len_base(ls)) << T.ll[sym]); E.len_nb[i] = (uint8_t)(T.ll[sym] + len_extra(ls));
    if (i < NDIST) { E.dc[i] = T.dc[i]; E.dl[i] = T.dl[i]; }
    if (i == 0) { E.eob_code = T.lc[256]; E.eob_len = T.ll[256]; }
}
// bits of one token, and the token as one LSB-first piece of at most 48 bits
DFL_HD uint32_t token_bits(const EmitTables &E, uint32_t t)
{
    if (!(t & 0x80000000u)) return E.lit_nb[t & 0xFF];
    const int li = (int)((t >> 16) & 0xFF), d = (int)(t & 0xFFFF) + 1, ds = dist_sym(d);
    return (uint32_t)E.len_nb[li] + E.dl[ds] + (uint32_t)dist_extra(ds);
}
DFL_HD uint64_t token_piece(const EmitTables &E, uint32_t t, uint32_t *nbits)
{
    if (!(t & 0x80000000u)) { *nbits = E.lit_nb[t & 0xFF]; return E.lit_cb[t & 0xFF]; }
    const int li = (int)((t >> 16) & 0xFF), d = (int)(t & 0xFFFF) + 1, ds = dist_sym(d);
    const uint64_t dpiece = (uint64_t)E.dc[ds] | ((uint64_t)(d - dist_base(ds)) << E.dl[ds]);                 // <= 15 + 13 bits
    *nbits = (uint32_t)E.len_nb[li] + E.dl[ds] + (uint32_t)dist_extra(ds);
    return (uint64_t)E.len_cb[li] | (dpiece << E.len_nb[li]);                                                   // <= 20 + 28 bits
}
DFL_HD void token_count(uint32_t t, uint32_t *lf, uint32_t *df)
{
    if (t & 0x80000000u) { lf[257 + len_sym((int)((t >> 16) & 0xFF) + 3)]++; df[dist_sym((int)(t & 0xFFFF) + 1)]++; } else lf[t & 0xFF]++;
}

} // namespace dfl
} // namespace b200
