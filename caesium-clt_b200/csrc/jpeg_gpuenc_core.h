// jpeg_gpuenc_core.h -- block-parallel formulation of the JPEG entropy ENCODER (jchuff.c / jcphuff.c semantics with
// optimised Huffman tables), written once as __host__ __device__ code: jpeg_gpuenc.cu wraps these bodies in CUDA
// kernels; tests/emul/ runs the very same bodies in plain loops on the CPU to validate the formulation without a GPU.
// This is SURVEY.md §8f rank 1 ("GPU-side Huffman encode"): it removes the host entropy-coding wall behind
// caesium::compress_in_memory (caesium-clt's src/compressor.rs:305).  Output bits are identical to jpeg_host.cpp's
// sequential writer (and therefore to oracle/jpeg_oracle.c).
//
// Formulation.  A scan is a sequence of blocks j = 0..n-1 in scan order.  Each block owns up to three consecutive
// pieces of the bitstream, [I_j][E_j][T_j]:
//   I_j  its inline symbols (DC difference; AC run/size symbols with ZRLs; in refinement scans each inline symbol is
//        followed by the correction bits that were pending inside the block),
//   E_j  an EOBn symbol, present iff j is the first block of an "EOB group" (its value is the group's block count),
//   T_j  the trailing correction bits of the block (refinement scans only) -- jcphuff.c buffers these (BE) and emits
//        them after the EOBn symbol of the group, which is exactly this order.
// A group ends before the next block that has inline symbols (it flushes the pending run first), after 0x7FFF blocks,
// or when more than MAX_CORR_BITS - DCTSIZE2 + 1 = 937 correction bits are pending (jcphuff.c emit_eobrun rules).
// Concatenating the pieces in block order reproduces the sequential encoder's output bit for bit.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define GE_HD __host__ __device__ __forceinline__
#else
#define GE_HD inline
#endif

namespace b200 {
namespace ge {

enum ScanMode { MODE_SEQ = 0, MODE_DC_FIRST = 1, MODE_AC_FIRST = 2, MODE_AC_REFINE = 3 };

constexpr int EOBRUN_MAX = 0x7FFF;
constexpr int CORR_FLUSH = 1000 - 64 + 1;      // flush when BE > 937

// One scan of one image.
struct Scan {
    const int16_t *coef;        // image base (zigzag blocks)
    int mode, ns, Ss, Se, Al;
    int comp[3];                // component indices in scan
    int hs[3], vs[3], bw[3];    // per component IN SCAN ORDER: sampling (interleaved only), allocated blocks per row
    long long comp_off[3];      // coefficient offset of the component, int16 units
    int tbl[3];                 // Huffman table id (0 luma / 1 chroma)
    int mcux, mcuy, blocks_per_mcu;   // interleaved geometry
    int rbw, rbh;               // single-component geometry (real blocks)
    int nblocks;                // units in this scan
    long long unit_base;        // index of unit 0 in the batch-wide per-unit arrays
    long long lu_base;          // ns > 1: index of unit 0 in the per-unit bit length / offset arrays (only these scans have them)
    int run_base, nruns;        // ns == 1 or a DC-first scan: the scan's first CTA run in the batch-wide run arrays, and its run count
    long long dc_base[3];       // DC-first scan with ns > 1: first entry of component i (scan order) in the batch-wide compact DC array
    int tab_base;              // index of this scan's first table in the batch-wide table array (4 per scan: [kind*2+tbl])
    long long word_base;        // first word of this scan's unstuffed bit buffer
    long long word_cap;         // capacity in 32-bit words
};

struct Table {                  // derived encoder table + the DHT payload
    uint32_t code_len[256];     // code << 8 | code length: one load per symbol in the length and emit passes (0: unused)
    uint8_t bits[17];
    uint8_t vals[256];
    int nvals;
};

// meta word per unit: bit0 event (has inline symbols), bit1 contributes to an EOB group, bits 8.. trailing correction bits
GE_HD uint32_t meta_pack(bool event, bool contrib, int tail) { return (event ? 1u : 0u) | (contrib ? 2u : 0u) | ((uint32_t)tail << 8); }
GE_HD bool meta_event(uint32_t m) { return m & 1u; }
GE_HD bool meta_contrib(uint32_t m) { return m & 2u; }
GE_HD int meta_tail(uint32_t m) { return (int)(m >> 8); }

GE_HD int nbits_of(unsigned v)
{
#if defined(__CUDA_ARCH__)
    return 32 - __clz((int)v);
#else
    return v ? 32 - __builtin_clz(v) : 0;
#endif
}

// scan-order unit -> block pointer, component slot i (index into Scan arrays) and, for DC coding, the previous block of
// the same component in scan order (nullptr at the start).
struct BlockRef { const int16_t *blk; const int16_t *prev; int slot; };

GE_HD BlockRef locate(const Scan &s, int u)
{
    BlockRef r;
    if (s.ns == 1) {
        const int row = u / s.rbw, col = u - row * s.rbw;
        const int16_t *base = s.coef + s.comp_off[0];
        r.blk = base + ((long long)row * s.bw[0] + col) * 64;
        r.slot = 0;
        if (u == 0) r.prev = nullptr;
        else { const int pu = u - 1, prow = pu / s.rbw, pcol = pu - prow * s.rbw; r.prev = base + ((long long)prow * s.bw[0] + pcol) * 64; }
        return r;
    }
    const int m = u / s.blocks_per_mcu;
    int q = u - m * s.blocks_per_mcu, i = 0;
    while (q >= s.hs[i] * s.vs[i]) { q -= s.hs[i] * s.vs[i]; i++; }
    const int my = m / s.mcux, mx = m - my * s.mcux;
    const int by = q / s.hs[i], bx = q - by * s.hs[i];
    const int16_t *base = s.coef + s.comp_off[i];
    r.slot = i;
    r.blk = base + ((long long)(my * s.vs[i] + by) * s.bw[i] + mx * s.hs[i] + bx) * 64;
    if (q > 0) { const int pq = q - 1, pby = pq / s.hs[i], pbx = pq - pby * s.hs[i]; r.prev = base + ((long long)(my * s.vs[i] + pby) * s.bw[i] + mx * s.hs[i] + pbx) * 64; }
    else if (m == 0) r.prev = nullptr;
    else { const int pm = m - 1, pmy = pm / s.mcux, pmx = pm - pmy * s.mcux; r.prev = base + ((long long)(pmy * s.vs[i] + s.vs[i] - 1) * s.bw[i] + pmx * s.hs[i] + s.hs[i] - 1) * 64; }
    return r;
}

// ---- bit masks over a block: bit k of mask(T) is set iff |coef[k]| >= T ----------------------------------------------
// The scans only ever ask "is |c| >> Al zero / one / more", i.e. threshold tests against 2^Al and 2^(Al+1); with the
// masks in hand every loop below visits the non-zero coefficients only (a handful per block) instead of all 63.
GE_HD int ctz64(unsigned long long m)
{
#if defined(__CUDA_ARCH__)
    return __ffsll((long long)m) - 1;
#else
    return __builtin_ctzll(m);
#endif
}
GE_HD int msb64(unsigned long long m)       // index of the highest set bit, -1 for 0
{
#if defined(__CUDA_ARCH__)
    return 63 - __clzll((long long)m);
#else
    return m ? 63 - __builtin_clzll(m) : -1;
#endif
}
GE_HD int popc64(unsigned long long m)
{
#if defined(__CUDA_ARCH__)
    return __popcll(m);
#else
    return __builtin_popcountll(m);
#endif
}
GE_HD unsigned long long band_mask(int Ss, int Se) { return (Se >= 63 ? ~0ull : ((1ull << (Se + 1)) - 1ull)) & ~((1ull << Ss) - 1ull); }

// Masks for the thresholds 1, 2 and 4: enough for first scans with Al <= 2 and refinement scans with Al <= 1 (the scripts
// in jpeg_scan_script use Al <= 1 / Al = 0).  One block read serves every scan that visits the block.
struct Masks3 { unsigned long long m[3]; };
GE_HD bool masks_cover(int mode, int Al) { return mode == MODE_AC_REFINE ? Al <= 1 : Al <= 2; }
// M.m[t] by selects: an array indexed with a runtime value would put the masks in local memory on the device
GE_HD unsigned long long mask_at(const Masks3 &M, int t) { return t == 0 ? M.m[0] : t == 1 ? M.m[1] : M.m[2]; }

// SWAR over the 32 coefficient pairs of a block (two int16 per 32-bit word, little endian): per word |c| of both halves,
// then for each threshold one add turns "half >= T" into bit 15 / bit 31, which is shifted onto the word's position in a
// 32-bit accumulator (even coefficients in the low half, odd ones in the high half); the two halves are interleaved once at
// the end.  ~600 integer operations per block instead of a compare-and-insert per coefficient and threshold.  The same code
// runs in the CPU emulation (tests/emul), so the bit tricks are covered without a GPU.
GE_HD uint32_t interleave16(uint32_t acc)       // bits 0..15 -> even positions, bits 16..31 -> odd positions
{
    uint32_t x = acc & 0xFFFFu, y = acc >> 16;
    x = (x | (x << 8)) & 0x00FF00FFu; x = (x | (x << 4)) & 0x0F0F0F0Fu; x = (x | (x << 2)) & 0x33333333u; x = (x | (x << 1)) & 0x55555555u;
    y = (y | (y << 8)) & 0x00FF00FFu; y = (y | (y << 4)) & 0x0F0F0F0Fu; y = (y | (y << 2)) & 0x33333333u; y = (y | (y << 1)) & 0x55555555u;
    return x | (y << 1);
}
GE_HD void masks_word(uint32_t w, int jj /*0..15: word inside its half*/, uint32_t (&acc)[3])
{
    const uint32_t sb = (w >> 15) & 0x00010001u;
    const uint32_t a = (w ^ (sb * 0xFFFFu)) + sb;                   // |lo| , |hi| (32768 for -32768): no carry between the halves
    const uint32_t pos = 0x00010001u << jj;
    acc[0] |= ((a + 0x7FFF7FFFu) >> (15 - jj)) & pos;              // half >= 1
    acc[1] |= (((a & 0xFFFEFFFEu) + 0x7FFF7FFFu) >> (15 - jj)) & pos;   // half >= 2
    acc[2] |= (((a & 0xFFFCFFFCu) + 0x7FFF7FFFu) >> (15 - jj)) & pos;   // half >= 4
}
GE_HD Masks3 make_masks3(const int16_t *__restrict__ blk)
{
    Masks3 M;
    uint32_t lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0};
#if defined(__CUDA_ARCH__)
    const uint4 *v = reinterpret_cast<const uint4 *>(blk);          // 8 x 128-bit loads
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const uint4 q = v[j];
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int i = 0; i < 4; i++) { if (j < 4) masks_word(w[i], (4 * j + i) & 15, lo); else masks_word(w[i], (4 * j + i) & 15, hi); }
    }
#else
    for (int j = 0; j < 32; j++) {
        const uint32_t w = (uint32_t)(uint16_t)blk[2 * j] | ((uint32_t)(uint16_t)blk[2 * j + 1] << 16);
        if (j < 16) masks_word(w, j, lo); else masks_word(w, j - 16, hi);
    }
#endif
    for (int t = 0; t < 3; t++) M.m[t] = ((unsigned long long)interleave16(hi[t]) << 32) | interleave16(lo[t]);
    return M;
}
// the definition the SWAR form is checked against in tests/emul: bit k of m[t] <=> |blk[k]| >= 2^t
inline Masks3 make_masks3_reference(const int16_t *blk)
{
    Masks3 M; M.m[0] = M.m[1] = M.m[2] = 0;
    for (int k = 0; k < 64; k++) { int a = blk[k]; if (a < 0) a = -a; for (int t = 0; t < 3; t++) if (a >= (1 << t)) M.m[t] |= 1ull << k; }
    return M;
}

// ---- classification (pass 0) ------------------------------------------------------------------------------------
// S: a Scan, or any descriptor with its mode, Ss, Se and Al (the device passes stage one per scan visit on chip)
template <class S>
GE_HD uint32_t classify_m(const S &s, const Masks3 &M)
{
    if (s.mode == MODE_SEQ || s.mode == MODE_DC_FIRST) return meta_pack(true, false, 0);
    const unsigned long long band = band_mask(s.Ss, s.Se);
    const unsigned long long mA = mask_at(M, s.Al) & band, mB = (s.mode == MODE_AC_REFINE ? mask_at(M, s.Al + 1) : 0ull) & band;
    if (s.mode == MODE_AC_FIRST) { const int last = msb64(mA); return meta_pack(last >= 0, last < s.Se, 0); }
    // AC refinement: inline symbols exist iff some coefficient becomes non-zero in this scan (|c| >> Al == 1).  After
    // the last such coefficient every remaining position is either zero (r++) or already non-zero (a pending correction
    // bit), so the block joins an EOB group (jcphuff.c: r > 0 || BR > 0) exactly when that coefficient is not at Se.
    const int last_new = msb64(mA & ~mB);
    int tail;                                   // already-non-zero coefficients after the last newly non-zero one
    if (last_new < 0) tail = popc64(mB);
    else if (last_new >= 63) tail = 0;
    else tail = popc64(mB & ~((2ull << last_new) - 1ull));
    return meta_pack(last_new >= 0, last_new < s.Se, tail);
}
// correction bits a block writes in a scan: one per coefficient of the band that was already non-zero (refinement scans only)
template <class S>
GE_HD int corr_bits_m(const S &s, const Masks3 &M)
{
    return s.mode == MODE_AC_REFINE ? popc64(mask_at(M, s.Al + 1) & band_mask(s.Ss, s.Se)) : 0;
}
GE_HD uint32_t classify(const Scan &s, const int16_t *blk)
{
    if (s.mode == MODE_SEQ || s.mode == MODE_DC_FIRST) return meta_pack(true, false, 0);
    return classify_m(s, make_masks3(blk));
}

// ---- symbol generation: one template, three sinks (histogram, length, emit) -----------------------------------------
// Sink interface: sym(kind /*0 DC,1 AC*/, tbl, symbol, nbits, extra) and raw(nbits, bits).
template <class Sink>
GE_HD void gen_dc(int value_shifted, int pred_shifted, int tbl, Sink &sk)
{
    int temp = value_shifted - pred_shifted, temp2 = temp;
    if (temp < 0) { temp = -temp; temp2--; }
    const int nb = nbits_of((unsigned)temp);
    sk.sym(0, tbl, nb, nb, (unsigned)temp2);
}

// The units of MCU m of a DC-first scan with ns > 1, in scan order, from the batch-wide compact DC array: component i of the scan
// has its DC coefficients at dc + s.dc_base[i], in MCU order, hs * vs per MCU, so the predecessor of every block is the entry
// before it (0 at the component's start).
template <class Sink>
GE_HD void gen_dc_mcu(const Scan &s, const int16_t *dc, int m, Sink &sk)
{
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int i = 0; i < 3; i++) {
        if (i >= s.ns) break;
        const int nb = s.hs[i] * s.vs[i];
        const int16_t *d = dc + s.dc_base[i] + (long long)m * nb;
        int prev = m ? d[-1] >> s.Al : 0;
        for (int q = 0; q < nb; q++) { const int v = d[q] >> s.Al; gen_dc(v, prev, s.tbl[i], sk); prev = v; }
    }
}

GE_HD int eob_symbol(unsigned count) { return (nbits_of(count) - 1) << 4; }     // EOBn: AC symbol of a group of `count` blocks
// The value bits that follow a Huffman symbol depend on the symbol alone: a DC symbol is its bit count; an AC run/size symbol
// carries `size` bits, EOBn (n << 4, n < 15) carries n, ZRL (0xF0) and EOB (0x00) none.  So a scan's size is
// sum(hist[symbol] * (code length + sym_extra_bits)) over its tables, plus the correction bits of a refinement scan.
GE_HD int sym_extra_bits(int kind, int symbol)
{
    if (kind == 0) return symbol;
    return (symbol & 15) ? (symbol & 15) : symbol == 0xF0 ? 0 : symbol >> 4;
}
template <class Sink>
GE_HD void gen_eob_token(unsigned count, int tbl, Sink &sk)
{
    sk.sym(1, tbl, eob_symbol(count), nbits_of(count) - 1, count);
}

// group_count: >0 iff this block opens an EOB group (then E_j carries that count).  The statistics pass runs it with
// group_count = 0: the inline symbols do not depend on the groups, and the EOBn symbols are counted where the groups are made.
// S as for classify_m; tbl = the block's Huffman table id, passed on to the sink.
template <class S, class Sink>
GE_HD void gen_block_m(const S &s, int tbl, const BlockRef &b, const Masks3 &M, unsigned group_count, Sink &sk)
{
    const int16_t *blk = b.blk;
    if (s.mode == MODE_DC_FIRST) { gen_dc(blk[0] >> s.Al, b.prev ? (b.prev[0] >> s.Al) : 0, tbl, sk); return; }
    if (s.mode == MODE_SEQ) {
        gen_dc(blk[0], b.prev ? b.prev[0] : 0, tbl, sk);
        int prevk = 0;
        for (unsigned long long m = M.m[0] & ~1ull; m; m &= m - 1) {
            const int k = ctz64(m);
            int r = k - prevk - 1; prevk = k;
            while (r > 15) { sk.sym(1, tbl, 0xF0, 0, 0); r -= 16; }
            int t = blk[k], t2 = t; if (t < 0) { t = -t; t2--; }
            const int nb = nbits_of((unsigned)t);
            sk.sym(1, tbl, (r << 4) + nb, nb, (unsigned)t2);
        }
        if (prevk != 63) sk.sym(1, tbl, 0, 0, 0);
        return;
    }
    const unsigned long long band = band_mask(s.Ss, s.Se);
    const unsigned long long mA = mask_at(M, s.Al) & band;                                              // |c| >= 2^Al
    const unsigned long long mB = (s.mode == MODE_AC_REFINE ? mask_at(M, s.Al + 1) : 0ull) & band;     // |c| >= 2^(Al+1)
    if (s.mode == MODE_AC_FIRST) {
        int prevk = s.Ss - 1;
        for (unsigned long long m = mA; m; m &= m - 1) {
            const int k = ctz64(m);
            int r = k - prevk - 1; prevk = k;
            while (r > 15) { sk.sym(1, tbl, 0xF0, 0, 0); r -= 16; }
            int t = blk[k], t2;
            if (t < 0) { t = (-t) >> s.Al; t2 = ~t; } else { t >>= s.Al; t2 = t; }
            const int nb = nbits_of((unsigned)t);
            sk.sym(1, tbl, (r << 4) + nb, nb, (unsigned)t2);
        }
        if (group_count) gen_eob_token(group_count, tbl, sk);
        return;
    }
    // MODE_AC_REFINE (jcphuff.c encode_mcu_AC_refine): pending correction bits are emitted right after each inline symbol.
    // mA & ~mB = coefficients that become non-zero in this scan, mB = already non-zero ones (one correction bit each).
    const unsigned long long newm = mA & ~mB;
    const int last_new = msb64(newm);
    const int EOB = last_new < 0 ? 0 : last_new;
    int r = 0, prevk = s.Ss - 1;
    int npend = 0; unsigned long long pend64 = 0;   // pending correction bits of this block (at most 63)
    for (unsigned long long m = mA; m; m &= m - 1) {
        const int k = ctz64(m);
        r += k - prevk - 1; prevk = k;
        while (r > 15 && k <= EOB) {
            sk.sym(1, tbl, 0xF0, 0, 0); r -= 16;
            if (npend) { sk.raw64(npend, pend64); npend = 0; pend64 = 0; }
        }
        int t = blk[k];
        const bool neg = t < 0;
        if (neg) t = -t;
        t >>= s.Al;
        if ((mB >> k) & 1ull) { pend64 = (pend64 << 1) | (unsigned)(t & 1); npend++; continue; }
        sk.sym(1, tbl, (r << 4) + 1, 1, neg ? 0u : 1u);
        if (npend) { sk.raw64(npend, pend64); npend = 0; pend64 = 0; }
        r = 0;
    }
    if (group_count) gen_eob_token(group_count, tbl, sk);
    if (npend) sk.raw64(npend, pend64);         // T_j: trailing correction bits, after the group's EOBn symbol
}
template <class Sink>
GE_HD void gen_block(const Scan &s, const BlockRef &b, unsigned group_count, Sink &sk)
{
    if (s.mode == MODE_DC_FIRST) { Masks3 none; none.m[0] = none.m[1] = none.m[2] = 0; gen_block_m(s, s.tbl[b.slot], b, none, group_count, sk); return; }
    gen_block_m(s, s.tbl[b.slot], b, make_masks3(b.blk), group_count, sk);
}

// ---- sinks --------------------------------------------------------------------------------------------------------
// Where the length and emit sinks find a symbol's `code << 8 | length` word (only the low byte, the length, for LenSink):
// ScanTabs looks it up in a scan's four Tables by kind and table id; KindTabs in one array per kind, the table id being
// fixed by the caller (the device passes stage the tables of a CTA's scan visits in shared memory this way).
struct ScanTabs {
    const Table *t = nullptr;
    ScanTabs() = default;
    GE_HD ScanTabs(const Table *p) : t(p) {}
    GE_HD uint32_t operator()(int kind, int tbl, int symbol) const { return t[kind * 2 + tbl].code_len[symbol]; }
};
template <class T>
struct KindTabs {
    T *dc, *ac;                 // T = const element type for lookups, a counter type for the statistics pass
    GE_HD uint32_t operator()(int kind, int, int symbol) const { return (kind ? ac : dc)[symbol]; }
};

template <class AddFn>
struct HistSink {               // add(index) must increment counter [kind*2 + tbl][symbol] (atomically on the device)
    AddFn add;
    GE_HD explicit HistSink(AddFn f) : add(f) {}
    GE_HD void sym(int kind, int tbl, int symbol, int, unsigned) { add((kind * 2 + tbl) * 256 + symbol); }
    GE_HD void raw64(int, unsigned long long) {}
};

template <class Tabs = ScanTabs>
struct LenSinkT {
    Tabs tabs;
    unsigned long long bits = 0;
    GE_HD void sym(int kind, int tbl, int symbol, int nb, unsigned) { bits += (tabs(kind, tbl, symbol) & 0xFFu) + nb; }
    GE_HD void raw64(int nb, unsigned long long) { bits += nb; }
};
using LenSink = LenSinkT<>;

GE_HD uint32_t shl_or_zero(uint32_t v, int s)      // v << s for s in [0, 32]
{
#if defined(__CUDA_ARCH__)
    return __funnelshift_lc(0u, v, (unsigned)s);
#else
    return s >= 32 ? 0u : v << s;
#endif
}

// MSB-first bit writer into a zero-initialised word buffer.  `cur` holds the n < 32 bits of the current word left-aligned
// (the first word starts with the previous block's n bits as zeros).  Only the first and the last word of a block's range can
// be shared with a neighbouring block: the first completed word and the one finish() writes go through `orw(word_index,
// value)`, which must OR atomically on the device; every completed word after the first is the block's own and is stored
// with `stw`.  A caller that writes the blocks one after another may pass its OR function for both.
template <class OrFn, class StFn = OrFn, class Tabs = ScanTabs>
struct EmitSink {
    Tabs tabs;
    OrFn orw;
    StFn stw;
    long long wpos, first;      // next word index, the block's first word
    uint32_t cur = 0; int n;
    GE_HD EmitSink(Tabs t, OrFn f, StFn g, long long word_base, unsigned long long bitoff)
        : tabs(t), orw(f), stw(g), wpos(word_base + (long long)(bitoff >> 5)), first(wpos), n((int)(bitoff & 31)) {}
    GE_HD EmitSink(Tabs t, OrFn f, long long word_base, unsigned long long bitoff) : EmitSink(t, f, f, word_base, bitoff) {}
    GE_HD void put(uint32_t code, int len)          // the low len bits of code (len <= 32, nothing above them set)
    {
        if (!len) return;
        const int fill = n + len;
        if (fill < 32) { cur |= code << (32 - fill); n = fill; return; }
        const int r = fill - 32;                    // bits of code left over for the next word
        const uint32_t w = cur | (code >> r);
        if (wpos == first) orw(wpos, w); else stw(wpos, w);
        wpos++;
        cur = shl_or_zero(code, 32 - r); n = r;
    }
    GE_HD void sym(int kind, int tbl, int symbol, int nb, unsigned extra)
    {
        // code and value bits leave as one piece: at most 16 + 16 bits
        const uint32_t e = tabs(kind, tbl, symbol);
        put(((e >> 8) << nb) | (extra & ((1u << nb) - 1u)), (int)(e & 0xFFu) + nb);
    }
    GE_HD void raw64(int nb, unsigned long long v)
    {
        if (nb > 32) { put((unsigned)(v >> 32), nb - 32); put((unsigned)v, 32); } else put((unsigned)v, nb);   // v < 2^nb
    }
    GE_HD void finish() { if (n > 0) orw(wpos, cur); }
    GE_HD unsigned long long bits_written(long long word_base) const { return (unsigned long long)(wpos - word_base) * 32 + n; }   // from a word-aligned start
};

// Copies bits [0, nbits) of the MSB-first word sequence src(0), src(1), ... (nothing set past nbits) to bit `bitoff` of a
// zero-initialised word buffer.  Destination words k = k0, k0 + dk, ... of the range are produced: the first and the last, which a
// neighbouring range may share, go through orw (atomic on the device), the others through stw.
template <class Src, class OrFn, class StFn>
GE_HD void place_bits(Src src, unsigned long long nbits, unsigned long long bitoff, OrFn &&orw, StFn &&stw, int k0 = 0, int dk = 1)
{
    if (!nbits) return;
    const int s = (int)(bitoff & 31);
    const long long w0 = (long long)(bitoff >> 5), nsrc = (long long)((nbits + 31) / 32), nout = (long long)((s + nbits + 31) / 32);
    for (long long k = k0; k < nout; k += dk) {
        const uint32_t hi = k > 0 ? src(k - 1) : 0u, lo = k < nsrc ? src(k) : 0u;
        const uint32_t v = s ? (hi << (32 - s)) | (lo >> s) : lo;
        if (k == 0 || k == nout - 1) { if (v) orw(w0 + k, v); }
        else stw(w0 + k, v);
    }
}

// ---- EOB groups (pass "groups"): called for every event unit b and once for b == nblocks (end of scan) -------------
// prev_ev = index of the last event unit before b (-1 if none); meta/tsum are the scan's per-unit arrays (tsum =
// exclusive prefix sum of trailing correction bits); writes gcount[j] = block count of the group opened at j, and calls
// counted(count) once per group, on the common path and on the overflow replay alike (the caller counts the EOBn symbol).
struct NoCount { GE_HD void operator()(uint32_t) const {} };
template <class CountFn = NoCount>
GE_HD void assign_groups(const uint32_t *meta, const uint32_t *tsum, int nblocks, int prev_ev, int b, uint32_t *gcount, CountFn &&counted = CountFn())
{
    auto group = [&](int j, uint32_t c) { gcount[j] = c; counted(c); };
    int gs = prev_ev < 0 ? 0 : (meta_contrib(meta[prev_ev]) ? prev_ev : prev_ev + 1);   // first contributor of the run
    if (gs >= b) return;
    const int count = b - gs;
    const uint32_t tend = b < nblocks ? tsum[b] : tsum[nblocks - 1] + (uint32_t)meta_tail(meta[nblocks - 1]);
    const uint32_t tailbits = tend - tsum[gs];          // modular difference: exact while a run holds < 2^32 bits
    if (count < EOBRUN_MAX && tailbits <= (uint32_t)CORR_FLUSH) { group(gs, (uint32_t)count); return; }
    // rare: the run overflows a counter; replay jcphuff.c's sequential rule over it
    int start = gs, n = 0; unsigned be = 0;
    for (int j = gs; j < b; j++) {
        n++; be += (unsigned)meta_tail(meta[j]);
        if (n == EOBRUN_MAX || be > (unsigned)CORR_FLUSH) { group(start, (uint32_t)n); start = j + 1; n = 0; be = 0; }
    }
    if (n > 0) group(start, (uint32_t)n);
}

// ---- jchuff.c jpeg_gen_optimal_table + jpeg_make_c_derived_tbl (single-thread form; freq has 256 entries) ------------
GE_HD void build_table(const uint32_t *freq_in, Table &t, int *codesize /*257*/, int *others /*257*/, long long *freq /*257*/)
{
    uint8_t bits[33];
    for (int i = 0; i < 33; i++) bits[i] = 0;
    for (int i = 0; i < 256; i++) { freq[i] = freq_in[i]; codesize[i] = 0; others[i] = -1; }
    freq[256] = 1; codesize[256] = 0; others[256] = -1;
    for (;;) {
        int c1 = -1, c2 = -1; long long v = 1000000000LL;
        for (int i = 0; i <= 256; i++) if (freq[i] && freq[i] <= v) { v = freq[i]; c1 = i; }
        v = 1000000000LL;
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
    int i = 16; while (i > 0 && bits[i] == 0) i--;
    if (i > 0) bits[i]--;
    for (int k = 0; k < 17; k++) t.bits[k] = bits[k];
    int p = 0;
    for (int l = 1; l <= 32; l++) for (int s = 0; s <= 255; s++) if (codesize[s] == l) t.vals[p++] = (uint8_t)s;
    t.nvals = p;
    for (int s = 0; s < 256; s++) t.code_len[s] = 0;
    uint32_t code = 0; int k = 0;
    for (int l = 1; l <= 16; l++) { for (int n = 0; n < t.bits[l]; n++, k++) t.code_len[t.vals[k]] = (code++ << 8) | (uint32_t)l; code <<= 1; }
}

} // namespace ge
} // namespace b200
