// jpeg_gpudec_core.h -- parallel decoding of a baseline (sequential Huffman, single interleaved or single-component
// scan, no restart markers) JPEG entropy-coded segment, written as __host__ __device__ code shared by the CUDA kernels
// (jpeg_gpudec.cu) and the serial CPU emulation in tests/emul/.  This is the decode half of SURVEY.md §8f rank 1; it
// replaces the host's jdhuff.c-style loop in front of caesium::compress_in_memory (caesium-clt's src/compressor.rs:305).
//
// Method (self-synchronising Huffman decoding, Klein & Wiseman 2003; Weissenberger & Schmidt 2018): the unstuffed bit
// stream is cut into subsequences of SUBSEQ_BITS bits.  A decoder state is (p, k, b) = bit position of the next
// codeword, zigzag index inside the current block (0 = a DC symbol is next), index of the block inside its MCU.
//   round 0 : thread i decodes subsequence i from the guess (i * S, 0, 0) and records where and in which state it
//             leaves the subsequence (its "exit").
//   round r : thread i restarts from thread i-1's recorded exit and re-decodes; when nobody's exit changes the exits
//             are the true ones by induction from thread 0.  Huffman codes re-synchronise quickly on photographic
//             data, so a handful of rounds suffice; streams that do not converge within the round budget (degenerate
//             periodic content) are handed to the host decoder by the caller.
//   count   : blocks completed per subsequence -> exclusive prefix sum -> first block index of every subsequence.
//   write   : thread i decodes once more from its true state and stores the blocks that START in its subsequence, whole
//             (decode_owned_blocks), with the DC as the raw difference, which it also hands to the dc pass.
//   dc      : per-component prefix sum over the DC differences in scan order.
#pragma once
#include <cstdint>
#include "jpeg_gpuenc_core.h"      // ge::Scan / ge::locate: scan-order unit -> block address

namespace b200 {
namespace gd {

struct DecTable {               // one Huffman table, jdhuff.c form (jpeg_make_d_derived_tbl): the REFERENCE the kernel form is checked against
    uint16_t look[512];         // 9-bit lookahead: (len << 8) | symbol, 0 = code longer than 9 bits (or invalid)
    int32_t maxcode[18];        // maxcode[l] = largest code of length l (-1 if none); maxcode[17] = sentinel
    int32_t valoff[17];         // vals index = valoff[l] + code
    uint8_t vals[256];
};

struct DecState { uint32_t p; uint16_t k; uint16_t b; };   // 8 bytes

GE_HD bool same_state(const DecState &a, const DecState &b) { return a.p == b.p && a.k == b.k && a.b == b.b; }

// 32 bits of the unstuffed stream starting at bit position p (big-endian bit order).  The stream buffer is 4-byte
// aligned and followed by at least 8 bytes of 0xFF padding, so bits past the end read as 1s (a real block that needs them
// is flagged ANOM_END: the host decoder reads 0s there) and two aligned word loads always suffice.
GE_HD uint32_t load_be32(const uint8_t *__restrict__ s, uint32_t word)
{
    const uint32_t w = reinterpret_cast<const uint32_t *>(s)[word];
#if defined(__CUDA_ARCH__)
    return __byte_perm(w, 0, 0x0123);
#else
    return __builtin_bswap32(w);
#endif
}
GE_HD uint32_t peek32(const uint8_t *__restrict__ s, uint32_t /*nbits_total*/, uint32_t p)
{
    const uint32_t wi = p >> 5, sh = p & 31;
    const uint32_t w0 = load_be32(s, wi), w1 = load_be32(s, wi + 1);
    return sh ? (w0 << sh) | (w1 >> (32 - sh)) : w0;
}

// A bit pattern that is no code of the table decodes as "length NO_CODE_LEN, symbol 0": one bit longer than any real code, so
// it can never be mistaken for a 16-bit code of symbol 0x00, and it still moves an unsynchronised decoder forward.
constexpr int NO_CODE_LEN = 17;

// decode one Huffman symbol from the top bits of `bits` (32 valid bits); returns symbol, *len = code length (>= 1)
GE_HD int decode_symbol(const DecTable &t, uint32_t bits, int *len)
{
    const uint32_t e = t.look[bits >> 23];
    if (e) { *len = (int)(e >> 8); return (int)(e & 0xFF); }
    const int code16 = (int)(bits >> 16);
    for (int l = 10; l <= 16; l++) {
        const int c = code16 >> (16 - l);
        if (c <= t.maxcode[l]) { *len = l; return t.vals[(t.valoff[l] + c) & 0xFF]; }
    }
    *len = NO_CODE_LEN;         // invalid code (reachable while unsynchronised or on corrupt data)
    return 0;
}

// What the write pass reports about the stream, per image.  Each is something the host decoder (jpeg_host.cpp) handles
// differently from decode_subsequence, so a real block that meets one must be decoded on the host:
//   ANOM_CODE  no code of the table (the host refuses the file), or a DC category above 15 (the host reads 16+ bits)
//   ANOM_RUN   a coefficient run past index 63 (the host ends the block without reading the value's bits)
//   ANOM_END   the stream ends before the last block does (the host reads 0-bits past the end, the device 1-bits)
// Symbols decoded from the padding after the last real block are not checked: they are normal on every clean file.
enum : uint32_t { ANOM_CODE = 1u, ANOM_RUN = 2u, ANOM_END = 4u };
GE_HD uint32_t symbol_anomaly(int len, int sym, bool dc, int k, uint32_t p_next, uint32_t nbits)
{
    return (len == NO_CODE_LEN || (dc && sym > 15) ? ANOM_CODE : 0u) |
           (!dc && (sym & 15) && k + (sym >> 4) > 63 ? ANOM_RUN : 0u) |
           (p_next > nbits ? ANOM_END : 0u);
}

// Only a sink that wants the anomalies defines anomaly(mask); for the others (the round passes' block counters) the call and the
// mask computation vanish.
template <class Sink> GE_HD auto report_anomaly(Sink &sk, uint32_t m, int) -> decltype(sk.anomaly(m), void()) { sk.anomaly(m); }
template <class Sink> GE_HD void report_anomaly(Sink &, uint32_t, long) {}

struct Geometry {               // what the decoder needs to know about the scan
    int blocks_per_mcu;
    int dc_tbl[10], ac_tbl[10]; // Huffman table ids (0..3) used by block q of the MCU
    uint32_t total_blocks;      // blocks in the scan
    uint32_t nbits;             // length of the unstuffed stream in bits
    uint32_t subseq_bits;
    uint32_t nsub;              // number of subsequences
};

// ---- decode tables, kernel form --------------------------------------------------------------------------------------------
// All Huffman tables of one image, laid out for a loop-free symbol decode: a 9-bit first-level table per Huffman table
// that resolves every code of up to 9 bits in one read, and for each 9-bit prefix under which longer codes live a
// second-level table of 2^(Lmax - 9) entries (Lmax = longest code under that prefix) drawn from one shared pool.  Canonical
// codes put the long codes at the top of the code space, so only a handful of prefixes need a second level (Annex K luminance
// AC: 5 prefixes, < 300 entries).  Entry format, both levels: (code length << 8) | symbol; first level only: bit 15 set =
// "second level": bits 11..13 = index bits - 1, bits 0..10 = pool offset.  A bit pattern that is no code at all decodes as
// (NO_CODE_LEN, 0), exactly what the canonical jdhuff.c search (decode_symbol above) answers for it.
constexpr int LOOK_BITS = 9, LOOK_N = 1 << LOOK_BITS, MAX_TABLES = 8, EXT_N = 1536;
struct DecTables {
    uint16_t look[MAX_TABLES * LOOK_N];     // first level of table slot t at look[t * LOOK_N]
    uint16_t ext[EXT_N];                    // second-level pool
    uint16_t sel[20];                       // [2 * q + (AC ? 1 : 0)] -> first-level offset of block q's DC / AC table
    uint16_t nlook, next;                   // slots / pool entries in use (what has to be staged)
    uint16_t ok, pad_;                      // 0: the tables did not fit the pool (the image is decoded on the host instead)
};

// Build the kernel form from DHT payloads.  dht_bits[kind*4+id] / dht_vals[...] = BITS[17] / HUFFVAL of table (kind, id), null if
// absent; the scan's table use comes from g.dc_tbl / g.ac_tbl.  Returns false (and leaves a harmless table set of 16-bit skips)
// when the second-level pool would overflow or a DHT is over-subscribed.
inline bool build_dec_tables(const uint8_t *const dht_bits[8], const uint8_t *const dht_vals[8], const Geometry &g, DecTables &T)
{
    const uint16_t INVALID = (uint16_t)(NO_CODE_LEN << 8);
    for (int i = 0; i < MAX_TABLES * LOOK_N; i++) T.look[i] = INVALID;
    for (int i = 0; i < EXT_N; i++) T.ext[i] = INVALID;
    for (int i = 0; i < 20; i++) T.sel[i] = 0;
    T.nlook = 1; T.next = 0; T.ok = 0; T.pad_ = 0;
    int slot_of[8]; for (int i = 0; i < 8; i++) slot_of[i] = -1;
    int nslot = 0; bool ok = true;
    for (int q = 0; q < g.blocks_per_mcu && q < 10; q++) for (int ac = 0; ac < 2; ac++) {
        const int t = ac * 4 + ((ac ? g.ac_tbl[q] : g.dc_tbl[q]) & 3);
        if (slot_of[t] < 0) slot_of[t] = nslot++;
        T.sel[2 * q + ac] = (uint16_t)(slot_of[t] * LOOK_N);
    }
    uint32_t next = 0;
    for (int t = 0; t < 8 && ok; t++) {
        if (slot_of[t] < 0) continue;
        if (!dht_bits[t]) { ok = false; break; }
        uint16_t *look = T.look + slot_of[t] * LOOK_N;
        const uint8_t *bits = dht_bits[t], *vals = dht_vals[t];
        // pass 1: canonical codes; short ones fill the first level, long ones record the longest length per prefix
        uint8_t lmax[LOOK_N]; for (int i = 0; i < LOOK_N; i++) lmax[i] = 0;
        uint32_t code = 0; int p = 0;
        for (int l = 1; l <= 16 && ok; l++) {
            for (int i = 0; i < bits[l]; i++, p++, code++) {
                if (p >= 256 || code >= (1u << l)) { ok = false; break; }
                if (l <= LOOK_BITS) { const uint32_t first = code << (LOOK_BITS - l); for (uint32_t k = 0; k < (1u << (LOOK_BITS - l)); k++) look[first + k] = (uint16_t)((l << 8) | vals[p]); }
                else { const uint32_t pre = code >> (l - LOOK_BITS); if (lmax[pre] < l) lmax[pre] = (uint8_t)l; }
            }
            code <<= 1;
        }
        if (!ok) break;
        // pass 2: second-level tables
        for (int pre = 0; pre < LOOK_N; pre++) if (lmax[pre]) {
            const uint32_t nb = lmax[pre] - LOOK_BITS;
            if (next + (1u << nb) > (uint32_t)EXT_N || next > 0x7FFu) { ok = false; break; }
            look[pre] = (uint16_t)(0x8000u | ((nb - 1) << 11) | next);
            next += 1u << nb;
        }
        if (!ok) break;
        code = 0; p = 0;
        for (int l = 1; l <= 16; l++) {
            for (int i = 0; i < bits[l]; i++, p++, code++) if (l > LOOK_BITS) {
                const uint32_t pre = code >> (l - LOOK_BITS), e = look[pre], nb = ((e >> 11) & 7) + 1, off = e & 0x7FF;
                const uint32_t low = code & ((1u << (l - LOOK_BITS)) - 1), first = low << (LOOK_BITS + nb - l);
                for (uint32_t k = 0; k < (1u << (LOOK_BITS + nb - l)); k++) T.ext[off + first + k] = (uint16_t)((l << 8) | vals[p]);
            }
            code <<= 1;
        }
    }
    if (!ok) {
        // a refused set is never trusted (T.ok = 0 sends the image to the host decoder): its entries only have to keep the passes
        // in bounds and moving, so every one is a plain 16-bit skip.  The kernels stage only the first nlook slots, so every
        // selector goes back to slot 0: one left on a later slot would read first-level entries that were never staged.
        const uint16_t SKIP = (uint16_t)(16 << 8);
        for (int i = 0; i < MAX_TABLES * LOOK_N; i++) T.look[i] = SKIP;
        for (int i = 0; i < EXT_N; i++) T.ext[i] = SKIP;
        for (int i = 0; i < 20; i++) T.sel[i] = 0;
        T.nlook = 1; T.next = 0; T.ok = 0;
        return false;
    }
    T.nlook = (uint16_t)(nslot ? nslot : 1); T.next = (uint16_t)next; T.ok = 1;
    return true;
}

// one symbol from the top bits of `bits` (32 valid bits) with the table at first-level offset `base`: (length << 8) | symbol
GE_HD uint32_t lookup_symbol(const DecTables &T, uint32_t base, uint32_t bits)
{
    uint32_t e = T.look[base + (bits >> (32 - LOOK_BITS))];
    if (e & 0x8000u) { const uint32_t nb = ((e >> 11) & 7u) + 1u; e = T.ext[(e & 0x7FFu) + ((bits << LOOK_BITS) >> (32 - nb))]; }
    return e;
}

// position of scan-order unit u inside the image's component-major array of DC differences (the DC prefix sum runs over it);
// *comp_start = where u's component begins in that array
GE_HD uint32_t dc_slot_index(const ge::Scan &s, uint32_t u, uint32_t *comp_start)
{
    if (s.ns == 1) { *comp_start = 0; return u; }
    const uint32_t m = u / s.blocks_per_mcu; int q = (int)(u - m * s.blocks_per_mcu), i = 0; uint32_t start = 0;
    const uint32_t mcus = (uint32_t)s.mcux * s.mcuy;
    while (q >= s.hs[i] * s.vs[i]) { q -= s.hs[i] * s.vs[i]; start += mcus * s.hs[i] * s.vs[i]; i++; }
    *comp_start = start;
    return start + m * s.hs[i] * s.vs[i] + q;
}

// ---- output addressing without divisions -------------------------------------------------------------------------------------
// Scan-order unit -> coefficient offset, walked incrementally: the write pass finishes a block every dozen symbols, and
// ge::locate()'s divisions were half of its instructions.  A non-interleaved scan is the special case "one block per MCU".
struct Walk {
    int bpm, mcux;              // blocks per MCU, MCUs per row (single-component scan: 1, real blocks per row)
    long long base[10];         // int16 offset of block q of MCU (0, 0)
    int colstep[10], rowstep[10];   // offset step to the next MCU in the row / to the next MCU row
    // the block's place in the image's component-major array of DC differences: dc_base[q] + MCU index * dc_step[q]
    uint32_t dc_base[10]; int dc_step[10];
};
inline Walk make_walk(const ge::Scan &s)
{
    Walk w{};
    if (s.ns == 1) { w.bpm = 1; w.mcux = s.rbw; w.base[0] = s.comp_off[0]; w.colstep[0] = 64; w.rowstep[0] = s.bw[0] * 64; w.dc_step[0] = 1; return w; }
    w.bpm = s.blocks_per_mcu; w.mcux = s.mcux;
    int q = 0; uint32_t comp_start = 0;
    for (int i = 0; i < s.ns; i++) {
        const int per_mcu = s.hs[i] * s.vs[i];
        for (int by = 0; by < s.vs[i]; by++) for (int bx = 0; bx < s.hs[i]; bx++, q++) if (q < 10) {
            w.base[q] = s.comp_off[i] + ((long long)by * s.bw[i] + bx) * 64;
            w.colstep[q] = s.hs[i] * 64; w.rowstep[q] = s.vs[i] * s.bw[i] * 64;
            w.dc_base[q] = comp_start + (uint32_t)(by * s.hs[i] + bx); w.dc_step[q] = per_mcu;
        }
        comp_start += (uint32_t)s.mcux * (uint32_t)s.mcuy * (uint32_t)per_mcu;
    }
    return w;
}
struct Cursor {                 // position of one scan-order unit
    int q, mx, my;
    GE_HD void seek(const Walk &w, uint32_t u) { const uint32_t m = u / (uint32_t)w.bpm; q = (int)(u - m * (uint32_t)w.bpm); my = (int)(m / (uint32_t)w.mcux); mx = (int)(m - (uint32_t)my * (uint32_t)w.mcux); }
    GE_HD void next(const Walk &w) { if (++q == w.bpm) { q = 0; if (++mx == w.mcux) { mx = 0; my++; } } }
    GE_HD long long offset(const Walk &w) const { return w.base[q] + (long long)my * w.rowstep[q] + (long long)mx * w.colstep[q]; }
    GE_HD uint32_t dc_slot(const Walk &w) const { return w.dc_base[q] + (uint32_t)(my * w.mcux + mx) * (uint32_t)w.dc_step[q]; }
};

// Decode from state `st` until the position leaves subsequence `i` (p >= (i+1)*S) or the stream ends.  Sink receives
// coef(k, value) for every coefficient (DC as raw difference), block_done(), and -- if it defines anomaly() -- the ANOM_* mask of
// every symbol and once more when the stream has ended.
// OWN = false is the form of the synchronisation rounds.  OWN = true is the write pass, where a block belongs to the subsequence
// in which its DC symbol starts, so that every block has exactly one writer and can be stored whole:
//   * a block entered in the middle (st.k != 0, the "head") is the previous thread's: it is decoded for its length only and the
//     sink hears nothing of it, neither coefficients nor anomalies nor its end;
//   * the thread then owns every block that starts at p < end and decodes PAST `end` until the last of them is complete (or the
//     stream is over: g.nbits is the only other bound).  A head that reaches `end` leaves the thread without a block of its own.
// `st` must be the true state.  The blocks completed inside the subsequence, and so first[] (the index of the block that is
// current at entry), mean what they mean in the rounds: the sink starts at first_owned_block(first[i], st).
GE_HD uint32_t first_owned_block(uint32_t first_i, const DecState &st) { return first_i + (st.k != 0 ? 1u : 0u); }
template <bool OWN, class Sink>
GE_HD DecState decode_span(const uint8_t *__restrict__ stream, const Geometry &g, const DecTables &T, uint32_t i, DecState st, Sink &sk)
{
    const uint32_t end = (i + 1) * g.subseq_bits < g.nbits ? (i + 1) * g.subseq_bits : g.nbits;
    uint32_t p = st.p; int k = st.k, b = st.b;
    bool head = OWN && k != 0;
    // Three-word window over the stream: w0 / w1 hold the words the next 32 bits come from, w2 is fetched one word ahead so
    // the load is off the critical path.  A symbol consumes at most 16 + 15 bits, so the window moves by at most one word.
    uint32_t wi = p >> 5;
    uint32_t w0 = load_be32(stream, wi), w1 = load_be32(stream, wi + 1), w2 = load_be32(stream, wi + 2);
    const int bpm = g.blocks_per_mcu;
    // table selectors of the MCU's blocks packed into two registers (3 bits per block: the first-level table slot), so that the
    // per-symbol table choice is a shift and a mask instead of a dependent shared-memory read in front of the table lookup
    uint32_t sel_dc = 0, sel_ac = 0;
    for (int q = 0; q < bpm && q < 10; q++) { sel_dc |= (uint32_t)(T.sel[2 * q] >> LOOK_BITS) << (3 * q); sel_ac |= (uint32_t)(T.sel[2 * q + 1] >> LOOK_BITS) << (3 * q); }
    while (p < end || (OWN && k != 0 && !head && p < g.nbits)) {
        if ((p >> 5) != wi) { wi = p >> 5; w0 = w1; w1 = w2; w2 = load_be32(stream, wi + 2); }
        const uint32_t sh = p & 31;
#if defined(__CUDA_ARCH__)
        const uint32_t bits = __funnelshift_l(w1, w0, sh);
#else
        const uint32_t bits = sh ? (w0 << sh) | (w1 >> (32 - sh)) : w0;
#endif
        // One uniform body for DC and AC symbols (a DC symbol is "run 0, category s at index 0"), selects instead of
        // branches: the lanes of a warp sit at unrelated points of their blocks, so divergent paths would serialise.
        const bool dc = k == 0;
        const uint32_t e = lookup_symbol(T, (((dc ? sel_dc : sel_ac) >> (3 * b)) & 7u) << LOOK_BITS, bits);
        const int len = (int)(e >> 8), sym = (int)(e & 0xFF);
        const int r = dc ? 0 : (sym >> 4), s = sym & 15;
        const uint32_t ext = s ? (bits << len) >> (32 - s) : 0u;
        const int v = s ? ((int)ext < (1 << (s - 1)) ? (int)ext - (1 << s) + 1 : (int)ext) : 0;
        const bool eob_or_zrl = !dc && s == 0;                                     // AC symbol without a value: ZRL or EOB
        if (!head) report_anomaly(sk, symbol_anomaly(len, sym, dc, k, p + (uint32_t)(len + s), g.nbits), 0);  // only the write sink looks
        int kw = k + r; if (kw > 63) kw = 63;                                       // corrupt / unsynchronised run: clamp
        if (!eob_or_zrl && !head) sk.coef(kw, v);
        k = eob_or_zrl ? (r == 15 ? k + 16 : 64) : kw + 1;
        p += (uint32_t)(len + s);
        if (k >= 64) {
            k = 0; b++; if (b == bpm) b = 0;
            if (head) head = false; else sk.block_done();
        }
    }
    if (p >= g.nbits) report_anomaly(sk, ANOM_END, 0);         // the stream is over: reported if the sink is still inside a real block
    DecState o; o.p = p; o.k = (uint16_t)k; o.b = (uint16_t)b;
    return o;
}
template <class Sink>
GE_HD DecState decode_subsequence(const uint8_t *__restrict__ stream, const Geometry &g, const DecTables &T, uint32_t i, DecState st, Sink &sk)
{
    return decode_span<false>(stream, g, T, i, st, sk);
}
template <class Sink>
GE_HD void decode_owned_blocks(const uint8_t *__restrict__ stream, const Geometry &g, const DecTables &T, uint32_t i, DecState st, Sink &sk)
{
    decode_span<true>(stream, g, T, i, st, sk);
}

struct NullSink { uint32_t nblk = 0; GE_HD void coef(int, int) {} GE_HD void block_done() { nblk++; } };

// jdhuff.c jpeg_make_d_derived_tbl from the DHT payload
inline void build_dec_table(const uint8_t bits[17], const uint8_t *vals, DecTable &t)
{
    for (int i = 0; i < 512; i++) t.look[i] = 0;
    for (int i = 0; i < 256; i++) t.vals[i] = vals[i];
    int code = 0, p = 0;
    for (int l = 1; l <= 16; l++) {
        t.valoff[l] = p - code;
        for (int i = 0; i < bits[l]; i++, p++, code++) {
            if (l <= 9) {
                const int first = code << (9 - l), cnt = 1 << (9 - l);
                if (first + cnt <= 512) for (int k = 0; k < cnt; k++) t.look[first + k] = (uint16_t)((l << 8) | vals[p]);
            }
        }
        t.maxcode[l] = bits[l] ? code - 1 : -1;
        code <<= 1;
    }
    t.maxcode[0] = -1; t.maxcode[17] = 0x7FFFFFFF; t.valoff[0] = 0;
}

} // namespace gd
} // namespace b200
