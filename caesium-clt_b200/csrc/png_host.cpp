// png_host.cpp -- see png_host.h.  Formats: PNG (ISO/IEC 15948), zlib (RFC 1950), DEFLATE (RFC 1951).  Restates the host
// duties of oxipng 9.1.5 + libdeflate (Cargo.lock:1161, :917) behind libcaesium png::lossless: decode the source, keep
// the chunks StripChunks::Safe keeps, and wrap the re-compressed image data.
#include "png_host.h"
#include "dfl_core.h"
#include "png_adam7_core.h"
#include <emmintrin.h>
#include <immintrin.h>
#include <algorithm>
#include <cstring>

namespace b200 {

// ---- checksums ------------------------------------------------------------------------------------------------------
static uint32_t g_crc[8][256];
static bool g_crc_init = [] {
    for (uint32_t i = 0; i < 256; i++) { uint32_t c = i; for (int k = 0; k < 8; k++) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1; g_crc[0][i] = c; }
    for (uint32_t i = 0; i < 256; i++) for (int t = 1; t < 8; t++) g_crc[t][i] = (g_crc[t - 1][i] >> 8) ^ g_crc[0][g_crc[t - 1][i] & 0xFF];
    return true; }();

static uint32_t crc32_table(uint32_t crc, const uint8_t *p, size_t n)
{   // slicing-by-8; crc is the running (pre-inverted) register
    (void)g_crc_init;
    while (n >= 8) {
        uint32_t a, b; memcpy(&a, p, 4); memcpy(&b, p + 4, 4); a ^= crc;
        crc = g_crc[7][a & 0xFF] ^ g_crc[6][(a >> 8) & 0xFF] ^ g_crc[5][(a >> 16) & 0xFF] ^ g_crc[4][a >> 24] ^
              g_crc[3][b & 0xFF] ^ g_crc[2][(b >> 8) & 0xFF] ^ g_crc[1][(b >> 16) & 0xFF] ^ g_crc[0][b >> 24];
        p += 8; n -= 8;
    }
    while (n--) crc = g_crc[0][(crc ^ *p++) & 0xFF] ^ (crc >> 8);
    return crc;
}

// Carry-less-multiply folding (Gopal et al., "Fast CRC computation for generic polynomials using PCLMULQDQ"; the constants are
// x^k mod P for the reflected CRC-32 polynomial): ~10x the table loop.  A 4096^2 RGBA PNG carries ~30 MB of IDAT whose chunk CRC
// is checked on the way in and written on the way out -- at table speed that was a fifth of the host time per image.
// n >= 64 and a multiple of 16; crc is the running (pre-inverted) register.
__attribute__((target("pclmul,sse4.1")))
static uint32_t crc32_clmul(uint32_t crc, const uint8_t *buf, size_t len)
{
    const __m128i k1k2 = _mm_set_epi64x(0x01c6e41596ll, 0x0154442bd4ll), k3k4 = _mm_set_epi64x(0x00ccaa009ell, 0x01751997d0ll);
    const __m128i k5k0 = _mm_set_epi64x(0, 0x0163cd6124ll), poly = _mm_set_epi64x(0x01f7011641ll, 0x01db710641ll);
    __m128i x0, x1, x2, x3, x4, x5, x6, x7, x8, y5, y6, y7, y8;
    x1 = _mm_loadu_si128((const __m128i *)(buf + 0x00)); x2 = _mm_loadu_si128((const __m128i *)(buf + 0x10));
    x3 = _mm_loadu_si128((const __m128i *)(buf + 0x20)); x4 = _mm_loadu_si128((const __m128i *)(buf + 0x30));
    x1 = _mm_xor_si128(x1, _mm_cvtsi32_si128((int)crc));
    x0 = k1k2;
    buf += 64; len -= 64;
    while (len >= 64) {
        x5 = _mm_clmulepi64_si128(x1, x0, 0x00); x6 = _mm_clmulepi64_si128(x2, x0, 0x00); x7 = _mm_clmulepi64_si128(x3, x0, 0x00); x8 = _mm_clmulepi64_si128(x4, x0, 0x00);
        x1 = _mm_clmulepi64_si128(x1, x0, 0x11); x2 = _mm_clmulepi64_si128(x2, x0, 0x11); x3 = _mm_clmulepi64_si128(x3, x0, 0x11); x4 = _mm_clmulepi64_si128(x4, x0, 0x11);
        y5 = _mm_loadu_si128((const __m128i *)(buf + 0x00)); y6 = _mm_loadu_si128((const __m128i *)(buf + 0x10));
        y7 = _mm_loadu_si128((const __m128i *)(buf + 0x20)); y8 = _mm_loadu_si128((const __m128i *)(buf + 0x30));
        x1 = _mm_xor_si128(_mm_xor_si128(x1, x5), y5); x2 = _mm_xor_si128(_mm_xor_si128(x2, x6), y6);
        x3 = _mm_xor_si128(_mm_xor_si128(x3, x7), y7); x4 = _mm_xor_si128(_mm_xor_si128(x4, x8), y8);
        buf += 64; len -= 64;
    }
    x0 = k3k4;
    x5 = _mm_clmulepi64_si128(x1, x0, 0x00); x1 = _mm_clmulepi64_si128(x1, x0, 0x11); x1 = _mm_xor_si128(_mm_xor_si128(x1, x2), x5);
    x5 = _mm_clmulepi64_si128(x1, x0, 0x00); x1 = _mm_clmulepi64_si128(x1, x0, 0x11); x1 = _mm_xor_si128(_mm_xor_si128(x1, x3), x5);
    x5 = _mm_clmulepi64_si128(x1, x0, 0x00); x1 = _mm_clmulepi64_si128(x1, x0, 0x11); x1 = _mm_xor_si128(_mm_xor_si128(x1, x4), x5);
    while (len >= 16) {
        x2 = _mm_loadu_si128((const __m128i *)buf);
        x5 = _mm_clmulepi64_si128(x1, x0, 0x00); x1 = _mm_clmulepi64_si128(x1, x0, 0x11); x1 = _mm_xor_si128(_mm_xor_si128(x1, x2), x5);
        buf += 16; len -= 16;
    }
    x2 = _mm_clmulepi64_si128(x1, x0, 0x10);
    x3 = _mm_setr_epi32(~0, 0, ~0, 0);
    x1 = _mm_srli_si128(x1, 8); x1 = _mm_xor_si128(x1, x2);
    x0 = k5k0;
    x2 = _mm_srli_si128(x1, 4); x1 = _mm_and_si128(x1, x3); x1 = _mm_clmulepi64_si128(x1, x0, 0x00); x1 = _mm_xor_si128(x1, x2);
    x0 = poly;
    x2 = _mm_and_si128(x1, x3); x2 = _mm_clmulepi64_si128(x2, x0, 0x10); x2 = _mm_and_si128(x2, x3); x2 = _mm_clmulepi64_si128(x2, x0, 0x00);
    x1 = _mm_xor_si128(x1, x2);
    return (uint32_t)_mm_extract_epi32(x1, 1);
}

uint32_t crc32_update(uint32_t crc, const uint8_t *p, size_t n)
{
    static const bool fast = [] {
        if (!__builtin_cpu_supports("pclmul") || !__builtin_cpu_supports("sse4.1")) return false;
        // trust, but verify once against the table loop (the constants are easy to get wrong)
        uint8_t t[256]; for (int i = 0; i < 256; i++) t[i] = (uint8_t)(i * 131 + 7);
        return crc32_clmul(0x12345678u, t, 256) == crc32_table(0x12345678u, t, 256) && crc32_clmul(~0u, t + 16, 64) == crc32_table(~0u, t + 16, 64);
    }();
    crc = ~crc;
    if (fast && n >= 128) {
        const size_t body = n & ~(size_t)15;
        crc = crc32_clmul(crc, p, body);
        p += body; n -= body;
    }
    return ~crc32_table(crc, p, n);
}

uint32_t adler32(const uint8_t *p, size_t n)
{
    uint32_t a = 1, b = 0;
    while (n) {
        size_t k = n < 5552 ? n : 5552; n -= k;
        // 16 bytes at a time: b += 16 a + 16 p0 + 15 p1 + ... + p15, a += sum -- no dependency between the byte terms
        for (; k >= 16; k -= 16, p += 16) {
            uint32_t s = 0, w = 0;
            for (int i = 0; i < 16; i++) { s += p[i]; w += (uint32_t)(16 - i) * p[i]; }
            b += 16 * a + w; a += s;
        }
        while (k--) { a += *p++; b += a; }
        a %= 65521; b %= 65521;
    }
    return (b << 16) | a;
}

// ---- inflate -----------------------------------------------------------------------------------------------------------
namespace {
struct InfTable {
    uint16_t fast[1 << 12]; uint16_t count[16]; uint16_t symbol[320]; int maxlen;   // fast: (len << 12) | sym, 0 = slow path
    // the same 12-bit lookup with the symbol already interpreted, for the unchecked inner loop of zlib_inflate (build_rich):
    // bits 0..3 code length (0 = leave the fast loop), bit 4 literal, bit 5 end of block, bits 8..11 extra-bit count,
    // bits 16..31 literal value / length base / distance base
    uint32_t rich[1 << 11];     // literal/length codes use all 11 index bits, distance codes the low 9 (longer codes: checked path)
};
enum { RICH_LIT = 1 << 4, RICH_EOB = 1 << 5 };

bool build_inf(InfTable &t, const uint8_t *lens, int n)
{
    memset(t.count, 0, sizeof(t.count));
    for (int i = 0; i < n; i++) t.count[lens[i]]++;
    t.count[0] = 0;
    int left = 1;
    for (int l = 1; l <= 15; l++) { left <<= 1; left -= t.count[l]; if (left < 0) return false; }
    uint16_t offs[16]; offs[1] = 0;
    for (int l = 1; l < 15; l++) offs[l + 1] = offs[l] + t.count[l];
    for (int i = 0; i < n; i++) if (lens[i]) t.symbol[offs[lens[i]]++] = (uint16_t)i;
    memset(t.fast, 0, sizeof(t.fast));
    // canonical codes, bit-reversed (DEFLATE packs Huffman codes starting from the LSB)
    int code = 0, idx = 0; t.maxlen = 0;
    for (int l = 1; l <= 15; l++) {
        for (int k = 0; k < t.count[l]; k++, idx++, code++) {
            t.maxlen = l;
            if (l <= 12) {
                int rev = 0; for (int b = 0; b < l; b++) if (code & (1 << b)) rev |= 1 << (l - 1 - b);
                for (int f = rev; f < 4096; f += 1 << l) t.fast[f] = (uint16_t)((l << 12) | t.symbol[idx]);
            }
        }
        code <<= 1;
    }
    return true;
}

struct InfBits {
    const uint8_t *p, *end; uint64_t acc = 0; int n = 0;
    inline void fill()
    {
        if (end - p >= 8) {                              // one unaligned 64-bit load tops the accumulator up to >= 56 bits
            uint64_t v; memcpy(&v, p, 8);
            acc |= v << n;
            const int adv = (63 - n) >> 3;
            p += adv; n += adv * 8;
            return;
        }
        while (n <= 56 && p < end) { acc |= (uint64_t)*p++ << n; n += 8; }
    }
    inline uint32_t peek(int k) { return (uint32_t)(acc & ((1ull << k) - 1)); }
    inline void drop(int k) { acc >>= k; n -= k; }
    inline uint32_t get(int k) { if (n < k) fill(); uint32_t v = peek(k); drop(k); return v; }
};

inline int inf_decode(InfBits &b, const InfTable &t)
{
    if (b.n < 15) b.fill();
    uint32_t e = t.fast[b.peek(12)];
    if (e) { b.drop(e >> 12); return e & 0xFFF; }
    int code = 0, first = 0, index = 0;
    for (int l = 1; l <= 15; l++) {
        code |= (int)(b.acc & 1); b.drop(1);
        int cnt = t.count[l];
        if (code - cnt < first) return t.symbol[index + (code - first)];
        index += cnt; first += cnt; first <<= 1; code <<= 1;
    }
    return -1;
}

const uint16_t kLenBase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
const uint8_t kLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
const uint16_t kDistBase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
const uint8_t kDistExtra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
const uint8_t kClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

constexpr int RICH_LIT_BITS = 11, RICH_DIST_BITS = 9;
void build_rich(InfTable &t, bool dist)
{
    const int bits = dist ? RICH_DIST_BITS : RICH_LIT_BITS;
    for (int f = 0; f < (1 << bits); f++) {
        const uint32_t e = t.fast[f]; uint32_t r = 0;
        if (e && (int)(e >> 12) <= bits) {
            const uint32_t len = e >> 12, s = e & 0xFFF;
            if (dist) { if (s < 30) r = len | ((uint32_t)kDistExtra[s] << 8) | ((uint32_t)kDistBase[s] << 16); }
            else if (s < 256) r = len | RICH_LIT | (s << 16);
            else if (s == 256) r = len | RICH_EOB;
            else if (s < 286) r = len | ((uint32_t)kLenExtra[s - 257] << 8) | ((uint32_t)kLenBase[s - 257] << 16);
        }
        t.rich[f] = r;             // 0: long code or invalid symbol -> the checked path deals with it
    }
}
} // namespace

// One body for both destinations: a vector that grows (stage entry points, conversions) or a caller's fixed buffer of
// cap >= limit + 4096 bytes (the lossless path inflates straight into pinned staging memory, no zero-fill, no second copy).
static bool inflate_body(const uint8_t *in, size_t n, std::vector<uint8_t> *vec, uint8_t *fixed, size_t fixed_cap, size_t size_hint, size_t *out_len, bool verify_adler,
                         uint32_t *stored_adler, std::string &err)
{
    if (n < 6) { err = "zlib stream too short"; return false; }
    if ((in[0] & 0x0F) != 8 || ((in[0] << 8) | in[1]) % 31 != 0 || (in[1] & 0x20)) { err = "bad zlib header"; return false; }
    InfBits b; b.p = in + 2; b.end = in + n;
    // Bytes are written through a raw pointer; a vector is trimmed at the end.  A caller that knows the decoded size (PNG:
    // (row_bytes + 1) * height from IHDR) passes it as size_hint and the stream may not inflate to more than that: an IDAT
    // that claims a 1x1 image and carries megabytes is refused instead of being expanded (decompression bomb).  DEFLATE
    // cannot expand by more than 1032:1, which bounds the first allocation when IHDR promises more than the input can hold.
    const size_t limit = size_hint ? size_hint : (size_t)-1;
    const size_t most = n > ((size_t)-1 >> 12) ? (size_t)-1 >> 1 : n * 1032 + 64;
    size_t cap, pos = 0;
    struct Dest {
        std::vector<uint8_t> *vec; uint8_t *base;
        bool grow(size_t &cap_, size_t want) { if (!vec) return false; cap_ = want; vec->resize(cap_ + 16); base = vec->data(); return true; }
    } out{vec, fixed};
    if (vec) { cap = std::min(size_hint ? size_hint : n * 4, most) + 4096; vec->resize(cap + 16); out.base = vec->data(); }
    else { if (fixed_cap < 1024) { err = "inflate buffer too small"; return false; } cap = fixed_cap - 16; }
    constexpr size_t MATCH_ROOM = 258 + 8;          // the longest match plus the 8-byte copy granularity
    static thread_local InfTable lit, dist;
    for (;;) {
        const uint32_t final = b.get(1), type = b.get(2);
        if (type == 0) {
            b.drop(b.n & 7);
            // give back whole buffered bytes
            while (b.n >= 8) { b.p--; b.n -= 8; } b.acc = 0; b.n = 0;
            if (b.end - b.p < 4) { err = "truncated stored block"; return false; }
            const uint32_t len = b.p[0] | (b.p[1] << 8), nlen = b.p[2] | (b.p[3] << 8);
            if ((len ^ 0xFFFF) != nlen || (size_t)(b.end - b.p - 4) < len) { err = "bad stored block"; return false; }
            if (len > limit - std::min(pos, limit)) { err = "IDAT too long"; return false; }
            if (cap - pos < len + 320 && !out.grow(cap, cap * 2 + len + 4096)) { err = "IDAT too long"; return false; }
            memcpy(out.base + pos, b.p + 4, len); pos += len; b.p += 4 + len;
        } else if (type == 1 || type == 2) {
            uint8_t lens[320];
            if (type == 1) {
                for (int i = 0; i < 288; i++) lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
                build_inf(lit, lens, 288);
                for (int i = 0; i < 30; i++) lens[i] = 5;
                build_inf(dist, lens, 30);
                build_rich(lit, false); build_rich(dist, true);
            } else {
                const int hlit = (int)b.get(5) + 257, hdist = (int)b.get(5) + 1, hclen = (int)b.get(4) + 4;
                uint8_t cl[19] = {0};
                for (int i = 0; i < hclen; i++) cl[kClOrder[i]] = (uint8_t)b.get(3);
                static thread_local InfTable clt;
                if (!build_inf(clt, cl, 19)) { err = "bad code-length code"; return false; }
                int i = 0;
                while (i < hlit + hdist) {
                    int s = inf_decode(b, clt);
                    if (s < 0) { err = "bad code-length symbol"; return false; }
                    if (s < 16) lens[i++] = (uint8_t)s;
                    else {
                        int rep, val = 0;
                        if (s == 16) { if (!i) { err = "repeat without previous length"; return false; } val = lens[i - 1]; rep = 3 + (int)b.get(2); }
                        else if (s == 17) rep = 3 + (int)b.get(3); else rep = 11 + (int)b.get(7);
                        if (i + rep > hlit + hdist) { err = "code lengths overflow"; return false; }
                        while (rep--) lens[i++] = (uint8_t)val;
                    }
                }
                if (!build_inf(lit, lens, hlit) || !build_inf(dist, lens + hlit, hdist)) { err = "bad Huffman code"; return false; }
                build_rich(lit, false); build_rich(dist, true);
            }
            for (;;) {
                if (cap - pos < 640 && !out.grow(cap, cap * 2 + 4096)) { err = "IDAT too long"; return false; }     // room for the fast loop's unchecked stretch
                uint8_t *o = out.base;
                // ---- unchecked inner loop: one 64-bit refill per iteration covers a whole match (15 + 5 + 15 + 13 bits) or up
                // to three literals; it runs while >= 16 input bytes and >= 320 output bytes remain and hands anything unusual
                // (codes longer than 12 bits, invalid symbols, distances past the start) to the checked code below, untouched
                {
                    const uint8_t *ip = b.p; uint64_t acc = b.acc; int nb = b.n;
                    uint8_t *op = o + pos, *const olimit = o + cap - 320;
                    const uint8_t *const ilimit = b.end - 16;
                    bool eob = false;
                    while (ip <= ilimit && op <= olimit) {
                        { uint64_t v; memcpy(&v, ip, 8); acc |= v << nb; ip += (63 - nb) >> 3; nb |= 56; }
                        uint32_t e = lit.rich[acc & ((1u << RICH_LIT_BITS) - 1)];
                        if (e & RICH_LIT) {
                            *op++ = (uint8_t)(e >> 16); acc >>= (e & 15); nb -= (int)(e & 15);
                            e = lit.rich[acc & ((1u << RICH_LIT_BITS) - 1)];
                            if (e & RICH_LIT) {
                                *op++ = (uint8_t)(e >> 16); acc >>= (e & 15); nb -= (int)(e & 15);
                                e = lit.rich[acc & ((1u << RICH_LIT_BITS) - 1)];
                                if (e & RICH_LIT) { *op++ = (uint8_t)(e >> 16); acc >>= (e & 15); nb -= (int)(e & 15); }
                            }
                            continue;
                        }
                        if (!(e & 15)) break;
                        if (e & RICH_EOB) { acc >>= (e & 15); nb -= (int)(e & 15); eob = true; break; }
                        // a match: decode everything on copies, commit only when it is sound
                        uint64_t a2 = acc >> (e & 15); int n2 = nb - (int)(e & 15);
                        const uint32_t lx = (e >> 8) & 15;
                        const size_t len = (e >> 16) + (size_t)(a2 & ((1u << lx) - 1)); a2 >>= lx; n2 -= (int)lx;
                        const uint32_t de = dist.rich[a2 & ((1u << RICH_DIST_BITS) - 1)];
                        if (!(de & 15)) break;
                        a2 >>= (de & 15); n2 -= (int)(de & 15);
                        const uint32_t dx = (de >> 8) & 15;
                        const size_t d = (de >> 16) + (size_t)(a2 & ((1u << dx) - 1)); a2 >>= dx; n2 -= (int)dx;
                        if (d > (size_t)(op - o)) break;
                        acc = a2; nb = n2;
                        const uint8_t *src = op - d;
                        if (d >= 8) { for (size_t k = 0; k < len; k += 8) memcpy(op + k, src + k, 8); }
                        else if (d == 1) memset(op, src[0], len);
                        else {
                            // distance 2..7 (the previous pixel of a filtered row: the commonest match in PNG data): an 8-byte
                            // pattern of the period, stored every `step` bytes where step is the largest multiple of d <= 8
                            uint8_t pat[8]; for (int i = 0; i < 8; i++) pat[i] = src[(size_t)i % d];
                            const size_t step = d * (8 / d);
                            for (size_t k = 0; k < len; k += step) memcpy(op + k, pat, 8);
                        }
                        op += len;
                    }
                    b.p = ip; b.acc = acc; b.n = nb; pos = (size_t)(op - o);
                    if (pos > limit) { err = "IDAT too long"; return false; }
                    if (eob) break;
                }
                // the fast loop may stop as close as 55 bytes to the end of the buffer: make room for one more whole match
                // before the checked path writes anything (ADVICE r1: heap overflow on an IDAT longer than IHDR implies)
                if (cap - pos < MATCH_ROOM + 64) { if (!out.grow(cap, cap * 2 + 4096)) { err = "IDAT too long"; return false; } o = out.base; }
                int s = inf_decode(b, lit);
                if (s < 0) { err = "bad literal/length code"; return false; }
                if (s < 256) o[pos++] = (uint8_t)s;
                else if (s == 256) break;
                else {
                    s -= 257; if (s >= 29) { err = "bad length symbol"; return false; }
                    const size_t len = kLenBase[s] + b.get(kLenExtra[s]);
                    const int ds = inf_decode(b, dist);
                    if (ds < 0 || ds >= 30) { err = "bad distance code"; return false; }
                    const size_t d = kDistBase[ds] + b.get(kDistExtra[ds]);
                    if (d > pos) { err = "distance too far back"; return false; }
                    uint8_t *dst = o + pos; const uint8_t *src = dst - d;
                    if (d >= 8) { for (size_t k = 0; k < len; k += 8) memcpy(dst + k, src + k, 8); }      // chunks never overlap their own source
                    else if (d == 1) memset(dst, src[0], len);
                    else for (size_t k = 0; k < len; k++) dst[k] = src[k];
                    pos += len;
                }
                if (pos > limit) { err = "IDAT too long"; return false; }
                if (b.p >= b.end && b.n <= 0) { err = "truncated deflate stream"; return false; }
            }
        } else { err = "bad block type"; return false; }
        if (final) break;
    }
    if (vec) vec->resize(pos);
    if (out_len) *out_len = pos;
    b.drop(b.n & 7);
    uint8_t tail[4]; for (int i = 0; i < 4; i++) tail[i] = (uint8_t)b.get(8);
    const uint32_t want = ((uint32_t)tail[0] << 24) | (tail[1] << 16) | (tail[2] << 8) | tail[3];
    if (stored_adler) *stored_adler = want;
    if (verify_adler && want != adler32(out.base, pos)) { err = "Adler-32 mismatch"; return false; }
    return true;
}

bool zlib_inflate(const uint8_t *in, size_t n, std::vector<uint8_t> &out, size_t size_hint, std::string &err)
{
    return inflate_body(in, n, &out, nullptr, 0, size_hint, nullptr, true, nullptr, err);
}

bool zlib_inflate_to(const uint8_t *in, size_t n, uint8_t *buf, size_t cap, size_t size_limit, size_t *out_len, uint32_t *stored_adler, std::string &err)
{
    if (!size_limit || cap < size_limit + 4096) { err = "inflate buffer too small"; return false; }
    return inflate_body(in, n, nullptr, buf, cap, size_limit, out_len, false, stored_adler, err);
}


// ---- PNG container -------------------------------------------------------------------------------------------------------
static uint32_t be32(const uint8_t *p) { return ((uint32_t)p[0] << 24) | (p[1] << 16) | (p[2] << 8) | p[3]; }
static void put32(std::vector<uint8_t> &o, uint32_t v) { o.push_back(v >> 24); o.push_back(v >> 16); o.push_back(v >> 8); o.push_back(v); }
static void put_chunk(std::vector<uint8_t> &o, const char *type, const uint8_t *data, size_t n)
{
    put32(o, (uint32_t)n);
    const size_t s = o.size();
    o.insert(o.end(), type, type + 4); o.insert(o.end(), data, data + n);
    put32(o, crc32_update(0, o.data() + s, 4 + n));
}

static inline int paeth(int a, int b, int c) { int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c); return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c); }

// Paeth reconstruction for 3- and 4-byte pixels: the channels of one pixel are independent, so they ride in four 16-bit
// lanes; the serial dependency is only pixel to pixel.  Loads/stores are 4 bytes wide (callers keep slack after the rows).
static void unfilter_paeth_sse2(const uint8_t *f, const uint8_t *up, uint8_t *r, size_t rb, size_t bpp)
{
    const __m128i zero = _mm_setzero_si128();
    __m128i a = zero, c = zero;                       // left and upper-left pixels (zero before the first pixel)
    for (size_t x = 0; x < rb; x += bpp) {
        uint32_t ub, fx; memcpy(&ub, up + x, 4); memcpy(&fx, f + x, 4);
        const __m128i b = _mm_unpacklo_epi8(_mm_cvtsi32_si128((int)ub), zero), v = _mm_unpacklo_epi8(_mm_cvtsi32_si128((int)fx), zero);
        __m128i pa = _mm_sub_epi16(b, c), pb = _mm_sub_epi16(a, c);              // p - a = b - c, p - b = a - c
        __m128i pc = _mm_add_epi16(pa, pb);                                      // p - c
        pa = _mm_max_epi16(pa, _mm_sub_epi16(zero, pa)); pb = _mm_max_epi16(pb, _mm_sub_epi16(zero, pb)); pc = _mm_max_epi16(pc, _mm_sub_epi16(zero, pc));
        const __m128i smallest = _mm_min_epi16(pc, _mm_min_epi16(pa, pb));
        const __m128i ma = _mm_cmpeq_epi16(smallest, pa), mb = _mm_cmpeq_epi16(smallest, pb);
        const __m128i bc = _mm_or_si128(_mm_and_si128(mb, b), _mm_andnot_si128(mb, c));
        const __m128i pred = _mm_or_si128(_mm_and_si128(ma, a), _mm_andnot_si128(ma, bc));
        const __m128i d = _mm_and_si128(_mm_add_epi16(v, pred), _mm_set1_epi16(0xFF));
        c = b; a = d;
        const uint32_t o = (uint32_t)_mm_cvtsi128_si32(_mm_packus_epi16(d, d));
        if (bpp == 4 || x + 4 <= rb) memcpy(r + x, &o, 4); else memcpy(r + x, &o, 3);
    }
}

bool png_parse_chunks(const uint8_t *d, size_t n, bool keep_all, PngInfo &info, PngIdat &idat_out, std::string &err)
{
    static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
    if (n < 8 + 25 || memcmp(d, sig, 8)) { err = "not a PNG"; return false; }
    info = PngInfo();
    std::vector<uint8_t> &idat = idat_out.joined; idat.clear();
    const uint8_t *first_idat = nullptr; size_t first_len = 0; int nidat = 0;
    size_t i = 8; bool have_ihdr = false, seen_idat = false, seen_end = false;
    while (i + 12 <= n) {
        const uint32_t L = be32(d + i);
        if (L > n - i - 12) { err = "truncated PNG chunk"; return false; }
        const uint8_t *type = d + i + 4, *data = d + i + 8;
        if (be32(data + L) != crc32_update(0, type, 4 + L)) { err = "PNG chunk CRC mismatch"; return false; }
        if (!memcmp(type, "IHDR", 4)) {
            if (L != 13) { err = "bad IHDR"; return false; }
            info.width = be32(data); info.height = be32(data + 4); info.bit_depth = data[8]; info.color_type = data[9]; info.interlace = data[12];
            if (!info.width || !info.height || data[10] || data[11]) { err = "bad IHDR"; return false; }
            static const int ch[7] = {1, 0, 3, 1, 2, 0, 4};
            if (info.color_type > 6 || !ch[info.color_type]) { err = "bad colour type"; return false; }
            // legal (colour type, bit depth) pairs of PNG 11.2.2 only: anything else would index samples with bd / 8 == 0,
            // divide by (1 << 0) - 1 or make zero-sized rows further down
            const int bd = info.bit_depth;
            const bool depth_ok = info.color_type == 0 ? (bd == 1 || bd == 2 || bd == 4 || bd == 8 || bd == 16)
                                : info.color_type == 3 ? (bd == 1 || bd == 2 || bd == 4 || bd == 8) : (bd == 8 || bd == 16);
            if (!depth_ok) { err = "bad bit depth for the colour type"; return false; }
            if (info.width > 0x7FFFFFFFu || info.height > 0x7FFFFFFFu) { err = "bad IHDR"; return false; }
            info.channels = ch[info.color_type]; info.bits_per_pixel = info.channels * info.bit_depth;
            info.bpp = std::max(1, info.bits_per_pixel / 8);
            info.row_bytes = ((size_t)info.width * info.bits_per_pixel + 7) / 8;
            have_ihdr = true;
        } else if (!memcmp(type, "IDAT", 4)) {
            // one IDAT chunk (the usual case for files a compressor wrote): inflate it where it lies; several: join them
            if (nidat == 0) { first_idat = data; first_len = L; }
            else { if (nidat == 1) idat.assign(first_idat, first_idat + first_len); idat.insert(idat.end(), data, data + L); }
            nidat++; seen_idat = true;
        }
        else if (!memcmp(type, "IEND", 4)) { seen_end = true; break; }
        else if (!memcmp(type, "PLTE", 4)) info.plte.assign(data, data + L);
        else if (!memcmp(type, "tRNS", 4)) info.trns.assign(data, data + L);
        else {
            // oxipng StripChunks::Safe keeps the chunks that affect rendering; with keep_metadata nothing is stripped
            static const char *safe[] = {"cICP", "iCCP", "sRGB", "pHYs", "gAMA", "cHRM", "sBIT", "acTL", "fcTL", "fdAT"};
            bool keep = keep_all;
            for (const char *s : safe) if (!memcmp(type, s, 4)) keep = true;
            if (keep) { std::vector<uint8_t> &dst = seen_idat ? info.kept_after_idat : info.kept_before_idat; dst.insert(dst.end(), d + i, d + i + 12 + L); }
        }
        i += 12 + L;
    }
    if (!have_ihdr || !seen_idat || !seen_end) { err = "incomplete PNG"; return false; }
    if (info.interlace > 1 || (info.interlace == 1 && !png_interlaced())) { err = "interlaced PNG is not supported on the GPU path"; return false; }
    // 1 TiB of samples: no overflow below.  The first test keeps png_inflated_size from overflowing; an Adam7 stream is larger (up to
    // about 15 h / 8 filter bytes and a padded last byte per pass row), so it is bounded on its own.
    const size_t stride = info.row_bytes + 1, most = (size_t)1 << 40;
    if (stride > most / info.height || png_inflated_size(info) > most) { err = "PNG dimensions too large"; return false; }
    if (nidat == 1) { idat_out.p = first_idat; idat_out.n = first_len; } else { idat_out.p = idat.data(); idat_out.n = idat.size(); }
    return true;
}

size_t png_inflated_size(const PngInfo &info)
{
    if (info.interlace != 1) return (info.row_bytes + 1) * (size_t)info.height;
    Adam7Layout L;
    adam7_layout(info.width, info.height, info.bits_per_pixel, L);
    return L.filt_bytes;
}

bool png_parse_inflate(const uint8_t *d, size_t n, bool keep_all, PngInfo &info, std::vector<uint8_t> &filt, std::string &err)
{
    PngIdat idat;
    if (!png_parse_chunks(d, n, keep_all, info, idat, err)) return false;
    const size_t nin = png_inflated_size(info);
    if (!zlib_inflate(idat.p, idat.n, filt, nin, err)) return false;
    if (filt.size() < nin) { err = "IDAT too short"; return false; }
    return true;
}

// PNG 9.2 reconstruction of h rows of rb bytes: filt holds each row's filter byte and filtered bytes, raw receives the rows.  Both
// have 16 bytes of slack after them (the 4-byte-wide Paeth path reads and stores past a 3-byte pixel); zero_row has rb + 16 zeros.
static bool unfilter_rows(const uint8_t *filt, uint8_t *raw, size_t h, size_t rb, size_t bpp, const uint8_t *zero_row, std::string &err)
{
    const size_t stride = rb + 1;
    for (size_t y = 0; y < h; y++) {
        const uint8_t *f = filt + y * stride; const int ft = f[0]; f++;
        uint8_t *r = raw + y * rb; const uint8_t *up = y ? r - rb : zero_row;
        switch (ft) {
            case 0: memcpy(r, f, rb); break;
            case 1:
                for (size_t x = 0; x < bpp && x < rb; x++) r[x] = f[x];
                for (size_t x = bpp; x < rb; x++) r[x] = (uint8_t)(f[x] + r[x - bpp]);
                break;
            case 2: for (size_t x = 0; x < rb; x++) r[x] = (uint8_t)(f[x] + up[x]); break;
            case 3:
                for (size_t x = 0; x < bpp && x < rb; x++) r[x] = (uint8_t)(f[x] + (up[x] >> 1));
                for (size_t x = bpp; x < rb; x++) r[x] = (uint8_t)(f[x] + ((r[x - bpp] + up[x]) >> 1));
                break;
            case 4:
                if ((bpp == 3 || bpp == 4) && rb >= bpp) unfilter_paeth_sse2(f, up, r, rb, bpp);
                else {
                    for (size_t x = 0; x < bpp && x < rb; x++) r[x] = (uint8_t)(f[x] + up[x]);          // a = c = 0: the predictor is b
                    for (size_t x = bpp; x < rb; x++) r[x] = (uint8_t)(f[x] + paeth(r[x - bpp], up[x], up[x - bpp]));
                }
                break;
            default: err = "bad filter type"; return false;
        }
    }
    return true;
}

bool png_decode(const uint8_t *d, size_t n, bool keep_all, PngInfo &info, std::vector<uint8_t> &raw, std::string &err)
{
    std::vector<uint8_t> filt;
    if (!png_parse_inflate(d, n, keep_all, info, filt, err)) return false;
    const size_t nraw = info.row_bytes * info.height, bpp = (size_t)info.bpp, rb = info.row_bytes;
    filt.resize(filt.size() + 16);
    const std::vector<uint8_t> zero_row(rb + 16, 0);
    if (info.interlace != 1) {
        raw.resize(nraw + 16);
        if (!unfilter_rows(filt.data(), raw.data(), info.height, rb, bpp, zero_row.data(), err)) return false;
        raw.resize(nraw);
        return true;
    }
    // Adam7: each pass is un-filtered as an image of its own into a pass-packed buffer, then the full rows are gathered from it
    Adam7Layout L;
    adam7_layout(info.width, info.height, info.bits_per_pixel, L);
    std::vector<uint8_t> packed(L.raw_bytes + 16);
    for (const Adam7Pass &P : L.pass)
        if (P.h && !unfilter_rows(filt.data() + P.filt_off, packed.data() + P.raw_off, P.h, P.rb, bpp, zero_row.data(), err)) return false;
    raw.resize(nraw);
    for (uint32_t y = 0; y < info.height; y++)
        for (size_t i = 0; i < rb; i++) raw[(size_t)y * rb + i] = adam7_gather_byte(packed.data(), L, info.bits_per_pixel, info.width, y, i);
    info.interlace = 0;
    return true;
}

static bool kept_has(const std::vector<uint8_t> &kept, const char *type)
{   // kept = serialised chunks: length (4, big endian) | type (4) | data | crc (4)
    size_t i = 0;
    while (i + 12 <= kept.size()) {
        const uint32_t L = be32(kept.data() + i);
        if (!memcmp(kept.data() + i + 4, type, 4)) return true;
        if (L > kept.size() - i - 12) break;
        i += 12 + (size_t)L;
    }
    return false;
}

bool png_palette_candidate(const PngInfo &info)
{
    if (info.bit_depth != 8 || (info.color_type != 2 && info.color_type != 6) || !info.trns.empty() || !info.plte.empty()) return false;
    for (const char *t : {"sBIT", "bKGD", "hIST", "acTL"}) if (kept_has(info.kept_before_idat, t) || kept_has(info.kept_after_idat, t)) return false;
    return true;
}

bool png_reduce_palette(PngInfo &info, std::vector<uint8_t> &raw)
{
    if (!png_palette_candidate(info)) return false;
    const size_t npix = (size_t)info.width * info.height; const int ch = info.channels;
    if (raw.size() < npix * (size_t)ch || npix == 0) return false;
    // distinct pixel values, first-appearance order; open addressing over 1024 slots; bail out at the 257th colour
    uint32_t key[1024]; int16_t slot_idx[1024]; memset(slot_idx, 0xFF, sizeof(slot_idx));
    uint32_t colours[256]; int ncol = 0; bool grey = true;
    {   // photographs leave here without touching memory: more than 256 values among the first few thousand pixels
        const size_t probe = std::min<size_t>(npix, 8192);
        const uint8_t *q = raw.data(); uint32_t seen[512]; uint8_t used[512]; memset(used, 0, sizeof(used)); int nseen = 0;
        for (size_t i = 0; i < probe; i++, q += ch) {
            const uint32_t v = (uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16) | ((uint32_t)(ch == 4 ? q[3] : 255) << 24);
            uint32_t h = (v * 2654435761u) >> 23;
            while (used[h] && seen[h] != v) h = (h + 1) & 511;
            if (!used[h]) { if (++nseen > 256) return false; used[h] = 1; seen[h] = v; }
        }
    }
    std::vector<uint8_t> idx(npix);
    const uint8_t *p = raw.data();
    uint32_t last = 0; int last_i = -1;
    for (size_t i = 0; i < npix; i++, p += ch) {
        const uint32_t v = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)(ch == 4 ? p[3] : 255) << 24);
        if (last_i >= 0 && v == last) { idx[i] = (uint8_t)last_i; continue; }      // runs: flat art is mostly this
        uint32_t h = (v * 2654435761u) >> 22;
        for (;;) {
            const int s = slot_idx[h];
            if (s < 0) {
                if (ncol == 256) return false;
                key[h] = v; slot_idx[h] = (int16_t)ncol; colours[ncol] = v;
                if (p[0] != p[1] || p[1] != p[2]) grey = false;
                last_i = ncol++; break;
            }
            if (key[h] == v) { last_i = s; break; }
            h = (h + 1) & 1023;
        }
        last = v; idx[i] = (uint8_t)last_i;
    }
    if (grey) return false;
    // entries that are not opaque go first (stable), so tRNS can stop at the last of them
    uint8_t remap[256]; int order[256], n = 0, ntrans = 0;
    for (int c = 0; c < ncol; c++) if ((colours[c] >> 24) != 255) order[n++] = c;
    ntrans = n;
    for (int c = 0; c < ncol; c++) if ((colours[c] >> 24) == 255) order[n++] = c;
    for (int k = 0; k < ncol; k++) remap[order[k]] = (uint8_t)k;
    if (ntrans) for (size_t i = 0; i < npix; i++) idx[i] = remap[idx[i]];
    info.plte.resize((size_t)ncol * 3); info.trns.resize((size_t)ntrans);
    for (int k = 0; k < ncol; k++) {
        const uint32_t v = colours[order[k]];
        info.plte[3 * k] = (uint8_t)v; info.plte[3 * k + 1] = (uint8_t)(v >> 8); info.plte[3 * k + 2] = (uint8_t)(v >> 16);
        if (k < ntrans) info.trns[k] = (uint8_t)(v >> 24);
    }
    // oxipng reduction::bit_depth for palettes: 16 / 4 / 2 entries fit 4 / 2 / 1 bits per index (rows packed MSB first, padded to bytes)
    const int depth = ncol <= 2 ? 1 : ncol <= 4 ? 2 : ncol <= 16 ? 4 : 8;
    info.color_type = 3; info.channels = 1; info.bit_depth = depth; info.bits_per_pixel = depth; info.bpp = 1;
    info.row_bytes = ((size_t)info.width * depth + 7) / 8;
    if (depth == 8) { raw.swap(idx); return true; }
    const int per = 8 / depth;
    raw.assign(info.row_bytes * info.height, 0);
    for (uint32_t y = 0; y < info.height; y++) {
        const uint8_t *src = idx.data() + (size_t)y * info.width; uint8_t *dst = raw.data() + (size_t)y * info.row_bytes;
        for (uint32_t x = 0; x < info.width; x++) dst[x / per] |= (uint8_t)(src[x] << (8 - depth - (x % per) * depth));
    }
    return true;
}

void png_write(const PngInfo &info, const std::vector<uint8_t> &z, std::vector<uint8_t> &out)
{
    static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
    out.clear(); out.reserve(z.size() + 1024 + info.kept_before_idat.size() + info.kept_after_idat.size());
    out.insert(out.end(), sig, sig + 8);
    uint8_t ih[13]; ih[0] = info.width >> 24; ih[1] = info.width >> 16; ih[2] = info.width >> 8; ih[3] = info.width;
    ih[4] = info.height >> 24; ih[5] = info.height >> 16; ih[6] = info.height >> 8; ih[7] = info.height;
    ih[8] = (uint8_t)info.bit_depth; ih[9] = (uint8_t)info.color_type; ih[10] = 0; ih[11] = 0; ih[12] = 0;
    put_chunk(out, "IHDR", ih, 13);
    out.insert(out.end(), info.kept_before_idat.begin(), info.kept_before_idat.end());
    if (!info.plte.empty()) put_chunk(out, "PLTE", info.plte.data(), info.plte.size());
    if (!info.trns.empty()) put_chunk(out, "tRNS", info.trns.data(), info.trns.size());
    put_chunk(out, "IDAT", z.data(), z.size());
    out.insert(out.end(), info.kept_after_idat.begin(), info.kept_after_idat.end());
    put_chunk(out, "IEND", nullptr, 0);
}

// ---- DEFLATE encoder over device-made LZ77 tokens --------------------------------------------------------------------------
namespace {
struct BitOut {                 // LSB-first bit writer over a vector grown in big steps; branch-free: every put stores the 8-byte
                                // accumulator at the write position and advances by the whole bytes it holds
    std::vector<uint8_t> &o; size_t pos; uint64_t acc = 0; int n = 0;          // n < 8 between puts
    explicit BitOut(std::vector<uint8_t> &out) : o(out), pos(out.size()) {}
    inline void reserve(size_t more) { if (o.size() < pos + more + 16) o.resize(std::max(o.size() * 2, pos + more + 16)); }
    inline void put(uint64_t v, int k)              // k <= 56; the caller has reserved the room
    {
        acc |= v << n; n += k;
        memcpy(o.data() + pos, &acc, 8);
        const int adv = n >> 3;
        pos += (size_t)adv; acc = adv >= 8 ? 0 : acc >> (adv * 8); n &= 7;
    }
    inline void flush() { if (n > 0) { o[pos++] = (uint8_t)acc; } acc = 0; n = 0; o.resize(pos); }
};

} // namespace

void deflate_tokens(const uint32_t *tok, size_t nt, uint32_t adler, std::vector<uint8_t> &out, size_t block_tokens)
{   // the block coder itself is dfl_core.h (shared with the device writer, png_deflate.cu); this is its sequential driver
    out.clear(); out.reserve(nt + nt / 4 + 1024);
    out.push_back(0x78); out.push_back(0xDA);
    BitOut bw(out);
    size_t pos = 0;
    bw.reserve(64);
    if (nt == 0) { bw.put(1, 1); bw.put(1, 2); bw.put(0, 7); }
    static thread_local dfl::BlockTables T; static thread_local dfl::HuffScratch S; static thread_local dfl::EmitTables E;
    auto put = [&](uint32_t v, int k) { bw.put(v, k); };
    while (pos < nt) {
        const size_t end = std::min(nt, pos + block_tokens);
        uint32_t lf[dfl::NLIT] = {0}, df[dfl::NDIST] = {0};
        for (size_t i = pos; i < end; i++) dfl::token_count(tok[i], lf, df);
        dfl::build_block_tables(lf, df, T, S);
        bw.reserve(512 + (end - pos) * 6);                  // header < 400 bytes; a token is at most 15 + 5 + 15 + 13 bits
        dfl::write_block_header(T, end == nt, put);
        for (int i = 0; i < 256; i++) dfl::fill_emit_entry(T, E, i);
        for (size_t i = pos; i < end; i++) { uint32_t nb; const uint64_t piece = dfl::token_piece(E, tok[i], &nb); bw.put(piece, (int)nb); }
        bw.put(E.eob_code, E.eob_len);
        pos = end;
    }
    bw.reserve(16);
    bw.flush();
    out.push_back(adler >> 24); out.push_back(adler >> 16); out.push_back(adler >> 8); out.push_back(adler);
}

} // namespace b200
