// vp8l_writer.h -- the host side of the VP8L bitstream writer shared by the ALPH coder (vp8l_alpha.cpp) and the lossless WebP encoder
// (vp8l_encode.cpp): an LSB-first bit writer and the length-limited (15-bit) canonical prefix codes of dfl_core.h with their
// serialisation (specification sections 6.2.1 / 6.2.2).
#pragma once
#include <cstdint>
#include <vector>
#include "dfl_core.h"
#include "vp8l_enc_core.h"

namespace b200 {

struct BitsLsb {
    std::vector<uint8_t> &o; uint64_t acc = 0; int n = 0;
    explicit BitsLsb(std::vector<uint8_t> &out) : o(out) {}
    void put(uint32_t v, int nb)
    {
        if (!nb) return;
        acc |= (uint64_t)(v & (nb >= 32 ? 0xFFFFFFFFu : ((1u << nb) - 1u))) << n; n += nb;
        while (n >= 8) { o.push_back((uint8_t)acc); acc >>= 8; n -= 8; }
    }
    void flush() { if (n > 0) { o.push_back((uint8_t)acc); acc = 0; n = 0; } }
    uint64_t bits() const { return (uint64_t)o.size() * 8 + (uint64_t)n; }
};

using Vp8lHuffScratch = dfl::HuffScratchN<VP8L_NGREEN>;

struct PrefixCode { std::vector<uint8_t> len; std::vector<uint16_t> code; int used = 0; };

// code lengths (limit 15) and canonical codes (bit-reversed for LSB-first output) of freq[0 .. n), n <= VP8L_NGREEN
void vp8l_make_code(const std::vector<uint32_t> &freq, PrefixCode &pc, Vp8lHuffScratch &S);
// the code's description in the bitstream
void vp8l_write_code(BitsLsb &bw, const PrefixCode &pc, Vp8lHuffScratch &S);
// one symbol; a code with a single symbol takes no bits
inline void vp8l_put_sym(BitsLsb &bw, const PrefixCode &pc, int s) { if (pc.used > 1) bw.put(pc.code[s], pc.len[s]); }

} // namespace b200
