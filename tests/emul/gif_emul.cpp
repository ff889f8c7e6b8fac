// The GIF leg's LZW walk (gif_core.h) compiled for the CPU, for tests/test_gif_host.py: the segments of n indices, packed as the
// device packs them (LSB first, no break between segments) and sub-blocked.
#include <cstdint>
#include <cstring>
#include <vector>
#include "../../caesium-clt_b200/csrc/gif_core.h"

using namespace b200;

extern "C" long long emul_gif_lzw(const uint8_t *idx, size_t n, int m, int seg, uint8_t *out, size_t cap)
{
    const size_t nseg = n ? (n + seg - 1) / seg : 1;
    std::vector<uint32_t> table(GIF_HASH);
    std::vector<uint16_t> codes((size_t)seg + seg / 1024 + 4);
    std::vector<uint8_t> bytes(nseg * codes.size() * 12 / 8 + 8, 0);
    unsigned long long bit = 0;
    for (size_t s = 0; s < nseg; s++) {
        const size_t at = s * seg, len = n - at < (size_t)seg ? n - at : (size_t)seg;
        unsigned b = 0;
        const int nc = gif_lzw_segment(idx + at, (int)len, m, s == 0, s == nseg - 1, table.data(), codes.data(), &b);
        for (int k = 0; k < nc; k++)
            for (int j = 0; j < (codes[k] >> 12); j++, bit++) bytes[bit >> 3] |= (uint8_t)((((codes[k] & 4095u) >> j) & 1) << (bit & 7));
    }
    const size_t nbytes = (size_t)((bit + 7) / 8), total = gif_blocks_size(nbytes);
    if (total > cap) return -1;
    for (size_t i = 0; i < total; i++) out[i] = gif_blocks_byte(bytes.data(), nbytes, i);
    return (long long)total;
}
