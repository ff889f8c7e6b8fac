// jpeg_gpuenc_stuff_core.h -- 0xFF byte stuffing of the device encoder's output scans: the per-thread bodies of k_ge_ffcount and
// k_ge_scatter (jpeg_gpuenc.cu), written once as __host__ __device__ code; tests/emul/stuff_emul.cpp runs the same bodies CTA by
// CTA on the CPU against a plain byte loop.
//
// A scan's unstuffed bytes are its bit buffer's words, big-endian within a word, with the padding ones of jchuff.c's flush_bits
// in the last byte (bytes past the scan's nbytes are not part of it).  k_ge_scanout starts every scan's words at a multiple of
// four words, so group g (bytes 16 g .. 16 g + 15) is one 16-byte load.  The groups are cut into tiles of `tile` groups, one per
// thread of a CTA, and the tiles into `nchunks` contiguous chunks, one per CTA: the number of 0xFF bytes in a chunk is all that the
// other CTAs of the scan need to know about it.
#pragma once
#include "jpeg_gpuenc_core.h"

namespace b200 {
namespace ge {

struct ScanGroup { uint32_t w[4]; };    // words 4 g .. 4 g + 3 of the scan's bit buffer, as read

// the groups [g0, g1) of chunk x: whole tiles, ceil(tiles / nchunks) per chunk (the last chunks may be short or empty)
GE_HD void stuff_chunk(uint32_t nbytes, uint32_t x, uint32_t nchunks, uint32_t tile, uint32_t &g0, uint32_t &g1)
{
    const uint32_t ng = (nbytes + 15) / 16, ntiles = (ng + tile - 1) / tile, per = (ntiles + nchunks - 1) / nchunks * tile;
    g0 = x * per < ng ? x * per : ng;
    g1 = (x + 1) * per < ng ? (x + 1) * per : ng;
}

// Group g (16 g < nbytes) as it goes out: the padding ones ORed into the scan's last byte, the bytes past it cleared (a cleared
// byte is 0x00, so it is never counted as an 0xFF).  Returns the group's byte count: 16, or fewer in the scan's last group.
GE_HD uint32_t stuff_group(ScanGroup &q, uint32_t g, uint32_t nbytes, uint32_t total_bits)
{
    const uint32_t left = nbytes - g * 16, n = left < 16 ? left : 16;
    const uint32_t pad = (total_bits & 7) ? (1u << (8 - (total_bits & 7))) - 1u : 0u;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int k = 0; k < 4; k++) {
        const int nk = (int)n - 4 * k;                              // bytes of word k that belong to the scan
        uint32_t w = nk <= 0 ? 0u : nk >= 4 ? q.w[k] : q.w[k] & ~(0xFFFFFFFFu >> (8 * nk));
        if (n == left && nk >= 1 && nk <= 4) w |= pad << (8 * (4 - nk));   // the scan's last byte is byte nk - 1 of word k
        q.w[k] = w;
    }
    return n;
}

// 0xFF bytes in a word: a byte of ~w is non-zero iff its high bit survives ((v & 0x7F) + 0x7F) | v, which carries into no
// neighbour
GE_HD uint32_t ff_bytes(uint32_t w)
{
    const uint32_t v = ~w;
    return (uint32_t)popc64(~(((v & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | v) & 0x80808080u);
}
GE_HD uint32_t stuff_ff_count(const ScanGroup &q) { return ff_bytes(q.w[0]) + ff_bytes(q.w[1]) + ff_bytes(q.w[2]) + ff_bytes(q.w[3]); }

// The group's n bytes, each 0xFF followed by a stuffed 0x00, at sb[o], sb[o + 1], ...; returns the position after them.
GE_HD uint32_t stuff_place_group(const ScanGroup &q, uint32_t n, uint32_t o, uint8_t *sb)
{
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int t = 0; t < 16; t++) {
        if ((uint32_t)t >= n) break;
        const uint32_t b = (q.w[t >> 2] >> (24 - 8 * (t & 3))) & 0xFFu;
        sb[o++] = (uint8_t)b;
        if (b == 0xFF) sb[o++] = 0;
    }
    return o;
}

// Thread `tid` of `nthreads` stores the output range [first, end) from the word buffer sbuf (word i = output bytes aligned + 4 i
// .. + 3, aligned = first & ~3, out 4-byte aligned): whole aligned words, except the words at either end of the range, which the
// neighbouring tile, chunk or scan shares and which leave byte by byte (gd::unstuff_store's rule).
GE_HD void stuff_store(const uint32_t *sbuf, uint32_t aligned, uint32_t first, uint32_t end, uint32_t tid, uint32_t nthreads, uint8_t *out)
{
    for (uint32_t a = aligned + 4 * tid; a < end; a += 4 * nthreads) {
        const uint32_t w = sbuf[(a - aligned) >> 2];
        if (a >= first && a + 4 <= end) *reinterpret_cast<uint32_t *>(out + a) = w;
        else for (uint32_t t = 0; t < 4; t++) if (a + t >= first && a + t < end) out[a + t] = (uint8_t)(w >> (8 * t));
    }
}

} // namespace ge
} // namespace b200
