// vp8l_kernels.h -- launchers of the lossless WebP (VP8L) encoder's kernels (vp8l_kernels.cu); the buffers are Vp8lDevice's.
#pragma once
#include <cstddef>
#include <cstdint>
#include <vector_types.h>
#include "vp8l_enc_core.h"
#include "vp8l_palette_core.h"

namespace b200 {

// the chosen prefix codes, laid out like one candidate's histograms (VP8L_HIST); a code with one symbol has length 0 everywhere
struct Vp8lCodes { uint16_t code[VP8L_HIST]; uint8_t len[VP8L_HIST]; };

struct Vp8lBuffers {
    uint8_t *planes;                    // R | G | B | A planes of n bytes each: the host entry's upload
    uint32_t *argb, *res, *best;        // n each: subtract-green pixels, residuals, best copy per pixel
    uint8_t *modes;                     // one per 16x16 tile
    int *cache_tab;                     // vp8l_cache_table_ints(nchunks)
    uint8_t *hits;                      // (VP8L_NCACHE - 1) x n
    uint2 *tok; uint32_t *cnt;          // n tokens (chunk b's at b * VP8L_CHUNK), nchunks counts
    uint32_t *hist;                     // VP8L_NCACHE x VP8L_HIST
    uint32_t *flags;                    // bit 0: some alpha below 255
    Vp8lCodes *codes;
    uint32_t *thread_off;               // nchunks x 256
    unsigned long long *chunk_bits, *chunk_start, *total;
    uint32_t *words;                    // the coded pixels, zeroed by launch_vp8l_emit
    unsigned long long *pal_set;        // VP8L_PAL_SET: the colours seen, as a set (vp8l_palette.cu)
    uint32_t *pal_info;                 // VP8L_PAL_INFO: colour count, overflow flag (over VP8L_PAL_MAX colours), ascending palette
};

size_t vp8l_cache_table_ints(int nchunks);
// R, G, B planes (+ alpha; nullptr: opaque) of w x h bytes anywhere on the device -> B.argb (subtract-green) and B.flags
int launch_vp8l_pack(const uint8_t *r, const uint8_t *g, const uint8_t *b, const uint8_t *a, const Vp8lBuffers &B, int w, int h, void *stream);
// predictor choice, colour-cache hits, match search, parse and the histograms of every cache candidate over B.argb
int launch_vp8l_analyse(const Vp8lBuffers &B, int w, int h, void *stream);
// the same without the predictor: B.res already holds the w x h pixels to code (the palette variant's packed index image)
int launch_vp8l_analyse_res(const Vp8lBuffers &B, int w, int h, void *stream);
// the colours of B.argb (w x h) -> B.pal_info (vp8l_palette.cu)
int launch_vp8l_palette(const Vp8lBuffers &B, int w, int h, void *stream);
// B.argb (w x h) -> B.res: the packed index image under B.pal_info's palette of `count` colours, vp8l_pal_width(w, xbits) x h
int launch_vp8l_palette_pack(const Vp8lBuffers &B, int w, int h, int count, void *stream);
// bit offsets of every chunk's and thread's tokens under B.codes for cache candidate `cand`; *B.total = bit_base + their bits
int launch_vp8l_size(const Vp8lBuffers &B, int w, int h, int cand, unsigned long long bit_base, void *stream);
// the tokens into B.words (words of them are zeroed first)
int launch_vp8l_emit(const Vp8lBuffers &B, int w, int h, int cand, size_t words, void *stream);

} // namespace b200
