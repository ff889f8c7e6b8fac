// CPU run of the Adam7 geometry (csrc/png_adam7_core.h) that k_png_adam7_unfilter / k_png_adam7_gather and the host decoder use:
// the pass table, sizes and offsets, and the gather of full-image rows from pass-packed rows, serially.  The test compares the
// results with a Python restatement.  Test infrastructure only.
#include <cstdint>
#include <cstddef>
#include "../../caesium-clt_b200/csrc/png_adam7_core.h"

using namespace b200;

// out: per pass w, h, rb, filt_off, raw_off (35 values), then filt_bytes and raw_bytes
extern "C" void emul_adam7_layout(uint32_t w, uint32_t h, int bits, uint64_t *out)
{
    Adam7Layout L;
    adam7_layout(w, h, bits, L);
    for (int p = 0; p < 7; p++) {
        const Adam7Pass &P = L.pass[p];
        const uint64_t v[5] = {P.w, P.h, P.rb, P.filt_off, P.raw_off};
        for (int k = 0; k < 5; k++) out[5 * p + k] = v[k];
    }
    out[35] = L.filt_bytes; out[36] = L.raw_bytes;
}

// packed: the passes' un-filtered rows one after another (L.raw_bytes); raw: h rows of (w * bits + 7) / 8 bytes
extern "C" void emul_adam7_gather(const uint8_t *packed, uint32_t w, uint32_t h, int bits, uint8_t *raw)
{
    Adam7Layout L;
    adam7_layout(w, h, bits, L);
    const size_t rb = ((size_t)w * bits + 7) / 8;
    for (uint32_t y = 0; y < h; y++)
        for (size_t i = 0; i < rb; i++) raw[(size_t)y * rb + i] = adam7_gather_byte(packed, L, bits, w, y, i);
}
