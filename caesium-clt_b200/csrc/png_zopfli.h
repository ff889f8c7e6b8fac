// png_zopfli.h -- the device side of the PNG `--zopfli` leg (png_zopfli.cu): an iterated optimal LZ77 parse over the rules of
// png_zopfli_core.h.
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>
#include "dev_buffer.h"

namespace b200 {

struct PngZopfli {
    DeviceBuffer<uint32_t> d_key, d_key2, d_val, d_val2, d_ent, d_bp, d_tok, d_best, d_segc, d_segn, d_offsets, d_hg, d_ha, d_hb, d_cost;
    DeviceBuffer<int32_t> d_prev;
    DeviceBuffer<unsigned long long> d_state;
    DeviceBuffer<uint8_t> d_temp, d_z;
    // The optimal parse of d_filt[0, n) (filter distance bpp, row stride), compacted into d_out (n words); its per-segment token
    // counts stay in d_segn and their exclusive prefix sum in d_offsets (nseg() entries).  d_gtok / d_gcounts: the greedy / lazy
    // parse of the same stream as k_png_parse left it (chunk-local slots of gchunk positions), whose statistics seed iteration 1.
    // Everything is enqueued on `stream`, with no host wait.
    bool tokens(const uint8_t *d_filt, size_t n, int bpp, int stride, const uint32_t *d_gtok, const uint32_t *d_gcounts, int gchunk, uint32_t *d_out,
                void *stream, std::string &err);
    static size_t nseg(size_t n);
};

} // namespace b200
