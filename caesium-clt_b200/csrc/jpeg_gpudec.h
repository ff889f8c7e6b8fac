// jpeg_gpudec.h -- device-side JPEG entropy DECODER for baseline single-scan files (see jpeg_gpudec_core.h), batched:
// one pass sequence decodes any number of images (blockIdx.y = image).
#pragma once
#include <cstdint>
#include <cstddef>
#include <string>
#include <vector>
#include "jpeg_gpudec_core.h"
#include "jpeg_host.h"

namespace b200 {

struct DecImage {               // one image of a decode batch (device-visible)
    uint32_t raw_off, nraw;     // entropy-coded segment inside the batch's raw buffer
    uint32_t stream_off;        // unstuffed stream inside the batch's stream buffer (word aligned, 0xFF padded)
    uint32_t grp_off, ngrp;     // 16-byte groups of the raw segment (un-stuffing)
    uint32_t sub_off;           // first subsequence of this image in the state arrays
    uint32_t blk_off;           // first block of this image in the DC arrays
    uint32_t verify;            // 1: the host did not walk the segment -- the un-stuff pass counts stuffed bytes (g.nbits / g.nsub are
                                // upper bounds until it has) and reports markers inside the segment
    gd::Geometry g;
    ge::Scan scan;              // output addressing (scan.coef = this image's coefficient buffer)
    gd::Walk walk;              // the same, in the division-free form the write pass steps through
};

class GpuDecoder {
public:
    GpuDecoder() = default;
    ~GpuDecoder();
    GpuDecoder(const GpuDecoder &) = delete;
    GpuDecoder &operator=(const GpuDecoder &) = delete;
    enum Result { OK = 0, NOT_CONVERGED = 1, FAILED = 2 };
    struct Item { const JpegReader *rd; const JpegReader::DeviceScan *ds; int16_t *d_coefs; Result result; };
    // Decode every item's scan straight into its d_coefs (device; fully overwritten).  Per item: OK, or NOT_CONVERGED
    // (the self-synchronisation did not settle within the round budget -- degenerate periodic streams -- or the stream is
    // damaged: a marker inside it, an invalid code, a run past index 63 or an end before the last block; the caller
    // decodes that image on the host instead).  Returns false on a CUDA failure.  Asynchronous work on `stream`, with one
    // short host sync per group of rounds.
    bool decode(std::vector<Item> &items, void *stream, std::string &err);
    // the same in steps: prepare() stages inputs and descriptors (H2D enqueued), enqueue() launches every pass without a host
    // wait (repeatable on unchanged inputs), finish() -- after the caller has waited for the stream -- fills items[].result
    bool prepare(std::vector<Item> &items, void *stream, std::string &err);       // host work only: nothing is put on the stream
    bool upload(void *stream, std::string &err);                                  // H2D of the staged inputs
    bool enqueue(void *stream, std::string &err);
    // identity of the launch sequence upload() + enqueue() would issue: equal signatures = the same driver calls with the same
    // arguments (sizes are high-water marks), i.e. a captured CUDA graph of them can be replayed
    unsigned long long signature() const;
    void finish(std::vector<Item> &items);
    size_t raw_bytes() const { return raw_total; }          // entropy-coded bytes staged by the last prepare()
    int rounds_used = 0, launches = 0;
    // subsequence size: swept 512 .. 8192 on the 4K bench set under full batch load (tools/throughput.py): 512 -> 3,400
    // images/s, 1024 -> 3,750, 2048 -> 3,970, 4096 -> 3,865, 8192 -> 3,560 (B200_DEC_SUBSEQ overrides)
    // ROUNDS: synchronisation rounds launched per batch, without a host check in between (a round whose image settled in an earlier
    // one leaves at once: ~2 us); the 4K bench set settles in <= 14.  An image that needs more is decoded on the host.
    static constexpr int SUBSEQ_BITS = 2048, ROUNDS = 24, MAX_ROUNDS = 64;
private:
    int nitems = 0;
    std::vector<DecImage> imgs; std::vector<int16_t *> coef_ptrs; std::vector<size_t> coef_bytes; std::vector<char> tables_ok;
    size_t raw_total = 0, o_img = 0, o_tab = 0, o_flag = 0, o_mark = 0, par_bytes = 0;
    size_t hw_raw = 0, hw_stream = 0, hw_grp = 0, hw_sub = 0, hw_blk = 0, hw_mgrp = 0, hw_msub = 0, hw_mblk = 0; int hw_n = 0;
    unsigned long long generation = 0;
    uint32_t grp_total = 0, sub_total = 0, blk_total = 0, max_grp = 0, max_sub = 0, max_blk = 0;
    uint8_t *h_raw = nullptr; size_t cap_hraw = 0;          // pinned staging of the entropy-coded segments
    uint8_t *d_raw = nullptr, *d_stream = nullptr; size_t cap_raw = 0, cap_stream = 0;
    uint32_t *d_cnt = nullptr, *d_off = nullptr; size_t cap_cnt = 0, cap_off = 0;
    gd::DecState *d_A = nullptr; size_t cap_A = 0;                             // exit state per subsequence (updated in place)
    uint8_t *d_chgA = nullptr, *d_chgB = nullptr; size_t cap_chgA = 0, cap_chgB = 0;   // epoch of the last change per subsequence; dirty flags per CTA (x2)
    uint32_t *d_nblk = nullptr, *d_first = nullptr; size_t cap_nblk = 0, cap_first = 0;
    int32_t *d_dc = nullptr, *d_dcs = nullptr; size_t cap_dc = 0, cap_dcs = 0;
    uint8_t *d_par = nullptr, *h_par = nullptr; size_t cap_par = 0, cap_hpar = 0;   // DecImage[] | DecTables[] | round flags
    uint8_t *d_temp = nullptr; size_t cap_temp = 0;
};

} // namespace b200
