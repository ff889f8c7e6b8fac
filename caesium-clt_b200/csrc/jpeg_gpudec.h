// jpeg_gpudec.h -- device-side JPEG entropy DECODER for baseline single-scan files (see jpeg_gpudec_core.h), batched:
// one pass sequence decodes any number of images (blockIdx.y = image).
#pragma once
#include <cstdint>
#include <cstddef>
#include <string>
#include <vector>
#include "dev_buffer.h"
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
    GpuDecoder(const GpuDecoder &) = delete;
    GpuDecoder &operator=(const GpuDecoder &) = delete;
    enum Result { OK = 0, NOT_CONVERGED = 1, FAILED = 2 };
    // defer_dc: leave each block's DC difference in the block and skip the DC scatter; whoever reads the blocks adds the prefix
    // sum from dc_sums() instead (the transform kernels do, CompWork::dc_sum).  One setting per batch.
    struct Item { const JpegReader *rd; const JpegReader::DeviceScan *ds; int16_t *d_coefs; Result result; bool defer_dc = false; };
    // Decode every item's scan straight into its d_coefs (device; fully overwritten, whatever it held before).  Per item: OK, or NOT_CONVERGED
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
    // Where the final DC of item n's frame component c comes from after enqueue() of a defer_dc batch: the DC of the block at
    // (bx, by) of the component is sum[slot] - (prev ? *prev : 0), slot = ((by / vs) * mcux + bx / hs) * hs * vs + (by % vs) * hs +
    // bx % hs.  sum = null when the batch does not defer the DC (the blocks hold it) or c is not in the scan.
    struct DcSums { const int32_t *sum, *prev; int hs, vs, mcux; };
    DcSums dc_sums(int n, int c) const;
    size_t raw_bytes() const { return raw_total; }          // entropy-coded bytes staged by the last prepare()
    int rounds_used = 0, launches = 0;
    // subsequence size: swept 512 .. 8192 on the 4K bench set under full batch load (tools/throughput.py): 512 -> 3,400
    // images/s, 1024 -> 3,750, 2048 -> 3,970, 4096 -> 3,865, 8192 -> 3,560 (B200_DEC_SUBSEQ overrides)
    // ROUNDS: synchronisation rounds launched per batch, without a host check in between (a round whose image settled in an earlier
    // one leaves at once: ~2 us); the 4K bench set settles in <= 14.  An image that needs more is decoded on the host.
    static constexpr int SUBSEQ_BITS = 2048, ROUNDS = 24, MAX_ROUNDS = 64;
private:
    int nitems = 0; bool defer_dc = false;
    std::vector<DecImage> imgs; std::vector<int16_t *> coef_ptrs; std::vector<size_t> coef_bytes; std::vector<char> tables_ok;
    size_t raw_total = 0, o_img = 0, o_tab = 0, o_flag = 0, o_mark = 0, par_bytes = 0;
    size_t hw_raw = 0, hw_stream = 0, hw_grp = 0, hw_sub = 0, hw_blk = 0, hw_mgrp = 0, hw_msub = 0, hw_mblk = 0; int hw_n = 0;
    unsigned long long generation = 0;          // bumped by every reallocation: captured graphs hold the old addresses
    uint32_t grp_total = 0, sub_total = 0, blk_total = 0, max_grp = 0, max_sub = 0, max_blk = 0;
    PinnedBuffer<uint8_t> h_raw;                        // staging of the entropy-coded segments
    DeviceBuffer<uint8_t> d_raw, d_stream;
    DeviceBuffer<uint32_t> d_cnt, d_off;
    DeviceBuffer<gd::DecState> d_A;                     // exit state per subsequence (updated in place)
    DeviceBuffer<uint8_t> d_chgA, d_chgB;               // epoch of the last change per subsequence; dirty flags per CTA (x2)
    DeviceBuffer<uint32_t> d_nblk, d_first;
    DeviceBuffer<int32_t> d_dc, d_dcs;
    DeviceBuffer<uint8_t> d_par; PinnedBuffer<uint8_t> h_par;   // DecImage[] | DecTables[] | round flags
    DeviceBuffer<uint8_t> d_temp;
};

} // namespace b200
