// jpeg_gpuenc.h -- device-side JPEG entropy encoder (see jpeg_gpuenc.cu / jpeg_gpuenc_core.h).
#pragma once
#include <cstdint>
#include <cstddef>
#include <string>
#include <vector>
#include "dev_buffer.h"
#include "jpeg_gpuenc_plan.h"

namespace b200 {

struct DhtOut { uint8_t bits[17]; uint8_t vals[256]; int32_t nvals; };
struct ScanOut { uint32_t total_bits, nbytes, word_base, arena_base; };   // filled on the device (k_ge_scanout)

// One encoder instance per slot (or per megabatch): owns its device / pinned buffers and grows them on demand.
class GpuEncoder {
public:
    GpuEncoder() = default;
    ~GpuEncoder();
    GpuEncoder(const GpuEncoder &) = delete;
    GpuEncoder &operator=(const GpuEncoder &) = delete;
    // Entropy-code `nimages` coefficient buffers of geometry g that already sit in device memory.  On success
    // results[image * scans_per_image + k] describes scan k (pointers into this object's pinned buffer, valid until the next call).
    // out_bytes_hint: expected total size of the entropy-coded output (0 = unknown); the output-side buffers are sized from it and
    // the pass sequence is repeated with exact sizes if it was too small.
    bool encode(const JpegGeom &g, bool progressive, int16_t *const *d_coefs, int nimages, void *stream, bool fill_dummy, std::string &err, size_t out_bytes_hint = 0);
    // The same in three steps (see jpeg_gpuenc.cu): prepare() sizes buffers and uploads descriptors, enqueue() launches every pass
    // without waiting (may be repeated on unchanged inputs), finish() waits, fetches the stuffed scans (fetch = false: leaves them
    // in HBM; results[].data == nullptr, lengths valid) and describes the result.
    bool prepare(const JpegGeom &g, bool progressive, int16_t *const *d_coefs, int nimages, void *stream, size_t out_bytes_hint, std::string &err);   // host work only
    bool upload(void *stream, std::string &err);                       // H2D of the descriptors
    bool enqueue(void *stream, bool fill_dummy, std::string &err);     // = front + sizes + mark + back
    // the pieces, for callers that replay the sequence as CUDA graphs (front + sizes in one graph, mark_sizes as a plain event
    // record, back in a second graph); signature() identifies the driver calls they would make
    bool enqueue_front(void *stream, bool fill_dummy, std::string &err);
    bool enqueue_sizes(void *stream, std::string &err);
    bool mark_sizes(void *stream, std::string &err);
    bool enqueue_back(void *stream, std::string &err);
    unsigned long long signature() const;
    bool finish(void *stream, bool fetch, std::string &err);
    int retries = 0;            // back halves repeated because the output estimate was too small
    double wait_sizes_ms = 0, wait_final_ms = 0;   // host time spent in finish()'s two waits (tracing)
    std::vector<EncodedScan> results;
    GpuEncPlan plan;
    bool overflow = false;      // the failure was "scan larger than its buffer": the caller may use the host encoder
    int launches = 0;
private:
    bool size_back_buffers(size_t image_bytes, std::string &err);
    unsigned long long generation = 0;      // bumped by every reallocation: captured graphs hold the old addresses
    int cap_nimg = 0;
    int nimg = 0;
    JpegGeom geom; bool prog = false;
    std::vector<int16_t *> coef_bases;
    void *ev_sizes = nullptr;
    uint32_t words_cap = 0;
    size_t est_image_bytes = 0, learned_image_bytes = 0, learned_for = 0;
    DeviceBuffer<uint32_t> d_flags;
    size_t o_scans = 0, o_total = 0, o_outlen = 0, o_dht = 0, o_comps = 0, o_flags = 0;
    DeviceBuffer<ge::Scan> d_scans;
    DeviceBuffer<BlockComp> d_comps;
    DeviceBuffer<uint32_t> d_meta, d_tail, d_tsum, d_gcount;
    DeviceBuffer<uint32_t> d_bitlen, d_bitoff;          // per unit of the interleaved scans coded unit by unit (Scan::lu_base)
    DeviceBuffer<int16_t> d_dc;                         // compact DC arrays for the DC-first interleaved scan (k_geb_classify, k_geb_dc_first)
    DeviceBuffer<uint32_t> d_corr;                      // correction bits per scan (k_geb_classify)
    DeviceBuffer<unsigned long long> d_tbits;           // bits coded with each table (k_ge_tables)
    DeviceBuffer<uint32_t> d_cursor, d_runlen, d_runoff, d_runpos, d_arena;   // CTA runs of the single-component scans (k_geb_emit, k_ge_place)
    DeviceBuffer<int> d_evkey, d_prev;
    DeviceBuffer<uint32_t> d_hist;
    DeviceBuffer<ge::Table> d_tabs;
    DeviceBuffer<DhtOut> d_dht;
    DeviceBuffer<uint32_t> d_total;
    DeviceBuffer<ScanOut> d_so;
    DeviceBuffer<uint32_t> d_words;
    DeviceBuffer<ge::Masks3> d_masks;                   // threshold masks per block, written by the classify pass
    DeviceBuffer<uint32_t> d_chunkff;                   // 0xFF bytes per chunk of each scan (k_ge_ffcount)
    DeviceBuffer<uint32_t> d_outoff, d_outlen;
    DeviceBuffer<uint8_t> d_out;
    DeviceBuffer<uint8_t> d_temp;
    PinnedBuffer<uint8_t> h_small;
    PinnedBuffer<uint8_t> h_out;
    size_t out_stride = 0, copy_bytes = 0;
};

} // namespace b200
