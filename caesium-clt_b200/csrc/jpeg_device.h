// jpeg_device.h -- device side of the JPEG path: per-GPU slot pools (stream + pinned staging + HBM buffers),
// work-list construction for the transform kernels, and the megabatch (K same-shaped images per launch sequence).
#pragma once
#include <cstdint>
#include <cstddef>
#include <memory>
#include <string>
#include <vector>
#include "dev_buffer.h"
#include "jpeg_host.h"
#include "jpeg_kernels.h"
#include "jpeg_gpudec.h"
#include "jpeg_gpuenc.h"

namespace b200 {

enum CompPath { PATH_FUSED = 0, PATH_C420 = 1, PATH_GENERIC = 2 };

// Per-image HBM footprint and per-component routing for an (input geometry, output geometry) pair.
struct ImagePlan {
    int path[4] = {0, 0, 0, 0};
    size_t in_bytes = 0, out_bytes = 0;
    size_t plane_off[4] = {0}, full_off[4] = {0}, dplane_off[4] = {0};
    size_t plane_bytes = 0, full_bytes = 0, dplane_bytes = 0;
    size_t scratch_bytes() const { return plane_bytes + full_bytes + dplane_bytes; }
};
bool plan_image(const JpegGeom &gin, const JpegGeom &gout, ImagePlan &plan, std::string &err);

// Work lists for one launch group (any number of images).  A non-empty trel list (every output-side item, see add_trellis_work)
// makes the FDCT kernels store raw DCT output and k_jpeg_trellis quantise it, with the JtTable array trel_t beside QuantDev trel_q.
struct WorkLists {
    std::vector<CompWork> fused, idct, c420, up, down, fdct, trel;
    int max_fused = 0, max_idct = 0, max_c420 = 0, max_fdct = 0, max_up_w = 0, max_up_h = 0, max_dn_w = 0, max_dn_h = 0, max_trel = 0;
    const QuantDev *trel_q = nullptr; const JtTable *trel_t = nullptr;
    size_t total() const { return fused.size() + idct.size() + c420.size() + up.size() + down.size() + fdct.size() + trel.size(); }
    void clear() { fused.clear(); idct.clear(); c420.clear(); up.clear(); down.clear(); fdct.clear(); trel.clear(); max_fused = max_idct = max_c420 = max_fdct = max_up_w = max_up_h = max_dn_w = max_dn_h = max_trel = 0; trel_q = nullptr; trel_t = nullptr; }
};
// Append one image's work.  d_dq: device uint16[4][64] (per input component, zigzag); d_q: device QuantDev[4] (per output slot).
void append_image_work(const JpegGeom &gin, const JpegGeom &gout, const ImagePlan &plan,
                       const int16_t *d_in, int16_t *d_out, uint8_t *d_scratch,
                       const uint16_t *d_dq, const QuantDev *d_q, WorkLists &wl);
// Copy lists into `h_work` (contiguous, order fused|idct|c420|up|down|fdct|trel); returns count.
size_t flatten_work(const WorkLists &wl, CompWork *h_work);
// Launch every non-empty list; d_work is the device copy of the flattened array.
int launch_work(const WorkLists &wl, const CompWork *d_work, void *stream);

// Trellis quantisation of lossy JPEG output (jpeg_trellis_core.h): the process-wide switch b200_set_jpeg_trellis sets; while never
// set, B200_JPEG_TRELLIS=1 turns it on (read once).  Off by default.  The transforms read it when they build their work lists; the
// resident pipe reads it once, at create.
bool jpeg_trellis();
void set_jpeg_trellis(bool on);

// ---- device runtime ------------------------------------------------------------------------------------------
struct PngDevice;
struct WebpDevice;
struct Vp8lDevice;
struct GifDevice;
struct Slot {
    int dev = 0;
    void *stream = nullptr;
    PinnedBuffer<int16_t> h_in, h_out;
    DeviceBuffer<int16_t> d_in, d_out;
    DeviceBuffer<uint8_t> d_scratch;
    PinnedBuffer<uint8_t> h_par; DeviceBuffer<uint8_t> d_par;                           // parameter block
    unsigned long long generation = 0;                                                   // bumped when d_in, d_out, d_scratch, h_par or d_par move
    std::unique_ptr<GpuEncoder> enc;                                                     // device entropy encoder (lazy)
    std::unique_ptr<GpuDecoder> dec;                                                     // device entropy decoder (lazy)
    std::unique_ptr<PngDevice> png;                                                      // lossless PNG state (lazy, png_device.cu)
    std::unique_ptr<WebpDevice> webp;                                                    // WebP / VP8 state (lazy, webp_device.cu)
    std::unique_ptr<Vp8lDevice> vp8l;                                                    // lossless WebP / VP8L state (lazy, vp8l_encode.cpp)
    std::unique_ptr<GifDevice> gif;                                                      // GIF state (lazy, gif_device.cu)
    // megabatch path: transform work lists of the current megabatch, and the captured launch sequence (two CUDA graphs, see
    // slot_run_group) with the signature it was captured for
    WorkLists group_wl; size_t group_par_bytes = 0, group_work_off = 0;
    void *graph_front = nullptr, *graph_back = nullptr; unsigned long long graph_sig = 0; bool graphs_broken = false;
    bool ensure(size_t in_bytes, size_t out_bytes, size_t scratch_bytes, size_t par_bytes, std::string &err);
    bool ensure_device(size_t in_bytes, size_t out_bytes, size_t scratch_bytes, size_t par_bytes, std::string &err);
    // the coders, created on first use
    GpuEncoder *encoder();
    GpuDecoder *decoder();
    PngDevice *png_dev();
    WebpDevice *webp_dev();
    Vp8lDevice *vp8l_dev();
    GifDevice *gif_dev();
    Slot();
    Slot(const Slot &) = delete;
    Slot &operator=(const Slot &) = delete;
    ~Slot();        // destroys the stream and the graphs, then the members free every buffer; the caller has made the slot's device current and its stream idle
};

int  runtime_init(int n_gpus, int only_device, std::string &err);   // returns device count (>0) or 0 with err
void runtime_shutdown();
int  runtime_device_count();
Slot *slot_acquire(int prefer_dev, std::string &err);               // blocks while all slots of the device are busy
void slot_release(Slot *s);
int  runtime_next_device();                                         // round-robin shard assignment
long long runtime_device_jobs(int dev_index);                       // slot acquisitions on that device so far
int  runtime_device_ordinal(int dev_index);                         // CUDA ordinal of the library's device number dev_index

// Run the transform for ONE image whose input coefficients already sit in s->h_in; result lands in s->h_out.
bool slot_transform(Slot *s, const JpegGeom &gin, const JpegGeom &gout, std::string &err, bool download = true, bool upload = true);
// D2H of the output coefficients left in HBM by a download=false transform (host-encoder fallback)
bool slot_download_coefs(Slot *s, size_t out_bytes, std::string &err);
// Entropy-decode a baseline single-scan file on the device into s->d_in (0 ok, 1 not converged -> host decode, 2 failed)
int slot_gpu_decode(Slot *s, const JpegReader &rd, const JpegReader::DeviceScan &ds, std::string &err);
// ---- megabatch (K same-shaped images per launch sequence; used by b200_compress_batch) ---------------------------------
struct GroupLayout {
    int K = 0; size_t in_stride = 0, out_stride = 0, scratch_stride = 0;
    // image k's coefficients: its input in s.d_in, or its output in s.d_out
    int16_t *coefs(const Slot &s, int k, bool input) const
    {
        return reinterpret_cast<int16_t *>(reinterpret_cast<uint8_t *>((input ? s.d_in : s.d_out).get()) + (input ? in_stride : out_stride) * k);
    }
};
bool slot_group_layout(Slot *s, const JpegGeom &gin, const JpegGeom &gout, int K, GroupLayout &L, std::string &err);   // sizes + ensure()
// one launch sequence serves images of one size, component count and sampling
inline bool same_shape(const JpegGeom &a, const JpegGeom &b)
{
    bool same = a.width == b.width && a.height == b.height && a.ncomp == b.ncomp;
    for (int c = 0; same && c < a.ncomp; c++) same = a.hs[c] == b.hs[c] && a.vs[c] == b.vs[c];
    return same;
}
// decode -> (transform) -> encode of one megabatch enqueued back to back, one idle host wait at the end; results in s->enc->results,
// items[k].result says which images the device decoder settled
bool slot_run_group(Slot *s, std::vector<GpuDecoder::Item> &items, const JpegGeom *const *gins, const JpegGeom &gout, const GroupLayout &L, bool progressive,
                    bool lossless, std::string &err);
bool slot_transform_group(Slot *s, const JpegGeom *const *gins, const JpegGeom &gout, const GroupLayout &L, bool trellis, std::string &err);
// H2D of s->h_out into s->d_out (entry point that encodes caller-supplied coefficients on the device)
bool slot_upload_out_coefs(Slot *s, size_t bytes, std::string &err);
// Entropy-code the output coefficients sitting in s->d_out on the device; result in s->enc->results
bool slot_gpu_encode(Slot *s, const JpegGeom &gout, bool progressive, std::string &err, bool from_input = false);
// the same without fetching the stuffed scans (results carry lengths only); slot_gpu_fetch() brings them over afterwards
bool slot_gpu_encode_sizes(Slot *s, const JpegGeom &gout, bool progressive, std::string &err);
bool slot_gpu_fetch(Slot *s, std::string &err);
// Resize path (CSParameters.width/height): gout carries the TARGET dimensions; decode -> RGB -> Lanczos3 -> YCbCr -> encode.
// rgb_out != nullptr: stop after the resize and hand back the three device planes (R, G, B of the TARGET size, pitch = target
// width; a greyscale source returns its single plane three times) -- the front end of the format-conversion paths.
// host_rgb != nullptr: the source is not a JPEG -- planar samples [ncomp][H][W] (RGB, or one grey plane) replace the decode
// front end; gin then only carries width / height / ncomp with 1x1 sampling.
bool slot_transform_resized(Slot *s, const JpegGeom &gin, const JpegGeom &gout, std::string &err, bool download = true, bool upload = true,
                            uint8_t **rgb_out = nullptr, const uint8_t *host_rgb = nullptr);
// D2H of nplanes device planes of n bytes each (rgb_out of slot_transform_resized) into one host buffer, synchronised
bool slot_fetch_planes(Slot *s, uint8_t *const *d_planes, int nplanes, size_t n, uint8_t *host, std::string &err);
// Same front end, but stop after IDCT + upsample and copy planar full-res samples into `planes` (host).
bool slot_decode_planes(Slot *s, const JpegGeom &gin, uint8_t *planes, std::string &err);

} // namespace b200
