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
#include "resize_kernels.h"

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
                       const uint16_t *d_dq, const QuantDev *d_q, WorkLists &wl, const GpuDecoder::DcSums *dc = nullptr);   // dc[c]: see CompWork::dc_sum
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
struct WebpAnimDevice;
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
    std::unique_ptr<WebpAnimDevice> webp_anim;                                           // animated WebP state (lazy, webp_anim_device.cu)
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
    WebpAnimDevice *webp_anim_dev();
    Resampler resampler{Grow::Slot};                                                     // K3 of the sample stages
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
// D2H of the output coefficients left in HBM by a download=false transform or coefs_from_samples (host encoder)
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
// D2H of nplanes device planes of n bytes each into one host buffer, synchronised
bool slot_fetch_planes(Slot *s, uint8_t *const *d_planes, int nplanes, size_t n, uint8_t *host, std::string &err);

// ---- sample stages: 8-bit planar samples on the slot, between a decode front end, K3 and the encode back end -------------------
// A caller chains them: samples_from_coefs or samples_from_host -> resize_samples -> coefs_from_samples (then the device entropy
// encoder, or slot_download_coefs for the host one), an encoder that reads device planes, or slot_fetch_planes.  Two facts of the
// slot make plan_samples fix every stage's region of d_scratch and of the parameter block before anything is enqueued:
// - Buffer::reserve frees the old memory, so a stage that grew a buffer would destroy the previous stage's output in it: nothing
//   grows between the stages of one chain.
// - h_par is pinned and goes up with cudaMemcpyAsync, and the stages of one chain do not wait for the stream: a stage that rewrote a
//   region an earlier stage has queued for upload would corrupt the queued copy.  So each stage writes and uploads only its own
//   regions (QuantDev q[4] at the start and the sink's work after the front end's), and the trellis tables stay at the end.
// The resize's tables and intermediate live in the slot's Resampler, which no other stage touches.
struct SamplePlan {
    int nc = 0, w = 0, h = 0, nw = 0, nh = 0;
    bool trellis = false;                     // coefs_from_samples runs the trellis pass (jpeg_trellis() when planned)
    // d_scratch: front's IDCT planes, then the full-resolution planes.  Every component takes PATH_GENERIC (IDCT + upsample), and
    // front.plane_bytes also holds the resized planes and the sink's downsampled planes: they are written after the IDCT planes die.
    ImagePlan front;
    size_t rz_off[4] = {0}, dpl_off[4] = {0};
    size_t in_bytes = 0, out_bytes = 0, scratch_bytes = 0, par_bytes = 0;
    size_t sink_off = 0;                      // the sink's work descriptors in the parameter block, after the front end's
};
// The chain from gin's samples (a JPEG's, or planar_geom for host planes) to nw x nh, and on to the coefficients of gout when the chain
// ends in coefs_from_samples (else gout is null).  Sizes the slot with one ensure().  Fails on fractional sampling ratios.
bool plan_samples(Slot *s, const JpegGeom &gin, int nw, int nh, const JpegGeom *gout, SamplePlan &p, std::string &err);
// Dequantisation, IDCT and upsampling of the coefficients in s->d_in (upload: s->h_in goes up first) into full-resolution planes,
// converted YCbCr -> RGB in place when rgb is set and there are three components.
bool samples_from_coefs(Slot *s, const JpegGeom &gin, const SamplePlan &p, bool upload, bool rgb, uint8_t **planes, std::string &err);
// host planes [nc][h][w] into the full-resolution planes
bool samples_from_host(Slot *s, const uint8_t *host, const SamplePlan &p, uint8_t **planes, std::string &err);
// K3 of the planes `in` to nw x nh; `out` are the resized planes, or `in` itself at the same size
bool resize_samples(Slot *s, uint8_t *const *in, const SamplePlan &p, uint8_t **out, std::string &err);
// RGB -> YCbCr in place (three components), K4 downsampling, K5 FDCT + quantisation (and the trellis pass) into s->d_out
bool coefs_from_samples(Slot *s, uint8_t *const *planes, const JpegGeom &gout, const SamplePlan &p, std::string &err);

} // namespace b200
