// jpeg_device.cu -- see jpeg_device.h.  Device runtime for the JPEG path of caesium::compress_in_memory
// (caesium-clt's src/compressor.rs:305): one pool of "slots" per GPU so that the blocking, one-image-per-thread
// callers of the reference's rayon map (compressor.rs:81-83) each get a private stream, pinned staging buffers and
// HBM buffers; images are sharded round-robin over the initialised GPUs (no cross-GPU traffic on this path).
#include <cuda_runtime.h>
#include <malloc.h>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <condition_variable>
#include <cstring>
#include <mutex>
#include <vector>
#include <atomic>
#include "jpeg_device.h"
#include "resize_kernels.h"
#include "jpeg_gpuenc.h"
#include "jpeg_gpudec.h"
#include "png_device.h"
#include "webp_device.h"
#include "vp8l_device.h"
#include "gif_device.h"
#include "webp_anim_device.h"
#include "stream_wait.h"
#include "launch_timer.h"

namespace b200 {

thread_local LaunchTimer *tl_launch_timer = nullptr;

static constexpr size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

bool plan_image(const JpegGeom &gin, const JpegGeom &gout, ImagePlan &p, std::string &err)
{
    p = ImagePlan();
    if (gin.ncomp != gout.ncomp || gin.width != gout.width || gin.height != gout.height) { err = "geometry mismatch between decode and encode side"; return false; }
    p.in_bytes = (size_t)gin.total_coefs * 2; p.out_bytes = (size_t)gout.total_coefs * 2;
    size_t off_plane = 0, off_full = 0, off_d = 0;
    for (int c = 0; c < gin.ncomp; c++) {
        if (gin.hmax % gin.hs[c] || gin.vmax % gin.vs[c] || gout.hmax % gout.hs[c] || gout.vmax % gout.vs[c]) { err = "fractional sampling ratio unsupported"; return false; }
        int uhx = gin.hmax / gin.hs[c], uvx = gin.vmax / gin.vs[c], dhx = gout.hmax / gout.hs[c], dvx = gout.vmax / gout.vs[c];
        if (uhx == 1 && uvx == 1 && dhx == 1 && dvx == 1) p.path[c] = PATH_FUSED;
        else if (uhx == 2 && uvx == 2 && dhx == 2 && dvx == 2) p.path[c] = PATH_C420;
        else p.path[c] = PATH_GENERIC;
        if (p.path[c] != PATH_FUSED) { p.plane_off[c] = off_plane; off_plane += align_up((size_t)gin.bw[c] * 8 * gin.bh[c] * 8, 256); }
        if (p.path[c] == PATH_GENERIC) {
            p.full_off[c] = off_full; off_full += align_up((size_t)gin.width * gin.height, 256);
            p.dplane_off[c] = off_d; off_d += align_up((size_t)gout.rbw[c] * 8 * gout.rbh[c] * 8, 256);
        }
    }
    p.plane_bytes = off_plane; p.full_bytes = off_full; p.dplane_bytes = off_d;
    return true;
}

void append_image_work(const JpegGeom &gin, const JpegGeom &gout, const ImagePlan &plan,
                       const int16_t *d_in, int16_t *d_out, uint8_t *d_scratch,
                       const uint16_t *d_dq, const QuantDev *d_q, WorkLists &wl, const GpuDecoder::DcSums *dc)
{
    for (int c = 0; c < gin.ncomp; c++) {
        CompWork w; memset(&w, 0, sizeof(w));
        w.cin = d_in + gin.comp_offset[c]; w.cout = d_out + gout.comp_offset[c];
        w.dq = d_dq + 64 * c; w.q = d_q + gout.tq[c];
        if (dc && dc[c].sum) { w.dc_sum = dc[c].sum; w.dc_prev = dc[c].prev; w.dc_hs = dc[c].hs; w.dc_vs = dc[c].vs; w.dc_mcux = dc[c].mcux; }
        w.bw_in = gin.bw[c]; w.bh_in = gin.bh[c]; w.rbw_in = gin.rbw[c]; w.rbh_in = gin.rbh[c]; w.cw = gin.cw[c]; w.ch = gin.ch[c];
        w.bw_out = gout.bw[c]; w.bh_out = gout.bh[c]; w.rbw_out = gout.rbw[c]; w.rbh_out = gout.rbh[c];
        w.W = gin.width; w.H = gin.height;
        w.pstride = gin.bw[c] * 8; w.fstride = gin.width;
        w.up_hx = gin.hmax / gin.hs[c]; w.up_vx = gin.vmax / gin.vs[c];
        w.dn_hx = gout.hmax / gout.hs[c]; w.dn_vx = gout.vmax / gout.vs[c];
        if (plan.path[c] != PATH_FUSED) w.plane = d_scratch + plan.plane_off[c];
        if (plan.path[c] == PATH_GENERIC) {
            w.full = d_scratch + plan.plane_bytes + plan.full_off[c];
            w.dplane = d_scratch + plan.plane_bytes + plan.full_bytes + plan.dplane_off[c];
        }
        const int t_in = work_tiles(w.rbw_in, w.rbh_in), t_out = work_tiles(w.rbw_out, w.rbh_out);
        switch (plan.path[c]) {
            case PATH_FUSED: wl.fused.push_back(w); wl.max_fused = std::max(wl.max_fused, t_out); break;
            case PATH_C420:
                wl.idct.push_back(w); wl.max_idct = std::max(wl.max_idct, t_in);
                wl.c420.push_back(w); wl.max_c420 = std::max(wl.max_c420, t_out);
                break;
            default:
                wl.idct.push_back(w); wl.max_idct = std::max(wl.max_idct, t_in);
                wl.up.push_back(w); wl.max_up_w = std::max(wl.max_up_w, w.W); wl.max_up_h = std::max(wl.max_up_h, w.H);
                wl.down.push_back(w); wl.max_dn_w = std::max(wl.max_dn_w, w.rbw_out * 8); wl.max_dn_h = std::max(wl.max_dn_h, w.rbh_out * 8);
                wl.fdct.push_back(w); wl.max_fdct = std::max(wl.max_fdct, t_out);
        }
    }
}

size_t flatten_work(const WorkLists &wl, CompWork *h)
{
    size_t n = 0;
    for (const auto *v : {&wl.fused, &wl.idct, &wl.c420, &wl.up, &wl.down, &wl.fdct, &wl.trel}) { if (!v->empty()) memcpy(h + n, v->data(), v->size() * sizeof(CompWork)); n += v->size(); }
    return n;
}

int launch_work(const WorkLists &wl, const CompWork *d, void *stream)
{
    int rc = 0;
    const CompWork *p_fused = d, *p_idct = p_fused + wl.fused.size(), *p_c420 = p_idct + wl.idct.size();
    const CompWork *p_up = p_c420 + wl.c420.size(), *p_down = p_up + wl.up.size(), *p_fdct = p_down + wl.down.size();
    const CompWork *p_trel = p_fdct + wl.fdct.size();
    const bool raw = !wl.trel.empty();
    if (!wl.fused.empty()) { rc = launch_fused_same(p_fused, (int)wl.fused.size(), wl.max_fused, stream, raw); LT_MARK("k_fused_same"); if (rc) return rc; }
    if (!wl.idct.empty()) { rc = launch_idct_plane(p_idct, (int)wl.idct.size(), wl.max_idct, stream); LT_MARK("k_idct_plane"); if (rc) return rc; }
    if (!wl.c420.empty()) { rc = launch_chroma420_refdct(p_c420, (int)wl.c420.size(), wl.max_c420, stream, raw); LT_MARK("k_chroma420_refdct"); if (rc) return rc; }
    if (!wl.up.empty()) { rc = launch_upsample(p_up, (int)wl.up.size(), wl.max_up_w, wl.max_up_h, stream); if (rc) return rc; }
    if (!wl.down.empty()) { rc = launch_downsample(p_down, (int)wl.down.size(), wl.max_dn_w, wl.max_dn_h, stream); if (rc) return rc; }
    if (!wl.fdct.empty()) { rc = launch_fdct_plane(p_fdct, (int)wl.fdct.size(), wl.max_fdct, stream, raw); if (rc) return rc; }
    if (raw) { rc = launch_jpeg_trellis(p_trel, (int)wl.trel.size(), wl.max_trel, wl.trel_q, wl.trel_t, stream); LT_MARK("k_jpeg_trellis"); if (rc) return rc; }
    return 0;
}

// every output-side item of wl (the ones an FDCT kernel writes) into its trellis list
static void add_trellis_work(WorkLists &wl)
{
    for (const auto *v : {&wl.fused, &wl.c420, &wl.fdct})
        for (const CompWork &w : *v) { wl.trel.push_back(w); wl.max_trel = std::max(wl.max_trel, w.rbw_out * w.rbh_out); }
}

namespace {
std::atomic<int> g_jpeg_trellis{-1};     // -1 unset (env B200_JPEG_TRELLIS); 1 = trellis quantisation, 0 = plain
}
bool jpeg_trellis()
{
    if (g_jpeg_trellis.load() < 0) {
        const char *e = getenv("B200_JPEG_TRELLIS");
        g_jpeg_trellis.store(e && !strcmp(e, "1") ? 1 : 0);
    }
    return g_jpeg_trellis.load() == 1;
}
void set_jpeg_trellis(bool on) { g_jpeg_trellis.store(on ? 1 : 0); }

// ================================================================================================================
// runtime: devices and slots
// ================================================================================================================
namespace {
struct DevicePool {
    int ordinal = 0;
    std::mutex mu; std::condition_variable cv;
    std::vector<Slot *> free_slots; int created = 0; int max_slots = 48;
    std::atomic<long long> jobs{0};             // slot acquisitions (a megabatch or a single image each)
};
std::mutex g_mu;
std::vector<DevicePool *> g_devs;
std::atomic<unsigned> g_rr{0};
bool g_inited = false;
}

int runtime_init(int n_gpus, int only_device, std::string &err)
{
    std::lock_guard<std::mutex> lk(g_mu);
    if (g_inited) return (int)g_devs.size();
    int count = 0;
    // How callers wait for their stream is decided in stream_wait.h (hybrid poll-then-sleep by default); B200_SYNC=block
    // additionally asks the driver for blocking synchronisation (no-op if a context already exists, e.g. torch's).
    // One stream per in-flight image, dozens in flight: with the default 8 hardware work queues, streams alias onto the
    // same queue and serialise behind each other.  32 is the maximum; only effective if set before the context exists.
    setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32", 0);
    const bool blocking = stream_wait_mode() == 1;
    // Every image hands a freshly malloc'ed file (~1 MB) to the caller, thousands per second from several threads.  With
    // glibc's defaults each of those is an mmap + page faults + munmap (or a heap that is trimmed back to the OS as soon as
    // the caller frees), all serialised on the process's mmap lock: measured, that alone cost 45 % of the end-to-end rate.
    // Keep freed memory in the allocator instead.  B200_MALLOPT=0 leaves the process's malloc settings untouched.
    {
        const char *mo = getenv("B200_MALLOPT");
        if (!(mo && !strcmp(mo, "0"))) { mallopt(M_MMAP_THRESHOLD, 32 << 20); mallopt(M_TRIM_THRESHOLD, 2000000000); mallopt(M_TOP_PAD, 64 << 20); }
    }
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count <= 0) { err = std::string("no CUDA device available (") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count 0") + "); this build has no CPU fallback"; return 0; }
    std::vector<int> ords;
    if (only_device >= 0) { if (only_device >= count) { err = "CUDA device ordinal out of range"; return 0; } ords.push_back(only_device); }
    else { int n = n_gpus <= 0 ? count : std::min(n_gpus, count); for (int i = 0; i < n; i++) ords.push_back(i); }
    for (int o : ords) {
        if (blocking && cudaSetDevice(o) == cudaSuccess) { cudaSetDeviceFlags(cudaDeviceScheduleBlockingSync); cudaGetLastError(); }
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, o) != cudaSuccess) { err = "cudaGetDeviceProperties failed"; return 0; }
        if (prop.major != 9 || prop.minor != 0) { err = "device " + std::to_string(o) + " is sm_" + std::to_string(prop.major) + std::to_string(prop.minor) + "; this library ships sm_90a kernels only"; for (auto *d : g_devs) delete d; g_devs.clear(); return 0; }
        auto *d = new DevicePool(); d->ordinal = o; g_devs.push_back(d);
    }
    g_inited = true;
    return (int)g_devs.size();
}

static void print_group_trace();
static void drop_graphs(Slot *s);
void runtime_shutdown()
{
    print_group_trace();
    std::lock_guard<std::mutex> lk(g_mu);
    for (auto *d : g_devs) {
        cudaSetDevice(d->ordinal);
        for (Slot *s : d->free_slots) delete s;
        delete d;
    }
    g_devs.clear(); g_inited = false;
}

Slot::~Slot()
{
    if (stream) cudaStreamDestroy((cudaStream_t)stream);
    drop_graphs(this);
}

Slot::Slot() = default;

GpuEncoder *Slot::encoder() { if (!enc) enc.reset(new GpuEncoder()); return enc.get(); }
GpuDecoder *Slot::decoder() { if (!dec) dec.reset(new GpuDecoder()); return dec.get(); }
PngDevice *Slot::png_dev() { if (!png) png.reset(new PngDevice()); return png.get(); }
WebpDevice *Slot::webp_dev() { if (!webp) webp.reset(new WebpDevice()); return webp.get(); }
Vp8lDevice *Slot::vp8l_dev() { if (!vp8l) vp8l.reset(new Vp8lDevice()); return vp8l.get(); }
GifDevice *Slot::gif_dev() { if (!gif) gif.reset(new GifDevice()); return gif.get(); }
WebpAnimDevice *Slot::webp_anim_dev() { if (!webp_anim) webp_anim.reset(new WebpAnimDevice()); return webp_anim.get(); }

int runtime_device_count() { std::lock_guard<std::mutex> lk(g_mu); return g_inited ? (int)g_devs.size() : 0; }
long long runtime_device_jobs(int i) { return g_devs.empty() || i < 0 || i >= (int)g_devs.size() ? 0 : g_devs[(size_t)i]->jobs.load(); }
int runtime_device_ordinal(int i) { return g_devs.empty() ? 0 : g_devs[(size_t)i % g_devs.size()]->ordinal; }
int runtime_next_device() { size_t n = g_devs.size(); return n ? (int)(g_rr.fetch_add(1) % n) : 0; }

Slot *slot_acquire(int prefer, std::string &err)
{
    if (g_devs.empty()) { err = "library not initialised (no CUDA device)"; return nullptr; }
    DevicePool *d = g_devs[(size_t)prefer % g_devs.size()];
    d->jobs++;
    std::unique_lock<std::mutex> lk(d->mu);
    for (;;) {
        if (!d->free_slots.empty()) { Slot *s = d->free_slots.back(); d->free_slots.pop_back(); lk.unlock(); cudaSetDevice(d->ordinal); return s; }
        if (d->created < d->max_slots) {
            d->created++; lk.unlock();
            cudaSetDevice(d->ordinal);
            Slot *s = new Slot(); s->dev = (int)((size_t)prefer % g_devs.size());
            cudaStream_t st;
            if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) { delete s; err = "cudaStreamCreate failed"; lk.lock(); d->created--; return nullptr; }
            s->stream = st;
            return s;
        }
        d->cv.wait(lk);
    }
}

void slot_release(Slot *s)
{
    if (!s) return;
    DevicePool *d = g_devs[(size_t)s->dev];
    { std::lock_guard<std::mutex> lk(d->mu); d->free_slots.push_back(s); }
    d->cv.notify_one();
}

bool Slot::ensure_device(size_t in_bytes, size_t out_bytes, size_t scratch_bytes, size_t par_bytes, std::string &err)
{   // megabatch path: coefficients never visit the host, so only the HBM side (and the small parameter block) grows
    return d_in.reserve(in_bytes, Grow::Slot, err, &generation) && d_out.reserve(out_bytes, Grow::Slot, err, &generation) &&
           d_scratch.reserve(std::max<size_t>(scratch_bytes, 256), Grow::Slot, err, &generation) &&
           h_par.reserve(par_bytes, Grow::Slot, err, &generation) && d_par.reserve(par_bytes, Grow::Slot, err, &generation);
}

bool Slot::ensure(size_t in_bytes, size_t out_bytes, size_t scratch_bytes, size_t par_bytes, std::string &err)
{
    return h_in.reserve(in_bytes, Grow::Slot, err) && h_out.reserve(out_bytes, Grow::Slot, err) &&
           ensure_device(in_bytes, out_bytes, scratch_bytes, par_bytes, err);
}

// Parameter block of a transform over K images, each part 256-byte aligned:
//   QuantDev q[4] (per output table) | uint16 dq[K][4][64] (per image and input component, zigzag) | CompWork work[]
// With trellis quantisation on, JtTable[4] (beside q[4], per output table) comes last.  The sample stages lay out K = 1 the same way
// (see SamplePlan).
static constexpr size_t par_dq_off = align_up(sizeof(QuantDev) * 4, 256);
static size_t par_work_off(int K) { return par_dq_off + align_up(sizeof(uint16_t) * 256 * K, 256); }
static constexpr size_t par_trellis_bytes = 256 + sizeof(JtTable) * 4;      // alignment + the tables
// the trellis tables of gout at the 256-aligned end `end` of the block; returns the new end
static size_t put_trellis(Slot *s, const JpegGeom &gout, size_t end, WorkLists &wl)
{
    const size_t off = align_up(end, 256);
    JtTable *t = reinterpret_cast<JtTable *>(s->h_par + off);
    for (int i = 0; i < 4; i++) if (gout.qt_present[i]) jt_make_table(gout.qt[i], i != 0, &t[i]);
    add_trellis_work(wl);
    wl.trel_q = reinterpret_cast<const QuantDev *>(s->d_par.get());
    wl.trel_t = reinterpret_cast<const JtTable *>(s->d_par + off);
    return off + sizeof(JtTable) * 4;
}

static void put_quant(Slot *s, const JpegGeom &gout)
{
    QuantDev *q = reinterpret_cast<QuantDev *>(s->h_par.get());
    for (int t = 0; t < 4; t++) if (gout.qt_present[t]) make_quant_dev(gout.qt[t], &q[t]);
}
static const QuantDev *dev_quant(const Slot *s) { return reinterpret_cast<const QuantDev *>(s->d_par.get()); }
// image k's dequantisation tables into the pinned block; returns where the kernels read them
static const uint16_t *put_dequant(Slot *s, int k, const JpegGeom &gin)
{
    uint16_t *dq = reinterpret_cast<uint16_t *>(s->h_par + par_dq_off) + 256 * k;
    for (int c = 0; c < gin.ncomp; c++) memcpy(dq + 64 * c, gin.qt[gin.tq[c]], 128);
    return reinterpret_cast<const uint16_t *>(s->d_par + par_dq_off) + 256 * k;
}

// Quantiser constants, per-image dequantisation tables and the work descriptors of the K images of L into the slot's pinned
// parameter block.  wl receives the work lists, par_bytes the size of the block, work_off the offset of the descriptors.
// dec: the decoder that decoded the K images of a megabatch (their DC from its prefix sums when it deferred the DC), or null
static bool fill_transform_params(Slot *s, const JpegGeom *const *gins, const JpegGeom &gout, const GroupLayout &L, bool trellis, const GpuDecoder *dec,
                                  WorkLists &wl, size_t &par_bytes, size_t &work_off, std::string &err)
{
    put_quant(s, gout);
    wl.clear();
    for (int k = 0; k < L.K; k++) {
        const JpegGeom &gin = *gins[k];
        ImagePlan plan;
        if (!plan_image(gin, gout, plan, err)) return false;
        GpuDecoder::DcSums dc[4];
        for (int c = 0; c < 4; c++) dc[c] = dec ? dec->dc_sums(k, c) : GpuDecoder::DcSums{nullptr, nullptr, 1, 1, 1};
        append_image_work(gin, gout, plan, L.coefs(*s, k, true), L.coefs(*s, k, false), s->d_scratch + L.scratch_stride * k,
                          put_dequant(s, k, gin), dev_quant(s), wl, dc);
    }
    work_off = par_work_off(L.K);
    if (!trellis) { par_bytes = work_off + flatten_work(wl, reinterpret_cast<CompWork *>(s->h_par + work_off)) * sizeof(CompWork); return true; }
    const size_t end = work_off + (wl.total() + wl.fused.size() + wl.c420.size() + wl.fdct.size()) * sizeof(CompWork);
    par_bytes = put_trellis(s, gout, end, wl);
    flatten_work(wl, reinterpret_cast<CompWork *>(s->h_par + work_off));
    return true;
}

bool slot_transform(Slot *s, const JpegGeom &gin, const JpegGeom &gout, std::string &err, bool download, bool upload)
{
    ImagePlan plan;
    if (!plan_image(gin, gout, plan, err)) return false;
    cudaStream_t st = (cudaStream_t)s->stream;
    if (!s->ensure(plan.in_bytes, plan.out_bytes, plan.scratch_bytes(), par_work_off(1) + sizeof(CompWork) * 4 * 7 + par_trellis_bytes, err)) return false;
    // a megabatch of one over the slot's own buffers (no strides needed); the work lists are local because s->group_wl and
    // the group_* sizes belong to the slot's last megabatch and feed the signature of its captured launch sequence
    GroupLayout L; L.K = 1;
    const JpegGeom *gins = &gin;
    WorkLists wl; size_t pbytes = 0, work_off = 0;
    if (!fill_transform_params(s, &gins, gout, L, jpeg_trellis(), nullptr, wl, pbytes, work_off, err)) return false;
    CU(cudaMemcpyAsync(s->d_par, s->h_par, pbytes, cudaMemcpyHostToDevice, st));
    if (upload) CU(cudaMemcpyAsync(s->d_in, s->h_in, plan.in_bytes, cudaMemcpyHostToDevice, st));
    const int rc = launch_work(wl, reinterpret_cast<const CompWork *>(s->d_par + work_off), st);
    if (!launch_ok(rc, "kernel launch", err)) return false;
    if (!download) return true;          // the coefficients stay in HBM for the device entropy encoder
    CU(cudaMemcpyAsync(s->h_out, s->d_out, plan.out_bytes, cudaMemcpyDeviceToHost, st));
    CU(stream_wait(st));
    return true;
}

// ---- megabatch: K same-shaped images per launch sequence (b200_compress_batch) -------------------------------------
// Buffers of image k live at d_in + k * in_stride etc.; the input coefficients are already in HBM (device decoder) and
// the output coefficients stay there (device encoder).
bool slot_group_layout(Slot *s, const JpegGeom &gin, const JpegGeom &gout, int K, GroupLayout &L, std::string &err)
{
    ImagePlan plan;
    if (!plan_image(gin, gout, plan, err)) return false;
    L.K = K;
    L.in_stride = align_up(plan.in_bytes, 256); L.out_stride = align_up(plan.out_bytes, 256); L.scratch_stride = align_up(std::max<size_t>(plan.scratch_bytes(), 256), 256);
    const size_t par = par_work_off(K) + sizeof(CompWork) * (size_t)K * 4 * 7 + 256 + par_trellis_bytes;
    return s->ensure_device(L.in_stride * K, L.out_stride * K, L.scratch_stride * K, par, err);
}

// host half: the parameter block into the slot's pinned memory, the work lists into s->group_wl
bool slot_transform_group_prepare(Slot *s, const JpegGeom *const *gins, const JpegGeom &gout, const GroupLayout &L, bool trellis, std::string &err)
{
    return fill_transform_params(s, gins, gout, L, trellis, s->dec.get(), s->group_wl, s->group_par_bytes, s->group_work_off, err);
}
// stream half: parameter block up, the transform kernels
bool slot_transform_group_enqueue(Slot *s, std::string &err)
{
    cudaStream_t st = (cudaStream_t)s->stream;
    CU(cudaMemcpyAsync(s->d_par, s->h_par, s->group_par_bytes, cudaMemcpyHostToDevice, st));
    const int rc = launch_work(s->group_wl, reinterpret_cast<const CompWork *>(s->d_par + s->group_work_off), st);
    if (!launch_ok(rc, "kernel launch", err)) return false;
    return true;
}
bool slot_transform_group(Slot *s, const JpegGeom *const *gins, const JpegGeom &gout, const GroupLayout &L, bool trellis, std::string &err)
{
    return slot_transform_group_prepare(s, gins, gout, L, trellis, err) && slot_transform_group_enqueue(s, err);
}

// (Measured and dropped: issuing the decode passes on a highest-priority stream so that their small latency-bound grids cut in
// front of other megabatches' 24k-CTA encoder grids LOWERED the batch rate by 20 % -- 4,430 -> 3,550 images/s with 8 group
// workers, 4,690 -> 4,030 with 16.  Everything of a megabatch stays on the slot's one stream.)
//
// One megabatch, front to back, with ONE host wait that leaves the GPU idle (the last): entropy decode (fixed number of rounds,
// flags read afterwards), transform, entropy encode (its sizes come back while the emit kernels run).  Round 1 waited three
// times per megabatch with an empty stream behind each wait.
// B200_TRACE: host wall-clock per megabatch, summed: staging (copy into pinned + tables), launching, the two waits
static std::atomic<long long> g_grp_ns[5];
static std::atomic<long long> g_grp_n{0};
static const bool g_grp_trace = getenv("B200_TRACE") != nullptr;
static void print_group_trace()
{
    const long long n = g_grp_n.load();
    if (!g_grp_trace || !n) return;
    static const char *names[] = {"stage inputs (memcpy to pinned, tables, H2D enqueue)", "enqueue decode + transform + encode (launch overhead)", "wait: sizes (GPU still busy)", "wait: final (after D2H enqueue)", "whole megabatch on the host"};
    fprintf(stderr, "[b200 trace] %lld megabatches; mean host ms per megabatch:\n", n);
    for (int i = 0; i < 5; i++) fprintf(stderr, "[b200 trace]   %-58s %8.3f\n", names[i], g_grp_ns[i].load() / 1e6 / (double)n);
}

// The launch sequence of a megabatch is ~70 driver calls (kernels, CUB scans, memsets, small copies).  Sixteen worker threads
// issuing them concurrently spend more time in the driver's process-wide lock than the kernels take to run (B200_TRACE showed
// 1.8 ms of pure enqueue time per megabatch, 24 us per call), and that -- not the GPU -- capped the C-ABI rate at 85 % of the
// device-resident rate.  The sequence is the same from megabatch to megabatch (sizes are high-water marks, buffers are reused), so
// it is captured once per slot as two CUDA graphs -- everything up to the scan sizes, and the bit-packing / stuffing half -- and
// replayed: three driver calls per megabatch.  A changed signature (other geometry, a grown buffer, a new high-water mark)
// re-captures.  B200_GRAPHS=0 issues the calls directly.
static bool graphs_enabled() { static const bool on = [] { const char *e = getenv("B200_GRAPHS"); return !(e && !strcmp(e, "0")); }(); return on; }
static void drop_graphs(Slot *s)
{
    if (s->graph_front) { cudaGraphExecDestroy((cudaGraphExec_t)s->graph_front); s->graph_front = nullptr; }
    if (s->graph_back) { cudaGraphExecDestroy((cudaGraphExec_t)s->graph_back); s->graph_back = nullptr; }
    s->graph_sig = 0;
}
template <class Fn> static bool capture_graph(cudaStream_t st, void *&exec_out, Fn fn, std::string &err)
{
    if (cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) != cudaSuccess) { cudaGetLastError(); return false; }
    const bool ok = fn();
    cudaGraph_t g = nullptr;
    const cudaError_t e = cudaStreamEndCapture(st, &g);
    if (!ok || e != cudaSuccess || !g) { if (g) cudaGraphDestroy(g); cudaGetLastError(); if (err.empty()) err = "graph capture failed"; return false; }
    cudaGraphExec_t ex = nullptr;
    const cudaError_t ei = cudaGraphInstantiate(&ex, g, 0);
    cudaGraphDestroy(g);
    if (ei != cudaSuccess) { cudaGetLastError(); err = std::string("cudaGraphInstantiate: ") + cudaGetErrorString(ei); return false; }
    exec_out = ex;
    return true;
}

bool slot_run_group(Slot *s, std::vector<GpuDecoder::Item> &items, const JpegGeom *const *gins, const JpegGeom &gout, const GroupLayout &L, bool progressive,
                    bool lossless, std::string &err)
{
    cudaStream_t st = (cudaStream_t)s->stream;
    const auto t0 = std::chrono::steady_clock::now();
    // ---- host half of all three stages (pinned staging, descriptors, plans); nothing touches the stream yet
    for (GpuDecoder::Item &it : items) it.defer_dc = !lossless;       // the transform adds the DC; --lossless encodes the blocks as decoded
    if (!s->decoder()->prepare(items, st, err)) return false;
    if (!lossless && !slot_transform_group_prepare(s, gins, gout, L, jpeg_trellis(), err)) return false;
    std::vector<int16_t *> bases((size_t)L.K);
    for (int k = 0; k < L.K; k++) bases[k] = L.coefs(*s, k, lossless);
    // a re-encode at lower quality (or a transcode with optimal tables) does not grow: the inputs' entropy-coded size sizes the output buffers
    if (!s->encoder()->prepare(gout, progressive, bases.data(), L.K, st, s->dec->raw_bytes(), err)) return false;
    const auto t1 = std::chrono::steady_clock::now();
    auto front = [&]() { return s->dec->upload(st, err) && s->dec->enqueue(st, err) && (lossless || slot_transform_group_enqueue(s, err)) &&
                                s->enc->upload(st, err) && s->enc->enqueue_front(st, true, err) && s->enc->enqueue_sizes(st, err); };
    auto back = [&]() { return s->enc->enqueue_back(st, err); };
    bool launched = false;
    if (graphs_enabled() && !s->graphs_broken) {
        unsigned long long sig = s->dec->signature() * 1099511628211ull ^ s->enc->signature();
        sig = (sig ^ s->generation ^ ((unsigned long long)s->group_par_bytes << 20) ^ (lossless ? 0x9e3779b97f4a7c15ull : 0)) * 1099511628211ull + (unsigned long long)L.K;
        if (!lossless && !s->group_wl.trel.empty()) sig = (sig ^ 0xc2b2ae3d27d4eb4full) * 1099511628211ull;     // the trellis pass is part of the sequence
        if (!s->graph_front || s->graph_sig != sig) {
            drop_graphs(s);
            std::string gerr;
            if (capture_graph(st, s->graph_front, front, gerr) && capture_graph(st, s->graph_back, back, gerr)) s->graph_sig = sig;
            else { drop_graphs(s); s->graphs_broken = true; }      // capture not possible here: issue the calls directly from now on
        }
        if (s->graph_front && s->graph_back) {
            if (cudaGraphLaunch((cudaGraphExec_t)s->graph_front, st) != cudaSuccess || !s->enc->mark_sizes(st, err) ||
                cudaGraphLaunch((cudaGraphExec_t)s->graph_back, st) != cudaSuccess) { err = std::string("cudaGraphLaunch: ") + cudaGetErrorString(cudaGetLastError()); return false; }
            launched = true;
        }
    }
    if (!launched && !(front() && s->enc->mark_sizes(st, err) && back())) return false;
    const auto t2 = std::chrono::steady_clock::now();
    if (!s->enc->finish(st, true, err)) return false;
    s->dec->finish(items);
    if (g_grp_trace) {
        const auto t3 = std::chrono::steady_clock::now();
        auto ns = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return (long long)std::chrono::duration_cast<std::chrono::nanoseconds>(b - a).count(); };
        g_grp_ns[0] += ns(t0, t1); g_grp_ns[1] += ns(t1, t2); g_grp_ns[2] += (long long)(s->enc->wait_sizes_ms * 1e6); g_grp_ns[3] += (long long)(s->enc->wait_final_ms * 1e6);
        g_grp_ns[4] += ns(t0, t3); g_grp_n++;
    }
    return true;
}

bool slot_download_coefs(Slot *s, size_t out_bytes, std::string &err)
{
    cudaStream_t st = (cudaStream_t)s->stream;
    CU(cudaMemcpyAsync(s->h_out, s->d_out, out_bytes, cudaMemcpyDeviceToHost, st));
    CU(stream_wait(st));
    return true;
}

int slot_gpu_decode(Slot *s, const JpegReader &rd, const JpegReader::DeviceScan &ds, std::string &err)
{   // 0 = coefficients are in s->d_in, 1 = not converged (decode on the host instead), 2 = failure
    std::vector<GpuDecoder::Item> items(1);
    items[0].rd = &rd; items[0].ds = &ds; items[0].d_coefs = s->d_in; items[0].result = GpuDecoder::FAILED;
    if (!s->decoder()->decode(items, s->stream, err)) return 2;
    return (int)items[0].result;
}

bool slot_upload_out_coefs(Slot *s, size_t bytes, std::string &err)
{
    cudaStream_t st = (cudaStream_t)s->stream;
    CU(cudaMemcpyAsync(s->d_out, s->h_out, bytes, cudaMemcpyHostToDevice, st));
    return true;
}

bool slot_gpu_encode(Slot *s, const JpegGeom &gout, bool progressive, std::string &err, bool from_input)
{
    int16_t *base = from_input ? s->d_in : s->d_out;
    return s->encoder()->encode(gout, progressive, &base, 1, s->stream, true, err);
}

bool slot_gpu_encode_sizes(Slot *s, const JpegGeom &gout, bool progressive, std::string &err)
{
    GpuEncoder *enc = s->encoder();
    int16_t *base = s->d_out;
    return enc->prepare(gout, progressive, &base, 1, s->stream, 0, err) && enc->upload(s->stream, err) && enc->enqueue(s->stream, true, err) && enc->finish(s->stream, false, err);
}
bool slot_gpu_fetch(Slot *s, std::string &err) { return s->enc && s->enc->finish(s->stream, true, err); }

bool slot_fetch_planes(Slot *s, uint8_t *const *d_planes, int nplanes, size_t n, uint8_t *host, std::string &err)
{
    cudaStream_t st = (cudaStream_t)s->stream;
    for (int c = 0; c < nplanes; c++) CU(cudaMemcpyAsync(host + (size_t)c * n, d_planes[c], n, cudaMemcpyDeviceToHost, st));
    CU(stream_wait(st));
    return true;
}

bool plan_samples(Slot *s, const JpegGeom &gin, int nw, int nh, const JpegGeom *gout, SamplePlan &p, std::string &err)
{
    p = SamplePlan();
    const int nc = gin.ncomp;
    if (gout && gout->ncomp != nc) { err = "component count mismatch"; return false; }
    p.nc = nc; p.w = gin.width; p.h = gin.height; p.nw = nw; p.nh = nh;
    size_t idct = 0, later = 0;
    for (int c = 0; c < nc; c++) {
        if (gin.hmax % gin.hs[c] || gin.vmax % gin.vs[c] || (gout && (gout->hmax % gout->hs[c] || gout->vmax % gout->vs[c]))) { err = "fractional sampling ratio unsupported"; return false; }
        p.front.path[c] = PATH_GENERIC;
        p.front.plane_off[c] = idct; idct += align_up((size_t)gin.bw[c] * 8 * gin.bh[c] * 8, 256);
        p.front.full_off[c] = p.front.full_bytes; p.front.full_bytes += align_up((size_t)gin.width * gin.height, 256);
    }
    for (int c = 0; (nw != p.w || nh != p.h) && c < nc; c++) { p.rz_off[c] = later; later += align_up((size_t)nw * nh, 256); }
    for (int c = 0; gout && c < nc; c++) { p.dpl_off[c] = later; later += align_up((size_t)gout->rbw[c] * 8 * gout->rbh[c] * 8, 256); }
    p.front.plane_bytes = std::max(idct, later);
    p.in_bytes = (size_t)gin.total_coefs * 2; p.out_bytes = gout ? (size_t)gout->total_coefs * 2 : 0;
    p.scratch_bytes = p.front.scratch_bytes();
    p.trellis = gout && jpeg_trellis();
    p.sink_off = par_work_off(1) + sizeof(CompWork) * 2 * nc;                  // front end: idct, up
    p.par_bytes = !gout ? p.sink_off : p.sink_off + sizeof(CompWork) * 3 * nc + (p.trellis ? par_trellis_bytes : 0);     // down, fdct, trel
    return s->ensure(p.in_bytes, p.out_bytes, p.scratch_bytes, p.par_bytes, err);
}

bool samples_from_coefs(Slot *s, const JpegGeom &gin, const SamplePlan &p, bool upload, bool rgb, uint8_t **planes, std::string &err)
{
    cudaStream_t st = (cudaStream_t)s->stream;
    JpegGeom g444 = gin;            // every component through IDCT + upsampling: planned against a 4:4:4 output of the same size
    for (int c = 0; c < gin.ncomp; c++) g444.hs[c] = g444.vs[c] = 1;
    g444.finalize();
    WorkLists wl;
    append_image_work(gin, g444, p.front, s->d_in, s->d_out, s->d_scratch, put_dequant(s, 0, gin), dev_quant(s), wl);
    wl.down.clear(); wl.fdct.clear();
    const size_t work_off = par_work_off(1), end = work_off + flatten_work(wl, reinterpret_cast<CompWork *>(s->h_par + work_off)) * sizeof(CompWork);
    CU(cudaMemcpyAsync(s->d_par + par_dq_off, s->h_par + par_dq_off, end - par_dq_off, cudaMemcpyHostToDevice, st));
    if (upload) CU(cudaMemcpyAsync(s->d_in, s->h_in, p.in_bytes, cudaMemcpyHostToDevice, st));
    if (!launch_ok(launch_work(wl, reinterpret_cast<const CompWork *>(s->d_par + work_off), st), "kernel launch", err)) return false;
    for (int c = 0; c < p.nc; c++) planes[c] = s->d_scratch + p.front.plane_bytes + p.front.full_off[c];
    if (rgb && p.nc == 3 && !launch_ok(launch_ycc_to_rgb(planes[0], planes[1], planes[2], (size_t)p.w * p.h, st), "ycc_to_rgb", err)) return false;
    return true;
}

bool samples_from_host(Slot *s, const uint8_t *host, const SamplePlan &p, uint8_t **planes, std::string &err)
{
    const size_t n = (size_t)p.w * p.h;
    for (int c = 0; c < p.nc; c++) {
        planes[c] = s->d_scratch + p.front.plane_bytes + p.front.full_off[c];
        CU(cudaMemcpyAsync(planes[c], host + c * n, n, cudaMemcpyHostToDevice, (cudaStream_t)s->stream));
    }
    return true;
}

bool resize_samples(Slot *s, uint8_t *const *in, const SamplePlan &p, uint8_t **out, std::string &err)
{
    const bool same = p.nw == p.w && p.nh == p.h;
    for (int c = 0; c < p.nc; c++) out[c] = same ? in[c] : s->d_scratch + p.rz_off[c];
    return s->resampler.run(in, p.w, p.h, out, p.nw, p.nh, p.nc, s->stream, err);
}

bool coefs_from_samples(Slot *s, uint8_t *const *planes, const JpegGeom &gout, const SamplePlan &p, std::string &err)
{
    cudaStream_t st = (cudaStream_t)s->stream;
    const int nc = gout.ncomp;
    if (nc == 3 && !launch_ok(launch_rgb_to_ycc(planes[0], planes[1], planes[2], (size_t)gout.width * gout.height, st), "rgb_to_ycc", err)) return false;
    put_quant(s, gout);
    WorkLists wl;
    for (int c = 0; c < nc; c++) {
        CompWork e; memset(&e, 0, sizeof(e));
        e.cout = s->d_out + gout.comp_offset[c]; e.q = dev_quant(s) + gout.tq[c];
        e.bw_out = gout.bw[c]; e.bh_out = gout.bh[c]; e.rbw_out = gout.rbw[c]; e.rbh_out = gout.rbh[c];
        e.W = gout.width; e.H = gout.height; e.fstride = gout.width; e.full = planes[c]; e.dplane = s->d_scratch + p.dpl_off[c];
        e.dn_hx = gout.hmax / gout.hs[c]; e.dn_vx = gout.vmax / gout.vs[c]; e.up_hx = e.up_vx = 1;
        wl.down.push_back(e); wl.max_dn_w = std::max(wl.max_dn_w, e.rbw_out * 8); wl.max_dn_h = std::max(wl.max_dn_h, e.rbh_out * 8);
        wl.fdct.push_back(e); wl.max_fdct = std::max(wl.max_fdct, work_tiles(e.rbw_out, e.rbh_out));
    }
    const size_t tables_end = p.trellis ? put_trellis(s, gout, p.sink_off + sizeof(CompWork) * 3 * nc, wl) : 0;
    const size_t works_end = p.sink_off + flatten_work(wl, reinterpret_cast<CompWork *>(s->h_par + p.sink_off)) * sizeof(CompWork);
    const size_t end = p.trellis ? tables_end : works_end;
    CU(cudaMemcpyAsync(s->d_par, s->h_par, sizeof(QuantDev) * 4, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(s->d_par + p.sink_off, s->h_par + p.sink_off, end - p.sink_off, cudaMemcpyHostToDevice, st));
    return launch_ok(launch_work(wl, reinterpret_cast<const CompWork *>(s->d_par + p.sink_off), st), "kernel launch", err);
}

} // namespace b200
