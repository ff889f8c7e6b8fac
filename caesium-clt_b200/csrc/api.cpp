// api.cpp -- the C-ABI of include/b200_caesium.h: format dispatch, parameter mapping and error mapping that
// libcaesium's lib.rs performs behind caesium::{compress,convert,compress_to_size}_in_memory
// (call sites caesium-clt's src/compressor.rs:287-306).  No CPU codec fallback exists anywhere below.
#include "../../include/b200_caesium.h"
#include "../../include/b200_caesium_png_lossy.h"
#include "../../include/b200_caesium_jpeg_trellis.h"
#include "../../include/b200_caesium_gif.h"
#include "../../include/b200_caesium_png_resize.h"
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <exception>
#include <fstream>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>
#include "jpeg_device.h"
#include "jpeg_host.h"
#include "jpeg_gpuenc.h"
#include "resize_kernels.h"
#include "png_host.h"
#include "png_device.h"
#include "png_quant.h"
#include "vp8_host.h"
#include "webp_device.h"
#include "vp8l_device.h"
#include "vp8_decode.h"
#include "vp8l_alpha.h"
#include "gif_host.h"
#include "gif_device.h"
#include "jpeg_pipe.h"
#include "topology.h"
#include "launch_timer.h"

using namespace b200;

namespace {

b200_status ok_status() { b200_status s; s.code = B200_OK; s.message = nullptr; return s; }
b200_status make_status(int code, const std::string &msg)
{   // CaesiumError Display: "{message} [{code}]"
    b200_status s; s.code = code;
    std::string m = msg + " [" + std::to_string(code) + "]";
    s.message = (char *)malloc(m.size() + 1);
    if (s.message) memcpy(s.message, m.c_str(), m.size() + 1);
    return s;
}

// a header the reader refused: RGB-coded sources are "recognised but not on this path" (code 3), everything else is corrupt input
b200_status header_status(const std::string &err) { return make_status(err.compare(0, 9, "RGB-coded") == 0 ? B200_ERR_UNSUPPORTED : B200_ERR_CORRUPT_INPUT, err); }

// Every leg that decodes a JPEG to samples (lossy compress, resize, conversion, compress-to-size) upsamples each component by
// hmax / hs x vmax / vs.  A factor that does not divide the largest one has no such ratio: libjpeg refuses the file the same
// way (jdsample.c, JERR_FRACT_SAMPLE_NOT_IMPL).  Each such leg asks this right after the header, before it reserves or launches
// anything, so that they all answer alike.  The coefficient-domain transcode (jpeg_optimize) has no upsampling and takes these files.
bool fractional_sampling(const JpegGeom &g)
{
    for (int c = 0; c < g.ncomp; c++)
        if (g.hmax % g.hs[c] || g.vmax % g.vs[c]) return true;
    return false;
}
const char *const kFractional = "fractional sampling ratio unsupported (upsampling needs factors that divide the largest ones)";

int g_forced_device = -1, g_forced_ngpus = 0;
std::atomic<int> g_entropy_mode{-1};     // -1 unset (env B200_ENTROPY); bit 0 = device entropy encoder, bit 1 = device entropy decoder (default 3)
std::atomic<int> g_png_lossy{-1};        // -1 unset (env B200_PNG_LOSSY); 1 = lossy PNG on the device's quantiser, 0 = refused (code 3)
std::atomic<int> g_gif{-1};              // -1 unset (env B200_GIF); 1 = GIF re-encoded on the device, 0 = refused (code 3)
std::atomic<int> g_png_resize{-1};       // -1 unset (env B200_PNG_RESIZE); 1 = PNG -> PNG with width / height on the device, 0 = refused (code 3)

// runtime_init is idempotent while initialised, so after b200_shutdown (which frees every slot's device buffers) the next call
// initialises again: a long-running host can hand the memory of one workload's slots back before starting another
bool ensure_runtime(std::string &err)
{
    if (runtime_device_count() > 0) return true;
    std::string e;
    if (runtime_init(g_forced_ngpus, g_forced_device, e) > 0) return true;
    err = e.empty() ? "no CUDA device available; this build has no CPU fallback" : e;
    return false;
}

// bit 0 = device entropy encoder, bit 1 = device entropy decoder; B200_ENTROPY is read once unless b200_set_entropy_mode chose
int entropy_mode()
{
    if (g_entropy_mode.load() < 0) {
        const char *e = getenv("B200_ENTROPY");
        g_entropy_mode.store(!e ? 3 : !strcmp(e, "host") ? 0 : !strcmp(e, "gpuenc") ? 1 : !strcmp(e, "gpudec") ? 2 : 3);
    }
    return g_entropy_mode.load();
}

// lossy PNG (png.optimize == false) on the device: b200_set_png_lossy, else B200_PNG_LOSSY=gpu, read once; off by default
bool png_lossy()
{
    if (g_png_lossy.load() < 0) {
        const char *e = getenv("B200_PNG_LOSSY");
        g_png_lossy.store(e && !strcmp(e, "gpu") ? 1 : 0);
    }
    return g_png_lossy.load() == 1;
}

// PNG -> PNG with a target size on the device: b200_set_png_resize, else B200_PNG_RESIZE=gpu, read once; off by default
bool png_resize()
{
    if (g_png_resize.load() < 0) {
        const char *e = getenv("B200_PNG_RESIZE");
        g_png_resize.store(e && !strcmp(e, "gpu") ? 1 : 0);
    }
    return g_png_resize.load() == 1;
}

// GIF sources on the device: b200_set_gif, else B200_GIF=gpu, read once; off by default
bool gif_on()
{
    if (g_gif.load() < 0) {
        const char *e = getenv("B200_GIF");
        g_gif.store(e && !strcmp(e, "gpu") ? 1 : 0);
    }
    return g_gif.load() == 1;
}

// One slot of one device (prefer_dev < 0: the next device round-robin), held until the lease goes out of scope.  The runtime
// must already be up (ensure_runtime): where a leg calls that decides which status a machine without a device answers.
class SlotLease {
public:
    explicit SlotLease(int prefer_dev) : s_(slot_acquire(prefer_dev < 0 ? runtime_next_device() : prefer_dev, err_)) {}
    ~SlotLease() { slot_release(s_); }
    SlotLease(const SlotLease &) = delete;
    SlotLease &operator=(const SlotLease &) = delete;
    operator Slot *() const { return s_; }
    Slot *operator->() const { return s_; }
    b200_status failure() const { return make_status(B200_ERR_CUDA, err_); }      // why no slot could be had
private:
    std::string err_;
    Slot *s_;
};

// the body of an entry point: no C++ exception crosses the C ABI
template <class Fn> b200_status guarded(Fn fn)
{
    try { return fn(); }
    catch (const std::exception &e) { return make_status(B200_ERR_OUT_OF_MEMORY, e.what()); }
    catch (...) { return make_status(B200_ERR_INVALID_ARGUMENT, "unexpected failure"); }
}

// a result handed to the caller in malloc'ed memory (released with b200_free); *n counts elements
template <class T> b200_status give(const std::vector<T> &v, T **out, size_t *n)
{
    *out = (T *)malloc(v.size() ? v.size() * sizeof(T) : 1);
    if (!*out) return make_status(B200_ERR_OUT_OF_MEMORY, "out of memory");
    memcpy(*out, v.data(), v.size() * sizeof(T)); *n = v.size();
    return ok_status();
}

// a PNG the decoder refused: interlaced files are "recognised but not on this path", everything else is corrupt input
b200_status png_status(const std::string &err) { return make_status(err.find("interlace") != std::string::npos ? B200_ERR_UNSUPPORTED : B200_ERR_CORRUPT_INPUT, err); }

// planar 8-bit samples with no JPEG behind them ([nc][h][w]: RGB or one grey plane): 1x1 sampling, one quantisation slot
JpegGeom planar_geom(uint32_t w, uint32_t h, int nc)
{
    JpegGeom g; g.width = (int)w; g.height = (int)h; g.ncomp = nc;
    for (int c = 0; c < nc; c++) { g.cid[c] = c + 1; g.hs[c] = g.vs[c] = 1; g.tq[c] = 0; }
    g.finalize();
    return g;
}
JpegGeom with_size(JpegGeom g, uint32_t w, uint32_t h) { g.width = (int)w; g.height = (int)h; g.finalize(); return g; }

// libcaesium resize::resize_image -> compute_dimensions (the source size when neither width nor height is set); source and
// target must fit the format: both sides at most 65535, the target at most `limit` (65535 for PNG, kJpegMaxDimension for JPEG,
// 16383 for WebP) and not empty
b200_status target_size(uint32_t w, uint32_t h, const b200_params *p, uint32_t limit, uint32_t &nw, uint32_t &nh, const char *msg)
{
    nw = w; nh = h;
    if (p->width || p->height) compute_resize_dimensions(w, h, p->width, p->height, nw, nh);
    if (nw == 0 || nh == 0 || nw > limit || nh > limit || w > 65535 || h > 65535) return make_status(B200_ERR_INVALID_ARGUMENT, msg);
    return ok_status();
}

void layout_from_geom(const JpegGeom &g, b200_jpeg_layout *l)
{
    memset(l, 0, sizeof(*l));
    l->width = g.width; l->height = g.height; l->ncomp = g.ncomp; l->progressive = g.progressive;
    for (int c = 0; c < g.ncomp; c++) {
        l->hs[c] = g.hs[c]; l->vs[c] = g.vs[c]; l->bw[c] = g.bw[c]; l->bh[c] = g.bh[c]; l->rbw[c] = g.rbw[c]; l->rbh[c] = g.rbh[c];
        l->comp_offset[c] = g.comp_offset[c];
        memcpy(l->qt[c], g.qt[g.tq[c]], 128);
    }
    l->total_coefs = g.total_coefs;
}

bool geom_from_layout(const b200_jpeg_layout *l, JpegGeom &g, std::string &err)
{
    g = JpegGeom();
    if (!l || l->width <= 0 || l->height <= 0 || (l->ncomp != 1 && l->ncomp != 3)) { err = "invalid JPEG layout"; return false; }
    g.width = l->width; g.height = l->height; g.ncomp = l->ncomp; g.progressive = l->progressive != 0;
    int nslots = 0;
    for (int c = 0; c < l->ncomp; c++) {
        if (l->hs[c] < 1 || l->hs[c] > 4 || l->vs[c] < 1 || l->vs[c] > 4) { err = "invalid sampling factors"; return false; }
        g.cid[c] = c + 1; g.hs[c] = l->hs[c]; g.vs[c] = l->vs[c];
        int slot = -1;
        for (int t = 0; t < nslots; t++) if (!memcmp(g.qt[t], l->qt[c], 128)) slot = t;
        if (c == 1 && slot == 0 && nslots == 1) slot = -1;          // keep luma / chroma in separate slots like jpeg_set_defaults
        if (slot < 0) { slot = nslots++; memcpy(g.qt[slot], l->qt[c], 128); g.qt_present[slot] = true; }
        g.tq[c] = slot;
    }
    g.finalize();
    for (int c = 0; c < l->ncomp; c++) if (l->bw[c] != g.bw[c] || l->bh[c] != g.bh[c] || l->comp_offset[c] != g.comp_offset[c]) { err = "layout block counts do not match its dimensions"; return false; }
    return true;
}

int usable_cores()
{   // cgroup v2 quota if any (the GPU boxes expose 128 logical CPUs but cap the container), else hardware_concurrency
    unsigned hc = std::thread::hardware_concurrency(); if (!hc) hc = 1;
    std::ifstream f("/sys/fs/cgroup/cpu.max");
    std::string a; long long period = 0;
    if (f && (f >> a >> period) && a != "max" && period > 0) {
        long long q = atoll(a.c_str());
        if (q > 0) { unsigned n = (unsigned)((q + period - 1) / period); if (n >= 1 && n < hc) hc = n; }
    }
    return (int)hc;
}

// B200_TRACE=1: wall-clock per stage of the per-image call, summed over all images, printed by b200_shutdown()
std::atomic<long long> g_stage_ns[8];
std::atomic<long long> g_stage_n{0};
const bool g_trace = getenv("B200_TRACE") != nullptr;
struct StageTimer {
    std::chrono::steady_clock::time_point t = std::chrono::steady_clock::now();
    void lap(int i)
    {
        if (!g_trace) return;
        auto n = std::chrono::steady_clock::now();
        const long long ns = std::chrono::duration_cast<std::chrono::nanoseconds>(n - t).count();
        g_stage_ns[i] += ns; t = n;
        if (i == 5) g_stage_n++;
        static const bool verbose = getenv("B200_TRACE") && atoi(getenv("B200_TRACE")) >= 2;
        if (verbose) fprintf(stderr, "[b200 trace] stage %d: %.3f ms\n", i, ns / 1e6);
    }
};
void print_trace()
{
    if (!g_trace || !g_stage_n.load()) return;
    static const char *names[] = {"parse+scan-for-markers", "device entropy decode (incl. syncs)", "host entropy decode", "transform launch", "device entropy encode (incl. syncs)", "assemble file"};
    fprintf(stderr, "[b200 trace] %lld images; mean ms per image and stage:\n", g_stage_n.load());
    for (int i = 0; i < 6; i++) fprintf(stderr, "[b200 trace]   %-38s %8.3f\n", names[i], g_stage_ns[i].load() / 1e6 / (double)g_stage_n.load());
}

// ---- JPEG through the device ---------------------------------------------------------------------------------
// Entropy DECODE on the device for baseline single-scan files (jpeg_gpudec.cu): the scan's bytes go up, the coefficients are
// born in HBM (on_device).  Progressive / multi-scan / restart-interval files, and the rare stream whose parallel decode does not
// settle, are Huffman-decoded into s->h_in on the calling thread instead.
b200_status decode_into_slot(Slot *s, JpegReader &rd, bool &on_device, std::string &err, StageTimer *tm = nullptr)
{
    on_device = false;
    JpegReader::DeviceScan ds;
    if ((entropy_mode() & 2) && rd.device_decodable(ds)) {
        if (tm) tm->lap(0);
        const int r = slot_gpu_decode(s, rd, ds, err);
        if (tm) tm->lap(1);
        if (r == 0) on_device = true;
        else if (r != 1) return make_status(B200_ERR_CUDA, err);
    }
    if (!on_device && !rd.decode(s->h_in, err)) return make_status(B200_ERR_CORRUPT_INPUT, err);
    return ok_status();
}

// Huffman statistics, table construction, bit packing and 0xFF stuffing of the coefficients in s->d_out on the device
// (jpeg_gpuenc.cu); the host only frames the scans.  A scan that outgrows its device buffer falls back to the host ENCODER
// (still the same coefficients from the CUDA transform).
b200_status encode_from_slot(Slot *s, const JpegGeom &gout, const JpegWriteOptions &wo, const JpegMeta *meta, std::vector<uint8_t> &out, std::string &err,
                             StageTimer *tm = nullptr)
{
    if (slot_gpu_encode(s, gout, wo.progressive, err)) {
        if (tm) tm->lap(4);
        const bool ok = jpeg_assemble(gout, wo, meta, s->enc->results.data(), (int)s->enc->results.size(), out, err);
        if (tm) tm->lap(5);
        return ok ? ok_status() : make_status(B200_ERR_INVALID_ARGUMENT, err);
    }
    if (!s->enc->overflow || !slot_download_coefs(s, (size_t)gout.total_coefs * 2, err)) return make_status(B200_ERR_CUDA, err);
    jpeg_fill_dummy_blocks(gout, s->h_out);
    if (!jpeg_write(gout, s->h_out, wo, meta, out, err)) return make_status(B200_ERR_INVALID_ARGUMENT, err);
    return ok_status();
}

b200_status jpeg_compress(const uint8_t *in, size_t in_len, const b200_params *p, int prefer_dev, std::vector<uint8_t> &out)
{
    std::string err;
    JpegReader rd(in, in_len);
    if (!rd.read_header(err)) return header_status(err);
    const JpegGeom &gin = rd.geom();
    JpegWriteOptions wo = write_options(p);
    if (p->jpeg_optimize) {
        // libcaesium jpeg::lossless: coefficient-domain transcode.  Baseline single-scan inputs are entropy-decoded and
        // re-encoded (optimal tables, progressive script) by the device coders; the coefficients never leave HBM.
        // Everything else (progressive input, no device) is transcoded on the calling thread -- there is no arithmetic
        // on this path, only entropy coding.
        wo.copy_jfif = true;
        std::string derr;
        JpegReader::DeviceScan ds;
        if (entropy_mode() == 3 && rd.device_decodable(ds) && ensure_runtime(derr)) {
            SlotLease s(prefer_dev);
            if (s) {
                if (s->ensure((size_t)gin.total_coefs * 2, 0, 0, 1 << 14, derr) && slot_gpu_decode(s, rd, ds, derr) == 0 &&
                    slot_gpu_encode(s, gin, wo.progressive, derr, true) &&
                    jpeg_assemble(gin, wo, &rd.meta(), s->enc->results.data(), (int)s->enc->results.size(), out, derr))
                    return ok_status();
                out.clear();
            }
        }
        std::vector<int16_t> coefs((size_t)gin.total_coefs);
        if (!rd.decode(coefs.data(), err)) return make_status(B200_ERR_CORRUPT_INPUT, err);
        jpeg_fill_dummy_blocks(gin, coefs.data());
        if (!jpeg_write(gin, coefs.data(), wo, &rd.meta(), out, err)) return make_status(B200_ERR_INVALID_ARGUMENT, err);
        return ok_status();
    }
    if (fractional_sampling(gin)) return make_status(B200_ERR_UNSUPPORTED, kFractional);
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    JpegGeom gout;
    if (!jpeg_output_geom(gin, (int)p->jpeg_quality, (int)p->jpeg_chroma_subsampling, gout, err)) return make_status(B200_ERR_INVALID_ARGUMENT, err);
    const bool resize = p->width || p->height;
    if (resize) {
        uint32_t nw, nh;
        const b200_status st = target_size((uint32_t)gin.width, (uint32_t)gin.height, p, kJpegMaxDimension, nw, nh, "invalid target dimensions");
        if (st.code) return st;
        gout = with_size(gout, nw, nh);
    }
    ImagePlan plan;
    if (!resize && !plan_image(gin, gout, plan, err)) return make_status(B200_ERR_UNSUPPORTED, err);
    if (resize) { plan.in_bytes = (size_t)gin.total_coefs * 2; plan.out_bytes = (size_t)gout.total_coefs * 2; }
    SlotLease s(prefer_dev);
    if (!s) return s.failure();
    if (!s->ensure(plan.in_bytes, plan.out_bytes, plan.scratch_bytes(), 1 << 14, err)) return make_status(B200_ERR_OUT_OF_MEMORY, err);
    const bool gpu_entropy = (entropy_mode() & 1) != 0;
    bool on_device;
    StageTimer tm;
    const b200_status st = decode_into_slot(s, rd, on_device, err, &tm);
    if (st.code) return st;
    tm.lap(2);
    SamplePlan sp;
    uint8_t *full[3], *rz[3];
    const bool ok = resize ? plan_samples(s, gin, gout.width, gout.height, &gout, sp, err) && samples_from_coefs(s, gin, sp, !on_device, true, full, err) &&
                                 resize_samples(s, full, sp, rz, err) && coefs_from_samples(s, rz, gout, sp, err)
                           : slot_transform(s, gin, gout, err, false, !on_device);
    if (!ok || (!gpu_entropy && !slot_download_coefs(s, plan.out_bytes, err))) return make_status(B200_ERR_CUDA, err);
    tm.lap(3);
    if (gpu_entropy) return encode_from_slot(s, gout, wo, &rd.meta(), out, err, &tm);
    jpeg_fill_dummy_blocks(gout, s->h_out);
    if (!jpeg_write(gout, s->h_out, wo, &rd.meta(), out, err)) return make_status(B200_ERR_INVALID_ARGUMENT, err);
    return ok_status();
}

// One megabatch: the images idx[] that are baseline single-scan JPEGs of one shape are decoded, transformed and encoded by
// ONE sequence of kernel launches on one slot.  done[k] = 1 for every image this function finished (successfully or with
// a final error in status[]); the caller runs the others through the per-image path.
void jpeg_compress_group(const uint8_t *const *in, const size_t *in_len, const std::vector<int> &idx, const b200_params *p, int dev,
                         uint8_t **out, size_t *out_len, b200_status *status, std::vector<char> &done)
{
    const int M = (int)idx.size();
    StageTimer tm;
    std::vector<std::unique_ptr<JpegReader>> rd((size_t)M);
    std::vector<JpegReader::DeviceScan> ds((size_t)M);
    std::vector<int> members;                       // positions k (into idx) that join the group
    std::string err;
    for (int k = 0; k < M; k++) {
        const int i = idx[k];
        if (b200_sniff_format(in[i], in_len[i]) != B200_FMT_JPEG) continue;
        rd[k].reset(new JpegReader(in[i], in_len[i]));
        if (!rd[k]->read_header(err) || !rd[k]->device_decodable(ds[k], true)) continue;      // the entropy-coded segment is walked on the device
        if (!members.empty() && !same_shape(rd[members[0]]->geom(), rd[k]->geom())) continue;
        members.push_back(k);
    }
    if (members.size() < 2) return;
    const JpegGeom &gin0 = rd[members[0]]->geom();
    const bool lossless = p->jpeg_optimize != 0;          // jpeg::lossless: decode -> encode, no transform, per-image tables kept
    JpegGeom gout;
    if (lossless) gout = gin0;
    else if (!jpeg_output_geom(gin0, (int)p->jpeg_quality, (int)p->jpeg_chroma_subsampling, gout, err)) return;
    SlotLease s(dev);
    if (!s) return;
    const int Kg = (int)members.size();
    GroupLayout L;
    if (!slot_group_layout(s, gin0, gout, Kg, L, err)) return;
    std::vector<GpuDecoder::Item> items((size_t)Kg);
    std::vector<const JpegGeom *> gins((size_t)Kg);
    for (int m = 0; m < Kg; m++) {
        const int k = members[m];
        items[m].rd = rd[k].get(); items[m].ds = &ds[k]; items[m].result = GpuDecoder::FAILED;
        items[m].d_coefs = L.coefs(*s, m, true);
        gins[m] = &rd[k]->geom();
    }
    tm.lap(0);
    JpegWriteOptions wo = write_options(p);
    wo.copy_jfif = lossless;
    if (!slot_run_group(s, items, gins.data(), gout, L, wo.progressive, lossless, err)) return;
    tm.lap(4);
    const int spi = s->enc->plan.scans_per_image;
    for (int m = 0; m < Kg; m++) {
        const int k = members[m], i = idx[k];
        if (items[m].result != GpuDecoder::OK) continue;          // not converged: the per-image path decodes it on the host
        out[i] = nullptr; out_len[i] = 0;
        if (!jpeg_assemble_malloc(lossless ? rd[k]->geom() : gout, wo, &rd[k]->meta(), s->enc->results.data() + (size_t)m * spi, spi, &out[i], &out_len[i], err)) status[i] = make_status(B200_ERR_INVALID_ARGUMENT, err);
        else status[i] = ok_status();
        done[k] = 1;
    }
    tm.lap(5);
}

b200_status png_lossy_compress(PngInfo &info, const PngIdat &idat, const b200_params *p, int prefer_dev, std::vector<uint8_t> &out, uint32_t nw, uint32_t nh);

// a failed PngDevice call: the input's fault (code 4); with a resize, a failed allocation is out of memory (code 7); else a CUDA error
b200_status png_device_status(const PngDevice *png, bool resize, const std::string &err)
{
    if (png->corrupt) return make_status(B200_ERR_CORRUPT_INPUT, err);
    if (resize && (!err.compare(0, 11, "cudaMalloc:") || !err.compare(0, 14, "cudaHostAlloc:"))) return make_status(B200_ERR_OUT_OF_MEMORY, err);
    return make_status(B200_ERR_CUDA, err);
}

// With width / height set (the resize switch on), the PNG leg resizes before coding: PngDevice expands the samples to the image crate's
// decoded type and resamples them with K3 between the un-filter and the back end.  target_size gives nw x nh (0 x 0 = no resize).
b200_status png_target(const PngInfo &info, const b200_params *p, uint32_t &nw, uint32_t &nh)
{
    nw = nh = 0;
    if (!p->width && !p->height) return ok_status();
    return target_size(info.width, info.height, p, 65535, nw, nh, "invalid target dimensions");
}

// ---- PNG (lossless) through the device ---------------------------------------------------------------------------
// libcaesium png::compress: optimize == true -> png::lossless (oxipng, level = png.optimization_level); otherwise the lossy
// palette quantiser (imagequant) when the lossy switch is on.  Resizing (width / height) runs on the device when the resize switch is on.
b200_status png_compress(const uint8_t *in, size_t in_len, const b200_params *p, int prefer_dev, std::vector<uint8_t> &out)
{
    if (!p->png_optimize && !png_lossy()) return make_status(B200_ERR_UNSUPPORTED, "lossy PNG (imagequant) is outside the GPU path (route to caesium::compress_in_memory)");
    if ((p->width || p->height) && !png_resize()) return make_status(B200_ERR_UNSUPPORTED, "PNG resize is outside the GPU path (route to caesium::compress_in_memory)");
    std::string err;
    PngInfo info; PngIdat idat;
    static const bool verbose = getenv("B200_TRACE") && atoi(getenv("B200_TRACE")) >= 2;
    const auto t0 = std::chrono::steady_clock::now();
    if (!png_parse_chunks(in, in_len, p->keep_metadata != 0, info, idat, err)) return png_status(err);
    uint32_t nw, nh;
    const b200_status tst = png_target(info, p, nw, nh);
    if (tst.code) return tst;
    if (!p->png_optimize) return png_lossy_compress(info, idat, p, prefer_dev, out, nw, nh);
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    std::vector<uint8_t> z;
    auto t1 = t0;
    double deflate_ms = 0;
    const uint32_t sw = info.width, sh = info.height;
    std::map<std::string, std::pair<double, int>> ev;      // B200_TRACE=2: device event times of the stages
    {   // the slot goes back before the container is written
        SlotLease s(prefer_dev);
        if (!s) return s.failure();
        PngDevice *png = s->png_dev();
        // the IDAT stream is inflated straight into the slot's pinned staging buffer; from there on everything is device work
        // (un-filter, checksum, reductions, filter trials, LZ77, DEFLATE coding) until the finished zlib stream comes back
        const size_t nin = (info.row_bytes + 1) * (size_t)info.height;
        size_t cap = 0, got = 0; uint32_t stored_adler = 0;
        uint8_t *buf = png->input_buffer(nin, cap, err);
        if (!buf) return make_status(B200_ERR_OUT_OF_MEMORY, err);
        if (!zlib_inflate_to(idat.p, idat.n, buf, cap, nin, &got, &stored_adler, err)) return make_status(B200_ERR_CORRUPT_INPUT, err);
        if (got < nin) return make_status(B200_ERR_CORRUPT_INPUT, "IDAT too short");
        t1 = std::chrono::steady_clock::now();
        LaunchTimer lt;
        if (verbose) { lt.begin((cudaStream_t)s->stream); tl_launch_timer = &lt; }
        const bool ok = png->compress_filtered(info, got, stored_adler, std::min((int)p->png_optimization_level, 6), s->stream, z, nullptr, err, nw, nh);
        tl_launch_timer = nullptr;
        if (verbose) { cudaStreamSynchronize((cudaStream_t)s->stream); lt.collect(ev); }
        if (!ok) return png_device_status(png, nw != 0, err);
        deflate_ms = png->last_deflate_ms;
    }
    const auto t3 = std::chrono::steady_clock::now();
    png_write(info, z, out);
    if (verbose) {
        auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
        fprintf(stderr, "[b200 trace] png %ux%u: parse + inflate %.1f ms, device (un-filter, filter trials, LZ77, DEFLATE coding; host Huffman %.1f) %.1f ms, container %.1f ms\n",
                info.width, info.height, ms(t0, t1), deflate_ms, ms(t1, t3), ms(t3, std::chrono::steady_clock::now()));
        auto at = [&](const char *k) { auto it = ev.find(k); return it == ev.end() ? 0.0 : it->second.first; };
        const double up = at("h2d") + at("png_unfilter"), rz = at("png_resize");
        fprintf(stderr, "[b200 trace] png stages %ux%u -> %ux%u: parse + inflate %.3f ms, h2d + un-filter %.3f ms, expand + K3 + pack %.3f ms, back end %.3f ms\n",
                sw, sh, info.width, info.height, ms(t0, t1), up, rz, ms(t1, t3) - up - rz);
    }
    return ok_status();
}

// chunks whose meaning depends on the colour type (sBIT, bKGD, hIST) do not survive quantisation, nor does a grey source's ICC
// profile (iCCP): a grey profile is invalid on the indexed colour output
void drop_colour_chunks(std::vector<uint8_t> &kept, bool grey_source)
{
    std::vector<uint8_t> out;
    for (size_t i = 0; i + 12 <= kept.size();) {
        const size_t L = (size_t)kept[i] << 24 | (size_t)kept[i + 1] << 16 | (size_t)kept[i + 2] << 8 | kept[i + 3];
        if (L > kept.size() - i - 12) break;
        const char *t = reinterpret_cast<const char *>(kept.data() + i + 4);
        if (memcmp(t, "sBIT", 4) && memcmp(t, "bKGD", 4) && memcmp(t, "hIST", 4) && (!grey_source || memcmp(t, "iCCP", 4))) out.insert(out.end(), kept.begin() + i, kept.begin() + i + 12 + L);
        i += 12 + L;
    }
    kept.swap(out);
}

// One lossy PNG try: the quantiser already holds the image (histogram built); palette at `quality`, dithering, indexed coding, file.
// B200_TRACE=2 prints the per-kernel event times.
b200_status png_lossy_code(Slot *s, PngInfo info, int quality, int level, std::vector<uint8_t> &out)
{
    static const bool verbose = getenv("B200_TRACE") && atoi(getenv("B200_TRACE")) >= 2;
    std::string err;
    std::vector<uint8_t> z;
    LaunchTimer lt;
    if (verbose) { lt.begin((cudaStream_t)s->stream); tl_launch_timer = &lt; }
    const auto t0 = std::chrono::steady_clock::now();
    const bool ok = s->png_dev()->code_quantized(info, quality < 0 ? 0 : quality > 100 ? 100 : quality, std::min(level, 6), s->stream, z, err);
    tl_launch_timer = nullptr;
    if (!ok) return make_status(B200_ERR_CUDA, err);
    if (verbose) {
        std::map<std::string, std::pair<double, int>> acc;
        lt.collect(acc);
        std::string kt;
        for (auto &kv : acc) { char b[96]; snprintf(b, sizeof b, " %s=%.4f", kv.first.c_str(), kv.second.first); kt += b; }
        fprintf(stderr, "[b200 trace] png-lossy %ux%u q%d: %d colours, device %.3f ms (median cut %.3f); kernels ms:%s\n", info.width, info.height, quality,
                (int)(info.plte.size() / 3), std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count(), s->png_dev()->quantiser()->last_cut_ms, kt.c_str());
    }
    png_write(info, z, out);
    return ok_status();
}

// a parsed PNG's IDAT inflated into the slot's staging buffer, un-filtered, (nw, nh > 0: resized,) expanded and histogrammed by the quantiser
b200_status png_lossy_load(Slot *s, PngInfo &info, const PngIdat &idat, uint32_t nw = 0, uint32_t nh = 0)
{
    std::string err;
    const bool grey = info.color_type == 0 || info.color_type == 4;
    drop_colour_chunks(info.kept_before_idat, grey); drop_colour_chunks(info.kept_after_idat, grey);
    PngDevice *png = s->png_dev();
    const size_t nin = (info.row_bytes + 1) * (size_t)info.height;
    size_t cap = 0, got = 0; uint32_t stored_adler = 0;
    uint8_t *buf = png->input_buffer(nin, cap, err);
    if (!buf) return make_status(B200_ERR_OUT_OF_MEMORY, err);
    if (!zlib_inflate_to(idat.p, idat.n, buf, cap, nin, &got, &stored_adler, err)) return make_status(B200_ERR_CORRUPT_INPUT, err);
    if (got < nin) return make_status(B200_ERR_CORRUPT_INPUT, "IDAT too short");
    if (!png->load_filtered_lossy(info, got, stored_adler, s->stream, err, nw, nh)) return png_device_status(png, nw != 0, err);
    return ok_status();
}

// lossy PNG (png.optimize == false, the switch on): palette quantisation with Floyd-Steinberg dithering on the device, then the
// lossless leg's filter trials, LZ77 and DEFLATE over the indexed image
b200_status png_lossy_compress(PngInfo &info, const PngIdat &idat, const b200_params *p, int prefer_dev, std::vector<uint8_t> &out, uint32_t nw, uint32_t nh)
{
    std::string err;
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    SlotLease s(prefer_dev);
    if (!s) return s.failure();
    const b200_status st = png_lossy_load(s, info, idat, nw, nh);
    if (st.code) return st;
    return png_lossy_code(s, info, (int)p->png_quality, (int)p->png_optimization_level, out);
}

// 8-bit planar samples ([nc][h][w], nc = 1 or 3) and an optional alpha plane -> lossless PNG (K6 filter selection, K7 LZ77) on the
// slot's PngDevice.  palette: try png_reduce_palette first.
b200_status png_from_planes(Slot *s, const uint8_t *planes, int nc, const uint8_t *alpha, uint32_t w, uint32_t h, bool palette, const b200_params *p,
                            std::vector<uint8_t> &out, std::string &err)
{
    if (!p->png_optimize) {             // lossy PNG (the callers refuse it while the switch is off): the planes go up as they are
        PngQuant *q = s->png_dev()->quantiser();
        if (!q->load_planes(planes, nc, alpha, (int)w, (int)h, s->stream, err) || !q->prepare(s->stream, err)) return make_status(B200_ERR_CUDA, err);
        PngInfo info; info.width = w; info.height = h;
        return png_lossy_code(s, info, (int)p->png_quality, (int)p->png_optimization_level, out);
    }
    const size_t n = (size_t)w * h;
    const int ch = nc + (alpha ? 1 : 0);
    std::vector<uint8_t> raw;
    if (ch == 1) raw.assign(planes, planes + n);
    else {
        raw.resize((size_t)ch * n);
        for (size_t i = 0; i < n; i++) {
            raw[ch * i] = planes[i]; raw[ch * i + 1] = planes[n + i]; raw[ch * i + 2] = planes[2 * n + i];
            if (alpha) raw[ch * i + 3] = alpha[i];
        }
    }
    PngInfo info; info.width = w; info.height = h; info.bit_depth = 8; info.color_type = ch == 1 ? 0 : ch == 3 ? 2 : 6; info.channels = ch;
    info.bits_per_pixel = 8 * ch; info.bpp = ch; info.row_bytes = (size_t)w * ch;
    if (palette) png_reduce_palette(info, raw);
    std::vector<uint8_t> z;
    if (!s->png_dev()->compress(info, raw, std::min((int)p->png_optimization_level, 6), s->stream, z, nullptr, err)) return make_status(B200_ERR_CUDA, err);
    png_write(info, z, out);
    return ok_status();
}

// Lanczos3 (K3) of nc host planes [nc][h][w] to nc device planes of nw x nh on the slot
bool resize_host_planes(Slot *s, const uint8_t *src, uint32_t w, uint32_t h, uint32_t nw, uint32_t nh, int nc, uint8_t **planes, std::string &err)
{
    SamplePlan sp;
    uint8_t *full[3];
    return plan_samples(s, planar_geom(w, h, nc), (int)nw, (int)nh, nullptr, sp, err) && samples_from_host(s, src, sp, full, err) && resize_samples(s, full, sp, planes, err);
}

// the same, fetched back into dst [nc][nh][nw]
bool resize_to_host(Slot *s, const uint8_t *src, uint32_t w, uint32_t h, uint32_t nw, uint32_t nh, int nc, std::vector<uint8_t> &dst, std::string &err)
{
    uint8_t *rz[3];
    dst.resize((size_t)nc * nw * nh);
    return resize_host_planes(s, src, w, h, nw, nh, nc, rz, err) && slot_fetch_planes(s, rz, nc, (size_t)nw * nh, dst.data(), err);
}

// ---- conversion to WebP (lossy VP8) ----------------------------------------------------------------------------------
// libcaesium convert: decode -> (resize) -> webp::compress at parameters.webp.quality.  JPEG sources are decoded on the
// device (entropy decode, IDCT, upsample, YCbCr -> RGB, Lanczos3 when width/height are set) and never leave HBM before K8.
b200_status jpeg_to_webp(const uint8_t *in, size_t in_len, const b200_params *p, int prefer_dev, std::vector<uint8_t> &out)
{
    std::string err;
    JpegReader rd(in, in_len);
    if (!rd.read_header(err)) return header_status(err);
    const JpegGeom &gin = rd.geom();
    if (fractional_sampling(gin)) return make_status(B200_ERR_UNSUPPORTED, kFractional);
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    uint32_t nw, nh;
    b200_status st = target_size((uint32_t)gin.width, (uint32_t)gin.height, p, 16383, nw, nh, "invalid target dimensions for WebP");
    if (st.code) return st;
    SlotLease s(prefer_dev);
    if (!s) return s.failure();
    static const bool verbose = getenv("B200_TRACE") && atoi(getenv("B200_TRACE")) >= 2;
    const auto t0 = std::chrono::steady_clock::now();
    if (!s->ensure((size_t)gin.total_coefs * 2, 0, 0, 1 << 14, err)) return make_status(B200_ERR_OUT_OF_MEMORY, err);
    bool on_device;
    if ((st = decode_into_slot(s, rd, on_device, err)).code) return st;
    const auto t1 = std::chrono::steady_clock::now();
    SamplePlan sp;
    uint8_t *full[3], *rgb[3];
    if (!(plan_samples(s, gin, (int)nw, (int)nh, nullptr, sp, err) && samples_from_coefs(s, gin, sp, !on_device, true, full, err) && resize_samples(s, full, sp, rgb, err)))
        return make_status(B200_ERR_CUDA, err);
    const auto t2 = std::chrono::steady_clock::now();
    WebpDevice *webp = s->webp_dev();
    const int g = gin.ncomp == 3;          // a grey source is its one plane three times
    if (!webp->encode_planes(rgb[0], rgb[g], rgb[2 * g], (int)nw, (int)nh, (int)p->webp_quality, s->stream, out, err)) return make_status(B200_ERR_CUDA, err);
    if (verbose) {
        auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
        fprintf(stderr, "[b200 trace] jpeg %dx%d -> webp %ux%u: segment walk + entropy decode (device %d) %.1f ms, transform + resize launch %.1f ms, VP8 (wait for the device %.1f ms, boolean coder %.1f ms) %.1f ms\n",
                gin.width, gin.height, nw, nh, (int)on_device, ms(t0, t1), ms(t1, t2), webp->last_wait_ms, webp->last_code_ms, ms(t2, std::chrono::steady_clock::now()));
    }
    return ok_status();
}

// JPEG -> PNG (lossless PNG only: png.optimize): device decode (+ K3 resize) to RGB, samples back to the host as PNG rows, then
// the lossless PNG leg (K6 filter selection, K7 LZ77).  A greyscale JPEG becomes a greyscale PNG.
b200_status jpeg_to_png(const uint8_t *in, size_t in_len, const b200_params *p, int prefer_dev, std::vector<uint8_t> &out)
{
    if (!p->png_optimize && !png_lossy()) return make_status(B200_ERR_UNSUPPORTED, "lossy PNG (imagequant) is outside the GPU path (route to caesium::convert_in_memory)");
    std::string err;
    JpegReader rd(in, in_len);
    if (!rd.read_header(err)) return header_status(err);
    const JpegGeom &gin = rd.geom();
    if (fractional_sampling(gin)) return make_status(B200_ERR_UNSUPPORTED, kFractional);
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    uint32_t nw, nh;
    b200_status st = target_size((uint32_t)gin.width, (uint32_t)gin.height, p, 65535, nw, nh, "invalid target dimensions");
    if (st.code) return st;
    SlotLease s(prefer_dev);
    if (!s) return s.failure();
    if (!s->ensure((size_t)gin.total_coefs * 2, 0, 0, 1 << 14, err)) return make_status(B200_ERR_OUT_OF_MEMORY, err);
    bool on_device;
    if ((st = decode_into_slot(s, rd, on_device, err)).code) return st;
    const int nc = gin.ncomp == 1 ? 1 : 3;
    SamplePlan sp;
    uint8_t *full[3], *rgb[3];
    std::vector<uint8_t> planes((size_t)nc * nw * nh);
    if (!(plan_samples(s, gin, (int)nw, (int)nh, nullptr, sp, err) && samples_from_coefs(s, gin, sp, !on_device, true, full, err) && resize_samples(s, full, sp, rgb, err) &&
          slot_fetch_planes(s, rgb, nc, (size_t)nw * nh, planes.data(), err)))
        return make_status(B200_ERR_CUDA, err);
    return png_from_planes(s, planes.data(), nc, nullptr, nw, nh, false, p, out, err);
}

// Decoded PNG samples -> 8-bit planar samples on the host: palette looked up, sub-byte greys scaled, 16-bit -> high byte,
// alpha dropped (like the image crate's to_rgb8 / to_luma8).  allow_grey: grey colour types stay one plane (JPEG target).
void png_expand_planar(const PngInfo &info, const std::vector<uint8_t> &raw, bool allow_grey, std::vector<uint8_t> &planes, int &nc)
{
    const size_t w = info.width, h = info.height, n = w * h;
    const int bd = info.bit_depth, ct = info.color_type;
    nc = (allow_grey && (ct == 0 || ct == 4)) ? 1 : 3;
    planes.resize((size_t)nc * n);
    for (size_t y = 0; y < h; y++) {
        const uint8_t *row = raw.data() + y * info.row_bytes;
        for (size_t x = 0; x < w; x++) {
            uint8_t r, g, b;
            if (ct == 2 || ct == 6) { const size_t o = x * info.channels * (bd / 8); r = row[o]; g = row[o + bd / 8]; b = row[o + 2 * (bd / 8)]; }
            else {
                unsigned v;
                if (bd >= 8) v = row[x * info.channels * (bd / 8)];
                else v = (row[(x * bd) >> 3] >> (8 - bd - ((x * bd) & 7))) & ((1u << bd) - 1);
                if (ct == 3) { if (3 * v + 2 < info.plte.size()) { r = info.plte[3 * v]; g = info.plte[3 * v + 1]; b = info.plte[3 * v + 2]; } else r = g = b = 0; }
                else { if (bd < 8) v = v * 255 / ((1u << bd) - 1); r = g = b = (uint8_t)v; }
            }
            planes[y * w + x] = r;
            if (nc == 3) { planes[n + y * w + x] = g; planes[2 * n + y * w + x] = b; }
        }
    }
}

// Planar 8-bit samples on the host ([nc][H][W]: RGB or one grey plane) -> JPEG: they take the resize path's back end (K3 Lanczos3 when
// width/height are set, RGB -> YCbCr, K4 box downsample, K5 FDCT + quantise) and the device Huffman encoder.
b200_status planes_to_jpeg(const std::vector<uint8_t> &planes, uint32_t w, uint32_t h, int nc, const b200_params *p, int prefer_dev, std::vector<uint8_t> &out)
{
    std::string err;
    uint32_t nw, nh;                                // the source's size unless width / height are set
    const b200_status st = target_size(w, h, p, kJpegMaxDimension, nw, nh, "invalid target dimensions");
    if (st.code) return st;
    const JpegGeom gin = planar_geom(w, h, nc);
    JpegGeom gout;
    if (!jpeg_output_geom(gin, (int)p->jpeg_quality, (int)p->jpeg_chroma_subsampling, gout, err)) return make_status(B200_ERR_INVALID_ARGUMENT, err);
    if (p->width || p->height) gout = with_size(gout, nw, nh);
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    SlotLease s(prefer_dev);
    if (!s) return s.failure();
    SamplePlan sp;
    uint8_t *full[3], *rz[3];
    if (!(plan_samples(s, gin, gout.width, gout.height, &gout, sp, err) && samples_from_host(s, planes.data(), sp, full, err) && resize_samples(s, full, sp, rz, err) &&
          coefs_from_samples(s, rz, gout, sp, err))) return make_status(B200_ERR_CUDA, err);
    return encode_from_slot(s, gout, write_options(p), nullptr, out, err);      // no source metadata: only `progressive` matters
}

b200_status png_to_jpeg(const uint8_t *in, size_t in_len, const b200_params *p, int prefer_dev, std::vector<uint8_t> &out)
{
    std::string err;
    PngInfo info; std::vector<uint8_t> raw;
    if (!png_decode(in, in_len, false, info, raw, err)) return png_status(err);
    std::vector<uint8_t> planes; int nc = 3;
    png_expand_planar(info, raw, true, planes, nc);
    return planes_to_jpeg(planes, info.width, info.height, nc, p, prefer_dev, out);
}

// Planar RGB on the host -> lossy WebP (K3 resize when width / height are set, then K8)
// alpha (optional): one 8-bit plane of the source's size.  It is resized like the colour planes, its LZ77 tokens come from K7 on the
// device, and the file becomes VP8X + ALPH (VP8L-coded, lossless -- libwebp's default alpha_quality 100) + VP8.
b200_status rgb_to_webp(const std::vector<uint8_t> &rgb, uint32_t w, uint32_t h, const b200_params *p, int prefer_dev, std::vector<uint8_t> &out,
                        const std::vector<uint8_t> *alpha = nullptr)
{
    std::string err;
    uint32_t nw, nh;
    const b200_status st = target_size(w, h, p, 16383, nw, nh, "invalid dimensions for WebP");
    if (st.code) return st;
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    SlotLease s(prefer_dev);
    if (!s) return s.failure();
    WebpDevice *webp = s->webp_dev();
    const bool resize = nw != w || nh != h;
    if (!resize) {
        if (!webp->encode_host_rgb(rgb.data(), (int)nw, (int)nh, (int)p->webp_quality, s->stream, out, err)) return make_status(B200_ERR_CUDA, err);
    } else {   // through the resize leg (K3 Lanczos3) first
        uint8_t *planes[3];
        if (!resize_host_planes(s, rgb.data(), w, h, nw, nh, 3, planes, err) || !webp->encode_planes(planes[0], planes[1], planes[2], (int)nw, (int)nh, (int)p->webp_quality, s->stream, out, err)) return make_status(B200_ERR_CUDA, err);
    }
    if (!alpha) return ok_status();
    const size_t n = (size_t)nw * nh;
    std::vector<uint8_t> resized;
    if (resize && !resize_to_host(s, alpha->data(), w, h, nw, nh, 1, resized, err)) return make_status(B200_ERR_CUDA, err);
    const uint8_t *ap = resize ? resized.data() : alpha->data();
    if (std::all_of(ap, ap + n, [](uint8_t v) { return v == 0xFF; })) return ok_status();
    std::vector<uint32_t> tokens; std::vector<uint8_t> alph, wrapped, residual;
    const int filter = webp_alpha_choose_filter(ap, (int)nw, (int)nh, residual);
    if (!s->png_dev()->plane_tokens(filter ? residual.data() : ap, n, (int)nw, s->stream, tokens, err)) return make_status(B200_ERR_CUDA, err);
    if (!(vp8l_alpha_from_tokens(tokens.data(), tokens.size(), (int)nw, (int)nh, alph, filter) && webp_wrap_alpha(out, alph, (int)nw, (int)nh, wrapped)))
        return make_status(B200_ERR_CUDA, "alpha plane could not be coded");
    out.swap(wrapped);
    return ok_status();
}

// The transparency of decoded PNG samples as one 8-bit plane (alpha channel: high byte of a 16-bit sample; tRNS: the palette's
// per-entry alpha or the colour key).  false: every pixel is opaque.
bool png_extract_alpha(const PngInfo &info, const std::vector<uint8_t> &raw, std::vector<uint8_t> &alpha)
{
    const size_t w = info.width, h = info.height;
    const int bd = info.bit_depth, ct = info.color_type;
    const bool channel = ct == 4 || ct == 6;
    if (!channel && info.trns.empty()) return false;
    alpha.assign(w * h, 0xFF);
    bool any = false;
    const size_t bps = bd >= 8 ? (size_t)bd / 8 : 1;
    for (size_t y = 0; y < h; y++) {
        const uint8_t *row = raw.data() + y * info.row_bytes;
        uint8_t *a = alpha.data() + y * w;
        for (size_t x = 0; x < w; x++) {
            uint8_t v = 0xFF;
            if (channel) v = row[(x * info.channels + info.channels - 1) * bps];
            else if (ct == 3) { const unsigned idx = (row[(x * bd) >> 3] >> (8 - bd - ((x * bd) & 7))) & ((1u << bd) - 1); if (idx < info.trns.size()) v = info.trns[idx]; }
            else if (ct == 0 && info.trns.size() >= 2) {
                const unsigned key = ((unsigned)info.trns[0] << 8) | info.trns[1];
                const unsigned sv = bd == 16 ? (((unsigned)row[2 * x] << 8) | row[2 * x + 1]) : bd == 8 ? row[x] : (row[(x * bd) >> 3] >> (8 - bd - ((x * bd) & 7))) & ((1u << bd) - 1);
                if (sv == key) v = 0;
            } else if (ct == 2 && info.trns.size() >= 6) {
                bool eq = true;
                for (int c = 0; c < 3 && eq; c++) {
                    const unsigned key = ((unsigned)info.trns[2 * c] << 8) | info.trns[2 * c + 1];
                    const unsigned sv = bd == 16 ? (((unsigned)row[(3 * x + c) * 2] << 8) | row[(3 * x + c) * 2 + 1]) : row[3 * x + c];
                    eq = sv == key;
                }
                if (eq) v = 0;
            }
            a[x] = v; any |= v != 0xFF;
        }
    }
    return any;
}

// WebP input (libcaesium webp::compress: decode, optional resize, re-encode at webp.quality): the VP8 bitstream is decoded on the
// calling thread (format plumbing, bit-exact with libwebp's decoder -- vp8_decode.cpp), the RGB goes through K3 / K8 like any other source.
b200_status webp_decode_status(const uint8_t *in, size_t in_len, WebpInfo &info, std::vector<uint8_t> &rgb, std::vector<uint8_t> *alpha = nullptr)
{
    std::string err;
    const int rc = webp_decode_rgb(in, in_len, info, rgb, err, alpha);
    if (rc == 1) return make_status(B200_ERR_UNSUPPORTED, err);
    if (rc) return make_status(B200_ERR_CORRUPT_INPUT, err);
    return ok_status();
}
// webp.lossless: decode as above, K3 on the RGB and alpha planes when width / height are set, then the lossless encoder (VP8L:
// subtract-green, per-tile predictors, colour cache, LZ77 at neighbourhood distances -- vp8l_kernels.cu).  Exact: RGB under fully
// transparent pixels is kept.  Like the lossy leg, no metadata is kept.
b200_status webp_lossless_compress(const uint8_t *in, size_t in_len, const b200_params *p, int prefer_dev, std::vector<uint8_t> &out)
{
    std::string err;
    static const bool verbose = getenv("B200_TRACE") && atoi(getenv("B200_TRACE")) >= 2;
    const auto t0 = std::chrono::steady_clock::now();
    WebpInfo info; std::vector<uint8_t> rgb, alpha;
    b200_status st = webp_decode_status(in, in_len, info, rgb, &alpha);
    if (st.code) return st;
    const uint32_t w = (uint32_t)info.width, h = (uint32_t)info.height;
    uint32_t nw, nh;
    if ((st = target_size(w, h, p, 16383, nw, nh, "invalid dimensions for WebP")).code) return st;
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    SlotLease s(prefer_dev);
    if (!s) return s.failure();
    const auto t1 = std::chrono::steady_clock::now();
    const uint8_t *src = rgb.data(), *ap = alpha.empty() ? nullptr : alpha.data();
    std::vector<uint8_t> planes, ra;
    if (nw != w || nh != h) {
        if (!resize_to_host(s, src, w, h, nw, nh, 3, planes, err) || (ap && !resize_to_host(s, ap, w, h, nw, nh, 1, ra, err))) return make_status(B200_ERR_CUDA, err);
        src = planes.data();
        if (ap) ap = ra.data();
    }
    const auto t2 = std::chrono::steady_clock::now();
    Vp8lDevice *v = s->vp8l_dev();
    LaunchTimer lt;
    if (verbose) { lt.begin((cudaStream_t)s->stream); tl_launch_timer = &lt; }
    const bool ok = v->encode(src, ap, (int)nw, (int)nh, s->stream, out, err);
    tl_launch_timer = nullptr;
    if (!ok) return make_status(B200_ERR_CUDA, err);
    if (verbose) {
        auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
        std::map<std::string, std::pair<double, int>> acc;
        lt.collect(acc);
        std::string kt;
        for (auto &kv : acc) { char b[96]; snprintf(b, sizeof b, " %s=%.4f", kv.first.c_str(), kv.second.first); kt += b; }
        fprintf(stderr, "[b200 trace] webp-lossless %ux%u -> %ux%u: host decode %.3f ms, resize %.3f ms, device encode %.3f ms (analysis wait %.3f, cache bits %d, codes + emission %.3f); kernels ms:%s\n",
                w, h, nw, nh, ms(t0, t1), ms(t1, t2), ms(t2, std::chrono::steady_clock::now()), v->last_analyse_ms, v->last_cache_bits, v->last_code_ms, kt.c_str());
    }
    return ok_status();
}

b200_status webp_compress(const uint8_t *in, size_t in_len, const b200_params *p, int prefer_dev, std::vector<uint8_t> &out)
{
    if (p->webp_lossless) return webp_lossless_compress(in, in_len, p, prefer_dev, out);
    WebpInfo info; std::vector<uint8_t> rgb, alpha;
    b200_status st = webp_decode_status(in, in_len, info, rgb, &alpha);
    if (st.code) return st;
    return rgb_to_webp(rgb, (uint32_t)info.width, (uint32_t)info.height, p, prefer_dev, out, alpha.empty() ? nullptr : &alpha);
}

// PNG source: samples are expanded to 8-bit RGB on the host (palette, grey, 16-bit -> high byte) and go through the same K8; an
// opaque alpha channel is discarded, real transparency becomes the file's alpha plane.
b200_status png_to_webp(const uint8_t *in, size_t in_len, const b200_params *p, int prefer_dev, std::vector<uint8_t> &out)
{
    std::string err;
    PngInfo info; std::vector<uint8_t> raw;
    if (!png_decode(in, in_len, false, info, raw, err)) return png_status(err);
    uint32_t nw, nh;
    const b200_status st = target_size(info.width, info.height, p, 16383, nw, nh, "invalid dimensions for WebP");
    if (st.code) return st;
    // transparency (alpha channel, tRNS) travels as the file's alpha plane: VP8X + ALPH next to the lossy frame
    std::vector<uint8_t> alpha;
    const bool has_alpha = png_extract_alpha(info, raw, alpha);
    std::vector<uint8_t> rgb; int nc = 3;
    png_expand_planar(info, raw, false, rgb, nc);
    return rgb_to_webp(rgb, info.width, info.height, p, prefer_dev, out, has_alpha ? &alpha : nullptr);
}

// Planar RGB on the host -> lossless PNG (K3 resize when asked, then the PNG leg's raw-sample entry point)
b200_status rgb_to_png(const std::vector<uint8_t> &rgb, uint32_t w, uint32_t h, const b200_params *p, int prefer_dev, std::vector<uint8_t> &out,
                       const std::vector<uint8_t> *alpha = nullptr)
{
    std::string err;
    uint32_t nw, nh;
    const b200_status st = target_size(w, h, p, 65535, nw, nh, "invalid target dimensions");
    if (st.code) return st;
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    SlotLease s(prefer_dev);
    if (!s) return s.failure();
    const uint8_t *src = rgb.data(), *ap = alpha ? alpha->data() : nullptr;
    std::vector<uint8_t> planes, ra;
    if (nw != w || nh != h) {   // transparency stays: the alpha plane takes the same Lanczos3 as the colour planes
        if (!resize_to_host(s, src, w, h, nw, nh, 3, planes, err) || (ap && !resize_to_host(s, ap, w, h, nw, nh, 1, ra, err))) return make_status(B200_ERR_CUDA, err);
        src = planes.data();
        if (ap) ap = ra.data();
    }
    return png_from_planes(s, src, 3, ap, nw, nh, true, p, out, err);
}

// libcaesium convert_in_memory for a source of format src: the conversions this path takes, the refusals in the reference's order
b200_status convert_dispatch(const uint8_t *in, size_t in_len, uint32_t src, uint32_t fmt, const b200_params *p, std::vector<uint8_t> &out)
{
    if (src == B200_FMT_UNKNOWN) return make_status(B200_ERR_UNKNOWN_FORMAT, "Unknown file type");
    if (src == fmt) return make_status(B200_ERR_SAME_FORMAT, "Cannot convert to the same format");
    if (fmt == B200_FMT_PNG && src == B200_FMT_JPEG) return jpeg_to_png(in, in_len, p, -1, out);
    if (src == B200_FMT_WEBP && (fmt == B200_FMT_JPEG || fmt == B200_FMT_PNG)) {
        // WebP source: decoded on the calling thread (vp8_decode.cpp), then the same back ends as a PNG source
        if (fmt == B200_FMT_JPEG && p->jpeg_optimize) return make_status(B200_ERR_UNSUPPORTED, "lossless conversion to JPEG is outside the GPU path (route to caesium::convert_in_memory)");
        if (fmt == B200_FMT_PNG && !p->png_optimize && !png_lossy()) return make_status(B200_ERR_UNSUPPORTED, "lossy PNG (imagequant) is outside the GPU path (route to caesium::convert_in_memory)");
        WebpInfo wi; std::vector<uint8_t> rgb, alpha;
        const b200_status s = webp_decode_status(in, in_len, wi, rgb, &alpha);
        if (s.code) return s;
        // a JPEG has no alpha (the image crate's to_rgb8 drops it); a PNG keeps it as an RGBA image
        return fmt == B200_FMT_JPEG ? planes_to_jpeg(rgb, (uint32_t)wi.width, (uint32_t)wi.height, 3, p, -1, out)
                                    : rgb_to_png(rgb, (uint32_t)wi.width, (uint32_t)wi.height, p, -1, out, alpha.empty() ? nullptr : &alpha);
    }
    const bool to_webp = fmt == B200_FMT_WEBP, png_to_jpg = fmt == B200_FMT_JPEG && src == B200_FMT_PNG;
    if (!to_webp && !png_to_jpg) return make_status(B200_ERR_UNSUPPORTED, "this conversion is outside the GPU path (route to caesium::convert_in_memory)");
    if (to_webp && p->webp_lossless) return make_status(B200_ERR_UNSUPPORTED, "lossless WebP (VP8L) is outside the GPU path (route to caesium::convert_in_memory)");
    if (png_to_jpg && p->jpeg_optimize) return make_status(B200_ERR_UNSUPPORTED, "lossless conversion to JPEG is outside the GPU path (route to caesium::convert_in_memory)");
    if (png_to_jpg) return png_to_jpeg(in, in_len, p, -1, out);
    if (src == B200_FMT_JPEG) return jpeg_to_webp(in, in_len, p, -1, out);
    if (src == B200_FMT_PNG) return png_to_webp(in, in_len, p, -1, out);
    return make_status(B200_ERR_UNSUPPORTED, "conversion from this format is outside the GPU path (route to caesium::convert_in_memory)");
}

// GIF (the switch on): decoded frame by frame on the calling thread, every composited canvas re-encoded on the device (palette
// quantiser at gif_quality, segmented LZW); the container is written here.  B200_TRACE=2 prints host decode against device time.
b200_status gif_compress(const uint8_t *in, size_t in_len, const b200_params *p, int prefer_dev, std::vector<uint8_t> &out)
{
    if (!gif_on()) return make_status(B200_ERR_UNSUPPORTED, "GIF is outside the GPU path (route to caesium::compress_in_memory)");
    if (p->width || p->height) return make_status(B200_ERR_UNSUPPORTED, "GIF resize is outside the GPU path (route to caesium::compress_in_memory)");
    static const bool verbose = getenv("B200_TRACE") && atoi(getenv("B200_TRACE")) >= 2;
    std::string err;
    GifReader rd;
    if (!rd.open(in, in_len, err)) return make_status(rd.unsupported ? B200_ERR_UNSUPPORTED : B200_ERR_CORRUPT_INPUT, err);
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    SlotLease s(prefer_dev);
    if (!s) return s.failure();
    const auto t0 = std::chrono::steady_clock::now();
    bool corrupt = false;
    const int q = (int)std::min<uint32_t>(p->gif_quality, 100);
    if (!s->gif_dev()->encode(rd, *s->png_dev()->quantiser(), q, s->stream, out, corrupt, err)) return make_status(corrupt ? B200_ERR_CORRUPT_INPUT : B200_ERR_CUDA, err);
    if (verbose) {
        const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        fprintf(stderr, "[b200 trace] gif %dx%d, %d frames q%d: host decode %.1f ms, device and container %.1f ms\n", rd.width, rd.height, rd.frames, q,
                s->gif_dev()->decode_ms, ms - s->gif_dev()->decode_ms);
    }
    return ok_status();
}

b200_status compress_dispatch(const uint8_t *in, size_t in_len, const b200_params *p, int prefer_dev, std::vector<uint8_t> &out)
{
    switch (b200_sniff_format(in, in_len)) {
        case B200_FMT_JPEG: return jpeg_compress(in, in_len, p, prefer_dev, out);
        case B200_FMT_PNG: return png_compress(in, in_len, p, prefer_dev, out);
        case B200_FMT_WEBP: return webp_compress(in, in_len, p, prefer_dev, out);
        case B200_FMT_GIF: return gif_compress(in, in_len, p, prefer_dev, out);
        case B200_FMT_TIFF: return make_status(B200_ERR_UNSUPPORTED, "TIFF is outside the GPU path (route to caesium::compress_in_memory)");
        default: return make_status(B200_ERR_UNKNOWN_FORMAT, "Unknown file type");
    }
}

// libcaesium compress_to_size: quality bisection in [1, 100] from 80, at most 10 tries, 2 % tolerance, the largest result under
// the limit wins.  `size_at(q, keep)` runs one try: it returns the output size at quality q and, when `keep` says so (the try
// is the best so far, or the smallest so far for return_smallest), leaves the file in `cur`.
template <class SizeAt>
static b200_status bisect_quality(SizeAt size_at, size_t max_output_size, bool return_smallest, uint32_t *quality_out, std::vector<uint8_t> &result)
{
    const size_t tolerance = max_output_size / 50;
    int lo = 1, hi = 100, q = 80;
    std::vector<uint8_t> best, smallest, cur; size_t best_size = 0, smallest_size = (size_t)-1;
    for (int tries = 0; tries < 10 && lo <= hi; tries++) {
        size_t sz = 0;
        auto want = [&](size_t size) { return (size <= max_output_size && size > best_size) || (return_smallest && size < smallest_size); };
        b200_status s = size_at(q, want, sz, cur);
        if (s.code) return s;
        if (sz < smallest_size) { smallest_size = sz; if (return_smallest) smallest = cur; }
        if (sz <= max_output_size) {
            if (sz > best_size) { best_size = sz; best.swap(cur); if (quality_out) *quality_out = (uint32_t)q; }
            if (max_output_size - sz <= tolerance) break;
            lo = q + 1;
        } else hi = q - 1;
        q = (lo + hi) / 2;
    }
    if (best_size) { result.swap(best); return ok_status(); }
    if (return_smallest && !smallest.empty()) { result.swap(smallest); return ok_status(); }
    return make_status(B200_ERR_TOO_LARGE, "Cannot compress to desired size");
}

// JPEG: the source is entropy-decoded ONCE, its coefficients stay in HBM, and every try re-runs only dequant/IDCT/resample/FDCT/
// quantise at the try's tables plus the device Huffman encoder; the encoder reports the scan lengths from the device and the
// stuffed bytes are fetched only for tries that become the answer (SURVEY.md 8f-2: "decode once, re-quantise many").
static b200_status jpeg_to_size(const uint8_t *in, size_t in_len, b200_params *params, size_t max_output_size, bool return_smallest, std::vector<uint8_t> &result)
{
    std::string err;
    JpegReader rd(in, in_len);
    if (!rd.read_header(err)) return header_status(err);
    const JpegGeom &gin = rd.geom();
    if (fractional_sampling(gin)) return make_status(B200_ERR_UNSUPPORTED, kFractional);
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    if (params->width || params->height || (entropy_mode() & 1) == 0) {
        // resize, or the host-entropy mode: every try is a whole compress call (the resized planes are not kept between tries)
        auto size_at = [&](int q, auto want, size_t &sz, std::vector<uint8_t> &cur) {
            b200_params p = *params; p.jpeg_quality = (uint32_t)q; p.jpeg_optimize = 0;
            b200_status s = compress_dispatch(in, in_len, &p, -1, cur);
            sz = cur.size(); (void)want;
            return s;
        };
        return bisect_quality(size_at, max_output_size, return_smallest, &params->jpeg_quality, result);
    }
    SlotLease s(-1);
    if (!s) return s.failure();
    JpegGeom g0;
    if (!jpeg_output_geom(gin, 80, (int)params->jpeg_chroma_subsampling, g0, err)) return make_status(B200_ERR_INVALID_ARGUMENT, err);
    ImagePlan plan;
    if (!plan_image(gin, g0, plan, err)) return make_status(B200_ERR_UNSUPPORTED, err);
    if (!s->ensure(plan.in_bytes, plan.out_bytes, plan.scratch_bytes(), 1 << 14, err)) return make_status(B200_ERR_OUT_OF_MEMORY, err);
    bool resident;                                  // coefficients already in s->d_in?
    const b200_status st = decode_into_slot(s, rd, resident, err);
    if (st.code) return st;
    const JpegWriteOptions wo = write_options(params);
    auto size_at = [&](int q, auto want, size_t &sz, std::vector<uint8_t> &cur) -> b200_status {
        JpegGeom gout; std::string e2;
        if (!jpeg_output_geom(gin, q, (int)params->jpeg_chroma_subsampling, gout, e2)) return make_status(B200_ERR_INVALID_ARGUMENT, e2);
        if (!slot_transform(s, gin, gout, e2, false, !resident)) return make_status(B200_ERR_CUDA, e2);
        resident = true;                            // the first try uploaded them if the host decoded
        if (!slot_gpu_encode_sizes(s, gout, wo.progressive, e2)) return make_status(B200_ERR_CUDA, e2);
        sz = jpeg_assembled_size(gout, wo, &rd.meta(), s->enc->results.data(), (int)s->enc->results.size());
        if (want(sz)) {
            if (!slot_gpu_fetch(s, e2)) return make_status(B200_ERR_CUDA, e2);
            if (!jpeg_assemble(gout, wo, &rd.meta(), s->enc->results.data(), (int)s->enc->results.size(), cur, e2)) return make_status(B200_ERR_INVALID_ARGUMENT, e2);
        }
        return ok_status();
    };
    return bisect_quality(size_at, max_output_size, return_smallest, &params->jpeg_quality, result);
}

} // namespace

extern "C" {

void b200_params_default(b200_params *p)
{   // CSParameters::new(): jpeg q80 auto-subsampling progressive, png q80 level 3, gif 80, webp 60... caesiumclt overwrites the qualities (compressor.rs:415-417)
    memset(p, 0, sizeof(*p));
    p->jpeg_quality = 80; p->jpeg_chroma_subsampling = B200_CS_AUTO; p->jpeg_progressive = 1; p->jpeg_preserve_icc = 1;
    p->png_quality = 80; p->png_optimization_level = 3; p->gif_quality = 80; p->webp_quality = 80;
}

int b200_init(int n_gpus) { g_forced_ngpus = n_gpus; std::string e; return ensure_runtime(e) ? B200_OK : B200_ERR_NO_DEVICE; }
int b200_init_device(int ordinal) { g_forced_device = ordinal; std::string e; return ensure_runtime(e) ? B200_OK : B200_ERR_NO_DEVICE; }
void b200_shutdown(void) { print_trace(); runtime_shutdown(); }
int b200_device_count(void) { return runtime_device_count(); }
long long b200_device_jobs(int index) { return runtime_device_jobs(index); }
int b200_device_numa_node(int index) { return index < 0 || index >= runtime_device_count() ? -1 : device_numa_node(runtime_device_ordinal(index)); }
const char *b200_version(void) { return "b200-caesium 0.1.0 (sm_90a)"; }
void b200_free(void *p) { free(p); }
int b200_set_entropy_mode(int mode) { if (mode < 0 || mode > 3) return B200_ERR_INVALID_ARGUMENT; g_entropy_mode.store(mode); return B200_OK; }
int b200_set_png_lossy(int on) { if (on < 0 || on > 1) return B200_ERR_INVALID_ARGUMENT; g_png_lossy.store(on); return B200_OK; }
int b200_set_gif(int on) { if (on < 0 || on > 1) return B200_ERR_INVALID_ARGUMENT; g_gif.store(on); return B200_OK; }
int b200_set_png_resize(int on) { if (on < 0 || on > 1) return B200_ERR_INVALID_ARGUMENT; g_png_resize.store(on); return B200_OK; }
int b200_set_jpeg_trellis(int on) { if (on < 0 || on > 1) return B200_ERR_INVALID_ARGUMENT; set_jpeg_trellis(on == 1); return B200_OK; }

uint32_t b200_sniff_format(const uint8_t *d, size_t n)
{   // the magic numbers `infer` checks (scan_files.rs:30-40, compressor.rs:259-264)
    if (!d) return B200_FMT_UNKNOWN;
    if (n >= 3 && d[0] == 0xFF && d[1] == 0xD8 && d[2] == 0xFF) return B200_FMT_JPEG;
    if (n >= 8 && !memcmp(d, "\x89PNG\r\n\x1a\n", 8)) return B200_FMT_PNG;
    if (n >= 6 && (!memcmp(d, "GIF87a", 6) || !memcmp(d, "GIF89a", 6))) return B200_FMT_GIF;
    if (n >= 12 && !memcmp(d, "RIFF", 4) && !memcmp(d + 8, "WEBP", 4)) return B200_FMT_WEBP;
    if (n >= 4 && (!memcmp(d, "II*\0", 4) || !memcmp(d, "MM\0*", 4))) return B200_FMT_TIFF;
    return B200_FMT_UNKNOWN;
}

// ---- call coalescing (opt-in: B200_COALESCE=1) ----------------------------------------------------------------------------------
// The reference calls the codec one image at a time from every rayon worker (compressor.rs:81-83, :305); the GPU wants several
// same-shaped JPEGs per launch sequence.  With coalescing on, concurrent b200_compress_in_memory calls on JPEG inputs with equal
// parameters meet in a queue: the first caller to find no collector waits a few hundred microseconds for company (or until
// B200_COALESCE_TARGET calls have gathered), takes every matching call out of the queue and runs them as ONE b200_compress_batch
// on its own thread; the others sleep until their result is in.  Several such batches can be in flight.  Per call the semantics
// (result bytes, status, ownership) are those of the direct path.  Off by default until its effect is measured on a GPU box.
namespace {
struct CoReq { const uint8_t *in; size_t len; uint8_t *out = nullptr; size_t out_len = 0; b200_status st{0, nullptr}; bool done = false; b200_params params; };
struct Coalescer {
    std::mutex mu; std::condition_variable cv;
    std::vector<CoReq *> pending; bool collecting = false;
};
Coalescer g_co;
std::atomic<long> g_co_calls{0}, g_co_batches{0};
struct CoReport { ~CoReport() { if (getenv("B200_TRACE") && g_co_batches.load()) fprintf(stderr, "[b200 trace] coalescing: %ld calls in %ld batches\n", g_co_calls.load(), g_co_batches.load()); } } g_co_report;
int coalesce_mode()       // 0 off, 1 on
{
    static const int m = [] { const char *e = getenv("B200_COALESCE"); return e && atoi(e) > 0 ? 1 : 0; }();
    return m;
}
bool same_params_abi(const b200_params &a, const b200_params &b)
{
    return a.keep_metadata == b.keep_metadata && a.jpeg_quality == b.jpeg_quality && a.jpeg_chroma_subsampling == b.jpeg_chroma_subsampling &&
           a.jpeg_progressive == b.jpeg_progressive && a.jpeg_optimize == b.jpeg_optimize && a.jpeg_preserve_icc == b.jpeg_preserve_icc &&
           a.png_quality == b.png_quality && a.png_optimization_level == b.png_optimization_level && a.png_force_zopfli == b.png_force_zopfli &&
           a.png_optimize == b.png_optimize && a.gif_quality == b.gif_quality && a.webp_quality == b.webp_quality && a.webp_lossless == b.webp_lossless &&
           a.width == b.width && a.height == b.height;
}
b200_status coalesced_compress(const uint8_t *in, size_t in_len, const b200_params *params, uint8_t **out, size_t *out_len)
{
    static const int target = [] { const char *e = getenv("B200_COALESCE_TARGET"); const int v = e ? atoi(e) : 0; return v >= 2 && v <= 1024 ? v : 16; }();
    static const int window_us = [] { const char *e = getenv("B200_COALESCE_US"); const int v = e ? atoi(e) : 0; return v >= 1 && v <= 100000 ? v : 400; }();
    CoReq me; me.in = in; me.len = in_len; me.params = *params;
    std::unique_lock<std::mutex> lk(g_co.mu);
    g_co.pending.push_back(&me);
    g_co.cv.notify_all();                                     // a collector may be waiting for company
    while (!me.done) {
        if (g_co.collecting) { g_co.cv.wait(lk); continue; }
        bool queued = false; for (CoReq *r : g_co.pending) if (r == &me) { queued = true; break; }
        if (!queued) { g_co.cv.wait(lk); continue; }         // my call is inside somebody's batch
        // become the collector for calls with my parameters
        g_co.collecting = true;
        const auto deadline = std::chrono::steady_clock::now() + std::chrono::microseconds(window_us);
        for (;;) {
            int have = 0; for (CoReq *r : g_co.pending) if (same_params_abi(r->params, me.params)) have++;
            if (have >= target || g_co.cv.wait_until(lk, deadline) == std::cv_status::timeout) break;
        }
        std::vector<CoReq *> batch, left;
        for (CoReq *r : g_co.pending) (same_params_abi(r->params, me.params) && (int)batch.size() < 4 * target ? batch : left).push_back(r);
        g_co.pending.swap(left);
        g_co.collecting = false;
        g_co.cv.notify_all();                                 // leftovers / new arrivals elect their own collector
        lk.unlock();
        const int n = (int)batch.size();
        g_co_calls += n; g_co_batches++;
        bool ran = false;
        try {
            std::vector<const uint8_t *> ins((size_t)n); std::vector<size_t> lens((size_t)n); std::vector<uint8_t *> outs((size_t)n, nullptr); std::vector<size_t> ol((size_t)n, 0);
            std::vector<b200_status> sts((size_t)n, b200_status{0, nullptr});
            for (int i = 0; i < n; i++) { ins[(size_t)i] = batch[(size_t)i]->in; lens[(size_t)i] = batch[(size_t)i]->len; }
            const int rc = b200_compress_batch(ins.data(), lens.data(), n, &me.params, std::min(n, 16), outs.data(), ol.data(), sts.data());
            lk.lock();
            for (int i = 0; i < n; i++) {
                CoReq *r = batch[(size_t)i];
                if (rc < 0) r->st = make_status(B200_ERR_INVALID_ARGUMENT, "batch call failed");
                else { r->st = sts[(size_t)i]; r->out = outs[(size_t)i]; r->out_len = ol[(size_t)i]; }
                r->done = true;
            }
            ran = true;
        } catch (...) {}
        if (!ran) {                                           // nobody may be left waiting on a batch that died (allocation failure)
            if (!lk.owns_lock()) lk.lock();
            for (CoReq *r : batch) if (!r->done) { r->st = make_status(B200_ERR_OUT_OF_MEMORY, "out of memory in the coalesced batch"); r->done = true; }
        }
        g_co.cv.notify_all();
    }
    lk.unlock();
    if (me.st.code) { if (me.out) b200_free(me.out); return me.st; }
    *out = me.out; *out_len = me.out_len;
    return me.st;
}
} // namespace

b200_status b200_compress_in_memory(const uint8_t *in, size_t in_len, const b200_params *params, uint8_t **out, size_t *out_len)
{
    if (!in || !params || !out || !out_len) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    *out = nullptr; *out_len = 0;
    if (coalesce_mode() && b200_sniff_format(in, in_len) == B200_FMT_JPEG) return guarded([&] { return coalesced_compress(in, in_len, params, out, out_len); });
    return guarded([&] {
        std::vector<uint8_t> v;
        const b200_status s = compress_dispatch(in, in_len, params, -1, v);
        return s.code ? s : give(v, out, out_len);
    });
}

b200_status b200_convert_in_memory(const uint8_t *in, size_t in_len, const b200_params *params, uint32_t fmt, uint8_t **out, size_t *out_len)
{
    if (!in || !params || !out || !out_len) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    *out = nullptr; *out_len = 0;
    return guarded([&] {
        std::vector<uint8_t> v;
        const b200_status s = convert_dispatch(in, in_len, b200_sniff_format(in, in_len), fmt, params, v);
        return s.code ? s : give(v, out, out_len);
    });
}

// WebP: the source is decoded once, its RGB uploaded once (resized once if asked); every try runs K8 at the try's quality and the
// host boolean coder.
static b200_status webp_to_size(const uint8_t *in, size_t in_len, b200_params *params, size_t max_output_size, bool return_smallest, std::vector<uint8_t> &result)
{
    if (params->webp_lossless) return make_status(B200_ERR_UNSUPPORTED, "lossless WebP (VP8L) is outside the GPU path (route to caesium::compress_to_size_in_memory)");
    std::string err;
    WebpInfo wi; std::vector<uint8_t> rgb, alpha;
    b200_status st = webp_decode_status(in, in_len, wi, rgb, &alpha);
    if (st.code) return st;
    if (!alpha.empty()) return make_status(B200_ERR_UNSUPPORTED, "compress_to_size on a WebP with an alpha plane is outside the GPU path (route to caesium::compress_to_size_in_memory)");
    uint32_t nw, nh;
    if ((st = target_size((uint32_t)wi.width, (uint32_t)wi.height, params, 16383, nw, nh, "invalid dimensions for WebP")).code) return st;
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    SlotLease s(-1);
    if (!s) return s.failure();
    WebpDevice *webp = s->webp_dev();
    uint8_t *planes[3];
    // the (possibly resized) RGB planes stay in the slot's scratch memory for all tries
    if (!resize_host_planes(s, rgb.data(), (uint32_t)wi.width, (uint32_t)wi.height, nw, nh, 3, planes, err)) return make_status(B200_ERR_CUDA, err);
    auto size_at = [&](int q, auto want, size_t &sz, std::vector<uint8_t> &cur) -> b200_status {
        std::string e2; (void)want;
        if (!webp->encode_planes(planes[0], planes[1], planes[2], (int)nw, (int)nh, q, s->stream, cur, e2)) return make_status(B200_ERR_CUDA, e2);
        sz = cur.size();
        return ok_status();
    };
    return bisect_quality(size_at, max_output_size, return_smallest, &params->webp_quality, result);
}

// PNG (the lossy switch on): the source is decoded, un-filtered, (resized,) expanded and histogrammed once; every try runs median cut,
// refinement, dithering and coding at its png_quality
static b200_status png_to_size(const uint8_t *in, size_t in_len, b200_params *params, size_t max_output_size, bool return_smallest, std::vector<uint8_t> &result)
{
    if (!png_lossy()) return make_status(B200_ERR_UNSUPPORTED, "compress_to_size on a PNG bisects the lossy (imagequant) quality, which is outside the GPU path (route to caesium::compress_to_size_in_memory)");
    if ((params->width || params->height) && !png_resize()) return make_status(B200_ERR_UNSUPPORTED, "PNG resize is outside the GPU path (route to caesium::compress_to_size_in_memory)");
    std::string err;
    PngInfo info; PngIdat idat;
    if (!png_parse_chunks(in, in_len, params->keep_metadata != 0, info, idat, err)) return png_status(err);
    uint32_t nw, nh;
    b200_status st = png_target(info, params, nw, nh);
    if (st.code) return st;
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    SlotLease s(-1);
    if (!s) return s.failure();
    st = png_lossy_load(s, info, idat, nw, nh);
    if (st.code) return st;
    auto size_at = [&](int q, auto want, size_t &sz, std::vector<uint8_t> &cur) -> b200_status {
        (void)want;
        const b200_status r = png_lossy_code(s, info, q, (int)params->png_optimization_level, cur);
        sz = cur.size();
        return r;
    };
    return bisect_quality(size_at, max_output_size, return_smallest, &params->png_quality, result);
}

b200_status b200_compress_to_size_in_memory(const uint8_t *in, size_t in_len, b200_params *params, size_t max_output_size, uint8_t return_smallest,
                                            uint8_t **out, size_t *out_len)
{
    if (!in || !params || !out || !out_len) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    *out = nullptr; *out_len = 0;
    return guarded([&] {
        // input already small enough is returned unchanged
        if (in_len <= max_output_size) { std::vector<uint8_t> v(in, in + in_len); return give(v, out, out_len); }
        uint32_t fmt = b200_sniff_format(in, in_len);
        std::vector<uint8_t> result;
        b200_status s;
        if (fmt == B200_FMT_JPEG) s = jpeg_to_size(in, in_len, params, max_output_size, return_smallest != 0, result);
        else if (fmt == B200_FMT_WEBP) s = webp_to_size(in, in_len, params, max_output_size, return_smallest != 0, result);
        else if (fmt == B200_FMT_PNG) s = png_to_size(in, in_len, params, max_output_size, return_smallest != 0, result);
        else s = make_status(fmt == B200_FMT_UNKNOWN ? B200_ERR_UNKNOWN_FORMAT : B200_ERR_UNSUPPORTED, "compress_to_size for this format is outside the GPU path (route to caesium::compress_to_size_in_memory)");
        return s.code ? s : give(result, out, out_len);
    });
}

int b200_compress_batch(const uint8_t *const *in, const size_t *in_len, int n, const b200_params *params, int n_threads,
                        uint8_t **out, size_t *out_len, b200_status *status)
{
    if (!in || !in_len || !params || !out || !out_len || !status || n < 0) return -1;
    if (n_threads <= 0) n_threads = usable_cores();
    if (n_threads > n) n_threads = n;
    std::atomic<int> failed{0};
    { std::string e; ensure_runtime(e); }
    const int ndev = std::max(1, runtime_device_count());
    // Megabatches: with both entropy stages on the device, consecutive images are processed K at a time -- one launch
    // sequence (decode rounds, transform, encode passes) for the whole group instead of one per image.  Images that do not
    // fit the group path (other formats, progressive input, resize, odd one out in shape) go through the per-image path.
    int K = 8; { const char *e = getenv("B200_MEGABATCH"); if (e) K = std::max(1, std::min(64, atoi(e))); }
    const bool grouped = runtime_device_count() > 0 && entropy_mode() == 3 && K > 1 && ((!params->width && !params->height) || params->jpeg_optimize);
    auto one = [&](int i, int dev) {
        out[i] = nullptr; out_len[i] = 0;
        status[i] = guarded([&] {
            std::vector<uint8_t> v;
            const b200_status s = compress_dispatch(in[i], in_len[i], params, dev, v);
            return s.code ? s : give(v, &out[i], &out_len[i]);
        });
        if (status[i].code) failed++;
    };
    auto run_threads = [](int nt, const std::function<void()> &fn) {
        std::vector<std::thread> th;
        for (int t = 1; t < nt; t++) th.emplace_back(fn);
        fn();
        for (auto &t : th) t.join();
    };
    // phase 1: JPEGs, K at a time (one megabatch = one long launch sequence on one slot of one device).  Megabatches are sharded
    // over the devices by bytes -- longest-processing-time-first: largest megabatch to the least loaded device (SURVEY.md 8e) --
    // and every device gets its own workers, bound to the CPUs of the device's NUMA node; a worker whose device runs dry takes
    // work from the most loaded one.  Whatever a megabatch could not take is left for phase 2.
    std::vector<int> rest;
    if (grouped) {
        std::vector<int> jpegs;
        for (int i = 0; i < n; i++) (b200_sniff_format(in[i], in_len[i]) == B200_FMT_JPEG ? jpegs : rest).push_back(i);
        if (jpegs.size() < 2) { rest.insert(rest.end(), jpegs.begin(), jpegs.end()); jpegs.clear(); }
        const int nj = (int)jpegs.size();
        if (nj) {
            const int nchunks = (nj + K - 1) / K;
            std::vector<size_t> cbytes((size_t)nchunks, 0);
            for (int c = 0; c < nchunks; c++) for (int j = c * K; j < std::min(nj, c * K + K); j++) cbytes[(size_t)c] += in_len[jpegs[(size_t)j]];
            std::vector<int> order((size_t)nchunks); for (int c = 0; c < nchunks; c++) order[(size_t)c] = c;
            std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return cbytes[(size_t)a] > cbytes[(size_t)b]; });
            std::vector<std::vector<int>> devq((size_t)ndev); std::vector<size_t> load((size_t)ndev, 0);
            for (int c : order) { int d = 0; for (int e = 1; e < ndev; e++) if (load[(size_t)e] < load[(size_t)d]) d = e; devq[(size_t)d].push_back(c); load[(size_t)d] += cbytes[(size_t)c]; }
            std::vector<std::atomic<int>> cursor((size_t)ndev); for (auto &c : cursor) c.store(0);
            std::mutex rest_mu;
            int max_workers = 16; { const char *e = getenv("B200_GROUP_WORKERS"); if (e) max_workers = std::max(1, std::min(32, atoi(e))); }
            std::atomic<int> worker_id{0};
            auto group_worker = [&]() {
                const int home = worker_id.fetch_add(1) % ndev;
                AffinityGuard pin(runtime_device_ordinal(home));
                for (;;) {
                    int dev = home, c = -1;
                    { const int k = cursor[(size_t)home].fetch_add(1); if (k < (int)devq[(size_t)home].size()) c = devq[(size_t)home][(size_t)k]; }
                    if (c < 0) {           // home queue empty: help the device with the most work left
                        int best = -1, left = 0;
                        for (int e = 0; e < ndev; e++) { const int l = (int)devq[(size_t)e].size() - cursor[(size_t)e].load(); if (l > left) { left = l; best = e; } }
                        if (best < 0) break;
                        const int k = cursor[(size_t)best].fetch_add(1);
                        if (k >= (int)devq[(size_t)best].size()) continue;
                        c = devq[(size_t)best][(size_t)k]; dev = best;
                    }
                    const int j0 = c * K, j1 = std::min(nj, j0 + K);
                    std::vector<int> idx(jpegs.begin() + j0, jpegs.begin() + j1);
                    std::vector<char> done(idx.size(), 0);
                    try { jpeg_compress_group(in, in_len, idx, params, dev, out, out_len, status, done); } catch (...) {}
                    for (size_t k = 0; k < idx.size(); k++) {
                        if (done[k]) { if (status[idx[k]].code) failed++; }
                        else { std::lock_guard<std::mutex> lk(rest_mu); rest.push_back(idx[k]); }
                    }
                }
            };
            run_threads(std::max(1, std::min(n_threads, std::min(max_workers * ndev, nchunks))), group_worker);
        }
    } else for (int i = 0; i < n; i++) rest.push_back(i);
    // phase 2: one image per call on every thread the caller allows (PNG, conversions' sources, progressive JPEGs, ...)
    if (!rest.empty()) {
        std::sort(rest.begin(), rest.end());
        std::atomic<int> nr{0};
        const int total = (int)rest.size();
        std::atomic<int> tid{0};
        run_threads(std::min(n_threads, total), [&]() {
            const int home = tid.fetch_add(1) % ndev;            // thread t serves device t % ndev from that device's NUMA node
            AffinityGuard pin(runtime_device_ordinal(home));
            for (;;) { const int r = nr.fetch_add(1); if (r >= total) break; one(rest[r], home); }
        });
    }
    return failed.load();
}

// ---- JPEG stage entry points ------------------------------------------------------------------------------------
b200_status b200_jpeg_decode_coefficients(const uint8_t *in, size_t in_len, b200_jpeg_layout *layout, int16_t **coefs)
{
    if (!in || !layout || !coefs) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    *coefs = nullptr;
    std::string err;
    JpegReader rd(in, in_len);
    if (!rd.read_header(err)) return header_status(err);
    int16_t *c = (int16_t *)malloc((size_t)rd.geom().total_coefs * 2 + 16);
    if (!c) return make_status(B200_ERR_OUT_OF_MEMORY, "out of memory");
    if (!rd.decode(c, err)) { free(c); return make_status(B200_ERR_CORRUPT_INPUT, err); }
    layout_from_geom(rd.geom(), layout);
    *coefs = c;
    return ok_status();
}

b200_status b200_jpeg_output_layout(const b200_jpeg_layout *in_layout, const b200_params *params, b200_jpeg_layout *out_layout)
{
    if (!in_layout || !params || !out_layout) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    std::string err; JpegGeom gin, gout;
    if (!geom_from_layout(in_layout, gin, err)) return make_status(B200_ERR_INVALID_ARGUMENT, err);
    if (!jpeg_output_geom(gin, (int)params->jpeg_quality, (int)params->jpeg_chroma_subsampling, gout, err)) return make_status(B200_ERR_INVALID_ARGUMENT, err);
    gout.progressive = params->jpeg_progressive != 0;
    layout_from_geom(gout, out_layout);
    return ok_status();
}

b200_status b200_jpeg_requantize(const b200_jpeg_layout *in_layout, const int16_t *in_coefs, const b200_jpeg_layout *out_layout, int16_t *out_coefs)
{
    if (!in_layout || !in_coefs || !out_layout || !out_coefs) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    std::string err; JpegGeom gin, gout;
    if (!geom_from_layout(in_layout, gin, err) || !geom_from_layout(out_layout, gout, err)) return make_status(B200_ERR_INVALID_ARGUMENT, err);
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    ImagePlan plan;
    if (!plan_image(gin, gout, plan, err)) return make_status(B200_ERR_UNSUPPORTED, err);
    SlotLease s(-1);
    if (!s) return s.failure();
    if (!s->ensure(plan.in_bytes, plan.out_bytes, plan.scratch_bytes(), 1 << 14, err)) return make_status(B200_ERR_OUT_OF_MEMORY, err);
    memcpy(s->h_in, in_coefs, plan.in_bytes);
    memset(s->h_out, 0, plan.out_bytes);
    if (!slot_transform(s, gin, gout, err)) return make_status(B200_ERR_CUDA, err);
    jpeg_fill_dummy_blocks(gout, s->h_out);
    memcpy(out_coefs, s->h_out, plan.out_bytes);
    return ok_status();
}

b200_status b200_jpeg_encode_coefficients(const b200_jpeg_layout *layout, const int16_t *coefs, int progressive, uint8_t **out, size_t *out_len)
{
    if (!layout || !coefs || !out || !out_len) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    std::string err; JpegGeom g;
    if (!geom_from_layout(layout, g, err)) return make_status(B200_ERR_INVALID_ARGUMENT, err);
    JpegWriteOptions wo; wo.progressive = progressive != 0;
    std::vector<uint8_t> v;
    if (!jpeg_write(g, coefs, wo, nullptr, v, err)) return make_status(B200_ERR_INVALID_ARGUMENT, err);
    return give(v, out, out_len);
}

b200_status b200_jpeg_encode_coefficients_device(const b200_jpeg_layout *layout, const int16_t *coefs, int progressive, uint8_t **out, size_t *out_len)
{
    if (!layout || !coefs || !out || !out_len) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    std::string err; JpegGeom g;
    if (!geom_from_layout(layout, g, err)) return make_status(B200_ERR_INVALID_ARGUMENT, err);
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    SlotLease s(-1);
    if (!s) return s.failure();
    const size_t bytes = (size_t)g.total_coefs * 2;
    if (!s->ensure(256, bytes, 256, 1 << 14, err)) return make_status(B200_ERR_OUT_OF_MEMORY, err);
    memcpy(s->h_out, coefs, bytes);
    if (!slot_upload_out_coefs(s, bytes, err)) return make_status(B200_ERR_CUDA, err);
    JpegWriteOptions wo; wo.progressive = progressive != 0;
    if (!slot_gpu_encode(s, g, wo.progressive, err)) return make_status(B200_ERR_CUDA, err);
    std::vector<uint8_t> v;
    if (!jpeg_assemble(g, wo, nullptr, s->enc->results.data(), (int)s->enc->results.size(), v, err)) return make_status(B200_ERR_INVALID_ARGUMENT, err);
    return give(v, out, out_len);
}

b200_status b200_jpeg_decode_planes(const b200_jpeg_layout *in_layout, const int16_t *in_coefs, uint8_t *planes)
{
    if (!in_layout || !in_coefs || !planes) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    std::string err; JpegGeom gin;
    if (!geom_from_layout(in_layout, gin, err)) return make_status(B200_ERR_INVALID_ARGUMENT, err);
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    SlotLease s(-1);
    if (!s) return s.failure();
    if (!s->ensure((size_t)gin.total_coefs * 2, 256, 256, 1 << 14, err)) return make_status(B200_ERR_OUT_OF_MEMORY, err);
    memcpy(s->h_in, in_coefs, (size_t)gin.total_coefs * 2);
    SamplePlan sp;
    uint8_t *full[3];
    if (!(plan_samples(s, gin, gin.width, gin.height, nullptr, sp, err) && samples_from_coefs(s, gin, sp, true, false, full, err) &&
          slot_fetch_planes(s, full, gin.ncomp, (size_t)gin.width * gin.height, planes, err))) return make_status(B200_ERR_CUDA, err);
    return ok_status();
}

void b200_jpeg_quant_table(int quality, int which, uint16_t out[64]) { jpeg_quant_table(quality, which, out); }

// ---- device-resident full path ------------------------------------------------------------------------------------------
struct b200_jpeg_pipe { JpegPipe *p; };
b200_status b200_jpeg_pipe_create(const uint8_t *const *in, const size_t *in_len, int n, const b200_params *params, int group, b200_jpeg_pipe **pipe)
{
    if (!in || !in_len || !params || !pipe || n <= 0) return make_status(B200_ERR_INVALID_ARGUMENT, "invalid argument");
    *pipe = nullptr;
    std::string err;
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    return guarded([&] {
        JpegPipe *P = pipe_create(in, in_len, n, params, group > 0 ? group : 8, err);
        if (!P) return make_status(B200_ERR_INVALID_ARGUMENT, err);
        *pipe = new b200_jpeg_pipe{P};
        return ok_status();
    });
}
b200_status b200_jpeg_pipe_run(b200_jpeg_pipe *p, void *cuda_stream, int which, int *launches)
{
    std::string err; if (!p) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    return pipe_run(p->p, cuda_stream, which, launches, err) ? ok_status() : make_status(B200_ERR_CUDA, err);
}
b200_status b200_jpeg_pipe_finish(b200_jpeg_pipe *p, size_t *out_sizes, int *not_settled, int *enc_retries)
{
    std::string err; if (!p) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    return pipe_finish(p->p, out_sizes, not_settled, enc_retries, err) ? ok_status() : make_status(B200_ERR_CUDA, err);
}
b200_status b200_jpeg_pipe_fetch(b200_jpeg_pipe *p, int index, uint8_t **out, size_t *out_len)
{
    std::string err; if (!p || !out || !out_len) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    std::vector<uint8_t> v;
    if (!pipe_fetch(p->p, index, v, err)) return make_status(B200_ERR_CUDA, err);
    return give(v, out, out_len);
}
b200_status b200_jpeg_pipe_kernel_times(b200_jpeg_pipe *p, int iters, char *text, size_t cap)
{
    std::string err; if (!p || !text || !cap || iters <= 0) return make_status(B200_ERR_INVALID_ARGUMENT, "invalid argument");
    std::map<std::string, std::pair<double, int>> t;
    if (!pipe_kernel_times(p->p, iters, t, err)) return make_status(B200_ERR_CUDA, err);
    std::string s;
    for (auto &kv : t) { char b[160]; snprintf(b, sizeof b, "%s %.6f %d\n", kv.first.c_str(), kv.second.first, kv.second.second); s += b; }
    if (s.size() + 1 > cap) return make_status(B200_ERR_INVALID_ARGUMENT, "text buffer too small");
    memcpy(text, s.c_str(), s.size() + 1);
    return ok_status();
}
void b200_jpeg_pipe_destroy(b200_jpeg_pipe *p) { if (p) { pipe_destroy(p->p); delete p; } }

// ---- PNG stage entry points ----------------------------------------------------------------------------------------
// palette_rgba / npalette set: the samples are first reduced to a palette where png_reduce_palette finds one
static b200_status png_decode_abi(const uint8_t *in, size_t in_len, b200_png_info *info, uint8_t **raw, uint8_t *palette_rgba, int *npalette)
{
    std::string err; PngInfo pi; std::vector<uint8_t> r;
    if (!png_decode(in, in_len, false, pi, r, err)) return png_status(err);
    if (npalette) {
        *npalette = 0;
        if (png_reduce_palette(pi, r)) {
            *npalette = (int)(pi.plte.size() / 3);
            for (int k = 0; k < *npalette; k++) {
                palette_rgba[4 * k] = pi.plte[3 * k]; palette_rgba[4 * k + 1] = pi.plte[3 * k + 1]; palette_rgba[4 * k + 2] = pi.plte[3 * k + 2];
                palette_rgba[4 * k + 3] = (size_t)k < pi.trns.size() ? pi.trns[k] : 255;
            }
        }
    }
    info->width = pi.width; info->height = pi.height; info->bit_depth = pi.bit_depth; info->color_type = pi.color_type; info->bpp = pi.bpp; info->row_bytes = pi.row_bytes;
    size_t n;
    return give(r, raw, &n);
}
b200_status b200_png_decode(const uint8_t *in, size_t in_len, b200_png_info *info, uint8_t **raw)
{
    if (!in || !info || !raw) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    return png_decode_abi(in, in_len, info, raw, nullptr, nullptr);
}
b200_status b200_png_decode_reduced(const uint8_t *in, size_t in_len, b200_png_info *info, uint8_t **raw, uint8_t *palette_rgba, int *npalette)
{
    if (!in || !info || !raw || !palette_rgba || !npalette) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    return png_decode_abi(in, in_len, info, raw, palette_rgba, npalette);
}
b200_status b200_png_filter(const uint8_t *raw, int h, int row_bytes, int bpp, int strategy, uint8_t *filtered)
{
    if (!raw || !filtered || h <= 0 || row_bytes <= 0 || bpp < 1 || bpp > 8 || strategy < 0 || strategy > 9) return make_status(B200_ERR_INVALID_ARGUMENT, "invalid argument");
    std::string err;
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    SlotLease s(-1);                                                 // makes the slot's device current for this thread
    if (!s) return s.failure();
    return png_stage_filter(raw, h, row_bytes, bpp, strategy, filtered, err) ? ok_status() : make_status(B200_ERR_CUDA, err);
}
b200_status b200_png_lz77(const uint8_t *filtered, size_t n, int bpp, int stride, uint32_t **tokens, size_t *ntokens, uint32_t *hist)
{
    if (!filtered || !n || !tokens || !ntokens || !hist || bpp < 1 || stride < 1) return make_status(B200_ERR_INVALID_ARGUMENT, "invalid argument");
    std::string err;
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    SlotLease s(-1);
    if (!s) return s.failure();
    std::vector<uint32_t> t;
    if (!png_stage_lz77(filtered, n, bpp, stride, t, hist, err)) return make_status(B200_ERR_CUDA, err);
    return give(t, tokens, ntokens);
}
b200_status b200_png_deflate_tokens(const uint32_t *tokens, size_t ntokens, uint32_t adler, uint8_t **out, size_t *out_len)
{
    if ((!tokens && ntokens) || !out || !out_len) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    std::vector<uint8_t> z; deflate_tokens(tokens, ntokens, adler, z);
    return give(z, out, out_len);
}
int b200_webp_alpha_filter(const uint8_t *alpha, int width, int height, uint8_t *filtered)
{
    if (!alpha || !filtered || width < 1 || height < 1) return -1;
    std::vector<uint8_t> f;
    const int k = webp_alpha_choose_filter(alpha, width, height, f);
    memcpy(filtered, k ? f.data() : alpha, (size_t)width * height);
    return k;
}
b200_status b200_webp_alpha_chunk(const uint32_t *tokens, size_t ntokens, int width, int height, int filter, uint8_t **out, size_t *out_len)
{
    if (!tokens || !out || !out_len || width < 1 || height < 1 || width > 16383 || height > 16383 || filter < 0 || filter > 3) return make_status(B200_ERR_INVALID_ARGUMENT, "invalid argument");
    std::vector<uint8_t> a;
    if (!vp8l_alpha_from_tokens(tokens, ntokens, width, height, a, filter)) return make_status(B200_ERR_INVALID_ARGUMENT, "the tokens do not cover the plane");
    return give(a, out, out_len);
}
b200_status b200_webp_wrap_alpha(const uint8_t *simple_file, size_t file_len, const uint8_t *alph, size_t alph_len, int width, int height, uint8_t **out, size_t *out_len)
{
    if (!simple_file || !alph || !out || !out_len || width < 1 || height < 1 || width > 16383 || height > 16383) return make_status(B200_ERR_INVALID_ARGUMENT, "invalid argument");
    std::vector<uint8_t> f(simple_file, simple_file + file_len), a(alph, alph + alph_len), o;
    if (!webp_wrap_alpha(f, a, width, height, o)) return make_status(B200_ERR_INVALID_ARGUMENT, "not a simple lossy WebP file");
    return give(o, out, out_len);
}
// ---- WebP stage entry points -----------------------------------------------------------------------------------------
b200_status b200_webp_encode_rgb(const uint8_t *rgb, int w, int h, int quality, uint8_t **out, size_t *out_len, int16_t *levels, uint8_t *modes)
{
    if (!rgb || !out || !out_len || w < 1 || h < 1 || w > 16383 || h > 16383) return make_status(B200_ERR_INVALID_ARGUMENT, "invalid argument");
    *out = nullptr; *out_len = 0;
    std::string err;
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    SlotLease s(-1);
    if (!s) return s.failure();
    std::vector<uint8_t> v;
    if (!s->webp_dev()->encode_host_rgb(rgb, w, h, quality, s->stream, v, err, levels, modes)) return make_status(B200_ERR_CUDA, err);
    return give(v, out, out_len);
}
b200_status b200_webp_decode(const uint8_t *in, size_t in_len, int *width, int *height, uint8_t **rgb)
{
    if (!in || !width || !height || !rgb) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    *rgb = nullptr;
    return guarded([&] {
        WebpInfo wi; std::vector<uint8_t> v, a;
        const b200_status s = webp_decode_status(in, in_len, wi, v, &a);
        if (s.code) return s;
        *width = wi.width; *height = wi.height;
        size_t n = 0;
        return give(v, rgb, &n);
    });
}
b200_status b200_webp_decode_rgba(const uint8_t *in, size_t in_len, int *width, int *height, uint8_t **rgb, uint8_t **alpha)
{
    if (!in || !width || !height || !rgb || !alpha) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    *rgb = nullptr; *alpha = nullptr;
    return guarded([&] {
        WebpInfo wi; std::vector<uint8_t> v, a;
        b200_status s = webp_decode_status(in, in_len, wi, v, &a);
        if (s.code) return s;
        *width = wi.width; *height = wi.height;
        size_t n = 0;
        if (!a.empty()) { s = give(a, alpha, &n); if (s.code) return s; }
        s = give(v, rgb, &n);
        if (s.code) { free(*alpha); *alpha = nullptr; }
        return s;
    });
}
b200_status b200_webp_write_levels(int w, int h, int quality, const int16_t *levels, const uint8_t *modes, uint8_t **out, size_t *out_len)
{
    if (!levels || !modes || !out || !out_len) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    std::vector<uint8_t> v;
    if (!vp8_write_file(w, h, vp8_qindex(quality < 0 ? 0 : quality > 100 ? 100 : quality), levels, modes, v)) return make_status(B200_ERR_INVALID_ARGUMENT, "frame cannot be written as VP8");
    return give(v, out, out_len);
}
unsigned long long b200_webp_d2h_bytes(void) { return webp_d2h_bytes_total(); }
int b200_webp_qindex(int quality, int factors[6])
{
    const int q = vp8_qindex(quality < 0 ? 0 : quality > 100 ? 100 : quality);
    if (factors) vp8_quant_factors(q, factors);
    return q;
}

b200_status b200_png_device_times(const uint8_t *in, size_t in_len, int level, int iters, char *text, size_t cap)
{
    if (!in || !text || !cap || iters <= 0) return make_status(B200_ERR_INVALID_ARGUMENT, "invalid argument");
    std::string err;
    PngInfo info0; PngIdat idat;
    if (!png_parse_chunks(in, in_len, false, info0, idat, err)) return make_status(B200_ERR_CORRUPT_INPUT, err);
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    std::map<std::string, std::pair<double, int>> acc;
    {
        SlotLease s(-1);
        if (!s) return s.failure();
        PngDevice *png = s->png_dev();
        const size_t nin = (info0.row_bytes + 1) * (size_t)info0.height;
        size_t bcap = 0, got = 0; uint32_t adler = 0;
        uint8_t *buf = png->input_buffer(nin, bcap, err);
        if (!buf) return make_status(B200_ERR_OUT_OF_MEMORY, err);
        if (!zlib_inflate_to(idat.p, idat.n, buf, bcap, nin, &got, &adler, err) || got < nin) return make_status(B200_ERR_CORRUPT_INPUT, err.empty() ? "IDAT too short" : err);
        std::vector<uint8_t> z;
        for (int it = 0; it <= iters; it++) {          // iteration 0 warms buffers up and is not counted
            PngInfo info = info0;
            LaunchTimer lt; lt.begin((cudaStream_t)s->stream);
            tl_launch_timer = it ? &lt : nullptr;
            const bool ok = png->compress_filtered(info, got, adler, level < 0 ? 0 : level > 6 ? 6 : level, s->stream, z, nullptr, err);
            tl_launch_timer = nullptr;
            if (!ok) return make_status(B200_ERR_CUDA, err);
            if (it) lt.collect(acc);
        }
    }
    std::string out;
    for (auto &kv : acc) { char b[160]; snprintf(b, sizeof b, "%s %.6f %d\n", kv.first.c_str(), kv.second.first / kv.second.second, kv.second.second / iters); out += b; }
    if (out.size() + 1 > cap) return make_status(B200_ERR_INVALID_ARGUMENT, "text buffer too small");
    memcpy(text, out.c_str(), out.size() + 1);
    return ok_status();
}

b200_status b200_png_quantize(const uint8_t *rgba, int width, int height, int quality, uint8_t *palette_rgba, int *npalette, uint8_t *indices)
{
    if (!rgba || !palette_rgba || !npalette || !indices || width < 1 || height < 1 || width > 65535 || height > 65535 || quality < 0 || quality > 100)
        return make_status(B200_ERR_INVALID_ARGUMENT, "invalid argument");
    std::string err;
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    return guarded([&] {
        SlotLease s(-1);
        if (!s) return s.failure();
        PngQuant *q = s->png_dev()->quantiser();
        std::vector<uint32_t> pal;
        if (!q->load_host(rgba, width, height, s->stream, err) || !q->prepare(s->stream, err) || !q->quantize(quality, s->stream, pal, err) ||
            !q->fetch_indices(indices, s->stream, err)) return make_status(B200_ERR_CUDA, err);
        for (size_t k = 0; k < pal.size(); k++) for (int c = 0; c < 4; c++) palette_rgba[4 * k + c] = (uint8_t)(pal[k] >> (8 * c));
        *npalette = (int)pal.size();
        return ok_status();
    });
}

b200_status b200_png_resize_samples(const uint8_t *in, size_t in_len, uint32_t width, uint32_t height, b200_png_info *info, uint8_t **raw)
{
    if (!in || !info || !raw) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    *raw = nullptr;
    return guarded([&] {
        std::string err;
        PngInfo pi; PngIdat idat;
        if (!png_parse_chunks(in, in_len, false, pi, idat, err)) return png_status(err);
        b200_params p; memset(&p, 0, sizeof p); p.width = width; p.height = height;
        uint32_t nw, nh;                                        // both 0: the expanded image at the source's size
        const b200_status st = target_size(pi.width, pi.height, &p, 65535, nw, nh, "invalid target dimensions");
        if (st.code) return st;
        if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
        SlotLease s(-1);
        if (!s) return s.failure();
        PngDevice *png = s->png_dev();
        const size_t nin = (pi.row_bytes + 1) * (size_t)pi.height;
        size_t cap = 0, got = 0; uint32_t stored_adler = 0;
        uint8_t *buf = png->input_buffer(nin, cap, err);
        if (!buf) return make_status(B200_ERR_OUT_OF_MEMORY, err);
        if (!zlib_inflate_to(idat.p, idat.n, buf, cap, nin, &got, &stored_adler, err)) return make_status(B200_ERR_CORRUPT_INPUT, err);
        if (got < nin) return make_status(B200_ERR_CORRUPT_INPUT, "IDAT too short");
        std::vector<uint8_t> r;
        if (!png->resize_filtered(pi, got, stored_adler, nw, nh, s->stream, r, err)) return png_device_status(png, true, err);
        info->width = pi.width; info->height = pi.height; info->bit_depth = pi.bit_depth; info->color_type = pi.color_type; info->bpp = pi.bpp; info->row_bytes = pi.row_bytes;
        size_t n;
        return give(r, raw, &n);
    });
}

b200_status b200_gif_decode(const uint8_t *in, size_t in_len, int *width, int *height, int *nframes, int *loop, uint8_t **rgba, int **delays)
{
    if (!in || !width || !height || !nframes || !loop || !rgba || !delays) return make_status(B200_ERR_INVALID_ARGUMENT, "null argument");
    *rgba = nullptr; *delays = nullptr;
    return guarded([&] {
        std::string err;
        GifReader rd;
        if (!rd.open(in, in_len, err)) return make_status(rd.unsupported ? B200_ERR_UNSUPPORTED : B200_ERR_CORRUPT_INPUT, err);
        const size_t npix = (size_t)rd.width * rd.height;
        std::vector<uint32_t> px(npix * (size_t)rd.frames);
        std::vector<int> dl((size_t)rd.frames);
        for (int f = 0; f < rd.frames; f++)
            if (!rd.next(px.data() + npix * f, dl[(size_t)f], err)) return make_status(B200_ERR_CORRUPT_INPUT, err.empty() ? "GIF frame missing" : err);
        size_t n = 0;
        std::vector<uint8_t> bytes(px.size() * 4);
        memcpy(bytes.data(), px.data(), bytes.size());
        b200_status s = give(dl, delays, &n);
        if (s.code) return s;
        s = give(bytes, rgba, &n);
        if (s.code) { free(*delays); *delays = nullptr; return s; }
        *width = rd.width; *height = rd.height; *nframes = rd.frames; *loop = rd.loop;
        return s;
    });
}

b200_status b200_gif_lzw(const uint8_t *indices, size_t n, int min_code_size, uint8_t **out, size_t *out_len)
{
    if (!indices || !out || !out_len || min_code_size < 2 || min_code_size > 8) return make_status(B200_ERR_INVALID_ARGUMENT, "invalid argument");
    *out = nullptr; *out_len = 0;
    for (size_t i = 0; i < n; i++) if (indices[i] >> min_code_size) return make_status(B200_ERR_INVALID_ARGUMENT, "index not below 2^min_code_size");
    std::string err;
    if (!ensure_runtime(err)) return make_status(B200_ERR_NO_DEVICE, err);
    return guarded([&] {
        SlotLease s(-1);
        if (!s) return s.failure();
        DeviceBuffer<uint8_t> d_idx;
        std::vector<uint8_t> v;
        if (!d_idx.reserve(n + 1, Grow::Exact, err)) return make_status(B200_ERR_OUT_OF_MEMORY, err);
        if (cudaMemcpyAsync(d_idx, indices, n, cudaMemcpyHostToDevice, (cudaStream_t)s->stream) != cudaSuccess || !s->gif_dev()->lzw(d_idx, n, min_code_size, s->stream, v, err))
            return make_status(B200_ERR_CUDA, err.empty() ? "upload failed" : err);
        return give(v, out, out_len);
    });
}

int b200_png_level_strategies(int level, int *out)
{
    const std::vector<int> v = png_level_strategies(level < 0 ? 0 : level > 6 ? 6 : level);
    if (out) for (size_t i = 0; i < v.size(); i++) out[i] = v[i];
    return (int)v.size();
}

} // extern "C"
