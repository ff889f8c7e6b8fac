// jpeg_pipe.cu -- the JPEG re-encode path with everything resident in HBM: n same-shaped baseline JPEGs are parsed once,
// their entropy-coded bytes uploaded once, and every run() enqueues the FULL device path -- Huffman decode, dequant/IDCT/
// chroma resample/FDCT/quantise, Huffman encode with optimal tables, byte stuffing -- for all of them, megabatch by megabatch
// on a set of streams, without a single host wait: scan bytes in HBM -> scan bytes in HBM.  This is what bench.py reports as
// `value` (SURVEY.md 8d: inputs resident when the timed region starts); b200_compress_batch runs the same launch sequences with
// the H2D / D2H copies and the file assembly around them (bench.py's `e2e`).  Reference path: caesium::compress_in_memory,
// caesium-clt's src/compressor.rs:305.
#include <cuda_runtime.h>
#include <map>
#include <memory>
#include <string>
#include <vector>
#include "jpeg_device.h"
#include "jpeg_pipe.h"
#include "launch_timer.h"
#include "stream_wait.h"

namespace b200 {

struct PipeGroup {
    Slot slot;                                  // private buffers + stream (not from the runtime's pool)
    cudaEvent_t done = nullptr;
    std::vector<int> members;                   // image indices
    std::vector<GpuDecoder::Item> items;
    std::vector<const JpegGeom *> gins;
    GroupLayout L;
    std::vector<int16_t *> bases;
};

struct JpegPipe {
    int n = 0, K = 0, dev = 0;
    bool lossless = false, progressive = true, trellis = false;
    JpegGeom gout;
    JpegWriteOptions wo;
    std::vector<std::unique_ptr<JpegReader>> rd;
    std::vector<JpegReader::DeviceScan> ds;
    std::vector<std::unique_ptr<PipeGroup>> groups;
    cudaEvent_t fork = nullptr;
    bool finished = false;
    ~JpegPipe();
};

JpegPipe::~JpegPipe()
{
    for (auto &g : groups) {
        if (g->slot.stream) cudaStreamSynchronize((cudaStream_t)g->slot.stream);
        if (g->done) cudaEventDestroy(g->done);
    }
    if (fork) cudaEventDestroy(fork);
    groups.clear();             // ~Slot: streams and buffers
}

JpegPipe *pipe_create(const uint8_t *const *in, const size_t *in_len, int n, const b200_params *p, int K, std::string &err)
{
    if (n <= 0 || K <= 0) { err = "empty pipe"; return nullptr; }
    std::unique_ptr<JpegPipe> P(new JpegPipe());
    P->n = n; P->K = K; P->lossless = p->jpeg_optimize != 0; P->progressive = p->jpeg_progressive != 0; P->trellis = !P->lossless && jpeg_trellis();
    P->wo = write_options(p); P->wo.copy_jfif = P->lossless;
    P->rd.resize((size_t)n); P->ds.resize((size_t)n);
    for (int i = 0; i < n; i++) {
        P->rd[i].reset(new JpegReader(in[i], in_len[i]));
        if (!P->rd[i]->read_header(err)) return nullptr;
        if (!P->rd[i]->device_decodable(P->ds[i])) { err = "input " + std::to_string(i) + " is not a baseline single-scan JPEG (the resident pipe takes only those)"; return nullptr; }
        if (!same_shape(P->rd[0]->geom(), P->rd[i]->geom())) { err = "inputs of a resident pipe must share one shape"; return nullptr; }
    }
    const JpegGeom &gin0 = P->rd[0]->geom();
    if (P->lossless) P->gout = gin0;
    else if (!jpeg_output_geom(gin0, (int)p->jpeg_quality, (int)p->jpeg_chroma_subsampling, P->gout, err)) return nullptr;
    {   // device of slot pool 0 (the runtime is initialised by the caller)
        Slot *s0 = slot_acquire(0, err); if (!s0) return nullptr; P->dev = s0->dev; slot_release(s0);
    }
    if (cudaEventCreateWithFlags(&P->fork, cudaEventDisableTiming) != cudaSuccess) { err = "cudaEventCreate failed"; return nullptr; }
    for (int i0 = 0; i0 < n; i0 += K) {
        std::unique_ptr<PipeGroup> G(new PipeGroup());
        const int Kg = std::min(K, n - i0);
        cudaStream_t st;
        if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) { err = "cudaStreamCreate failed"; return nullptr; }
        G->slot.stream = st; G->slot.dev = P->dev;
        if (cudaEventCreateWithFlags(&G->done, cudaEventDisableTiming) != cudaSuccess) { err = "cudaEventCreate failed"; return nullptr; }
        if (!slot_group_layout(&G->slot, gin0, P->gout, Kg, G->L, err)) return nullptr;
        G->items.resize((size_t)Kg); G->gins.resize((size_t)Kg); G->bases.resize((size_t)Kg);
        size_t raw = 0;
        for (int m = 0; m < Kg; m++) {
            const int i = i0 + m;
            G->members.push_back(i);
            G->items[m].rd = P->rd[i].get(); G->items[m].ds = &P->ds[i]; G->items[m].result = GpuDecoder::FAILED;
            G->items[m].d_coefs = G->L.coefs(G->slot, m, true); G->items[m].defer_dc = !P->lossless;
            G->gins[m] = &P->rd[i]->geom();
            G->bases[m] = G->L.coefs(G->slot, m, P->lossless);
            raw += P->ds[i].ecs_end - P->ds[i].ecs_begin;
        }
        if (!G->slot.decoder()->prepare(G->items, st, err) || !G->slot.dec->upload(st, err)) return nullptr;       // entropy-coded bytes + tables go up here, once
        if (!G->slot.encoder()->prepare(P->gout, P->progressive, G->bases.data(), Kg, st, raw, err) || !G->slot.enc->upload(st, err)) return nullptr;
        if (cudaStreamSynchronize(st) != cudaSuccess) { err = "upload failed"; return nullptr; }
        P->groups.push_back(std::move(G));
    }
    return P.release();
}

static bool enqueue_group(JpegPipe *P, PipeGroup &G, int which, int *launches, std::string &err)
{
    Slot *s = &G.slot;
    int n = 0;
    if (which == 0 || which == 1) { if (!s->dec->enqueue(s->stream, err)) return false; n += s->dec->launches; }
    if (!P->lossless && (which == 0 || which == 2)) { if (!slot_transform_group(s, G.gins.data(), P->gout, G.L, P->trellis, err)) return false; n += P->trellis ? 4 : 3; }
    if (which == 0 || which == 3) { if (!s->enc->enqueue(s->stream, true, err)) return false; n += s->enc->launches; }
    if (launches) *launches += n;
    return true;
}

bool pipe_run(JpegPipe *P, void *stream_, int which, int *launches, std::string &err)
{
    cudaStream_t caller = (cudaStream_t)stream_;
    cudaSetDevice(runtime_device_ordinal(P->dev));
    if (launches) *launches = 0;
    P->finished = false;
    CU(cudaEventRecord(P->fork, caller));
    for (auto &G : P->groups) {
        cudaStream_t st = (cudaStream_t)G->slot.stream;
        CU(cudaStreamWaitEvent(st, P->fork, 0));
        if (!enqueue_group(P, *G, which, launches, err)) return false;
        CU(cudaEventRecord(G->done, st));
        CU(cudaStreamWaitEvent(caller, G->done, 0));
    }
    return true;
}

bool pipe_finish(JpegPipe *P, size_t *out_sizes, int *not_settled, int *enc_retries, std::string &err)
{
    cudaSetDevice(runtime_device_ordinal(P->dev));
    int bad = 0, retries = 0;
    for (auto &G : P->groups) {
        Slot *s = &G->slot;
        CU(cudaStreamSynchronize((cudaStream_t)s->stream));
        const int r0 = s->enc->retries;
        if (!s->enc->finish(s->stream, false, err)) return false;
        retries += s->enc->retries - r0;
        s->dec->finish(G->items);
        const int spi = s->enc->plan.scans_per_image;
        for (size_t m = 0; m < G->members.size(); m++) {
            if (G->items[m].result != GpuDecoder::OK) bad++;
            size_t tot = 0; for (int k = 0; k < spi; k++) tot += s->enc->results[m * spi + k].len;
            if (out_sizes) out_sizes[G->members[m]] = tot;
        }
    }
    if (not_settled) *not_settled = bad;
    if (enc_retries) *enc_retries = retries;
    P->finished = true;
    return true;
}

bool pipe_fetch(JpegPipe *P, int index, std::vector<uint8_t> &file, std::string &err)
{
    if (index < 0 || index >= P->n) { err = "bad image index"; return false; }
    if (!P->finished) { err = "pipe_fetch before pipe_finish"; return false; }
    cudaSetDevice(runtime_device_ordinal(P->dev));
    PipeGroup &G = *P->groups[(size_t)(index / P->K)];
    Slot *s = &G.slot;
    const int m = index % P->K, spi = s->enc->plan.scans_per_image;
    if (!s->enc->finish(s->stream, true, err)) return false;               // sizes are known: this only fetches the stuffed scans
    return jpeg_assemble(P->lossless ? P->rd[index]->geom() : P->gout, P->wo, &P->rd[index]->meta(), s->enc->results.data() + (size_t)m * spi, spi, file, err);
}

// One megabatch alone on its stream with an event after every launch: name -> (ms per launch, launches per megabatch), averaged
// over `iters` runs.  The table bench.py turns into per-kernel roofline fractions.
bool pipe_kernel_times(JpegPipe *P, int iters, std::map<std::string, std::pair<double, int>> &out, std::string &err)
{
    cudaSetDevice(runtime_device_ordinal(P->dev));
    PipeGroup &G = *P->groups[0];
    cudaStream_t st = (cudaStream_t)G.slot.stream;
    CU(cudaDeviceSynchronize());
    std::map<std::string, std::pair<double, int>> acc;
    for (int it = 0; it < iters; it++) {
        LaunchTrace tr(st, true);
        if (!enqueue_group(P, G, 0, nullptr, err)) return false;
        CU(cudaStreamSynchronize(st));
        tr.lt.collect(acc);
    }
    out.clear();
    for (auto &kv : acc) out[kv.first] = std::make_pair(kv.second.first / kv.second.second, kv.second.second / iters);
    return true;
}

void pipe_destroy(JpegPipe *P) { if (P) { cudaSetDevice(runtime_device_ordinal(P->dev)); delete P; } }
int pipe_group_size(const JpegPipe *P) { return P->K; }
int pipe_groups(const JpegPipe *P) { return (int)P->groups.size(); }

} // namespace b200
