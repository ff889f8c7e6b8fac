// png_quant.cu -- the lossy PNG leg's palette quantiser (libcaesium png::compress with optimize == false reaches imagequant;
// this is the device's own quantiser, rules in png_quant_core.h): expand to RGBA8, a dense histogram of 2^20 cells, compaction of
// the occupied cells (CUB), median cut over the cells (the host picks each split from O(boxes) statistics the device computes),
// k-means refinement, exact nearest-entry candidate lists, Floyd-Steinberg as a wavefront, index packing.
#include <cuda_runtime.h>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <algorithm>
#include <chrono>
#include <climits>
#include <cstring>
#include "png_quant.h"
#include "png_quant_core.h"
#include "png_kernels.h"
#include "stream_wait.h"
#include "launch_timer.h"

namespace b200 {

#define KCHECK(name) do { LT_MARK(name); if (!launch_ok(cudaGetLastError(), name, err)) return false; } while (0)

static const int kSmall = 32 * 1024;          // pinned readback buffer

// image-sized buffers: the smallest power of two >= 64 KiB and >= need + need / 4; the rest are allocated at their exact size
template <class B> static bool grow(B &buf, size_t need, std::string &err) { return buf.reserve(need, Grow::Pow2Quarter, err); }
template <class B> static bool fixed(B &buf, size_t bytes, std::string &err) { return buf.reserve(bytes, Grow::Exact, err); }

// ---- kernels -------------------------------------------------------------------------------------------------------------------
// any PNG colour type / bit depth -> RGBA8 (16 bits: the high byte; sub-byte grey scaled to 8 bits; palette and tRNS through lut;
// a colour key gives alpha 0)
__global__ void k_pq_expand(const uint8_t *__restrict__ raw, size_t rb, int w, int h, int ct, int bd, const uint32_t *__restrict__ lut,
                            int has_key, int k0, int k1, int k2, uint32_t *__restrict__ rgba)
{
    const size_t npix = (size_t)w * h;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (size_t)gridDim.x * blockDim.x) {
        const int y = (int)(i / w), x = (int)(i % w);
        const uint8_t *row = raw + (size_t)y * rb;
        const int bps = bd == 16 ? 2 : 1;
        uint32_t out;
        if (ct == 2 || ct == 6) {
            const int ch = ct == 2 ? 3 : 4;
            const uint8_t *p = row + (size_t)x * ch * bps;
            const uint32_t r = p[0], g = p[bps], b = p[2 * bps];
            uint32_t a = ct == 6 ? p[3 * bps] : 255;
            if (has_key && ct == 2) {
                const int s0 = bps == 2 ? (p[0] << 8 | p[1]) : p[0], s1 = bps == 2 ? (p[2] << 8 | p[3]) : p[1], s2 = bps == 2 ? (p[4] << 8 | p[5]) : p[2];
                if (s0 == k0 && s1 == k1 && s2 == k2) a = 0;
            }
            out = r | g << 8 | b << 16 | a << 24;
        } else if (ct == 4) {
            const uint8_t *p = row + (size_t)x * 2 * bps;
            out = (uint32_t)p[0] * 0x010101u | (uint32_t)p[bps] << 24;
        } else {
            int v;
            if (bd == 16) v = row[2 * x] << 8 | row[2 * x + 1];
            else if (bd == 8) v = row[x];
            else v = (row[(x * bd) >> 3] >> (8 - bd - ((x * bd) & 7))) & ((1 << bd) - 1);
            if (ct == 3) out = lut[v & 255];
            else {
                const uint32_t g = bd == 16 ? (uint32_t)(v >> 8) : bd == 8 ? (uint32_t)v : (uint32_t)(v * 255 / ((1 << bd) - 1));
                out = g * 0x010101u | (has_key && v == k0 ? 0u : 255u << 24);
            }
        }
        rgba[i] = out;
    }
}

// planes [nc][n] (+ an alpha plane after them) -> RGBA8
__global__ void k_pq_planes(const uint8_t *__restrict__ planes, size_t n, int nc, int has_alpha, uint32_t *__restrict__ rgba)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t r = planes[i], g = nc == 3 ? planes[n + i] : r, b = nc == 3 ? planes[2 * n + i] : r;
        const uint32_t a = has_alpha ? planes[(size_t)nc * n + i] : 255u;
        rgba[i] = r | g << 8 | b << 16 | a << 24;
    }
}

// fully transparent pixels are not counted: they take the reserved entry (*clear = 1 when there is one)
__global__ void k_pq_hist(const uint32_t *__restrict__ rgba, size_t npix, unsigned long long *__restrict__ count, unsigned long long *__restrict__ sums,
                          uint32_t *__restrict__ clear)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (size_t)gridDim.x * blockDim.x) {
        int p[4]; pq_premul(rgba[i], p);
        if (p[3] == 0) { if (!*(volatile uint32_t *)clear) *clear = 1; continue; }
        const uint32_t c = pq_cell(p);
        atomicAdd(&count[c], 1ull);
#pragma unroll
        for (int k = 0; k < 4; k++) if (p[k]) atomicAdd(&sums[4 * (size_t)c + k], (unsigned long long)p[k]);
    }
}

struct PqOccupied {
    const unsigned long long *count;
    __host__ __device__ bool operator()(const uint32_t c) const { return count[c] != 0; }
};

__device__ __forceinline__ void pq_rep(const unsigned long long *count, const unsigned long long *sums, uint32_t cell, int v[4], unsigned long long &n)
{
    n = count[cell];
#pragma unroll
    for (int k = 0; k < 4; k++) v[k] = (int)((sums[4 * (size_t)cell + k] + n / 2) / n);
}

// one median-cut split: cells of box b with coordinate > t on `axis` move to box k (axis < 0: nothing moves); statistics of both
// boxes (PqBox layout) are summed into box[0] / box[1]
__global__ void __launch_bounds__(256) k_pq_split(const uint32_t *__restrict__ cells, int ncells, const unsigned long long *__restrict__ count,
                                                  const unsigned long long *__restrict__ sums, uint8_t *__restrict__ label, int b, int axis, int t, int k,
                                                  unsigned long long *__restrict__ box)
{
    __shared__ unsigned long long sb[2 * PQ_BOX_WORDS];
    for (int i = threadIdx.x; i < 2 * PQ_BOX_WORDS; i += blockDim.x) sb[i] = 0;
    __syncthreads();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ncells; i += gridDim.x * blockDim.x) {
        if (label[i] != b) continue;
        const uint32_t cell = cells[i];
        int side = 0;
        if (axis >= 0 && pq_cell_coord(cell, axis) > t) { label[i] = (uint8_t)k; side = 1; }
        int v[4]; unsigned long long n; pq_rep(count, sums, cell, v, n);
        unsigned long long *s = sb + side * PQ_BOX_WORDS;
        atomicAdd(&s[0], n);
#pragma unroll
        for (int c = 0; c < 4; c++) {
            atomicAdd(&s[1 + c], n * (unsigned long long)v[c]);
            atomicAdd(&s[5 + c], n * (unsigned long long)(v[c] * v[c]));
            atomicAdd(&s[9 + c * PQ_BINS + pq_cell_coord(cell, c)], n);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * PQ_BOX_WORDS; i += blockDim.x) if (sb[i]) atomicAdd(&box[i], sb[i]);
}

// per entry: pixel count and exact premultiplied sums of its cells; a cell's entry is its box (coords == nullptr) or the nearest entry
__global__ void __launch_bounds__(256) k_pq_accum(const uint32_t *__restrict__ cells, int ncells, const unsigned long long *__restrict__ count,
                                                  const unsigned long long *__restrict__ sums, const uint8_t *__restrict__ label,
                                                  const uint32_t *__restrict__ coords, int n, unsigned long long *__restrict__ acc)
{
    __shared__ unsigned long long sa[PQ_MAX_COLOURS * 5];
    __shared__ uint32_t sc[PQ_MAX_COLOURS];
    for (int i = threadIdx.x; i < PQ_MAX_COLOURS * 5; i += blockDim.x) sa[i] = 0;
    if (coords) for (int i = threadIdx.x; i < n; i += blockDim.x) sc[i] = coords[i];
    __syncthreads();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ncells; i += gridDim.x * blockDim.x) {
        const uint32_t cell = cells[i];
        int v[4]; unsigned long long cn; pq_rep(count, sums, cell, v, cn);
        const int e = coords ? pq_nearest(v, sc, n) : label[i];
        unsigned long long *a = sa + 5 * e;
        atomicAdd(&a[0], cn);
#pragma unroll
        for (int c = 0; c < 4; c++) atomicAdd(&a[1 + c], sums[4 * (size_t)cell + c]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < PQ_MAX_COLOURS * 5; i += blockDim.x) if (sa[i]) atomicAdd(&acc[i], sa[i]);
}

// exact nearest-entry candidates of one grid cell (16 values per channel): every entry whose least distance to the cell is at most
// the smallest greatest distance of any entry, in index order.  A scan of the list in order with strict < is the exhaustive search.
__global__ void __launch_bounds__(256) k_pq_cands(const uint32_t *__restrict__ coords, int n, uint8_t *__restrict__ cand, uint16_t *__restrict__ ncand)
{
    __shared__ int sh_min[8], sh_cnt[8];
    const uint32_t cell = blockIdx.x;
    const int k = threadIdx.x, lane = k & 31, warp = k >> 5;
    int dmin = INT_MAX, dmax = INT_MAX;
    if (k < n) {
        dmin = dmax = 0;
        const uint32_t e = coords[k];
#pragma unroll
        for (int c = 0; c < 4; c++) {
            const int v = (int)((e >> (8 * c)) & 255), lo = (int)((cell >> (12 - 4 * c)) & 15) * 16, hi = lo + 15;
            const int d = v < lo ? lo - v : v > hi ? v - hi : 0;
            const int m = max(abs(v - lo), abs(v - hi));
            dmin += d * d; dmax += m * m;
        }
    }
    const int wmin = __reduce_min_sync(0xFFFFFFFFu, dmax);
    if (lane == 0) sh_min[warp] = wmin;
    __syncthreads();
    int D = sh_min[0];
    for (int i = 1; i < 8; i++) D = min(D, sh_min[i]);
    const bool take = k < n && dmin <= D;
    const unsigned bal = __ballot_sync(0xFFFFFFFFu, take);
    if (lane == 0) sh_cnt[warp] = __popc(bal);
    __syncthreads();
    int off = 0, tot = 0;
    for (int i = 0; i < 8; i++) { if (i < warp) off += sh_cnt[i]; tot += sh_cnt[i]; }
    if (take) cand[(size_t)cell * 256 + off + __popc(bal & ((1u << lane) - 1))] = (uint8_t)k;
    if (k == 0) ncand[cell] = (uint16_t)tot;
}

__device__ __forceinline__ int pq_err(unsigned long long e, int c) { return (int)(int16_t)(e >> (16 * c)); }

// Floyd-Steinberg as a wavefront (the k_png_unfilter pattern): one warp owns 32 consecutive rows, lane l works on row 32 g + l and at
// step t on pixel t - 2 l, two pixels behind the lane above -- what it needs from the row above (errors at x + 1, x, x - 1) are
// that lane's results of the previous three steps and arrive by shuffle.  Lane 0 reads the previous group's last row from HBM
// behind that group's progress counter; groups are handed out by an atomic ticket, so a waiting warp only waits for a running one.
__global__ void __launch_bounds__(32) k_pq_dither(const uint32_t *__restrict__ rgba, int w, int h, const uint32_t *__restrict__ coords, int n,
                                                  const uint8_t *__restrict__ cand, const uint16_t *__restrict__ ncand, int off,
                                                  uint8_t *__restrict__ idx, unsigned long long *edge, uint32_t *__restrict__ ticket,
                                                  volatile uint32_t *__restrict__ progress)
{
    __shared__ uint32_t sc[PQ_MAX_COLOURS];
    __shared__ unsigned long long ring[64];
    const int lane = threadIdx.x;
    for (int k = lane; k < n; k += 32) sc[k] = coords[k];
    int g = 0;
    if (lane == 0) g = (int)atomicAdd(ticket, 1u);
    g = __shfl_sync(0xFFFFFFFFu, g, 0);
    __syncwarp();
    const int y = g * 32 + lane;
    const bool live = y < h;
    const unsigned long long *above = g > 0 ? edge + (size_t)(g - 1) * w : nullptr;
    unsigned long long *mine = edge + (size_t)g * w;
    unsigned long long r1 = 0, r2 = 0, r3 = 0;         // this row's errors of the previous three steps (four int16 each)
    const int steps = w + 62;
    for (int t = 0; t < steps; t++) {
        if (above && (t & 31) == 0 && t < w) {
            const uint32_t need = (uint32_t)min(t + 33, w);
            if (lane == 0) { while (progress[g - 1] < need) __nanosleep(100); }
            __syncwarp();
            __threadfence();
            const int px = t + 1 + lane;
            if (px < w) ring[px & 63] = __ldcg(above + px);
            if (t == 0 && lane == 0) ring[0] = __ldcg(above);
            __syncwarp();
        }
        const int x = t - 2 * lane;
        unsigned long long ur = __shfl_up_sync(0xFFFFFFFFu, r1, 1), uu = __shfl_up_sync(0xFFFFFFFFu, r2, 1), ul = __shfl_up_sync(0xFFFFFFFFu, r3, 1);
        if (lane == 0) {
            ur = uu = ul = 0;
            if (above && x < w) {
                if (x + 1 < w) ur = ring[(x + 1) & 63];
                uu = ring[x & 63];
                if (x >= 1) ul = ring[(x - 1) & 63];
            }
        }
        unsigned long long e = 0;
        if (live && x >= 0 && x < w) {
            int p[4]; pq_premul(rgba[(size_t)y * w + x], p);
            int k = 0;
            if (p[3] != 0) {
                int tt[4];
#pragma unroll
                for (int c = 0; c < 4; c++)
                    tt[c] = pq_clamp255(p[c] + pq_fs_round(7 * pq_err(r1, c) + 3 * pq_err(ur, c) + 5 * pq_err(uu, c) + pq_err(ul, c)));
                const uint32_t cell = pq_grid(tt);
                const int m = ncand[cell];
                const uint32_t *cl = reinterpret_cast<const uint32_t *>(cand + (size_t)cell * 256);
                int bd = INT_MAX;
                for (int j = 0; j < m; j += 4) {
                    const uint32_t wd = __ldg(cl + (j >> 2));
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        if (j + q >= m) break;
                        const int kk = (int)((wd >> (8 * q)) & 255);
                        const int d = pq_dist(tt, sc[kk]);
                        if (d < bd) { bd = d; k = kk; }
                    }
                }
                const uint32_t ck = sc[k];
#pragma unroll
                for (int c = 0; c < 4; c++) e |= (unsigned long long)(uint16_t)(int16_t)(tt[c] - (int)((ck >> (8 * c)) & 255)) << (16 * c);
            }
            idx[(size_t)y * w + x] = (uint8_t)(p[3] ? off + k : 0);        // fully transparent: the reserved entry 0
            if (lane == 31) {
                mine[x] = e;
                if ((x & 31) == 31 || x == w - 1) { __threadfence(); progress[g] = (uint32_t)(x + 1); }
            }
        }
        r3 = r2; r2 = r1; r1 = e;
    }
}

// exact path: the index of every pixel in the sorted palette keys
__global__ void k_pq_exact(const uint32_t *__restrict__ rgba, size_t npix, const unsigned long long *__restrict__ keys, int n, uint8_t *__restrict__ idx)
{
    __shared__ unsigned long long sk[256];
    for (int i = threadIdx.x; i < n; i += blockDim.x) sk[i] = keys[i];
    __syncthreads();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (size_t)gridDim.x * blockDim.x) {
        const unsigned long long key = pq_exact_key(rgba[i]);
        int lo = 0, hi = n - 1;
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (sk[mid] < key) lo = mid + 1; else hi = mid; }
        idx[i] = (uint8_t)lo;
    }
}

// indices -> PNG rows of `depth`-bit samples, MSB first, one thread per output byte
__global__ void k_pq_pack(const uint8_t *__restrict__ idx, int w, int h, int depth, size_t rb, uint8_t *__restrict__ dst)
{
    const size_t nb = rb * h;
    const int per = 8 / depth;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nb; i += (size_t)gridDim.x * blockDim.x) {
        const int y = (int)(i / rb), xb = (int)(i % rb);
        const uint8_t *src = idx + (size_t)y * w;
        uint32_t v = 0;
        for (int q = 0; q < per; q++) {
            const int x = xb * per + q;
            if (x < w) v |= (uint32_t)src[x] << (8 - depth - q * depth);
        }
        dst[i] = (uint8_t)v;
    }
}

static unsigned grid_for(size_t n, int threads) { return (unsigned)std::max<size_t>(1, std::min<size_t>((n + threads - 1) / threads, 132 * 16)); }

// ---- host driver -----------------------------------------------------------------------------------------------------------------
bool PngQuant::load_host(const uint8_t *rgba, int width, int height, void *stream, std::string &err)
{
    w = width; h = height;
    const size_t n = (size_t)w * h * 4;
    if (!grow(d_rgba, n + 64, err)) return false;
    CU(cudaMemcpyAsync(d_rgba, rgba, n, cudaMemcpyHostToDevice, (cudaStream_t)stream));
    return true;
}

uint32_t *PngQuant::rgba_for(int width, int height, std::string &err)
{
    w = width; h = height;
    return grow(d_rgba, (size_t)w * h * 4 + 64, err) ? d_rgba.get() : nullptr;
}

bool PngQuant::load_planes(const uint8_t *planes, int nc, const uint8_t *alpha, int width, int height, void *stream, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream;
    w = width; h = height;
    const size_t n = (size_t)w * h;
    if (!grow(d_rgba, n * 4 + 64, err) || !grow(d_planes, n * (nc + 1) + 64, err)) return false;
    CU(cudaMemcpyAsync(d_planes, planes, n * nc, cudaMemcpyHostToDevice, st));
    if (alpha) CU(cudaMemcpyAsync(d_planes + n * nc, alpha, n, cudaMemcpyHostToDevice, st));
    k_pq_planes<<<grid_for(n, 256), 256, 0, st>>>(d_planes, n, nc, alpha ? 1 : 0, d_rgba);
    KCHECK("k_pq_planes");
    return true;
}

bool PngQuant::expand(const uint8_t *d_raw, const PngInfo &info, void *stream_, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    w = (int)info.width; h = (int)info.height;
    const size_t npix = (size_t)w * h;
    if (!grow(d_rgba, npix * 4 + 64, err)) return false;
    if (!fixed(d_lut, 256 * 4, err) || !fixed(h_small, kSmall, err)) return false;
    int has_key = 0, key[3] = {0, 0, 0};
    const int ct = info.color_type;
    if (ct == 3) {
        uint32_t *lut = reinterpret_cast<uint32_t *>(h_small.get());
        for (int i = 0; i < 256; i++) {
            uint32_t r = 0, g = 0, b = 0;
            if ((size_t)(3 * i + 2) < info.plte.size()) { r = info.plte[3 * i]; g = info.plte[3 * i + 1]; b = info.plte[3 * i + 2]; }
            const uint32_t a = (size_t)i < info.trns.size() ? info.trns[i] : 255;
            lut[i] = r | g << 8 | b << 16 | a << 24;
        }
        CU(cudaMemcpyAsync(d_lut, lut, 1024, cudaMemcpyHostToDevice, st));
    } else if (ct == 0 && info.trns.size() >= 2) { has_key = 1; key[0] = info.trns[0] << 8 | info.trns[1]; }
    else if (ct == 2 && info.trns.size() >= 6) { has_key = 1; for (int c = 0; c < 3; c++) key[c] = info.trns[2 * c] << 8 | info.trns[2 * c + 1]; }
    k_pq_expand<<<grid_for(npix, 256), 256, 0, st>>>(d_raw, info.row_bytes, w, h, ct, info.bit_depth, d_lut, has_key, key[0], key[1], key[2], d_rgba);
    KCHECK("k_pq_expand");
    if (ct == 3) CU(stream_wait(st));          // the lut staging buffer is reused by the next readback
    return true;
}

bool PngQuant::prepare(void *stream_, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const size_t npix = (size_t)w * h;
    if (!fixed(d_count, (size_t)PQ_NCELLS * 8, err) || !fixed(d_sums, (size_t)PQ_NCELLS * 32, err) || !fixed(d_cells, (size_t)PQ_NCELLS * 4 + 64, err) ||
        !fixed(d_label, PQ_NCELLS, err) || !fixed(d_box, 2 * PQ_BOX_WORDS * 8, err) || !fixed(d_acc, PQ_MAX_COLOURS * 5 * 8, err) ||
        !fixed(d_coords, PQ_MAX_COLOURS * 4, err) || !fixed(d_keys, 256 * 8, err) || !fixed(d_set, 2048 * 4, err) || !fixed(d_flags, 64, err) ||
        !fixed(d_cand, (size_t)PQ_GRID * 256, err) || !fixed(d_ncand, (size_t)PQ_GRID * 2, err) || !fixed(h_small, kSmall, err)) return false;
    size_t tb = 0;
    cub::DeviceSelect::If(nullptr, tb, thrust::counting_iterator<uint32_t>(0), d_cells.get(), d_flags.get(), PQ_NCELLS, PqOccupied{d_count}, st);
    if (!grow(d_temp, tb + 256, err) || !grow(d_idx, npix + 64, err)) return false;
    CU(cudaMemsetAsync(d_count, 0, (size_t)PQ_NCELLS * 8, st));
    CU(cudaMemsetAsync(d_sums, 0, (size_t)PQ_NCELLS * 32, st));
    CU(cudaMemsetAsync(d_flags, 0, 64, st));
    k_pq_hist<<<grid_for(npix, 256), 256, 0, st>>>(d_rgba, npix, d_count, d_sums, d_flags + 8);
    KCHECK("k_pq_hist");
    tb = d_temp.capacity();
    cudaError_t e = cub::DeviceSelect::If(d_temp, tb, thrust::counting_iterator<uint32_t>(0), d_cells.get(), d_flags.get(), PQ_NCELLS, PqOccupied{d_count}, st);
    if (e != cudaSuccess) { err = std::string("cub select: ") + cudaGetErrorString(e); return false; }
    LT_MARK("cub_select");
    // the distinct-value probe of the lossless leg over the RGBA samples (flags[2], saturating above 256)
    if (launch_png_colours(reinterpret_cast<const uint8_t *>(d_rgba.get()), npix, 4, d_set, d_flags + 4, st)) { err = "png colours launch failed"; return false; }
    CU(cudaMemcpyAsync(h_small, d_flags, 48, cudaMemcpyDeviceToHost, st));
    CU(stream_wait(st)); LT_MARK("host_wait");
    const uint32_t *f = reinterpret_cast<const uint32_t *>(h_small.get());
    ncells = (int)f[0]; distinct = (int)f[6]; clear = (int)f[8];
    last_cut_ms = 0;
    return true;
}

namespace {
struct SplitCtx { PngQuant *q; cudaStream_t st; std::string *err; };
int split_cb(void *ctx_, int b, int axis, int t, int k, PqBox *sb, PqBox *sk)
{
    SplitCtx *c = static_cast<SplitCtx *>(ctx_);
    PngQuant *q = c->q;
    if (cudaMemsetAsync(q->d_box, 0, 2 * PQ_BOX_WORDS * 8, c->st) != cudaSuccess) { *c->err = "memset failed"; return 1; }
    k_pq_split<<<grid_for((size_t)q->ncells, 256), 256, 0, c->st>>>(q->d_cells, q->ncells, q->d_count, q->d_sums, q->d_label, b, axis, t, k, q->d_box);
    LT_MARK("k_pq_split");
    if (cudaMemcpyAsync(q->h_small, q->d_box, 2 * PQ_BOX_WORDS * 8, cudaMemcpyDeviceToHost, c->st) != cudaSuccess || stream_wait(c->st) != cudaSuccess) {
        *c->err = std::string("median cut: ") + cudaGetErrorString(cudaGetLastError()); return 1;
    }
    LT_MARK("host_wait");
    memcpy(sb, q->h_small, sizeof(PqBox));
    if (sk) memcpy(sk, q->h_small + sizeof(PqBox), sizeof(PqBox));
    return 0;
}
} // namespace

bool PngQuant::quantize(int quality, void *stream_, std::vector<uint32_t> &palette, std::string &err, bool allow_exact)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const size_t npix = (size_t)w * h;
    palette.clear();
    if (allow_exact && exact()) {
        // the distinct values from the probe's set (keys 1 << 32 | value), sorted by pq_exact_key
        CU(cudaMemcpyAsync(h_small, d_set, 1024 * 8, cudaMemcpyDeviceToHost, st));
        CU(stream_wait(st)); LT_MARK("host_wait");
        const unsigned long long *set = reinterpret_cast<const unsigned long long *>(h_small.get());
        std::vector<unsigned long long> keys;
        for (int i = 0; i < 1024; i++) if (set[i]) keys.push_back(pq_exact_key((uint32_t)set[i]));
        std::sort(keys.begin(), keys.end());
        for (unsigned long long k : keys) palette.push_back((uint32_t)k);
        CU(cudaMemcpyAsync(d_keys, keys.data(), keys.size() * 8, cudaMemcpyHostToDevice, st));
        k_pq_exact<<<grid_for(npix, 256), 256, 0, st>>>(d_rgba, npix, d_keys, (int)keys.size(), d_idx);
        KCHECK("k_pq_exact");
        return true;
    }
    if (!ncells) {              // every pixel fully transparent: the reserved entry alone
        palette.assign(1, 0u);
        CU(cudaMemsetAsync(d_idx, 0, npix, st));
        return true;
    }
    const auto t0 = std::chrono::steady_clock::now();
    CU(cudaMemsetAsync(d_label, 0, (size_t)ncells, st));
    SplitCtx ctx{this, st, &err};
    std::vector<PqBox> boxes(PQ_MAX_COLOURS);
    const int nb = pq_median_cut(&ctx, split_cb, quality, PQ_MAX_COLOURS - clear, boxes.data());
    if (nb < 0) return false;
    last_cut_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    // box means, then the refinement passes
    uint32_t ent[PQ_MAX_COLOURS], coords[PQ_MAX_COLOURS];
    unsigned long long *acc = reinterpret_cast<unsigned long long *>(h_small.get());
    int n = nb;
    for (int pass = 0; pass <= PQ_REFINE_PASSES; pass++) {
        if (pass) {
            for (int k = 0; k < n; k++) coords[k] = pq_entry_coords(ent[k]);
            CU(cudaMemcpyAsync(d_coords, coords, (size_t)n * 4, cudaMemcpyHostToDevice, st));
        }
        CU(cudaMemsetAsync(d_acc, 0, PQ_MAX_COLOURS * 5 * 8, st));
        k_pq_accum<<<grid_for((size_t)ncells, 256), 256, 0, st>>>(d_cells, ncells, d_count, d_sums, d_label, pass ? d_coords.get() : nullptr, n, d_acc);
        KCHECK(pass ? "k_pq_refine" : "k_pq_box_means");
        CU(cudaMemcpyAsync(acc, d_acc, (size_t)n * 5 * 8, cudaMemcpyDeviceToHost, st));
        CU(stream_wait(st)); LT_MARK("host_wait");
        n = pq_entries_from_sums(acc, n, ent);
    }
    pq_order(ent, n);
    // palette: the reserved transparent entry, then the quantised entries (d_coords holds only those)
    for (int k = 0; k < n; k++) coords[k] = pq_entry_coords(ent[k]);
    palette.assign((size_t)clear, 0u);
    palette.insert(palette.end(), ent, ent + n);
    CU(cudaMemcpyAsync(d_coords, coords, (size_t)n * 4, cudaMemcpyHostToDevice, st));
    k_pq_cands<<<PQ_GRID, 256, 0, st>>>(d_coords, n, d_cand, d_ncand);
    KCHECK("k_pq_cands");
    const int groups = (h + 31) / 32;
    if (!grow(d_edge, (size_t)groups * w * 8 + 64, err) || !grow(d_sync, (size_t)(groups + 2) * 4, err)) return false;
    CU(cudaMemsetAsync(d_sync, 0, (size_t)(groups + 2) * 4, st));
    k_pq_dither<<<groups, 32, 0, st>>>(d_rgba, w, h, d_coords, n, d_cand, d_ncand, clear, d_idx, d_edge, d_sync, d_sync + 2);
    KCHECK("k_pq_dither");
    return true;
}

bool PngQuant::fetch_indices(uint8_t *idx, void *stream, std::string &err)
{
    CU(cudaMemcpyAsync(idx, d_idx, (size_t)w * h, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    CU(stream_wait((cudaStream_t)stream));
    return true;
}

bool PngQuant::fetch_rgba(std::vector<uint8_t> &rgba, void *stream, std::string &err)
{
    rgba.resize((size_t)w * h * 4);
    CU(cudaMemcpyAsync(rgba.data(), d_rgba, rgba.size(), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    CU(stream_wait((cudaStream_t)stream));
    return true;
}

bool PngQuant::pack(uint8_t *d_dst, int depth, void *stream, std::string &err)
{
    const size_t rb = ((size_t)w * depth + 7) / 8;
    k_pq_pack<<<grid_for(rb * h, 256), 256, 0, (cudaStream_t)stream>>>(d_idx, w, h, depth, rb, d_dst);
    KCHECK("k_pq_pack");
    return true;
}

} // namespace b200
