// gif_device.cu -- host driver of the GIF leg (gif_device.h): canvases up, difference boxes back, crop and mask into the palette
// quantiser, segmented LZW, and only finished image data back to the host, which writes the container.
#include <cuda_runtime.h>
#include <cub/device/device_scan.cuh>
#include <algorithm>
#include <chrono>
#include <cstring>
#include "gif_device.h"
#include "gif_host.h"
#include "gif_kernels.h"
#include "png_quant.h"
#include "stream_wait.h"

namespace b200 {

namespace {
// image-sized buffers as the quantiser grows its own; the rest at their exact size
template <class B> bool grow(B &buf, size_t need, std::string &err) { return buf.reserve(need, Grow::Pow2Quarter, err); }
template <class B> bool fixed(B &buf, size_t bytes, std::string &err) { return buf.reserve(bytes, Grow::Exact, err); }

GifRect box_rect(const uint32_t *b, int w, int h) { GifRect r = {w - (int)b[0], h - (int)b[1], (int)b[2], (int)b[3]}; if (!b[2]) r = GifRect{0, 0, 0, 0}; return r; }
} // namespace

bool GifDevice::lzw(const uint8_t *d_idx, size_t n, int m, void *stream_, std::vector<uint8_t> &out, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    const int nseg = (int)std::max<size_t>(1, (n + GIF_SEG - 1) / GIF_SEG);
    const size_t words = (size_t)nseg * GIF_SEG_CODES * 12 / 32 + 2, cap = gif_blocks_size(words * 4);
    size_t tb = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tb, d_bits.get(), d_off.get(), nseg + 1, st);
    if (!grow(d_codes, (size_t)nseg * GIF_SEG_CODES * 2, err) || !grow(d_ncodes, (size_t)nseg * 4, err) || !grow(d_bits, (size_t)(nseg + 1) * 8, err) ||
        !grow(d_off, (size_t)(nseg + 1) * 8, err) || !grow(d_temp, tb + 256, err) || !grow(d_words, words * 4, err) || !grow(d_blocks, cap, err) ||
        !fixed(h_box, 64, err)) return false;
    CU(cudaMemsetAsync(d_bits, 0, (size_t)(nseg + 1) * 8, st));
    CU(cudaMemsetAsync(d_words, 0, words * 4, st));
    if (!launch_ok(launch_gif_walk(d_idx, n, m, nseg, d_codes, d_ncodes, d_bits, st), "k_gif_walk", err)) return false;
    tb = d_temp.capacity();
    CU(cub::DeviceScan::ExclusiveSum(d_temp.get(), tb, d_bits.get(), d_off.get(), nseg + 1, st));
    if (!launch_ok(launch_gif_emit(d_codes, d_ncodes, d_off, nseg, d_words, st), "k_gif_emit", err) ||
        !launch_ok(launch_gif_blocks(reinterpret_cast<const uint8_t *>(d_words.get()), d_off, nseg, cap, d_blocks, st), "k_gif_blocks", err)) return false;
    CU(cudaMemcpyAsync(h_box, d_off + nseg, 8, cudaMemcpyDeviceToHost, st));
    CU(stream_wait(st));
    unsigned long long total_bits;
    memcpy(&total_bits, h_box.get(), 8);
    const size_t size = gif_blocks_size((size_t)((total_bits + 7) / 8));
    if (!grow(h_out, size, err)) return false;
    CU(cudaMemcpyAsync(h_out, d_blocks, size, cudaMemcpyDeviceToHost, st));
    CU(stream_wait(st));
    out.insert(out.end(), h_out.get(), h_out.get() + size);
    return true;
}

bool GifDevice::code_frame(PngQuant &q, int quality, int delay, int disposal, GifRect r, void *stream, std::vector<uint8_t> &out, std::string &err)
{
    std::vector<uint32_t> pal;
    if (!q.prepare(stream, err) || !q.quantize(quality, stream, pal, err, quality == 100)) return false;
    uint8_t head[8 + 10 + 768 + 1];
    const int hn = gif_put_frame_head(head, delay, disposal, r, pal.data(), (int)pal.size());
    out.insert(out.end(), head, head + hn);
    return lzw(q.d_idx, (size_t)(r.x1 - r.x0) * (r.y1 - r.y0), gif_min_code_size((int)pal.size()), stream, out, err);
}

bool GifDevice::encode_canvas(PngQuant &q, int W, int H, int quality, void *stream, std::vector<uint8_t> &out, std::string &err)
{
    out.resize(64);
    out.resize((size_t)gif_put_header(out.data(), W, H, -1));
    if (!code_frame(q, quality, 0, 1, GifRect{0, 0, W, H}, stream, out, err)) return false;
    out.push_back(0x3B);
    return true;
}

bool GifDevice::canvas_from_planes(PngQuant &q, const uint8_t *r, const uint8_t *g, const uint8_t *b, const uint8_t *a, int W, int H, void *stream, std::string &err)
{
    uint32_t *d_rgba = q.rgba_for(W, H, err);
    return d_rgba && launch_ok(launch_gif_canvas(r, g, b, a, (size_t)W * H, d_rgba, stream), "k_gif_canvas", err);
}

bool GifDevice::canvas_from_host(PngQuant &q, const uint8_t *rgb, const uint8_t *a, int W, int H, void *stream, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream;
    const size_t n = (size_t)W * H;
    if (!grow(d_planes, 4 * n, err)) return false;
    CU(cudaMemcpyAsync(d_planes, rgb, 3 * n, cudaMemcpyHostToDevice, st));
    if (a) CU(cudaMemcpyAsync(d_planes + 3 * n, a, n, cudaMemcpyHostToDevice, st));
    return canvas_from_planes(q, d_planes, d_planes + n, d_planes + 2 * n, a ? d_planes + 3 * n : nullptr, W, H, stream, err);
}

bool GifDevice::canvas_from_rgba(PngQuant &q, void *stream, std::string &err)
{
    return launch_ok(launch_gif_canvas_rgba(q.d_rgba, (size_t)q.w * q.h, stream), "k_gif_canvas_rgba", err);
}

bool GifDevice::encode(GifReader &rd, PngQuant &q, int quality, void *stream_, std::vector<uint8_t> &out, bool &corrupt, std::string &err)
{
    cudaStream_t st = (cudaStream_t)stream_;
    corrupt = false;
    decode_ms = 0;
    const int W = rd.width, H = rd.height;
    const size_t npix = (size_t)W * H;
    for (auto &c : d_canvas) if (!grow(c, npix * 4, err)) return false;
    if (!grow(h_canvas, npix * 4, err) || !fixed(d_box, 64, err) || !fixed(h_box, 64, err)) return false;
    const GifRect whole = {0, 0, W, H}, none = {0, 0, 0, 0};
    out.resize(64);
    out.resize((size_t)gif_put_header(out.data(), W, H, rd.loop));

    // the pending frame: its canvas (slot cur), the one before it (slot prev; frame 0 has none), its delay and changed box
    int prev = -1, cur = -1, delay_pending = 0;
    GifRect changed = whole, redraw = none;
    bool first = true;
    auto write_frame = [&](GifRect clears) -> bool {
        const GifRect r = first ? whole : gif_union(gif_union(changed, clears), redraw);
        const int disposal = gif_rect_empty(clears) ? 1 : 2;
        uint32_t *d_rgba = q.rgba_for(r.x1 - r.x0, r.y1 - r.y0, err);
        if (!d_rgba) return false;
        if (!launch_ok(launch_gif_crop(first ? d_canvas[cur] : d_canvas[prev], d_canvas[cur], W, r, first ? whole : redraw, d_rgba, st), "k_gif_crop", err) ||
            !code_frame(q, quality, delay_pending, disposal, r, st, out, err)) return false;
        redraw = disposal == 2 ? r : none;
        first = false;
        return true;
    };
    for (;;) {
        int delay = 0;
        const auto t0 = std::chrono::steady_clock::now();
        const bool more = rd.next(h_canvas, delay, err);
        decode_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        if (!more) {
            if (!err.empty()) { corrupt = true; return false; }
            break;
        }
        int nx = 0;
        while (nx == prev || nx == cur) nx++;
        CU(cudaMemcpyAsync(d_canvas[nx], h_canvas, npix * 4, cudaMemcpyHostToDevice, st));
        if (cur < 0) {
            CU(stream_wait(st));           // the staging buffer takes the next frame
            cur = nx; delay_pending = delay;
            continue;
        }
        CU(cudaMemsetAsync(d_box, 0, 32, st));
        if (!launch_ok(launch_gif_diff(d_canvas[cur], d_canvas[nx], W, H, d_box, st), "k_gif_diff", err)) return false;
        CU(cudaMemcpyAsync(h_box, d_box, 32, cudaMemcpyDeviceToHost, st));
        CU(stream_wait(st));
        const GifRect d = box_rect(h_box, W, H), k = box_rect(h_box + 4, W, H);
        if (gif_rect_empty(d)) { delay_pending = std::min(delay_pending + delay, (int)GIF_MAX_DELAY); continue; }
        if (!write_frame(k)) return false;
        prev = cur; cur = nx; delay_pending = delay; changed = d;
    }
    if (!write_frame(none)) return false;
    out.push_back(0x3B);
    return true;
}

} // namespace b200
