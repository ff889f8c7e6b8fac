// png_resize.cu -- the two ends of the PNG resize leg (libcaesium png::compress_in_memory with width / height set: the image crate
// decodes with EXPAND, resize_exact(.., Lanczos3), re-encodes, then oxipng or imagequant).  Expansion turns the un-filtered rows into
// one plane per channel of the decoded type, K3 resamples the planes (resize_kernels.cu), packing writes PNG rows for the back end.
// Both are one thread per pixel, HBM-bound.
#include <cuda_runtime.h>
#include <algorithm>
#include "png_resize.h"

namespace b200 {

PngDecodedType png_decoded_type(const PngInfo &info)
{
    const int depth = info.bit_depth == 16 ? 16 : 8;
    switch (info.color_type) {
        case 0: return info.trns.size() >= 2 ? PngDecodedType{4, 2, depth} : PngDecodedType{0, 1, depth};
        case 2: return info.trns.size() >= 6 ? PngDecodedType{6, 4, depth} : PngDecodedType{2, 3, depth};
        case 3: return info.trns.empty() ? PngDecodedType{2, 3, 8} : PngDecodedType{6, 4, 8};
        case 4: return {4, 2, depth};
        default: return {6, 4, depth};
    }
}

void png_resized_info(PngInfo &info, uint32_t nw, uint32_t nh)
{
    const PngDecodedType t = png_decoded_type(info);
    info.width = nw; info.height = nh;
    info.color_type = t.color_type; info.bit_depth = t.depth; info.channels = t.channels; info.interlace = 0;
    info.bits_per_pixel = t.channels * t.depth; info.bpp = t.channels * t.depth / 8;
    info.row_bytes = (size_t)nw * info.bpp;
    info.plte.clear(); info.trns.clear();
    info.kept_before_idat.clear(); info.kept_after_idat.clear();
}

PngLut png_palette_lut(const PngInfo &info)
{
    PngLut lut;
    for (int i = 0; i < 256; i++) {
        uint32_t r = 0, g = 0, b = 0;
        if ((size_t)(3 * i + 2) < info.plte.size()) { r = info.plte[3 * i]; g = info.plte[3 * i + 1]; b = info.plte[3 * i + 2]; }
        const uint32_t a = (size_t)i < info.trns.size() ? info.trns[i] : 255;
        lut.v[i] = r | g << 8 | b << 16 | a << 24;
    }
    return lut;
}

// one sample of a row: 16 bits big-endian, 8 bits, or a sub-byte grey / index (MSB first)
__device__ __forceinline__ int png_sample(const uint8_t *row, size_t k, int bd)
{
    if (bd == 16) return row[2 * k] << 8 | row[2 * k + 1];
    if (bd == 8) return row[k];
    return (row[(k * bd) >> 3] >> (8 - bd - (int)((k * bd) & 7))) & ((1 << bd) - 1);
}

template <class T>
__global__ void k_png_expand_planes(const uint8_t *__restrict__ raw, size_t rb, int w, int h, int ct, int bd, const PngLut lut, int has_key,
                                    int k0, int k1, int k2, int och, T *__restrict__ planes)
{
    const size_t npix = (size_t)w * h;
    const T amax = sizeof(T) == 1 ? 255 : 65535;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (size_t)gridDim.x * blockDim.x) {
        const int y = (int)(i / w), x = (int)(i % w);
        const uint8_t *row = raw + (size_t)y * rb;
        if (ct == 3) {
            const uint32_t c = lut.v[png_sample(row, x, bd) & 255];
            for (int k = 0; k < och; k++) planes[k * npix + i] = (T)((c >> (8 * k)) & 255);
        } else if (ct == 0) {
            const int v = png_sample(row, x, bd);
            planes[i] = (T)(bd < 8 ? v * 255 / ((1 << bd) - 1) : v);
            if (och == 2) planes[npix + i] = has_key && v == k0 ? (T)0 : amax;
        } else {
            const int nin = ct == 2 ? 3 : ct == 4 ? 2 : 4;
            int s[4];
            for (int k = 0; k < nin; k++) { s[k] = png_sample(row, (size_t)x * nin + k, bd); planes[k * npix + i] = (T)s[k]; }
            if (ct == 2 && och == 4) planes[3 * npix + i] = has_key && s[0] == k0 && s[1] == k1 && s[2] == k2 ? (T)0 : amax;
        }
    }
}

template <class T>
__global__ void k_png_pack_planes(const T *__restrict__ planes, int ch, size_t npix, uint8_t *__restrict__ raw)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (size_t)gridDim.x * blockDim.x)
        for (int k = 0; k < ch; k++) {
            const unsigned v = planes[k * npix + i];
            if (sizeof(T) == 1) raw[i * ch + k] = (uint8_t)v;
            else { raw[2 * (i * ch + k)] = (uint8_t)(v >> 8); raw[2 * (i * ch + k) + 1] = (uint8_t)v; }
        }
}

static int grid_of(size_t n) { return (int)std::min<size_t>((n + 255) / 256, (size_t)1 << 20); }

int launch_png_expand_planes(const uint8_t *d_raw, const PngInfo &info, const PngLut &lut, void *planes, void *stream)
{
    const PngDecodedType t = png_decoded_type(info);
    const int ct = info.color_type, bd = info.bit_depth;
    int has_key = 0, key[3] = {0, 0, 0};
    if (ct == 0 && t.channels == 2) { has_key = 1; key[0] = info.trns[0] << 8 | info.trns[1]; }
    if (ct == 2 && t.channels == 4) { has_key = 1; for (int c = 0; c < 3; c++) key[c] = info.trns[2 * c] << 8 | info.trns[2 * c + 1]; }
    const size_t npix = (size_t)info.width * info.height;
    cudaStream_t st = (cudaStream_t)stream;
    if (t.depth == 16)
        k_png_expand_planes<uint16_t><<<grid_of(npix), 256, 0, st>>>(d_raw, info.row_bytes, (int)info.width, (int)info.height, ct, bd, lut, has_key,
                                                                     key[0], key[1], key[2], t.channels, static_cast<uint16_t *>(planes));
    else
        k_png_expand_planes<uint8_t><<<grid_of(npix), 256, 0, st>>>(d_raw, info.row_bytes, (int)info.width, (int)info.height, ct, bd, lut, has_key,
                                                                    key[0], key[1], key[2], t.channels, static_cast<uint8_t *>(planes));
    return (int)cudaGetLastError();
}

int launch_png_pack_planes(const void *planes, int channels, int depth, int w, int h, uint8_t *d_raw, void *stream)
{
    const size_t npix = (size_t)w * h;
    cudaStream_t st = (cudaStream_t)stream;
    if (depth == 16) k_png_pack_planes<uint16_t><<<grid_of(npix), 256, 0, st>>>(static_cast<const uint16_t *>(planes), channels, npix, d_raw);
    else k_png_pack_planes<uint8_t><<<grid_of(npix), 256, 0, st>>>(static_cast<const uint8_t *>(planes), channels, npix, d_raw);
    return (int)cudaGetLastError();
}

} // namespace b200
