// jpeg_kernels.h -- device work descriptors and launchers for the JPEG transform kernels
// (K1 dequant+IDCT, K2 chroma upsample, K4 downsample, K5 FDCT+quantise+zigzag and their fusions;
// SURVEY.md §8a row a6).  Plain C++ declarations so host translation units need no CUDA headers.
#pragma once
#include <cstdint>
#include <cstddef>
#include "jpeg_trellis_core.h"

namespace b200 {

// Output quantiser of one component, in ZIGZAG order.  mozjpeg's non-trellis quantize() is round-half-away-from-zero division
// by d = quantval << 3 (the ISLOW FDCT output is scaled by 8):  q = sign(x) * floor((|x| + d/2) / d).  Because d is even that is
//     q = floor((x + d/2 + (x >> 31)) / d)                      (one formula for both signs; x >> 31 = -1 for x < 0)
// and with a bias B*d that makes the dividend non-negative for every x >= -32768 (B = ceil(32769 / d)):
//     q + B = floor(y / d),  y = x + (x >> 31) + c,  c = d/2 + B*d,  0 <= y < 2^20
// floor(y / d) = umulhi(y, m) >> sh with m = ceil(2^s / d) << (32 - min(s, 32)), sh = max(s - 32, 0), s = 20 + ceil(log2 d):
// exact for y < 2^20 (e = m'*d - 2^s < d <= 2^(s-20), so y*e < 2^s).  No abs, no sign select.  The bias comes off when two
// results are packed into one 32-bit word:  word = ((q_even + B_even) + ((q_odd + B_odd) << 16) + kpair) ^ 0x8000 with
// kpair = 0x8000 - B_even - (B_odd << 16): the 0x8000 keeps the low half from borrowing, the XOR takes it out again.
struct QuantDev {
    uint32_t m[64];
    uint32_t c[64];
    uint32_t kpair[32];
    uint8_t sh[64];
    uint32_t any_shift;     // some sh != 0 (quantval > 512): the kernels then take the variant that applies sh
};

#if defined(__CUDACC__)
#define B200_HD __host__ __device__ __forceinline__
#else
#define B200_HD inline
#endif
// the integer sequence the kernels execute for one coefficient (biased result) -- shared with the CPU check in tests/emul
B200_HD uint32_t quant_biased(int x, uint32_t m, uint32_t c, uint32_t sh)
{
    const uint32_t y = (uint32_t)(x + (x >> 31)) + c;
#if defined(__CUDA_ARCH__)
    return __umulhi(y, m) >> sh;
#else
    return (uint32_t)(((unsigned long long)y * m) >> 32) >> sh;
#endif
}
B200_HD uint32_t quant_pack(uint32_t qb_even, uint32_t qb_odd, uint32_t kpair) { return (qb_even + (qb_odd << 16) + kpair) ^ 0x8000u; }

inline void make_quant_dev(const uint16_t qt_zigzag[64], QuantDev *out)
{
    uint32_t B[64];
    out->any_shift = 0;
    for (int k = 0; k < 64; k++) {
        uint32_t d = (uint32_t)qt_zigzag[k] << 3;       // jcdctmgr.c: ISLOW divisor = quantval << 3
        if (d == 0) d = 8;
        int l = 0; while ((1u << l) < d) l++;            // ceil(log2 d)
        const int s = 20 + l;
        const unsigned long long mfull = ((1ull << s) + d - 1) / d;      // ceil(2^s / d) < 2^21
        if (s <= 32) { out->m[k] = (uint32_t)(mfull << (32 - s)); out->sh[k] = 0; }
        else         { out->m[k] = (uint32_t)mfull; out->sh[k] = (uint8_t)(s - 32); out->any_shift = 1; }
        B[k] = (32769u + d - 1) / d;
        out->c[k] = (d >> 1) + B[k] * d;
    }
    for (int j = 0; j < 32; j++) out->kpair[j] = 0x8000u - B[2 * j] - (B[2 * j + 1] << 16);
}

// One unit of device work: one component of one image.
struct CompWork {
    const int16_t *cin;     // input coefficients  [bh_in*bw_in][64] zigzag, quantised
    int16_t *cout;          // output coefficients [bh_out*bw_out][64] zigzag
    uint8_t *plane;         // component-resolution samples, (bh_in*8) rows x pstride
    uint8_t *full;          // full-resolution plane W x H (generic path only), stride = fstride
    uint8_t *dplane;        // downsampled padded plane (rbh_out*8) x (rbw_out*8) (generic path only)
    const uint16_t *dq;     // 64 dequantisation multipliers, zigzag order
    const QuantDev *q;      // output quantiser
    int32_t bw_in, bh_in;   // allocated blocks of the input component
    int32_t rbw_in, rbh_in; // real blocks of the input component
    int32_t cw, ch;         // real sample dims of the input component
    int32_t bw_out, bh_out, rbw_out, rbh_out;
    int32_t W, H;           // image dims
    int32_t pstride, fstride;
    int32_t up_hx, up_vx;   // decoder upsampling ratio  (hmax/hs, vmax/vs of the input)
    int32_t dn_hx, dn_vx;   // encoder downsampling ratio (hmax/hs, vmax/vs of the output)
    // dc_sum != null: the input blocks hold their DC DIFFERENCE (GpuDecoder::Item::defer_dc); the DC of block (bx, by) is
    // dc_sum[slot] - (dc_prev ? *dc_prev : 0), slot as GpuDecoder::DcSums says
    const int32_t *dc_sum, *dc_prev;
    int32_t dc_hs, dc_vs, dc_mcux;
};

inline int work_tiles(int rbw, int rbh) { return ((rbw + 31) / 32) * rbh; }   // row-aligned tiles of 32 blocks

// Launchers.  `work` is a DEVICE array of n descriptors; max_tiles = max over the n items of
// work_tiles(real blocks across, down) for the grid the kernel iterates (sizes grid.x).  All asynchronous on `stream` (cudaStream_t).
// Return cudaError_t as int.
// raw = true: the FDCT kernels store the unquantised zigzag DCT output instead, for launch_jpeg_trellis to quantise.
int launch_fused_same(const CompWork *work, int n, int max_tiles, void *stream, bool raw = false);       // IDCT -> FDCT+quant, same geometry
int launch_idct_plane(const CompWork *work, int n, int max_tiles, void *stream);       // IDCT -> u8 plane
int launch_chroma420_refdct(const CompWork *work, int n, int max_tiles, void *stream, bool raw = false); // h2v2 fancy up o h2v2 box down o FDCT+quant
int launch_upsample(const CompWork *work, int n, int max_w, int max_h, void *stream);   // plane -> full
int launch_downsample(const CompWork *work, int n, int max_w, int max_h, void *stream); // full -> dplane
int launch_fdct_plane(const CompWork *work, int n, int max_tiles, void *stream, bool raw = false);       // dplane -> coefficients
// trellis quantisation in place of the raw coefficients of the real blocks of n items (max_blocks = max rbw_out * rbh_out);
// item i uses tables[w.q - qbase], the JtTable beside its QuantDev
int launch_jpeg_trellis(const CompWork *work, int n, int max_blocks, const QuantDev *qbase, const JtTable *tables, void *stream);
int launch_memset_warm(void *p, size_t n, void *stream);

} // namespace b200
