// dev_bits.h -- LSB-first bit writing on the device for the entropy coders whose pieces are placed by a prefix sum of their bit
// lengths (png_deflate.cu's DEFLATE blocks, vp8l_kernels.cu's VP8L tokens): every writer starts at its own bit position in zeroed
// 32-bit words and shares the first and last word with its neighbours, so every flush is an atomic OR.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace b200 {

struct DevBits {
    uint32_t *words; unsigned long long wpos; unsigned long long acc; int n;
    __device__ __forceinline__ DevBits(uint32_t *w, unsigned long long bitpos) : words(w), wpos(bitpos >> 5), acc(0), n((int)(bitpos & 31)) {}
    __device__ __forceinline__ void put32(uint32_t v, int k)      // k <= 32, n < 32 on entry
    {
        if (!k) return;
        acc |= (unsigned long long)v << n; n += k;
        if (n >= 32) { const uint32_t w = (uint32_t)acc; if (w) atomicOr(&words[wpos], w); wpos++; acc >>= 32; n -= 32; }
    }
    __device__ __forceinline__ void put(unsigned long long v, int k)   // k <= 48
    {
        if (k > 32) { put32((uint32_t)v, 32); put32((uint32_t)(v >> 32), k - 32); } else put32((uint32_t)v, k);
    }
    __device__ __forceinline__ void finish() { if (n > 0) { const uint32_t w = (uint32_t)acc; if (w) atomicOr(&words[wpos], w); } }
};

} // namespace b200
