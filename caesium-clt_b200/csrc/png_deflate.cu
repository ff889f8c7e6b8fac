// png_deflate.cu -- DEFLATE entropy coding of the lossless PNG path ON THE DEVICE (round-1 verdict: "inflate/unfilter/Huffman on
// host dominate").  Input: the LZ77 token stream K7 left in HBM.  Output: the zlib payload (dynamic-Huffman blocks of 65,536 tokens)
// in HBM, bit-identical to what png_host.cpp's deflate_tokens() writes -- both run the block coder of dfl_core.h.
//   k_dfl_hist    per block: litlen / distance symbol counts                         (CTA per block, shared-memory histogram)
//   k_dfl_tables  per block: code lengths, canonical codes, coded header, emit tables (one thread per block builds, the warp fills)
//   k_dfl_len     per block: bits of every 256-token chunk -> chunk offsets inside the block, block size in bits
//   k_dfl_scan    block sizes -> start bit of every block, total size                 (one CTA)
//   k_dfl_emit    per block: header, tokens, end-of-block code, OR-ed LSB-first into the zeroed output words
// Reference path: caesium::compress_in_memory -> png::lossless -> oxipng (caesium-clt's src/compressor.rs:428,436-437).
#include <cuda_runtime.h>
#include <cstdint>
#include "dfl_core.h"
#include "png_deflate.h"
#include "launch_timer.h"
#include "dev_bits.h"

namespace b200 {

using namespace dfl;

constexpr int DFL_THREADS = 256;

__device__ __forceinline__ uint32_t block_count(uint32_t ntok, int block_tokens) { return (ntok + (uint32_t)block_tokens - 1) / (uint32_t)block_tokens; }

__global__ void __launch_bounds__(DFL_THREADS) k_dfl_hist(const uint32_t *__restrict__ tok, const uint32_t *__restrict__ ntok_p, int block_tokens, uint32_t *__restrict__ hist)
{
    __shared__ uint32_t h[320];
    const uint32_t ntok = *ntok_p, b = blockIdx.x;
    if (b >= block_count(ntok, block_tokens)) return;
    for (int i = threadIdx.x; i < 320; i += blockDim.x) h[i] = 0;
    __syncthreads();
    const uint32_t begin = b * (uint32_t)block_tokens, end = min(ntok, begin + (uint32_t)block_tokens);
    for (uint32_t i = begin + threadIdx.x; i < end; i += blockDim.x) {
        const uint32_t t = tok[i];
        if (t & 0x80000000u) { atomicAdd(&h[257 + len_sym((int)((t >> 16) & 0xFF) + 3)], 1u); atomicAdd(&h[288 + dist_sym((int)(t & 0xFFFF) + 1)], 1u); }
        else atomicAdd(&h[t & 0xFF], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 320; i += blockDim.x) hist[(size_t)b * 320 + i] = h[i];
}

__global__ void __launch_bounds__(32) k_dfl_tables(const uint32_t *__restrict__ hist, const uint32_t *__restrict__ ntok_p, int block_tokens, BlockTables *__restrict__ tabs, EmitTables *__restrict__ emit)
{
    __shared__ HuffScratch S;
    __shared__ BlockTables T;
    __shared__ uint32_t lf[NLIT], df[NDIST];
    const uint32_t b = blockIdx.x;
    if (b >= block_count(*ntok_p, block_tokens)) return;
    for (int i = threadIdx.x; i < NLIT; i += 32) lf[i] = hist[(size_t)b * 320 + i];
    if (threadIdx.x < NDIST) df[threadIdx.x] = hist[(size_t)b * 320 + 288 + threadIdx.x];
    if (threadIdx.x == 0) lf[256] = 1;                    // the end-of-block symbol (build_block_tables counts it too)
    __syncwarp();
    // the litlen leaves sorted by (count, symbol) with the whole warp: rank of a leaf = leaves that precede it
    __shared__ int nleaf;
    if (threadIdx.x == 0) nleaf = 0;
    __syncwarp();
    for (int i = threadIdx.x; i < NLIT; i += 32) {
        const uint32_t f = lf[i];
        if (!f) continue;
        int r = 0;
        for (int j = 0; j < NLIT; j++) { const uint32_t g = lf[j]; r += (g != 0) && (g < f || (g == f && j < i)); }
        S.order[r] = (uint16_t)i;
        atomicAdd(&nleaf, 1);
    }
    __syncwarp();
    if (threadIdx.x == 0) build_block_tables(lf, df, T, S, nleaf);
    __syncwarp();
    EmitTables &E = emit[b];
    for (int i = threadIdx.x; i < 256; i += 32) fill_emit_entry(T, E, i);
    const uint32_t *src = reinterpret_cast<const uint32_t *>(&T); uint32_t *dst = reinterpret_cast<uint32_t *>(&tabs[b]);
    for (int i = threadIdx.x; i < (int)(sizeof(BlockTables) / 4); i += 32) dst[i] = src[i];
}

// chunk c of a block = its tokens [c * per, (c + 1) * per), per = block_tokens / DFL_THREADS (block_tokens is a multiple of it)
__global__ void __launch_bounds__(DFL_THREADS) k_dfl_len(const uint32_t *__restrict__ tok, const uint32_t *__restrict__ ntok_p, int block_tokens, const BlockTables *__restrict__ tabs,
                                                          const EmitTables *__restrict__ emit, uint32_t *__restrict__ chunk_off, unsigned long long *__restrict__ block_bits)
{
    __shared__ EmitTables E;
    __shared__ uint32_t part[DFL_THREADS];
    const uint32_t ntok = *ntok_p, b = blockIdx.x;
    if (b >= block_count(ntok, block_tokens)) return;
    { const uint32_t *src = reinterpret_cast<const uint32_t *>(&emit[b]); uint32_t *dst = reinterpret_cast<uint32_t *>(&E);
      for (int i = threadIdx.x; i < (int)(sizeof(EmitTables) / 4); i += blockDim.x) dst[i] = src[i]; }
    __syncthreads();
    const uint32_t per = (uint32_t)block_tokens / DFL_THREADS;
    const uint32_t begin = b * (uint32_t)block_tokens + threadIdx.x * per, end = min(ntok, min(begin + per, (b + 1) * (uint32_t)block_tokens));
    uint32_t bits = 0;
    for (uint32_t i = begin; i < end; i++) bits += token_bits(E, tok[i]);
    part[threadIdx.x] = bits;
    __syncthreads();
    // exclusive scan of 256 values (Hillis-Steele on shared memory)
    uint32_t v = bits;
    for (int d = 1; d < DFL_THREADS; d <<= 1) {
        const uint32_t add = threadIdx.x >= (unsigned)d ? part[threadIdx.x - d] : 0u;
        __syncthreads();
        v += add; part[threadIdx.x] = v;
        __syncthreads();
    }
    const uint32_t hdr = tabs[b].header_bits;
    chunk_off[(size_t)b * DFL_THREADS + threadIdx.x] = hdr + v - bits;
    if (threadIdx.x == DFL_THREADS - 1) block_bits[b] = (unsigned long long)hdr + v + E.eob_len;
}

// start bit of every block (after the two zlib header bytes) and the total; one CTA, blocks in chunks of its size
__global__ void __launch_bounds__(1024) k_dfl_scan(const unsigned long long *__restrict__ block_bits, const uint32_t *__restrict__ ntok_p, int block_tokens,
                                                    unsigned long long *__restrict__ block_start, unsigned long long *__restrict__ total /*[0] bits incl. header, [1] = ntok*/)
{
    __shared__ unsigned long long part[1024];
    __shared__ unsigned long long carry;
    const uint32_t nb = block_count(*ntok_p, block_tokens);
    if (threadIdx.x == 0) carry = 16;
    __syncthreads();
    for (uint32_t base = 0; base < nb; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        const unsigned long long mine = i < nb ? block_bits[i] : 0ull;
        unsigned long long v = mine;
        part[threadIdx.x] = v;
        __syncthreads();
        for (int d = 1; d < 1024; d <<= 1) {
            const unsigned long long add = threadIdx.x >= (unsigned)d ? part[threadIdx.x - d] : 0ull;
            __syncthreads();
            v += add; part[threadIdx.x] = v;
            __syncthreads();
        }
        if (i < nb) block_start[i] = carry + v - mine;
        __syncthreads();
        if (threadIdx.x == 1023) carry += v;
        __syncthreads();
    }
    if (threadIdx.x == 0) { total[0] = carry; total[1] = *ntok_p; }
}

__global__ void __launch_bounds__(DFL_THREADS) k_dfl_emit(const uint32_t *__restrict__ tok, const uint32_t *__restrict__ ntok_p, int block_tokens, const BlockTables *__restrict__ tabs,
                                                           const EmitTables *__restrict__ emit, const uint32_t *__restrict__ chunk_off, const unsigned long long *__restrict__ block_bits,
                                                           const unsigned long long *__restrict__ block_start, const unsigned long long *__restrict__ total, uint32_t *__restrict__ words,
                                                           unsigned long long cap_bits)
{
    __shared__ EmitTables E;
    const uint32_t ntok = *ntok_p, b = blockIdx.x, nb = block_count(ntok, block_tokens);
    if (b >= nb || total[0] > cap_bits) return;          // does not fit the output buffer: the host codes the tokens itself
    { const uint32_t *src = reinterpret_cast<const uint32_t *>(&emit[b]); uint32_t *dst = reinterpret_cast<uint32_t *>(&E);
      for (int i = threadIdx.x; i < (int)(sizeof(EmitTables) / 4); i += blockDim.x) dst[i] = src[i]; }
    __syncthreads();
    const unsigned long long start = block_start[b];
    if (threadIdx.x == 0) {          // the block header: a few hundred bits, sequential
        DevBits w(words, start);
        auto put = [&](uint32_t v, int k) { w.put32(v, k); };
        write_block_header(tabs[b], b == nb - 1, put);
        w.finish();
    }
    const uint32_t per = (uint32_t)block_tokens / DFL_THREADS;
    const uint32_t begin = b * (uint32_t)block_tokens + threadIdx.x * per, end = min(ntok, min(begin + per, (b + 1) * (uint32_t)block_tokens));
    if (begin < end) {
        DevBits w(words, start + chunk_off[(size_t)b * DFL_THREADS + threadIdx.x]);
        for (uint32_t i = begin; i < end; i++) { uint32_t k; const unsigned long long piece = token_piece(E, tok[i], &k); w.put(piece, (int)k); }
        w.finish();
    }
    if (threadIdx.x == DFL_THREADS - 1) { DevBits w(words, start + block_bits[b] - E.eob_len); w.put32(E.eob_code, E.eob_len); w.finish(); }
}

size_t png_deflate_scratch_bytes(size_t max_tokens, int block_tokens)
{
    const size_t nb = (max_tokens + block_tokens - 1) / block_tokens + 1;
    return nb * (320 * 4 + sizeof(BlockTables) + sizeof(EmitTables) + DFL_THREADS * 4 + 8 + 8) + 4096;
}

int launch_png_deflate(const uint32_t *d_tok, const uint32_t *d_ntok, size_t max_tokens, int block_tokens, uint8_t *d_scratch, uint32_t *d_words, size_t words_cap_bytes,
                       unsigned long long *d_total, void *stream_)
{
    cudaStream_t st = (cudaStream_t)stream_;
    if (block_tokens % DFL_THREADS) return (int)cudaErrorInvalidValue;
    const size_t nb = (max_tokens + block_tokens - 1) / block_tokens + 1;
    uint8_t *p = d_scratch;
    auto take = [&](size_t bytes) { uint8_t *q = p; p += (bytes + 255) / 256 * 256; return q; };
    uint32_t *hist = (uint32_t *)take(nb * 320 * 4);
    BlockTables *tabs = (BlockTables *)take(nb * sizeof(BlockTables));
    EmitTables *emit = (EmitTables *)take(nb * sizeof(EmitTables));
    uint32_t *chunk_off = (uint32_t *)take(nb * DFL_THREADS * 4);
    unsigned long long *block_bits = (unsigned long long *)take(nb * 8), *block_start = (unsigned long long *)take(nb * 8);
    k_dfl_hist<<<(unsigned)nb, DFL_THREADS, 0, st>>>(d_tok, d_ntok, block_tokens, hist); LT_MARK("k_dfl_hist");
    k_dfl_tables<<<(unsigned)nb, 32, 0, st>>>(hist, d_ntok, block_tokens, tabs, emit); LT_MARK("k_dfl_tables");
    k_dfl_len<<<(unsigned)nb, DFL_THREADS, 0, st>>>(d_tok, d_ntok, block_tokens, tabs, emit, chunk_off, block_bits); LT_MARK("k_dfl_len");
    k_dfl_scan<<<1, 1024, 0, st>>>(block_bits, d_ntok, block_tokens, block_start, d_total); LT_MARK("k_dfl_scan");
    cudaMemsetAsync(d_words, 0, words_cap_bytes, st); LT_MARK("memset");
    k_dfl_emit<<<(unsigned)nb, DFL_THREADS, 0, st>>>(d_tok, d_ntok, block_tokens, tabs, emit, chunk_off, block_bits, block_start, d_total, d_words, (unsigned long long)words_cap_bytes * 8 - 64);
    LT_MARK("k_dfl_emit");
    return (int)cudaGetLastError();
}

} // namespace b200
