// dev_buffer.h -- the one owner of device and pinned host memory in this library: a move-only buffer that grows on demand, the
// rounding rules the owners grow by, and the CUDA error checks the device modules share.
#pragma once
#include <cstddef>

namespace b200 {

// How reserve() rounds a request of `need` bytes up.  Each owner keeps the rule it was measured with: slots only grow, so the rule
// fixes a slot's device-memory footprint, and bench.py sizes its PNG leg's callers against that footprint.
enum class Grow {
    Exact,          // need: fixed-size buffers
    Slot,           // need + need / 8, rounded up to 64 KiB: the JPEG slot's coefficient, scratch and parameter buffers
    Pow2,           // the smallest power of two >= 64 KiB and >= need (WebP, VP8L)
    Pow2Quarter,    // ... >= need + need / 4 (PNG, the PNG quantiser)
    Pow2Half,       // ... >= need + need / 2 (the JPEG entropy encoder and decoder, whose sizes follow image content)
};

constexpr size_t grow_bytes(size_t need, Grow rule)
{
    if (rule == Grow::Exact) return need;
    if (rule == Grow::Slot) return (need + need / 8 + 0xFFFF) / 0x10000 * 0x10000;
    const size_t want = rule == Grow::Pow2Half ? need + need / 2 : rule == Grow::Pow2Quarter ? need + need / 4 : need;
    size_t bytes = size_t(1) << 16;
    while (bytes < want) bytes <<= 1;
    return bytes;
}

} // namespace b200

#ifndef B200_GROW_RULES_ONLY        // the CPU test of the rules above compiles without CUDA
#include <cuda_runtime.h>
#include <string>
#include <utility>

// err = "<expr>: <CUDA error>" and return false when a runtime call fails
#define CU(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) { err = std::string(#expr) + ": " + cudaGetErrorString(e_); return false; } } while (0)

namespace b200 {

// A kernel launcher's return code (a cudaError_t, 0 = launched) into err = "<what>: <CUDA error>"; false when it failed.
inline bool launch_ok(int rc, const char *what, std::string &err)
{
    if (!rc) return true;
    err = std::string(what) + ": " + cudaGetErrorString((cudaError_t)rc);
    return false;
}

enum class Mem { Device, Pinned };

// An owning buffer of T in device memory (cudaMalloc) or pinned host memory (cudaHostAlloc).  It converts to T * so that launch
// lines read as with a raw pointer; templated calls (CUB) take get().
template <class T, Mem M = Mem::Device> class Buffer {
public:
    Buffer() = default;
    Buffer(const Buffer &) = delete;
    Buffer &operator=(const Buffer &) = delete;
    Buffer(Buffer &&o) noexcept { swap(o); }
    Buffer &operator=(Buffer &&o) noexcept { Buffer(std::move(o)).swap(*this); return *this; }
    ~Buffer() { release(); }

    // Room for `need` bytes.  A buffer that large already is left as it is.  Otherwise the old memory is freed, grow_bytes(need,
    // rule) bytes are allocated and *generation, if given, is bumped: a captured CUDA graph holds the old address.  On failure the
    // buffer is empty and err says why.
    bool reserve(size_t need, Grow rule, std::string &err, unsigned long long *generation = nullptr)
    {
        if (need <= cap_) return true;
        if (generation) ++*generation;
        release();
        const size_t bytes = grow_bytes(need, rule);
        void *q = nullptr;
        const cudaError_t e = M == Mem::Pinned ? cudaHostAlloc(&q, bytes, cudaHostAllocDefault) : cudaMalloc(&q, bytes);
        if (e != cudaSuccess) { err = std::string(M == Mem::Pinned ? "cudaHostAlloc: " : "cudaMalloc: ") + cudaGetErrorString(e); return false; }
        p_ = static_cast<T *>(q); cap_ = bytes;
        return true;
    }
    T *get() const { return p_; }
    operator T *() const { return p_; }
    size_t capacity() const { return cap_; }          // bytes
    void swap(Buffer &o) noexcept { std::swap(p_, o.p_); std::swap(cap_, o.cap_); }

private:
    void release()
    {
        if (p_) { if (M == Mem::Pinned) cudaFreeHost(p_); else cudaFree(p_); }
        p_ = nullptr; cap_ = 0;
    }
    T *p_ = nullptr;
    size_t cap_ = 0;
};
template <class T> using DeviceBuffer = Buffer<T, Mem::Device>;
template <class T> using PinnedBuffer = Buffer<T, Mem::Pinned>;

} // namespace b200
#endif
