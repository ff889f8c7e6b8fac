// launch_timer.h -- optional per-launch timing of a pass sequence with CUDA events on the launching stream.  bench.py's
// per-kernel roofline table comes from here: one megabatch is run alone on one stream with an event recorded after every
// launch, so the differences are the kernels' own durations (no overlap with other megabatches).  Off (a null pointer test)
// everywhere else.
#pragma once
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <string>
#include <vector>

namespace b200 {

struct LaunchTimer {
    struct Mark { const char *name; cudaEvent_t ev; };
    std::vector<Mark> marks;
    cudaStream_t st = nullptr;
    void begin(cudaStream_t s) { st = s; mark("begin"); }
    void mark(const char *name) { cudaEvent_t e; if (cudaEventCreate(&e) != cudaSuccess) return; cudaEventRecord(e, st); marks.push_back({name, e}); }
    // after the stream has been waited for: add each interval to acc[name] = (total ms, launches)
    void collect(std::map<std::string, std::pair<double, int>> &acc)
    {
        for (size_t i = 1; i < marks.size(); i++) {
            float ms = 0; if (cudaEventElapsedTime(&ms, marks[i - 1].ev, marks[i].ev) != cudaSuccess) continue;
            auto &a = acc[marks[i].name]; a.first += ms; a.second++;
        }
        for (auto &m : marks) cudaEventDestroy(m.ev);
        marks.clear();
    }
};
extern thread_local LaunchTimer *tl_launch_timer;
#define LT_MARK(name) do { if (::b200::tl_launch_timer) ::b200::tl_launch_timer->mark(name); } while (0)

// B200_TRACE's level, read once (unset: 0).  At 2 and above the legs print one line per call with their stage and kernel times.
inline int trace_level()
{
    static const int level = [] { const char *e = getenv("B200_TRACE"); return e ? atoi(e) : 0; }();
    return level;
}

// A LaunchTimer on `stream`, installed as this thread's tl_launch_timer while `on`.  The pointer is cleared when the scope ends,
// however it ends, so that no later LT_MARK writes through a timer that is gone.
struct LaunchTrace {
    LaunchTimer lt;
    LaunchTrace(void *stream, bool on) { if (on) { lt.begin((cudaStream_t)stream); tl_launch_timer = &lt; } }
    ~LaunchTrace() { tl_launch_timer = nullptr; }
    LaunchTrace(const LaunchTrace &) = delete;
    LaunchTrace &operator=(const LaunchTrace &) = delete;
    // after the stream has been waited for: " name=ms" per kernel name, in name order
    std::string kernel_ms()
    {
        std::map<std::string, std::pair<double, int>> acc;
        lt.collect(acc);
        std::string s;
        for (auto &kv : acc) { char b[96]; snprintf(b, sizeof b, " %s=%.4f", kv.first.c_str(), kv.second.first); s += b; }
        return s;
    }
};

} // namespace b200
