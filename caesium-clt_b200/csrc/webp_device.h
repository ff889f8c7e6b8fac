// webp_device.h -- per-worker device state of the WebP (lossy VP8) leg: planar RGB in HBM -> K8 -> levels/modes -> host writer.
#pragma once
#include <cstdint>
#include <cstddef>
#include <string>
#include <vector>
#include "dev_buffer.h"

namespace b200 {

// bytes this leg has copied device -> host so far, all devices (diagnostics: bench.py reports the per-step figure from it)
unsigned long long webp_d2h_bytes_total();

struct WebpDevice {
    DeviceBuffer<uint8_t> d_planes;         // Y,U,V source + RY,RU,RV reconstruction, macroblock-padded
    DeviceBuffer<uint8_t> d_rgb;            // staging for callers whose RGB starts on the host
    DeviceBuffer<int16_t> d_levels;
    DeviceBuffer<uint8_t> d_modes;
    DeviceBuffer<int> d_progress;
    PinnedBuffer<uint8_t> h_out;            // levels | modes
    PinnedBuffer<uint8_t> h_rgb;            // staging for host RGB
    DeviceBuffer<uint32_t> d_tokwork;       // mask | counts | offsets | tallies
    DeviceBuffer<uint8_t> d_toktemp;        // scan scratch
    DeviceBuffer<uint16_t> d_tokens;        // the frame's decision records
    PinnedBuffer<uint8_t> h_tokens;         // records
    double last_wait_ms = 0, last_code_ms = 0;                 // tracing: wait for the kernels + D2H, host boolean coder of the last encode
    // d_r/d_g/d_b: device planes (pitch w).  Produces the .webp file; optionally also hands back the levels/modes (tests).
    bool encode_planes(const uint8_t *d_r, const uint8_t *d_g, const uint8_t *d_b, int w, int h, int quality, void *stream,
                       std::vector<uint8_t> &out, std::string &err, int16_t *levels_out = nullptr, uint8_t *modes_out = nullptr);
    // rgb: host, planar [3][h][w]
    bool encode_host_rgb(const uint8_t *rgb, int w, int h, int quality, void *stream, std::vector<uint8_t> &out, std::string &err,
                         int16_t *levels_out = nullptr, uint8_t *modes_out = nullptr);
};

} // namespace b200
