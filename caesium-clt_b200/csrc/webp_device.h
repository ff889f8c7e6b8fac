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
// the B_PRED switch (b200_set_webp_bpred / B200_WEBP_BPRED=gpu), asked by encode_planes, which every lossy WebP leg goes through
bool webp_bpred();

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
    // d_r/d_g/d_b: device planes (pitch w).  Produces the .webp file; optionally also hands back the levels/modes/sub-block modes
    // (tests).  With the B_PRED switch on (or force_bpred) macroblocks may take 4x4 prediction; a frame whose first partition would
    // then overflow is coded 16x16-only instead.
    bool encode_planes(const uint8_t *d_r, const uint8_t *d_g, const uint8_t *d_b, int w, int h, int quality, void *stream,
                       std::vector<uint8_t> &out, std::string &err, int16_t *levels_out = nullptr, uint8_t *modes_out = nullptr,
                       uint8_t *bmodes_out = nullptr, bool force_bpred = false);
    // rgb: host, planar [3][h][w]
    bool encode_host_rgb(const uint8_t *rgb, int w, int h, int quality, void *stream, std::vector<uint8_t> &out, std::string &err,
                         int16_t *levels_out = nullptr, uint8_t *modes_out = nullptr, uint8_t *bmodes_out = nullptr, bool force_bpred = false);
private:
    // one frame with (bpred) or without 4x4 prediction; overflow: the frame failed only because its first partition is too large
    bool encode_frame(const uint8_t *d_r, const uint8_t *d_g, const uint8_t *d_b, int w, int h, int quality, void *stream, std::vector<uint8_t> &out,
                      std::string &err, int16_t *levels_out, uint8_t *modes_out, uint8_t *bmodes_out, bool bpred, bool &overflow);
};

} // namespace b200
