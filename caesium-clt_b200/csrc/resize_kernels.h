// resize_kernels.h -- launchers for K3 (Lanczos3) and the colour conversions, plus the host-side weight tables.
#pragma once
#include <cstdint>
#include <cstddef>
#include <vector>

namespace b200 {

// Tap windows + normalised f32 weights for one axis (image 0.25.9 imageops/sample.rs horizontal_sample/vertical_sample).
struct ResizeAxis {
    int in_size = 0, out_size = 0, cap = 0;        // cap = row pitch of `weights`
    std::vector<int> left, count;
    std::vector<float> weights;                     // [out_size][cap]
};
void make_resize_axis(int in_size, int out_size, ResizeAxis &ax);
// libcaesium resize.rs compute_dimensions
void compute_resize_dimensions(uint32_t ow, uint32_t oh, uint32_t dw, uint32_t dh, uint32_t &nw, uint32_t &nh);

int launch_resize_v(const uint8_t *in, int w, int h, int stride, float *out, int nh, const int *left, const int *count, const float *weights, int cap, void *stream);
int launch_resize_h(const float *in, int w, uint8_t *out, int nw, int nh, int ostride, const int *left, const int *count, const float *weights, int cap, void *stream);
// the same passes over `planes` planes in one launch each (plane k at in + k * in_pitch / out + k * out_pitch, in samples);
// T = uint8_t or uint16_t (clamped to [0, 255] or [0, 65535] before rounding)
template <class T>
int launch_resize_v_planes(const T *in, int w, int h, int stride, size_t in_pitch, float *out, int nh, size_t out_pitch, int planes,
                           const int *left, const int *count, const float *weights, int cap, void *stream);
template <class T>
int launch_resize_h_planes(const float *in, int w, size_t in_pitch, T *out, int nw, int nh, int ostride, size_t out_pitch, int planes,
                           const int *left, const int *count, const float *weights, int cap, void *stream);
int launch_ycc_to_rgb(uint8_t *p0, uint8_t *p1, uint8_t *p2, size_t n, void *stream);
int launch_rgb_to_ycc(uint8_t *p0, uint8_t *p1, uint8_t *p2, size_t n, void *stream);

} // namespace b200
