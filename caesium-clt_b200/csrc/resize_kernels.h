// resize_kernels.h -- the K3 (Lanczos3) resampler, the colour conversions, and the host-side weight tables.
#pragma once
#include <cstdint>
#include <cstddef>
#include <string>
#include <vector>
#include "dev_buffer.h"

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

// K3 of `planes` device planes of T (uint8_t or uint16_t, clamped to [0, 255] or [0, 65535] before rounding), in[k] of w x h
// samples, into out[k] of nw x nh, one plane at a time: the vertical pass into one f32 plane, then the horizontal pass.  At the
// same size nothing is enqueued (imageops::resize copies): the caller reads the input planes.  The buffers grow by the owner's rule.
struct Resampler {
    explicit Resampler(Grow rule) : rule(rule) {}
    template <class T>
    bool run(const T *const *in, int w, int h, T *const *out, int nw, int nh, int planes, void *stream, std::string &err);

    Grow rule;
    // Both axes' tap tables: left | count | weights of the vertical axis, then of the horizontal one.  The host rewrites h_tab for
    // every resize, so the stream must have passed the previous upload from it first: every owner waits for its stream between two
    // resizes.
    PinnedBuffer<uint8_t> h_tab; DeviceBuffer<uint8_t> d_tab;
    DeviceBuffer<float> d_tmp;                      // the vertical pass of one plane, w x nh
};

int launch_ycc_to_rgb(uint8_t *p0, uint8_t *p1, uint8_t *p2, size_t n, void *stream);
int launch_rgb_to_ycc(uint8_t *p0, uint8_t *p1, uint8_t *p2, size_t n, void *stream);

} // namespace b200
