// resize_host.cpp -- host half of K3: the per-axis tap windows and normalised Lanczos3 weights of image 0.25.9
// imageops/sample.rs (reached via libcaesium resize::resize_image when CSParameters.width/height are set,
// caesium-clt's src/compressor.rs:439-443).  f32 throughout, libm sinf, no FMA contraction (Makefile passes
// -ffp-contract=off) so the tables match oracle/resize_oracle.c bit for bit.
#include "resize_kernels.h"
#include <cmath>

namespace b200 {

static float sinc_(float t) { float a = t * 3.14159265358979323846f; return t == 0.0f ? 1.0f : sinf(a) / a; }
static float lanczos3(float x) { return fabsf(x) < 3.0f ? sinc_(x) * sinc_(x / 3.0f) : 0.0f; }

void compute_resize_dimensions(uint32_t ow, uint32_t oh, uint32_t dw, uint32_t dh, uint32_t &nw, uint32_t &nh)
{
    if (dw > 0 && dh > 0) { nw = dw; nh = dh; return; }
    float n_width = (float)dw, n_height = (float)dh;
    float ratio = (float)ow / (float)oh;
    if (dh == 0) n_height = roundf(n_width / ratio);
    if (dw == 0) n_width = roundf(n_height * ratio);
    nw = (uint32_t)n_width; nh = (uint32_t)n_height;
}

void make_resize_axis(int in_size, int out_size, ResizeAxis &ax)
{
    ax.in_size = in_size; ax.out_size = out_size;
    ax.left.assign(out_size, 0); ax.count.assign(out_size, 0);
    const float ratio = (float)in_size / (float)out_size;
    const float sratio = ratio < 1.0f ? 1.0f : ratio;
    const float src_support = 3.0f * sratio;
    ax.cap = (int)(2.0f * src_support) + 4;
    ax.weights.assign((size_t)out_size * ax.cap, 0.0f);
    for (int o = 0; o < out_size; o++) {
        float inputx = ((float)o + 0.5f) * ratio;
        long l = (long)floorf(inputx - src_support);
        if (l < 0) l = 0;
        if (l > in_size - 1) l = in_size - 1;
        long r = (long)ceilf(inputx + src_support);
        if (r < l + 1) r = l + 1;
        if (r > in_size) r = in_size;
        inputx = inputx - 0.5f;
        int n = (int)(r - l);
        if (n > ax.cap) n = ax.cap;                 // cannot happen: cap >= 2*support + 4
        ax.left[o] = (int)l; ax.count[o] = n;
        float *w = ax.weights.data() + (size_t)o * ax.cap, sum = 0.0f;
        for (int i = 0; i < n; i++) { w[i] = lanczos3(((float)(l + i) - inputx) / sratio); sum += w[i]; }
        for (int i = 0; i < n; i++) w[i] /= sum;
    }
}

} // namespace b200
