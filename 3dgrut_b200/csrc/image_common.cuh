// 3dgrut_b200/csrc/image_common.cuh -- what the image loss (gut_loss.cu) and the image metrics (gut_metrics.cu) share: the 16x16 SSIM
// tile with its 5-pixel halo, the 11-tap Gaussian window, and how a pixel of the prediction is loaded -- composited onto the background,
// post-processed, masked -- before either of them sees it.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace gutb200 {

namespace {

constexpr int kT = 16;          // output tile
constexpr int kR = 5;           // window radius
constexpr int kS = kT + 2 * kR; // staged tile
constexpr float kC1 = 0.01f * 0.01f, kC2 = 0.03f * 0.03f;

struct Window {
    float w[11];
};

// The normalised Gaussian window of SSIM (11 taps, sigma 1.5), built in fp64 and rounded once.
inline Window gaussian_window() {
    Window win;
    double g[11], total = 0.0;
    for (int i = 0; i < 11; ++i) {
        const double x = i - 5;
        g[i] = exp(-(x * x) / (2.0 * 1.5 * 1.5));
        total += g[i];
    }
    for (int i = 0; i < 11; ++i) win.w[i] = static_cast<float>(g[i] / total);
    return win;
}

// Extra inputs and outputs of the composited loss; unread by the plain kernels.
struct Composite {
    const float* alpha;     // [H,W]: the prediction's alpha when it is not channel 3 of the prediction (PS == 3)
    const float* bg_image;  // [H,W,3] background (BG == 2)
    const float* mask;      // [H,W] (MASK)
    float* d_alpha;         // [H,W]: d loss / d alpha when the gradient has no alpha channel (GS == 3)
    double* acc;            // [2] fp64 sums of the composited kernels (the head of the scratch), copied to sums2 by loss_grad_kernel
    float* sums;            // sums2
    float bg[3];            // constant background (BG == 1)
};

constexpr float kSrgbLimit = 0.0031308f, kSrgbExp = 1.0f / 2.4f;

// linear-to-sRGB (post_processing_linear_to_srgb.py:43-67): the branch is taken on c itself, the power on max(c, 1e-8)
__device__ __forceinline__ float linear_to_srgb(float c) {
    return c > kSrgbLimit ? 1.055f * powf(fmaxf(c, 1e-8f), kSrgbExp) - 0.055f : 12.92f * c;
}

// its derivative through the branch taken (torch.where): (1.055 / 2.4) c^(1/2.4 - 1) above the limit, 12.92 below
__device__ __forceinline__ float linear_to_srgb_slope(float c) {
    return c > kSrgbLimit ? (1.055f / 2.4f) * powf(c, kSrgbExp - 1.0f) : 12.92f;
}

// x = the prediction of pixel p, channel c, composited onto the background (before any post-processing and the mask).
template <int PS, int BG>
__device__ __forceinline__ float composite(float x, const float* __restrict__ pred, const Composite& cp, int64_t p, int c) {
    if constexpr (BG != 0) {
        const float a = PS == 4 ? pred[p * 4 + 3] : cp.alpha[p];
        const float b = BG == 1 ? cp.bg[c] : cp.bg_image[p * 3 + c];
        x = x + b * (1.0f - a);
    }
    return x;
}

// x and y of pixel p, channel c, as the loss sees them: the prediction composited onto the background and post-processed (POST), both
// multiplied by the mask.
template <int PS, int BG, bool MASK, int POST = 0>
__device__ __forceinline__ void load_xy(const float* __restrict__ pred, const float* __restrict__ target, const Composite& cp, int64_t p, int c,
                                        float& x, float& y) {
    x = pred[p * PS + c];
    y = target[p * 3 + c];
    x = composite<PS, BG>(x, pred, cp, p, c);
    if constexpr (POST == 1) x = linear_to_srgb(x);
    if constexpr (MASK) {
        const float m = cp.mask[p];
        x = x * m;
        y = y * m;
    }
}

}  // namespace

}  // namespace gutb200
