// 3dgrut_b200/csrc/gut_loss.cu -- image loss of the training step and its gradient w.r.t. the rendered image (SURVEY.md 8f row 3).
//
//     loss = lambda_l1 * mean|x - y| + lambda_ssim * (1 - SSIM(x, y))                     threedgrut/trainer.py:698-739
// l1_loss: threedgrut/model/losses.py:20-21.  ssim: losses.py:30-33 -> fused_ssim(img1, img2, padding="valid") of the third-party
// package fused-ssim @ 1272e21 (requirements_extra.txt:2; not under the reference tree): per channel, 11x11 Gaussian window (sigma 1.5,
// separable), zero padding, C1 = 0.01^2, C2 = 0.03^2, 5-pixel border cropped before the mean.  Restated from the published algorithm,
// not from that package's source.
//
// Two kernels over 16x16 pixel tiles with a 5-pixel halo staged in shared memory, separable convolutions (horizontal then vertical):
//   ssim_stats_kernel   x = prediction ([H,W,4] as the renderer writes it, channels 0..2), y = target [H,W,3]: the five windowed moments,
//                       the SSIM map, the sums for the two loss terms, and the three partial-derivative maps already multiplied by
//                       d loss / d map (stored [H,W,9])
//   loss_grad_kernel    convolves those maps and assembles d loss / d x, written as [H,W,4] with a zero alpha gradient -- directly the
//                       d_rgba argument of gutb200_backward.
// Both are templated on the pixel strides of the prediction and the gradient, so that gutb200_image_loss_rgb runs the same arithmetic on
// the 3DGRT layout (rgb [H,W,3] in, d_rgb [H,W,3] out, directly the d_rgb argument of grtb200_trace_bwd).
//
// gutb200_image_loss_composited adds the two image-side parts of the training loss (threedgrut/model/background.py:80-93,
// trainer.py:691-694) where the kernels load x and y, and their chain rule where loss_grad_kernel writes:
//     x = (rgb + bg (1 - alpha)) m,  y = target m          bg: constant colour or [H,W,3] image; m: optional [H,W] mask
//     d rgb_c = m dL/dx_c,  d alpha = -sum_c bg_c m dL/dx_c
// The background mode (BG) and the mask (MASK) are template parameters beside the strides; BG = 0 (black) with no mask is the plain loss.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/gut_b200.h"

namespace gutb200 {

namespace {

constexpr int kT = 16;          // output tile
constexpr int kR = 5;           // window radius
constexpr int kS = kT + 2 * kR; // staged tile
constexpr float kC1 = 0.01f * 0.01f, kC2 = 0.03f * 0.03f;

struct Window {
    float w[11];
};

// Extra inputs and outputs of the composited loss; unused (all null) by the plain entries.
struct Composite {
    const float* alpha;     // [H,W]: the prediction's alpha when it is not channel 3 of the prediction (PS == 3)
    const float* bg_image;  // [H,W,3] background (BG == 2)
    const float* mask;      // [H,W] (MASK)
    float* d_alpha;         // [H,W]: d loss / d alpha when the gradient has no alpha channel (GS == 3)
    double* acc;            // [2] fp64 sums of the composited kernels (the head of the scratch), copied to sums2 by loss_grad_kernel
    float* sums;            // sums2
    float bg[3];            // constant background (BG == 1)
};

// x and y of pixel p, channel c, as the loss sees them: the prediction composited onto the background, both multiplied by the mask.
template <int PS, int BG, bool MASK>
__device__ __forceinline__ void load_xy(const float* __restrict__ pred, const float* __restrict__ target, const Composite& cp, int64_t p, int c,
                                        float& x, float& y) {
    x = pred[p * PS + c];
    y = target[p * 3 + c];
    if constexpr (BG != 0) {
        const float a = PS == 4 ? pred[p * 4 + 3] : cp.alpha[p];
        const float b = BG == 1 ? cp.bg[c] : cp.bg_image[p * 3 + c];
        x = x + b * (1.0f - a);
    }
    if constexpr (MASK) {
        const float m = cp.mask[p];
        x = x * m;
        y = y * m;
    }
}

__device__ __forceinline__ float block_sum(float v, float* scratch) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    const int warp = (threadIdx.y * kT + threadIdx.x) >> 5, lane = (threadIdx.y * kT + threadIdx.x) & 31;
    if (lane == 0) scratch[warp] = v;
    __syncthreads();
    float total = 0.f;
    if (warp == 0) {
        total = lane < (kT * kT / 32) ? scratch[lane] : 0.f;
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) total += __shfl_xor_sync(0xFFFFFFFFu, total, o);
    }
    __syncthreads();
    return total;  // valid in thread (0,0)
}

// PS: floats per pixel of the prediction (4: the 3DGUT [H,W,4] image, 3: the 3DGRT rgb [H,W,3]); only the loads depend on it.
template <int PS, int BG = 0, bool MASK = false>
__global__ void __launch_bounds__(kT * kT) ssim_stats_kernel(int H, int W, const float* __restrict__ pred_rgba, const float* __restrict__ target,
                                                             Composite cp, Window win, float g_scale /* -lambda_ssim / count */,
                                                             float* __restrict__ dmaps,
                                                             float* __restrict__ sums /* [2]: sum |x-y|, sum of the valid SSIM map */) {
    __shared__ float sx[kS][kS + 1], sy[kS][kS + 1];
    __shared__ float hz[5][kS][kT + 1];
    __shared__ float scratch[8];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kT + tx;
    const int x0 = blockIdx.x * kT, y0 = blockIdx.y * kT;
    const int px = x0 + tx, py = y0 + ty;
    const bool inside = (px < W) && (py < H);
    const bool valid = inside && (px >= kR) && (py >= kR) && (px < W - kR) && (py < H - kR);
    float l1_acc = 0.f, ssim_acc = 0.f;
    for (int c = 0; c < 3; ++c) {
        for (int i = tid; i < kS * kS; i += kT * kT) {
            const int ly = i / kS, lx = i - ly * kS;
            const int gx = x0 + lx - kR, gy = y0 + ly - kR;
            const bool in = (gx >= 0) && (gy >= 0) && (gx < W) && (gy < H);
            const int64_t p = static_cast<int64_t>(gy) * W + gx;
            float xv = 0.f, yv = 0.f;
            if (in) load_xy<PS, BG, MASK>(pred_rgba, target, cp, p, c, xv, yv);
            sx[ly][lx] = xv;
            sy[ly][lx] = yv;
        }
        __syncthreads();
        // horizontal pass: kS rows x kT columns x 5 quantities
        for (int i = tid; i < kS * kT; i += kT * kT) {
            const int ly = i / kT, lx = i - ly * kT;
            float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f, a4 = 0.f;
#pragma unroll
            for (int k = 0; k < 11; ++k) {
                const float xv = sx[ly][lx + k], yv = sy[ly][lx + k], wk = win.w[k];
                a0 += wk * xv; a1 += wk * yv; a2 += wk * xv * xv; a3 += wk * yv * yv; a4 += wk * xv * yv;
            }
            hz[0][ly][lx] = a0; hz[1][ly][lx] = a1; hz[2][ly][lx] = a2; hz[3][ly][lx] = a3; hz[4][ly][lx] = a4;
        }
        __syncthreads();
        float mu1 = 0.f, mu2 = 0.f, ex2 = 0.f, ey2 = 0.f, exy = 0.f;
#pragma unroll
        for (int k = 0; k < 11; ++k) {
            const float wk = win.w[k];
            mu1 += wk * hz[0][ty + k][tx]; mu2 += wk * hz[1][ty + k][tx]; ex2 += wk * hz[2][ty + k][tx];
            ey2 += wk * hz[3][ty + k][tx]; exy += wk * hz[4][ty + k][tx];
        }
        const float s1 = ex2 - mu1 * mu1, s2 = ey2 - mu2 * mu2, s12 = exy - mu1 * mu2;
        const float a = 2.f * mu1 * mu2 + kC1, b = 2.f * s12 + kC2, cc = mu1 * mu1 + mu2 * mu2 + kC1, d = s1 + s2 + kC2;
        const float icd = 1.0f / (cc * d);
        const float map = a * b * icd;
        if (inside) {
            const float xv = sx[ty + kR][tx + kR], yv = sy[ty + kR][tx + kR];
            l1_acc += fabsf(xv - yv);
            if (valid) ssim_acc += map;
            const float g = valid ? g_scale : 0.f;
            const float dm_ds1 = -(a * b) * icd / d;
            const float dm_ds12 = 2.f * a * icd;
            const float dm_dmu1 = 2.f * mu2 * b * icd - 2.f * mu1 * a * b * icd / cc - 2.f * mu1 * dm_ds1 - mu2 * dm_ds12;
            float* o = dmaps + (static_cast<int64_t>(py) * W + px) * 9 + c * 3;
            o[0] = g * dm_dmu1; o[1] = g * dm_ds1; o[2] = g * dm_ds12;
        }
        __syncthreads();
    }
    const float l1_block = block_sum(l1_acc, scratch);
    const float ss_block = block_sum(ssim_acc, scratch);
    if (tid == 0) {
        if constexpr (BG != 0 || MASK) {  // fp64 totals: the 1e-6 bar of the means holds at 800x800 with masked (partly constant) images
            atomicAdd(cp.acc + 0, static_cast<double>(l1_block));
            atomicAdd(cp.acc + 1, static_cast<double>(ss_block));
        } else {
            atomicAdd(sums + 0, l1_block);
            atomicAdd(sums + 1, ss_block);
        }
    }
}

// GS: floats per pixel of the gradient (4: d_rgba, one 16-byte store, its alpha gradient zero unless BG != 0; 3: d_rgb, plus cp.d_alpha
// in the composited entry).
template <int PS, int GS, int BG = 0, bool MASK = false>
__global__ void __launch_bounds__(kT * kT) loss_grad_kernel(int H, int W, const float* __restrict__ pred_rgba, const float* __restrict__ target,
                                                            Composite cp, Window win, float l1_scale /* lambda_l1 / (H W 3) */,
                                                            const float* __restrict__ dmaps, float* __restrict__ d_rgba) {
    __shared__ float sm[3][kS][kS + 1];
    __shared__ float hz[3][kS][kT + 1];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kT + tx;
    const int x0 = blockIdx.x * kT, y0 = blockIdx.y * kT;
    const int px = x0 + tx, py = y0 + ty;
    const bool inside = (px < W) && (py < H);
    if constexpr (BG != 0 || MASK) {
        if (blockIdx.x == 0 && blockIdx.y == 0 && tid == 0) {  // every block of ssim_stats_kernel has finished (stream order)
            cp.sums[0] = static_cast<float>(cp.acc[0]);
            cp.sums[1] = static_cast<float>(cp.acc[1]);
        }
    }
    float grad[3] = {0.f, 0.f, 0.f};
    for (int c = 0; c < 3; ++c) {
        for (int i = tid; i < kS * kS; i += kT * kT) {
            const int ly = i / kS, lx = i - ly * kS;
            const int gx = x0 + lx - kR, gy = y0 + ly - kR;
            const bool in = (gx >= 0) && (gy >= 0) && (gx < W) && (gy < H);
            const float* m = dmaps + (static_cast<int64_t>(gy) * W + gx) * 9 + c * 3;
            sm[0][ly][lx] = in ? m[0] : 0.f;
            sm[1][ly][lx] = in ? m[1] : 0.f;
            sm[2][ly][lx] = in ? m[2] : 0.f;
        }
        __syncthreads();
        for (int i = tid; i < kS * kT; i += kT * kT) {
            const int ly = i / kT, lx = i - ly * kT;
            float a0 = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll
            for (int k = 0; k < 11; ++k) {
                const float wk = win.w[k];
                a0 += wk * sm[0][ly][lx + k]; a1 += wk * sm[1][ly][lx + k]; a2 += wk * sm[2][ly][lx + k];
            }
            hz[0][ly][lx] = a0; hz[1][ly][lx] = a1; hz[2][ly][lx] = a2;
        }
        __syncthreads();
        float c0 = 0.f, c1 = 0.f, c2 = 0.f;
#pragma unroll
        for (int k = 0; k < 11; ++k) {
            const float wk = win.w[k];
            c0 += wk * hz[0][ty + k][tx]; c1 += wk * hz[1][ty + k][tx]; c2 += wk * hz[2][ty + k][tx];
        }
        if (inside) {
            const int64_t p = static_cast<int64_t>(py) * W + px;
            float xv, yv;
            load_xy<PS, BG, MASK>(pred_rgba, target, cp, p, c, xv, yv);
            const float diff = xv - yv;
            const float sgn = diff > 0.f ? 1.f : (diff < 0.f ? -1.f : 0.f);
            grad[c] = c0 + 2.f * xv * c1 + yv * c2 + l1_scale * sgn;
        }
        __syncthreads();
    }
    if (!inside) return;
    const int64_t p = static_cast<int64_t>(py) * W + px;
    // chain rule through the mask and the composite: grad is d loss / d x of the masked composite
    if constexpr (MASK) {
        const float m = cp.mask[p];
        grad[0] *= m; grad[1] *= m; grad[2] *= m;
    }
    float d_alpha = 0.f;
    if constexpr (BG == 1) d_alpha = -(cp.bg[0] * grad[0] + cp.bg[1] * grad[1] + cp.bg[2] * grad[2]);
    if constexpr (BG == 2) {
        const float* b = cp.bg_image + p * 3;
        d_alpha = -(b[0] * grad[0] + b[1] * grad[1] + b[2] * grad[2]);
    }
    if (GS == 4) {
        reinterpret_cast<float4*>(d_rgba)[p] = make_float4(grad[0], grad[1], grad[2], d_alpha);
    } else {
        d_rgba[p * GS + 0] = grad[0];
        d_rgba[p * GS + 1] = grad[1];
        d_rgba[p * GS + 2] = grad[2];
        if constexpr (BG != 0 || MASK) cp.d_alpha[p] = d_alpha;
    }
}

template <int PS, int GS, int BG = 0, bool MASK = false>
int image_loss(void* stream, int32_t height, int32_t width, const float* pred, const float* target_rgb, float lambda_l1, float lambda_ssim,
               void* scratch, float* d_pred, float* sums2, Composite cp = Composite{}) {
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    Window win;
    double g[11], total = 0.0;
    for (int i = 0; i < 11; ++i) {
        const double x = i - 5;
        g[i] = exp(-(x * x) / (2.0 * 1.5 * 1.5));
        total += g[i];
    }
    for (int i = 0; i < 11; ++i) win.w[i] = static_cast<float>(g[i] / total);
    const double count = (height > 10 && width > 10) ? static_cast<double>(height - 10) * (width - 10) * 3.0 : 1.0;
    const dim3 block(kT, kT), grid((width + kT - 1) / kT, (height + kT - 1) / kT);
    float* dmaps = static_cast<float*>(scratch);
    if constexpr (BG != 0 || MASK) {
        // the composited kernels keep their two sums in fp64 at the head of the scratch (its 16 spare bytes), the maps after them
        cp.acc = static_cast<double*>(scratch);
        cp.sums = sums2;
        dmaps = reinterpret_cast<float*>(static_cast<char*>(scratch) + 16);
        if (cudaMemsetAsync(cp.acc, 0, 2 * sizeof(double), s) != cudaSuccess) return 2;
    } else {
        if (cudaMemsetAsync(sums2, 0, 2 * sizeof(float), s) != cudaSuccess) return 2;
    }
    ssim_stats_kernel<PS, BG, MASK><<<grid, block, 0, s>>>(height, width, pred, target_rgb, cp, win, static_cast<float>(-lambda_ssim / count),
                                                           dmaps, sums2);
    loss_grad_kernel<PS, GS, BG, MASK><<<grid, block, 0, s>>>(height, width, pred, target_rgb, cp, win,
                                                              static_cast<float>(lambda_l1 / (static_cast<double>(height) * width * 3.0)), dmaps,
                                                              d_pred);
    return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

template <int L>
int image_loss_composited(void* stream, int32_t height, int32_t width, const float* pred, const float* target_rgb, float lambda_l1,
                          float lambda_ssim, void* scratch, float* d_pred, float* sums2, const Composite& cp, int bg_mode, bool mask) {
    if (bg_mode == 0 && !mask) {
        // black, no mask: the plain loss; the split layout's alpha gradient is zero
        if (L == 3 && cudaMemsetAsync(cp.d_alpha, 0, static_cast<size_t>(height) * width * sizeof(float), static_cast<cudaStream_t>(stream)) != cudaSuccess)
            return 2;
        return image_loss<L, L>(stream, height, width, pred, target_rgb, lambda_l1, lambda_ssim, scratch, d_pred, sums2);
    }
#define GUT_LOSS_CASE(BG_, M_) \
    if (bg_mode == BG_ && mask == M_) return image_loss<L, L, BG_, M_>(stream, height, width, pred, target_rgb, lambda_l1, lambda_ssim, scratch, d_pred, sums2, cp);
    GUT_LOSS_CASE(0, true)
    GUT_LOSS_CASE(1, false)
    GUT_LOSS_CASE(1, true)
    GUT_LOSS_CASE(2, false)
    GUT_LOSS_CASE(2, true)
#undef GUT_LOSS_CASE
    return 1;
}

}  // namespace

}  // namespace gutb200

extern "C" {

size_t gutb200_image_loss_scratch_bytes(int32_t height, int32_t width) {
    return static_cast<size_t>(height) * static_cast<size_t>(width) * 9 * sizeof(float) + 16;
}

int gutb200_image_loss(void* stream, int32_t height, int32_t width, const float* pred_rgba, const float* target_rgb, float lambda_l1,
                       float lambda_ssim, void* scratch, float* d_rgba, float* sums2) {
    if (height <= 0 || width <= 0 || !pred_rgba || !target_rgb || !scratch || !d_rgba || !sums2) return 1;
    if ((reinterpret_cast<uintptr_t>(d_rgba) & 15) != 0) return 3;
    return gutb200::image_loss<4, 4>(stream, height, width, pred_rgba, target_rgb, lambda_l1, lambda_ssim, scratch, d_rgba, sums2);
}

// The same loss on the 3DGRT layout: prediction rgb [H,W,3] (alpha is a separate output there and takes no part), gradient d_rgb [H,W,3].
int gutb200_image_loss_rgb(void* stream, int32_t height, int32_t width, const float* pred_rgb, const float* target_rgb, float lambda_l1,
                           float lambda_ssim, void* scratch, float* d_rgb, float* sums2) {
    if (height <= 0 || width <= 0 || !pred_rgb || !target_rgb || !scratch || !d_rgb || !sums2) return 1;
    return gutb200::image_loss<3, 3>(stream, height, width, pred_rgb, target_rgb, lambda_l1, lambda_ssim, scratch, d_rgb, sums2);
}

// The loss on the composited, masked prediction (see the top of this file), for either layout:
//   layout 4: pred [H,W,4] rgba, d_pred [H,W,4] = d_rgba with its alpha gradient (16-byte aligned); pred_alpha / d_alpha unused
//   layout 3: pred [H,W,3] rgb + pred_alpha [H,W], d_pred [H,W,3] = d_rgb + d_alpha [H,W]
// background_rgb: 3 host floats, or NULL (black); background_image: [H,W,3] device image (takes precedence), or NULL.  A black background
// is skipped entirely: no alpha gradient.  mask: [H,W] device floats, or NULL.
int gutb200_image_loss_composited(void* stream, int32_t height, int32_t width, int32_t layout, const float* pred, const float* pred_alpha,
                                  const float* target_rgb, const float* background_rgb, const float* background_image, const float* mask,
                                  float lambda_l1, float lambda_ssim, void* scratch, float* d_pred, float* d_alpha, float* sums2) {
    if (height <= 0 || width <= 0 || !pred || !target_rgb || !scratch || !d_pred || !sums2) return 1;
    if (layout != 3 && layout != 4) return 1;
    if (layout == 3 && (!pred_alpha || !d_alpha)) return 1;
    if (layout == 4 && (reinterpret_cast<uintptr_t>(d_pred) & 15) != 0) return 3;
    gutb200::Composite cp{};
    cp.alpha = pred_alpha;
    cp.d_alpha = d_alpha;
    cp.mask = mask;
    int bg_mode = 0;
    if (background_image) {
        cp.bg_image = background_image;
        bg_mode = 2;
    } else if (background_rgb && (background_rgb[0] != 0.f || background_rgb[1] != 0.f || background_rgb[2] != 0.f)) {
        for (int c = 0; c < 3; ++c) cp.bg[c] = background_rgb[c];
        bg_mode = 1;
    }
    if (layout == 4)
        return gutb200::image_loss_composited<4>(stream, height, width, pred, target_rgb, lambda_l1, lambda_ssim, scratch, d_pred, sums2, cp,
                                                 bg_mode, mask != nullptr);
    return gutb200::image_loss_composited<3>(stream, height, width, pred, target_rgb, lambda_l1, lambda_ssim, scratch, d_pred, sums2, cp, bg_mode,
                                             mask != nullptr);
}

}  // extern "C"
