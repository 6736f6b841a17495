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
template <int PS>
__global__ void __launch_bounds__(kT * kT) ssim_stats_kernel(int H, int W, const float* __restrict__ pred_rgba, const float* __restrict__ target,
                                                             Window win, float g_scale /* -lambda_ssim / count */, float* __restrict__ dmaps,
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
            sx[ly][lx] = in ? pred_rgba[p * PS + c] : 0.f;
            sy[ly][lx] = in ? target[p * 3 + c] : 0.f;
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
        atomicAdd(sums + 0, l1_block);
        atomicAdd(sums + 1, ss_block);
    }
}

// GS: floats per pixel of the gradient (4: d_rgba with a zero alpha gradient, one 16-byte store; 3: d_rgb).
template <int PS, int GS>
__global__ void __launch_bounds__(kT * kT) loss_grad_kernel(int H, int W, const float* __restrict__ pred_rgba, const float* __restrict__ target,
                                                            Window win, float l1_scale /* lambda_l1 / (H W 3) */, const float* __restrict__ dmaps,
                                                            float* __restrict__ d_rgba) {
    __shared__ float sm[3][kS][kS + 1];
    __shared__ float hz[3][kS][kT + 1];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kT + tx;
    const int x0 = blockIdx.x * kT, y0 = blockIdx.y * kT;
    const int px = x0 + tx, py = y0 + ty;
    const bool inside = (px < W) && (py < H);
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
            const float xv = pred_rgba[p * PS + c], yv = target[p * 3 + c];
            const float diff = xv - yv;
            const float sgn = diff > 0.f ? 1.f : (diff < 0.f ? -1.f : 0.f);
            grad[c] = c0 + 2.f * xv * c1 + yv * c2 + l1_scale * sgn;
        }
        __syncthreads();
    }
    if (!inside) return;
    const int64_t p = static_cast<int64_t>(py) * W + px;
    if (GS == 4) {
        reinterpret_cast<float4*>(d_rgba)[p] = make_float4(grad[0], grad[1], grad[2], 0.f);
    } else {
        d_rgba[p * GS + 0] = grad[0];
        d_rgba[p * GS + 1] = grad[1];
        d_rgba[p * GS + 2] = grad[2];
    }
}

template <int PS, int GS>
int image_loss(void* stream, int32_t height, int32_t width, const float* pred, const float* target_rgb, float lambda_l1, float lambda_ssim,
               void* scratch, float* d_pred, float* sums2) {
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
    if (cudaMemsetAsync(sums2, 0, 2 * sizeof(float), s) != cudaSuccess) return 2;
    const dim3 block(kT, kT), grid((width + kT - 1) / kT, (height + kT - 1) / kT);
    float* dmaps = static_cast<float*>(scratch);
    ssim_stats_kernel<PS><<<grid, block, 0, s>>>(height, width, pred, target_rgb, win, static_cast<float>(-lambda_ssim / count), dmaps, sums2);
    loss_grad_kernel<PS, GS><<<grid, block, 0, s>>>(height, width, pred, target_rgb, win,
                                                    static_cast<float>(lambda_l1 / (static_cast<double>(height) * width * 3.0)), dmaps, d_pred);
    return cudaGetLastError() == cudaSuccess ? 0 : 2;
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

}  // extern "C"
