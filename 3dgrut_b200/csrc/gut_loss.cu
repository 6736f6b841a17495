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
// Both are templated on the pixel strides of the prediction and the gradient, so that layout 3 of gutb200_image_loss runs the same
// arithmetic on the 3DGRT layout (rgb [H,W,3] in, d_rgb [H,W,3] out, directly the d_rgb argument of grtb200_trace_bwd).
//
// A background and a mask add the two image-side parts of the training loss (threedgrut/model/background.py:80-93,
// trainer.py:691-694) where the kernels load x and y, and their chain rule where loss_grad_kernel writes:
//     x = (rgb + bg (1 - alpha)) m,  y = target m          bg: constant colour or [H,W,3] image; m: optional [H,W] mask
//     d rgb_c = m dL/dx_c,  d alpha = -sum_c bg_c m dL/dx_c
// The background mode (BG) and the mask (MASK) are template parameters beside the strides; BG = 0 (black) with no mask is the plain loss.
//
// post_processing = 1 adds the reference's `post_processing.method: linear-to-srgb` (threedgrut/utils/
// post_processing_linear_to_srgb.py, applied after the background and before the loss, trainer.py:1165-1172) as a third template
// parameter, POST (0 none, 1 linear-to-sRGB), between the composite and the mask:
//     x = s(c) m,  c = rgb + bg (1 - alpha),   s(c) = 1.055 max(c, 1e-8)^(1/2.4) - 0.055 if c > 0.0031308, else 12.92 c   (no clamp: HDR)
//     d rgb_c = m s'(c_c) dL/dx_c,  d alpha = -sum_c bg_c m s'(c_c) dL/dx_c
// POST = 0 compiles every existing instantiation to the code it had without this parameter.
//
// The one C entry point, gutb200_image_loss, turns (layout, background mode, mask, post-processing) into those template arguments in one
// dispatch: 2 x 3 x 2 x 2 instantiations of each kernel.
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <type_traits>

#include "../../include/gut_b200.h"
#include "image_common.cuh"

namespace gutb200 {

void set_context_free_error(const std::string& msg);  // gut_api.cu: the message gutb200_last_error(NULL) returns

namespace {

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
template <int PS, int BG = 0, bool MASK = false, int POST = 0>
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
            if (in) load_xy<PS, BG, MASK, POST>(pred_rgba, target, cp, p, c, xv, yv);
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
        if constexpr (BG != 0 || MASK || POST != 0) {  // fp64 totals: the 1e-6 bar of the means holds at 800x800 with masked (partly constant) images
            atomicAdd(cp.acc + 0, static_cast<double>(l1_block));
            atomicAdd(cp.acc + 1, static_cast<double>(ss_block));
        } else {
            atomicAdd(sums + 0, l1_block);
            atomicAdd(sums + 1, ss_block);
        }
    }
}

// GS: floats per pixel of the gradient (4: d_rgba, one 16-byte store, its alpha gradient zero unless BG != 0; 3: d_rgb, plus cp.d_alpha
// in the composited instantiations).
template <int PS, int GS, int BG = 0, bool MASK = false, int POST = 0>
__global__ void __launch_bounds__(kT * kT) loss_grad_kernel(int H, int W, const float* __restrict__ pred_rgba, const float* __restrict__ target,
                                                            Composite cp, Window win, float l1_scale /* lambda_l1 / (H W 3) */,
                                                            const float* __restrict__ dmaps, float* __restrict__ d_rgba) {
    __shared__ float sm[3][kS][kS + 1];
    __shared__ float hz[3][kS][kT + 1];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kT + tx;
    const int x0 = blockIdx.x * kT, y0 = blockIdx.y * kT;
    const int px = x0 + tx, py = y0 + ty;
    const bool inside = (px < W) && (py < H);
    if constexpr (BG != 0 || MASK || POST != 0) {
        if (blockIdx.x == 0 && blockIdx.y == 0 && tid == 0) {  // every block of ssim_stats_kernel has finished (stream order)
            cp.sums[0] = static_cast<float>(cp.acc[0]);
            cp.sums[1] = static_cast<float>(cp.acc[1]);
        }
    }
    float grad[3] = {0.f, 0.f, 0.f};
    float slope[3];  // s'(c) of the post-processing (POST)
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
            load_xy<PS, BG, MASK, POST>(pred_rgba, target, cp, p, c, xv, yv);
            if constexpr (POST == 1) slope[c] = linear_to_srgb_slope(composite<PS, BG>(pred_rgba[p * PS + c], pred_rgba, cp, p, c));
            const float diff = xv - yv;
            const float sgn = diff > 0.f ? 1.f : (diff < 0.f ? -1.f : 0.f);
            grad[c] = c0 + 2.f * xv * c1 + yv * c2 + l1_scale * sgn;
        }
        __syncthreads();
    }
    if (!inside) return;
    const int64_t p = static_cast<int64_t>(py) * W + px;
    // chain rule through the mask, the post-processing and the composite: grad is d loss / d x of the masked composite
    if constexpr (POST != 0) {
        grad[0] *= slope[0]; grad[1] *= slope[1]; grad[2] *= slope[2];
    }
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
        if constexpr (BG != 0 || MASK || POST != 0) cp.d_alpha[p] = d_alpha;
    }
}

template <int PS, int GS, int BG, bool MASK, int POST>
cudaError_t image_loss(void* stream, int32_t height, int32_t width, const float* pred, const float* target_rgb, float lambda_l1,
                       float lambda_ssim, void* scratch, float* d_pred, float* sums2, Composite cp) {
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const Window win = gaussian_window();
    const double count = (height > 10 && width > 10) ? static_cast<double>(height - 10) * (width - 10) * 3.0 : 1.0;
    const dim3 block(kT, kT), grid((width + kT - 1) / kT, (height + kT - 1) / kT);
    float* dmaps = static_cast<float*>(scratch);
    cudaError_t e;
    if constexpr (BG != 0 || MASK || POST != 0) {
        // the composited kernels keep their two sums in fp64 at the head of the scratch (its 16 spare bytes), the maps after them
        cp.acc = static_cast<double*>(scratch);
        cp.sums = sums2;
        dmaps = reinterpret_cast<float*>(static_cast<char*>(scratch) + 16);
        e = cudaMemsetAsync(cp.acc, 0, 2 * sizeof(double), s);
    } else {
        e = cudaMemsetAsync(sums2, 0, 2 * sizeof(float), s);
        // the plain kernels write no alpha gradient: on the split layout it is zero
        if (e == cudaSuccess && GS == 3 && cp.d_alpha) e = cudaMemsetAsync(cp.d_alpha, 0, static_cast<size_t>(height) * width * sizeof(float), s);
    }
    if (e != cudaSuccess) return e;
    ssim_stats_kernel<PS, BG, MASK, POST><<<grid, block, 0, s>>>(height, width, pred, target_rgb, cp, win,
                                                                 static_cast<float>(-lambda_ssim / count), dmaps, sums2);
    loss_grad_kernel<PS, GS, BG, MASK, POST><<<grid, block, 0, s>>>(height, width, pred, target_rgb, cp, win,
                                                                    static_cast<float>(lambda_l1 / (static_cast<double>(height) * width * 3.0)),
                                                                    dmaps, d_pred);
    return cudaGetLastError();
}

// The runtime value v in [0, N) as a template argument: f(std::integral_constant<int, v>()), as grt.cu's with_kind does.
template <int N, class F>
cudaError_t with_value(int v, F&& f) {
    if constexpr (N == 1)
        return f(std::integral_constant<int, 0>());
    else
        return v == N - 1 ? f(std::integral_constant<int, N - 1>()) : with_value<N - 1>(v, f);
}

}  // namespace

}  // namespace gutb200

extern "C" {

size_t gutb200_image_loss_scratch_bytes(int32_t height, int32_t width) {
    return static_cast<size_t>(height) * static_cast<size_t>(width) * 9 * sizeof(float) + 16;
}

int gutb200_image_loss(void* stream, int32_t height, int32_t width, int32_t layout, const float* pred, const float* pred_alpha,
                       const float* target_rgb, const float* background_rgb, const float* background_image, const float* mask,
                       float lambda_l1, float lambda_ssim, void* scratch, float* d_pred, float* d_alpha, float* sums2, int32_t post_processing) {
    const auto fail = [](int rc, const std::string& why) {
        gutb200::set_context_free_error("gutb200_image_loss: " + why);
        return rc;
    };
    if (height <= 0 || width <= 0 || !pred || !target_rgb || !scratch || !d_pred || !sums2)
        return fail(1, "needs a positive height and width and non-null pred, target_rgb, scratch, d_pred and sums2");
    if (layout != 3 && layout != 4) return fail(1, "layout=" + std::to_string(layout) + " (3 = rgb + alpha, 4 = rgba)");
    if (post_processing != 0 && post_processing != 1)
        return fail(1, "post_processing=" + std::to_string(post_processing) + " is not built (0 = none, 1 = linear-to-sRGB)");
    gutb200::Composite cp{};
    cp.alpha = pred_alpha;
    cp.d_alpha = d_alpha;
    cp.mask = mask;
    int bg_mode = 0;  // a black background is skipped entirely: no alpha gradient
    if (background_image) {
        cp.bg_image = background_image;
        bg_mode = 2;
    } else if (background_rgb && (background_rgb[0] != 0.f || background_rgb[1] != 0.f || background_rgb[2] != 0.f)) {
        for (int c = 0; c < 3; ++c) cp.bg[c] = background_rgb[c];
        bg_mode = 1;
    }
    if (layout == 3 && bg_mode != 0 && !pred_alpha) return fail(1, "layout 3 with a background needs pred_alpha");
    if (layout == 3 && (bg_mode != 0 || mask || post_processing != 0) && !d_alpha)
        return fail(1, "layout 3 with a background, a mask or post-processing needs d_alpha");
    if (layout == 4 && (reinterpret_cast<uintptr_t>(d_pred) & 15) != 0) return fail(3, "layout 4 stores d_pred 16 bytes at a time: align it");
    const cudaError_t e = gutb200::with_value<2>(layout == 4, [&](auto wide) {
        return gutb200::with_value<3>(bg_mode, [&](auto bg) {
            return gutb200::with_value<2>(mask != nullptr, [&](auto masked) {
                return gutb200::with_value<2>(post_processing, [&](auto post) {
                    constexpr int L = decltype(wide)::value ? 4 : 3;
                    return gutb200::image_loss<L, L, decltype(bg)::value, decltype(masked)::value != 0, decltype(post)::value>(
                        stream, height, width, pred, target_rgb, lambda_l1, lambda_ssim, scratch, d_pred, sums2, cp);
                });
            });
        });
    });
    return e == cudaSuccess ? 0 : fail(2, cudaGetErrorString(e));
}

}  // extern "C"
