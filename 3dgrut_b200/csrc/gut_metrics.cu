// 3dgrut_b200/csrc/gut_metrics.cu -- the test-set metrics of a rendered frame as the reference evaluator computes them
// (threedgrut/render.py:294-369, trainer.py:641-657, 1350-1364), in four launches with no host synchronisation.
//
//     x = s(rgb + bg (1 - alpha))        the prediction the metrics see: composited, then post-processed (s = identity or linear-to-sRGB)
//     psnr     = 10 log10(1 / mean (x - y)^2)                         torchmetrics PeakSignalNoiseRatio(data_range=1); +inf when x == y
//     ssim     = mean over the (H-10)(W-10) 3 interior of the SSIM map, 11-tap Gaussian window (sigma 1.5), C1 = 0.01^2, C2 = 0.03^2, the
//                variances clamped at 0 (torchmetrics StructuralSimilarityIndexMeasure(data_range=1.0): reflect pad 5, crop 5)
//     a, b     per channel over all HW pixels (threedgrut/utils/color_correct.py:96-145, color_correct_affine(x, y)):
//                var = max(E[y^2] - E[y]^2, 1e-8), a = (E[xy] - E[x] E[y]) / var, b = E[x] - a E[y], then a -> 1 where |a| < 1e-8
//     x_cc     = clip((x - b) / a, 0, 1);  cc_psnr, cc_ssim = psnr, ssim of x_cc against y
//     l1       = mean |x - y|;  hits: mean, unbiased std, min, max of the hit counts (trainer.py:641-644)
//     u8       = trunc(clamp(fl(fl(x 255) + 0.5), 0, 255)): the bytes torchvision.utils.save_image writes (for x and y)
//
//   metrics_pass_kernel<CC = false>  loads x, y on the SSIM tile of gut_loss.cu (image_common.cuh; the separable passes in fp64) and
//                                    writes per block: sum (x-y)^2, sum |x-y|, sum of the interior SSIM map, per channel sum x, y, y^2,
//                                    xy, and the hit sums / min / max; optionally the PNG bytes
//   finalise_kernel<false>           one block sums the partials in a fixed order (fp64) -> psnr, ssim, l1, hit statistics, a, b
//   metrics_pass_kernel<CC = true>   stages x_cc = clip((x - b) / a, 0, 1) into the SSIM tile (never written to memory): sum (x_cc - y)^2
//                                    and the interior SSIM map
//   finalise_kernel<true>            -> cc_psnr, cc_ssim
// No atomics: every block writes its own partials and the finalising block sums them in block order, so the same inputs give the same
// bits on every run.  The unit is built without fast-math and without contraction (-fmad=false): the composite rounds as its torch
// expression does, a, b are applied with IEEE division, and the quantisation rounds the product and the sum separately.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <string>
#include <type_traits>

#include "../../include/gut_b200.h"
#include "image_common.cuh"

namespace gutb200 {

void set_context_free_error(const std::string& msg);  // gut_api.cu: the message gutb200_last_error(NULL) returns

namespace {

// per-block partials of the first pass (fp64)
enum { kSq = 0, kL1 = 1, kSsim = 2, kSumX = 3, kSumY = 6, kSumYY = 9, kSumXY = 12, kHitSum = 15, kHitSq = 16, kHitMin = 17, kHitMax = 18,
       kQ1 = 19 };
// and of the second: sum (x_cc - y)^2, sum of the interior cc SSIM map
enum { kQ2 = 2 };
constexpr int kThreads = kT * kT;
constexpr double kC1d = 0.01 * 0.01, kC2d = 0.03 * 0.03;

// The SSIM window in fp64: the windowed moments are taken in fp64, so that E[x^2] - E[x]^2 does not cancel away the variance of a
// nearly flat window (the metric is a mean over few pixels on small frames, and is compared across runs at 1e-6).
struct WindowF64 {
    double w[11];
};

WindowF64 gaussian_window_f64() {
    WindowF64 win;
    double total = 0.0;
    for (int i = 0; i < 11; ++i) {
        const double x = i - 5;
        win.w[i] = exp(-(x * x) / (2.0 * 1.5 * 1.5));
        total += win.w[i];
    }
    for (int i = 0; i < 11; ++i) win.w[i] /= total;
    return win;
}

// Reduce v[0..Q) over the block in a fixed order; the totals are valid in thread 0.  op: 0 sum, 1 min, 2 max (per entry, from kinds).
template <int Q>
__device__ __forceinline__ void block_reduce(double (&v)[Q], const int (&kinds)[Q], double* red /* [8][Q] */) {
    const int tid = threadIdx.y * kT + threadIdx.x, warp = tid >> 5, lane = tid & 31;
#pragma unroll
    for (int q = 0; q < Q; ++q) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double u = __shfl_xor_sync(0xFFFFFFFFu, v[q], o);
            v[q] = kinds[q] == 0 ? v[q] + u : (kinds[q] == 1 ? fmin(v[q], u) : fmax(v[q], u));
        }
        if (lane == 0) red[warp * Q + q] = v[q];
    }
    __syncthreads();
    if (tid == 0) {
#pragma unroll
        for (int q = 0; q < Q; ++q) {
            double t = red[q];
            for (int w = 1; w < kThreads / 32; ++w) {
                const double u = red[w * Q + q];
                t = kinds[q] == 0 ? t + u : (kinds[q] == 1 ? fmin(t, u) : fmax(t, u));
            }
            v[q] = t;
        }
    }
}

__device__ __forceinline__ uint8_t to_u8(float v) {  // torchvision.utils.save_image: mul(255).add_(0.5).clamp_(0, 255).to(uint8)
    const float s = fminf(fmaxf(__fadd_rn(__fmul_rn(v, 255.0f), 0.5f), 0.0f), 255.0f);
    return static_cast<uint8_t>(s);
}

struct Outputs {
    const int32_t* hits;      // [H,W] or NULL
    uint8_t* pred_u8;         // [H,W,3] or NULL
    uint8_t* target_u8;       // [H,W,3] or NULL
    const float* ab;          // [6] = a[3], b[3] (CC pass)
    double* partials;         // [blocks, Q]
};

// PS, BG, POST as in gut_loss.cu (no mask).  CC: the second pass, on x_cc.
template <int PS, int BG, int POST, bool CC>
__global__ void __launch_bounds__(kThreads) metrics_pass_kernel(int H, int W, const float* __restrict__ pred, const float* __restrict__ target,
                                                                Composite cp, WindowF64 win, Outputs o) {
    constexpr int Q = CC ? kQ2 : kQ1;
    __shared__ float sx[kS][kS + 1], sy[kS][kS + 1];
    __shared__ double hz[5][kS][kT + 1];
    __shared__ double red[(kThreads / 32) * Q];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kT + tx;
    const int x0 = blockIdx.x * kT, y0 = blockIdx.y * kT;
    const int px = x0 + tx, py = y0 + ty;
    const bool inside = (px < W) && (py < H);
    const bool valid = inside && (px >= kR) && (py >= kR) && (px < W - kR) && (py < H - kR);
    const int64_t pc = static_cast<int64_t>(py) * W + px;
    double v[Q];
    int kinds[Q];
#pragma unroll
    for (int q = 0; q < Q; ++q) {
        v[q] = 0.0;
        kinds[q] = 0;
    }
    if constexpr (!CC) {
        kinds[kHitMin] = 1;
        kinds[kHitMax] = 2;
        v[kHitMin] = INFINITY;
        v[kHitMax] = -INFINITY;
        if (inside && o.hits) {
            const double h = static_cast<double>(o.hits[pc]);
            v[kHitSum] = h;
            v[kHitSq] = h * h;
            v[kHitMin] = h;
            v[kHitMax] = h;
        }
    }
    for (int c = 0; c < 3; ++c) {
        float a = 1.f, b = 0.f;
        if constexpr (CC) {
            a = o.ab[c];
            b = o.ab[3 + c];
        }
        for (int i = tid; i < kS * kS; i += kThreads) {
            const int ly = i / kS, lx = i - ly * kS;
            const int gx = x0 + lx - kR, gy = y0 + ly - kR;
            const bool in = (gx >= 0) && (gy >= 0) && (gx < W) && (gy < H);
            const int64_t p = static_cast<int64_t>(gy) * W + gx;
            float xv = 0.f, yv = 0.f;
            if (in) {
                load_xy<PS, BG, false, POST>(pred, target, cp, p, c, xv, yv);
                if constexpr (CC) xv = fminf(fmaxf(__fdiv_rn(__fsub_rn(xv, b), a), 0.f), 1.f);
            }
            sx[ly][lx] = xv;
            sy[ly][lx] = yv;
        }
        __syncthreads();
        for (int i = tid; i < kS * kT; i += kThreads) {
            const int ly = i / kT, lx = i - ly * kT;
            double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0, a4 = 0.0;
#pragma unroll
            for (int k = 0; k < 11; ++k) {
                const double xv = sx[ly][lx + k], yv = sy[ly][lx + k], wk = win.w[k];
                a0 += wk * xv; a1 += wk * yv; a2 += wk * (xv * xv); a3 += wk * (yv * yv); a4 += wk * (xv * yv);
            }
            hz[0][ly][lx] = a0; hz[1][ly][lx] = a1; hz[2][ly][lx] = a2; hz[3][ly][lx] = a3; hz[4][ly][lx] = a4;
        }
        __syncthreads();
        if (inside) {
            const float xv = sx[ty + kR][tx + kR], yv = sy[ty + kR][tx + kR];
            const double d = static_cast<double>(xv) - static_cast<double>(yv);
            v[0] += d * d;
            if constexpr (!CC) {
                v[kL1] += fabs(d);
                v[kSumX + c] += xv;
                v[kSumY + c] += yv;
                v[kSumYY + c] += static_cast<double>(yv) * yv;
                v[kSumXY + c] += static_cast<double>(xv) * yv;
                if (o.pred_u8) o.pred_u8[pc * 3 + c] = to_u8(xv);
                if (o.target_u8) o.target_u8[pc * 3 + c] = to_u8(yv);
            }
            if (valid) {
                double mu1 = 0.0, mu2 = 0.0, ex2 = 0.0, ey2 = 0.0, exy = 0.0;
#pragma unroll
                for (int k = 0; k < 11; ++k) {
                    const double wk = win.w[k];
                    mu1 += wk * hz[0][ty + k][tx]; mu2 += wk * hz[1][ty + k][tx]; ex2 += wk * hz[2][ty + k][tx];
                    ey2 += wk * hz[3][ty + k][tx]; exy += wk * hz[4][ty + k][tx];
                }
                // torchmetrics clamps both variances at 0 (the training loss's SSIM does not)
                const double s1 = fmax(ex2 - mu1 * mu1, 0.0), s2 = fmax(ey2 - mu2 * mu2, 0.0), s12 = exy - mu1 * mu2;
                const double num = (2.0 * mu1 * mu2 + kC1d) * (2.0 * s12 + kC2d), den = (mu1 * mu1 + mu2 * mu2 + kC1d) * (s1 + s2 + kC2d);
                v[CC ? 1 : kSsim] += num / den;
            }
        }
        __syncthreads();
    }
    block_reduce<Q>(v, kinds, red);
    if (tid == 0) {
        double* dst = o.partials + (static_cast<int64_t>(blockIdx.y) * gridDim.x + blockIdx.x) * Q;
#pragma unroll
        for (int q = 0; q < Q; ++q) dst[q] = v[q];
    }
}

__device__ __forceinline__ double psnr_of(double sq, double count) { return 10.0 * log10(1.0 / (sq / count)); }

// One block: sums the partials of every block of the pass in block order and writes its fields of out[GUTB200_METRICS_K].
template <bool CC>
__global__ void __launch_bounds__(kThreads) finalise_kernel(int H, int W, int blocks, const double* __restrict__ partials, int has_hits,
                                                            float* __restrict__ ab, double* __restrict__ out) {
    constexpr int Q = CC ? kQ2 : kQ1;
    __shared__ double red[(kThreads / 32) * Q];
    const int tid = threadIdx.y * kT + threadIdx.x;
    double v[Q];
    int kinds[Q];
#pragma unroll
    for (int q = 0; q < Q; ++q) {
        kinds[q] = 0;
        v[q] = 0.0;
    }
    if constexpr (!CC) {
        kinds[kHitMin] = 1;
        kinds[kHitMax] = 2;
        v[kHitMin] = INFINITY;
        v[kHitMax] = -INFINITY;
    }
    for (int i = tid; i < blocks; i += kThreads) {
        const double* p = partials + static_cast<int64_t>(i) * Q;
#pragma unroll
        for (int q = 0; q < Q; ++q) v[q] = kinds[q] == 0 ? v[q] + p[q] : (kinds[q] == 1 ? fmin(v[q], p[q]) : fmax(v[q], p[q]));
    }
    block_reduce<Q>(v, kinds, red);
    if (tid != 0) return;
    const double hw = static_cast<double>(H) * W, count = 3.0 * hw, interior = 3.0 * (H - 10.0) * (W - 10.0);
    if constexpr (CC) {
        out[GUTB200_METRIC_CC_PSNR] = psnr_of(v[0], count);
        out[GUTB200_METRIC_CC_SSIM] = v[1] / interior;
    } else {
        out[GUTB200_METRIC_PSNR] = psnr_of(v[kSq], count);
        out[GUTB200_METRIC_SSIM] = v[kSsim] / interior;
        out[GUTB200_METRIC_CC_PSNR] = NAN;  // until the second pass finalises
        out[GUTB200_METRIC_CC_SSIM] = NAN;
        out[GUTB200_METRIC_L1] = v[kL1] / count;
        if (has_hits) {
            const double mean = v[kHitSum] / hw;
            out[GUTB200_METRIC_HITS_MEAN] = mean;
            out[GUTB200_METRIC_HITS_STD] = hw > 1.0 ? sqrt(fmax(v[kHitSq] - v[kHitSum] * mean, 0.0) / (hw - 1.0)) : NAN;
            out[GUTB200_METRIC_HITS_MIN] = v[kHitMin];
            out[GUTB200_METRIC_HITS_MAX] = v[kHitMax];
        } else {
            out[GUTB200_METRIC_HITS_MEAN] = out[GUTB200_METRIC_HITS_STD] = out[GUTB200_METRIC_HITS_MIN] = out[GUTB200_METRIC_HITS_MAX] = NAN;
        }
        for (int c = 0; c < 3; ++c) {  // color_correct_affine: b takes the slope before it is replaced by 1
            const double ex = v[kSumX + c] / hw, ey = v[kSumY + c] / hw, eyy = v[kSumYY + c] / hw, exy = v[kSumXY + c] / hw;
            const double var = fmax(eyy - ey * ey, 1e-8);
            double a = (exy - ey * ex) / var;
            const double b = ex - a * ey;
            if (fabs(a) < 1e-8) a = 1.0;
            ab[c] = static_cast<float>(a);
            ab[3 + c] = static_cast<float>(b);
            out[GUTB200_METRIC_A + c] = a;
            out[GUTB200_METRIC_B + c] = b;
        }
    }
}

template <int PS, int BG, int POST>
cudaError_t image_metrics(cudaStream_t s, int H, int W, const float* pred, const float* target, Composite cp, Outputs o, void* scratch,
                          double* out) {
    const WindowF64 win = gaussian_window_f64();
    const dim3 block(kT, kT), grid((W + kT - 1) / kT, (H + kT - 1) / kT);
    const int blocks = static_cast<int>(grid.x * grid.y);
    double* part1 = static_cast<double*>(scratch);
    double* part2 = part1 + static_cast<size_t>(blocks) * kQ1;
    float* ab = reinterpret_cast<float*>(part2 + static_cast<size_t>(blocks) * kQ2);
    o.partials = part1;
    metrics_pass_kernel<PS, BG, POST, false><<<grid, block, 0, s>>>(H, W, pred, target, cp, win, o);
    finalise_kernel<false><<<1, block, 0, s>>>(H, W, blocks, part1, o.hits != nullptr, ab, out);
    Outputs o2{};
    o2.ab = ab;
    o2.partials = part2;
    metrics_pass_kernel<PS, BG, POST, true><<<grid, block, 0, s>>>(H, W, pred, target, cp, win, o2);
    finalise_kernel<true><<<1, block, 0, s>>>(H, W, blocks, part2, 0, ab, out);
    return cudaGetLastError();
}

template <int N, class F>
cudaError_t with_value(int v, F&& f) {
    if constexpr (N == 1)
        return f(std::integral_constant<int, 0>());
    else
        return v == N - 1 ? f(std::integral_constant<int, N - 1>()) : with_value<N - 1>(v, f);
}

size_t blocks_of(int32_t height, int32_t width) {
    return static_cast<size_t>((width + kT - 1) / kT) * static_cast<size_t>((height + kT - 1) / kT);
}

}  // namespace

}  // namespace gutb200

extern "C" {

size_t gutb200_image_metrics_scratch_bytes(int32_t height, int32_t width) {
    if (height <= 0 || width <= 0) return 0;
    return gutb200::blocks_of(height, width) * (gutb200::kQ1 + gutb200::kQ2) * sizeof(double) + 6 * sizeof(float);
}

int gutb200_image_metrics(void* stream, int32_t height, int32_t width, int32_t layout, const float* pred, const float* pred_alpha,
                          const float* target_rgb, const float* background_rgb, int32_t post_processing, const int32_t* hits, void* scratch,
                          double* out, uint8_t* pred_u8, uint8_t* target_u8) {
    const auto fail = [](int rc, const std::string& why) {
        gutb200::set_context_free_error("gutb200_image_metrics: " + why);
        return rc;
    };
    if (height < 11 || width < 11)
        return fail(1, "height and width must be at least 11 (the SSIM window's reflect pad and crop leave no interior below that); got " +
                           std::to_string(height) + "x" + std::to_string(width));
    if (!pred || !target_rgb || !scratch || !out) return fail(1, "needs non-null pred, target_rgb, scratch and out");
    if (layout != 3 && layout != 4) return fail(1, "layout=" + std::to_string(layout) + " (3 = rgb + alpha, 4 = rgba)");
    if (post_processing != 0 && post_processing != 1)
        return fail(1, "post_processing=" + std::to_string(post_processing) + " is not built (0 = none, 1 = linear-to-sRGB)");
    gutb200::Composite cp{};
    cp.alpha = pred_alpha;
    int bg_mode = 0;  // black: nothing is composited
    if (background_rgb && (background_rgb[0] != 0.f || background_rgb[1] != 0.f || background_rgb[2] != 0.f)) {
        for (int c = 0; c < 3; ++c) cp.bg[c] = background_rgb[c];
        bg_mode = 1;
    }
    if (layout == 3 && bg_mode != 0 && !pred_alpha) return fail(1, "layout 3 with a background needs pred_alpha");
    if ((reinterpret_cast<uintptr_t>(scratch) & 7) != 0) return fail(1, "scratch must be 8-byte aligned");
    gutb200::Outputs o{};
    o.hits = hits;
    o.pred_u8 = pred_u8;
    o.target_u8 = target_u8;
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const cudaError_t e = gutb200::with_value<2>(layout == 4, [&](auto wide) {
        return gutb200::with_value<2>(bg_mode, [&](auto bg) {
            return gutb200::with_value<2>(post_processing, [&](auto post) {
                constexpr int L = decltype(wide)::value ? 4 : 3;
                return gutb200::image_metrics<L, decltype(bg)::value, decltype(post)::value>(s, height, width, pred, target_rgb, cp, o, scratch,
                                                                                             out);
            });
        });
    });
    return e == cudaSuccess ? 0 : fail(2, cudaGetErrorString(e));
}

}  // extern "C"
