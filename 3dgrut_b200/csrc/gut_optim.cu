// 3dgrut_b200/csrc/gut_optim.cu -- optimizer step of the Gaussian parameters (SURVEY.md section 8f row 2, "next" row).
//
//   selective_adam_kernel   drop-in for selective_adam_update_kernel of the reference plugin
//                           (threedgrut/optimizers/optimizers.cu:49-83): Adam without bias correction on the rows whose
//                           visibility flag is set, one launch per parameter tensor.
//   gaussian_adam_kernel    ours: ONE launch for all six parameter tensors of the SH model, taking the renderer's gradients
//                           ([N,12] w.r.t. post-activation position/density/quaternion/scale and [N,48] w.r.t. the SH coefficients,
//                           i.e. after the view-parallel exchange) and applying the activation chain rule the reference leaves to
//                           autograd (threedgrut/model/model.py:102-118 with utils/misc.py:46-50: density = sigmoid(raw),
//                           scale = exp(raw), rotation = normalize(raw)) followed by the Adam update, either torch.optim.Adam's
//                           (bias-corrected, model.py:807-810) or the selective one.
// gutb200_gaussian_adam_step_reg adds the opacity and scale regularisers of the reference loss (trainer.py:722-736:
// lambda_opacity mean|sigmoid(raw density)| + lambda_scale mean|exp(raw scale)|) to the activated density / scale gradients before the
// chain rule: + lambda_opacity / N and + lambda_scale / (3 N).  They are a template flag (REG) of the kernel, so the plain entry is unchanged.
// nht_adam_kernel is the same step for the NHT model (template variant of the same group code): features [N,48] are used raw, and the
// feature decoder's flat parameter vector is a sixth group with its own Adam (betas, eps, L2 weight decay, step count; never selective),
// as the reference trains it with a torch.optim.Adam of its own (trainer.py:573-577).  Groups in frozen_mask launch no block: parameters
// and moments stay untouched, as torch's Adam skips a parameter whose grad is None (colour refinement, trainer.py:168-195).
// All are streaming kernels: every byte is read and written once, coalesced (element-wise index space; the quaternion rows as
// float4).  Algorithmic bytes per Gaussian of the fused step: 59 x (4 param r + 4 param w + 8 moments r + 8 moments w) + 240
// gradient + 4 visibility = 1660 B.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/gut_b200.h"

namespace gutb200 {

namespace {

struct AdamHyper {
    float b1, b2, eps;
    float bc1, bc2_sqrt;  // bias corrections 1 - b1^t and sqrt(1 - b2^t); both 1 in selective mode
    int selective;
};

__device__ __forceinline__ float adam_update(float p, float g, float& m, float& v, float lr, const AdamHyper& h) {
    m = h.b1 * m + (1.0f - h.b1) * g;
    v = h.b2 * v + (1.0f - h.b2) * g * g;
    // selective: step = -lr m / (sqrt(v) + eps)                                   (optimizers.cu:74)
    // adam:      step = -(lr / bc1) m / (sqrt(v) / sqrt(bc2) + eps)               (torch.optim.Adam, single-tensor path)
    const float denom = sqrtf(v) / h.bc2_sqrt + h.eps;
    return p - (lr / h.bc1) * m / denom;
}

__global__ void __launch_bounds__(256) selective_adam_kernel(float* __restrict__ param, const float* __restrict__ grad, float* __restrict__ m,
                                                             float* __restrict__ v, const uint8_t* __restrict__ visibility, float lr,
                                                             AdamHyper h, int64_t total, int width) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= total) return;
    if (visibility && !visibility[i / width]) return;
    float mi = m[i], vi = v[i];
    param[i] = adam_update(param[i], grad[i], mi, vi, lr, h);
    m[i] = mi;
    v[i] = vi;
}

struct GaussianAdamArgs {
    float* param[6];        // positions [N,3], density [N,1], rotation [N,4], scale [N,3], albedo [N,3], specular [N,45] (raw, pre-activation)
    float* m[6];
    float* v[6];
    float lr[6];
    unsigned block_end[6];     // exclusive prefix of the blocks of each group: a block works on ONE group (no divergence)
    const float* d_particles;  // [N,12] dL/d(pos3, density, quat4 (wxyz), scale3, pad) w.r.t. the ACTIVATED values
    const float* d_sph;        // [N,48]
    const float* visibility;   // [N] float bits (the renderer's output) or nullptr
    int64_t n;
    AdamHyper h;
    float reg_density;         // lambda_opacity / N, added to d density (REG only)
    float reg_scale;           // lambda_scale / (3 N), added to every d scale (REG only)
};

struct NhtAdamArgs {
    float* param[6];           // positions [N,3], density [N,1], rotation [N,4], scale [N,3], features [N,48] (raw), decoder params [n_decoder]
    float* m[6];
    float* v[6];
    float lr[6];
    unsigned block_end[6];     // as in GaussianAdamArgs; a frozen group has no blocks
    const float* d_particles;  // [N,12] w.r.t. the activated values
    const float* d_features;   // [N,48] (the features are used raw: no chain rule)
    const float* d_decoder;    // [n_decoder]
    const float* visibility;   // [N] float bits or nullptr (Gaussian groups only)
    int64_t n;
    int64_t n_decoder;
    AdamHyper h[6];            // per group: its own step count; the decoder its own betas / eps and never selective
    float weight_decay;        // decoder: L2 on the gradient, g + weight_decay p (torch.optim.Adam weight_decay)
    float reg_density;
    float reg_scale;
};

// the hyper-parameters and the element count of group G (W floats per Gaussian)
template <int G> __device__ __forceinline__ const AdamHyper& group_hyper(const GaussianAdamArgs& a) { return a.h; }
template <int G> __device__ __forceinline__ const AdamHyper& group_hyper(const NhtAdamArgs& a) { return a.h[G]; }
template <int G, int W> __device__ __forceinline__ int64_t group_total(const GaussianAdamArgs& a) { return a.n * W; }
template <int G, int W> __device__ __forceinline__ int64_t group_total(const NhtAdamArgs& a) { return G == 5 ? a.n_decoder : a.n * W; }

// gradient w.r.t. the RAW value p of the [N,12]-record groups (positions, density, scale), shared by both layouts
template <int G, bool REG, class A>
__device__ __forceinline__ float particle_gradient(const A& a, int64_t row, int col, float p) {
    if (G == 0) return a.d_particles[row * 12 + col];
    if (G == 1) {
        const float s = 1.0f / (1.0f + expf(-p));   // density = sigmoid(raw)
        float g = a.d_particles[row * 12 + 3];
        if constexpr (REG) g = g + a.reg_density;
        return g * s * (1.0f - s);
    }
    float g = a.d_particles[row * 12 + 8 + col];
    if constexpr (REG) g = g + a.reg_scale;
    return g * expf(p);   // scale = exp(raw)
}

// gradient of element (row, col) of group G w.r.t. the RAW parameter value p
template <int G, bool REG>
__device__ __forceinline__ float raw_gradient(const GaussianAdamArgs& a, int64_t row, int col, float p) {
    if (G == 4) return a.d_sph[row * 48 + col];                        // features = cat(albedo [N,3], specular [N,45])  (model.py:94-96)
    if (G == 5) return a.d_sph[row * 48 + 3 + col];
    return particle_gradient<G, REG>(a, row, col, p);
}

template <int G, bool REG>
__device__ __forceinline__ float raw_gradient(const NhtAdamArgs& a, int64_t row, int col, float p) {
    if (G == 4) return a.d_features[row * 48 + col];                   // NHT features are raw (model.py:225)
    if (G == 5) return a.d_decoder[row] + a.weight_decay * p;
    return particle_gradient<G, REG>(a, row, col, p);
}

// flat groups: a thread owns 4 consecutive floats of the [N*W] array (16-byte loads and stores of param / moments)
template <int G, int W, bool REG, class A>
__device__ __forceinline__ void flat_group(const A& a, int64_t t) {
    const int64_t total = group_total<G, W>(a), e0 = t * 4;
    if (e0 >= total) return;
    float* P = a.param[G] + e0;
    float* M = a.m[G] + e0;
    float* V = a.v[G] + e0;
    const float lr = a.lr[G];
    const AdamHyper& h = group_hyper<G>(a);
    const bool masked = h.selective && a.visibility;
    if (e0 + 3 < total) {
        float4 p = *reinterpret_cast<float4*>(P), m = *reinterpret_cast<float4*>(M), v = *reinterpret_cast<float4*>(V);
        float pe[4] = {p.x, p.y, p.z, p.w}, me[4] = {m.x, m.y, m.z, m.w}, ve[4] = {v.x, v.y, v.z, v.w};
        bool any = false;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int64_t e = e0 + k, row = e / W;
            const int col = static_cast<int>(e - row * W);
            if (masked && (__float_as_uint(a.visibility[row]) == 0u)) continue;
            any = true;
            pe[k] = adam_update(pe[k], raw_gradient<G, REG>(a, row, col, pe[k]), me[k], ve[k], lr, h);
        }
        if (!any) return;  // nothing visible: leave the 48 bytes alone
        *reinterpret_cast<float4*>(P) = make_float4(pe[0], pe[1], pe[2], pe[3]);
        *reinterpret_cast<float4*>(M) = make_float4(me[0], me[1], me[2], me[3]);
        *reinterpret_cast<float4*>(V) = make_float4(ve[0], ve[1], ve[2], ve[3]);
    } else {
        for (int64_t e = e0; e < total; ++e) {
            const int64_t row = e / W;
            const int col = static_cast<int>(e - row * W);
            if (masked && (__float_as_uint(a.visibility[row]) == 0u)) continue;
            float m = a.m[G][e], v = a.v[G][e];
            const float p = a.param[G][e];
            a.param[G][e] = adam_update(p, raw_gradient<G, REG>(a, row, col, p), m, v, lr, h);
            a.m[G][e] = m;
            a.v[G][e] = v;
        }
    }
}

// rotation = normalize(raw), one row (float4) per thread: d raw = (g - q (q . g)) / max(|raw|, 1e-12)   (torch.nn.functional.normalize,
// eps 1e-12)
template <class A>
__device__ __forceinline__ void rotation_group(const A& a, int64_t t) {
    const AdamHyper& h = group_hyper<2>(a);
    const int64_t row = t;
    if (row >= a.n) return;
    if (h.selective && a.visibility && (__float_as_uint(a.visibility[row]) == 0u)) return;
    const float lr = a.lr[2];
    float4* P = reinterpret_cast<float4*>(a.param[2]) + row;
    float4* M = reinterpret_cast<float4*>(a.m[2]) + row;
    float4* V = reinterpret_cast<float4*>(a.v[2]) + row;
    const float4 r = *P;
    const float4 g = *reinterpret_cast<const float4*>(a.d_particles + row * 12 + 4);
    const float len = fmaxf(sqrtf(r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w), 1e-12f);
    const float il = 1.0f / len;
    const float qx = r.x * il, qy = r.y * il, qz = r.z * il, qw = r.w * il;
    const float dot = qx * g.x + qy * g.y + qz * g.z + qw * g.w;
    float4 m = *M, v = *V, out;
    out.x = adam_update(r.x, (g.x - qx * dot) * il, m.x, v.x, lr, h);
    out.y = adam_update(r.y, (g.y - qy * dot) * il, m.y, v.y, lr, h);
    out.z = adam_update(r.z, (g.z - qz * dot) * il, m.z, v.z, lr, h);
    out.w = adam_update(r.w, (g.w - qw * dot) * il, m.w, v.w, lr, h);
    *P = out;
    *M = m;
    *V = v;
}

// a block works on ONE group: the group whose block range holds blockIdx.x (empty ranges -- frozen groups -- are skipped)
template <class A>
__device__ __forceinline__ int block_group(const A& a, int64_t& t) {
    const unsigned blk = blockIdx.x;
    int group = 0;
#pragma unroll
    for (int k = 0; k < 5; ++k) group += blk >= a.block_end[k] ? 1 : 0;
    const unsigned first = group == 0 ? 0u : a.block_end[group - 1];
    t = static_cast<int64_t>(blk - first) * blockDim.x + threadIdx.x;
    return group;
}

template <bool REG>
__global__ void __launch_bounds__(256, 4) gaussian_adam_kernel(GaussianAdamArgs a) {
    int64_t t;
    switch (block_group(a, t)) {
        case 0: flat_group<0, 3, REG>(a, t); break;
        case 1: flat_group<1, 1, REG>(a, t); break;
        case 3: flat_group<3, 3, REG>(a, t); break;
        case 4: flat_group<4, 3, REG>(a, t); break;
        case 5: flat_group<5, 45, REG>(a, t); break;
        default: rotation_group(a, t);
    }
}

// The NHT model's step: the Gaussian groups with [N,48] raw features, and the decoder's flat parameter vector as a sixth group
template <bool REG>
__global__ void __launch_bounds__(256, 4) nht_adam_kernel(NhtAdamArgs a) {
    int64_t t;
    switch (block_group(a, t)) {
        case 0: flat_group<0, 3, REG>(a, t); break;
        case 1: flat_group<1, 1, REG>(a, t); break;
        case 3: flat_group<3, 3, REG>(a, t); break;
        case 4: flat_group<4, 48, REG>(a, t); break;
        case 5: flat_group<5, 1, REG>(a, t); break;
        default: rotation_group(a, t);
    }
}

AdamHyper make_hyper(float b1, float b2, float eps, int64_t step, int selective) {
    AdamHyper h;
    h.b1 = b1; h.b2 = b2; h.eps = eps; h.selective = selective;
    h.bc1 = 1.f; h.bc2_sqrt = 1.f;
    if (!selective) {
        double p1 = 1.0, p2 = 1.0;
        for (int64_t k = 0; k < step; ++k) { p1 *= b1; p2 *= b2; if (p1 < 1e-300 && p2 < 1e-300) break; }
        h.bc1 = static_cast<float>(1.0 - p1);
        h.bc2_sqrt = static_cast<float>(sqrt(1.0 - p2));
    }
    return h;
}

int gaussian_adam_step(void* stream, int64_t n, float* const* params6, float* const* exp_avg6, float* const* exp_avg_sq6, const float* lr6,
                       float b1, float b2, float eps, int64_t step, int32_t selective, const float* d_particles, const float* d_sph,
                       const float* visibility, float reg_density, float reg_scale) {
    if (n < 0 || !params6 || !exp_avg6 || !exp_avg_sq6 || !lr6 || !d_particles || !d_sph) return 1;
    if (!selective && step < 1) return 1;
    if (n == 0) return 0;
    GaussianAdamArgs a;
    for (int k = 0; k < 6; ++k) {
        if (!params6[k] || !exp_avg6[k] || !exp_avg_sq6[k]) return 1;
        a.param[k] = params6[k];
        a.m[k] = exp_avg6[k];
        a.v[k] = exp_avg_sq6[k];
        a.lr[k] = lr6[k];
    }
    for (int k = 0; k < 6; ++k) {  // parameters and moments are accessed 16 bytes at a time
        if ((reinterpret_cast<uintptr_t>(a.param[k]) | reinterpret_cast<uintptr_t>(a.m[k]) | reinterpret_cast<uintptr_t>(a.v[k])) & 15) return 3;
    }
    if (reinterpret_cast<uintptr_t>(d_particles) & 15) return 3;
    a.d_particles = d_particles;
    a.d_sph = d_sph;
    a.visibility = visibility;
    a.n = n;
    a.h = make_hyper(b1, b2, eps, step, selective);
    a.reg_density = reg_density;
    a.reg_scale = reg_scale;
    const int widths[6] = {3, 1, 4, 3, 3, 45};
    unsigned blocks = 0;
    for (int k = 0; k < 6; ++k) {
        const int64_t threads = k == 2 ? n : (n * widths[k] + 3) / 4;  // rotation: one row per thread; flat groups: 4 floats per thread
        blocks += static_cast<unsigned>((threads + 255) / 256);
        a.block_end[k] = blocks;
    }
    if (reg_density == 0.f && reg_scale == 0.f)
        gaussian_adam_kernel<false><<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
    else
        gaussian_adam_kernel<true><<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
    return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

int nht_adam_step(void* stream, int64_t n, int64_t n_decoder, float* const* params6, float* const* exp_avg6, float* const* exp_avg_sq6,
                  const float* lr6, const int64_t* steps6, float b1, float b2, float eps, int32_t selective, float decoder_b1, float decoder_b2,
                  float decoder_eps, float decoder_weight_decay, int32_t frozen_mask, const float* d_particles, const float* d_features,
                  const float* d_decoder, const float* visibility, float reg_density, float reg_scale) {
    if (n < 0 || n_decoder < 0 || !params6 || !exp_avg6 || !exp_avg_sq6 || !lr6 || !steps6) return 1;
    NhtAdamArgs a;
    const int widths[6] = {3, 1, 4, 3, 48, 1};
    unsigned blocks = 0;
    for (int k = 0; k < 6; ++k) {
        const bool frozen = (frozen_mask >> k) & 1;
        const int64_t count = k == 5 ? n_decoder : n;
        a.param[k] = params6[k];
        a.m[k] = exp_avg6[k];
        a.v[k] = exp_avg_sq6[k];
        a.lr[k] = lr6[k];
        if (!frozen && count > 0) {
            if (!params6[k] || !exp_avg6[k] || !exp_avg_sq6[k]) return 1;
            if ((reinterpret_cast<uintptr_t>(a.param[k]) | reinterpret_cast<uintptr_t>(a.m[k]) | reinterpret_cast<uintptr_t>(a.v[k])) & 15) return 3;
            const bool sel = k < 5 && selective;
            if (!sel && steps6[k] < 1) return 1;
            a.h[k] = k == 5 ? make_hyper(decoder_b1, decoder_b2, decoder_eps, steps6[k], 0) : make_hyper(b1, b2, eps, steps6[k], selective);
            // rotation: one row per thread; flat groups: 4 floats per thread
            const int64_t threads = k == 2 ? count : (count * widths[k] + 3) / 4;
            blocks += static_cast<unsigned>((threads + 255) / 256);
        } else {
            a.h[k] = make_hyper(b1, b2, eps, 0, 1);  // never read: the group launches no block
        }
        a.block_end[k] = blocks;
    }
    const bool gaussians = (~frozen_mask & 0x1f) != 0 && n > 0, decoder = !(frozen_mask & 0x20) && n_decoder > 0;
    if ((gaussians && !d_particles) || (gaussians && !(frozen_mask & 0x10) && !d_features) || (decoder && !d_decoder)) return 1;
    if (reinterpret_cast<uintptr_t>(d_particles) & 15) return 3;
    if (blocks == 0) return 0;
    a.d_particles = d_particles;
    a.d_features = d_features;
    a.d_decoder = d_decoder;
    a.visibility = visibility;
    a.n = n;
    a.n_decoder = n_decoder;
    a.weight_decay = decoder_weight_decay;
    a.reg_density = reg_density;
    a.reg_scale = reg_scale;
    if (reg_density == 0.f && reg_scale == 0.f)
        nht_adam_kernel<false><<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
    else
        nht_adam_kernel<true><<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
    return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

}  // namespace

}  // namespace gutb200

extern "C" {

int gutb200_selective_adam_update(void* stream, float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                                  const uint8_t* visibility, float lr, float b1, float b2, float eps, int64_t n, int64_t m) {
    using namespace gutb200;
    if (n < 0 || m <= 0 || !param || !grad || !exp_avg || !exp_avg_sq) return 1;
    const int64_t total = n * m;
    if (total == 0) return 0;
    if (m > 0x7FFFFFFF) return 1;
    const AdamHyper h = make_hyper(b1, b2, eps, 0, 1);
    const unsigned blocks = static_cast<unsigned>((total + 255) / 256);
    selective_adam_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(param, grad, exp_avg, exp_avg_sq, visibility, lr, h, total,
                                                                                 static_cast<int>(m));
    return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

int gutb200_gaussian_adam_step(void* stream, int64_t n, float* const* params6, float* const* exp_avg6, float* const* exp_avg_sq6,
                               const float* lr6, float b1, float b2, float eps, int64_t step, int32_t selective, const float* d_particles,
                               const float* d_sph, const float* visibility) {
    return gutb200::gaussian_adam_step(stream, n, params6, exp_avg6, exp_avg_sq6, lr6, b1, b2, eps, step, selective, d_particles, d_sph,
                                       visibility, 0.f, 0.f);
}

int gutb200_gaussian_adam_step_reg(void* stream, int64_t n, float* const* params6, float* const* exp_avg6, float* const* exp_avg_sq6,
                                   const float* lr6, float b1, float b2, float eps, int64_t step, int32_t selective, const float* d_particles,
                                   const float* d_sph, const float* visibility, float reg_density, float reg_scale) {
    return gutb200::gaussian_adam_step(stream, n, params6, exp_avg6, exp_avg_sq6, lr6, b1, b2, eps, step, selective, d_particles, d_sph,
                                       visibility, reg_density, reg_scale);
}

int gutb200_nht_adam_step(void* stream, int64_t n, int64_t n_decoder, float* const* params6, float* const* exp_avg6,
                          float* const* exp_avg_sq6, const float* lr6, const int64_t* steps6, float b1, float b2, float eps, int32_t selective,
                          float decoder_b1, float decoder_b2, float decoder_eps, float decoder_weight_decay, int32_t frozen_mask,
                          const float* d_particles, const float* d_features, const float* d_decoder, const float* visibility, float reg_density,
                          float reg_scale) {
    return gutb200::nht_adam_step(stream, n, n_decoder, params6, exp_avg6, exp_avg_sq6, lr6, steps6, b1, b2, eps, selective, decoder_b1,
                                  decoder_b2, decoder_eps, decoder_weight_decay, frozen_mask, d_particles, d_features, d_decoder, visibility,
                                  reg_density, reg_scale);
}

}  // extern "C"
