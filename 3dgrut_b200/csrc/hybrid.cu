// 3dgrut_b200/csrc/hybrid.cu -- device code of the 3DGRUT hybrid training step (train_step_hybrid.GaussianTrainStepHybrid): primary camera
// rays through 3DGUT, their mirror reflections off a plane through 3DGRT, the two images composited (hybrid.py: mirror_rays, render_hybrid).
//
//   hybrid_rays_kernel            camera rays [P,3] + the host 3x4 camera-to-world -> world secondary origins / directions [P,3], hit [P]
//   hybrid_composite_kernel       rgb = primary_rgb + reflectivity (1 - alpha_p) hit secondary_rgb           [H,W,4] + [P,3] -> [H,W,3]
//   hybrid_composite_bwd_kernel   its adjoint: the 3DGUT d_rgba [H,W,4] and the 3DGRT d_rgb [P,3]
//
// One thread per pixel, no shared memory, no synchronisation.  The unit is built with -fmad=false and every expression keeps the operation
// order of the torch code in hybrid.py, so the forward outputs are those of its elementwise kernels bit for bit (the ray transform `rays @ R.T`
// is a matmul there, whose summation order is the library's: rays agree to rounding).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/gut_b200.h"

namespace gutb200 {

namespace {

constexpr int kBlock = 256;

struct Mirror {
    float r[12];   // camera-to-world rows [R | t], row-major 3x4
    float p0[3];   // plane point
    float n[3];    // unit plane normal
};

__global__ void __launch_bounds__(kBlock) hybrid_rays_kernel(int64_t pixels, const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                                             Mirror m, float* __restrict__ out_o, float* __restrict__ out_d,
                                                             float* __restrict__ out_hit) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * kBlock + threadIdx.x;
    if (i >= pixels) return;
    const float ox = rays_o[i * 3 + 0], oy = rays_o[i * 3 + 1], oz = rays_o[i * 3 + 2];
    const float dx = rays_d[i * 3 + 0], dy = rays_d[i * 3 + 1], dz = rays_d[i * 3 + 2];
    float o[3], d[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float* r = m.r + 4 * k;
        o[k] = ((r[0] * ox + r[1] * oy) + r[2] * oz) + r[3];   // rays_ori @ R.T + t
        d[k] = (r[0] * dx + r[1] * dy) + r[2] * dz;            // rays_dir @ R.T
    }
    const float denom = (d[0] * m.n[0] + d[1] * m.n[1]) + d[2] * m.n[2];
    const float num = ((m.p0[0] - o[0]) * m.n[0] + (m.p0[1] - o[1]) * m.n[1]) + (m.p0[2] - o[2]) * m.n[2];
    const float s = num / (fabsf(denom) > 1e-8f ? denom : 1e-8f);  // torch.where(|denom| > 1e-8, denom, 1e-8): +1e-8 for either sign
    const bool hit = s > 0.f && denom < 0.f;
    const float twice = 2.0f * denom;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        out_o[i * 3 + k] = hit ? o[k] + s * d[k] : o[k];
        out_d[i * 3 + k] = hit ? d[k] - twice * m.n[k] : d[k];
    }
    out_hit[i] = hit ? 1.f : 0.f;
}

__global__ void __launch_bounds__(kBlock) hybrid_composite_kernel(int64_t pixels, const float* __restrict__ primary_rgba,
                                                                  const float* __restrict__ secondary_rgb, const float* __restrict__ hit,
                                                                  float reflectivity, float* __restrict__ out_rgb) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * kBlock + threadIdx.x;
    if (i >= pixels) return;
    const float4 p = reinterpret_cast<const float4*>(primary_rgba)[i];
    const float w = (reflectivity * (1.0f - p.w)) * hit[i];  // render_hybrid: reflectivity * (1 - opacity) * hit
    out_rgb[i * 3 + 0] = p.x + w * secondary_rgb[i * 3 + 0];
    out_rgb[i * 3 + 1] = p.y + w * secondary_rgb[i * 3 + 1];
    out_rgb[i * 3 + 2] = p.z + w * secondary_rgb[i * 3 + 2];
}

__global__ void __launch_bounds__(kBlock) hybrid_composite_bwd_kernel(int64_t pixels, const float* __restrict__ primary_rgba,
                                                                      const float* __restrict__ secondary_rgb, const float* __restrict__ hit,
                                                                      float reflectivity, const float* __restrict__ d_rgb,
                                                                      const float* __restrict__ d_alpha, float* __restrict__ d_primary_rgba,
                                                                      float* __restrict__ d_secondary_rgb) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * kBlock + threadIdx.x;
    if (i >= pixels) return;
    const float a = primary_rgba[i * 4 + 3], h = hit[i];
    const float g0 = d_rgb[i * 3 + 0], g1 = d_rgb[i * 3 + 1], g2 = d_rgb[i * 3 + 2];
    const float s0 = secondary_rgb[i * 3 + 0], s1 = secondary_rgb[i * 3 + 1], s2 = secondary_rgb[i * 3 + 2];
    const float w = (reflectivity * (1.0f - a)) * h;
    const float dot = (g0 * s0 + g1 * s1) + g2 * s2;  // d loss / d w
    const float da = (d_alpha ? d_alpha[i] : 0.f) - (reflectivity * h) * dot;
    reinterpret_cast<float4*>(d_primary_rgba)[i] = make_float4(g0, g1, g2, da);
    d_secondary_rgb[i * 3 + 0] = w * g0;
    d_secondary_rgb[i * 3 + 1] = w * g1;
    d_secondary_rgb[i * 3 + 2] = w * g2;
}

inline unsigned blocks_for(int64_t pixels) { return static_cast<unsigned>((pixels + kBlock - 1) / kBlock); }

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

}  // namespace gutb200

extern "C" {

int gutb200_hybrid_rays(void* stream, int64_t pixels, const float* rays_o, const float* rays_d, const float* T_to_world_host,
                        const float* plane_point_host, const float* plane_normal_host, float* out_o, float* out_d, float* out_hit) {
    if (pixels < 0 || !T_to_world_host || !plane_point_host || !plane_normal_host) return 1;
    if (pixels == 0) return 0;
    if (!rays_o || !rays_d || !out_o || !out_d || !out_hit) return 1;
    gutb200::Mirror m;
    for (int k = 0; k < 12; ++k) m.r[k] = T_to_world_host[k];
    for (int k = 0; k < 3; ++k) {
        m.p0[k] = plane_point_host[k];
        m.n[k] = plane_normal_host[k];
    }
    gutb200::hybrid_rays_kernel<<<gutb200::blocks_for(pixels), gutb200::kBlock, 0, static_cast<cudaStream_t>(stream)>>>(pixels, rays_o, rays_d, m,
                                                                                                                        out_o, out_d, out_hit);
    return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

int gutb200_hybrid_composite(void* stream, int64_t pixels, const float* primary_rgba, const float* secondary_rgb, const float* hit,
                             float reflectivity, float* out_rgb) {
    if (pixels < 0) return 1;
    if (pixels == 0) return 0;
    if (!primary_rgba || !secondary_rgb || !hit || !out_rgb) return 1;
    if (!gutb200::aligned16(primary_rgba)) return 3;
    gutb200::hybrid_composite_kernel<<<gutb200::blocks_for(pixels), gutb200::kBlock, 0, static_cast<cudaStream_t>(stream)>>>(
        pixels, primary_rgba, secondary_rgb, hit, reflectivity, out_rgb);
    return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

int gutb200_hybrid_composite_bwd(void* stream, int64_t pixels, const float* primary_rgba, const float* secondary_rgb, const float* hit,
                                 float reflectivity, const float* d_rgb, const float* d_alpha, float* d_primary_rgba, float* d_secondary_rgb) {
    if (pixels < 0) return 1;
    if (pixels == 0) return 0;
    if (!primary_rgba || !secondary_rgb || !hit || !d_rgb || !d_primary_rgba || !d_secondary_rgb) return 1;
    if (!gutb200::aligned16(d_primary_rgba)) return 3;
    gutb200::hybrid_composite_bwd_kernel<<<gutb200::blocks_for(pixels), gutb200::kBlock, 0, static_cast<cudaStream_t>(stream)>>>(
        pixels, primary_rgba, secondary_rgb, hit, reflectivity, d_rgb, d_alpha, d_primary_rgba, d_secondary_rgb);
    return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

}  // extern "C"
