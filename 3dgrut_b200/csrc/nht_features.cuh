// 3dgrut_b200/csrc/nht_features.cuh -- Neural Harmonic Texture (NHT) feature maths shared by both tracers (gut_render_nht.cu,
// grt.cu): barycentric weights of the canonical hit point, the blend of the 4 x 12 vertex features and the adjoint of both with
// respect to the hit point.  Restated (not copied) from neuralHarmonicFeaturesParticle.slang:46-66 (canonical tetrahedron),
// :123-134 (barycentric weights), :152-189 (blend + sincos); the 3DGRT copy of that file equals the 3DGUT one.
// Configuration built: 48 features per particle = 4 tetrahedron vertices x 12, barycentric interpolation, sincos x 1 frequency,
// so 24 ray features (DESIGN.md sections 12, 13).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

namespace gutb200 {

constexpr int kNhtBase = 12;                    // features per tetrahedron vertex
constexpr int kNhtOut = 2 * kNhtBase;           // ray features (sin, cos of every blended feature)
constexpr int kNhtRow = 4 * kNhtBase;           // particle feature row

// tetrahedron vertices / 12: w_k = 1/4 + vk12[k] . P
static __constant__ float kVk12[4][3] = {{0.2041241452319315f, -0.11785113019775793f, -0.08333333333333333f},
                                   {-0.2041241452319315f, -0.11785113019775793f, -0.08333333333333333f},
                                   {0.0f, 0.23570226039551587f, -0.08333333333333333f},
                                   {0.0f, 0.0f, 0.25f}};

__device__ __forceinline__ void bary_weights(float px, float py, float pz, float (&w)[4]) {
#pragma unroll
    for (int k = 0; k < 4; ++k) w[k] = 0.25f + (kVk12[k][0] * px + kVk12[k][1] * py + kVk12[k][2] * pz);
}

// blended base features of row `f` (12 float4 = [vertex][12], fp32)
__device__ __forceinline__ void blend(const float4* __restrict__ f, const float (&w)[4], float (&b)[kNhtBase]) {
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        float4 a = f[q];
        b[q * 4 + 0] = w[0] * a.x; b[q * 4 + 1] = w[0] * a.y; b[q * 4 + 2] = w[0] * a.z; b[q * 4 + 3] = w[0] * a.w;
    }
#pragma unroll
    for (int k = 1; k < 4; ++k)
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            const float4 a = f[k * 3 + q];
            b[q * 4 + 0] += w[k] * a.x; b[q * 4 + 1] += w[k] * a.y; b[q * 4 + 2] += w[k] * a.z; b[q * 4 + 3] += w[k] * a.w;
        }
}

// float4 q (0..11) of a particle's feature row in global memory: fp32 rows are 12 float4, fp16 rows 6 x 16 bytes widened on load
template <bool HALF>
__device__ __forceinline__ float4 feature_quad(const void* __restrict__ features, uint32_t pid, int q) {
    if (HALF) {
        const uint2 v = __ldg(reinterpret_cast<const uint2*>(features) + static_cast<size_t>(pid) * 12 + q);
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&v.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
        return make_float4(a.x, a.y, b.x, b.y);
    }
    return __ldg(reinterpret_cast<const float4*>(features) + static_cast<size_t>(pid) * 12 + q);
}

// blend of a feature row read from global memory (no staging): same arithmetic order as blend()
template <bool HALF>
__device__ __forceinline__ void blend_global(const void* __restrict__ features, uint32_t pid, const float (&w)[4], float (&b)[kNhtBase]) {
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        const float4 a = feature_quad<HALF>(features, pid, q);
        b[q * 4 + 0] = w[0] * a.x; b[q * 4 + 1] = w[0] * a.y; b[q * 4 + 2] = w[0] * a.z; b[q * 4 + 3] = w[0] * a.w;
    }
#pragma unroll
    for (int k = 1; k < 4; ++k)
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            const float4 a = feature_quad<HALF>(features, pid, k * 3 + q);
            b[q * 4 + 0] += w[k] * a.x; b[q * 4 + 1] += w[k] * a.y; b[q * 4 + 2] += w[k] * a.z; b[q * 4 + 3] += w[k] * a.w;
        }
}

// Adjoint of blend(bary_weights(P)) with respect to P, for a row in global memory: with e[n] = dL/db_n, accumulates
// Pg += sum_k (sum_n e_n f[k*12+n]) v_k / 12.  (gut_render_nht.cu keeps its own loop over the staged row.)
template <bool HALF>
__device__ __forceinline__ void point_grad_global(const void* __restrict__ features, uint32_t pid, const float (&e)[kNhtBase], float& pgx,
                                                  float& pgy, float& pgz) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        float h = 0.f;
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            const float4 f = feature_quad<HALF>(features, pid, k * 3 + q);
            h += f.x * e[q * 4] + f.y * e[q * 4 + 1] + f.z * e[q * 4 + 2] + f.w * e[q * 4 + 3];
        }
        pgx += h * kVk12[k][0]; pgy += h * kVk12[k][1]; pgz += h * kVk12[k][2];
    }
}

}  // namespace gutb200
