// 3dgrut_b200/csrc/gut_render_nht.cu -- per-tile compositing of Neural Harmonic Texture (NHT) features and its adjoint (3DGUT path).
//
// Reference semantics restated (not copied) from
//   threedgut_tracer/include/3dgut/kernels/slang/models/neuralHarmonicFeaturesParticle.slang:46-66 (canonical tetrahedron),
//     :123-134 (barycentric weights), :152-189 (blend + sincos), :199-212 (integration)
//   kernels/slang/models/gaussianParticles.slang:181-190 (canonical hit point), :231 (alpha clamp), :420-479 (backward)
//   kernels/cuda/renderers/gutKBufferRenderer.cuh:546-640 (per-ray backward, k-buffer = 0)
// Configuration built: 48 features per particle = 4 tetrahedron vertices x 12, barycentric interpolation, sincos x 1 frequency,
// so 24 ray features (DESIGN.md section 12).
//
// Per accepted (pixel, particle) pair, with gro / grd the canonical ray origin / unit direction of the SH path:
//   P   = gro + grd pd,  pd = -(grd . gro)                       canonical hit point
//   w_k = 1/4 + (v_k . P) / 12                                  barycentric weights of P in the tetrahedron v_0..v_3 (inradius 1);
//                                                               not clamped: P outside the tetrahedron extrapolates
//   b_n = sum_k w_k f[k*12 + n],  out[2n] = sin b_n, out[2n+1] = cos b_n
//   feat += out * alpha T   (when alpha T > 0; no max(., 0) as on the SH radiance)
// The forward is the shared tile walk (render_tile.cuh: sub-tile screens, hit words) with a feature payload; the batch is 128 entries so
// that the 48-float feature rows of a batch (24 KB) are staged on chip next to the geometry records.
#include <cuda_fp16.h>

#include "gut_common.cuh"
#include "nht_features.cuh"
#include "render_tile.cuh"
#include "subtile_cull.cuh"

namespace gutb200 {

namespace {

constexpr int kNhtBatch = 128;
constexpr int kNhtChannels = kNhtOut + 1;       // output channels: features, then opacity

// stage the feature rows of entries [base, base + count) into feat[entry][12 float4]; all threads of the CTA take part
template <bool HALF>
__device__ __forceinline__ void stage_features(float4 (*feat)[12], const void* __restrict__ features, const uint32_t* __restrict__ sorted_values,
                                               uint32_t base, int count, int tid) {
    if (HALF) {  // 96-byte rows: 6 x 16 bytes = 8 halves each
        const uint4* src = reinterpret_cast<const uint4*>(features);
        for (int f = tid; f < count * 6; f += kTilePixels) {
            const int e = f / 6, part = f - e * 6;
            const uint32_t idx = sorted_values[base + e];
            const uint4 v = __ldg(src + static_cast<size_t>(idx) * 6 + part);
            const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&v.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
            const float2 c = __half22float2(*reinterpret_cast<const __half2*>(&v.z)), d = __half22float2(*reinterpret_cast<const __half2*>(&v.w));
            feat[e][part * 2] = make_float4(a.x, a.y, b.x, b.y);
            feat[e][part * 2 + 1] = make_float4(c.x, c.y, d.x, d.y);
        }
    } else {
        const float4* src = reinterpret_cast<const float4*>(features);
        for (int f = tid; f < count * 12; f += kTilePixels) {
            const int e = f / 12, part = f - e * 12;
            const uint32_t idx = sorted_values[base + e];
            feat[e][part] = __ldg(src + static_cast<size_t>(idx) * 12 + part);
        }
    }
}

// ----------------------------------------------------------------------------------------------------------
// forward: the shared walk (render_tile.cuh) with the feature payload.  Staged record: FwdRecords, then the feature row.

struct NhtFwdSmem : FwdRecords<kNhtBatch> {
    float4 feat[kNhtBatch][12];
};

template <bool HALF>
struct FeaturePayload {
    float4 (*feat)[12];
    const void* __restrict__ features;
    float acc[kNhtOut];
    __device__ __forceinline__ void entry(int, uint32_t) {}
    __device__ __forceinline__ void batch(const uint32_t* __restrict__ sorted_values, uint32_t base, int count, int tid) {
        stage_features<HALF>(feat, features, sorted_values, base, count, tid);
    }
    __device__ __forceinline__ void add(int j, float w, float px, float py, float pz) {
        float wk[4], b[kNhtBase];
        bary_weights(px, py, pz, wk);
        blend(feat[j], wk, b);
#pragma unroll
        for (int n = 0; n < kNhtBase; ++n) {
            float s, c;
            sincosf(b[n], &s, &c);
            acc[2 * n] += s * w;
            acc[2 * n + 1] += c * w;
        }
    }
};

template <int DEG, bool HALF>
__global__ void __launch_bounds__(kTilePixels) render_forward_nht_kernel(FrameCamera cam, FrameConfig cfg, const float* __restrict__ rays_o,
                                                                         const float* __restrict__ rays_d, const float* __restrict__ particles,
                                                                         const void* __restrict__ features,
                                                                         const uint32_t* __restrict__ sorted_values,
                                                                         const uint32_t* __restrict__ ranges, const uint32_t* __restrict__ tile_order,
                                                                         const uint32_t* __restrict__ chunk_base, uint32_t* __restrict__ hit_words,
                                                                         float* __restrict__ out_features_alpha, float* __restrict__ out_dist,
                                                                         float* __restrict__ out_hits) {
    __shared__ NhtFwdSmem sm;
    const int tid = threadIdx.x;
    const TileRay tr = tile_ray(cam, rays_o, rays_d, tile_order, tid);
    float T = 1.f, dist = 0.f;
    FeaturePayload<HALF> pay{sm.feat, features};
#pragma unroll
    for (int c = 0; c < kNhtOut; ++c) pay.acc[c] = 0.f;
    uint32_t hits = 0;
    forward_list<DEG, false>(cam, cfg, sm, pay, tr, tid, rays_o, particles, sorted_values, ranges, chunk_base, hit_words, T, dist, hits, nullptr);

    const int64_t pix = tr.pix;
    if (!tr.inside) return;
    float* o = out_features_alpha + pix * kNhtChannels;
    if (tr.valid) {
#pragma unroll
        for (int c = 0; c < kNhtOut; ++c) o[c] = pay.acc[c];
        o[kNhtOut] = 1.0f - T;
        out_dist[pix] = dist;
        out_hits[pix] = static_cast<float>(hits);
    } else {
#pragma unroll
        for (int c = 0; c < kNhtChannels; ++c) o[c] = 0.f;
        out_dist[pix] = 1e06f;
        out_hits[pix] = 0.f;
    }
}

// ----------------------------------------------------------------------------------------------------------
// backward.
//
// Per accepted pair the adjoint is the SH path's (gut_render.cu, G7) with three changes:
//   * radiance -> features: the residual behind the pair is peeled front to back without a clamp, res = (F_out - F_acc) / T_next, so
//     only the dot products  sum_c F_out,c g_c  (per pixel) and  sum_c F_acc,c g_c  (running) are needed;
//   * alpha = min(max_alpha, response density) is differentiated: a clamped pair passes no gradient through response or density
//     (gaussianParticles.slang:231 under bwd_diff);
//   * the features depend on the hit point P = (I - grd grd^T) gro.  With Pg = dL/dP = alpha T sum_k h_k v_k / 12,
//     h_k = sum_n e_n f[k*12+n],  e_n = g_2n cos b_n - g_2n+1 sin b_n,  s = grd . Pg:
//         groGrd  += Pg - grd s
//         grduGrd += (pd Pg - s gro - 2 pd s grd) / |grdu|        (general adjoint of normalize(); the SH path's closed form
//                                                                  grduGrd = (pd / |grdu|) groGrd holds only for its own term)
//     so the canonical sums G, W of the SH path carry it and G8 maps them unchanged.
// The feature gradient of the pair is the outer product  d f[k*12+n] = w_k (alpha T e_n).  Each lane writes its 16 geometry slots
// and the 4 + 12 factors into a per-warp scratch row; lane l then sums feature entries l and l + 32 (or geometry slot l - 16) over the
// 32 rows, so one (warp, particle) pair lands 48 + 16 sums instead of 32 rows of 64 floats.  The warp walks the union of its four
// quarters' hit words.

struct NhtBwdSmem : BwdRecords<kNhtBatch> {
    float4 feat[kNhtBatch][12];
    uint32_t idx[kNhtBatch];
    uint32_t hw[(kNhtBatch / 32) * kWordsPerChunk];
    float rows[kTilePixels / 32][32][33];  // [warp][lane][slot], padded: lane-strided writes hit distinct banks
};

struct NhtBwdRay {
    float Tint, Tgrad, Dint, Dgrad, FiG;  // saved transmittance / distance, their gradients, sum_c F_out,c g_c
    float T, D, FG;                       // running transmittance, distance, sum_c F_acc,c g_c
    float g[kNhtOut];                     // feature gradient of the pixel
};

// the feature terms of backward_pair (render_tile.cuh): g[16..19] = barycentric weights w_k, g[20..31] = alpha T e_n, depth slots 13..15
struct FeatureHit {
    static constexpr int kDepthSlot = 13;
    static constexpr bool kHitPoint = true;
    float fg;  // sum_c out_c g_c
    // features at the hit point
    __device__ __forceinline__ void at_hit(const NhtBwdSmem& sm, int j, const NhtBwdRay& st, float px, float py, float pz, float weight,
                                           float (&g)[32]) {
        float wk[4], b[kNhtBase];
        bary_weights(px, py, pz, wk);
        blend(sm.feat[j], wk, b);
        fg = 0.f;
#pragma unroll
        for (int n = 0; n < kNhtBase; ++n) {
            float s, c;
            sincosf(b[n], &s, &c);
            fg += s * st.g[2 * n] + c * st.g[2 * n + 1];
            g[20 + n] = weight * (st.g[2 * n] * c - st.g[2 * n + 1] * s);  // alpha T e_n
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) g[16 + k] = wk[k];
    }
    __device__ __forceinline__ float common(const FrameConfig& cfg, NhtBwdRay& st, float T, float weight, float inv_next, float raw_alpha,
                                            float partial, float (&)[32]) {
        st.FG += weight * fg;
        const float res_g = (st.FiG - st.FG) * inv_next;  // sum_c res_c g_c, no clamp
        float common = partial + T * (fg - res_g);
        if (raw_alpha > cfg.max_alpha) common = 0.f;  // d min(max_alpha, x) / dx = 0
        return common;
    }
    // Pg = sum_k (alpha T h_k) v_k / 12
    __device__ __forceinline__ void hit_point_grad(const NhtBwdSmem& sm, int j, const float (&g)[32], float& pgx, float& pgy, float& pgz) {
        pgx = 0.f; pgy = 0.f; pgz = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            float h = 0.f;
#pragma unroll
            for (int q = 0; q < 3; ++q) {
                const float4 f = sm.feat[j][k * 3 + q];
                h += f.x * g[20 + q * 4] + f.y * g[21 + q * 4] + f.z * g[22 + q * 4] + f.w * g[23 + q * 4];
            }
            pgx += h * kVk12[k][0]; pgy += h * kVk12[k][1]; pgz += h * kVk12[k][2];
        }
    }
};

template <int DEG, bool FAST, bool HALF>
__device__ __forceinline__ void backward_tile_nht(const FrameConfig& cfg, NhtBwdSmem& sm, const Ray& ray, float ofx, float ofy, float ofz, int tid,
                                                  int lane, uint32_t begin, uint32_t end, const float* __restrict__ particles,
                                                  const void* __restrict__ features, const uint32_t* __restrict__ sorted_values,
                                                  const uint32_t* __restrict__ hit_words, bool use_words, bool alive, NhtBwdRay& st,
                                                  float* __restrict__ grad_acc, float* __restrict__ d_features) {
    const float dox = ray.ox - ofx, doy = ray.oy - ofy, doz = ray.oz - ofz;
    const bool depth_grads = __any_sync(kFull, alive && (st.Dgrad != 0.f));
    float (*rows)[33] = sm.rows[tid >> 5];
    // lane l sums feature entry l and, for l < 16, feature entry l + 32, else geometry slot l - 16 (accumulator slots 0..12, 16..18)
    const int fk0 = lane / kNhtBase, fn0 = lane - fk0 * kNhtBase;
    const int o1 = lane + 32, fk1 = o1 / kNhtBase, fn1 = o1 - fk1 * kNhtBase;
    const int gslot = lane - 16, gdst = gslot < 13 ? gslot : gslot + 3;
    backward_batches<FAST>(sm, sm.hw, ofx, ofy, ofz, tid, begin, end, particles, sorted_values, hit_words, use_words, alive,
        [&](uint32_t idx) { sm.idx[tid] = idx; },
        [&](uint32_t base, int count) { stage_features<HALF>(sm.feat, features, sorted_values, base, count, tid); },
        [&](int count) {
        for (int c = 0; c < count; c += 32) {
            if (__all_sync(kFull, !alive)) break;
            const uint32_t* hw = sm.hw + (c >> 5) * kWordsPerChunk + (tid >> 5) * 4;
            unsigned todo = hw[0] | hw[1] | hw[2] | hw[3];
            if (count - c < 32) todo &= (1u << (count - c)) - 1u;
            while (todo) {
                const int j = c + __ffs(todo) - 1;
                todo &= todo - 1;
                float g[32];
#pragma unroll
                for (int i = 0; i < 32; ++i) g[i] = 0.f;
                bool hit = false;
                if (alive) hit = backward_pair<DEG, FAST, FeatureHit>(cfg, sm, j, ray, dox, doy, doz, depth_grads, st, alive, g);
                if (__ballot_sync(kFull, hit)) {
#pragma unroll
                    for (int i = 0; i < 32; ++i) rows[lane][i] = g[i];
                    __syncwarp();
                    float f0 = 0.f, f1 = 0.f;
#pragma unroll 8
                    for (int i = 0; i < 32; ++i) {
                        const float* rw = rows[i];
                        f0 += rw[16 + fk0] * rw[20 + fn0];
                        f1 += lane < 16 ? rw[16 + fk1] * rw[20 + fn1] : rw[gslot];
                    }
                    const size_t p = sm.idx[j];
                    if (f0 != 0.f) atomicAdd(d_features + p * kNhtRow + lane, f0);
                    if (f1 != 0.f) {
                        if (lane < 16) atomicAdd(d_features + p * kNhtRow + o1, f1);
                        else atomicAdd(grad_acc + p * kGradRow + gdst, f1);
                    }
                    __syncwarp();
                    if (__all_sync(kFull, !alive)) break;
                }
            }
        }
    });
}

template <int DEG, bool HALF>
__global__ void __launch_bounds__(kTilePixels) render_backward_nht_kernel(FrameCamera cam, FrameConfig cfg, const float* __restrict__ rays_o,
                                                                          const float* __restrict__ rays_d, const float* __restrict__ particles,
                                                                          const void* __restrict__ features,
                                                                          const uint32_t* __restrict__ sorted_values,
                                                                          const uint32_t* __restrict__ ranges, const uint32_t* __restrict__ tile_order,
                                                                          const uint32_t* __restrict__ chunk_base, const uint32_t* __restrict__ hit_words,
                                                                          const float* __restrict__ out_features_alpha,
                                                                          const float* __restrict__ d_features_alpha, const float* __restrict__ out_dist,
                                                                          const float* __restrict__ d_dist, float* __restrict__ grad_acc,
                                                                          float* __restrict__ d_features) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    NhtBwdSmem& sm = *reinterpret_cast<NhtBwdSmem*>(smem_raw);
    const int tid = threadIdx.x;
    const TileRay tr = tile_ray(cam, rays_o, rays_d, tile_order, tid);
    const int64_t pix = tr.pix;

    NhtBwdRay st;
    st.Tint = 1.f; st.Tgrad = 0.f; st.Dint = 0.f; st.Dgrad = 0.f; st.FiG = 0.f;
    st.T = 1.f; st.D = 0.f; st.FG = 0.f;
#pragma unroll
    for (int c = 0; c < kNhtOut; ++c) st.g[c] = 0.f;
    if (tr.valid) {
        const float* o = out_features_alpha + pix * kNhtChannels;
        const float* d = d_features_alpha + pix * kNhtChannels;
#pragma unroll
        for (int c = 0; c < kNhtOut; ++c) {
            st.g[c] = d[c];
            st.FiG += o[c] * st.g[c];
        }
        st.Tint = 1.f - o[kNhtOut];
        st.Tgrad = -1.f * d[kNhtOut];
        st.Dint = out_dist[pix];
        st.Dgrad = d_dist[pix];
    }

    float ofx, ofy, ofz;
    const bool fast = frame_common_origin(cam, rays_o, tr.inside, pix, ofx, ofy, ofz);
    const uint32_t begin = ranges[tr.tile * 2], end = ranges[tr.tile * 2 + 1];
    const uint32_t* words = hit_words + static_cast<size_t>(chunk_base[tr.tile]) * kWordsPerChunk;
    const bool use_words = (cfg.subtile_culling & 4) != 0;
    if (fast)
        backward_tile_nht<DEG, true, HALF>(cfg, sm, tr.ray, ofx, ofy, ofz, tid, tid & 31, begin, end, particles, features, sorted_values, words, use_words, tr.valid, st, grad_acc, d_features);
    else
        backward_tile_nht<DEG, false, HALF>(cfg, sm, tr.ray, ofx, ofy, ofz, tid, tid & 31, begin, end, particles, features, sorted_values, words, use_words, tr.valid, st, grad_acc, d_features);
}

}  // namespace

void launch_render_forward_nht(cudaStream_t s, const FrameCamera& cam, const FrameConfig& cfg, const float* rays_o, const float* rays_d,
                               const float* particles, const void* features, bool half, const uint32_t* sorted_values, const uint32_t* ranges,
                               const uint32_t* tile_order, const uint32_t* chunk_base, uint32_t* hit_words, float* out_features_alpha,
                               float* out_dist, float* out_hits) {
    const unsigned grid = cam.grid_x * cam.grid_y;
#define GUT_NHT_FWD(DEG_, HALF_) render_forward_nht_kernel<DEG_, HALF_><<<grid, kTilePixels, 0, s>>>(cam, cfg, rays_o, rays_d, particles, features, sorted_values, ranges, tile_order, chunk_base, hit_words, out_features_alpha, out_dist, out_hits)
    if (cfg.kernel_degree == 4) {
        if (half) GUT_NHT_FWD(4, true); else GUT_NHT_FWD(4, false);
    } else {
        if (half) GUT_NHT_FWD(2, true); else GUT_NHT_FWD(2, false);
    }
#undef GUT_NHT_FWD
}

cudaError_t launch_render_backward_nht(cudaStream_t s, const FrameCamera& cam, const FrameConfig& cfg, const float* rays_o, const float* rays_d,
                                       const float* particles, const void* features, bool half, const uint32_t* sorted_values,
                                       const uint32_t* ranges, const uint32_t* tile_order, const uint32_t* chunk_base, const uint32_t* hit_words,
                                       const float* out_features_alpha, const float* d_features_alpha, const float* out_dist, const float* d_dist,
                                       float* grad_acc, float* d_features) {
    const unsigned grid = cam.grid_x * cam.grid_y;
    const int bytes = static_cast<int>(sizeof(NhtBwdSmem));
    cudaError_t e = cudaSuccess;
#define GUT_NHT_BWD(DEG_, HALF_)                                                                                                          \
    do {                                                                                                                                  \
        e = cudaFuncSetAttribute(render_backward_nht_kernel<DEG_, HALF_>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);          \
        if (e != cudaSuccess) return e;                                                                                                   \
        render_backward_nht_kernel<DEG_, HALF_><<<grid, kTilePixels, bytes, s>>>(cam, cfg, rays_o, rays_d, particles, features, sorted_values, \
                                                                                  ranges, tile_order, chunk_base, hit_words, out_features_alpha, \
                                                                                  d_features_alpha, out_dist, d_dist, grad_acc, d_features);   \
    } while (0)
    if (cfg.kernel_degree == 4) {
        if (half) GUT_NHT_BWD(4, true); else GUT_NHT_BWD(4, false);
    } else {
        if (half) GUT_NHT_BWD(2, true); else GUT_NHT_BWD(2, false);
    }
#undef GUT_NHT_BWD
    return cudaGetLastError();
}

}  // namespace gutb200
