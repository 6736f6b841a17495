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
// The tile walk, the sub-tile screens and the hit words are those of gut_render.cu; the batch is 128 entries so that the 48-float
// feature rows of a batch (24 KB) are staged on chip next to the geometry records.
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
// forward.  Staged record: rows of M = diag(1/s) R^T with the canonical tile origin (UNIFORM) or the position in .w, (s, density),
// then the feature row.

struct NhtFwdSmem {
    float4 m0[kNhtBatch], m1[kNhtBatch], m2[kNhtBatch], sd[kNhtBatch];
    float4 feat[kNhtBatch][12];
};

template <int DEG, bool UNIFORM>
__device__ __forceinline__ bool forward_pair_nht(const FrameConfig& cfg, const NhtFwdSmem& sm, int j, const Ray& ray, bool& alive, float& T,
                                                 float (&acc)[kNhtOut], float& dist, uint32_t& hits) {
    const float4 m0 = sm.m0[j], m1 = sm.m1[j], m2 = sm.m2[j];
    float gox, goy, goz;
    if (UNIFORM) {
        gox = m0.w; goy = m1.w; goz = m2.w;
    } else {
        const float vx = ray.ox - m0.w, vy = ray.oy - m1.w, vz = ray.oz - m2.w;
        gox = m0.x * vx + m0.y * vy + m0.z * vz;
        goy = m1.x * vx + m1.y * vy + m1.z * vz;
        goz = m2.x * vx + m2.y * vy + m2.z * vz;
    }
    const float ax = m0.x * ray.dx + m0.y * ray.dy + m0.z * ray.dz;
    const float ay = m1.x * ray.dx + m1.y * ray.dy + m1.z * ray.dz;
    const float az = m2.x * ray.dx + m2.y * ray.dy + m2.z * ray.dz;
    const float l = ax * ax + ay * ay + az * az;
    const float il = l > 0.f ? rsqrtf(l) : 1.f;
    const float gdx = ax * il, gdy = ay * il, gdz = az * il;
    const float ccx = gdy * goz - gdz * goy, ccy = gdz * gox - gdx * goz, ccz = gdx * goy - gdy * gox;
    const float gray = ccx * ccx + ccy * ccy + ccz * ccz;
    const float gres = kernel_response<DEG>(gray);
    const float4 sd = sm.sd[j];
    const float alpha = fminf(cfg.max_alpha, gres * sd.w);
    const bool accept = (gres > cfg.min_kernel_density) && (alpha > cfg.min_alpha);
    if (accept) {
        const float pd = -(gdx * gox + gdy * goy + gdz * goz);
        const float hx = sd.x * gdx * pd, hy = sd.y * gdy * pd, hz = sd.z * gdz * pd;
        const float t = sqrtf(hx * hx + hy * hy + hz * hz);
        if ((t > ray.tmin) && (t < ray.tmax)) {
            const float w = alpha * T;
            dist += t * w;
            T *= (1.f - alpha);
            if (w > 0.f) {
                float wk[4], b[kNhtBase];
                bary_weights(gox + gdx * pd, goy + gdy * pd, goz + gdz * pd, wk);
                blend(sm.feat[j], wk, b);
#pragma unroll
                for (int n = 0; n < kNhtBase; ++n) {
                    float s, c;
                    sincosf(b[n], &s, &c);
                    acc[2 * n] += s * w;
                    acc[2 * n + 1] += c * w;
                }
                hits++;
            }
            if (T < cfg.min_transmittance) alive = false;
        }
    }
    return accept;
}

template <int DEG, bool UNIFORM, bool HALF>
__device__ __forceinline__ void forward_tile_nht(const FrameConfig& cfg, NhtFwdSmem& sm, const WarpFrame& wf, const Ray& ray, float o0x, float o0y,
                                                 float o0z, int tid, uint32_t begin, uint32_t end, const float* __restrict__ particles,
                                                 const void* __restrict__ features, const uint32_t* __restrict__ sorted_values,
                                                 uint32_t* __restrict__ hit_words, bool& alive, float& T, float (&acc)[kNhtOut], float& dist,
                                                 uint32_t& hits) {
    const int lane = tid & 31;
    for (uint32_t base = begin; base < end; base += kNhtBatch) {
        if (__syncthreads_and(!alive)) break;
        const int count = min(kNhtBatch, static_cast<int>(end - base));
        if (tid < count) {
            const uint32_t idx = sorted_values[base + tid];
            const float4* p4 = reinterpret_cast<const float4*>(particles) + static_cast<size_t>(idx) * 3;
            const float4 a = __ldg(p4), q = __ldg(p4 + 1), s = __ldg(p4 + 2);
            const float r = q.x, x = q.y, y = q.z, z = q.w;
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, xz = x * z, yz = y * z;
            const float rx = r * x, ry = r * y, rz = r * z;
            const float isx = 1.0f / s.x, isy = 1.0f / s.y, isz = 1.0f / s.z;
            float4 m0 = make_float4(isx * (1.f - 2.f * (yy + zz)), isx * (2.f * (xy + rz)), isx * (2.f * (xz - ry)), a.x);
            float4 m1 = make_float4(isy * (2.f * (xy - rz)), isy * (1.f - 2.f * (xx + zz)), isy * (2.f * (yz + rx)), a.y);
            float4 m2 = make_float4(isz * (2.f * (xz + ry)), isz * (2.f * (yz - rx)), isz * (1.f - 2.f * (xx + yy)), a.z);
            if (UNIFORM) {
                const float vx = o0x - a.x, vy = o0y - a.y, vz = o0z - a.z;
                m0.w = m0.x * vx + m0.y * vy + m0.z * vz;
                m1.w = m1.x * vx + m1.y * vy + m1.z * vz;
                m2.w = m2.x * vx + m2.y * vy + m2.z * vz;
            }
            sm.m0[tid] = m0;
            sm.m1[tid] = m1;
            sm.m2[tid] = m2;
            sm.sd[tid] = make_float4(s.x, s.y, s.z, a.w);
        }
        stage_features<HALF>(sm.feat, features, sorted_values, base, count, tid);
        __syncthreads();
        uint32_t* words = hit_words + (static_cast<size_t>(base - begin) >> 5) * kWordsPerChunk + (tid >> 5) * 4;
        const int quarter = lane_quarter(lane);
        const unsigned my_quarter = quarter_lanes(quarter);
        const bool writer = (lane & 0x0B) == 0;
        if (UNIFORM) {
            for (int c = 0; c < count; c += 32) {
                if (!__any_sync(kFull, alive)) break;
                const int e = c + lane;
                bool cand = e < count;
                if (wf.on && cand) {
                    const float4 m0 = sm.m0[e], m1 = sm.m1[e], m2 = sm.m2[e];
                    cand = block_candidate<DEG>(cfg, wf, m0.x, m0.y, m0.z, m1.x, m1.y, m1.z, m2.x, m2.y, m2.z, m0.w, m1.w, m2.w, sm.sd[e].w);
                }
                unsigned todo = __ballot_sync(kFull, cand);
                uint32_t word = 0;
                while (todo) {
                    const int b = __ffs(todo) - 1;
                    todo &= todo - 1;
                    bool acc_pair = false;
                    if (alive) acc_pair = forward_pair_nht<DEG, true>(cfg, sm, c + b, ray, alive, T, acc, dist, hits);
                    if (__ballot_sync(kFull, acc_pair) & my_quarter) word |= 1u << b;
                }
                if (writer) words[(c >> 5) * kWordsPerChunk + quarter] = word;
            }
        } else {  // per-pixel origins: no screening, all-ones words
            if (writer)
                for (int c = 0; c < count; c += 32) words[(c >> 5) * kWordsPerChunk + quarter] = 0xFFFFFFFFu;
            for (int j = 0; alive && j < count; ++j) forward_pair_nht<DEG, false>(cfg, sm, j, ray, alive, T, acc, dist, hits);
        }
    }
}

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
    const int tile = tile_order[blockIdx.x];
    const int tid = threadIdx.x;
    int px, py;
    tile_pixel(tile, cam.grid_x, tid, px, py);
    const bool inside = (px < cam.width) && (py < cam.height);
    const int64_t pix = static_cast<int64_t>(py) * cam.width + px;

    Ray ray;
    ray.alive = false;
    if (inside) ray = make_ray(cam, rays_o, rays_d, pix);
    const bool valid = inside && ray.alive;
    float o0x, o0y, o0z;
    const bool uniform = tile_common_origin(cam, rays_o, tile, inside, pix, o0x, o0y, o0z);
    const WarpFrame wf = make_warp_frame(cam, ray, valid, uniform && (cfg.subtile_culling & 2), tid & 31);

    float T = 1.f, dist = 0.f, acc[kNhtOut];
#pragma unroll
    for (int c = 0; c < kNhtOut; ++c) acc[c] = 0.f;
    uint32_t hits = 0;
    bool alive = valid;
    const uint32_t begin = ranges[tile * 2], end = ranges[tile * 2 + 1];
    uint32_t* words = hit_words + static_cast<size_t>(chunk_base[tile]) * kWordsPerChunk;
    if (uniform)
        forward_tile_nht<DEG, true, HALF>(cfg, sm, wf, ray, o0x, o0y, o0z, tid, begin, end, particles, features, sorted_values, words, alive, T, acc, dist, hits);
    else
        forward_tile_nht<DEG, false, HALF>(cfg, sm, wf, ray, o0x, o0y, o0z, tid, begin, end, particles, features, sorted_values, words, alive, T, acc, dist, hits);

    if (!inside) return;
    float* o = out_features_alpha + pix * kNhtChannels;
    if (valid) {
#pragma unroll
        for (int c = 0; c < kNhtOut; ++c) o[c] = acc[c];
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

struct NhtBwdSmem {
    float4 r0[kNhtBatch], r1[kNhtBatch], r2[kNhtBatch], sc[kNhtBatch], is[kNhtBatch];
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

template <int DEG, bool FAST>
__device__ __forceinline__ bool backward_pair_nht(const FrameConfig& cfg, const NhtBwdSmem& sm, int j, const Ray& ray, float dox, float doy,
                                                  float doz, bool depth_grads, NhtBwdRay& st, bool& alive, float (&g)[32]) {
    const float4 r0 = sm.r0[j], r1 = sm.r1[j], r2 = sm.r2[j], sc = sm.sc[j], is = sm.is[j];
    float gox, goy, goz;
    if (FAST) {
        gox = r0.w; goy = r1.w; goz = r2.w;
    } else {
        const float pcx = ray.ox - r0.w, pcy = ray.oy - r1.w, pcz = ray.oz - r2.w;
        gox = is.x * (r0.x * pcx + r0.y * pcy + r0.z * pcz);
        goy = is.y * (r1.x * pcx + r1.y * pcy + r1.z * pcz);
        goz = is.z * (r2.x * pcx + r2.y * pcy + r2.z * pcz);
    }
    const float drx = r0.x * ray.dx + r0.y * ray.dy + r0.z * ray.dz;
    const float dry = r1.x * ray.dx + r1.y * ray.dy + r1.z * ray.dz;
    const float drz = r2.x * ray.dx + r2.y * ray.dy + r2.z * ray.dz;
    const float ux = is.x * drx, uy = is.y * dry, uz = is.z * drz;
    const float l = ux * ux + uy * uy + uz * uz;
    const float il = l > 0.f ? rsqrtf(l) : 1.f;
    const float gdx = ux * il, gdy = uy * il, gdz = uz * il;
    const float ccx = gdy * goz - gdz * goy, ccy = gdz * gox - gdx * goz, ccz = gdx * goy - gdy * gox;
    const float gray = ccx * ccx + ccy * ccy + ccz * ccz;
    const float gres = kernel_response<DEG>(gray);
    const float dns = sc.w;
    const float raw_alpha = gres * dns;
    const float alpha = fminf(cfg.max_alpha, raw_alpha);
    if (!((gres > cfg.min_kernel_density) && (alpha > cfg.min_alpha))) return false;

    const float T = st.T;
    const float weight = alpha * T;
    const float nextT = (1.f - alpha) * T;
    const bool last = nextT <= cfg.min_transmittance;
    const float inv_next = last ? 0.f : 1.0f / nextT;
    const float pd = -(gdx * gox + gdy * goy + gdz * goz);

    // features at the hit point
    const float Px = gox + gdx * pd, Py = goy + gdy * pd, Pz = goz + gdz * pd;
    float wk[4], b[kNhtBase];
    bary_weights(Px, Py, Pz, wk);
    blend(sm.feat[j], wk, b);
    float fg = 0.f;  // sum_c out_c g_c
#pragma unroll
    for (int n = 0; n < kNhtBase; ++n) {
        float s, c;
        sincosf(b[n], &s, &c);
        fg += s * st.g[2 * n] + c * st.g[2 * n + 1];
        g[20 + n] = weight * (st.g[2 * n] * c - st.g[2 * n + 1] * s);  // alpha T e_n
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) g[16 + k] = wk[k];

    // depth branch, as in the SH path
    float a_hit = 0.f, sd = 0.f, hgx = 0.f, hgy = 0.f, hgz = 0.f, ddx = 0.f, ddy = 0.f, ddz = 0.f;
    if (depth_grads) {
        ddx = gdx * pd; ddy = gdy * pd; ddz = gdz * pd;
        const float hx = sc.x * ddx, hy = sc.y * ddy, hz = sc.z * ddz;
        const float gsq = hx * hx + hy * hy + hz * hz;
        const float gdist = sqrtf(gsq);
        st.D += weight * gdist;
        const float resD = fmaxf((st.Dint - st.D) * inv_next, 0.f);
        a_hit = (gdist - resD) * T * st.Dgrad;
        const float hs = gsq > 0.f ? (weight / gdist) * st.Dgrad : 0.f;
        hgx = hx * hs; hgy = hy * hs; hgz = hz * hs;
        sd = hgx * sc.x * gdx + hgy * sc.y * gdy + hgz * sc.z * gdz;
    }
    const float resT = alpha < 0.999999f ? st.Tint / (1.f - alpha) : T;
    const float a_dns = resT * -st.Tgrad;
    st.FG += weight * fg;
    const float res_g = (st.FiG - st.FG) * inv_next;  // sum_c res_c g_c, no clamp
    float common = a_hit + a_dns + T * (fg - res_g);
    if (raw_alpha > cfg.max_alpha) common = 0.f;  // d min(max_alpha, x) / dx = 0
    g[3] = gres * common;
    const float gray_g = kernel_response_grad<DEG>(gray, gres, dns * common);
    const float kx = 2.f * ccx * gray_g, ky = 2.f * ccy * gray_g, kz = 2.f * ccz * gray_g;
    float go_gx = ky * gdz - kz * gdy, go_gy = kz * gdx - kx * gdz, go_gz = kx * gdy - ky * gdx;
    float ug_x, ug_y, ug_z;
    if (depth_grads) {
        const float sd2 = 2.f * sd;
        const float vx = (go_gx + sc.x * hgx) - sd2 * gdx, vy = (go_gy + sc.y * hgy) - sd2 * gdy, vz = (go_gz + sc.z * hgz) - sd2 * gdz;
        ug_x = il * (pd * vx - sd * gox); ug_y = il * (pd * vy - sd * goy); ug_z = il * (pd * vz - sd * goz);
        go_gx -= gdx * sd; go_gy -= gdy * sd; go_gz -= gdz * sd;
        g[13] = ddx * hgx; g[14] = ddy * hgy; g[15] = ddz * hgz;
    } else {
        const float tq = pd * il;
        ug_x = tq * go_gx; ug_y = tq * go_gy; ug_z = tq * go_gz;
        g[13] = g[14] = g[15] = 0.f;
    }
    // hit-point term: Pg = sum_k (alpha T h_k) v_k / 12
    float pgx = 0.f, pgy = 0.f, pgz = 0.f;
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
    const float s = gdx * pgx + gdy * pgy + gdz * pgz;
    go_gx += pgx - gdx * s; go_gy += pgy - gdy * s; go_gz += pgz - gdz * s;
    const float ps2 = 2.f * pd * s;
    ug_x += il * (pd * pgx - s * gox - ps2 * gdx);
    ug_y += il * (pd * pgy - s * goy - ps2 * gdy);
    ug_z += il * (pd * pgz - s * goz - ps2 * gdz);

    g[0] = go_gx; g[1] = go_gy; g[2] = go_gz;
    g[4] = ug_x * ray.dx; g[5] = ug_x * ray.dy; g[6] = ug_x * ray.dz;
    g[7] = ug_y * ray.dx; g[8] = ug_y * ray.dy; g[9] = ug_y * ray.dz;
    g[10] = ug_z * ray.dx; g[11] = ug_z * ray.dy; g[12] = ug_z * ray.dz;
    if (!FAST) {
        g[4] += go_gx * dox; g[5] += go_gx * doy; g[6] += go_gx * doz;
        g[7] += go_gy * dox; g[8] += go_gy * doy; g[9] += go_gy * doz;
        g[10] += go_gz * dox; g[11] += go_gz * doy; g[12] += go_gz * doz;
    }
    st.T = nextT;
    if (nextT < cfg.min_transmittance) alive = false;
    return true;
}

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
    for (uint32_t base = begin; base < end; base += kNhtBatch) {
        if (__syncthreads_and(!alive)) break;
        const int count = min(kNhtBatch, static_cast<int>(end - base));
        if (tid < (kNhtBatch / 32) * kWordsPerChunk) {
            const uint32_t chunk = (base - begin) / 32 + (tid >> 5);
            const bool in_list = base + (tid >> 5) * 32 < end;
            sm.hw[tid] = (use_words && in_list) ? hit_words[static_cast<size_t>(chunk) * kWordsPerChunk + (tid & 31)] : 0xFFFFFFFFu;
        }
        if (tid < count) {
            const uint32_t idx = sorted_values[base + tid];
            const float4* p4 = reinterpret_cast<const float4*>(particles) + static_cast<size_t>(idx) * 3;
            const float4 a = __ldg(p4), q = __ldg(p4 + 1), s = __ldg(p4 + 2);
            const float r = q.x, x = q.y, y = q.z, z = q.w;
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, xz = x * z, yz = y * z;
            const float rx = r * x, ry = r * y, rz = r * z;
            float4 t0 = make_float4(1.f - 2.f * (yy + zz), 2.f * (xy + rz), 2.f * (xz - ry), a.x);
            float4 t1 = make_float4(2.f * (xy - rz), 1.f - 2.f * (xx + zz), 2.f * (yz + rx), a.y);
            float4 t2 = make_float4(2.f * (xz + ry), 2.f * (yz - rx), 1.f - 2.f * (xx + yy), a.z);
            if (FAST) {
                const float vx = ofx - a.x, vy = ofy - a.y, vz = ofz - a.z;
                t0.w = (t0.x * vx + t0.y * vy + t0.z * vz) / s.x;
                t1.w = (t1.x * vx + t1.y * vy + t1.z * vz) / s.y;
                t2.w = (t2.x * vx + t2.y * vy + t2.z * vz) / s.z;
            }
            sm.r0[tid] = t0;
            sm.r1[tid] = t1;
            sm.r2[tid] = t2;
            sm.sc[tid] = make_float4(s.x, s.y, s.z, a.w);
            sm.is[tid] = make_float4(1.0f / s.x, 1.0f / s.y, 1.0f / s.z, 0.f);
            sm.idx[tid] = idx;
        }
        stage_features<HALF>(sm.feat, features, sorted_values, base, count, tid);
        __syncthreads();
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
                if (alive) hit = backward_pair_nht<DEG, FAST>(cfg, sm, j, ray, dox, doy, doz, depth_grads, st, alive, g);
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
    }
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
    const int tile = tile_order[blockIdx.x];
    const int tid = threadIdx.x;
    const int lane = tid & 31;
    int px, py;
    tile_pixel(tile, cam.grid_x, tid, px, py);
    const bool inside = (px < cam.width) && (py < cam.height);
    const int64_t pix = static_cast<int64_t>(py) * cam.width + px;

    Ray ray;
    ray.alive = false;
    if (inside) ray = make_ray(cam, rays_o, rays_d, pix);
    const bool alive = inside && ray.alive;

    NhtBwdRay st;
    st.Tint = 1.f; st.Tgrad = 0.f; st.Dint = 0.f; st.Dgrad = 0.f; st.FiG = 0.f;
    st.T = 1.f; st.D = 0.f; st.FG = 0.f;
#pragma unroll
    for (int c = 0; c < kNhtOut; ++c) st.g[c] = 0.f;
    if (alive) {
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
    const bool fast = frame_common_origin(cam, rays_o, inside, pix, ofx, ofy, ofz);
    const uint32_t begin = ranges[tile * 2], end = ranges[tile * 2 + 1];
    const uint32_t* words = hit_words + static_cast<size_t>(chunk_base[tile]) * kWordsPerChunk;
    const bool use_words = (cfg.subtile_culling & 4) != 0;
    if (fast)
        backward_tile_nht<DEG, true, HALF>(cfg, sm, ray, ofx, ofy, ofz, tid, lane, begin, end, particles, features, sorted_values, words, use_words, alive, st, grad_acc, d_features);
    else
        backward_tile_nht<DEG, false, HALF>(cfg, sm, ray, ofx, ofy, ofz, tid, lane, begin, end, particles, features, sorted_values, words, use_words, alive, st, grad_acc, d_features);
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
