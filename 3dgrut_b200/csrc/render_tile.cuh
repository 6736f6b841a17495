// 3dgrut_b200/csrc/render_tile.cuh -- per-tile code shared by the 3DGUT compositing kernels (gut_render.cu: radiance,
// gut_render_nht.cu: Neural Harmonic Texture features): rays, kernel response, pixel layout of a tile CTA, common-origin tests, warp
// frames of the sub-tile screens, hit-word lane groups, the kernel prologue, the forward's list walk and the backward's batch loop
// and pair adjoint.
#pragma once
#include "gut_common.cuh"
#include "subtile_cull.cuh"

namespace gutb200 {

namespace {

constexpr unsigned kFull = 0xFFFFFFFFu;
struct Ray {
    float ox, oy, oz, dx, dy, dz, tmin, tmax;
    bool alive;
};

// initializeRay (kernels/cuda/common/rayPayload.cuh:76-108) with the +-1e6 scene box of splatRaster.cpp:240
__device__ __forceinline__ Ray make_ray(const FrameCamera& cam, const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                        int64_t pix) {
    Ray r;
    const float rox = rays_o[pix * 3 + 0], roy = rays_o[pix * 3 + 1], roz = rays_o[pix * 3 + 2];
    const float rdx = rays_d[pix * 3 + 0], rdy = rays_d[pix * 3 + 1], rdz = rays_d[pix * 3 + 2];
    const float* m = cam.s2w;
    r.ox = m[0] * rox + m[3] * roy + m[6] * roz + m[9];
    r.oy = m[1] * rox + m[4] * roy + m[7] * roz + m[10];
    r.oz = m[2] * rox + m[5] * roy + m[8] * roz + m[11];
    r.dx = m[0] * rdx + m[3] * rdy + m[6] * rdz;
    r.dy = m[1] * rdx + m[4] * rdy + m[7] * rdz;
    r.dz = m[2] * rdx + m[5] * rdy + m[8] * rdz;
    const float lo = -1e06f, hi = 1e06f;
    float tmin = (lo - r.ox) / r.dx, tmax = (hi - r.ox) / r.dx, t;
    if (tmin > tmax) { t = tmin; tmin = tmax; tmax = t; }
    float tymin = (lo - r.oy) / r.dy, tymax = (hi - r.oy) / r.dy;
    if (tymin > tymax) { t = tymin; tymin = tymax; tymax = t; }
    bool miss = (tmin > tymax) || (tymin > tmax);
    tmin = fmaxf(tmin, tymin);
    tmax = fminf(tmax, tymax);
    float tzmin = (lo - r.oz) / r.dz, tzmax = (hi - r.oz) / r.dz;
    if (tzmin > tzmax) { t = tzmin; tzmin = tzmax; tzmax = t; }
    miss = miss || (tmin > tzmax) || (tzmin > tmax);
    tmin = fmaxf(tmin, tzmin);
    tmax = fminf(tmax, tzmax);
    r.tmin = miss ? 3.4028235e+38f : fmaxf(tmin, 0.0f);
    r.tmax = miss ? 3.4028235e+38f : tmax;
    r.alive = r.tmax > r.tmin;
    return r;
}

template <int DEG>
__device__ __forceinline__ float kernel_response(float gray) {
    // generalized Gaussian exp(-4.5/3^DEG * |x|^DEG) on the squared canonical distance (gaussianParticles.cuh:267-308)
    if (DEG == 4) return __expf(-0.0555555555556f * gray * gray);
    return __expf(-0.5f * gray);
}

template <int DEG>
__device__ __forceinline__ float kernel_response_grad(float gray, float gres, float gres_grad) {
    if (DEG == 4) return (-0.0555555555556f * 2.0f) * gray * gres * gres_grad;  // gaussianParticles.cuh:239-243
    return -0.5f * gres * gres_grad;                                             // :259-263
}

__device__ __forceinline__ WarpFrame make_warp_frame(const FrameCamera& cam, const Ray& ray, bool alive, bool enabled, int lane) {
    WarpFrame wf;
    wf.on = false;
    const unsigned live = __ballot_sync(kFull, alive);
    if (!enabled || live == 0u) return wf;
    const int src = __ffs(live) - 1;
    float dx = __shfl_sync(kFull, ray.dx, src), dy = __shfl_sync(kFull, ray.dy, src), dz = __shfl_sync(kFull, ray.dz, src);
    if (!frame_axes(cam.s2w, dx, dy, dz, wf)) return wf;
    // this lane's ray in the frame; every live ray must point within 60 degrees of e3
    float u = 0.f, v = 0.f;
    const bool fine = !alive || ray_uv(wf, ray.dx, ray.dy, ray.dz, u, v);
    float ulo = alive ? u : 3.0e38f, uhi = alive ? u : -3.0e38f, vlo = alive ? v : 3.0e38f, vhi = alive ? v : -3.0e38f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        ulo = fminf(ulo, __shfl_xor_sync(kFull, ulo, o));
        uhi = fmaxf(uhi, __shfl_xor_sync(kFull, uhi, o));
        vlo = fminf(vlo, __shfl_xor_sync(kFull, vlo, o));
        vhi = fmaxf(vhi, __shfl_xor_sync(kFull, vhi, o));
    }
    // half a pixel of slack is not needed: the rectangle is the hull of the rays themselves
    wf.ulo = ulo; wf.uhi = uhi; wf.vlo = vlo; wf.vhi = vhi;
    wf.umax = fmaxf(fmaxf(fabsf(ulo), fabsf(uhi)), fmaxf(fabsf(vlo), fabsf(vhi)));
    wf.on = __all_sync(kFull, fine);
    return wf;
}

// pixel of thread `tid` in tile (tx,ty): a warp covers an 8x4 pixel block (not a 16x2 strip) -- hits are spatially
// coherent, so a compact footprint keeps more lanes on the same side of the accept branch
__device__ __forceinline__ void tile_pixel(int tile, int grid_x, int tid, int& px, int& py) {
    const int tx = tile % grid_x, ty = tile / grid_x;
    px = tx * kTile + ((tid >> 5) & 1) * 8 + (tid & 7);
    py = ty * kTile + (tid >> 6) * 4 + ((tid >> 3) & 3);
}

// world-space origin of the tile's first pixel; when every ray of the tile starts there (always the case for the
// camera rays the projection stage assumes) the canonical origin S^-1 R^T (o - mu) is computed once per staged
// particle instead of once per (pixel, particle)
__device__ __forceinline__ bool tile_common_origin(const FrameCamera& cam, const float* __restrict__ rays_o, int tile, bool inside,
                                                   int64_t pix, float& ox, float& oy, float& oz) {
    const int tx = tile % cam.grid_x, ty = tile / cam.grid_x;
    const int64_t pix0 = static_cast<int64_t>(ty * kTile) * cam.width + tx * kTile;
    const float ax = rays_o[pix0 * 3 + 0], ay = rays_o[pix0 * 3 + 1], az = rays_o[pix0 * 3 + 2];
    bool same = true;
    if (inside) same = (rays_o[pix * 3 + 0] == ax) && (rays_o[pix * 3 + 1] == ay) && (rays_o[pix * 3 + 2] == az);
    const float* m = cam.s2w;
    ox = m[0] * ax + m[3] * ay + m[6] * az + m[9];
    oy = m[1] * ax + m[4] * ay + m[7] * az + m[10];
    oz = m[2] * ax + m[5] * ay + m[8] * az + m[11];
    return __syncthreads_and(same);
}

// Lane bits of a warp's 8x4 pixel block: b0..b2 = x, b3..b4 = y (tile_pixel).  Quarter q = b2 | b4 << 1 is a 4x2-pixel block; the
// forward records one hit word per (32-entry chunk, warp, quarter); halves (4x4 pixels, split by b2) and the whole warp OR them.
__device__ __forceinline__ int lane_quarter(int lane) { return ((lane >> 2) & 1) | ((lane >> 3) & 2); }
__device__ __forceinline__ unsigned quarter_lanes(int q) { return (0x0F0Fu << ((q & 1) * 4)) << ((q >> 1) * 16); }
constexpr int kWordsPerChunk = (kTilePixels / 32) * 4;  // 8 warps x 4 quarters
// world-space origin of the frame's first ray; a tile is FAST when every one of its rays starts there (always the case for camera rays)
__device__ __forceinline__ bool frame_common_origin(const FrameCamera& cam, const float* __restrict__ rays_o, bool inside, int64_t pix,
                                                    float& ox, float& oy, float& oz) {
    const float ax = rays_o[0], ay = rays_o[1], az = rays_o[2];
    bool same = true;
    if (inside) same = (rays_o[pix * 3 + 0] == ax) && (rays_o[pix * 3 + 1] == ay) && (rays_o[pix * 3 + 2] == az);
    const float* m = cam.s2w;
    ox = m[0] * ax + m[3] * ay + m[6] * az + m[9];
    oy = m[1] * ax + m[4] * ay + m[7] * az + m[10];
    oz = m[2] * ax + m[5] * ay + m[8] * az + m[11];
    return __syncthreads_and(same);
}

// every thread's pixel and camera ray in the tile of this CTA (the prologue of every compositing kernel)
struct TileRay {
    int tile;
    bool inside, valid;  // pixel inside the image / and its ray meets the scene box
    int64_t pix;
    Ray ray;
};

__device__ __forceinline__ TileRay tile_ray(const FrameCamera& cam, const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                            const uint32_t* __restrict__ tile_order, int tid) {
    TileRay t;
    t.tile = tile_order[blockIdx.x];  // heaviest tiles first (tile_scan_kernel's order): shortens the tail of the grid
    int px, py;
    tile_pixel(t.tile, cam.grid_x, tid, px, py);
    t.inside = (px < cam.width) && (py < cam.height);
    t.pix = static_cast<int64_t>(py) * cam.width + px;
    t.ray.alive = false;
    if (t.inside) t.ray = make_ray(cam, rays_o, rays_d, t.pix);
    t.valid = t.inside && t.ray.alive;
    return t;
}

// rows of quaternionWXYZToMatrix (the columns of R) for q = (w, x, y, z)
__device__ __forceinline__ void rotation_rows(const float4& q, float3& r0, float3& r1, float3& r2) {
    const float r = q.x, x = q.y, y = q.z, z = q.w;
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, xz = x * z, yz = y * z;
    const float rx = r * x, ry = r * y, rz = r * z;
    r0 = make_float3(1.f - 2.f * (yy + zz), 2.f * (xy + rz), 2.f * (xz - ry));
    r1 = make_float3(2.f * (xy - rz), 1.f - 2.f * (xx + zz), 2.f * (yz + rx));
    r2 = make_float3(2.f * (xz + ry), 2.f * (yz - rx), 1.f - 2.f * (xx + yy));
}

// ----------------------------------------------------------------------------------------------------------
// Forward walk, shared by both kinds.  A batch of B list entries is staged as geometry records (below) plus the kind's payload rows;
// the payload (gut_render.cu: radiance, gut_render_nht.cu: features) provides
//   entry(slot, idx)                       stage the row of particle idx (threads with an entry)
//   batch(sorted_values, base, count, tid) stage rows with all threads of the CTA
//   add(j, w, px, py, pz)                  accumulate staged entry j with weight w = alpha T at the canonical hit point p
//
// Staged geometry record: rows of M = diag(1/s) R^T with the canonical tile origin (UNIFORM) or the particle position in .w, then
// (s, density).

template <int B>
struct FwdRecords {
    float4 m0[B], m1[B], m2[B], sd[B];
};

template <bool UNIFORM, int B>
__device__ __forceinline__ void stage_fwd_record(FwdRecords<B>& sm, int slot, const float* __restrict__ particles, uint32_t idx, float o0x,
                                                 float o0y, float o0z) {
    const float4* p4 = reinterpret_cast<const float4*>(particles) + static_cast<size_t>(idx) * 3;
    const float4 a = __ldg(p4), q = __ldg(p4 + 1), s = __ldg(p4 + 2);
    float3 r0, r1, r2;
    rotation_rows(q, r0, r1, r2);
    const float isx = 1.0f / s.x, isy = 1.0f / s.y, isz = 1.0f / s.z;
    float4 m0 = make_float4(isx * r0.x, isx * r0.y, isx * r0.z, a.x);
    float4 m1 = make_float4(isy * r1.x, isy * r1.y, isy * r1.z, a.y);
    float4 m2 = make_float4(isz * r2.x, isz * r2.y, isz * r2.z, a.z);
    if (UNIFORM) {  // .w carries the canonical origin instead of the particle position
        const float vx = o0x - a.x, vy = o0y - a.y, vz = o0z - a.z;
        m0.w = m0.x * vx + m0.y * vy + m0.z * vz;
        m1.w = m1.x * vx + m1.y * vy + m1.z * vz;
        m2.w = m2.x * vx + m2.y * vy + m2.z * vz;
    }
    sm.m0[slot] = m0;
    sm.m1[slot] = m1;
    sm.m2[slot] = m2;
    sm.sd[slot] = make_float4(s.x, s.y, s.z, a.w);
}

// exact test + compositing of one (pixel, staged entry j) pair; returns whether the accept test passed (before the t-range test:
// the reference's backward does not re-apply the range test, DESIGN.md section 5)
template <int DEG, bool UNIFORM, int B, class Payload>
__device__ __forceinline__ bool forward_pair(const FrameConfig& cfg, const FwdRecords<B>& sm, Payload& pay, int j, const Ray& ray, bool& alive,
                                             float& T, float& dist, uint32_t& hits) {
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
                pay.add(j, w, gox + gdx * pd, goy + gdy * pd, goz + gdz * pd);
                hits++;
            }
            if (T < cfg.min_transmittance) alive = false;
        }
    }
    return accept;
}

// Work counters (debug entry point gutb200_debug_work_counters; COUNT instantiations of the radiance forward never run on the product path).
//   0 tests_ref   (pixel, entry) pairs the reference's loop evaluates: every live pixel tests every entry of its tile list
//   1 tests_exec  lane-level exact tests our forward executes after sub-tile culling
//   2 hits        accepted pairs (the set the backward's adjoint runs on)
//   3 fwd_iters   warp iterations of the forward's exact test     4 hit_iters  warp iterations with >= 1 accepting lane (= backward's iterations)
//   5 screens     lane-level sub-tile culling screens             6 bwd_lanes  live lanes summed over hit_iters (lane-level tests of the backward)
//   7 iters16 / 8 iters8   backward iterations when half-warps (4x4 pixels) / quarter-warps (4x2) walk their own entries in lockstep
//   9 sub16_hits / 10 sub8_hits   (half-warp, entry) / (quarter-warp, entry) pairs with >= 1 accepting lane (= gradient rows flushed)
struct WorkCounters {
    unsigned long long v[16];
};

template <int DEG, bool UNIFORM, bool COUNT, int B, class Payload>
__device__ __forceinline__ void forward_tile(const FrameConfig& cfg, FwdRecords<B>& sm, Payload& pay, const WarpFrame& wf, const Ray& ray, float o0x,
                                             float o0y, float o0z, int tid, uint32_t begin, uint32_t end, const float* __restrict__ particles,
                                             const uint32_t* __restrict__ sorted_values, uint32_t* __restrict__ hit_words, bool& alive, float& T,
                                             float& dist, uint32_t& hits, WorkCounters* __restrict__ ctr) {
    const int lane = tid & 31;
    unsigned long long c_ref = 0, c_exec = 0, c_hits = 0, c_iters = 0, c_hit_iters = 0, c_screens = 0, c_bwd_lanes = 0;
    unsigned long long c_iters16 = 0, c_iters8 = 0, c_sub16 = 0, c_sub8 = 0;
    for (uint32_t base = begin; base < end; base += B) {
        if (__syncthreads_and(!alive)) break;
        const int count = min(B, static_cast<int>(end - base));
        const uint32_t k = base + tid;
        if ((B >= kTilePixels || tid < B) && k < end) {  // a batch shorter than the CTA stages on its first B threads
            const uint32_t idx = sorted_values[k];
            stage_fwd_record<UNIFORM>(sm, tid, particles, idx, o0x, o0y, o0z);
            pay.entry(tid, idx);
        }
        pay.batch(sorted_values, base, count, tid);
        __syncthreads();
        // this warp's hit words of the batch: bit e of word c/32 = "some pixel of the warp's 8x4 block accepted entry c + e" -- the backward
        // walks only those entries (a necessary condition of its own exact test, so it drops nothing it would have accepted)
        uint32_t* words = hit_words + (static_cast<size_t>(base - begin) >> 5) * kWordsPerChunk + (tid >> 5) * 4;
        const int quarter = lane_quarter(lane);
        const unsigned my_quarter = quarter_lanes(quarter);
        const bool writer = (lane & 0x0B) == 0;  // lanes 0, 4, 16, 20: one per quarter
        if (UNIFORM) {
            // chunks of 32 entries: lane k screens entry k against the warp's pixel block, the warp walks the survivors
            for (int c = 0; c < count; c += 32) {
                if (!__any_sync(kFull, alive)) break;
                const int e = c + lane;
                bool cand = e < count;
                if (wf.on && cand) {
                    const float4 m0 = sm.m0[e], m1 = sm.m1[e], m2 = sm.m2[e];
                    cand = block_candidate<DEG>(cfg, wf, m0.x, m0.y, m0.z, m1.x, m1.y, m1.z, m2.x, m2.y, m2.z, m0.w, m1.w, m2.w, sm.sd[e].w);
                    if (COUNT) c_screens++;
                }
                unsigned todo = __ballot_sync(kFull, cand);
                uint32_t word = 0;
                int prev = c;
                while (todo) {
                    const int b = __ffs(todo) - 1;
                    const int j = c + b;
                    todo &= todo - 1;
                    int live_n = 0;
                    if (COUNT) {
                        live_n = __popc(__ballot_sync(kFull, alive));
                        c_ref += static_cast<unsigned long long>(live_n) * (j - prev + 1);
                        prev = j + 1;
                        c_iters++;
                        if (alive) c_exec++;
                    }
                    bool acc = false;
                    if (alive) acc = forward_pair<DEG, true>(cfg, sm, pay, j, ray, alive, T, dist, hits);
                    const unsigned accs = __ballot_sync(kFull, acc);
                    if (accs & my_quarter) word |= 1u << b;  // this lane's quarter (4x2 pixels) accepted entry j
                    if (COUNT && accs) {
                        c_hit_iters++;
                        c_bwd_lanes += live_n;
                        c_hits += acc ? 1 : 0;
                    }
                }
                if (COUNT) {
                    const unsigned live = __ballot_sync(kFull, alive);
                    c_ref += static_cast<unsigned long long>(__popc(live)) * (min(c + 32, count) - prev);
                    // lockstep iteration counts of the sub-block walks: halves split by b2, quarters by (b2, b4)
                    const uint32_t wq = word, wh = word | __shfl_xor_sync(kFull, word, 16);
                    const int p16 = __popc(wh), p8 = __popc(wq);
                    const int m16 = max(p16, __shfl_xor_sync(kFull, p16, 4));
                    int m8 = max(p8, __shfl_xor_sync(kFull, p8, 4));
                    m8 = max(m8, __shfl_xor_sync(kFull, m8, 16));
                    c_iters16 += m16;
                    c_iters8 += m8;
                    c_sub16 += p16 + __shfl_xor_sync(kFull, p16, 4);
                    int s8 = p8 + __shfl_xor_sync(kFull, p8, 4);
                    s8 += __shfl_xor_sync(kFull, s8, 16);
                    c_sub8 += s8;
                }
                if (writer) words[(c >> 5) * kWordsPerChunk + quarter] = word;
            }
        } else {
            // per-pixel origins: no warp-level screening; the backward gets all-ones words for these tiles
            if (writer)
                for (int c = 0; c < count; c += 32) words[(c >> 5) * kWordsPerChunk + quarter] = 0xFFFFFFFFu;
            for (int j = 0; alive && j < count; ++j) {
                const bool acc = forward_pair<DEG, false>(cfg, sm, pay, j, ray, alive, T, dist, hits);
                if (COUNT) {
                    c_exec++;
                    c_hits += acc ? 1 : 0;
                }
            }
        }
    }
    if (COUNT) {
        // c_ref, c_iters, c_hit_iters are warp-uniform (lane 0 reports); the others are per lane
        if (!UNIFORM) c_ref = 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            c_exec += __shfl_xor_sync(kFull, c_exec, o);
            c_hits += __shfl_xor_sync(kFull, c_hits, o);
            c_screens += __shfl_xor_sync(kFull, c_screens, o);
        }
        if (lane == 0) {
            if (!UNIFORM) c_ref = c_exec;
            atomicAdd(&ctr->v[0], c_ref);
            atomicAdd(&ctr->v[1], c_exec);
            atomicAdd(&ctr->v[2], c_hits);
            atomicAdd(&ctr->v[3], c_iters);
            atomicAdd(&ctr->v[4], c_hit_iters);
            atomicAdd(&ctr->v[5], c_screens);
            atomicAdd(&ctr->v[6], c_bwd_lanes);
            atomicAdd(&ctr->v[7], c_iters16);
            atomicAdd(&ctr->v[8], c_iters8);
            atomicAdd(&ctr->v[9], c_sub16);
            atomicAdd(&ctr->v[10], c_sub8);
        }
    }
}

// the tile's list walk of a forward kernel: common-origin test, warp frames, then forward_tile on the uniform or per-pixel-origin path
template <int DEG, bool COUNT, int B, class Payload>
__device__ __forceinline__ void forward_list(const FrameCamera& cam, const FrameConfig& cfg, FwdRecords<B>& sm, Payload& pay, const TileRay& tr,
                                             int tid, const float* __restrict__ rays_o, const float* __restrict__ particles,
                                             const uint32_t* __restrict__ sorted_values, const uint32_t* __restrict__ ranges,
                                             const uint32_t* __restrict__ chunk_base, uint32_t* __restrict__ hit_words, float& T, float& dist,
                                             uint32_t& hits, WorkCounters* __restrict__ ctr) {
    float o0x, o0y, o0z;
    const bool uniform = tile_common_origin(cam, rays_o, tr.tile, tr.inside, tr.pix, o0x, o0y, o0z);
    const WarpFrame wf = make_warp_frame(cam, tr.ray, tr.valid, uniform && (cfg.subtile_culling & 2), tid & 31);
    bool alive = tr.valid;
    const uint32_t begin = ranges[tr.tile * 2], end = ranges[tr.tile * 2 + 1];
    uint32_t* words = hit_words + static_cast<size_t>(chunk_base[tr.tile]) * kWordsPerChunk;
    if (uniform)
        forward_tile<DEG, true, COUNT>(cfg, sm, pay, wf, tr.ray, o0x, o0y, o0z, tid, begin, end, particles, sorted_values, words, alive, T, dist, hits, ctr);
    else
        forward_tile<DEG, false, COUNT>(cfg, sm, pay, wf, tr.ray, o0x, o0y, o0z, tid, begin, end, particles, sorted_values, words, alive, T, dist, hits, ctr);
}

// ----------------------------------------------------------------------------------------------------------
// Backward, shared by both kinds.
//
// Staged geometry record: r0, r1, r2 = rows of quaternionWXYZToMatrix (columns of R); .w = canonical frame origin S^-1 R (o_f - mu)
// (FAST) | position (GENERAL); sc = scale.xyz, density; is = 1/scale.xyz, _.
// The rotation rows are kept apart from 1/scale (the forward stages M = S^-1 R^T): the backward's accept test applies 1/s after the
// rotation, as the reference's adjoint does.  With the forward's record the test moves by the last bits, borderline pairs flip, and
// on a 500-Gaussian scene the gradients drifted from 4.7e-4 to 1.8e-3 relative to the CPU restatement of the reference.

template <int B>
struct BwdRecords {
    float4 r0[B], r1[B], r2[B], sc[B], is[B];
};

template <bool FAST, int B>
__device__ __forceinline__ void stage_bwd_record(BwdRecords<B>& sm, int slot, const float* __restrict__ particles, uint32_t idx, float ofx,
                                                 float ofy, float ofz) {
    const float4* p4 = reinterpret_cast<const float4*>(particles) + static_cast<size_t>(idx) * 3;
    const float4 a = __ldg(p4), q = __ldg(p4 + 1), s = __ldg(p4 + 2);
    float3 r0, r1, r2;
    rotation_rows(q, r0, r1, r2);
    float4 t0 = make_float4(r0.x, r0.y, r0.z, a.x);
    float4 t1 = make_float4(r1.x, r1.y, r1.z, a.y);
    float4 t2 = make_float4(r2.x, r2.y, r2.z, a.z);
    if (FAST) {  // .w carries the canonical frame origin instead of the particle position
        const float vx = ofx - a.x, vy = ofy - a.y, vz = ofz - a.z;
        t0.w = (t0.x * vx + t0.y * vy + t0.z * vz) / s.x;
        t1.w = (t1.x * vx + t1.y * vy + t1.z * vz) / s.y;
        t2.w = (t2.x * vx + t2.y * vy + t2.z * vz) / s.z;
    }
    sm.r0[slot] = t0;
    sm.r1[slot] = t1;
    sm.r2[slot] = t2;
    sm.sc[slot] = make_float4(s.x, s.y, s.z, a.w);
    sm.is[slot] = make_float4(1.0f / s.x, 1.0f / s.y, 1.0f / s.z, 0.f);
}

// The batch loop of a backward tile: per batch of B entries, the forward's hit words of the batch into hw[chunk][warp][quarter], the
// geometry records and the kind's rows (entry(idx) on the threads with an entry, batch(base, count) on all), then walk(count).
template <bool FAST, int B, class Entry, class Batch, class Walk>
__device__ __forceinline__ void backward_batches(BwdRecords<B>& sm, uint32_t* hw, float ofx, float ofy, float ofz, int tid, uint32_t begin,
                                                 uint32_t end, const float* __restrict__ particles, const uint32_t* __restrict__ sorted_values,
                                                 const uint32_t* __restrict__ hit_words, bool use_words, const bool& alive, Entry&& entry,
                                                 Batch&& batch, Walk&& walk) {
    constexpr int kWords = (B / 32) * kWordsPerChunk;
    for (uint32_t base = begin; base < end; base += B) {
        if (__syncthreads_and(!alive)) break;
        const int count = min(B, static_cast<int>(end - base));
        if (kWords >= kTilePixels || tid < kWords) {
            const uint32_t chunk = (base - begin) / 32 + (tid >> 5);
            const bool in_list = base + (tid >> 5) * 32 < end;
            hw[tid] = (use_words && in_list) ? hit_words[static_cast<size_t>(chunk) * kWordsPerChunk + (tid & 31)] : 0xFFFFFFFFu;
        }
        const uint32_t k = base + tid;
        if ((B >= kTilePixels || tid < B) && k < end) {  // a batch shorter than the CTA stages on its first B threads
            const uint32_t idx = sorted_values[k];
            stage_bwd_record<FAST>(sm, tid, particles, idx, ofx, ofy, ofz);
            entry(idx);
        }
        batch(base, count);
        __syncthreads();
        walk(count);
    }
}

// Exact test + adjoint of one (pixel, staged entry j) pair (processHitBwd, gaussianParticles.cuh:484-751); fills g[] and returns true
// on a hit.  Everything but what the pair contributes to the ray's payload is the same for both kinds; Kind (a per-pair object) holds
// the rest:
//   kDepthSlot                                  first of the 3 g slots of the depth branch's direct scale part
//   at_hit(sm, j, st, px, py, pz, weight, g)    per-pair payload terms at the canonical hit point p, before the depth branch
//   common(cfg, st, T, weight, inv_next, raw_alpha, partial, g) -> dL/d(alpha) / T, given partial = the depth and opacity parts
//   kHitPoint, hit_point_grad(sm, j, g, pg)     whether the payload depends on p, and dL/dp
template <int DEG, bool FAST, class Kind, class Smem, class St, int NG>
__device__ __forceinline__ bool backward_pair(const FrameConfig& cfg, const Smem& sm, int j, const Ray& ray, float dox, float doy, float doz,
                                              bool depth_grads, St& st, bool& alive, float (&g)[NG]) {
    const float4 r0 = sm.r0[j], r1 = sm.r1[j], r2 = sm.r2[j], sc = sm.sc[j], is = sm.is[j];
    float gox, goy, goz;                                                                          // gro
    if (FAST) {
        gox = r0.w; goy = r1.w; goz = r2.w;
    } else {
        const float pcx = ray.ox - r0.w, pcy = ray.oy - r1.w, pcz = ray.oz - r2.w;                  // gposc
        gox = is.x * (r0.x * pcx + r0.y * pcy + r0.z * pcz);
        goy = is.y * (r1.x * pcx + r1.y * pcy + r1.z * pcz);
        goz = is.z * (r2.x * pcx + r2.y * pcy + r2.z * pcz);
    }
    const float drx = r0.x * ray.dx + r0.y * ray.dy + r0.z * ray.dz;                                // rayDirR
    const float dry = r1.x * ray.dx + r1.y * ray.dy + r1.z * ray.dz;
    const float drz = r2.x * ray.dx + r2.y * ray.dy + r2.z * ray.dz;
    const float ux = is.x * drx, uy = is.y * dry, uz = is.z * drz;                                  // grdu
    const float l = ux * ux + uy * uy + uz * uz;
    const float il = l > 0.f ? rsqrtf(l) : 1.f;
    const float gdx = ux * il, gdy = uy * il, gdz = uz * il;                                        // grd
    const float ccx = gdy * goz - gdz * goy, ccy = gdz * gox - gdx * goz, ccz = gdx * goy - gdy * gox;  // gcrod
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
    Kind kind;
    kind.at_hit(sm, j, st, gox + gdx * pd, goy + gdy * pd, goz + gdz * pd, weight, g);

    // depth branch (:545-580); skipped by warps whose pixels carry no distance gradient (an RGB-only loss)
    float a_hit = 0.f, sd = 0.f, hgx = 0.f, hgy = 0.f, hgz = 0.f, ddx = 0.f, ddy = 0.f, ddz = 0.f;
    if (depth_grads) {
        ddx = gdx * pd; ddy = gdy * pd; ddz = gdz * pd;                                             // grdd
        const float hx = sc.x * ddx, hy = sc.y * ddy, hz = sc.z * ddz;                              // grds
        const float gsq = hx * hx + hy * hy + hz * hz;
        const float gdist = sqrtf(gsq);
        st.D += weight * gdist;
        const float resD = fmaxf((st.Dint - st.D) * inv_next, 0.f);
        a_hit = (gdist - resD) * T * st.Dgrad;
        const float hs = gsq > 0.f ? (weight / gdist) * st.Dgrad : 0.f;
        hgx = hx * hs; hgy = hy * hs; hgz = hz * hs;                                                // grdsRayHitGrd
        sd = hgx * sc.x * gdx + hgy * sc.y * gdy + hgz * sc.z * gdz;                                // grdScaledDot
    }
    // opacity branch (:586-587)
    const float resT = alpha < 0.999999f ? st.Tint / (1.f - alpha) : T;
    const float a_dns = resT * -st.Tgrad;
    const float common = kind.common(cfg, st, T, weight, inv_next, raw_alpha, a_hit + a_dns, g);
    g[3] = gres * common;                                                                           // d density (:624-627)
    const float gray_g = kernel_response_grad<DEG>(gray, gres, dns * common);                       // (:639-648)
    // gray = |grd x gro|^2  (:684-702)
    const float kx = 2.f * ccx * gray_g, ky = 2.f * ccy * gray_g, kz = 2.f * ccz * gray_g;          // gcrodGrd
    float go_gx = ky * gdz - kz * gdy, go_gy = kz * gdx - kx * gdz, go_gz = kx * gdy - ky * gdx;    // groGrd
    float ug_x, ug_y, ug_z;                                                                         // grduGrd
    if (depth_grads) {
        // + grdRayHitGrd = S grdsRayHitGrd pd - gro sd, groRayHitGrd = -grd sd (:560-580), then grd = normalize(grdu) (:729-731): with
        // P = k x grd (the groGrd above) the projection (I - grd grd^T) of grdGrd = gro x k + S hg pd - gro sd is, term by term,
        // pd P,  pd (S hg - grd sd)  and  -sd (gro + pd grd), i.e.  grduGrd = (pd (P + S hg - 2 sd grd) - sd gro) / |grdu|
        const float sd2 = 2.f * sd;
        const float vx = (go_gx + sc.x * hgx) - sd2 * gdx, vy = (go_gy + sc.y * hgy) - sd2 * gdy, vz = (go_gz + sc.z * hgz) - sd2 * gdz;
        ug_x = il * (pd * vx - sd * gox); ug_y = il * (pd * vy - sd * goy); ug_z = il * (pd * vz - sd * goz);
        go_gx -= gdx * sd; go_gy -= gdy * sd; go_gz -= gdz * sd;
        constexpr int D = Kind::kDepthSlot;                                                         // gsclRayHitGrd (:705-713)
        g[D] = ddx * hgx; g[D + 1] = ddy * hgy; g[D + 2] = ddz * hgz;
    } else {  // the same chain in closed form (gut_render.cu, G7 section comment): grduGrd = (pd / |grdu|) groGrd
        const float tq = pd * il;
        ug_x = tq * go_gx; ug_y = tq * go_gy; ug_z = tq * go_gz;
    }
    if constexpr (Kind::kHitPoint) {
        // hit point p = gro + grd pd with dL/dp = pg, s = grd . pg:  groGrd += pg - grd s,  grduGrd += (pd pg - s gro - 2 pd s grd) / |grdu|
        // (the general adjoint of normalize(); the closed form above holds only for the kernel response's own term)
        float pgx, pgy, pgz;
        kind.hit_point_grad(sm, j, g, pgx, pgy, pgz);
        const float s = gdx * pgx + gdy * pgy + gdz * pgz;
        go_gx += pgx - gdx * s; go_gy += pgy - gdy * s; go_gz += pgz - gdz * s;
        const float ps2 = 2.f * pd * s;
        ug_x += il * (pd * pgx - s * gox - ps2 * gdx);
        ug_y += il * (pd * pgy - s * goy - ps2 * gdy);
        ug_z += il * (pd * pgz - s * goz - ps2 * gdz);
    }
    g[0] = go_gx; g[1] = go_gy; g[2] = go_gz;          // canonical: G8 turns the sums into d pos, the gro part of d scale and of d quat
    // W rows: grduGrd_i * d  (+ groGrd_i * (o - o_f) for pixels off the frame origin); G8 scales row i by 1/s_i (rayDirRGrd, gposcrGrd)
    // and contracts it with R for d scale (:733-738) and with the quaternion Jacobian for d quat (matmul_bw_quat, :719-747)
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

}  // namespace

}  // namespace gutb200
