// 3dgrut_b200/csrc/render_tile.cuh -- per-tile ray set-up shared by the 3DGUT compositing kernels (gut_render.cu: radiance,
// gut_render_nht.cu: Neural Harmonic Texture features): rays, kernel response, pixel layout of a tile CTA, common-origin tests, warp
// frames of the sub-tile screens, hit-word lane groups and the per-pixel backward state.
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
// per-pixel backward state (initializeBackwardRay, kernels/cuda/common/rayPayloadBackward.cuh:31-73)
struct BwdRay {
    float Cix, Ciy, Ciz, Cgx, Cgy, Cgz, Tint, Tgrad, Dint, Dgrad;
    float T, Cx, Cy, Cz, D;
};
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

}  // namespace

}  // namespace gutb200
