// 3dgrut_b200/csrc/mesh_bvh.cuh -- closest-hit queries against the triangle LBVH of the playground meshes (DESIGN.md section 22).
// playground.cu builds the tree with the stages of lbvh.cuh; grt.cu's playground trace and playground.cu's query entry both walk it
// with mesh_closest_hit below.
//
// The triangle test is Moller-Trumbore written with round-to-nearest intrinsics (__fmul_rn, __fadd_rn, ...): they are never contracted
// into FMAs and never replaced by approximations, so the same hit comes out of a --use_fast_math unit (grt.cu) and a plain one
// (playground.cu), and a float32 restatement of the same expression order reproduces it bit for bit.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/grt_b200.h"
#include "lbvh.cuh"

namespace gutb200 {

// What a trace needs of a built mesh BVH (device pointers).  Plain types only: the view crosses translation units.
struct MeshView {
    int ntri;
    const float4* nodes;       // BvhNode records (4 float4 each), ntri - 1 of them (1 for a single triangle)
    const float4* tris;        // [F][3]: v0, e1 = v1 - v0, e2 = v2 - v0 (world space; .w unused)
    const int* faces;          // [F,3] vertex indices
    const float* vnormals;     // [V,3] world-space unit vertex normals
    const int* tri_material;   // [F] row of `materials`
    const float4* materials;   // [M][2]: (kind, ior, 0, 0), (r, g, b, 0)
};

// the device view of a built mesh handle (playground.cu); a null handle is the empty mesh set
MeshView mesh_view(const grtb200_mesh* mesh);

}  // namespace gutb200

namespace {

constexpr float kMeshTMin = 1e-5f;  // TRACE_MESH_TMIN
constexpr float kMeshTMax = 1e5f;   // TRACE_MESH_TMAX
constexpr int kMeshStack = 64;      // the Karras topology is at most 64 levels deep (lbvh.cuh)

struct MeshHit {
    float t, u, v;  // distance along the ray (in units of |d|) and barycentrics of v1, v2
    int tri;        // -1: no hit in (kMeshTMin, kMeshTMax)
};

__device__ __forceinline__ float dot_rn(float ax, float ay, float az, float bx, float by, float bz) {
    return __fadd_rn(__fadd_rn(__fmul_rn(ax, bx), __fmul_rn(ay, by)), __fmul_rn(az, bz));
}

// Moller-Trumbore, both faces: true with (t, u, v) when the ray meets triangle `tri` at t in (kMeshTMin, kMeshTMax)
__device__ __forceinline__ bool tri_intersect(const float4* __restrict__ tris, int tri, float ox, float oy, float oz, float dx, float dy,
                                              float dz, float& t, float& u, float& v) {
    const float4 v0 = __ldg(tris + 3 * tri), e1 = __ldg(tris + 3 * tri + 1), e2 = __ldg(tris + 3 * tri + 2);
    const float px = __fsub_rn(__fmul_rn(dy, e2.z), __fmul_rn(dz, e2.y));
    const float py = __fsub_rn(__fmul_rn(dz, e2.x), __fmul_rn(dx, e2.z));
    const float pz = __fsub_rn(__fmul_rn(dx, e2.y), __fmul_rn(dy, e2.x));
    const float det = dot_rn(e1.x, e1.y, e1.z, px, py, pz);
    if (det == 0.f) return false;
    const float inv = __fdiv_rn(1.f, det);
    const float sx = __fsub_rn(ox, v0.x), sy = __fsub_rn(oy, v0.y), sz = __fsub_rn(oz, v0.z);
    u = __fmul_rn(dot_rn(sx, sy, sz, px, py, pz), inv);
    if (!(u >= 0.f && u <= 1.f)) return false;
    const float qx = __fsub_rn(__fmul_rn(sy, e1.z), __fmul_rn(sz, e1.y));
    const float qy = __fsub_rn(__fmul_rn(sz, e1.x), __fmul_rn(sx, e1.z));
    const float qz = __fsub_rn(__fmul_rn(sx, e1.y), __fmul_rn(sy, e1.x));
    v = __fmul_rn(dot_rn(dx, dy, dz, qx, qy, qz), inv);
    if (!(v >= 0.f && __fadd_rn(u, v) <= 1.f)) return false;
    t = __fmul_rn(dot_rn(e2.x, e2.y, e2.z, qx, qy, qz), inv);
    return t > kMeshTMin && t < kMeshTMax;
}

// The closest triangle hit of one ray (per-thread walk), ties broken by the lowest triangle index.  The box tests are widened by a
// relative 2e-6 (boxes are padded at the build too), so a subtree is skipped only when no triangle in it can be hit at t <= the best t.
__device__ __forceinline__ MeshHit mesh_closest_hit(const gutb200::MeshView& M, float ox, float oy, float oz, float dx, float dy, float dz) {
    MeshHit best{kMeshTMax, 0.f, 0.f, -1};
    if (M.ntri <= 0) return best;
    const float ix = 1.0f / (fabsf(dx) > 1e-20f ? dx : copysignf(1e-20f, dx));
    const float iy = 1.0f / (fabsf(dy) > 1e-20f ? dy : copysignf(1e-20f, dy));
    const float iz = 1.0f / (fabsf(dz) > 1e-20f ? dz : copysignf(1e-20f, dz));
    int stack[kMeshStack];
    int sp = 0;
    stack[sp++] = 0;
    while (sp > 0) {
        const float4* np = M.nodes + 4 * stack[--sp];
        const float4 b0 = __ldg(np), b1 = __ldg(np + 1), b2 = __ldg(np + 2), mt = __ldg(np + 3);
        const float hi = best.t * 1.000002f;
        float a0 = (b0.x - ox) * ix, a1 = (b0.w - ox) * ix;
        float ln = fminf(a0, a1), lf = fmaxf(a0, a1);
        a0 = (b0.y - oy) * iy; a1 = (b1.x - oy) * iy;
        ln = fmaxf(ln, fminf(a0, a1)); lf = fminf(lf, fmaxf(a0, a1));
        a0 = (b0.z - oz) * iz; a1 = (b1.y - oz) * iz;
        ln = fmaxf(ln, fminf(a0, a1)); lf = fminf(lf, fmaxf(a0, a1));
        float rn, rf;
        a0 = (b1.z - ox) * ix; a1 = (b2.y - ox) * ix;
        rn = fminf(a0, a1); rf = fmaxf(a0, a1);
        a0 = (b1.w - oy) * iy; a1 = (b2.z - oy) * iy;
        rn = fmaxf(rn, fminf(a0, a1)); rf = fminf(rf, fmaxf(a0, a1));
        a0 = (b2.x - oz) * iz; a1 = (b2.w - oz) * iz;
        rn = fmaxf(rn, fminf(a0, a1)); rf = fminf(rf, fmaxf(a0, a1));
        const bool lhit = fmaxf(ln, kMeshTMin) <= fminf(lf, hi) * 1.000002f;
        const bool rhit = fmaxf(rn, kMeshTMin) <= fminf(rf, hi) * 1.000002f;
        const int lc = __float_as_int(mt.x), rc = __float_as_int(mt.y);
        int kids[2] = {lc, rc};
        const bool hits[2] = {lhit, rhit};
        // visit the nearer child first: push the far one first
        const int first = (lhit && rhit && ln > rn) ? 0 : 1;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const int c = kids[k ^ first], h = hits[k ^ first];
            if (!h) continue;
            if (c < 0) {
                float t, u, v;
                const int tri = ~c;
                if (tri_intersect(M.tris, tri, ox, oy, oz, dx, dy, dz, t, u, v) && (t < best.t || (t == best.t && tri < best.tri)))
                    best = MeshHit{t, u, v, tri};
            } else if (sp < kMeshStack) {
                stack[sp++] = c;
            }
        }
    }
    return best;
}

}  // namespace
