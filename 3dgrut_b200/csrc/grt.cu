// 3dgrut_b200/csrc/grt.cu -- native 3DGRT: Morton-code LBVH over per-Gaussian bounding proxies and an ordered
// software ray tracer with volumetric integration and its adjoint.  C ABI: include/grt_b200.h.
//
// The path runs on the SMs (no RT cores are used), so the OptiX instance-AS of the reference (threedgrt_tracer/src/optixTracer.cpp:543-593,799-887)
// and its traversal (src/kernels/cuda/referenceOptix.cu) are replaced by our own kernels:
//   proxy_kernel      per particle: instance transform inverse, world box, conservative radius, scene box (atomics)
//                     <- computeGaussianEnclosingInstancesKernel + kernelScale (src/particlePrimitives.cu:27-51,543-610)
//   morton_kernel     32-bit key = size-class bit + 30-bit Morton code of the proxy centre in the scene box
//   (CUB radix sort of (key, particle) pairs -- library)
//   leaf_kernel       leaves of `leaf` consecutive sorted particles: leaf key, leaf box, proxies stored in leaf order
//   hierarchy_kernel  Karras LBVH topology over the leaves, one thread per internal node
//   refit_kernel      bottom-up boxes, both child boxes stored in the 64-byte parent node (one fetch per visit)
//   trace_kernel<PRIM,DEG,BWD,COUNT,FK>  a warp owns an 8x4 block of rays; per optixTrace-equivalent query the 16 nearest hits are gathered
//                     (t* order -- entry t for icosahedra --, strict comparisons, same bubble insertion as __anyhit__ah) -- coherent blocks walk the tree as a
//                     PACKET (one stack, warp-uniform control flow, per-lane payloads), others one traversal per thread -- then the
//                     hits are integrated / differentiated in order (__raygen__rg of referenceOptix.cu / referenceBwdOptix.cu).
//                     The forward also records each ray's accepted hits;
//   replay_bwd_kernel replays those lists in the backward (no traversal, so one instantiation serves both primitives);
//                     trace_kernel<PRIM,DEG,true> re-traces only overflowed rays.
// Both kernels share one ray prologue (ray_pixel, world_ray), one k-nearest query loop for the forward and one for the re-trace and one hit adjoint
// (backward_hit); the feature kind FK (ShRadiance or NhtFeatures, DESIGN.md section 13; ShRadianceNormals, the SH forward that also sums
// the rays' normals, section 17) supplies only what it accumulates.
// Candidate rule (DESIGN.md section 9), primitive_type instances: the ray segment of the query meets the proxy's oriented box and
// the custom intersection of the reference accepts (intersectInstanceParticle); icosahedron: the ray enters the proxy on the query's
// (tmin, tmax), keyed by the entry t (front-facing triangle hit).  Subtrees entered beyond the current 16th hit are culled, which is
// what OptiX does when the any-hit program shrinks the ray's tmax.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <type_traits>

#include "../../include/grt_b200.h"
#include "hit_math.cuh"
#include "lbvh.cuh"
#include "mesh_bvh.cuh"
#include "nht_features.cuh"

namespace gutb200 {
size_t sort32_temp_bytes(int64_t n);
void run_sort32_pairs(cudaStream_t s, void* temp, size_t temp_bytes, const uint32_t* kin, uint32_t* kout, const uint32_t* vin,
                      uint32_t* vout, int64_t n, int end_bit);
}  // namespace gutb200

using namespace gutb200;

namespace {

constexpr int kK = 16;            // PipelineParameters::MaxNumHitPerTrace
constexpr float kInf = 1e20f;     // RayHit::InfiniteDistance
constexpr uint32_t kNone = 0xFFFFFFFFu;
constexpr float kEpsT = 1e-9f;
constexpr int kStack = 64;
// What a trace integrates: SH radiance (grtb200_trace) or Neural Harmonic Texture features with fp32 / fp16 rows (grtb200_trace_nht);
// kFeatShNormals is the SH radiance forward that also accumulates the ray's normal (grtb200_trace_normals, DESIGN.md section 17).  It
// has no backward of its own: its hit lists and its forward key are those of kFeatSH.
constexpr int kFeatSH = 0, kFeatNht = 1, kFeatNhtHalf = 2, kFeatShNormals = 3;
constexpr int kTraceThreads = 128;  // threads per trace / replay CTA: the NHT per-thread shared rows below are [kNhtOut][128]
#ifndef GRT_BLOCKS_PER_SM
#define GRT_BLOCKS_PER_SM 6
#endif
constexpr int kTraceBlocksPerSm = GRT_BLOCKS_PER_SM;  // 6 -> at most 80 registers, 24 warps per SM (64K registers per SM on sm_90)
// Measured at C4 on an H100 80GB HBM3 (700 W), bench.py --workload c4 --steps 30, two runs each: 4 -> 103.5, 5 -> 110.1, 6 -> 112.0,
// 8 -> 106.9 frames/s.

struct __align__(16) Proxy {  // rows of A^-1 = diag(1/kscl) R^T with the centre in .w
    float4 a0, a1, a2;
};
struct __align__(16) LeafProxy {  // proxy in leaf (sorted) order: 64 B, the particles of one leaf are contiguous
    float4 a0, a1, a2;
    uint32_t pid, pad0, pad1, pad2;
};
// BvhNode, Box, the scene-box reduction, Morton codes, hierarchy_kernel and refit_kernel: lbvh.cuh (shared with gut_knn.cu)

// kernelScale (particlePrimitives.cu:27-51), generalized Gaussian branch
__device__ __forceinline__ float kernel_scale(float density, float min_response, int clamping, float degree) {
    const float modulation = clamping ? density : 1.0f;
    const float minr = fminf(min_response / modulation, 0.97f);
    const float a = -4.5f / powf(3.0f, degree);
    return powf(logf(minr) / a, 1.0f / degree);
}

// primitive_type: icosahedron (computeGaussianEnclosingIcosaHedronKernel, particlePrimitives.cu:435-494).  In the instance space of
// a particle (x = A^-1 (w - mu), the unit cube of `instances`) the proxy is a fixed icosahedron with inradius 1: its vertices are
// (+-1, +-phi, 0) and their cyclic permutations times kIcoVrtScale.  It is centrally symmetric, so it is the intersection of the 10
// slabs |n_k . x| <= 1 whose normals are the dodecahedron directions; kIcoSlab holds n_k * sqrt(3) (so that the slab bound is
// sqrt(3)) and one normal of each antipodal pair.  The CPU tests derive the same table from the reference's faces.
constexpr float kPhi = 1.618033988749895f;
constexpr float kIcoVrtScale = 0.5f * 1.323169076499215f;  // icosaVrtScale: inradius 1
constexpr float kInvPhi = 0.618033988749895f;
constexpr float kSqrt3 = 1.7320508075688772f;
// one vertex of each antipodal pair of the reference's table (vertices 0-5; 6-11 are their negations)
__device__ constexpr float kIcoVrt[6][3] = {{-1.f, kPhi, 0.f}, {1.f, kPhi, 0.f}, {0.f, 1.f, -kPhi}, {-kPhi, 0.f, -1.f}, {-kPhi, 0.f, 1.f},
                                             {0.f, 1.f, kPhi}};
__device__ constexpr float kIcoSlab[10][3] = {{1.f, 1.f, 1.f}, {1.f, 1.f, -1.f}, {1.f, -1.f, 1.f}, {-1.f, 1.f, 1.f},
                                              {0.f, kPhi, kInvPhi}, {0.f, kPhi, -kInvPhi}, {kInvPhi, 0.f, kPhi},
                                              {-kInvPhi, 0.f, kPhi}, {kPhi, kInvPhi, 0.f}, {kPhi, -kInvPhi, 0.f}};

// n . (x, y, z) for a compile-time normal of kIcoSlab: zero terms are left out, +-1 factors fold to adds
__device__ __forceinline__ float slab_dot(const float (&n)[3], float x, float y, float z) {
    if (n[0] == 0.f) return fmaf(n[1], y, n[2] * z);
    if (n[1] == 0.f) return fmaf(n[0], x, n[2] * z);
    if (n[2] == 0.f) return fmaf(n[0], x, n[1] * y);
    return fmaf(n[0], x, fmaf(n[1], y, n[2] * z));
}

// PS, RS, SS, DS: floats between consecutive particles in pos / rot / scl / dns -- 3, 4, 3, 1 for the four separate arrays of
// grtb200_build_bvh, 12 for all four when they point into the [N,12] particle record (grtb200_build_bvh_packed).  Only the loads differ.
template <int PS, int RS, int SS, int DS>
__global__ void __launch_bounds__(256) proxy_kernel(int n, const float* __restrict__ pos, const float* __restrict__ rot,
                                                    const float* __restrict__ scl, const float* __restrict__ dns, float min_response,
                                                    int clamping, float degree, int primitive, Proxy* __restrict__ proxies,
                                                    Box* __restrict__ boxes, int* __restrict__ scene /*[6] ordered ints*/) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float ks = kernel_scale(dns[i * DS], min_response, clamping, degree);
    const float kx = ks * scl[i * SS], ky = ks * scl[i * SS + 1], kz = ks * scl[i * SS + 2];
    const float r = rot[i * RS], x = rot[i * RS + 1], y = rot[i * RS + 2], z = rot[i * RS + 3];
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, xz = x * z, yz = y * z, rx = r * x, ry = r * y, rz = r * z;
    // c0,c1,c2 = columns of R
    const float c0x = 1.f - 2.f * (yy + zz), c0y = 2.f * (xy + rz), c0z = 2.f * (xz - ry);
    const float c1x = 2.f * (xy - rz), c1y = 1.f - 2.f * (xx + zz), c1z = 2.f * (yz + rx);
    const float c2x = 2.f * (xz + ry), c2y = 2.f * (yz - rx), c2z = 1.f - 2.f * (xx + yy);
    const float px = pos[i * PS], py = pos[i * PS + 1], pz = pos[i * PS + 2];
    Proxy p;
    p.a0 = make_float4(c0x / kx, c0y / kx, c0z / kx, px);
    p.a1 = make_float4(c1x / ky, c1y / ky, c1z / ky, py);
    p.a2 = make_float4(c2x / kz, c2y / kz, c2z / kz, pz);
    proxies[i] = p;
    float hx, hy, hz, radius;
    if (primitive == GRTB200_PRIMITIVE_ICOSAHEDRON) {
        // world box of the 12 transformed vertices (the vertices stick out of the unit cube: |y| = phi * kIcoVrtScale = 1.0705);
        // radius = the largest vertex distance from the centre (size class of the Morton key)
        hx = hy = hz = 0.f;
        float r2 = 0.f;
#pragma unroll
        for (int v = 0; v < 6; ++v) {
            const float ex = kIcoVrt[v][0] * kIcoVrtScale * kx, ey = kIcoVrt[v][1] * kIcoVrtScale * ky, ez = kIcoVrt[v][2] * kIcoVrtScale * kz;
            hx = fmaxf(hx, fabsf(c0x * ex + c1x * ey + c2x * ez));
            hy = fmaxf(hy, fabsf(c0y * ex + c1y * ey + c2y * ez));
            hz = fmaxf(hz, fabsf(c0z * ex + c1z * ey + c2z * ez));
            r2 = fmaxf(r2, ex * ex + ey * ey + ez * ez);
        }
        radius = sqrtf(r2);
    } else {
        // world box of the oriented box (== box of its 8 transformed corners, particlePrimitives.cu:566-583)
        hx = fabsf(c0x) * kx + fabsf(c1x) * ky + fabsf(c2x) * kz;
        hy = fabsf(c0y) * kx + fabsf(c1y) * ky + fabsf(c2y) * kz;
        hz = fabsf(c0z) * kx + fabsf(c1z) * ky + fabsf(c2z) * kz;
        radius = sqrtf(kx * kx + ky * ky + kz * kz);
    }
    Box b;
    b.lo = make_float4(px - hx, py - hy, pz - hz, radius);
    b.hi = make_float4(px + hx, py + hy, pz + hz, 0.f);
    boxes[i] = b;
    scene_box_extend(scene, b.lo.x, b.lo.y, b.lo.z, b.hi.x, b.hi.y, b.hi.z);
}

// The two top bits of the key are a size class of the proxy (radius relative to the scene diagonal), so the LBVH splits the particles
// by size first and each class gets its own spatial subtree -- large proxies no longer inflate the boxes of the subtrees that hold
// the many small ones (the crudest form of the "extended Morton code").  Class 0: rel < kSmallProxy, class 1: the rest; a zero scene
// diagonal (rel NaN or infinite) gives class 3.
constexpr float kSmallProxy = 1.f / 48.f;

__global__ void __launch_bounds__(256) morton_kernel(int n, const Proxy* __restrict__ proxies, const Box* __restrict__ boxes,
                                                     const int* __restrict__ scene, uint32_t* __restrict__ codes,
                                                     uint32_t* __restrict__ ids) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const SceneBox sb = scene_box(scene);
    const Proxy p = proxies[i];
    const float diag = sqrtf(sb.ex * sb.ex + sb.ey * sb.ey + sb.ez * sb.ez);
    const float rel = boxes[i].lo.w / diag;   // proxy radius / scene diagonal
    const uint32_t cls = rel < kSmallProxy ? 0u : (rel < 3e38f ? 1u : 3u);
    codes[i] = (cls << 30) | morton30(sb, p.a0.w, p.a1.w, p.a2.w);
    ids[i] = static_cast<uint32_t>(i);
}

// Leaves hold up to `leaf` consecutive particles of the sorted order: one thread per leaf writes the leaf's key (its first particle's),
// its box (union) and the particles' proxies in leaf order.  Fewer, fatter leaves remove the bottom levels of the tree, where most
// node visits happen; the particles of a leaf are tested back to back from one 64*leaf-byte record.
// kLeaf particles per leaf: C4 on an H100 80GB HBM3 (700 W), bench.py --workload c4 --steps 30, two runs each: 1 -> 109.8,
// 2 -> 112.0, 4 -> 108.6, 8 -> 98.9 frames/s
constexpr int kLeaf = 2;
__global__ void __launch_bounds__(256) leaf_kernel(int n, int leaf, const uint32_t* __restrict__ codes_sorted,
                                                   const uint32_t* __restrict__ ids_sorted, const Proxy* __restrict__ proxies,
                                                   const Box* __restrict__ boxes, uint32_t* __restrict__ leaf_codes,
                                                   uint32_t* __restrict__ leaf_ids, Box* __restrict__ leaf_boxes,
                                                   LeafProxy* __restrict__ leaf_proxies) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    const int first = g * leaf;
    if (first >= n) return;
    const int last = min(first + leaf, n);
    Box u;
    u.lo = make_float4(3e38f, 3e38f, 3e38f, 0.f);
    u.hi = make_float4(-3e38f, -3e38f, -3e38f, 0.f);
    for (int k = first; k < last; ++k) {
        const uint32_t pid = ids_sorted[k];
        const Box b = boxes[pid];
        u.lo = make_float4(fminf(u.lo.x, b.lo.x), fminf(u.lo.y, b.lo.y), fminf(u.lo.z, b.lo.z), fmaxf(u.lo.w, b.lo.w));
        u.hi = make_float4(fmaxf(u.hi.x, b.hi.x), fmaxf(u.hi.y, b.hi.y), fmaxf(u.hi.z, b.hi.z), 0.f);
        const Proxy p = proxies[pid];
        LeafProxy q;
        q.a0 = p.a0; q.a1 = p.a1; q.a2 = p.a2;
        q.pid = pid; q.pad0 = q.pad1 = q.pad2 = 0u;
        leaf_proxies[k] = q;
    }
    leaf_codes[g] = codes_sorted[first];
    leaf_ids[g] = static_cast<uint32_t>(g);
    leaf_boxes[g] = u;
}

// one leaf: a root whose left child is the only leaf and whose right child is the point (3e38, 3e38, 3e38), which no ray segment
// reaches.  (An inverted box min > max would not do: the slab test orders each axis' two planes, so it reads as the whole space and
// the leaf's particles were visited, and counted, twice.)
__global__ void single_leaf_kernel(const Box* __restrict__ leaf_boxes, BvhNode* __restrict__ nodes) {
    const Box l = leaf_boxes[0];
    BvhNode nd;
    nd.b0 = make_float4(l.lo.x, l.lo.y, l.lo.z, l.hi.x);
    nd.b1 = make_float4(l.hi.y, l.hi.z, 3e38f, 3e38f);
    nd.b2 = make_float4(3e38f, 3e38f, 3e38f, 3e38f);
    nd.meta = make_float4(__int_as_float(~0), __int_as_float(~0), l.lo.w, 0.f);
    nodes[0] = nd;
}

// ---------------------------------------------------------------------------------------------------------------

struct TraceParams {
    int n, width, height, batch;   // rays are [batch, height, width, 3]
    int sph_degree;
    float min_transmittance, min_response, min_alpha, max_alpha;
    float r2w[12];                 // row-major 3x4
    float scene[6];
    const float* particles;
    const float* sph;              // NHT kinds: the [N,48] feature rows (fp32, or fp16 for kFeatNhtHalf)
    const float* rays_o;
    const float* rays_d;
    const LeafProxy* proxies;      // leaf order
    const BvhNode* nodes;
    int leaf;                      // particles per leaf
    // hit-list cache (ours): the forward records each ray's accepted hits, the backward replays them instead of re-tracing
    uint32_t* hit_list;            // [hit_cap][rays] particle ids (coalesced across the rays of a warp); nullptr = off
    uint32_t* hit_count;           // [rays] number of hits the backward must visit; kNone = more than hit_cap, re-trace this ray
    int hit_cap;
    int64_t rays;
    int only_overflow;             // backward re-trace launch: handle only the rays whose list overflowed
    // forward outputs / backward inputs; NHT kinds: out_rgb / d_rgb are the [R,24] ray features and their gradient, d_sph the
    // [N,48] fp32 feature gradient
    float* out_rgb; float* out_alpha; float* out_dist; float* out_hits; float* visibility;
    const float* d_rgb; const float* d_alpha; const float* d_dist;
    float* d_particles; float* d_sph;
    unsigned long long* counters;  // debug work counters (grtb200_debug_trace_counters); only the COUNT instantiation touches them
    float* out_normals;            // [R,3] accumulated normals; only the kFeatShNormals forward touches them
};

// work counters of one forward trace (lane-level unless noted): 0 rays, 1 k-nearest queries, 2 node visits (one per warp and node in
// packet mode -- the node record is fetched once for the warp -- else one per lane), 3 box tests (lanes that took part in a node visit),
// 4 proxy tests, 5 candidate hits processed, 6 accepted hits, 7 rays walked as packets
struct LaneCounters {
    unsigned long long queries = 0, nodes = 0, boxes = 0, proxies = 0, cands = 0, hits = 0;
};

// one k-nearest query == one optixTrace of the reference: the 16 smallest t* in (tmin, tmax) in ascending order
//
// PACKET = true: the 32 rays of a warp (an 8x4 pixel block of coherent rays) walk the tree TOGETHER -- one traversal stack with
// warp-uniform control flow, a subtree is entered when ANY lane's ray needs it, node records are fetched once per warp (uniform
// address) and every lane keeps its own 16-slot payload and its own cull bound.  Per-ray results are the same as with
// PACKET = false (each lane still tests exactly the leaves its own ray reaches); what changes is that no lane idles while others
// traverse (a per-thread walk leaves most lanes of a warp idle).  Lanes with want == false take part in the votes
// with an empty ray interval.
// proxy test of one leaf for this lane's ray + insertion into the sorted payload
template <int PRIM>
__device__ __forceinline__ void proxy_visit(const LeafProxy* __restrict__ lp, float ox, float oy, float oz, float dx, float dy, float dz,
                                            float tmin, float tmax, float (&kt)[kK], uint32_t (&kid)[kK]) {
    const float4* pp = reinterpret_cast<const float4*>(lp);
    const float4 a0 = __ldg(pp), a1 = __ldg(pp + 1), a2 = __ldg(pp + 2);
    const float vx = ox - a0.w, vy = oy - a1.w, vz = oz - a2.w;
    const float oix = a0.x * vx + a0.y * vy + a0.z * vz, oiy = a1.x * vx + a1.y * vy + a1.z * vz,
                oiz = a2.x * vx + a2.y * vy + a2.z * vz;
    const float dix = a0.x * dx + a0.y * dy + a0.z * dz, diy = a1.x * dx + a1.y * dy + a1.z * dz,
                diz = a2.x * dx + a2.y * dy + a2.z * dz;
    float ht;
    if (PRIM == GRTB200_PRIMITIVE_ICOSAHEDRON) {
        // ray vs the 10 slabs of the icosahedron: entry = the largest slab entry, exit = the smallest slab exit.  The reference
        // reports the front-facing triangle hit (OPTIX_RAY_FLAG_CULL_BACK_FACING_TRIANGLES, referenceOptix.cu:62) with
        // t = optixGetRayTmax(): the entry t of a ray that enters the proxy on (tmin, tmax).  A ray starting inside the proxy
        // (entry <= tmin) only meets back faces and never sees the particle; no closest-approach test applies.
        float tin = -kInf, tout = tmax;
#pragma unroll
        for (int k = 0; k < 10; ++k) {
            const float s = slab_dot(kIcoSlab[k], oix, oiy, oiz), sd = slab_dot(kIcoSlab[k], dix, diy, diz);
            const float q0 = (-kSqrt3 - s) / sd, q1 = (kSqrt3 - s) / sd;
            tin = fmaxf(tin, fminf(q0, q1));
            tout = fminf(tout, fmaxf(q0, q1));
        }
        if (!((tin <= tout) && (tin > tmin) && (tin < tmax))) return;
        ht = tin;
    } else {
        // ray segment vs the unit cube of instance space (the custom primitive's AABB)
        float tin = tmin, tout = tmax, q0, q1;
        q0 = (-1.f - oix) / dix; q1 = (1.f - oix) / dix;
        tin = fmaxf(tin, fminf(q0, q1)); tout = fminf(tout, fmaxf(q0, q1));
        q0 = (-1.f - oiy) / diy; q1 = (1.f - oiy) / diy;
        tin = fmaxf(tin, fminf(q0, q1)); tout = fminf(tout, fmaxf(q0, q1));
        q0 = (-1.f - oiz) / diz; q1 = (1.f - oiz) / diz;
        tin = fmaxf(tin, fminf(q0, q1)); tout = fminf(tout, fmaxf(q0, q1));
        if (!(tin <= tout)) return;
        // intersectInstanceParticle (gaussianParticles.cuh:449-465)
        const float dd = dix * dix + diy * diy + diz * diz;
        const float den = 1.f / dd;
        ht = -(oix * dix + oiy * diy + oiz * diz) * den;
        if (!((ht > tmin) && (ht < tmax))) return;
        const float il = dd > 0.f ? rsqrtf(dd) : 1.f;
        const float n0 = dix * il, n1 = diy * il, n2 = diz * il;
        const float c0 = n1 * oiz - n2 * oiy, c1 = n2 * oix - n0 * oiz, c2 = n0 * oiy - n1 * oix;
        if (!((c0 * c0 + c1 * c1 + c2 * c2) * den < 9.f)) return;
    }
    // __anyhit__ah (referenceOptix.cu:222-248): bubble the hit into the sorted 16-slot payload
    if (ht < kt[kK - 1]) {
        uint32_t hid = __ldg(&lp->pid);
#pragma unroll
        for (int i = 0; i < kK; ++i) {
            if (ht < kt[i]) {
                const float tt = kt[i];
                const uint32_t ti = kid[i];
                kt[i] = ht;
                kid[i] = hid;
                ht = tt;
                hid = ti;
            }
        }
    }
}

// all particles of leaf g for this lane's ray
template <int PRIM, bool COUNT>
__device__ __forceinline__ void leaf_visit(const TraceParams& P, uint32_t g, float ox, float oy, float oz, float dx, float dy, float dz,
                                           float tmin, float tmax, float (&kt)[kK], uint32_t (&kid)[kK], LaneCounters& cc) {
    const int first = static_cast<int>(g) * P.leaf, last = min(first + P.leaf, P.n);
    if (COUNT) cc.proxies += static_cast<unsigned long long>(last - first);
#pragma unroll 1
    for (int k = first; k < last; ++k) proxy_visit<PRIM>(P.proxies + k, ox, oy, oz, dx, dy, dz, tmin, tmax, kt, kid);
}

template <int PRIM, bool PACKET, bool COUNT>
__device__ __forceinline__ void knn_query(const TraceParams& P, bool want, float ox, float oy, float oz, float dx, float dy, float dz,
                                          float idx_, float idy_, float idz_, float tmin, float tmax, float (&kt)[kK], uint32_t (&kid)[kK],
                                          LaneCounters& cc, int* __restrict__ warp_stack) {
    if (COUNT && want) cc.queries++;
#pragma unroll
    for (int i = 0; i < kK; ++i) {
        kt[i] = kInf;
        kid[i] = kNone;
    }
    if (PACKET && !want) {  // empty interval: every slab test of this lane fails
        tmin = 1.f;
        tmax = 0.f;
    }
    // slab planes as one FMA each: t = plane * (1/d) + (-o/d); `slack` covers the rounding difference to (plane - o) / d, so the
    // box test stays a superset of the exact proxy test of the leaves
    const float nox = -ox * idx_, noy = -oy * idy_, noz = -oz * idz_;
    // degenerate axes (|1/d| clamped to 1e20 for axis-parallel rays, trace_rays) are left out: their slab interval is (-huge, +huge) or
    // empty with the right sign, and |-o/d| ~ 1e20 there would inflate the slack until the other axes' tests never reject
    const float slack = 4e-7f * ((fabsf(idx_) < 1e19f ? fabsf(nox) : 0.f) + (fabsf(idy_) < 1e19f ? fabsf(noy) : 0.f) +
                                 (fabsf(idz_) < 1e19f ? fabsf(noz) : 0.f)) + 1e-30f;
    // a packet has ONE traversal stack (warp-uniform control flow): it lives in shared memory, every lane stores the same value to the
    // same word and reads back what it stored; per-thread walks keep a private stack
    int local_stack[PACKET ? 1 : kStack];
    int* stack = PACKET ? warp_stack : local_stack;
    int sp = 0;
    stack[sp++] = 0;
    while (sp > 0) {
        const int ni = stack[--sp];
        if (COUNT) {
            if (PACKET) {
                if ((threadIdx.x & 31) == 0) cc.nodes++;
                if (want) cc.boxes++;
            } else {
                cc.nodes++;
                cc.boxes++;
            }
        }
        const float4* np = reinterpret_cast<const float4*>(P.nodes + ni);
        const float4 b0 = __ldg(np), b1 = __ldg(np + 1), b2 = __ldg(np + 2), mt = __ldg(np + 3);
        const float bound = kt[kK - 1];  // kInf until 16 hits are held
        // slab tests of both children against [tmin, tmax]
        float l0 = fmaf(b0.x, idx_, nox), l1 = fmaf(b0.w, idx_, nox);
        float lt0 = fminf(l0, l1), lt1 = fmaxf(l0, l1);
        l0 = fmaf(b0.y, idy_, noy); l1 = fmaf(b1.x, idy_, noy);
        lt0 = fmaxf(lt0, fminf(l0, l1)); lt1 = fminf(lt1, fmaxf(l0, l1));
        l0 = fmaf(b0.z, idz_, noz); l1 = fmaf(b1.y, idz_, noz);
        lt0 = fmaxf(lt0, fminf(l0, l1)); lt1 = fminf(lt1, fmaxf(l0, l1));
        lt0 = fmaxf(lt0, tmin); lt1 = fminf(lt1, tmax);
        float r0 = fmaf(b1.z, idx_, nox), r1 = fmaf(b2.y, idx_, nox);
        float rt0 = fminf(r0, r1), rt1 = fmaxf(r0, r1);
        r0 = fmaf(b1.w, idy_, noy); r1 = fmaf(b2.z, idy_, noy);
        rt0 = fmaxf(rt0, fminf(r0, r1)); rt1 = fminf(rt1, fmaxf(r0, r1));
        r0 = fmaf(b2.x, idz_, noz); r1 = fmaf(b2.w, idz_, noz);
        rt0 = fmaxf(rt0, fminf(r0, r1)); rt1 = fminf(rt1, fmaxf(r0, r1));
        rt0 = fmaxf(rt0, tmin); rt1 = fminf(rt1, tmax);
        // like OptiX, cull a subtree whose box is entered beyond the current 16th hit (ray tmax shrinks to it)
        const bool lhit = (lt0 <= lt1 + slack) && (lt0 < bound);
        const bool rhit = (rt0 <= rt1 + slack) && (rt0 < bound);
        const int lc = __float_as_int(mt.x), rc = __float_as_int(mt.y);
        bool lpush = lhit && (lc >= 0), rpush = rhit && (rc >= 0);
        if (PACKET) {  // a subtree is entered when ANY lane needs it
            lpush = (lc >= 0) && __any_sync(0xFFFFFFFFu, lhit);
            rpush = (rc >= 0) && __any_sync(0xFFFFFFFFu, rhit);
        }
        if (lpush && rpush) {
            // nearer child on top of the stack; a packet follows the majority of the lanes that need both
            bool left_far = lt0 > rt0;
            if (PACKET) left_far = 2 * __popc(__ballot_sync(0xFFFFFFFFu, lhit && rhit && (lt0 > rt0))) > __popc(__ballot_sync(0xFFFFFFFFu, lhit && rhit));
            if (sp + 1 < kStack) {
                stack[sp] = left_far ? lc : rc;
                stack[sp + 1] = left_far ? rc : lc;
                sp += 2;
            }
        } else if (lpush || rpush) {
            if (sp < kStack) stack[sp++] = lpush ? lc : rc;
        }
        // leaves are tested immediately, by the lanes whose ray reaches them
        if ((lc < 0) && lhit) leaf_visit<PRIM, COUNT>(P, static_cast<uint32_t>(~lc), ox, oy, oz, dx, dy, dz, tmin, tmax, kt, kid, cc);
        if ((rc < 0) && rhit) leaf_visit<PRIM, COUNT>(P, static_cast<uint32_t>(~rc), ox, oy, oz, dx, dy, dz, tmin, tmax, kt, kid, cc);
    }
}

__device__ __forceinline__ void scene_clip(const float* bb, float ox, float oy, float oz, float idx_, float idy_, float idz_, float& t0,
                                           float& t1) {  // intersectAABB (referenceOptix.cu:33-39)
    const float ax = (bb[0] - ox) * idx_, bx = (bb[3] - ox) * idx_;
    const float ay = (bb[1] - oy) * idy_, by = (bb[4] - oy) * idy_;
    const float az = (bb[2] - oz) * idz_, bz = (bb[5] - oz) * idz_;
    t0 = fmaxf(0.f, fmaxf(fminf(ax, bx), fmaxf(fminf(ay, by), fminf(az, bz))));
    t1 = fminf(fmaxf(ax, bx), fminf(fmaxf(ay, by), fmaxf(az, bz)));
}

// The ray of one thread of a trace or replay CTA: a warp covers an 8x4 pixel block of one image (traversal coherence).
struct TraceRay {
    int64_t ray;                   // index into [batch, height, width]
    bool valid;                    // the pixel lies inside the image
    float ox, oy, oz, dx, dy, dz;  // world-space origin and direction
};

// The pixel of this thread; false: the warp lies past the last pixel block (whole warps only).  A lane outside the image takes the ray of
// the nearest pixel inside it, so that the lanes of a packet all take part in its votes; it is not `valid`.
__device__ __forceinline__ bool ray_pixel(const TraceParams& P, TraceRay& r) {
    const int bw = (P.width + 7) / 8, bh = (P.height + 3) / 4;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int per_image = bw * bh;
    if (warp >= per_image * P.batch) return false;
    const int img = warp / per_image, blk = warp % per_image;
    const int px = (blk % bw) * 8 + (lane & 7), py = (blk / bw) * 4 + (lane >> 3);
    r.valid = (px < P.width) && (py < P.height);
    r.ray = (static_cast<int64_t>(img) * P.height + min(py, P.height - 1)) * P.width + min(px, P.width - 1);
    return true;
}

// the world-space ray of r.ray: rayWorldOrigin / rayWorldDirection (pipelineParameters.h:96-114)
__device__ __forceinline__ void world_ray(const TraceParams& P, TraceRay& r) {
    const int64_t ray = r.ray;
    const float rox = P.rays_o[ray * 3], roy = P.rays_o[ray * 3 + 1], roz = P.rays_o[ray * 3 + 2];
    const float rdx = P.rays_d[ray * 3], rdy = P.rays_d[ray * 3 + 1], rdz = P.rays_d[ray * 3 + 2];
    const float* m = P.r2w;
    r.ox = m[0] * rox + m[1] * roy + m[2] * roz + m[3];
    r.oy = m[4] * rox + m[5] * roy + m[6] * roz + m[7];
    r.oz = m[8] * rox + m[9] * roy + m[10] * roz + m[11];
    r.dx = m[0] * rdx + m[1] * rdy + m[2] * rdz;
    r.dy = m[4] * rdx + m[5] * rdy + m[6] * rdz;
    r.dz = m[8] * rdx + m[9] * rdy + m[10] * rdz;
}

// The backward's per-ray values that every kind has: the forward's transmittance and distance, their gradients, and the running
// transmittance and distance of the hits visited so far.
struct RayGrad {
    float Tint, Tgrad, Dint, Dgrad;
    float T = 1.f, D = 0.f;
    __device__ __forceinline__ RayGrad(const TraceParams& P, int64_t ray)
        : Tint(1.0f - P.out_alpha[ray]), Tgrad(-1.0f * P.d_alpha[ray]), Dint(P.out_dist[ray * 2]), Dgrad(P.d_dist[ray]) {}
};

// What a trace integrates.  The walk (trace_rays, replay_bwd_kernel) does not depend on it; a kind supplies
//   forward:  clear() its accumulators; chunk() once per k-nearest query; add() an accepted hit of particle frame f and weight
//             w = alpha T, true when the hit counts and marks its particle visible; store() the ray's output;
//   backward: init() from the forward's output and its gradient; chunk(); adjoint(), its part of the adjoint of an accepted hit, which
//             fills the particle gradient; scatter() its own gradient row of the particle.

// SH radiance (grtb200_trace): sph = the [N,48] coefficients, out_rgb / d_rgb = [R,3].
struct ShRadiance {
    float basis[16];                     // of the ray direction, recomputed per chunk: 16 registers less across the traversal
    float Cx, Cy, Cz;                    // radiance accumulated so far
    float Cix, Ciy, Ciz, Cgx, Cgy, Cgz;  // backward: the forward's radiance and its gradient
    float mr, mg, mb;                    // backward: radiance gradient of the current hit

    __device__ __forceinline__ explicit ShRadiance(float*) {}
    __device__ __forceinline__ void clear() { Cx = Cy = Cz = 0.f; }
    __device__ __forceinline__ void chunk(const TraceParams& P, float dx, float dy, float dz) { sh_basis16(P.sph_degree, dx, dy, dz, basis); }
    __device__ __forceinline__ bool add(const TraceParams& P, uint32_t pid, const ParticleFrame&, const CanonicalHit&, float w) {
        const float4* c4 = reinterpret_cast<const float4*>(P.sph + static_cast<size_t>(pid) * 48);
        float cf[48];
#pragma unroll
        for (int k = 0; k < 12; ++k) {
            const float4 v = __ldg(c4 + k);
            cf[k * 4] = v.x; cf[k * 4 + 1] = v.y; cf[k * 4 + 2] = v.z; cf[k * 4 + 3] = v.w;
        }
        float r = 0.5f, g = 0.5f, b = 0.5f;
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            r += basis[k] * cf[k * 3];
            g += basis[k] * cf[k * 3 + 1];
            b += basis[k] * cf[k * 3 + 2];
        }
        Cx += fmaxf(r, 0.f) * w; Cy += fmaxf(g, 0.f) * w; Cz += fmaxf(b, 0.f) * w;
        return true;
    }
    __device__ __forceinline__ void store(const TraceParams& P, int64_t ray) {
        P.out_rgb[ray * 3] = Cx; P.out_rgb[ray * 3 + 1] = Cy; P.out_rgb[ray * 3 + 2] = Cz;
    }

    __device__ __forceinline__ void init(const TraceParams& P, int64_t ray) {
        Cix = P.out_rgb[ray * 3]; Ciy = P.out_rgb[ray * 3 + 1]; Ciz = P.out_rgb[ray * 3 + 2];
        Cgx = P.d_rgb[ray * 3]; Cgy = P.d_rgb[ray * 3 + 1]; Cgz = P.d_rgb[ray * 3 + 2];
        clear();
    }
    template <int DEG>
    __device__ __forceinline__ void adjoint(const TraceParams& P, uint32_t pid, const ParticleFrame& f, const CanonicalHit& h, float dx, float dy,
                                            float dz, RayGrad& st, float (&gr)[11]) {
        const float4* c4 = reinterpret_cast<const float4*>(P.sph + static_cast<size_t>(pid) * 48);
        float r = 0.5f, g = 0.5f, b = 0.5f;
#pragma unroll
        for (int k = 0; k < 12; ++k) {
            const float4 v = __ldg(c4 + k);
            const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int flat = k * 4 + q, j = flat / 3, c = flat % 3;
                if (c == 0) r += basis[j] * e[q];
                if (c == 1) g += basis[j] * e[q];
                if (c == 2) b += basis[j] * e[q];
            }
        }
        float rg[3];
        hit_adjoint<DEG>(f, h, dx, dy, dz, fmaxf(r, 0.f), fmaxf(g, 0.f), fmaxf(b, 0.f), P.min_transmittance, st.Tint, st.Tgrad, Cix, Ciy,
                         Ciz, Cgx, Cgy, Cgz, st.Dint, st.Dgrad, st.T, Cx, Cy, Cz, st.D, gr, rg);
        // radianceFromSpHBwd<true> (gaussianParticles.cuh:101-177): clamp mask on the unclamped radiance
        mr = r > 0.f ? rg[0] : 0.f; mg = g > 0.f ? rg[1] : 0.f; mb = b > 0.f ? rg[2] : 0.f;
    }
    __device__ __forceinline__ void scatter(const TraceParams& P, uint32_t pid) {
        float4* ds = reinterpret_cast<float4*>(P.d_sph + static_cast<size_t>(pid) * 48);
        const int ncoef = (P.sph_degree + 1) * (P.sph_degree + 1);
#pragma unroll
        for (int k = 0; k < 12; ++k) {
            if (k * 4 < ncoef * 3) {  // the basis is zero beyond the active degree
                float e[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int flat = k * 4 + q, j = flat / 3, c = flat % 3;
                    e[q] = basis[j] * (c == 0 ? mr : (c == 1 ? mg : mb));
                }
                atomicAdd(ds + k, make_float4(e[0], e[1], e[2], e[3]));
            }
        }
    }
};

// SH radiance plus the ray's normal (grtb200_trace_normals): forward only, out_normals = [R,3] unnormalised.  Per accepted hit, as
// processHit accumulates rayNormal (gaussianParticles.cuh:397-401, referenceOptix.cu:103-186), with gro / grd the canonical ray and
// grayDist = |grd x gro|^2 of the accept test:
//   normal += w safe_normalize((gro + grd (dot(grd, -gro) - sqrt(9 - grayDist))) * (R s))
// `*` element-wise and R s = operator*(float33, float3) of the quaternion matrix and the scale (mathUtils.h:450-455): sum_i s_i row_i.
// It is not the ellipsoid's geometric normal; it is what the reference's "normals" view shows.  9 - grayDist < 0 needs a response
// below exp(-4.5), i.e. min_response < 0.0111: there the sqrt is NaN, as in the reference.
struct ShRadianceNormals : ShRadiance {
    float Nx, Ny, Nz;

    __device__ __forceinline__ explicit ShRadianceNormals(float* row) : ShRadiance(row) {}
    __device__ __forceinline__ void clear() {
        ShRadiance::clear();
        Nx = Ny = Nz = 0.f;
    }
    __device__ __forceinline__ bool add(const TraceParams& P, uint32_t pid, const ParticleFrame& f, const CanonicalHit& h, float w) {
        ShRadiance::add(P, pid, f, h, w);
        const float sx = f.r0x * f.sx + f.r1x * f.sy + f.r2x * f.sz;  // particleRotation * particleScale
        const float sy = f.r0y * f.sx + f.r1y * f.sy + f.r2y * f.sz;
        const float sz = f.r0z * f.sx + f.r1z * f.sy + f.r2z * f.sz;
        const float pd = -(h.gdx * h.gox + h.gdy * h.goy + h.gdz * h.goz) - sqrtf(9.0f - h.gray);
        const float vx = (h.gox + h.gdx * pd) * sx, vy = (h.goy + h.gdy * pd) * sy, vz = (h.goz + h.gdz * pd) * sz;
        const float l = vx * vx + vy * vy + vz * vz;
        const float il = l > 0.f ? rsqrtf(l) : 1.f;  // safe_normalize
        Nx += w * (vx * il); Ny += w * (vy * il); Nz += w * (vz * il);
        return true;
    }
    __device__ __forceinline__ void store(const TraceParams& P, int64_t ray) {
        ShRadiance::store(P, ray);
        P.out_normals[ray * 3] = Nx; P.out_normals[ray * 3 + 1] = Ny; P.out_normals[ray * 3 + 2] = Nz;
    }
};

// Neural Harmonic Texture features (grtb200_trace_nht, DESIGN.md section 13) with fp32 or fp16 (HALF) rows: sph = the [N,48] feature
// rows, out_rgb / d_rgb = the [R,24] ray features, d_sph = the [N,48] fp32 feature gradient.  The ray's 24 accumulators (forward) or
// gradients (backward) live in `feat`, this thread's row of the CTA's lane-interleaved [kNhtOut][kTraceThreads] shared array: they do
// not fit next to the 16-slot payload in the 80 registers of a trace thread.
template <bool HALF>
struct NhtFeatures {
    float* feat;
    float FiG, FG;                  // backward: sum_c F_out,c g_c of the ray, and the running sum_c F_acc,c g_c
    float wk[4], e[kNhtBase];       // backward: barycentric weights and alpha T dL/db_n of the current hit

    __device__ __forceinline__ explicit NhtFeatures(float* row) : feat(row) {}
    __device__ __forceinline__ void clear() {
#pragma unroll
        for (int c = 0; c < kNhtOut; ++c) feat[c * kTraceThreads] = 0.f;
    }
    __device__ __forceinline__ void chunk(const TraceParams&, float, float, float) {}
    // the barycentric weights wk of the canonical hit point P = gro + grd pd and the 12 blended base features b there
    // (neuralHarmonicFeaturesParticle.slang); the ray features are out[2n] = sin b_n, out[2n+1] = cos b_n
    __device__ __forceinline__ void hit_features(const TraceParams& P, uint32_t pid, const CanonicalHit& h, float (&b)[kNhtBase]) {
        const float pd = -(h.gdx * h.gox + h.gdy * h.goy + h.gdz * h.goz);
        bary_weights(h.gox + h.gdx * pd, h.goy + h.gdy * pd, h.goz + h.gdz * pd, wk);
        blend_global<HALF>(P.sph, pid, wk, b);
    }
    __device__ __forceinline__ bool add(const TraceParams& P, uint32_t pid, const ParticleFrame&, const CanonicalHit& h, float w) {
        // referenceSlangOptix.cu:144-176: features, hit count and visibility only where the hit weight is > 0
        if (!(w > 0.f)) return false;
        float fb[kNhtBase];
        hit_features(P, pid, h, fb);
#pragma unroll
        for (int n = 0; n < kNhtBase; ++n) {
            float sn, cn;
            sincosf(fb[n], &sn, &cn);
            feat[(2 * n) * kTraceThreads] += sn * w;
            feat[(2 * n + 1) * kTraceThreads] += cn * w;
        }
        return true;
    }
    __device__ __forceinline__ void store(const TraceParams& P, int64_t ray) {
#pragma unroll
        for (int c = 0; c < kNhtOut; ++c) P.out_rgb[ray * kNhtOut + c] = feat[c * kTraceThreads];
    }

    __device__ __forceinline__ void init(const TraceParams& P, int64_t ray) {
        FiG = 0.f;
        FG = 0.f;
#pragma unroll
        for (int c = 0; c < kNhtOut; ++c) {
            const float g = P.d_rgb[ray * kNhtOut + c];
            feat[c * kTraceThreads] = g;
            FiG += P.out_rgb[ray * kNhtOut + c] * g;
        }
    }
    // referenceSlangBwdOptix.cu: particleFeaturesIntegrateBwdToBuffer + particleDensityProcessHitBwdToBuffer
    template <int DEG>
    __device__ __forceinline__ void adjoint(const TraceParams& P, uint32_t pid, const ParticleFrame& f, const CanonicalHit& h, float dx, float dy,
                                            float dz, RayGrad& st, float (&gr)[11]) {
        const float weight = h.alpha * st.T;
        float b[kNhtBase];
        hit_features(P, pid, h, b);
        float fg = 0.f;  // sum_c out_c g_c of this hit
#pragma unroll
        for (int n = 0; n < kNhtBase; ++n) {
            float sn, cn;
            sincosf(b[n], &sn, &cn);
            const float g0 = feat[(2 * n) * kTraceThreads], g1 = feat[(2 * n + 1) * kTraceThreads];
            fg += sn * g0 + cn * g1;
            e[n] = weight * (g0 * cn - g1 * sn);  // alpha T dL/db_n
        }
        float pgx = 0.f, pgy = 0.f, pgz = 0.f;
        point_grad_global<HALF>(P.sph, pid, e, pgx, pgy, pgz);
        hit_adjoint_nht<DEG>(f, h, dx, dy, dz, fg, pgx, pgy, pgz, P.min_transmittance, st.Tint, st.Tgrad, FiG, st.Dint, st.Dgrad, st.T, FG,
                             st.D, gr);
    }
    // d f[12k + n] = w_k alpha T e_n: 12 red.global.add.v4.f32 per hit
    __device__ __forceinline__ void scatter(const TraceParams& P, uint32_t pid) {
        float4* df = reinterpret_cast<float4*>(P.d_sph + static_cast<size_t>(pid) * kNhtRow);
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int q = 0; q < 3; ++q)
                atomicAdd(df + k * 3 + q, make_float4(wk[k] * e[q * 4], wk[k] * e[q * 4 + 1], wk[k] * e[q * 4 + 2], wk[k] * e[q * 4 + 3]));
    }
};

template <int FK>
using Kind = std::conditional_t<FK == kFeatSH, ShRadiance,
                                std::conditional_t<FK == kFeatShNormals, ShRadianceNormals, NhtFeatures<FK == kFeatNhtHalf>>>;

// this thread's feature row (NhtFeatures); nullptr for SH radiance, which keeps its accumulators in registers
template <int FK>
__device__ __forceinline__ float* feature_row() {
    if constexpr (FK == kFeatSH || FK == kFeatShNormals) {
        return nullptr;
    } else {
        __shared__ float s_feat[kNhtOut][kTraceThreads];  // lane-interleaved ([channel][thread]: conflict-free), 12 KB per CTA
        return &s_feat[0][threadIdx.x];
    }
}

// adjoint of one candidate hit of a ray: re-evaluates the accept test, adds the kind's adjoint (processHitBwd) and scatters the gradients
template <int DEG, class K>
__device__ __forceinline__ void backward_hit(const TraceParams& P, uint32_t pid, const TraceRay& r, RayGrad& st, K& kind) {
    const ParticleFrame f = load_frame(P.particles, pid);
    const CanonicalHit h = canonical_hit<DEG>(f, r.ox, r.oy, r.oz, r.dx, r.dy, r.dz, P.min_response, P.min_alpha, P.max_alpha);
    if (!h.accept) return;
    float gr[11];
    kind.template adjoint<DEG>(P, pid, f, h, r.dx, r.dy, r.dz, st, gr);
    // 16-byte vector reductions (red.global.add.v4.f32): 3 + 12 instead of 11 + 48 scalar atomics per hit
    float4* dp = reinterpret_cast<float4*>(P.d_particles + static_cast<size_t>(pid) * 12);
    atomicAdd(dp, make_float4(gr[0], gr[1], gr[2], gr[3]));
    atomicAdd(dp + 1, make_float4(gr[4], gr[5], gr[6], gr[7]));
    atomicAdd(dp + 2, make_float4(gr[8], gr[9], gr[10], 0.f));
    kind.scatter(P, pid);
}

// The forward state of one ray across its k-nearest queries: transmittance, integrated distance, the largest hit distance processed so
// far, the accepted hits counted for the output and, for the hit lists, the accepted hits so far and those of them at distance `last`.
// A playground ray carries it, T above all, from one segment to the next.
struct FwdState {
    float T, D, last, hits;
    uint32_t nrec, nlast;
};

// The forward's walk (one optixTrace of __raygen__rg per iteration) over the hits at t in (s.last + kEpsT, t1 + kEpsT) while T is above
// min_transmittance, integrating every accepted hit into `kind` and `s`.  PACKET: every lane of the warp calls it (`want` false: the lane
// only takes part in the votes).  tix..tiz: the clamped inverse direction of the node slab tests.
template <int PRIM, int DEG, bool PACKET, bool COUNT, int FK>
__device__ __forceinline__ void forward_walk(const TraceParams& P, const TraceRay& r, bool want, float tix, float tiy, float tiz, float t1,
                                             Kind<FK>& kind, FwdState& s, LaneCounters& cc, int* __restrict__ warp_stack) {
    float kt[kK];
    uint32_t kid[kK];
    while (true) {  // one k-nearest query (optixTrace of __raygen__rg) per iteration
        want = want && (s.last <= t1) && (s.T > P.min_transmittance);
        if (PACKET ? !__any_sync(0xFFFFFFFFu, want) : !want) break;
        knn_query<PRIM, PACKET, COUNT>(P, want, r.ox, r.oy, r.oz, r.dx, r.dy, r.dz, tix, tiy, tiz, s.last + kEpsT, t1 + kEpsT, kt, kid, cc, warp_stack);
        if (kid[0] == kNone) want = false;
        if (!want) continue;
        float lt[kK];
        uint32_t li[kK];
#pragma unroll
        for (int i = 0; i < kK; ++i) { lt[i] = kt[i]; li[i] = kid[i]; }
        kind.chunk(P, r.dx, r.dy, r.dz);
#pragma unroll 1
        for (int i = 0; i < kK; ++i) {
            const uint32_t pid = li[i];
            if ((pid == kNone) || !(s.T > P.min_transmittance)) continue;
            const ParticleFrame f = load_frame(P.particles, pid);
            const CanonicalHit h = canonical_hit<DEG>(f, r.ox, r.oy, r.oz, r.dx, r.dy, r.dz, P.min_response, P.min_alpha, P.max_alpha);
            if (COUNT) {
                cc.cands++;
                cc.hits += h.accept ? 1 : 0;
            }
            if (h.accept) {
                const float w = h.alpha * s.T;
                if (kind.add(P, pid, f, h, w)) {
                    s.hits += 1.f;
                    P.visibility[pid] = __int_as_float(1);  // benign race, same value (referenceOptix.cu:158-161)
                }
                s.T *= (1.f - h.alpha);
                s.D += hit_distance(f, h) * w;
                if (P.hit_list && s.nrec < static_cast<uint32_t>(P.hit_cap)) P.hit_list[static_cast<int64_t>(s.nrec) * P.rays + r.ray] = pid;
                s.nrec++;
            }
            if (lt[i] > s.last) {  // hits arrive in ascending t
                s.last = lt[i];
                s.nlast = 0;
            }
            s.nlast += h.accept ? 1u : 0u;
        }
        if (li[kK - 1] == kNone) want = false;  // fewer than 16 hits: the ray is exhausted, the reference's next trace would return nothing
    }
}

// Per-ray work after the rays are set up: the forward (BWD = false; COUNT: the work counters instead of the image) or the re-trace of
// the backward, each one loop of k-nearest queries for every feature kind.  PACKET: the warp's 32 rays traverse together (warp-uniform
// loops, every lane of the warp must call this, `r.valid` marks the lanes that own a ray).  The two loops differ in their interval, stop
// rule and per-candidate work; they are kept as plain loops because routing the candidate work through a shared loop and a lambda cost
// the SH re-trace two more spill slots at the 80-register cap.
template <int PRIM, int DEG, bool BWD, bool PACKET, bool COUNT, int FK>
__device__ __forceinline__ void trace_rays(const TraceParams& P, const TraceRay& r, int* __restrict__ warp_stack, float* __restrict__ feat) {
    LaneCounters cc;
    const float idx_ = 1.0f / r.dx, idy_ = 1.0f / r.dy, idz_ = 1.0f / r.dz;
    // inverse direction for the node slab tests: a zero component (axis-parallel ray) would make the FMA form plane * inf + (-o * inf) a
    // NaN and cull everything; 1e-20 keeps both products finite (|plane|, |o| << 1e18) and the slab interval (-huge, +huge) as it should be
    const float tix = 1.0f / (fabsf(r.dx) > 1e-20f ? r.dx : copysignf(1e-20f, r.dx));
    const float tiy = 1.0f / (fabsf(r.dy) > 1e-20f ? r.dy : copysignf(1e-20f, r.dy));
    const float tiz = 1.0f / (fabsf(r.dz) > 1e-20f ? r.dz : copysignf(1e-20f, r.dz));

    float t0, t1;
    scene_clip(P.scene, r.ox, r.oy, r.oz, idx_, idy_, idz_, t0, t1);

    Kind<FK> kind(feat);
    bool want = r.valid && (P.n > 0);
    if constexpr (!BWD) {
        FwdState s{1.f, 0.f, fmaxf(0.f, t0 - kEpsT), 0.f, 0u, 0u};
        kind.clear();
        forward_walk<PRIM, DEG, PACKET, COUNT, FK>(P, r, want, tix, tiy, tiz, t1, kind, s, cc, warp_stack);
        const float T = s.T, D = s.D, last = s.last, hits = s.hits;
        const uint32_t nrec = s.nrec, nlast = s.nlast;
        if (COUNT) {
            unsigned long long v[8] = {r.valid ? 1ull : 0ull, cc.queries, cc.nodes, cc.boxes, cc.proxies, cc.cands, cc.hits, (PACKET && r.valid) ? 1ull : 0ull};
#pragma unroll
            for (int k = 0; k < 8; ++k) {
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xFFFFFFFFu, v[k], o);
                if ((threadIdx.x & 31) == 0 && v[k]) atomicAdd(&P.counters[k], v[k]);
            }
            return;  // the counting pass writes no image
        }
        if (r.valid) {
            const int64_t ray = r.ray;
            kind.store(P, ray);
            P.out_alpha[ray] = 1.f - T;
            P.out_dist[ray * 2] = D;
            P.out_dist[ray * 2 + 1] = last;
            P.out_hits[ray] = hits;
            // the backward's re-trace ends before fminf(last, t1) + kEpsT (referenceBwdOptix.cu:115,125): strictly before the last
            // processed hit distance while kEpsT is below half an ulp of it, so the accepted hits AT that distance are not replayed
            // either -- several of them when particles coincide (fresh clones).  Closer than ~0.0168 the sum rounds up past `last`
            // and the re-trace does visit them (rays starting inside the cloud); the replay must too.
            const bool drop_last = !(last < fminf(last, t1) + kEpsT);
            if (P.hit_count) P.hit_count[ray] = nrec > static_cast<uint32_t>(P.hit_cap) ? kNone : nrec - (drop_last ? nlast : 0u);
        }
    } else {  // referenceBwdOptix.cu / referenceSlangBwdOptix.cu:103-230
        kind.init(P, r.ray);
        RayGrad st(P, r.ray);
        float start = fmaxf(0.f, t0 - kEpsT);
        const float end = fminf(P.out_dist[r.ray * 2 + 1], t1) + kEpsT;
        if (P.only_overflow && want) want = P.hit_count[r.ray] == kNone;
        float kt[kK];
        uint32_t kid[kK];
        while (true) {
            want = want && (start < end);
            if (PACKET ? !__any_sync(0xFFFFFFFFu, want) : !want) break;
            knn_query<PRIM, PACKET, COUNT>(P, want, r.ox, r.oy, r.oz, r.dx, r.dy, r.dz, tix, tiy, tiz, start + kEpsT, end, kt, kid, cc, warp_stack);
            if (kid[0] == kNone) want = false;
            if (!want) continue;
            float lt[kK];
            uint32_t li[kK];
#pragma unroll
            for (int i = 0; i < kK; ++i) { lt[i] = kt[i]; li[i] = kid[i]; }
            kind.chunk(P, r.dx, r.dy, r.dz);
#pragma unroll 1
            for (int i = 0; i < kK; ++i) {
                const uint32_t pid = li[i];
                if (pid == kNone) continue;
                backward_hit<DEG>(P, pid, r, st, kind);
                start = fmaxf(start, lt[i]);
            }
            if (li[kK - 1] == kNone) want = false;
        }
    }
}

// packet traversal pays when the warp's rays are coherent: directions within ~6 degrees of lane 0's and origins within 2 % of the scene
// diagonal; otherwise every thread walks the tree on its own.  Every lane of the warp calls this.
__device__ __forceinline__ bool coherent_warp(const TraceParams& P, const TraceRay& r) {
    const float dx = r.dx, dy = r.dy, dz = r.dz, ox = r.ox, oy = r.oy, oz = r.oz;
    const float fx = __shfl_sync(0xFFFFFFFFu, dx, 0), fy = __shfl_sync(0xFFFFFFFFu, dy, 0), fz = __shfl_sync(0xFFFFFFFFu, dz, 0);
    const float gx = __shfl_sync(0xFFFFFFFFu, ox, 0), gy = __shfl_sync(0xFFFFFFFFu, oy, 0), gz = __shfl_sync(0xFFFFFFFFu, oz, 0);
    const float dot = dx * fx + dy * fy + dz * fz, n1 = dx * dx + dy * dy + dz * dz, n0 = fx * fx + fy * fy + fz * fz;
    const float ex = P.scene[3] - P.scene[0], ey = P.scene[4] - P.scene[1], ez = P.scene[5] - P.scene[2];
    const float sx = ox - gx, sy = oy - gy, sz = oz - gz;
    const bool near_first = (dot > 0.f) && (dot * dot > 0.99f * n1 * n0) && (sx * sx + sy * sy + sz * sz <= 4e-4f * (ex * ex + ey * ey + ez * ez));
    return __all_sync(0xFFFFFFFFu, near_first);
}

template <int PRIM, int DEG, bool BWD, bool COUNT, int FK>
__global__ void __launch_bounds__(128, kTraceBlocksPerSm) trace_kernel(TraceParams P) {
    __shared__ int s_stack[4][kStack];  // one traversal stack per warp (packet walks)
    float* feat = feature_row<FK>();
    TraceRay r;
    if (!ray_pixel(P, r)) return;
    world_ray(P, r);
    int* warp_stack = s_stack[threadIdx.x >> 5];
    if (coherent_warp(P, r)) {
        trace_rays<PRIM, DEG, BWD, true, COUNT, FK>(P, r, warp_stack, feat);
    } else if (COUNT || r.valid) {   // the counting pass ends in warp shuffles: every lane takes part
        trace_rays<PRIM, DEG, BWD, false, COUNT, FK>(P, r, warp_stack, feat);
    }
}

// Backward from the hit lists the forward recorded: no traversal, one thread per ray, list reads coalesced across the warp.
// Rays whose list overflowed (hit_count == kNone) are left to the re-trace launch that follows.
template <int DEG, int FK>
__global__ void __launch_bounds__(128) replay_bwd_kernel(TraceParams P) {
    TraceRay r;
    if (!ray_pixel(P, r) || !r.valid) return;
    const uint32_t count = P.hit_count[r.ray];
    if (count == kNone || count == 0u) return;
    world_ray(P, r);
    Kind<FK> kind(feature_row<FK>());
    kind.chunk(P, r.dx, r.dy, r.dz);
    RayGrad st(P, r.ray);
    kind.init(P, r.ray);
#pragma unroll 1
    for (uint32_t i = 0; i < count; ++i) backward_hit<DEG>(P, P.hit_list[static_cast<int64_t>(i) * P.rays + r.ray], r, st, kind);
}

// ---- playground: meshes inside the scene (grtb200_trace_playground, DESIGN.md section 22) ----------------------------------------------
// The constants of the reference's playgroundKernel.cu / handleGlass.
constexpr int kMaxBounces = 32;          // MAX_BOUNCES: mirror reflections (and total internal reflections)
constexpr int kMaxSegments = 1000;       // TIMEOUT_ITERATIONS
constexpr float kRefractShift = 1e-5f;   // REFRACTION_EPS_SHIFT
constexpr float kOutsideIor = 1.0003f;   // n1
constexpr float kStopAlpha = 0.995f;
constexpr float kBounceTMin = 1e-9f;     // tmin of a Gaussian segment after a bounce
constexpr float kRayMaxT = 1e9f;         // ray_max_t where the caller gives none

struct PlaygroundParams {
    TraceParams P;                 // the Gaussians, rays and options of grtb200_trace (SH radiance)
    gutb200::MeshView mesh;
    const float* ray_max_t;        // [R] or nullptr (kRayMaxT)
    float bg[3];
    int smooth;                    // interpolated vertex normals, else the triangle's own
};

// The Gaussians of ray r on (a, b) inside the scene box: the forward walk of grtb200_trace, starting from the state s (T and the radiance
// in `kind` carried from the segments before).  With a = 0 and b past the scene box this is grtb200_trace's walk exactly.
template <int PRIM, int DEG, bool PACKET>
__device__ __forceinline__ void gaussian_segment(const TraceParams& P, const TraceRay& r, bool want, float a, float b, ShRadiance& kind,
                                                 FwdState& s, int* __restrict__ warp_stack) {
    const float idx_ = 1.0f / r.dx, idy_ = 1.0f / r.dy, idz_ = 1.0f / r.dz;
    const float tix = 1.0f / (fabsf(r.dx) > 1e-20f ? r.dx : copysignf(1e-20f, r.dx));
    const float tiy = 1.0f / (fabsf(r.dy) > 1e-20f ? r.dy : copysignf(1e-20f, r.dy));
    const float tiz = 1.0f / (fabsf(r.dz) > 1e-20f ? r.dz : copysignf(1e-20f, r.dz));
    float t0, t1;
    scene_clip(P.scene, r.ox, r.oy, r.oz, idx_, idy_, idz_, t0, t1);
    t0 = fmaxf(t0, a);
    t1 = fminf(t1, b);
    s.last = fmaxf(0.f, t0 - kEpsT);
    LaneCounters cc;
    forward_walk<PRIM, DEG, PACKET, false, kFeatSH>(P, r, want && (P.n > 0), tix, tiy, tiz, t1, kind, s, cc, warp_stack);
}

__device__ __forceinline__ void normalize3(float& x, float& y, float& z) {
    const float l2 = x * x + y * y + z * z;
    const float il = l2 > 0.f ? rsqrtf(l2) : 1.f;  // safe_normalize
    x *= il; y *= il; z *= il;
}

// the unit normal at hit h: normalize(cross(e1, e2)), or the vertex normals interpolated with the barycentrics (1 - u - v, u, v)
__device__ __forceinline__ void hit_normal(const PlaygroundParams& G, const MeshHit& h, float& nx, float& ny, float& nz) {
    if (G.smooth) {
        const int a = G.mesh.faces[3 * h.tri], b = G.mesh.faces[3 * h.tri + 1], c = G.mesh.faces[3 * h.tri + 2];
        const float w = 1.f - h.u - h.v;
        const float* vn = G.mesh.vnormals;
        nx = w * vn[3 * a] + h.u * vn[3 * b] + h.v * vn[3 * c];
        ny = w * vn[3 * a + 1] + h.u * vn[3 * b + 1] + h.v * vn[3 * c + 1];
        nz = w * vn[3 * a + 2] + h.u * vn[3 * b + 2] + h.v * vn[3 * c + 2];
    } else {
        const float4 e1 = G.mesh.tris[3 * h.tri + 1], e2 = G.mesh.tris[3 * h.tri + 2];
        nx = e1.y * e2.z - e1.z * e2.y;
        ny = e1.z * e2.x - e1.x * e2.z;
        nz = e1.x * e2.y - e1.y * e2.x;
    }
    normalize3(nx, ny, nz);
}

// One ray: the first segment as grtb200_trace walks it (as a packet when the warp is coherent), then per thread a closest mesh hit, the
// material's bounce and the Gaussians of the next segment, until the ray leaves every mesh, meets a diffuse surface, reaches alpha 0.995,
// 32 bounces or 1000 segments.  One transmittance T is carried through all of it: mirror and glass are lossless, a diffuse hit adds
// T c |dot(d, n)| and makes the ray opaque.
template <int PRIM, int DEG>
__global__ void __launch_bounds__(128) playground_kernel(PlaygroundParams G, float* __restrict__ out_rgb, float* __restrict__ out_alpha) {
    __shared__ int s_stack[4][kStack];
    const TraceParams& P = G.P;
    TraceRay r;
    if (!ray_pixel(P, r)) return;
    world_ray(P, r);
    int* warp_stack = s_stack[threadIdx.x >> 5];
    const float tmax = G.ray_max_t ? G.ray_max_t[r.ray] : kRayMaxT;
    MeshHit h = mesh_closest_hit(G.mesh, r.ox, r.oy, r.oz, r.dx, r.dy, r.dz);
    ShRadiance kind(nullptr);
    kind.clear();
    FwdState s{1.f, 0.f, 0.f, 0.f, 0u, 0u};
    const float end0 = h.tri >= 0 ? h.t : tmax;
    if (coherent_warp(P, r))
        gaussian_segment<PRIM, DEG, true>(P, r, r.valid, 0.f, end0, kind, s, warp_stack);
    else if (r.valid)
        gaussian_segment<PRIM, DEG, false>(P, r, true, 0.f, end0, kind, s, warp_stack);
    if (!r.valid) return;
    int bounces = 0, segments = 1;
#pragma unroll 1
    while (h.tri >= 0) {
        const int m = G.mesh.tri_material[h.tri];
        const float4 mk = G.mesh.materials[2 * m], mc = G.mesh.materials[2 * m + 1];
        const int kind_m = static_cast<int>(mk.x);
        float nx, ny, nz;
        hit_normal(G, h, nx, ny, nz);
        float dx = r.dx, dy = r.dy, dz = r.dz;
        normalize3(dx, dy, dz);
        const float dn = dx * nx + dy * ny + dz * nz;
        if (kind_m == GRTB200_MATERIAL_DIFFUSE) {  // get_diffuse_color without a texture: opaque, ends the ray
            const float shade = fabsf(dn);
            kind.Cx += s.T * mc.x * shade;
            kind.Cy += s.T * mc.y * shade;
            kind.Cz += s.T * mc.z * shade;
            s.T = 0.f;
            break;
        }
        // the normal turned against the ray: the front face when dot(d, n) < 0
        const float sg = dn < 0.f ? 1.f : -1.f;
        const float fx = sg * nx, fy = sg * ny, fz = sg * nz;
        const float cos_i = -(dx * fx + dy * fy + dz * fz);  // >= 0
        float t = h.t;
        float ex, ey, ez;
        bool reflect = kind_m == GRTB200_MATERIAL_MIRROR;
        if (!reflect) {  // glass: Snell refraction, n1 outside, the mesh's ior inside (refract / handleGlass)
            const float eta = mk.y / kOutsideIor;
            const float ri = dn < 0.f ? 1.f / eta : eta;
            const float ct = fminf(cos_i, 1.f);
            const float st = sqrtf(fmaxf(0.f, 1.f - ct * ct));
            if (ri * st <= 1.f) {
                const float px = ri * (dx + ct * fx), py = ri * (dy + ct * fy), pz = ri * (dz + ct * fz);
                const float q = -sqrtf(fabsf(1.f - (px * px + py * py + pz * pz)));
                ex = px + q * fx; ey = py + q * fy; ez = pz + q * fz;
                normalize3(ex, ey, ez);
                t += kRefractShift;
            } else {
                reflect = true;  // total internal reflection
            }
        }
        if (reflect) {  // handleMirror: d - 2 dot(d, n) n about the turned normal
            ex = dx + 2.f * cos_i * fx; ey = dy + 2.f * cos_i * fy; ez = dz + 2.f * cos_i * fz;
            normalize3(ex, ey, ez);
            ++bounces;
        }
        r.ox += t * r.dx; r.oy += t * r.dy; r.oz += t * r.dz;
        r.dx = ex; r.dy = ey; r.dz = ez;
        if (!(1.f - s.T < kStopAlpha) || bounces >= kMaxBounces || segments >= kMaxSegments) break;
        h = mesh_closest_hit(G.mesh, r.ox, r.oy, r.oz, r.dx, r.dy, r.dz);
        gaussian_segment<PRIM, DEG, false>(P, r, true, kBounceTMin, h.tri >= 0 ? h.t : tmax, kind, s, warp_stack);
        ++segments;
    }
    // the background on 1 - alpha (BackgroundColor at evaluation), rounded as rgb + bg * (1 - alpha), then clamped to [0, 1]
    const float alpha = 1.f - s.T, keep = __fsub_rn(1.f, alpha);
    const int64_t ray = r.ray;
    out_rgb[ray * 3] = fminf(fmaxf(__fadd_rn(kind.Cx, __fmul_rn(G.bg[0], keep)), 0.f), 1.f);
    out_rgb[ray * 3 + 1] = fminf(fmaxf(__fadd_rn(kind.Cy, __fmul_rn(G.bg[1], keep)), 0.f), 1.f);
    out_rgb[ray * 3 + 2] = fminf(fmaxf(__fadd_rn(kind.Cz, __fmul_rn(G.bg[2], keep)), 0.f), 1.f);
    out_alpha[ray] = fminf(fmaxf(alpha, 0.f), 1.f);
}

int fail(grtb200_ctx* c, const char* fmt, ...);

}  // namespace

struct grtb200_ctx {
    grtb200_config cfg;
    int device = 0;
    std::string error;
    int64_t n = -1;
    int64_t launches = 0;
    cudaStream_t build_stream = nullptr;
    void *proxies = nullptr, *leaf_boxes = nullptr, *node_boxes = nullptr, *nodes = nullptr, *codes = nullptr, *ids = nullptr,
         *codes_sorted = nullptr, *ids_sorted = nullptr, *children = nullptr, *parent = nullptr, *leaf_parent = nullptr, *flags = nullptr,
         *scene = nullptr, *sort_temp = nullptr, *grp_codes = nullptr, *grp_ids = nullptr, *grp_boxes = nullptr, *grp_proxies = nullptr;
    size_t cap = 0, sort_temp_bytes = 0;
    // hit-list cache of the last forward (see TraceParams)
    void *hit_list = nullptr, *hit_count = nullptr;
    size_t hit_list_bytes = 0, hit_count_bytes = 0;
    int hit_cap = 96, hit_cap_used = 0;
    bool record_hits = true;          // grtb200_set_replay: inference-only callers switch the hit-list cache off
    size_t hit_budget_bytes = size_t(1) << 30;  // cap of the hit-list cache: the per-ray capacity shrinks for large ray batches
    uint64_t build_generation = 0;
    struct { const float* rays_o; const float* rays_d; const float* particles; const float* out_rgb; const float* out_dist; int64_t rays; int64_t n; uint64_t generation; float r2w[12]; bool valid; int sph_degree; float min_transmittance; int feature_kind; } fwd_key = {};
    float scene_host[6] = {0, 0, 0, 0, 0, 0};
    bool scene_valid = false;
};

namespace {

int fail(grtb200_ctx* c, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (c) c->error = buf;
    return 1;
}

#define GRT_CUDA(ctx, expr)                                                                          \
    do {                                                                                             \
        cudaError_t e__ = (expr);                                                                    \
        if (e__ != cudaSuccess) return fail(ctx, "%s failed: %s", #expr, cudaGetErrorString(e__));   \
    } while (0)

void release(grtb200_ctx* c) {
    void** ptrs[] = {&c->proxies, &c->leaf_boxes, &c->node_boxes, &c->nodes, &c->codes, &c->ids, &c->codes_sorted, &c->ids_sorted,
                     &c->children, &c->parent, &c->leaf_parent, &c->flags, &c->sort_temp, &c->grp_codes, &c->grp_ids, &c->grp_boxes,
                     &c->grp_proxies};
    for (void** p : ptrs) {
        if (*p) cudaFree(*p);
        *p = nullptr;
    }
    c->cap = 0;
    c->sort_temp_bytes = 0;
}

int fill_params(grtb200_ctx* c, TraceParams& P, int64_t n, const float* particles, const float* sph, int sph_degree, float min_t,
                int batch, int height, int width, const float* rays_o, const float* rays_d, const float* r2w, cudaStream_t s) {
    if (batch < 0 || height < 0 || width < 0) return fail(c, "invalid ray shape");
    if (c->n != n) return fail(c, "trace with %lld particles but the BVH was built over %lld (call build_bvh first)",
                               static_cast<long long>(n), static_cast<long long>(c->n));
    if (c->cfg.kernel_degree != 2 && c->cfg.kernel_degree != 4) return fail(c, "kernel_degree %d not built (2 or 4)", c->cfg.kernel_degree);
    if (sph_degree < 0 || sph_degree > 3) return fail(c, "sph_degree %d out of range", sph_degree);
    if (!c->scene_valid && n > 0) {
        int ord[6];
        GRT_CUDA(c, cudaMemcpyAsync(ord, c->scene, sizeof(ord), cudaMemcpyDeviceToHost, s));
        GRT_CUDA(c, cudaStreamSynchronize(s));  // 24-byte read-back once per build, as the reference does (optixTracer.cpp:870-886)
        for (int i = 0; i < 6; ++i) {
            const int v = ord[i] >= 0 ? ord[i] : ord[i] ^ 0x7FFFFFFF;
            memcpy(&c->scene_host[i], &v, 4);
        }
        c->scene_valid = true;
    }
    memset(&P, 0, sizeof(P));
    P.n = static_cast<int>(n);
    P.width = width;
    P.height = height;
    P.batch = batch;
    P.sph_degree = sph_degree;
    P.min_transmittance = min_t;
    P.min_response = c->cfg.min_response;
    P.min_alpha = c->cfg.min_alpha;
    P.max_alpha = c->cfg.max_alpha;
    memcpy(P.r2w, r2w, sizeof(P.r2w));
    memcpy(P.scene, c->scene_host, sizeof(P.scene));
    P.particles = particles;
    P.sph = sph;
    P.rays_o = rays_o;
    P.rays_d = rays_d;
    P.proxies = static_cast<const LeafProxy*>(c->grp_proxies);
    P.leaf = kLeaf;
    P.nodes = static_cast<const BvhNode*>(c->nodes);
    return 0;
}

// CTAs of a trace or replay launch: one warp per 8x4 pixel block, 128 threads per CTA
unsigned ray_blocks(const TraceParams& P) {
    const int bw = (P.width + 7) / 8, bh = (P.height + 3) / 4;
    const int64_t warps = static_cast<int64_t>(bw) * bh * P.batch;
    return static_cast<unsigned>((warps * 32 + 127) / 128);
}

// forward (BWD = false), backward re-trace (BWD = true) or the counting pass (COUNT = true) for the config's primitive and degree
template <bool BWD, bool COUNT, int FK>
void launch_trace(const grtb200_config& cfg, const TraceParams& P, cudaStream_t s) {
    const unsigned blocks = ray_blocks(P);
    if (blocks == 0) return;
    constexpr int kInst = GRTB200_PRIMITIVE_INSTANCES, kIco = GRTB200_PRIMITIVE_ICOSAHEDRON;
    const bool ico = cfg.primitive == kIco;
    if (cfg.kernel_degree == 4) {
        if (ico)
            trace_kernel<kIco, 4, BWD, COUNT, FK><<<blocks, 128, 0, s>>>(P);
        else
            trace_kernel<kInst, 4, BWD, COUNT, FK><<<blocks, 128, 0, s>>>(P);
    } else {
        if (ico)
            trace_kernel<kIco, 2, BWD, COUNT, FK><<<blocks, 128, 0, s>>>(P);
        else
            trace_kernel<kInst, 2, BWD, COUNT, FK><<<blocks, 128, 0, s>>>(P);
    }
}

// false: no rays, nothing launched
template <int FK>
bool launch_replay(const grtb200_config& cfg, const TraceParams& P, cudaStream_t s) {
    const unsigned blocks = ray_blocks(P);
    if (blocks == 0) return false;
    if (cfg.kernel_degree == 4)
        replay_bwd_kernel<4, FK><<<blocks, 128, 0, s>>>(P);
    else
        replay_bwd_kernel<2, FK><<<blocks, 128, 0, s>>>(P);
    return true;
}

// The feature kind fk as a template argument: f(std::integral_constant<int, FK>()).  Every forward, re-trace and replay launch goes
// through here.
template <class F>
void with_kind(int fk, F&& f) {
    if (fk == kFeatNhtHalf)
        f(std::integral_constant<int, kFeatNhtHalf>());
    else if (fk == kFeatNht)
        f(std::integral_constant<int, kFeatNht>());
    else
        f(std::integral_constant<int, kFeatSH>());
}

}  // namespace

extern "C" {

void grtb200_default_config(grtb200_config* c) {  // configs/render/3dgrt.yaml
    c->kernel_degree = 4;
    c->min_response = 0.0113f;
    c->min_alpha = 1.0f / 255.0f;
    c->max_alpha = 0.99f;
    c->density_clamping = 1;
    c->primitive = GRTB200_PRIMITIVE_INSTANCES;
}

int grtb200_create(const grtb200_config* cfg, int device, grtb200_ctx** out) {
    if (!cfg || !out) return 1;
    *out = nullptr;
    if (cfg->primitive != GRTB200_PRIMITIVE_INSTANCES && cfg->primitive != GRTB200_PRIMITIVE_ICOSAHEDRON) return 5;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count) return 2;  // no CPU fallback
    grtb200_ctx* c = new (std::nothrow) grtb200_ctx();
    if (!c) return 3;
    c->cfg = *cfg;
    c->device = device;
    if (cudaSetDevice(device) != cudaSuccess || cudaMalloc(&c->scene, 6 * sizeof(int)) != cudaSuccess) {
        delete c;
        return 4;
    }
    *out = c;
    return 0;
}

void grtb200_destroy(grtb200_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    release(c);
    if (c->scene) cudaFree(c->scene);
    if (c->hit_list) cudaFree(c->hit_list);
    if (c->hit_count) cudaFree(c->hit_count);
    delete c;
}

const char* grtb200_last_error(const grtb200_ctx* c) { return c ? c->error.c_str() : "null context"; }
int64_t grtb200_launch_count(const grtb200_ctx* c) { return c ? c->launches : 0; }

// Both build entries: `packed` says that pos / rot / scl / dns point into the [N,12] particle record (row stride 12 floats).
static int build_bvh(grtb200_ctx* c, void* stream, int64_t n, const float* pos, const float* rot, const float* scl, const float* dns,
                     bool packed) {
    if (!c) return 1;
    if (n < 0 || n > 0x3FFFFFFF) return fail(c, "particle count %lld out of range", static_cast<long long>(n));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    GRT_CUDA(c, cudaSetDevice(c->device));
    c->n = n;
    c->scene_valid = false;
    c->build_generation++;
    c->fwd_key.valid = false;
    if (n == 0) {
        for (float& v : c->scene_host) v = 0.f;
        c->scene_valid = true;
        return 0;
    }
    if (static_cast<size_t>(n) > c->cap) {
        GRT_CUDA(c, cudaStreamSynchronize(s));
        release(c);
        const size_t cap = static_cast<size_t>(n) + static_cast<size_t>(n) / 8 + 16;
        GRT_CUDA(c, cudaMalloc(&c->proxies, cap * sizeof(Proxy)));
        GRT_CUDA(c, cudaMalloc(&c->leaf_boxes, cap * sizeof(Box)));
        GRT_CUDA(c, cudaMalloc(&c->node_boxes, cap * sizeof(Box)));
        GRT_CUDA(c, cudaMalloc(&c->nodes, cap * sizeof(BvhNode)));
        GRT_CUDA(c, cudaMalloc(&c->codes, cap * 4));
        GRT_CUDA(c, cudaMalloc(&c->ids, cap * 4));
        GRT_CUDA(c, cudaMalloc(&c->codes_sorted, cap * 4));
        GRT_CUDA(c, cudaMalloc(&c->ids_sorted, cap * 4));
        GRT_CUDA(c, cudaMalloc(&c->children, cap * sizeof(int2)));
        GRT_CUDA(c, cudaMalloc(&c->parent, cap * 4));
        GRT_CUDA(c, cudaMalloc(&c->leaf_parent, cap * 4));
        GRT_CUDA(c, cudaMalloc(&c->flags, cap * 4));
        GRT_CUDA(c, cudaMalloc(&c->grp_codes, cap * 4));
        GRT_CUDA(c, cudaMalloc(&c->grp_ids, cap * 4));
        GRT_CUDA(c, cudaMalloc(&c->grp_boxes, cap * sizeof(Box)));
        GRT_CUDA(c, cudaMalloc(&c->grp_proxies, cap * sizeof(LeafProxy)));
        c->sort_temp_bytes = sort32_temp_bytes(static_cast<int64_t>(cap)) + 16;
        GRT_CUDA(c, cudaMalloc(&c->sort_temp, c->sort_temp_bytes));
        c->cap = cap;
    }
    const int ni = static_cast<int>(n);
    const unsigned blocks = (ni + 255) / 256;
    GRT_CUDA(c, cudaMemcpyAsync(c->scene, kSceneBoxInit, sizeof(kSceneBoxInit), cudaMemcpyHostToDevice, s));
    if (packed)
        proxy_kernel<12, 12, 12, 12><<<blocks, 256, 0, s>>>(ni, pos, rot, scl, dns, c->cfg.min_response, c->cfg.density_clamping,
                                                            static_cast<float>(c->cfg.kernel_degree), c->cfg.primitive,
                                                            static_cast<Proxy*>(c->proxies), static_cast<Box*>(c->leaf_boxes),
                                                            static_cast<int*>(c->scene));
    else
        proxy_kernel<3, 4, 3, 1><<<blocks, 256, 0, s>>>(ni, pos, rot, scl, dns, c->cfg.min_response, c->cfg.density_clamping,
                                                        static_cast<float>(c->cfg.kernel_degree), c->cfg.primitive,
                                                        static_cast<Proxy*>(c->proxies), static_cast<Box*>(c->leaf_boxes),
                                                        static_cast<int*>(c->scene));
    c->launches++;
    {
        const int ng = (ni + kLeaf - 1) / kLeaf;
        const unsigned gblocks = (ng + 255) / 256;
        morton_kernel<<<blocks, 256, 0, s>>>(ni, static_cast<const Proxy*>(c->proxies), static_cast<const Box*>(c->leaf_boxes),
                                             static_cast<const int*>(c->scene), static_cast<uint32_t*>(c->codes), static_cast<uint32_t*>(c->ids));
        run_sort32_pairs(s, c->sort_temp, c->sort_temp_bytes, static_cast<const uint32_t*>(c->codes), static_cast<uint32_t*>(c->codes_sorted),
                         static_cast<const uint32_t*>(c->ids), static_cast<uint32_t*>(c->ids_sorted), n, 32);
        leaf_kernel<<<gblocks, 256, 0, s>>>(ni, kLeaf, static_cast<const uint32_t*>(c->codes_sorted), static_cast<const uint32_t*>(c->ids_sorted),
                                            static_cast<const Proxy*>(c->proxies), static_cast<const Box*>(c->leaf_boxes),
                                            static_cast<uint32_t*>(c->grp_codes), static_cast<uint32_t*>(c->grp_ids),
                                            static_cast<Box*>(c->grp_boxes), static_cast<LeafProxy*>(c->grp_proxies));
        c->launches += 2;
        if (ng == 1) {
            single_leaf_kernel<<<1, 1, 0, s>>>(static_cast<const Box*>(c->grp_boxes), static_cast<BvhNode*>(c->nodes));
            c->launches++;
        } else {
            GRT_CUDA(c, cudaMemsetAsync(c->flags, 0, static_cast<size_t>(ng) * 4, s));
            hierarchy_kernel<<<gblocks, 256, 0, s>>>(ng, static_cast<const uint32_t*>(c->grp_codes), static_cast<const uint32_t*>(c->grp_ids),
                                                     static_cast<int2*>(c->children), static_cast<int*>(c->parent),
                                                     static_cast<int*>(c->leaf_parent));
            refit_kernel<<<gblocks, 256, 0, s>>>(ng, static_cast<const int2*>(c->children), static_cast<const int*>(c->parent),
                                                 static_cast<const int*>(c->leaf_parent), static_cast<const Box*>(c->grp_boxes),
                                                 static_cast<Box*>(c->node_boxes), static_cast<int*>(c->flags), static_cast<BvhNode*>(c->nodes));
            c->launches += 2;
        }
    }
    GRT_CUDA(c, cudaGetLastError());
    return 0;
}

int grtb200_build_bvh(grtb200_ctx* c, void* stream, int64_t n, const float* pos, const float* rot, const float* scl, const float* dns,
                      int32_t /*rebuild*/, int32_t /*allow_update*/) {
    return build_bvh(c, stream, n, pos, rot, scl, dns, false);
}

// The particle record [N,12] = pos3, density, quat(wxyz), scale3, pad is what grtb200_trace reads: a training step that keeps its
// activated particles in that layout builds from it directly instead of copying out four arrays.
int grtb200_build_bvh_packed(grtb200_ctx* c, void* stream, int64_t n, const float* particles) {
    if (!c) return 1;
    if (!particles && n > 0) return fail(c, "particles is null");
    return build_bvh(c, stream, n, particles, particles + 4, particles + 8, particles + 3, true);
}

int grtb200_scene_aabb(grtb200_ctx* c, float* aabb6) {
    if (!c || c->n < 0) return fail(c, "no BVH built");
    if (!c->scene_valid) {
        int ord[6];
        GRT_CUDA(c, cudaSetDevice(c->device));
        GRT_CUDA(c, cudaDeviceSynchronize());
        GRT_CUDA(c, cudaMemcpy(ord, c->scene, sizeof(ord), cudaMemcpyDeviceToHost));
        for (int i = 0; i < 6; ++i) {
            const int v = ord[i] >= 0 ? ord[i] : ord[i] ^ 0x7FFFFFFF;
            memcpy(&c->scene_host[i], &v, 4);
        }
        c->scene_valid = true;
    }
    memcpy(aabb6, c->scene_host, sizeof(c->scene_host));
    return 0;
}

// Forward of either feature kind: fk = kFeatSH (sph [N,48] SH coefficients, out_rgb [R,3]) or an NHT kind (sph = the [N,48] feature
// rows, out_rgb = the [R,24] ray features).  out_normals (SH only, else nullptr): the kFeatShNormals forward also writes the [R,3]
// normals; it records the same hit lists under the same key as the plain SH forward, so the SH backward replays them.
static int trace_fwd(grtb200_ctx* c, int fk, void* stream, int64_t n, const float* particles, const float* sph, int32_t sph_degree,
                     float min_transmittance, int32_t batch, int32_t height, int32_t width, const float* rays_o, const float* rays_d,
                     const float* ray_to_world_host, float* out_rgb, float* out_alpha, float* out_dist, float* out_hits, float* visibility,
                     float* out_normals = nullptr) {
    if (!c) return 1;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    GRT_CUDA(c, cudaSetDevice(c->device));
    TraceParams P;
    if (int rc = fill_params(c, P, n, particles, sph, sph_degree, min_transmittance, batch, height, width, rays_o, rays_d, ray_to_world_host, s)) return rc;
    P.out_rgb = out_rgb; P.out_alpha = out_alpha; P.out_dist = out_dist; P.out_hits = out_hits; P.visibility = visibility;
    P.out_normals = out_normals;
    if (n > 0) GRT_CUDA(c, cudaMemsetAsync(visibility, 0, static_cast<size_t>(n) * 4, s));
    // hit-list cache for the backward of this forward (grow-only; GRTB200_HITCAP=0 turns it off, the backward then re-traces)
    c->fwd_key.valid = false;
    int cap = c->record_hits ? c->hit_cap : 0;
    if (const char* e = std::getenv("GRTB200_HITCAP")) cap = std::max(0, std::min(1024, std::atoi(e)));
    const int64_t rays = static_cast<int64_t>(batch) * height * width;
    if (cap > 0 && rays > 0)  // keep the cache inside its byte budget (1080p x 96 x 4 B would be 0.8 GB, 4K 3.2 GB); overflowed rays re-trace
        cap = static_cast<int>(std::min<int64_t>(cap, std::max<int64_t>(8, static_cast<int64_t>(c->hit_budget_bytes / 4) / rays)));
    if (cap > 0 && rays > 0 && n > 0) {
        const size_t need = static_cast<size_t>(rays) * cap * 4, need_c = static_cast<size_t>(rays) * 4;
        if (need > c->hit_list_bytes) {
            GRT_CUDA(c, cudaStreamSynchronize(s));
            if (c->hit_list) cudaFree(c->hit_list);
            c->hit_list = nullptr;
            c->hit_list_bytes = 0;
            GRT_CUDA(c, cudaMalloc(&c->hit_list, need));
            c->hit_list_bytes = need;
        }
        if (need_c > c->hit_count_bytes) {
            GRT_CUDA(c, cudaStreamSynchronize(s));
            if (c->hit_count) cudaFree(c->hit_count);
            c->hit_count = nullptr;
            c->hit_count_bytes = 0;
            GRT_CUDA(c, cudaMalloc(&c->hit_count, need_c));
            c->hit_count_bytes = need_c;
        }
        P.hit_list = static_cast<uint32_t*>(c->hit_list);
        P.hit_count = static_cast<uint32_t*>(c->hit_count);
        P.hit_cap = cap;
        P.rays = rays;
        c->fwd_key = {rays_o, rays_d, particles, out_rgb, out_dist, rays, n, c->build_generation, {}, true};
        memcpy(c->fwd_key.r2w, P.r2w, sizeof(P.r2w));
        c->fwd_key.sph_degree = sph_degree;
        c->fwd_key.min_transmittance = min_transmittance;
        c->fwd_key.feature_kind = fk;
        c->hit_cap_used = cap;
    }
    if (out_normals)
        launch_trace<false, false, kFeatShNormals>(c->cfg, P, s);
    else
        with_kind(fk, [&](auto k) { launch_trace<false, false, decltype(k)::value>(c->cfg, P, s); });
    c->launches++;
    GRT_CUDA(c, cudaGetLastError());
    return 0;
}

int grtb200_trace_normals(grtb200_ctx* c, void* stream, int64_t n, const float* particles, const float* sph, int32_t sph_degree,
                          float min_transmittance, int32_t batch, int32_t height, int32_t width, const float* rays_o, const float* rays_d,
                          const float* ray_to_world_host, float* out_rgb, float* out_alpha, float* out_dist, float* out_hits, float* visibility,
                          float* out_normals) {
    if (!c) return 1;
    if (!out_normals) return fail(c, "out_normals is null (grtb200_trace writes no normals)");
    return trace_fwd(c, kFeatSH, stream, n, particles, sph, sph_degree, min_transmittance, batch, height, width, rays_o, rays_d,
                     ray_to_world_host, out_rgb, out_alpha, out_dist, out_hits, visibility, out_normals);
}

int grtb200_trace(grtb200_ctx* c, void* stream, int64_t n, const float* particles, const float* sph, int32_t sph_degree,
                  float min_transmittance, int32_t batch, int32_t height, int32_t width, const float* rays_o, const float* rays_d,
                  const float* ray_to_world_host, float* out_rgb, float* out_alpha, float* out_dist, float* out_hits, float* visibility) {
    return trace_fwd(c, kFeatSH, stream, n, particles, sph, sph_degree, min_transmittance, batch, height, width, rays_o, rays_d,
                     ray_to_world_host, out_rgb, out_alpha, out_dist, out_hits, visibility);
}

// the NHT kind of a feature row layout; -1 (with the context's error set) for a layout that is not built
static int nht_kind(grtb200_ctx* c, int32_t feature_dim, int32_t features_half) {
    if (feature_dim != kNhtRow) {
        fail(c, "feature_dim %d not built: NHT features are built for 48 = 4 tetrahedron vertices x 12", feature_dim);
        return -1;
    }
    return features_half ? kFeatNhtHalf : kFeatNht;
}

int grtb200_trace_nht(grtb200_ctx* c, void* stream, int64_t n, const float* particles, const void* features, int32_t feature_dim,
                      int32_t features_half, float min_transmittance, int32_t batch, int32_t height, int32_t width, const float* rays_o,
                      const float* rays_d, const float* ray_to_world_host, float* out_features, float* out_alpha, float* out_dist,
                      float* out_hits, float* visibility) {
    if (!c) return 1;
    const int fk = nht_kind(c, feature_dim, features_half);
    if (fk < 0) return 1;
    return trace_fwd(c, fk, stream, n, particles, static_cast<const float*>(features), 0, min_transmittance, batch, height, width, rays_o,
                     rays_d, ray_to_world_host, out_features, out_alpha, out_dist, out_hits, visibility);
}

// Work counters of one forward trace (debug, synchronises; writes no image): counters8 = { rays, k-nearest queries, node visits (one per
// warp and node for packet-walked rays, else one per lane), box tests, proxy tests, candidate hits processed, accepted hits, rays walked
// as packets } -- the units of SURVEY.md 8d "3DGRT work units".
int grtb200_debug_trace_counters(grtb200_ctx* c, void* stream, int64_t n, const float* particles, const float* sph, int32_t sph_degree,
                                 float min_transmittance, int32_t batch, int32_t height, int32_t width, const float* rays_o, const float* rays_d,
                                 const float* ray_to_world_host, float* visibility_scratch, uint64_t* counters8) {
    if (!c || !counters8) return 1;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    GRT_CUDA(c, cudaSetDevice(c->device));
    TraceParams P;
    if (int rc = fill_params(c, P, n, particles, sph, sph_degree, min_transmittance, batch, height, width, rays_o, rays_d, ray_to_world_host, s)) return rc;
    P.visibility = visibility_scratch;
    P.hit_list = nullptr;
    P.hit_count = nullptr;
    unsigned long long* d = nullptr;
    GRT_CUDA(c, cudaMalloc(&d, 64));
    cudaMemsetAsync(d, 0, 64, s);
    P.counters = d;
    launch_trace<false, true, kFeatSH>(c->cfg, P, s);
    cudaError_t e = cudaStreamSynchronize(s);
    if (e == cudaSuccess) e = cudaMemcpy(counters8, d, 64, cudaMemcpyDeviceToHost);
    cudaFree(d);
    GRT_CUDA(c, e);
    return 0;
}

// Switch the forward's hit-list recording (replayed by the backward) on / off: inference-only renders need no cache.  Turning it off frees it.
int grtb200_set_replay(grtb200_ctx* c, int32_t enable) {
    if (!c) return 1;
    c->record_hits = enable != 0;
    if (!c->record_hits) {
        GRT_CUDA(c, cudaSetDevice(c->device));
        c->fwd_key.valid = false;
        if (c->hit_list) {
            GRT_CUDA(c, cudaDeviceSynchronize());
            cudaFree(c->hit_list);
            c->hit_list = nullptr;
            c->hit_list_bytes = 0;
        }
    }
    return 0;
}

// Backward of either feature kind (see trace_fwd); d_sph is the [N,48] fp32 SH or feature gradient.  The replay and the re-trace add
// into d_particles / d_sph; accumulate = false zeroes them first.
static int trace_bwd(grtb200_ctx* c, int fk, void* stream, int64_t n, const float* particles, const float* sph, int32_t sph_degree,
                     float min_transmittance, int32_t batch, int32_t height, int32_t width, const float* rays_o, const float* rays_d,
                     const float* ray_to_world_host, const float* out_rgb, const float* out_alpha, const float* out_dist,
                     const float* d_rgb, const float* d_alpha, const float* d_dist, float* d_particles, float* d_sph, bool accumulate = false) {
    if (!c) return 1;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    GRT_CUDA(c, cudaSetDevice(c->device));
    TraceParams P;
    if (int rc = fill_params(c, P, n, particles, sph, sph_degree, min_transmittance, batch, height, width, rays_o, rays_d, ray_to_world_host, s)) return rc;
    P.out_rgb = const_cast<float*>(out_rgb); P.out_alpha = const_cast<float*>(out_alpha); P.out_dist = const_cast<float*>(out_dist);
    P.d_rgb = d_rgb; P.d_alpha = d_alpha; P.d_dist = d_dist;
    P.d_particles = d_particles; P.d_sph = d_sph;
    if (n > 0 && !accumulate) {
        GRT_CUDA(c, cudaMemsetAsync(d_particles, 0, static_cast<size_t>(n) * 48, s));
        GRT_CUDA(c, cudaMemsetAsync(d_sph, 0, static_cast<size_t>(n) * 192, s));
    }
    const int64_t rays = static_cast<int64_t>(batch) * height * width;
    const bool replay = c->fwd_key.valid && c->fwd_key.rays_o == rays_o && c->fwd_key.rays_d == rays_d && c->fwd_key.particles == particles &&
                        c->fwd_key.out_rgb == out_rgb && c->fwd_key.out_dist == out_dist && memcmp(c->fwd_key.r2w, P.r2w, sizeof(P.r2w)) == 0 &&
                        c->fwd_key.rays == rays && c->fwd_key.n == n && c->fwd_key.generation == c->build_generation && n > 0 &&
                        c->fwd_key.sph_degree == sph_degree && c->fwd_key.min_transmittance == min_transmittance &&
                        c->fwd_key.feature_kind == fk;
    if (replay) {  // the lists of the forward these outputs came from: replay them, re-trace only the rays that overflowed
        P.hit_list = static_cast<uint32_t*>(c->hit_list);
        P.hit_count = static_cast<uint32_t*>(c->hit_count);
        P.hit_cap = c->hit_cap_used;
        P.rays = rays;
        bool launched = false;
        with_kind(fk, [&](auto k) { launched = launch_replay<decltype(k)::value>(c->cfg, P, s); });
        c->launches += launched ? 1 : 0;
        P.only_overflow = 1;
    }
    with_kind(fk, [&](auto k) { launch_trace<true, false, decltype(k)::value>(c->cfg, P, s); });
    c->launches++;
    GRT_CUDA(c, cudaGetLastError());
    return 0;
}

int grtb200_trace_bwd(grtb200_ctx* c, void* stream, int64_t n, const float* particles, const float* sph, int32_t sph_degree,
                      float min_transmittance, int32_t batch, int32_t height, int32_t width, const float* rays_o, const float* rays_d,
                      const float* ray_to_world_host, const float* out_rgb, const float* out_alpha, const float* out_dist,
                      const float* d_rgb, const float* d_alpha, const float* d_dist, float* d_particles, float* d_sph) {
    return trace_bwd(c, kFeatSH, stream, n, particles, sph, sph_degree, min_transmittance, batch, height, width, rays_o, rays_d,
                     ray_to_world_host, out_rgb, out_alpha, out_dist, d_rgb, d_alpha, d_dist, d_particles, d_sph);
}

int grtb200_trace_bwd_accumulate(grtb200_ctx* c, void* stream, int64_t n, const float* particles, const float* sph, int32_t sph_degree,
                                 float min_transmittance, int32_t batch, int32_t height, int32_t width, const float* rays_o,
                                 const float* rays_d, const float* ray_to_world_host, const float* out_rgb, const float* out_alpha,
                                 const float* out_dist, const float* d_rgb, const float* d_alpha, const float* d_dist, float* d_particles,
                                 float* d_sph) {
    return trace_bwd(c, kFeatSH, stream, n, particles, sph, sph_degree, min_transmittance, batch, height, width, rays_o, rays_d,
                     ray_to_world_host, out_rgb, out_alpha, out_dist, d_rgb, d_alpha, d_dist, d_particles, d_sph, true);
}

int grtb200_trace_bwd_nht(grtb200_ctx* c, void* stream, int64_t n, const float* particles, const void* features, int32_t feature_dim,
                          int32_t features_half, float min_transmittance, int32_t batch, int32_t height, int32_t width, const float* rays_o,
                          const float* rays_d, const float* ray_to_world_host, const float* out_features, const float* out_alpha,
                          const float* out_dist, const float* d_features_out, const float* d_alpha, const float* d_dist, float* d_particles,
                          float* d_features) {
    if (!c) return 1;
    const int fk = nht_kind(c, feature_dim, features_half);
    if (fk < 0) return 1;
    return trace_bwd(c, fk, stream, n, particles, static_cast<const float*>(features), 0, min_transmittance, batch, height, width, rays_o,
                     rays_d, ray_to_world_host, out_features, out_alpha, out_dist, d_features_out, d_alpha, d_dist, d_particles, d_features);
}

// Playground render (DESIGN.md section 22): fill_params as grtb200_trace, the mesh view of `mesh`, one launch.
int grtb200_trace_playground(grtb200_ctx* c, void* stream, const grtb200_mesh* mesh, int64_t n, const float* particles, const float* sph,
                             int32_t sph_degree, float min_transmittance, int32_t batch, int32_t height, int32_t width, const float* rays_o,
                             const float* rays_d, const float* ray_to_world_host, const float* ray_max_t, const float* background_host,
                             int32_t smooth_normals, float* out_rgb, float* out_alpha, float* visibility) {
    if (!c) return 1;
    if (!background_host || !out_rgb || !out_alpha || (n > 0 && !visibility)) return fail(c, "trace_playground: null background or output");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    GRT_CUDA(c, cudaSetDevice(c->device));
    PlaygroundParams G;
    if (int rc = fill_params(c, G.P, n, particles, sph, sph_degree, min_transmittance, batch, height, width, rays_o, rays_d, ray_to_world_host, s))
        return rc;
    G.P.visibility = visibility;
    G.mesh = gutb200::mesh_view(mesh);
    G.ray_max_t = ray_max_t;
    for (int k = 0; k < 3; ++k) G.bg[k] = background_host[k];
    G.smooth = smooth_normals != 0;
    if (n > 0) GRT_CUDA(c, cudaMemsetAsync(visibility, 0, static_cast<size_t>(n) * 4, s));
    const unsigned blocks = ray_blocks(G.P);
    if (blocks == 0) return 0;
    constexpr int kInst = GRTB200_PRIMITIVE_INSTANCES, kIco = GRTB200_PRIMITIVE_ICOSAHEDRON;
    const bool ico = c->cfg.primitive == kIco;
    if (c->cfg.kernel_degree == 4) {
        if (ico)
            playground_kernel<kIco, 4><<<blocks, 128, 0, s>>>(G, out_rgb, out_alpha);
        else
            playground_kernel<kInst, 4><<<blocks, 128, 0, s>>>(G, out_rgb, out_alpha);
    } else {
        if (ico)
            playground_kernel<kIco, 2><<<blocks, 128, 0, s>>>(G, out_rgb, out_alpha);
        else
            playground_kernel<kInst, 2><<<blocks, 128, 0, s>>>(G, out_rgb, out_alpha);
    }
    c->launches++;
    GRT_CUDA(c, cudaGetLastError());
    return 0;
}

}  // extern "C"
