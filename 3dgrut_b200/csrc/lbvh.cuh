// 3dgrut_b200/csrc/lbvh.cuh -- the LBVH build stages shared by the 3DGRT proxy tree (grt.cu) and the k-nearest-neighbour point tree
// (gut_knn.cu): the scene-box reduction, 30-bit Morton codes in that box, the Karras topology over sorted keys and the bottom-up refit
// into 64-byte nodes that hold both child boxes.  (The sort between the Morton codes and the topology is run_sort32_pairs, gut_sort.cu.)
// Everything here sits in the unnamed namespace: each translation unit that includes the header compiles its own copy with its own
// numerics flags.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

struct __align__(16) BvhNode {
    float4 b0;    // lmin.xyz, lmax.x
    float4 b1;    // lmax.yz, rmin.xy
    float4 b2;    // rmin.z, rmax.xyz
    float4 meta;  // left, right (int bits: >=0 internal, <0 leaf ~leaf index), left slack, right slack
};
struct __align__(16) Box {
    float4 lo;  // min.xyz, slack (3DGRT: largest proxy half-diagonal below; 0 for points)
    float4 hi;  // max.xyz, unused
};

// ---- scene box: six ordered ints reduced with atomicMin / atomicMax -------------------------------------------------------------------

__device__ __forceinline__ int float_order(float f) {  // monotone float -> int map for atomicMin/Max
    const int i = __float_as_int(f);
    return i >= 0 ? i : i ^ 0x7FFFFFFF;
}
__device__ __forceinline__ float order_float(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7FFFFFFF); }

// the empty box: min = +FLT_MAX, max = ordered(-FLT_MAX); the host copies it into the six ints before the reduction
constexpr int kSceneBoxInit[6] = {0x7F7FFFFF, 0x7F7FFFFF, 0x7F7FFFFF, static_cast<int>(0xFF7FFFFFu ^ 0x7FFFFFFFu),
                                  static_cast<int>(0xFF7FFFFFu ^ 0x7FFFFFFFu), static_cast<int>(0xFF7FFFFFu ^ 0x7FFFFFFFu)};

__device__ __forceinline__ void scene_box_extend(int* scene, float lx, float ly, float lz, float hx, float hy, float hz) {
    atomicMin(scene + 0, float_order(lx)); atomicMin(scene + 1, float_order(ly)); atomicMin(scene + 2, float_order(lz));
    atomicMax(scene + 3, float_order(hx)); atomicMax(scene + 4, float_order(hy)); atomicMax(scene + 5, float_order(hz));
}

// ---- Morton codes -------------------------------------------------------------------------------------------------------------------

__device__ __forceinline__ uint32_t expand_bits(uint32_t v) {
    v = (v * 0x00010001u) & 0xFF0000FFu;
    v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u;
    v = (v * 0x00000005u) & 0x49249249u;
    return v;
}

struct SceneBox {
    float lx, ly, lz;  // min corner
    float ex, ey, ez;  // extent, at least 1e-20
};

__device__ __forceinline__ SceneBox scene_box(const int* __restrict__ scene) {
    SceneBox b;
    b.lx = order_float(scene[0]); b.ly = order_float(scene[1]); b.lz = order_float(scene[2]);
    b.ex = fmaxf(order_float(scene[3]) - b.lx, 1e-20f);
    b.ey = fmaxf(order_float(scene[4]) - b.ly, 1e-20f);
    b.ez = fmaxf(order_float(scene[5]) - b.lz, 1e-20f);
    return b;
}

// 10 bits per axis of (x, y, z) in the scene box, interleaved x-major; points outside the box clamp to its faces
__device__ __forceinline__ uint32_t morton30(const SceneBox& b, float x, float y, float z) {
    const float ux = fminf(fmaxf((x - b.lx) / b.ex * 1024.f, 0.f), 1023.f);
    const float uy = fminf(fmaxf((y - b.ly) / b.ey * 1024.f, 0.f), 1023.f);
    const float uz = fminf(fmaxf((z - b.lz) / b.ez * 1024.f, 0.f), 1023.f);
    return expand_bits(static_cast<uint32_t>(ux)) * 4 + expand_bits(static_cast<uint32_t>(uy)) * 2 + expand_bits(static_cast<uint32_t>(uz));
}

// ---- Karras topology and refit ------------------------------------------------------------------------------------------------------

// common-prefix length of sorted keys i and j (index as tie breaker); -1 outside the range
__device__ __forceinline__ int delta(const uint32_t* __restrict__ codes, int n, int i, int j) {
    if (j < 0 || j >= n) return -1;
    const uint32_t a = codes[i], b = codes[j];
    if (a == b) return 32 + __clz(static_cast<uint32_t>(i) ^ static_cast<uint32_t>(j));
    return __clz(a ^ b);
}

// Karras 2012: one thread per internal node; children are (internal index) or ~(leaf id) for leaves.  Each level below the root
// lengthens the common prefix of the 64-bit (code, index) keys under it, so no path from the root is longer than 64 nodes.
__global__ void __launch_bounds__(256) hierarchy_kernel(int n, const uint32_t* __restrict__ codes, const uint32_t* __restrict__ ids,
                                                        int2* __restrict__ children, int* __restrict__ parent,
                                                        int* __restrict__ leaf_parent) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n - 1) return;
    const int d = (delta(codes, n, i, i + 1) - delta(codes, n, i, i - 1)) >= 0 ? 1 : -1;
    const int dmin = delta(codes, n, i, i - d);
    int lmax = 2;
    while (delta(codes, n, i, i + lmax * d) > dmin) lmax *= 2;
    int l = 0;
    for (int t = lmax / 2; t >= 1; t /= 2)
        if (delta(codes, n, i, i + (l + t) * d) > dmin) l += t;
    const int j = i + l * d;
    const int dnode = delta(codes, n, i, j);
    int s = 0, t = l;
    do {
        t = (t + 1) >> 1;
        if (delta(codes, n, i, i + (s + t) * d) > dnode) s += t;
    } while (t > 1);
    const int gamma = i + s * d + min(d, 0);
    const int lo = min(i, j), hi = max(i, j);
    int left, right;
    if (lo == gamma) {
        left = ~static_cast<int>(ids[gamma]);
        leaf_parent[gamma] = i;
    } else {
        left = gamma;
        parent[gamma] = i;
    }
    if (hi == gamma + 1) {
        right = ~static_cast<int>(ids[gamma + 1]);
        leaf_parent[gamma + 1] = i;
    } else {
        right = gamma + 1;
        parent[gamma + 1] = i;
    }
    children[i] = make_int2(left, right);
    if (i == 0) parent[0] = -1;
}

// Bottom-up boxes, one thread per leaf: the second thread to reach a node writes it.  The atomic decides only which thread does the
// work; a node's boxes are min / max of its children's whichever thread writes them, so the nodes are the same on every run.
__global__ void __launch_bounds__(256) refit_kernel(int n, const int2* __restrict__ children, const int* __restrict__ parent,
                                                    const int* __restrict__ leaf_parent, const Box* __restrict__ leaf_boxes,
                                                    Box* __restrict__ node_boxes, int* __restrict__ flags, BvhNode* __restrict__ nodes) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int cur = leaf_parent[i];
    while (cur >= 0) {
        __threadfence();
        if (atomicAdd(flags + cur, 1) == 0) return;  // first arrival: the sibling subtree is not finished yet
        __threadfence();
        const int2 ch = children[cur];
        const Box l = ch.x < 0 ? leaf_boxes[~ch.x] : node_boxes[ch.x];
        const Box r = ch.y < 0 ? leaf_boxes[~ch.y] : node_boxes[ch.y];
        BvhNode nd;
        nd.b0 = make_float4(l.lo.x, l.lo.y, l.lo.z, l.hi.x);
        nd.b1 = make_float4(l.hi.y, l.hi.z, r.lo.x, r.lo.y);
        nd.b2 = make_float4(r.lo.z, r.hi.x, r.hi.y, r.hi.z);
        nd.meta = make_float4(__int_as_float(ch.x), __int_as_float(ch.y), l.lo.w, r.lo.w);
        nodes[cur] = nd;
        Box u;
        u.lo = make_float4(fminf(l.lo.x, r.lo.x), fminf(l.lo.y, r.lo.y), fminf(l.lo.z, r.lo.z), fmaxf(l.lo.w, r.lo.w));
        u.hi = make_float4(fmaxf(l.hi.x, r.hi.x), fmaxf(l.hi.y, r.hi.y), fmaxf(l.hi.z, r.hi.z), 0.f);
        node_boxes[cur] = u;
        cur = parent[cur];
    }
}

}  // namespace
