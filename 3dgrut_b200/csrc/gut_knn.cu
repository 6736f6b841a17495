// 3dgrut_b200/csrc/gut_knn.cu -- exact k-nearest-neighbour search (k <= 4) for the initial Gaussian scales (initialization.py).
// C ABI: gutb200_knn / gutb200_knn_workspace_bytes (include/gut_b200.h).  DESIGN.md section 19.
//
// The point tree is built from the 3DGRT LBVH stages (lbvh.cuh, gut_sort.cu):
//   box_kernel        scene box of the targets (warp min / max, then the shared ordered-int atomics)
//   morton_kernel     30-bit Morton code of each target in that box
//   (CUB radix sort of (code, target) pairs -- library)
//   bucket_kernel     buckets of kBucket consecutive sorted targets: the targets as float4 (x, y, z, index bits) in sorted order, the
//                     bucket's box and key.  Buckets are bounded by count, not by code: a dense core puts many targets on one code.
//   hierarchy_kernel  Karras topology over the buckets
//   refit_kernel      both child boxes in each 64-byte node
//   query_kernel<K,SELF>  one thread per query; self queries run in sorted order (neighbouring threads walk similar paths) and seed the
//                     k best from their own bucket, then walk the tree nearer child first.
// Exactness: a box is skipped only when its lower bound is strictly greater than the current k-th best distance, and that bound is computed
// with the distance's own operations (per axis a difference, squares, two adds left to right; this file is built with -fmad=false), so
// that it can never round above the distance of a point inside the box.  Determinism: the result is the k smallest (distance, index) pairs
// in lexicographic order, which does not depend on the order in which the walk meets them.
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "../../include/gut_b200.h"
#include "lbvh.cuh"

namespace gutb200 {
size_t sort32_temp_bytes(int64_t n);
void run_sort32_pairs(cudaStream_t s, void* temp, size_t temp_bytes, const uint32_t* kin, uint32_t* kout, const uint32_t* vin,
                      uint32_t* vout, int64_t n, int end_bit);
void set_context_free_error(const std::string& msg);  // gut_api.cu: the message gutb200_last_error(NULL) returns
}  // namespace gutb200

using namespace gutb200;

namespace {

constexpr int kBucket = 16;   // targets per leaf bucket
constexpr int kStack = 64;    // the Karras tree is at most 64 levels deep (lbvh.cuh)
constexpr int kQueryThreads = 128;  // 8 CTAs per SM: at most 64 registers, and the K = 4 walk then keeps its state out of local memory

__global__ void __launch_bounds__(256) box_kernel(int m, const float* __restrict__ pts, int* __restrict__ scene) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < m;
    const float x = live ? pts[3 * i] : 3e38f, y = live ? pts[3 * i + 1] : 3e38f, z = live ? pts[3 * i + 2] : 3e38f;
    const int lx = __reduce_min_sync(0xFFFFFFFFu, float_order(x)), ly = __reduce_min_sync(0xFFFFFFFFu, float_order(y)),
              lz = __reduce_min_sync(0xFFFFFFFFu, float_order(z));
    const int hx = __reduce_max_sync(0xFFFFFFFFu, float_order(live ? x : -3e38f)),
              hy = __reduce_max_sync(0xFFFFFFFFu, float_order(live ? y : -3e38f)),
              hz = __reduce_max_sync(0xFFFFFFFFu, float_order(live ? z : -3e38f));
    if ((threadIdx.x & 31) == 0 && i < m)
        scene_box_extend(scene, order_float(lx), order_float(ly), order_float(lz), order_float(hx), order_float(hy), order_float(hz));
}

__global__ void __launch_bounds__(256) morton_kernel(int m, const float* __restrict__ pts, const int* __restrict__ scene,
                                                     uint32_t* __restrict__ codes, uint32_t* __restrict__ ids) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    codes[i] = morton30(scene_box(scene), pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
    ids[i] = static_cast<uint32_t>(i);
}

__global__ void __launch_bounds__(256) bucket_kernel(int m, int ng, const uint32_t* __restrict__ codes_sorted,
                                                     const uint32_t* __restrict__ ids_sorted, const float* __restrict__ pts,
                                                     float4* __restrict__ sorted, uint32_t* __restrict__ leaf_codes,
                                                     uint32_t* __restrict__ leaf_ids, Box* __restrict__ leaf_boxes) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= ng) return;
    const int first = g * kBucket, last = min(first + kBucket, m);
    Box u;
    u.lo = make_float4(3e38f, 3e38f, 3e38f, 0.f);
    u.hi = make_float4(-3e38f, -3e38f, -3e38f, 0.f);
    for (int s = first; s < last; ++s) {
        const uint32_t id = ids_sorted[s];
        const float x = pts[3 * id], y = pts[3 * id + 1], z = pts[3 * id + 2];
        sorted[s] = make_float4(x, y, z, __int_as_float(static_cast<int>(id)));
        u.lo = make_float4(fminf(u.lo.x, x), fminf(u.lo.y, y), fminf(u.lo.z, z), 0.f);
        u.hi = make_float4(fmaxf(u.hi.x, x), fmaxf(u.hi.y, y), fmaxf(u.hi.z, z), 0.f);
    }
    leaf_codes[g] = codes_sorted[first];
    leaf_ids[g] = static_cast<uint32_t>(g);
    leaf_boxes[g] = u;
}

// (da, ia) before (db, ib): the order the rows are sorted in
__device__ __forceinline__ bool before(float da, int ia, float db, int ib) { return da < db || (da == db && ia < ib); }

template <int K>
struct Best {
    float d[K];
    int i[K];

    __device__ __forceinline__ void init() {
#pragma unroll
        for (int s = 0; s < K; ++s) {
            d[s] = __int_as_float(0x7F800000);  // +inf
            i[s] = 0x7FFFFFFF;
        }
    }
    __device__ __forceinline__ float worst() const { return d[K - 1]; }
    __device__ __forceinline__ void insert(float dn, int in) {
        if (!before(dn, in, d[K - 1], i[K - 1])) return;
        d[K - 1] = dn;
        i[K - 1] = in;
#pragma unroll
        for (int s = K - 1; s > 0; --s) {
            if (before(d[s], i[s], d[s - 1], i[s - 1])) {
                const float td = d[s]; d[s] = d[s - 1]; d[s - 1] = td;
                const int ti = i[s]; i[s] = i[s - 1]; i[s - 1] = ti;
            }
        }
    }
};

// the squared distance, evaluated (qx-px)^2 + (qy-py)^2 + (qz-pz)^2 left to right without contraction
__device__ __forceinline__ float dist2(float qx, float qy, float qz, float px, float py, float pz) {
    const float dx = qx - px, dy = qy - py, dz = qz - pz;
    return dx * dx + dy * dy + dz * dz;
}

// Lower bound of dist2(q, p) over the points p of the box [lo, hi].  Per axis, a point with lo <= p <= hi has q - p at least q - hi and
// p - q at least lo - q in exact arithmetic; rounding to nearest is monotone and odd, so the rounded gap here is at most |q - p| as
// dist2 rounds it, and the squares and the two adds keep that order.
__device__ __forceinline__ float box_bound(float qx, float qy, float qz, float lx, float ly, float lz, float hx, float hy, float hz) {
    const float ex = fmaxf(fmaxf(lx - qx, qx - hx), 0.f), ey = fmaxf(fmaxf(ly - qy, qy - hy), 0.f), ez = fmaxf(fmaxf(lz - qz, qz - hz), 0.f);
    return ex * ex + ey * ey + ez * ez;
}

template <int K>
__device__ __forceinline__ void scan_bucket(const float4* __restrict__ sorted, int m, int g, float qx, float qy, float qz, int self,
                                            Best<K>& best) {
    const int first = g * kBucket, last = min(first + kBucket, m);
    for (int s = first; s < last; ++s) {
        const float4 p = sorted[s];
        const int id = __float_as_int(p.w);
        if (id == self) continue;
        best.insert(dist2(qx, qy, qz, p.x, p.y, p.z), id);
    }
}

// SELF: thread t is the query at sorted position t (target sorted[t], which it excludes); else thread t is queries[t].
template <int K, bool SELF>
__global__ void __launch_bounds__(kQueryThreads, 8) query_kernel(int nq, int m, int ng, const float* __restrict__ queries,
                                                              const float4* __restrict__ sorted, const BvhNode* __restrict__ nodes,
                                                              int32_t* __restrict__ out_idx, float* __restrict__ out_dist) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nq) return;
    float qx, qy, qz;
    int self = -1, skip = -1, row = t;
    Best<K> best;
    best.init();
    if (SELF) {
        const float4 q = sorted[t];
        qx = q.x; qy = q.y; qz = q.z;
        self = row = __float_as_int(q.w);
        skip = t / kBucket;
        scan_bucket<K>(sorted, m, skip, qx, qy, qz, self, best);
    } else {
        qx = queries[3 * t]; qy = queries[3 * t + 1]; qz = queries[3 * t + 2];
    }
    if (ng == 1) {
        if (skip != 0) scan_bucket<K>(sorted, m, 0, qx, qy, qz, self, best);
    } else {
        int stack[kStack];
        float stack_bound[kStack];
        int sp = 0, node = 0;
        while (true) {
            const BvhNode nd = nodes[node];
            int a = __float_as_int(nd.meta.x), b = __float_as_int(nd.meta.y);
            float ba = box_bound(qx, qy, qz, nd.b0.x, nd.b0.y, nd.b0.z, nd.b0.w, nd.b1.x, nd.b1.y);
            float bb = box_bound(qx, qy, qz, nd.b1.z, nd.b1.w, nd.b2.x, nd.b2.y, nd.b2.z, nd.b2.w);
            if (bb < ba) {
                const int tc = a; a = b; b = tc;
                const float tb = ba; ba = bb; bb = tb;
            }
            int next = -1;
            if (ba <= best.worst()) {
                if (a >= 0) next = a;
                else if (~a != skip) scan_bucket<K>(sorted, m, ~a, qx, qy, qz, self, best);
            }
            if (bb <= best.worst()) {
                if (b < 0) {
                    if (~b != skip) scan_bucket<K>(sorted, m, ~b, qx, qy, qz, self, best);
                } else if (next < 0) {
                    next = b;
                } else {
                    stack[sp] = b;
                    stack_bound[sp] = bb;
                    ++sp;
                }
            }
            while (next < 0 && sp > 0) {
                --sp;
                if (stack_bound[sp] <= best.worst()) next = stack[sp];
            }
            if (next < 0) break;
            node = next;
        }
    }
#pragma unroll
    for (int s = 0; s < K; ++s) {
        out_idx[static_cast<int64_t>(row) * K + s] = best.i[s];
        if (out_dist) out_dist[static_cast<int64_t>(row) * K + s] = best.d[s];
    }
}

template <int K>
void launch_query(cudaStream_t s, bool self, int nq, int m, int ng, const float* queries, const float4* sorted, const BvhNode* nodes,
                  int32_t* out_idx, float* out_dist) {
    const unsigned blocks = (nq + kQueryThreads - 1) / kQueryThreads;
    if (self)
        query_kernel<K, true><<<blocks, kQueryThreads, 0, s>>>(nq, m, ng, queries, sorted, nodes, out_idx, out_dist);
    else
        query_kernel<K, false><<<blocks, kQueryThreads, 0, s>>>(nq, m, ng, queries, sorted, nodes, out_idx, out_dist);
}

// The workspace: every array 256-byte aligned, in this order.
struct Layout {
    size_t scene, codes, ids, codes_sorted, ids_sorted, sorted, leaf_codes, leaf_ids, leaf_boxes, node_boxes, nodes, children, parent,
        leaf_parent, flags, sort_temp, sort_bytes, total;
};

Layout layout(int64_t m) {
    const size_t n = static_cast<size_t>(m), ng = (n + kBucket - 1) / kBucket;
    Layout L{};
    size_t off = 0;
    auto take = [&off](size_t bytes) {
        const size_t at = off;
        off += (bytes + 255) & ~static_cast<size_t>(255);
        return at;
    };
    L.scene = take(6 * sizeof(int));
    L.codes = take(n * 4);
    L.ids = take(n * 4);
    L.codes_sorted = take(n * 4);
    L.ids_sorted = take(n * 4);
    L.sorted = take(n * sizeof(float4));
    L.leaf_codes = take(ng * 4);
    L.leaf_ids = take(ng * 4);
    L.leaf_boxes = take(ng * sizeof(Box));
    L.node_boxes = take(ng * sizeof(Box));
    L.nodes = take(ng * sizeof(BvhNode));
    L.children = take(ng * sizeof(int2));
    L.parent = take(ng * 4);
    L.leaf_parent = take(ng * 4);
    L.flags = take(ng * 4);
    L.sort_bytes = sort32_temp_bytes(m);
    L.sort_temp = take(L.sort_bytes);
    L.total = off;
    return L;
}

int knn_fail(const std::string& msg) {
    set_context_free_error("gutb200_knn: " + msg);
    return 1;
}

}  // namespace

extern "C" {

size_t gutb200_knn_workspace_bytes(int64_t n_targets) {
    if (n_targets < 1 || n_targets > INT32_MAX) return 0;
    return layout(n_targets).total;
}

int gutb200_knn(void* stream, int64_t n_targets, const float* targets, int64_t n_queries, const float* queries, int32_t k, void* workspace,
                size_t workspace_bytes, int32_t* out_idx, float* out_dist) {
    const bool self = queries == nullptr;
    if (k < 1 || k > 4) return knn_fail("k=" + std::to_string(k) + " is outside 1..4");
    if (n_targets > INT32_MAX || n_queries > INT32_MAX)
        return knn_fail("n_targets=" + std::to_string(n_targets) + ", n_queries=" + std::to_string(n_queries) + ": sizes above INT32_MAX");
    if (n_queries < 0) return knn_fail("n_queries=" + std::to_string(n_queries) + " is negative");
    if (self && n_queries != n_targets)
        return knn_fail("queries is NULL (the targets query themselves) but n_queries=" + std::to_string(n_queries) + " != n_targets=" +
                        std::to_string(n_targets));
    const int64_t need = self ? k + 1 : k;
    if (n_targets < need)
        return knn_fail("n_targets=" + std::to_string(n_targets) + " < " + std::to_string(need) + (self ? " (k + 1 with self-exclusion)" : " (k)"));
    if (!targets || !workspace || !out_idx) return knn_fail("targets, workspace and out_idx must not be NULL");
    const Layout L = layout(n_targets);
    if (workspace_bytes < L.total)
        return knn_fail("workspace_bytes=" + std::to_string(workspace_bytes) + " < gutb200_knn_workspace_bytes(n_targets)=" + std::to_string(L.total));
    if (n_queries == 0) return 0;

    cudaStream_t s = static_cast<cudaStream_t>(stream);
    char* ws = static_cast<char*>(workspace);
    int* scene = reinterpret_cast<int*>(ws + L.scene);
    uint32_t* codes = reinterpret_cast<uint32_t*>(ws + L.codes);
    uint32_t* ids = reinterpret_cast<uint32_t*>(ws + L.ids);
    uint32_t* codes_sorted = reinterpret_cast<uint32_t*>(ws + L.codes_sorted);
    uint32_t* ids_sorted = reinterpret_cast<uint32_t*>(ws + L.ids_sorted);
    float4* sorted = reinterpret_cast<float4*>(ws + L.sorted);
    uint32_t* leaf_codes = reinterpret_cast<uint32_t*>(ws + L.leaf_codes);
    uint32_t* leaf_ids = reinterpret_cast<uint32_t*>(ws + L.leaf_ids);
    Box* leaf_boxes = reinterpret_cast<Box*>(ws + L.leaf_boxes);
    Box* node_boxes = reinterpret_cast<Box*>(ws + L.node_boxes);
    BvhNode* nodes = reinterpret_cast<BvhNode*>(ws + L.nodes);
    int2* children = reinterpret_cast<int2*>(ws + L.children);
    int* parent = reinterpret_cast<int*>(ws + L.parent);
    int* leaf_parent = reinterpret_cast<int*>(ws + L.leaf_parent);
    int* flags = reinterpret_cast<int*>(ws + L.flags);

    const int m = static_cast<int>(n_targets), nq = static_cast<int>(n_queries);
    const int ng = (m + kBucket - 1) / kBucket;
    const unsigned blocks = (m + 255) / 256, gblocks = (ng + 255) / 256;
    cudaError_t e = cudaMemcpyAsync(scene, kSceneBoxInit, sizeof(kSceneBoxInit), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess && ng > 1) e = cudaMemsetAsync(flags, 0, static_cast<size_t>(ng) * 4, s);
    if (e != cudaSuccess) return knn_fail(cudaGetErrorString(e));
    box_kernel<<<blocks, 256, 0, s>>>(m, targets, scene);
    morton_kernel<<<blocks, 256, 0, s>>>(m, targets, scene, codes, ids);
    run_sort32_pairs(s, ws + L.sort_temp, L.sort_bytes, codes, codes_sorted, ids, ids_sorted, n_targets, 30);
    bucket_kernel<<<gblocks, 256, 0, s>>>(m, ng, codes_sorted, ids_sorted, targets, sorted, leaf_codes, leaf_ids, leaf_boxes);
    if (ng > 1) {
        hierarchy_kernel<<<gblocks, 256, 0, s>>>(ng, leaf_codes, leaf_ids, children, parent, leaf_parent);
        refit_kernel<<<gblocks, 256, 0, s>>>(ng, children, parent, leaf_parent, leaf_boxes, node_boxes, flags, nodes);
    }
    switch (k) {
        case 1: launch_query<1>(s, self, nq, m, ng, queries, sorted, nodes, out_idx, out_dist); break;
        case 2: launch_query<2>(s, self, nq, m, ng, queries, sorted, nodes, out_idx, out_dist); break;
        case 3: launch_query<3>(s, self, nq, m, ng, queries, sorted, nodes, out_idx, out_dist); break;
        default: launch_query<4>(s, self, nq, m, ng, queries, sorted, nodes, out_idx, out_dist); break;
    }
    e = cudaGetLastError();
    if (e != cudaSuccess) return knn_fail(cudaGetErrorString(e));
    return 0;
}

}  // extern "C"
