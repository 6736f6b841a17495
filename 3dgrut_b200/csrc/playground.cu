// 3dgrut_b200/csrc/playground.cu -- the triangle LBVH of the playground meshes (DESIGN.md section 22).  C ABI: include/grt_b200.h.
//
// One build per change of the meshes: a box and a centroid per triangle, 30-bit Morton codes of the centroids in their bounding box
// (lbvh.cuh), the same radix sort of (key, triangle) pairs as the 3DGRT build (run_sort32_pairs), the Karras topology and the
// bottom-up refit (lbvh.cuh).  Leaves hold one triangle each; a leaf's index in the tree is its triangle index.  The tree, the
// triangles, the vertex normals and the material table are device copies owned by the grtb200_mesh handle, so the caller's arrays may go
// away after the build.  The closest-hit walk is mesh_bvh.cuh; grtb200_mesh_closest_hit runs it on a batch of world-space rays.
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <new>
#include <string>

#include "../../include/grt_b200.h"
#include "mesh_bvh.cuh"

namespace gutb200 {
size_t sort32_temp_bytes(int64_t n);
void run_sort32_pairs(cudaStream_t s, void* temp, size_t temp_bytes, const uint32_t* kin, uint32_t* kout, const uint32_t* vin,
                      uint32_t* vout, int64_t n, int end_bit);
}  // namespace gutb200

struct grtb200_mesh {
    int device = 0;
    std::string error;
    int ntri = 0, nvert = 0, nmat = 0;
    void *nodes = nullptr, *tris = nullptr, *faces = nullptr, *vnormals = nullptr, *tri_material = nullptr, *materials = nullptr;
};

namespace {

int fail(grtb200_mesh* m, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (m) m->error = buf;
    return 1;
}

#define MESH_CUDA(m, expr)                                                                           \
    do {                                                                                             \
        cudaError_t e__ = (expr);                                                                    \
        if (e__ != cudaSuccess) return fail(m, "%s failed: %s", #expr, cudaGetErrorString(e__));     \
    } while (0)

void release(grtb200_mesh* m) {
    void** ptrs[] = {&m->nodes, &m->tris, &m->faces, &m->vnormals, &m->tri_material, &m->materials};
    for (void** p : ptrs) {
        if (*p) cudaFree(*p);
        *p = nullptr;
    }
    m->ntri = m->nvert = m->nmat = 0;
}

// per triangle: (v0, e1, e2), its box padded by 1e-6 of its largest coordinate (the walk's slab tests round), its centroid into the
// centroid box
__global__ void __launch_bounds__(256) triangle_kernel(int nf, const float* __restrict__ vertices, const int* __restrict__ faces,
                                                       float4* __restrict__ tris, Box* __restrict__ boxes, float4* __restrict__ centroids,
                                                       int* __restrict__ scene) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nf) return;
    const int a = faces[3 * i], b = faces[3 * i + 1], c = faces[3 * i + 2];
    const float ax = vertices[3 * a], ay = vertices[3 * a + 1], az = vertices[3 * a + 2];
    const float bx = vertices[3 * b], by = vertices[3 * b + 1], bz = vertices[3 * b + 2];
    const float cx = vertices[3 * c], cy = vertices[3 * c + 1], cz = vertices[3 * c + 2];
    tris[3 * i] = make_float4(ax, ay, az, 0.f);
    tris[3 * i + 1] = make_float4(__fsub_rn(bx, ax), __fsub_rn(by, ay), __fsub_rn(bz, az), 0.f);
    tris[3 * i + 2] = make_float4(__fsub_rn(cx, ax), __fsub_rn(cy, ay), __fsub_rn(cz, az), 0.f);
    const float lx = fminf(ax, fminf(bx, cx)), ly = fminf(ay, fminf(by, cy)), lz = fminf(az, fminf(bz, cz));
    const float hx = fmaxf(ax, fmaxf(bx, cx)), hy = fmaxf(ay, fmaxf(by, cy)), hz = fmaxf(az, fmaxf(bz, cz));
    const float big = fmaxf(fmaxf(fmaxf(fabsf(lx), fabsf(hx)), fmaxf(fabsf(ly), fabsf(hy))), fmaxf(fabsf(lz), fabsf(hz)));
    const float pad = 1e-6f * big + 1e-30f;
    Box bx_;
    bx_.lo = make_float4(lx - pad, ly - pad, lz - pad, 0.f);
    bx_.hi = make_float4(hx + pad, hy + pad, hz + pad, 0.f);
    boxes[i] = bx_;
    const float mx = (ax + bx + cx) * (1.f / 3.f), my = (ay + by + cy) * (1.f / 3.f), mz = (az + bz + cz) * (1.f / 3.f);
    centroids[i] = make_float4(mx, my, mz, 0.f);
    scene_box_extend(scene, mx, my, mz, mx, my, mz);
}

__global__ void __launch_bounds__(256) centroid_morton_kernel(int nf, const float4* __restrict__ centroids, const int* __restrict__ scene,
                                                              uint32_t* __restrict__ codes, uint32_t* __restrict__ ids) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nf) return;
    const SceneBox sb = scene_box(scene);
    const float4 c = centroids[i];
    codes[i] = morton30(sb, c.x, c.y, c.z);
    ids[i] = static_cast<uint32_t>(i);
}

// one triangle: its box on the left, an unreachable point (3e38, 3e38, 3e38) on the right (as grt.cu's single_leaf_kernel)
__global__ void single_triangle_kernel(const Box* __restrict__ boxes, BvhNode* __restrict__ nodes) {
    const Box l = boxes[0];
    BvhNode nd;
    nd.b0 = make_float4(l.lo.x, l.lo.y, l.lo.z, l.hi.x);
    nd.b1 = make_float4(l.hi.y, l.hi.z, 3e38f, 3e38f);
    nd.b2 = make_float4(3e38f, 3e38f, 3e38f, 3e38f);
    nd.meta = make_float4(__int_as_float(~0), __int_as_float(~0), 0.f, 0.f);
    nodes[0] = nd;
}

__global__ void __launch_bounds__(128) closest_hit_kernel(gutb200::MeshView M, int64_t nrays, const float* __restrict__ rays_o,
                                                          const float* __restrict__ rays_d, float* __restrict__ out_t, int* __restrict__ out_tri) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= nrays) return;
    const MeshHit h = mesh_closest_hit(M, rays_o[3 * i], rays_o[3 * i + 1], rays_o[3 * i + 2], rays_d[3 * i], rays_d[3 * i + 1], rays_d[3 * i + 2]);
    out_t[i] = h.tri >= 0 ? h.t : kMeshTMax;
    out_tri[i] = h.tri;
}

}  // namespace

namespace gutb200 {

MeshView mesh_view(const grtb200_mesh* m) {
    MeshView v;
    v.ntri = m ? m->ntri : 0;
    v.nodes = m ? static_cast<const float4*>(m->nodes) : nullptr;
    v.tris = m ? static_cast<const float4*>(m->tris) : nullptr;
    v.faces = m ? static_cast<const int*>(m->faces) : nullptr;
    v.vnormals = m ? static_cast<const float*>(m->vnormals) : nullptr;
    v.tri_material = m ? static_cast<const int*>(m->tri_material) : nullptr;
    v.materials = m ? static_cast<const float4*>(m->materials) : nullptr;
    return v;
}

}  // namespace gutb200

extern "C" {

int grtb200_mesh_create(int device, grtb200_mesh** out) {
    if (!out) return 1;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count) return 2;  // no CPU fallback
    grtb200_mesh* m = new (std::nothrow) grtb200_mesh();
    if (!m) return 3;
    m->device = device;
    *out = m;
    return 0;
}

void grtb200_mesh_destroy(grtb200_mesh* m) {
    if (!m) return;
    cudaSetDevice(m->device);
    cudaDeviceSynchronize();
    release(m);
    delete m;
}

const char* grtb200_mesh_last_error(const grtb200_mesh* m) { return m ? m->error.c_str() : "null mesh"; }

int grtb200_build_mesh_bvh(grtb200_mesh* m, void* stream, int64_t n_vertices, const float* vertices, const float* vertex_normals,
                           int64_t n_faces, const int32_t* faces, const int32_t* face_material, int32_t n_materials, const float* materials) {
    if (!m) return 1;
    if (n_faces < 0 || n_faces > 0x3FFFFFFF || n_vertices < 0 || n_vertices > 0x3FFFFFFF)
        return fail(m, "mesh size out of range: %lld vertices, %lld faces", static_cast<long long>(n_vertices), static_cast<long long>(n_faces));
    if (n_faces > 0 && (!vertices || !vertex_normals || !faces || !face_material || !materials || n_materials <= 0))
        return fail(m, "mesh arrays are null or the material table is empty");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    MESH_CUDA(m, cudaSetDevice(m->device));
    MESH_CUDA(m, cudaStreamSynchronize(s));  // the previous tree may still be read by work queued on this stream
    release(m);
    if (n_faces == 0) return 0;
    const int nf = static_cast<int>(n_faces);
    const size_t nv = static_cast<size_t>(n_vertices);
    MESH_CUDA(m, cudaMalloc(&m->nodes, static_cast<size_t>(nf) * sizeof(BvhNode)));
    MESH_CUDA(m, cudaMalloc(&m->tris, static_cast<size_t>(nf) * 3 * sizeof(float4)));
    MESH_CUDA(m, cudaMalloc(&m->faces, static_cast<size_t>(nf) * 3 * 4));
    MESH_CUDA(m, cudaMalloc(&m->vnormals, nv * 3 * 4 + 4));
    MESH_CUDA(m, cudaMalloc(&m->tri_material, static_cast<size_t>(nf) * 4));
    MESH_CUDA(m, cudaMalloc(&m->materials, static_cast<size_t>(n_materials) * 2 * sizeof(float4)));
    MESH_CUDA(m, cudaMemcpyAsync(m->faces, faces, static_cast<size_t>(nf) * 3 * 4, cudaMemcpyDeviceToDevice, s));
    MESH_CUDA(m, cudaMemcpyAsync(m->vnormals, vertex_normals, nv * 3 * 4, cudaMemcpyDeviceToDevice, s));
    MESH_CUDA(m, cudaMemcpyAsync(m->tri_material, face_material, static_cast<size_t>(nf) * 4, cudaMemcpyDeviceToDevice, s));
    MESH_CUDA(m, cudaMemcpyAsync(m->materials, materials, static_cast<size_t>(n_materials) * 2 * sizeof(float4), cudaMemcpyDeviceToDevice, s));
    // build scratch, freed before returning (a rebuild happens only when the meshes change)
    const size_t cap = static_cast<size_t>(nf) + 16;
    void *boxes = nullptr, *node_boxes = nullptr, *centroids = nullptr, *codes = nullptr, *ids = nullptr, *codes_sorted = nullptr,
         *ids_sorted = nullptr, *children = nullptr, *parent = nullptr, *leaf_parent = nullptr, *flags = nullptr, *scene = nullptr,
         *temp = nullptr;
    const size_t temp_bytes = gutb200::sort32_temp_bytes(static_cast<int64_t>(cap)) + 16;
    void** scratch[] = {&boxes, &node_boxes, &centroids, &codes, &ids, &codes_sorted, &ids_sorted, &children, &parent, &leaf_parent, &flags,
                        &scene, &temp};
    const size_t bytes[] = {cap * sizeof(Box), cap * sizeof(Box), cap * sizeof(float4), cap * 4, cap * 4, cap * 4, cap * 4, cap * sizeof(int2),
                            cap * 4, cap * 4, cap * 4, 6 * sizeof(int), temp_bytes};
    cudaError_t e = cudaSuccess;
    for (int k = 0; k < 13 && e == cudaSuccess; ++k) e = cudaMalloc(scratch[k], bytes[k]);
    const unsigned blocks = (nf + 255) / 256;
    if (e == cudaSuccess) e = cudaMemcpyAsync(scene, kSceneBoxInit, sizeof(kSceneBoxInit), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) {
        triangle_kernel<<<blocks, 256, 0, s>>>(nf, vertices, faces, static_cast<float4*>(m->tris), static_cast<Box*>(boxes),
                                               static_cast<float4*>(centroids), static_cast<int*>(scene));
        centroid_morton_kernel<<<blocks, 256, 0, s>>>(nf, static_cast<const float4*>(centroids), static_cast<const int*>(scene),
                                                      static_cast<uint32_t*>(codes), static_cast<uint32_t*>(ids));
        gutb200::run_sort32_pairs(s, temp, temp_bytes, static_cast<const uint32_t*>(codes), static_cast<uint32_t*>(codes_sorted),
                                  static_cast<const uint32_t*>(ids), static_cast<uint32_t*>(ids_sorted), nf, 30);
        if (nf == 1) {
            single_triangle_kernel<<<1, 1, 0, s>>>(static_cast<const Box*>(boxes), static_cast<BvhNode*>(m->nodes));
        } else {
            e = cudaMemsetAsync(flags, 0, static_cast<size_t>(nf) * 4, s);
            hierarchy_kernel<<<blocks, 256, 0, s>>>(nf, static_cast<const uint32_t*>(codes_sorted), static_cast<const uint32_t*>(ids_sorted),
                                                    static_cast<int2*>(children), static_cast<int*>(parent), static_cast<int*>(leaf_parent));
            refit_kernel<<<blocks, 256, 0, s>>>(nf, static_cast<const int2*>(children), static_cast<const int*>(parent),
                                                static_cast<const int*>(leaf_parent), static_cast<const Box*>(boxes),
                                                static_cast<Box*>(node_boxes), static_cast<int*>(flags), static_cast<BvhNode*>(m->nodes));
        }
        if (e == cudaSuccess) e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);  // before the scratch is freed
    }
    for (void** p : scratch)
        if (*p) cudaFree(*p);
    if (e != cudaSuccess) {
        release(m);
        return fail(m, "mesh BVH build failed: %s", cudaGetErrorString(e));
    }
    m->ntri = nf;
    m->nvert = static_cast<int>(n_vertices);
    m->nmat = n_materials;
    return 0;
}

int grtb200_mesh_closest_hit(grtb200_mesh* m, void* stream, int64_t n_rays, const float* rays_o, const float* rays_d, float* out_t,
                             int32_t* out_tri) {
    if (!m) return 1;
    if (n_rays < 0) return fail(m, "n_rays %lld out of range", static_cast<long long>(n_rays));
    if (n_rays == 0) return 0;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    MESH_CUDA(m, cudaSetDevice(m->device));
    const unsigned blocks = static_cast<unsigned>((n_rays + 127) / 128);
    closest_hit_kernel<<<blocks, 128, 0, s>>>(gutb200::mesh_view(m), n_rays, rays_o, rays_d, out_t, out_tri);
    MESH_CUDA(m, cudaGetLastError());
    return 0;
}

}  // extern "C"
