/*
 * include/grt_b200.h -- C ABI of the H100-native (sm_90a) 3DGRT tracer (same shared library: 3dgrut_b200/libgut_b200.so).
 *
 * Replaces the OptiX-backed pybind class of the reference (threedgrt_tracer/bindings.cpp:32-38,
 * include/3dgrt/optixTracer.h:128-177) -- no RT cores are used, so the acceleration structure is a Morton-code
 * LBVH built and traversed by our own kernels:
 *
 *   grtb200_create / destroy   <- OptixTracer::OptixTracer / ~OptixTracer        (src/optixTracer.cpp:153-343)
 *   grtb200_build_bvh          <- OptixTracer::buildBVH                           (src/optixTracer.cpp:616-890)
 *   grtb200_build_bvh_packed   the same build from the [N,12] particle record (ours: the no-autograd training step)
 *   grtb200_trace              <- OptixTracer::trace   -> __raygen__rg            (src/optixTracer.cpp:893-960, src/kernels/cuda/referenceOptix.cu:103-186)
 *   grtb200_trace_normals      grtb200_trace that also sums the rays' normals (render.enable_normals)
 *   grtb200_trace_bwd          <- OptixTracer::traceBwd -> bwd __raygen__rg        (src/optixTracer.cpp:962-1031, src/kernels/cuda/referenceBwdOptix.cu:103-170)
 *   grtb200_trace_nht / grtb200_trace_bwd_nht  the same with NHT features         (src/kernels/cuda/referenceSlangOptix.cu, referenceSlangBwdOptix.cu)
 *
 * Layouts (fp32): particles [N,12] = pos3, density, quat(wxyz), scale3, pad; sph [N,48]; rays_o/rays_d [B,H,W,3]
 * (R = B*H*W rays, ray space); ray_to_world = first three rows of T_to_world, row major [3,4], HOST pointer
 * (the reference copies it to the host too, optixTracer.cpp:931); out_rgb [R,3], out_alpha [R], out_dist [R,2] =
 * (integrated distance, distance of the last processed hit), out_hits [R], visibility [N].
 * All other pointers are device pointers; `stream` is a cudaStream_t.  Returns 0 on success.
 *
 * Forward state kept for the backward (ours, no reference twin): grtb200_trace records each ray's accepted hits in a buffer owned
 * by the context; grtb200_trace_bwd replays them when it is called with the forward's arguments (same ray / particle / output
 * pointers, pose and BVH) and otherwise re-traces like the reference (src/kernels/cuda/referenceBwdOptix.cu:103-170).
 * The environment variable GRTB200_HITCAP=k, read at each forward, sets the hits recorded per ray (0 = always re-trace); rays with
 * more hits than that are re-traced by the backward.
 */
#ifndef GRT_B200_H
#define GRT_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct grtb200_config {
    int32_t kernel_degree;   /* render.particle_kernel_degree: 4 (3DGRT default) or 2   */
    float min_response;      /* render.particle_kernel_min_response  0.0113              */
    float min_alpha;         /* alphaMinThreshold 1/255 (optixTracer.cpp:928)            */
    float max_alpha;         /* render.particle_kernel_max_alpha 0.99                    */
    int32_t density_clamping; /* render.particle_kernel_density_clamping (true)          */
    int32_t primitive;       /* render.primitive_type: 0 instances (default), 1 icosahedron */
} grtb200_config;

/* grtb200_config.primitive */
#define GRTB200_PRIMITIVE_INSTANCES 0
#define GRTB200_PRIMITIVE_ICOSAHEDRON 1

typedef struct grtb200_ctx grtb200_ctx;

void grtb200_default_config(grtb200_config* cfg);
/* Returns 2 without a usable CUDA device and 5 when cfg->primitive is not one of GRTB200_PRIMITIVE_*. */
int grtb200_create(const grtb200_config* cfg, int device, grtb200_ctx** out);
void grtb200_destroy(grtb200_ctx* ctx);
const char* grtb200_last_error(const grtb200_ctx* ctx);

/* (Re)build the LBVH over the particles' bounding proxies (cfg->primitive: the instance box or the icosahedron; both are traced
 * in the instance space of the particle, no triangles are stored).  `rebuild`/`allow_update` are accepted for API
 * compatibility; every call is a full rebuild (the reference's default config also rebuilds every step). */
int grtb200_build_bvh(grtb200_ctx* ctx, void* stream, int64_t n, const float* pos, const float* rot, const float* scl,
                      const float* dns, int32_t rebuild, int32_t allow_update);

/* The same build from the [N,12] particle record that grtb200_trace reads (pos = cols 0-2, density = col 3, quat = cols 4-7, scale =
 * cols 8-10): the same proxies, scene box and LBVH as grtb200_build_bvh on the same values, bit for bit, without copying the four
 * arrays out first.  Every call is a full rebuild. */
int grtb200_build_bvh_packed(grtb200_ctx* ctx, void* stream, int64_t n, const float* particles);

int grtb200_trace(grtb200_ctx* ctx, void* stream, int64_t n, const float* particles, const float* sph, int32_t sph_degree,
                  float min_transmittance, int32_t batch, int32_t height, int32_t width, const float* rays_o,
                  const float* rays_d, const float* ray_to_world_host, float* out_rgb, float* out_alpha, float* out_dist,
                  float* out_hits, float* visibility);

/* grtb200_trace that also writes the rays' normals (render.enable_normals; <- the `normal` accumulator of processHit,
 * include/3dgrt/kernels/cuda/gaussianParticles.cuh:397-401): out_normals [R,3] = sum over the accepted hits of
 * weight * safe_normalize((gro + grd (dot(grd, -gro) - sqrt(9 - grayDist))) * (R s)), unnormalised, written for every ray (zero where
 * no hit is accepted).  Every other output is bit-identical to grtb200_trace's, and the hit lists it records are replayed by
 * grtb200_trace_bwd / grtb200_trace_bwd_accumulate exactly as grtb200_trace's are.  There is no gradient of the normals (the reference's
 * backward has none).  A particle_kernel_min_response below exp(-4.5) = 0.0111 makes sqrt(9 - grayDist) NaN for some hits, as in the
 * reference.  out_normals must not be null. */
int grtb200_trace_normals(grtb200_ctx* ctx, void* stream, int64_t n, const float* particles, const float* sph, int32_t sph_degree,
                          float min_transmittance, int32_t batch, int32_t height, int32_t width, const float* rays_o,
                          const float* rays_d, const float* ray_to_world_host, float* out_rgb, float* out_alpha, float* out_dist,
                          float* out_hits, float* visibility, float* out_normals);

int grtb200_trace_bwd(grtb200_ctx* ctx, void* stream, int64_t n, const float* particles, const float* sph, int32_t sph_degree,
                      float min_transmittance, int32_t batch, int32_t height, int32_t width, const float* rays_o,
                      const float* rays_d, const float* ray_to_world_host, const float* out_rgb, const float* out_alpha,
                      const float* out_dist, const float* d_rgb, const float* d_alpha, const float* d_dist, float* d_particles,
                      float* d_sph);
/* grtb200_trace_bwd that adds this trace's gradients to what d_particles / d_sph already hold instead of zeroing them first (ours): two
 * passes -- e.g. the 3DGUT primary and the 3DGRT secondary rays of the hybrid step -- write one gradient buffer. */
int grtb200_trace_bwd_accumulate(grtb200_ctx* ctx, void* stream, int64_t n, const float* particles, const float* sph, int32_t sph_degree,
                                 float min_transmittance, int32_t batch, int32_t height, int32_t width, const float* rays_o,
                                 const float* rays_d, const float* ray_to_world_host, const float* out_rgb, const float* out_alpha,
                                 const float* out_dist, const float* d_rgb, const float* d_alpha, const float* d_dist, float* d_particles,
                                 float* d_sph);

/* Neural Harmonic Texture (NHT) features instead of SH radiance (model.feature_type: nht; <- the referenceSlang / referenceSlangBwd
 * pipelines, src/kernels/cuda/referenceSlangOptix.cu:103-200, referenceSlangBwdOptix.cu:103-230).  features: [N,feature_dim] rows,
 * fp32, or fp16 when features_half != 0; only feature_dim = 48 (4 tetrahedron vertices x 12, barycentric, sincos x 1) is built, other
 * dims are refused.  out_features [R,24] fp32 (sin / cos of the 12 blended features), d_features_out its gradient, d_features [N,48]
 * fp32 (zeroed by the call).  Every other argument, output and the hit-list replay are as in grtb200_trace / grtb200_trace_bwd; the
 * backward replays only the lists of an NHT forward with the same feature row layout and otherwise re-traces. */
int grtb200_trace_nht(grtb200_ctx* ctx, void* stream, int64_t n, const float* particles, const void* features, int32_t feature_dim,
                      int32_t features_half, float min_transmittance, int32_t batch, int32_t height, int32_t width, const float* rays_o,
                      const float* rays_d, const float* ray_to_world_host, float* out_features, float* out_alpha, float* out_dist,
                      float* out_hits, float* visibility);

int grtb200_trace_bwd_nht(grtb200_ctx* ctx, void* stream, int64_t n, const float* particles, const void* features, int32_t feature_dim,
                          int32_t features_half, float min_transmittance, int32_t batch, int32_t height, int32_t width, const float* rays_o,
                          const float* rays_d, const float* ray_to_world_host, const float* out_features, const float* out_alpha,
                          const float* out_dist, const float* d_features_out, const float* d_alpha, const float* d_dist, float* d_particles,
                          float* d_features);

/* Scene bounding box of the last build: min xyz, max xyz (host array of 6 floats; synchronises). */
int grtb200_scene_aabb(grtb200_ctx* ctx, float* aabb6);

int64_t grtb200_launch_count(const grtb200_ctx* ctx);

/* The forward records each ray's accepted hits so that the backward replays them instead of re-tracing (ours; bounded to 1 GiB, the per-ray
 * capacity shrinks for large ray batches).  enable = 0 switches the recording off and frees the cache: inference-only callers. */
int grtb200_set_replay(grtb200_ctx* ctx, int32_t enable);

/* Measurement helper (debug, synchronises, writes no image): work counters of one forward trace with the arguments of grtb200_trace.
 * counters8 = { rays, k-nearest queries, node visits (one per warp and node for packet-walked rays, else per lane), box tests,
 * proxy tests, candidate hits processed, accepted hits, rays walked as packets }; visibility_scratch: device [N] floats. */
int grtb200_debug_trace_counters(grtb200_ctx* ctx, void* stream, int64_t n, const float* particles, const float* sph, int32_t sph_degree,
                                 float min_transmittance, int32_t batch, int32_t height, int32_t width, const float* rays_o,
                                 const float* rays_d, const float* ray_to_world_host, float* visibility_scratch, uint64_t* counters8);

/* ---- Playground: triangle meshes inside a trained scene (forward only; DESIGN.md section 22) -------------------------------------------
 *
 *   grtb200_mesh_create / destroy / last_error   a handle that owns one LBVH over the triangles of all inserted meshes
 *   grtb200_build_mesh_bvh                       (re)build it: call when the meshes change, not per frame
 *   grtb200_mesh_closest_hit                     closest hit of world-space rays (t in (1e-5, 1e5), both faces, ties -> lowest index)
 *   grtb200_trace_playground                     <- the Playground's __raygen__rg (threedgrut_playground/src/kernels/cuda/playgroundKernel.cu)
 *
 * Mesh layouts (device, world space): vertices [V,3] fp32; vertex_normals [V,3] fp32 unit normals; faces [F,3] int32; face_material [F]
 * int32 rows of materials [M,8] fp32 = (kind, ior, 0, 0, r, g, b, 0) with kind one of GRTB200_MATERIAL_*.  The build copies all of it.
 */
#define GRTB200_MATERIAL_MIRROR 0
#define GRTB200_MATERIAL_GLASS 1
#define GRTB200_MATERIAL_DIFFUSE 2

typedef struct grtb200_mesh grtb200_mesh;

/* Returns 2 without a usable CUDA device. */
int grtb200_mesh_create(int device, grtb200_mesh** out);
void grtb200_mesh_destroy(grtb200_mesh* mesh);
const char* grtb200_mesh_last_error(const grtb200_mesh* mesh);
/* Synchronises `stream` (before replacing the previous tree and after the build).  n_faces = 0 leaves an empty mesh set. */
int grtb200_build_mesh_bvh(grtb200_mesh* mesh, void* stream, int64_t n_vertices, const float* vertices, const float* vertex_normals,
                           int64_t n_faces, const int32_t* faces, const int32_t* face_material, int32_t n_materials, const float* materials);
/* rays_o / rays_d [R,3] world space; out_t [R] (1e5 where nothing is hit), out_tri [R] int32 (-1 where nothing is hit). */
int grtb200_mesh_closest_hit(grtb200_mesh* mesh, void* stream, int64_t n_rays, const float* rays_o, const float* rays_d, float* out_t,
                             int32_t* out_tri);

/* Forward render of the Gaussians of the last grtb200_build_bvh with the meshes of `mesh` (null: no meshes) inserted.  Arguments up to
 * ray_to_world_host are grtb200_trace's (SH radiance).  Each ray alternates a closest mesh hit and the k-nearest Gaussian walk of
 * grtb200_trace on the segment up to it (to ray_max_t [R], or 1e9 where ray_max_t is null, when no mesh is hit), with one transmittance
 * carried through every segment; mirror and glass redirect the ray (at most 32 mirror bounces, 1000 segments), diffuse ends it.  The ray
 * stops once its alpha reaches 0.995.  smooth_normals: interpolated vertex normals, else the triangle's own.  background_host: 3 floats
 * (host), composited on 1 - alpha.  out_rgb [R,3] and out_alpha [R] are clamped to [0, 1]; visibility [N] marks the Gaussians hit.  A ray
 * that meets no mesh gets grtb200_trace's radiance and alpha exactly (then composited and clamped).  Records no hit lists. */
int grtb200_trace_playground(grtb200_ctx* ctx, void* stream, const grtb200_mesh* mesh, int64_t n, const float* particles, const float* sph,
                             int32_t sph_degree, float min_transmittance, int32_t batch, int32_t height, int32_t width, const float* rays_o,
                             const float* rays_d, const float* ray_to_world_host, const float* ray_max_t, const float* background_host,
                             int32_t smooth_normals, float* out_rgb, float* out_alpha, float* visibility);

#ifdef __cplusplus
}
#endif
#endif
