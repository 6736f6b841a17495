// 3dgrut_b200/csrc/gut_api.cu -- C ABI (include/gut_b200.h) and host orchestration of the 3DGUT path.
//
// Mirrors the host side of the reference (threedgut_tracer/src/splatRaster.cpp:184-350 and
// src/gutRenderer.cu:99-232,241-519): per-object scratch cache that only grows, forward context reused by the
// following backward, all work enqueued on the caller's stream.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>

#include "gut_common.cuh"

using namespace gutb200;

namespace {

// ---------------------------------------------------------------------------------------------------------
// host pose maths, fp32, same operation order as tcnn's vec.h used by include/3dgut/sensors/sensors.h:44-73

struct Quat {
    float w, x, y, z;
};
struct Mat3 {
    float m[3][3];  // column major: m[c][r]
};
struct Pose {
    float t[3];
    Quat q;
};

Mat3 to_mat3(const Quat& q) {
    const float qxx = q.x * q.x, qyy = q.y * q.y, qzz = q.z * q.z;
    const float qxz = q.x * q.z, qxy = q.x * q.y, qyz = q.y * q.z;
    const float qwx = q.w * q.x, qwy = q.w * q.y, qwz = q.w * q.z;
    Mat3 r;
    r.m[0][0] = 1.f - 2.f * (qyy + qzz); r.m[0][1] = 2.f * (qxy + qwz); r.m[0][2] = 2.f * (qxz - qwy);
    r.m[1][0] = 2.f * (qxy - qwz); r.m[1][1] = 1.f - 2.f * (qxx + qzz); r.m[1][2] = 2.f * (qyz + qwx);
    r.m[2][0] = 2.f * (qxz + qwy); r.m[2][1] = 2.f * (qyz - qwx); r.m[2][2] = 1.f - 2.f * (qxx + qyy);
    return r;
}

Quat to_quat(const Mat3& a) {
    const float(*m)[3] = a.m;
    Quat q;
    const float tr = m[0][0] + m[1][1] + m[2][2];
    if (tr > 0.f) {
        const float S = std::sqrt(tr + 1.f) * 2.f;
        q = {0.25f * S, (m[1][2] - m[2][1]) / S, (m[2][0] - m[0][2]) / S, (m[0][1] - m[1][0]) / S};
    } else if (m[0][0] > m[1][1] && m[0][0] > m[2][2]) {
        const float S = std::sqrt(1.f + m[0][0] - m[1][1] - m[2][2]) * 2.f;
        q = {(m[1][2] - m[2][1]) / S, 0.25f * S, (m[1][0] + m[0][1]) / S, (m[2][0] + m[0][2]) / S};
    } else if (m[1][1] > m[2][2]) {
        const float S = std::sqrt(1.f + m[1][1] - m[0][0] - m[2][2]) * 2.f;
        q = {(m[2][0] - m[0][2]) / S, (m[1][0] + m[0][1]) / S, 0.25f * S, (m[2][1] + m[1][2]) / S};
    } else {
        const float S = std::sqrt(1.f + m[2][2] - m[0][0] - m[1][1]) * 2.f;
        q = {(m[0][1] - m[1][0]) / S, (m[2][0] + m[0][2]) / S, (m[2][1] + m[1][2]) / S, 0.25f * S};
    }
    return q;
}

Quat slerp(const Quat& x, const Quat& y, float t) {
    Quat z = y;
    float c = (x.w * y.w + x.x * y.x) + (x.y * y.y + x.z * y.z);
    if (c < 0.f) {
        z = {-y.w, -y.x, -y.y, -y.z};
        c = -c;
    }
    if (c > 1.f - 1.1920929e-07f) {
        const float a = 1.f - t;
        return {x.w * a + z.w * t, x.x * a + z.x * t, x.y * a + z.y * t, x.z * a + z.z * t};
    }
    const float ang = std::acos(c);
    const float s0 = std::sin((1.f - t) * ang), s1 = std::sin(t * ang), sd = std::sin(ang);
    return {(s0 * x.w + s1 * z.w) / sd, (s0 * x.x + s1 * z.x) / sd, (s0 * x.y + s1 * z.y) / sd, (s0 * x.z + s1 * z.z) / sd};
}

Pose pose_from7(const float* p) { return Pose{{p[0], p[1], p[2]}, Quat{p[6], p[3], p[4], p[5]}}; }

Pose pose_inverse(const Pose& p) {
    const Mat3 r = to_mat3(p.q);
    Mat3 inv;
    for (int c = 0; c < 3; ++c)
        for (int k = 0; k < 3; ++k) inv.m[c][k] = r.m[k][c];
    Pose o;
    o.q = to_quat(inv);
    for (int j = 0; j < 3; ++j) {
        float acc = 0.f;
        acc += (-1.0f * inv.m[0][j]) * p.t[0];
        acc += (-1.0f * inv.m[1][j]) * p.t[1];
        acc += (-1.0f * inv.m[2][j]) * p.t[2];
        o.t[j] = acc;
    }
    return o;
}

void pose_cols(const Pose& p, float cols[12]) {
    const Mat3 r = to_mat3(p.q);
    for (int c = 0; c < 3; ++c)
        for (int k = 0; k < 3; ++k) cols[c * 3 + k] = r.m[c][k];
    cols[9] = p.t[0];
    cols[10] = p.t[1];
    cols[11] = p.t[2];
}

// ---------------------------------------------------------------------------------------------------------

struct DeviceBuffer {
    void* ptr = nullptr;
    size_t bytes = 0;
    // grow-only like the reference's CudaBuffer (src/cudaBuffer.cpp:44-119); new memory is zero-filled
    cudaError_t reserve(size_t want, cudaStream_t s, bool zero = false) {
        if (want <= bytes) return cudaSuccess;
        if (ptr) {
            cudaError_t e = cudaFreeAsync(ptr, s);
            if (e != cudaSuccess) return e;
            ptr = nullptr;
            bytes = 0;
        }
        const size_t padded = (want + (want >> 3) + 255) & ~size_t(255);
        cudaError_t e = cudaMallocAsync(&ptr, padded, s);
        if (e != cudaSuccess) return e;
        bytes = padded;
        if (zero) e = cudaMemsetAsync(ptr, 0, padded, s);
        return e;
    }
    void release() {
        if (ptr) cudaFree(ptr);
        ptr = nullptr;
        bytes = 0;
    }
    template <typename T>
    T* as() const { return static_cast<T*>(ptr); }
};

}  // namespace

struct gutb200_ctx {
    gutb200_config cfg;
    int device = 0;
    std::string error;
    cudaStream_t own_stream = nullptr;

    // forward context (reused by backward): per particle
    DeviceBuffer tiles_count, proj, depth, rgb, grad_acc;
    // per intersection: 64-bit (depth bits << 32 | particle) keys in per-tile slices, sorted particle indices, hit words
    DeviceBuffer keys64, keys64_alt, vals_out, hit_words;
    // per tile: list-length histogram, slot counters, ranges, heaviest-first order, hit-word slice offsets; {I, overflow} on the device;
    // per-CTA partial sums of the tile scan
    DeviceBuffer tile_hist, tile_fill, sub_base, ranges, tile_order, chunk_base, totals, scan_parts;
    cudaEvent_t ev_total = nullptr;
    gutb200_camera fwd_camera{};   // the camera of the forward whose context the backward replays
    // host staging for the *_host entry points
    DeviceBuffer h_particles, h_sph, h_rays_o, h_rays_d, h_rgba, h_dist, h_hits, h_vis, h_drgba, h_ddist, h_dpart, h_dsph;
    uint32_t* pinned_total = nullptr;

    FrameCamera cam{};
    FrameConfig fcfg{};
    int64_t n = -1, num_isect = 0, num_tiles = 0;
    bool have_forward = false;
    bool fwd_nht = false;          // the forward rendered NHT features (gutb200_forward_nht): only gutb200_backward_nht may follow
    cudaStream_t fwd_stream = nullptr;

    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    double fwd_ms = 0, bwd_ms = 0;
    int fwd_calls = 0, bwd_calls = 0;
    bool fwd_pending = false, bwd_pending = false;
    int64_t launches = 0;

    // per-stage device timers (enable_timings >= 2): project, scan, expand, sort, ranges, render, render_bwd, project_bwd
    cudaEvent_t st_ev[8][2] = {};
    bool st_pending[8] = {};
    double st_ms[8] = {};
    int st_calls[8] = {};
};

namespace {

int fail(gutb200_ctx* c, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (c) c->error = buf;
    return 1;
}

#define GUT_CUDA(ctx, expr)                                                                             \
    do {                                                                                                \
        cudaError_t e__ = (expr);                                                                       \
        if (e__ != cudaSuccess) return fail(ctx, "%s failed: %s", #expr, cudaGetErrorString(e__));      \
    } while (0)

void fill_frame(gutb200_ctx* c, const gutb200_camera* cam) {
    FrameCamera& f = c->cam;
    f.width = cam->width;
    f.height = cam->height;
    f.grid_x = (cam->width + kTile - 1) / kTile;
    f.grid_y = (cam->height + kTile - 1) / kTile;
    f.fx = cam->focal[0]; f.fy = cam->focal[1];
    f.cx = cam->principal[0]; f.cy = cam->principal[1];
    memcpy(f.radial, cam->radial, sizeof(f.radial));
    memcpy(f.tangential, cam->tangential, sizeof(f.tangential));
    memcpy(f.thin_prism, cam->thin_prism, sizeof(f.thin_prism));
    f.has_distortion = 0;
    for (float v : cam->radial) f.has_distortion |= (v != 0.f);
    for (float v : cam->tangential) f.has_distortion |= (v != 0.f);
    for (float v : cam->thin_prism) f.has_distortion |= (v != 0.f);
    f.res_x = static_cast<float>(cam->width);
    f.res_y = static_cast<float>(cam->height);
    f.model = cam->model;
    f.max_angle = cam->max_angle;
    f.ft_reference_poly = cam->ftheta_reference_poly;
    memcpy(f.ft_bw, cam->ftheta_bw, sizeof(f.ft_bw));
    memcpy(f.ft_fw, cam->ftheta_fw, sizeof(f.ft_fw));
    memcpy(f.ft_cde, cam->ftheta_cde, sizeof(f.ft_cde));
    const Pose ps = pose_from7(cam->pose_start), pe = pose_from7(cam->pose_end);
    const Mat3 rs = to_mat3(ps.q);
    for (int cc = 0; cc < 3; ++cc)
        for (int k = 0; k < 3; ++k) f.rot_start[cc * 3 + k] = rs.m[cc][k];
    for (int k = 0; k < 3; ++k) f.t_start[k] = ps.t[k];
    f.rolling_shutter = cam->rolling_shutter;
    f.rs_iterations = c->cfg.n_rolling_shutter_iterations;
    f.q_start[0] = ps.q.w; f.q_start[1] = ps.q.x; f.q_start[2] = ps.q.y; f.q_start[3] = ps.q.z;
    f.q_end[0] = pe.q.w; f.q_end[1] = pe.q.x; f.q_end[2] = pe.q.y; f.q_end[3] = pe.q.z;
    for (int k = 0; k < 3; ++k) f.t_end[k] = pe.t[k];
    // pose at mid exposure (gutRenderer.cu:266-267)
    Pose mid;
    mid.q = slerp(ps.q, pe.q, 0.5f);
    for (int k = 0; k < 3; ++k) mid.t[k] = ps.t[k] * (1.f - 0.5f) + pe.t[k] * 0.5f;
    const Pose inv = pose_inverse(mid);
    pose_cols(mid, f.view);
    pose_cols(inv, f.s2w);
    for (int k = 0; k < 3; ++k) f.cam_pos[k] = inv.t[k];

    FrameConfig& g = c->fcfg;
    const gutb200_config& s = c->cfg;
    g.kernel_degree = s.kernel_degree;
    g.min_kernel_density = s.min_kernel_density;
    g.min_alpha = s.min_alpha;
    g.max_alpha = s.max_alpha;
    g.min_transmittance = s.min_transmittance;
    g.ut_delta = s.ut_delta;
    g.ut_margin = s.ut_margin;
    const float D = 3.f;
    const float lambda = s.ut_alpha * s.ut_alpha * (D + s.ut_kappa) - D;
    g.w0_mean = lambda / (D + lambda);
    g.wi = 1.f / (2.f * (D + lambda));
    g.w0_cov = lambda / (D + lambda) + (1.f - s.ut_alpha * s.ut_alpha + s.ut_beta);
    g.rect_bounding = s.rect_bounding;
    g.tight_opacity_bounding = s.tight_opacity_bounding;
    g.tile_culling = s.tile_culling;
    g.global_z_order = s.global_z_order;
    g.subtile_culling = s.subtile_culling;
    g.k_buffer_size = s.k_buffer_size;
}

int check_args(gutb200_ctx* c, const gutb200_camera* cam, int64_t n, const void* particles, int32_t sph_degree) {
    if (!c) return 1;
    if (sph_degree < 0 || sph_degree > 3) return fail(c, "sph_degree %d out of range (0..3)", sph_degree);
    if (!cam || cam->width <= 0 || cam->height <= 0) return fail(c, "invalid camera resolution");
    if (cam->rolling_shutter < 0 || cam->rolling_shutter > 4) return fail(c, "rolling_shutter %d out of range (0 global, 1..4 readout directions)", cam->rolling_shutter);
    if (cam->model < 0 || cam->model > 2) return fail(c, "camera model %d unknown (0 = OpenCV pinhole, 1 = OpenCV fisheye, 2 = f-theta)", cam->model);
    if (n < 0 || n > 0x7FFFFFFF) return fail(c, "particle count %lld out of range", static_cast<long long>(n));
    if (reinterpret_cast<uintptr_t>(particles) & 15) return fail(c, "particle buffer must be 16-byte aligned");
    if (c->cfg.k_buffer_size < 0 || c->cfg.k_buffer_size > 16) return fail(c, "k_buffer_size %d out of range (0..16)", c->cfg.k_buffer_size);
    if (c->cfg.kernel_degree != 2 && c->cfg.kernel_degree != 4) return fail(c, "kernel_degree %d not built (2 or 4)", c->cfg.kernel_degree);
    if (((c->cfg.subtile_culling >> 4) & 3) == 3)
        return fail(c, "subtile_culling sub-block code 3 (bits 4-5) not built (0 = quarter-warps, 1 = half-warps, 2 = whole warps)");
    return 0;
}

struct StageTimer {  // RAII event pair around one stage on the launching stream
    gutb200_ctx* c;
    int id;
    cudaStream_t s;
    bool on;
    StageTimer(gutb200_ctx* ctx, int stage, cudaStream_t stream) : c(ctx), id(stage), s(stream), on(ctx->cfg.enable_timings >= 2) {
        if (on) {
            if (!c->st_ev[id][0]) {
                cudaEventCreate(&c->st_ev[id][0]);
                cudaEventCreate(&c->st_ev[id][1]);
            }
            cudaEventRecord(c->st_ev[id][0], s);
        }
    }
    ~StageTimer() {
        if (on) {
            cudaEventRecord(c->st_ev[id][1], s);
            c->st_pending[id] = true;
        }
    }
};

void drain_timers(gutb200_ctx* c) {
    float ms = 0.f;
    for (int i = 0; i < 8; ++i) {
        if (c->st_pending[i] && cudaEventSynchronize(c->st_ev[i][1]) == cudaSuccess &&
            cudaEventElapsedTime(&ms, c->st_ev[i][0], c->st_ev[i][1]) == cudaSuccess) {
            c->st_ms[i] += ms;
            c->st_calls[i]++;
        }
        c->st_pending[i] = false;
    }
    if (c->fwd_pending && cudaEventSynchronize(c->ev[1]) == cudaSuccess && cudaEventElapsedTime(&ms, c->ev[0], c->ev[1]) == cudaSuccess) {
        c->fwd_ms += ms;
        c->fwd_calls++;
    }
    c->fwd_pending = false;
    if (c->bwd_pending && cudaEventSynchronize(c->ev[3]) == cudaSuccess && cudaEventElapsedTime(&ms, c->ev[2], c->ev[3]) == cudaSuccess) {
        c->bwd_ms += ms;
        c->bwd_calls++;
    }
    c->bwd_pending = false;
}

}  // namespace

extern "C" {

const char* gutb200_version(void) { return "3dgrut_b200 0.1 (sm_90a)"; }

void gutb200_default_config(gutb200_config* c) {  // configs/render/3dgut.yaml, include/3dgut/threedgut.cuh:54-89
    c->kernel_degree = 2;
    c->min_kernel_density = 0.0113f;
    c->min_alpha = 1.0f / 255.0f;
    c->max_alpha = 0.99f;
    c->min_transmittance = 0.0001f;
    c->ut_alpha = 1.0f;
    c->ut_beta = 2.0f;
    c->ut_kappa = 0.0f;
    c->ut_delta = static_cast<float>(1.7320508075688772);
    c->ut_margin = 0.1f;
    c->rect_bounding = 1;
    c->tight_opacity_bounding = 1;
    c->tile_culling = 1;
    c->global_z_order = 1;
    c->enable_timings = 0;
    c->subtile_culling = 7;  // bit 1: sub-tile screens in render; bit 2: renderBackward walks the forward's hit words (bit 0: unused since round 2)
    c->n_rolling_shutter_iterations = 5;  // configs/render/3dgut.yaml:18
    c->k_buffer_size = 0;                 // configs/render/3dgut.yaml: k_buffer_size 0 (unsorted)
    if (const char* e = std::getenv("GUTB200_SUBTILE_CULLING")) c->subtile_culling = std::atoi(e);  // A/B switch for profiling
}

int gutb200_create(const gutb200_config* cfg, int device, gutb200_ctx** out) {
    if (!cfg || !out) return 1;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count) return 2;  // no CPU fallback
    gutb200_ctx* c = new (std::nothrow) gutb200_ctx();
    if (!c) return 3;
    c->cfg = *cfg;
    c->device = device;
    if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaMallocHost(reinterpret_cast<void**>(&c->pinned_total), 2 * sizeof(uint32_t)) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_total, cudaEventDisableTiming) != cudaSuccess) {
        delete c;
        return 4;
    }
    for (auto& e : c->ev) cudaEventCreate(&e);
    *out = c;
    return 0;
}

void gutb200_destroy(gutb200_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    DeviceBuffer* bufs[] = {&c->tiles_count, &c->proj, &c->depth, &c->rgb, &c->grad_acc, &c->keys64, &c->keys64_alt, &c->vals_out, &c->hit_words, &c->tile_hist,
                            &c->tile_fill, &c->scan_parts, &c->sub_base, &c->ranges, &c->tile_order, &c->chunk_base, &c->totals, &c->h_particles, &c->h_sph,
                            &c->h_rays_o, &c->h_rays_d, &c->h_rgba, &c->h_dist, &c->h_hits, &c->h_vis, &c->h_drgba, &c->h_ddist,
                            &c->h_dpart, &c->h_dsph};
    for (DeviceBuffer* b : bufs) b->release();
    if (c->pinned_total) cudaFreeHost(c->pinned_total);
    for (auto& e : c->ev)
        if (e) cudaEventDestroy(e);
    if (c->ev_total) cudaEventDestroy(c->ev_total);
    for (auto& pair : c->st_ev)
        for (auto& e : pair)
            if (e) cudaEventDestroy(e);
    if (c->own_stream) cudaStreamDestroy(c->own_stream);
    delete c;
}

const char* gutb200_last_error(const gutb200_ctx* c) { return c ? c->error.c_str() : "null context"; }

int64_t gutb200_launch_count(const gutb200_ctx* c) { return c ? c->launches : 0; }

}  // extern "C"

namespace {

// NHT features: the configuration the kernels build (48 features = 4 vertices x 12, barycentric, sincos x 1)
int check_nht_args(gutb200_ctx* c, const void* features, int32_t feature_dim, int32_t features_half) {
    if (feature_dim != 48) return fail(c, "NHT feature_dim %d not built (48 = 4 tetrahedron vertices x 12 features)", feature_dim);
    if (features_half != 0 && features_half != 1) return fail(c, "features_half must be 0 (fp32) or 1 (fp16), got %d", features_half);
    if (reinterpret_cast<uintptr_t>(features) & 15) return fail(c, "feature buffer must be 16-byte aligned");
    if (c->cfg.k_buffer_size > 0) return fail(c, "NHT features are not built with the k-buffer (k_buffer_size %d > 0)", c->cfg.k_buffer_size);
    return 0;
}

// nht = false: SH radiance (`sph`, `sph_degree`, out [H,W,4]); nht = true: NHT features (`sph` = features, `half`, out [H,W,25])
int forward_impl(gutb200_ctx* c, void* stream, const gutb200_camera* cam, int64_t n, const float* particles, const void* sph,
                 int32_t sph_degree, bool nht, bool half, const float* rays_o, const float* rays_d, float* out_rgba, float* out_dist,
                 float* out_hits, float* visibility) {
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    GUT_CUDA(c, cudaSetDevice(c->device));
    c->have_forward = false;
    fill_frame(c, cam);
    const int64_t tiles = static_cast<int64_t>(c->cam.grid_x) * c->cam.grid_y;
    const size_t nn = static_cast<size_t>(n > 0 ? n : 1);

    if (c->cfg.enable_timings) {
        drain_timers(c);
        GUT_CUDA(c, cudaEventRecord(c->ev[0], s));
    }

    GUT_CUDA(c, c->tiles_count.reserve(nn * 4, s));
    GUT_CUDA(c, c->proj.reserve(nn * sizeof(ProjRecord), s));
    GUT_CUDA(c, c->depth.reserve(nn * 4, s));
    GUT_CUDA(c, c->rgb.reserve(nn * 12, s));
    const size_t tt = static_cast<size_t>(tiles);
    GUT_CUDA(c, c->tile_hist.reserve(tt * kTileSubs * 4, s));
    GUT_CUDA(c, c->tile_fill.reserve(tt * kTileSubs * 4, s));
    GUT_CUDA(c, c->sub_base.reserve(tt * kTileSubs * 4, s));
    GUT_CUDA(c, c->ranges.reserve(tt * 8, s));
    GUT_CUDA(c, c->tile_order.reserve(tt * 4, s));
    GUT_CUDA(c, c->chunk_base.reserve(tt * 4, s));
    GUT_CUDA(c, c->totals.reserve(16, s));
    GUT_CUDA(c, c->scan_parts.reserve(tile_scan_parts_words(static_cast<int>(tiles)) * 4, s));

    // The frame is enqueued in one go.  The list total I is needed on the host only to SIZE the key / value / hit-word buffers, so the
    // kernels that depend on it are launched speculatively against the capacity those (grow-only) buffers already have, and the host
    // reads I after everything is queued -- the GPU keeps working through the round trip the reference stalls on
    // (gutRenderer.cu:313-321).  If I does not fit (first frame, or the scene grew past the 12.5 % head-room) tile_scan publishes empty
    // ranges, the speculative kernels find nothing to do, and the tail of the frame is queued again after the buffers have grown.
    auto bin_and_render = [&](uint32_t capacity) -> int {
        {
            StageTimer t(c, 1, s);
            launch_tile_scan(s, static_cast<int>(tiles), c->tile_hist.as<uint32_t>(), capacity, c->ranges.as<uint32_t>(), c->sub_base.as<uint32_t>(),
                             c->chunk_base.as<uint32_t>(), c->tile_order.as<uint32_t>(), c->tile_fill.as<uint32_t>(), c->totals.as<uint32_t>(),
                             c->scan_parts.as<uint32_t>());
        }
        GUT_CUDA(c, cudaMemcpyAsync(c->pinned_total, c->totals.ptr, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        GUT_CUDA(c, cudaEventRecord(c->ev_total, s));
        c->launches += 2;
        if (capacity > 0 && n > 0) {
            {
                StageTimer t(c, 2, s);
                launch_expand_place(s, c->cam, c->fcfg, n, c->proj.as<ProjRecord>(), c->depth.as<float>(), c->tile_hist.as<uint32_t>(),
                                    c->sub_base.as<uint32_t>(), c->totals.as<uint32_t>(), capacity, c->tile_fill.as<uint32_t>(),
                                    c->keys64.as<unsigned long long>());
            }
            {
                StageTimer t(c, 3, s);
                GUT_CUDA(c, launch_tile_sort(s, static_cast<int>(tiles), c->tile_order.as<uint32_t>(), c->ranges.as<uint32_t>(), c->totals.as<uint32_t>(),
                                             c->keys64.as<unsigned long long>(), c->keys64_alt.as<unsigned long long>(), c->vals_out.as<uint32_t>()));
            }
            c->launches += 2;
        }
        {
            StageTimer t(c, 5, s);
            if (c->fcfg.k_buffer_size == 0)  // chunks a forward warp never reaches must read as "no hit" in the backward
                GUT_CUDA(c, cudaMemsetAsync(c->hit_words.ptr, 0, hit_words_capacity(capacity, tiles) * 4, s));
            if (nht)
                launch_render_forward_nht(s, c->cam, c->fcfg, rays_o, rays_d, particles, sph, half, c->vals_out.as<uint32_t>(),
                                          c->ranges.as<uint32_t>(), c->tile_order.as<uint32_t>(), c->chunk_base.as<uint32_t>(),
                                          c->hit_words.as<uint32_t>(), out_rgba, out_dist, out_hits);
            else if (c->fcfg.k_buffer_size > 0)  // sorted 3DGUT (gut_render_kbuffer.cu)
                launch_render_forward_kbuffer(s, c->cam, c->fcfg, c->fcfg.k_buffer_size, rays_o, rays_d, particles, c->rgb.as<float>(),
                                              c->vals_out.as<uint32_t>(), c->ranges.as<uint32_t>(), out_rgba, out_dist, out_hits);
            else
                launch_render_forward(s, c->cam, c->fcfg, rays_o, rays_d, particles, c->rgb.as<float>(), c->vals_out.as<uint32_t>(),
                                      c->ranges.as<uint32_t>(), c->tile_order.as<uint32_t>(), c->chunk_base.as<uint32_t>(),
                                      c->hit_words.as<uint32_t>(), out_rgba, out_dist, out_hits);
        }
        c->launches++;
        return 0;
    };

    uint32_t total = 0;
    GUT_CUDA(c, cudaMemsetAsync(c->tile_hist.ptr, 0, tt * kTileSubs * 4, s));
    if (n > 0) {
        StageTimer t(c, 0, s);
        launch_project(s, c->cam, c->fcfg, n, particles, static_cast<const float*>(sph), sph_degree, c->tiles_count.as<uint32_t>(),
                       c->proj.as<ProjRecord>(), c->depth.as<float>(), c->rgb.as<float>(), visibility, c->tile_hist.as<uint32_t>(), !nht);
        c->launches++;
    }
    GUT_CUDA(c, c->vals_out.reserve(16, s));
    GUT_CUDA(c, c->hit_words.reserve(hit_words_capacity(0, tiles) * 4, s));
    uint32_t capacity = static_cast<uint32_t>(std::min<size_t>(std::min(c->keys64.bytes, c->keys64_alt.bytes) / 8, 0xFFFFFFF0u));
    // the three per-intersection buffers grow together; `capacity` is the smallest of them in entries
    capacity = static_cast<uint32_t>(std::min<size_t>(capacity, c->vals_out.bytes / 4));
    while (capacity > 0 && hit_words_capacity(capacity, tiles) * 4 > c->hit_words.bytes) capacity = capacity > 4096 ? capacity - 4096 : 0;
    if (int rc = bin_and_render(capacity)) return rc;
    GUT_CUDA(c, cudaEventSynchronize(c->ev_total));
    total = c->pinned_total[0];
    if (c->pinned_total[1] != 0u) {  // did not fit: grow (grow-only, 12.5 % head-room) and queue the tail of the frame again
        GUT_CUDA(c, c->keys64.reserve(static_cast<size_t>(total) * 8, s));
        GUT_CUDA(c, c->keys64_alt.reserve(static_cast<size_t>(total) * 8, s));
        GUT_CUDA(c, c->vals_out.reserve(static_cast<size_t>(total) * 4 + 16, s));
        GUT_CUDA(c, c->hit_words.reserve(hit_words_capacity(total + (total >> 3) + 64, tiles) * 4, s));
        capacity = total;
        if (int rc = bin_and_render(capacity)) return rc;
        GUT_CUDA(c, cudaEventSynchronize(c->ev_total));
        if (c->pinned_total[1] != 0u || c->pinned_total[0] != total) return fail(c, "internal error: intersection count changed between two passes");
    }
    GUT_CUDA(c, cudaGetLastError());
    if (c->cfg.enable_timings) {
        GUT_CUDA(c, cudaEventRecord(c->ev[1], s));
        c->fwd_pending = true;
    }
    c->n = n;
    c->num_isect = total;
    c->num_tiles = tiles;
    c->fwd_stream = s;
    c->fwd_camera = *cam;
    c->fwd_nht = nht;
    c->have_forward = true;
    return 0;
}

}  // namespace

extern "C" {

int gutb200_forward(gutb200_ctx* c, void* stream, const gutb200_camera* cam, int64_t n, const float* particles, const float* sph,
                    int32_t sph_degree, const float* rays_o, const float* rays_d, float* out_rgba, float* out_dist, float* out_hits,
                    float* visibility) {
    if (int rc = check_args(c, cam, n, particles, sph_degree)) return rc;
    return forward_impl(c, stream, cam, n, particles, sph, sph_degree, false, false, rays_o, rays_d, out_rgba, out_dist, out_hits, visibility);
}

int gutb200_forward_nht(gutb200_ctx* c, void* stream, const gutb200_camera* cam, int64_t n, const float* particles, const void* features,
                        int32_t feature_dim, int32_t features_half, const float* rays_o, const float* rays_d, float* out_features_alpha,
                        float* out_dist, float* out_hits, float* visibility) {
    if (int rc = check_args(c, cam, n, particles, 0)) return rc;
    if (int rc = check_nht_args(c, features, feature_dim, features_half)) return rc;
    return forward_impl(c, stream, cam, n, particles, features, 0, true, features_half != 0, rays_o, rays_d, out_features_alpha, out_dist,
                        out_hits, visibility);
}

// `nht`: the adjoint of gutb200_forward_nht (`sph` = the features, `half`, out / d_rgba [H,W,25], d_sph = d_features [N,48])
static int backward_impl(gutb200_ctx* c, void* stream, const gutb200_camera* cam, int64_t n, const float* particles, const void* sph,
                         int32_t sph_degree, bool nht, bool half, const float* rays_o, const float* rays_d, const float* out_rgba,
                         const float* d_rgba, const float* out_dist, const float* d_dist, float* d_particles, float* d_sph, bool compact) {
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    // the backward replays the sorted lists of the immediately preceding forward (gutRenderer.cu:436-440)
    if (!c->have_forward || c->fwd_stream != s || c->n != n || c->cam.width != cam->width || c->cam.height != cam->height)
        return fail(c, "backward needs the forward context of the same stream / particle count / resolution");
    // the lists, the projection and the hit words are those of the forward's camera: a different view in between is an error, not a silent mix
    if (memcmp(&c->fwd_camera, cam, sizeof(gutb200_camera)) != 0)
        return fail(c, "backward was called with a camera that differs from the immediately preceding forward's (poses / intrinsics)");
    if (c->fwd_nht != nht)
        return fail(c, nht ? "gutb200_backward_nht needs a gutb200_forward_nht before it (the preceding forward rendered SH radiance)"
                           : "the preceding forward rendered NHT features: its adjoint is gutb200_backward_nht");
    GUT_CUDA(c, cudaSetDevice(c->device));
    if (c->cfg.enable_timings) {
        GUT_CUDA(c, cudaEventRecord(c->ev[2], s));
    }
    const size_t nn = static_cast<size_t>(n > 0 ? n : 1);
    GUT_CUDA(c, c->grad_acc.reserve(nn * kGradRow * 4, s, /*zero=*/true));
    if (nht && n > 0) GUT_CUDA(c, cudaMemsetAsync(d_sph, 0, static_cast<size_t>(n) * 48 * sizeof(float), s));  // the feature adjoint adds into it
    if (c->num_isect > 0) {
        StageTimer t(c, 6, s);
        if (nht)
            GUT_CUDA(c, launch_render_backward_nht(s, c->cam, c->fcfg, rays_o, rays_d, particles, sph, half, c->vals_out.as<uint32_t>(),
                                                   c->ranges.as<uint32_t>(), c->tile_order.as<uint32_t>(), c->chunk_base.as<uint32_t>(),
                                                   c->hit_words.as<uint32_t>(), out_rgba, d_rgba, out_dist, d_dist, c->grad_acc.as<float>(),
                                                   d_sph));
        else if (c->fcfg.k_buffer_size > 0)
            launch_render_backward_kbuffer(s, c->cam, c->fcfg, c->fcfg.k_buffer_size, rays_o, rays_d, particles, c->rgb.as<float>(),
                                           c->vals_out.as<uint32_t>(), c->ranges.as<uint32_t>(), out_rgba, d_rgba, out_dist, d_dist,
                                           c->grad_acc.as<float>());
        else
            launch_render_backward(s, c->cam, c->fcfg, rays_o, rays_d, particles, c->rgb.as<float>(), c->vals_out.as<uint32_t>(),
                                   c->ranges.as<uint32_t>(), c->tile_order.as<uint32_t>(), c->chunk_base.as<uint32_t>(),
                                   c->hit_words.as<uint32_t>(), out_rgba, d_rgba, out_dist, d_dist, c->grad_acc.as<float>());
        c->launches++;
    }
    if (n > 0) {
        StageTimer t(c, 7, s);
        launch_project_backward(s, c->cam, n, particles, static_cast<const float*>(sph), sph_degree, c->rgb.as<float>(),
                                c->tiles_count.as<uint32_t>(), rays_o, c->grad_acc.as<float>(), d_particles, d_sph, compact,
                                /*canon=*/c->fcfg.k_buffer_size == 0, /*radiance=*/!nht);
        c->launches++;
    }
    GUT_CUDA(c, cudaGetLastError());
    if (c->cfg.enable_timings) {
        GUT_CUDA(c, cudaEventRecord(c->ev[3], s));
        c->bwd_pending = true;
    }
    return 0;
}

int gutb200_backward(gutb200_ctx* c, void* stream, const gutb200_camera* cam, int64_t n, const float* particles, const float* sph,
                     int32_t sph_degree, const float* rays_o, const float* rays_d, const float* out_rgba, const float* d_rgba,
                     const float* out_dist, const float* d_dist, float* d_particles, float* d_sph) {
    if (int rc = check_args(c, cam, n, particles, sph_degree)) return rc;
    return backward_impl(c, stream, cam, n, particles, sph, sph_degree, false, false, rays_o, rays_d, out_rgba, d_rgba, out_dist, d_dist, d_particles,
                         d_sph, false);
}

int gutb200_backward_nht(gutb200_ctx* c, void* stream, const gutb200_camera* cam, int64_t n, const float* particles, const void* features,
                         int32_t feature_dim, int32_t features_half, const float* rays_o, const float* rays_d, const float* out_features_alpha,
                         const float* d_features_alpha, const float* out_dist, const float* d_dist, float* d_particles, float* d_features) {
    if (int rc = check_args(c, cam, n, particles, 0)) return rc;
    if (int rc = check_nht_args(c, features, feature_dim, features_half)) return rc;
    return backward_impl(c, stream, cam, n, particles, features, 0, true, features_half != 0, rays_o, rays_d, out_features_alpha, d_features_alpha,
                         out_dist, d_dist, d_particles, d_features, false);
}

int gutb200_backward_compact(gutb200_ctx* c, void* stream, const gutb200_camera* cam, int64_t n, const float* particles, const float* sph,
                             int32_t sph_degree, const float* rays_o, const float* rays_d, const float* out_rgba, const float* d_rgba,
                             const float* out_dist, const float* d_dist, float* d_particles, float* d_radiance) {
    if (int rc = check_args(c, cam, n, particles, sph_degree)) return rc;
    return backward_impl(c, stream, cam, n, particles, sph, sph_degree, false, false, rays_o, rays_d, out_rgba, d_rgba, out_dist, d_dist, d_particles,
                         d_radiance, true);
}

int gutb200_sph_grad_from_views(gutb200_ctx* c, void* stream, int64_t n, const float* particles, int32_t sph_degree, int32_t views,
                                const float* view_positions_host, const float* d_radiance_all, float* d_sph) {
    if (!c) return 1;
    if (views < 1 || views > 64) return fail(c, "views %d out of range (1..64)", views);
    if (n < 0 || !view_positions_host) return fail(c, "invalid arguments");
    if (sph_degree < 0 || sph_degree > 3) return fail(c, "sph_degree %d out of range", sph_degree);
    GUT_CUDA(c, cudaSetDevice(c->device));
    launch_sph_from_views(static_cast<cudaStream_t>(stream), n, particles, sph_degree, views, view_positions_host, d_radiance_all, d_sph);
    c->launches++;
    GUT_CUDA(c, cudaGetLastError());
    return 0;
}

int gutb200_camera_position(const gutb200_camera* cam, float* pos3) {
    if (!cam || !pos3) return 1;
    // the sensor position the kernels use: translation of the inverse mid-exposure pose (fill_frame)
    const Pose ps = pose_from7(cam->pose_start), pe = pose_from7(cam->pose_end);
    Pose mid;
    mid.q = slerp(ps.q, pe.q, 0.5f);
    for (int k = 0; k < 3; ++k) mid.t[k] = ps.t[k] * (1.f - 0.5f) + pe.t[k] * 0.5f;
    const Pose inv = pose_inverse(mid);
    for (int k = 0; k < 3; ++k) pos3[k] = inv.t[k];
    return 0;
}

int gutb200_forward_host(gutb200_ctx* c, const gutb200_camera* cam, int64_t n, const float* particles, const float* sph,
                         int32_t sph_degree, const float* rays_o, const float* rays_d, float* out_rgba, float* out_dist,
                         float* out_hits, float* visibility) {
    if (!c || !cam) return 1;
    cudaStream_t s = c->own_stream;
    const size_t np = static_cast<size_t>(n), px = static_cast<size_t>(cam->width) * cam->height;
    GUT_CUDA(c, cudaSetDevice(c->device));
    GUT_CUDA(c, c->h_particles.reserve(np * 48 + 16, s));
    GUT_CUDA(c, c->h_sph.reserve(np * 192 + 16, s));
    GUT_CUDA(c, c->h_rays_o.reserve(px * 12, s));
    GUT_CUDA(c, c->h_rays_d.reserve(px * 12, s));
    GUT_CUDA(c, c->h_rgba.reserve(px * 16, s));
    GUT_CUDA(c, c->h_dist.reserve(px * 4, s));
    GUT_CUDA(c, c->h_hits.reserve(px * 4, s));
    GUT_CUDA(c, c->h_vis.reserve(np * 4 + 16, s));
    GUT_CUDA(c, cudaMemcpyAsync(c->h_particles.ptr, particles, np * 48, cudaMemcpyHostToDevice, s));
    GUT_CUDA(c, cudaMemcpyAsync(c->h_sph.ptr, sph, np * 192, cudaMemcpyHostToDevice, s));
    GUT_CUDA(c, cudaMemcpyAsync(c->h_rays_o.ptr, rays_o, px * 12, cudaMemcpyHostToDevice, s));
    GUT_CUDA(c, cudaMemcpyAsync(c->h_rays_d.ptr, rays_d, px * 12, cudaMemcpyHostToDevice, s));
    if (int rc = gutb200_forward(c, s, cam, n, c->h_particles.as<float>(), c->h_sph.as<float>(), sph_degree, c->h_rays_o.as<float>(),
                                 c->h_rays_d.as<float>(), c->h_rgba.as<float>(), c->h_dist.as<float>(), c->h_hits.as<float>(),
                                 c->h_vis.as<float>()))
        return rc;
    GUT_CUDA(c, cudaMemcpyAsync(out_rgba, c->h_rgba.ptr, px * 16, cudaMemcpyDeviceToHost, s));
    GUT_CUDA(c, cudaMemcpyAsync(out_dist, c->h_dist.ptr, px * 4, cudaMemcpyDeviceToHost, s));
    GUT_CUDA(c, cudaMemcpyAsync(out_hits, c->h_hits.ptr, px * 4, cudaMemcpyDeviceToHost, s));
    if (np) GUT_CUDA(c, cudaMemcpyAsync(visibility, c->h_vis.ptr, np * 4, cudaMemcpyDeviceToHost, s));
    GUT_CUDA(c, cudaStreamSynchronize(s));
    return 0;
}

int gutb200_backward_host(gutb200_ctx* c, const gutb200_camera* cam, int64_t n, const float* particles, const float* sph,
                          int32_t sph_degree, const float* rays_o, const float* rays_d, const float* out_rgba, const float* d_rgba,
                          const float* out_dist, const float* d_dist, float* d_particles, float* d_sph) {
    if (!c || !cam) return 1;
    (void)particles; (void)sph; (void)rays_o; (void)rays_d;  // still resident from forward_host (same contract as the reference ctx)
    if (!c->have_forward || c->fwd_stream != c->own_stream)
        return fail(c, "backward needs the forward context of the same stream / particle count / resolution");
    cudaStream_t s = c->own_stream;
    const size_t np = static_cast<size_t>(n), px = static_cast<size_t>(cam->width) * cam->height;
    GUT_CUDA(c, cudaSetDevice(c->device));
    GUT_CUDA(c, c->h_drgba.reserve(px * 16, s));
    GUT_CUDA(c, c->h_ddist.reserve(px * 4, s));
    GUT_CUDA(c, c->h_dpart.reserve(np * 48 + 16, s));
    GUT_CUDA(c, c->h_dsph.reserve(np * 192 + 16, s));
    GUT_CUDA(c, cudaMemcpyAsync(c->h_rgba.ptr, out_rgba, px * 16, cudaMemcpyHostToDevice, s));
    GUT_CUDA(c, cudaMemcpyAsync(c->h_dist.ptr, out_dist, px * 4, cudaMemcpyHostToDevice, s));
    GUT_CUDA(c, cudaMemcpyAsync(c->h_drgba.ptr, d_rgba, px * 16, cudaMemcpyHostToDevice, s));
    GUT_CUDA(c, cudaMemcpyAsync(c->h_ddist.ptr, d_dist, px * 4, cudaMemcpyHostToDevice, s));
    if (int rc = gutb200_backward(c, s, cam, n, c->h_particles.as<float>(), c->h_sph.as<float>(), sph_degree, c->h_rays_o.as<float>(),
                                  c->h_rays_d.as<float>(), c->h_rgba.as<float>(), c->h_drgba.as<float>(), c->h_dist.as<float>(),
                                  c->h_ddist.as<float>(), c->h_dpart.as<float>(), c->h_dsph.as<float>()))
        return rc;
    if (np) {
        GUT_CUDA(c, cudaMemcpyAsync(d_particles, c->h_dpart.ptr, np * 48, cudaMemcpyDeviceToHost, s));
        GUT_CUDA(c, cudaMemcpyAsync(d_sph, c->h_dsph.ptr, np * 192, cudaMemcpyDeviceToHost, s));
    }
    GUT_CUDA(c, cudaStreamSynchronize(s));
    return 0;
}

int gutb200_last_stats(gutb200_ctx* c, int64_t* n, int64_t* num_intersections, int64_t* num_visible, int64_t* num_tiles) {
    if (!c || !c->have_forward) return fail(c, "no forward context");
    GUT_CUDA(c, cudaSetDevice(c->device));
    GUT_CUDA(c, cudaStreamSynchronize(c->fwd_stream));
    if (n) *n = c->n;
    if (num_intersections) *num_intersections = c->num_isect;
    if (num_tiles) *num_tiles = c->num_tiles;
    if (num_visible) {
        int64_t v = 0;
        if (c->n > 0) {
            uint32_t* h = new (std::nothrow) uint32_t[c->n];
            if (!h) return fail(c, "out of host memory");
            cudaError_t e = cudaMemcpy(h, c->tiles_count.ptr, static_cast<size_t>(c->n) * 4, cudaMemcpyDeviceToHost);
            for (int64_t i = 0; e == cudaSuccess && i < c->n; ++i) v += h[i] > 0;
            delete[] h;
            GUT_CUDA(c, e);
        }
        *num_visible = v;
    }
    return 0;
}

int gutb200_debug_copy(gutb200_ctx* c, int what, void* dst, size_t bytes) {
    if (!c || !c->have_forward) return fail(c, "no forward context");
    GUT_CUDA(c, cudaSetDevice(c->device));
    GUT_CUDA(c, cudaStreamSynchronize(c->fwd_stream));
    const void* src = nullptr;
    size_t have = 0;
    const size_t n = static_cast<size_t>(c->n), I = static_cast<size_t>(c->num_isect), T = static_cast<size_t>(c->num_tiles);
    switch (what) {
        case GUTB200_DBG_TILES_COUNT: src = c->tiles_count.ptr; have = n * 4; break;
        case GUTB200_DBG_SORTED_KEYS: {  // the reference's 64-bit keys, rebuilt from (tile, particle -> depth bits)
            if (bytes != I * 8) return fail(c, "debug buffer %d holds %zu bytes, caller asked for %zu", what, I * 8, bytes);
            if (I == 0) return 0;
            void* tmp = nullptr;
            GUT_CUDA(c, cudaMalloc(&tmp, I * 8));
            launch_synth_tile_keys(c->fwd_stream, static_cast<int>(T), c->ranges.as<uint32_t>(), c->vals_out.as<uint32_t>(), c->depth.as<float>(),
                                   static_cast<uint64_t*>(tmp));
            cudaError_t e = cudaStreamSynchronize(c->fwd_stream);
            if (e == cudaSuccess) e = cudaMemcpy(dst, tmp, I * 8, cudaMemcpyDeviceToHost);
            cudaFree(tmp);
            GUT_CUDA(c, e);
            return 0;
        }
        case GUTB200_DBG_SORTED_VALUES: src = c->vals_out.ptr; have = I * 4; break;
        case GUTB200_DBG_TILE_RANGES: src = c->ranges.ptr; have = T * 8; break;
        case GUTB200_DBG_DEPTH: src = c->depth.ptr; have = n * 4; break;
        case GUTB200_DBG_RGB: src = c->rgb.ptr; have = n * 12; break;
        case GUTB200_DBG_PROJ: src = c->proj.ptr; have = n * sizeof(ProjRecord); break;
        default: return fail(c, "unknown debug buffer %d", what);
    }
    if (bytes != have) return fail(c, "debug buffer %d holds %zu bytes, caller asked for %zu", what, have, bytes);
    if (have) GUT_CUDA(c, cudaMemcpy(dst, src, have, cudaMemcpyDeviceToHost));
    return 0;
}

// Work counters of the last forward (debug): re-walks its lists with the counting instantiation of the forward kernel.
// counters16: tests_ref, tests_exec, hits, fwd_iters, hit_iters, screens, bwd_lanes, iters16, iters8, sub16_hits, sub8_hits, 0.. (WorkCounters, gut_render.cu)
int gutb200_debug_work_counters(gutb200_ctx* c, const float* particles, const float* rays_o, const float* rays_d, uint64_t* counters16) {
    if (!c || !c->have_forward) return fail(c, "no forward context");
    if (c->fcfg.k_buffer_size != 0) return fail(c, "work counters exist for the unsorted path (k_buffer_size 0) only");
    if (c->fwd_nht) return fail(c, "work counters exist for the SH radiance forward only");
    GUT_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t s = c->fwd_stream;
    unsigned long long* dctr = nullptr;
    GUT_CUDA(c, cudaMalloc(&dctr, 128));
    cudaMemsetAsync(dctr, 0, 128, s);
    for (int i = 0; i < 16; ++i) counters16[i] = 0;
    if (c->num_isect > 0)
        launch_count_work(s, c->cam, c->fcfg, rays_o, rays_d, particles, c->rgb.as<float>(), c->vals_out.as<uint32_t>(), c->ranges.as<uint32_t>(),
                          c->tile_order.as<uint32_t>(), c->chunk_base.as<uint32_t>(), c->hit_words.as<uint32_t>(), dctr);
    cudaError_t e = cudaStreamSynchronize(s);
    if (e == cudaSuccess) e = cudaMemcpy(counters16, dctr, 128, cudaMemcpyDeviceToHost);
    cudaFree(dctr);
    GUT_CUDA(c, e);
    return 0;
}

// FP32 FMA throughput of this GPU (debug): best of `repeats` launches of the micro-benchmark in gut_debug.cu, in TFLOP/s
int gutb200_debug_fma_peak(gutb200_ctx* c, int repeats, float* tflops) {
    if (!c || !tflops) return 1;
    GUT_CUDA(c, cudaSetDevice(c->device));
    cudaDeviceProp prop;
    GUT_CUDA(c, cudaGetDeviceProperties(&prop, c->device));
    const int blocks = prop.multiProcessorCount * 8, iters = 2048;
    float* sink = nullptr;
    GUT_CUDA(c, cudaMalloc(&sink, 4));
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    float best = 0.f;
    for (int r = 0; r < repeats + 1; ++r) {  // first launch is a warm-up
        cudaEventRecord(a, c->own_stream);
        launch_fma_peak(c->own_stream, blocks, iters, sink);
        cudaEventRecord(b, c->own_stream);
        cudaEventSynchronize(b);
        float ms = 0.f;
        cudaEventElapsedTime(&ms, a, b);
        const double flops = static_cast<double>(blocks) * 256.0 * iters * 16.0 * 8.0 * 2.0;
        if (r > 0 && ms > 0.f) best = fmaxf(best, static_cast<float>(flops / (ms * 1e-3) / 1e12));
    }
    cudaEventDestroy(a);
    cudaEventDestroy(b);
    cudaFree(sink);
    *tflops = best;
    GUT_CUDA(c, cudaGetLastError());
    return 0;
}

int gutb200_set_timings(gutb200_ctx* c, int level) {
    if (!c) return 1;
    drain_timers(c);
    c->cfg.enable_timings = level;
    return 0;
}

int gutb200_collect_stage_times(gutb200_ctx* c, float* mean_ms /*[8]*/) {
    if (!c || !mean_ms) return 1;
    drain_timers(c);
    for (int i = 0; i < 8; ++i) {
        mean_ms[i] = c->st_calls[i] ? static_cast<float>(c->st_ms[i] / c->st_calls[i]) : 0.f;
        c->st_ms[i] = 0;
        c->st_calls[i] = 0;
    }
    return 0;
}

int gutb200_collect_times(gutb200_ctx* c, float* forward_ms, float* backward_ms) {
    if (!c) return 1;
    drain_timers(c);
    if (forward_ms) *forward_ms = c->fwd_calls ? static_cast<float>(c->fwd_ms / c->fwd_calls) : 0.f;
    if (backward_ms) *backward_ms = c->bwd_calls ? static_cast<float>(c->bwd_ms / c->bwd_calls) : 0.f;
    c->fwd_ms = c->bwd_ms = 0;
    c->fwd_calls = c->bwd_calls = 0;
    return 0;
}

}  // extern "C"
