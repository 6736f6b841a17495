// 3dgrut_b200/csrc/gut_project.cu -- per-particle stages of the 3DGUT forward: unscented projection + tile counting + per-tile
// histogram (G1), key expansion into the tiles' slices (G3).  Tile ranges (G2 / G5) and the per-tile sort (G4) live in gut_binning.cu.
//
// Built with -fmad=false and IEEE div/sqrt: tile counts and sort keys are INTEGER outputs that must be
// bit-identical to the checker, so every fp32 operation here is written in the order the reference writes it
// (threedgut_tracer/include/3dgut/kernels/cuda/renderers/gutProjector.cuh) and nothing is contracted.
// These kernels are HBM-bound (DESIGN.md section 4), the un-fused multiplies cost nothing measurable.
//
// Hopper specifics: the 48-byte particle records of a CTA are one contiguous 12 KB span, fetched with a single
// TMA bulk copy (cp.async.bulk + mbarrier) into shared memory instead of 3 strided LDG.128 per thread; record
// reads from shared memory are conflict-free (stride 12 words, LDS.128 phases of 8 lanes).
#include "gut_common.cuh"
#include "tma.cuh"

namespace gutb200 {

namespace {

constexpr int kProjThreads = 256;
constexpr int kSmallBox = 8;  // footprints above this many tiles are walked by the whole warp

struct TileBox {
    int x0, y0, x1, y1;
};

// computeTileSpaceBBox (gutProjector.cuh:32-43)
__device__ __forceinline__ TileBox tile_box(int gx, int gy, float cx, float cy, float ex, float ey) {
    TileBox b;
    b.x0 = min(gx, max(0, static_cast<int>(floorf((cx - 0.5f - ex) / 16.0f))));
    b.y0 = min(gy, max(0, static_cast<int>(floorf((cy - 0.5f - ey) / 16.0f))));
    b.x1 = min(gx, max(0, static_cast<int>(ceilf((cx - 0.5f + ex) / 16.0f))));
    b.y1 = min(gy, max(0, static_cast<int>(ceilf((cy - 0.5f + ey) / 16.0f))));
    return b;
}

__device__ __forceinline__ float sat(float x) { return fminf(fmaxf(x, 0.f), 1.f); }

// tileMinParticlePowerResponse (gutProjector.cuh:49-78): smallest power of the 2-D conic over a tile.
__device__ __forceinline__ float tile_min_power(float tx, float ty, float ca, float cb, float cc, float mx, float my) {
    const float ts = 16.0f;
    const float tminx = ts * tx, tminy = ts * ty;
    const float tmaxx = ts + tminx, tmaxy = ts + tminy;
    const float mox = tminx - mx, moy = tminy - my;
    const float lax = mox > 0.0f ? 1.f : 0.f, lay = moy > 0.0f ? 1.f : 0.f;
    const float nrx = lax + (mx > tmaxx ? 1.f : 0.f);
    const float nry = lay + (my > tmaxy ? 1.f : 0.f);
    if ((nrx + nry) > 0.0f) {
        const float px = tmaxx * (1.f - lax) + tminx * lax;
        const float py = tmaxy * (1.f - lay) + tminy * lay;
        const float dxx = copysignf(ts, mox), dxy = copysignf(ts, moy);
        const float dfx = mx - px, dfy = my - py;
        const float rcx = 1.0f / (ts * ts * ca);
        const float rcy = 1.0f / (ts * ts * cc);
        const float tx_ = nry * sat((dxx * ca * dfx + dxx * cb * dfy) * rcx);
        const float ty_ = nrx * sat((dxy * cb * dfx + dxy * cc * dfy) * rcy);
        const float mdx = mx - (px + tx_ * dxx);
        const float mdy = my - (py + ty_ * dxy);
        return 0.5f * (ca * mdx * mdx + cc * mdy * mdy) + cb * mdx * mdy;
    }
    return 0.f;
}

// OpenCV pinhole projection of a sensor-space point (cameraProjections.cuh:67-118)
__device__ __forceinline__ bool project_pinhole(const FrameCamera& cam, float tol, float x, float y, float z, float& ox, float& oy) {
    if (z <= 0.f) {
        ox = 0.f;
        oy = 0.f;
        return false;
    }
    const float u = x / z, v = y / z;
    if (!cam.has_distortion) {
        // all distortion coefficients are zero: icD == 1 and delta == 0 exactly, so the general expression below
        // reduces to this one bit for bit
        ox = u * cam.fx + cam.cx;
        oy = v * cam.fy + cam.cy;
        const float mx0 = cam.res_x * tol, my0 = cam.res_y * tol;
        return (ox > -mx0) && (oy > -my0) && (ox < cam.res_x + mx0) && (oy < cam.res_y + my0);
    }
    const float uu = u * u, vv = v * v;
    const float r2 = uu + vv;
    const float a1 = 2.f * u * v;
    const float a2 = r2 + 2.f * uu;
    const float a3 = r2 + 2.f * vv;
    const float num = 1.f + r2 * (cam.radial[0] + r2 * (cam.radial[1] + r2 * cam.radial[2]));
    const float den = 1.f + r2 * (cam.radial[3] + r2 * (cam.radial[4] + r2 * cam.radial[5]));
    const float icd = num / den;
    const float dx = cam.tangential[0] * a1 + cam.tangential[1] * a2 + r2 * (cam.thin_prism[0] + r2 * cam.thin_prism[1]);
    const float dy = cam.tangential[0] * a3 + cam.tangential[1] * a1 + r2 * (cam.thin_prism[2] + r2 * cam.thin_prism[3]);
    const float ndx = icd * u + dx, ndy = icd * v + dy;
    const bool valid_radial = (icd > 0.8f) && (icd < 1.2f);
    if (valid_radial) {
        ox = ndx * cam.fx + cam.cx;
        oy = ndy * cam.fy + cam.cy;
    } else {
        const float clip = hypotf(cam.res_x, cam.res_y);
        const float f = clip / sqrtf(r2);
        ox = f * u + cam.cx;
        oy = f * v + cam.cy;
    }
    const float mx = cam.res_x * tol, my = cam.res_y * tol;
    const bool inside = (ox > -mx) && (oy > -my) && (ox < cam.res_x + mx) && (oy < cam.res_y + my);
    return valid_radial && inside;
}

// OpenCV fisheye projection of a sensor-space point (cameraProjections.cuh:25-35 stableNorm2, :38-48 Horner, :120-146)
__device__ __forceinline__ bool project_fisheye(const FrameCamera& cam, float tol, float x, float y, float z, float& ox, float& oy) {
    const float ax = fabsf(x), ay = fabsf(y);
    const float mn = fminf(ax, ay), mx = fmaxf(ax, ay);
    float rho = 0.f;
    if (mx > 0.f) {
        const float ratio = mn / mx;
        rho = mx * sqrtf(1.f + ratio * ratio);
    }
    if (rho <= 0.f) rho = 1.1920929e-07f;  // FLT_EPSILON
    const float theta_full = atan2f(rho, z);
    const float theta = fminf(theta_full, cam.max_angle);  // FOV-clamped projections are marked invalid below
    const float theta2 = theta * theta;
    float poly = cam.radial[3];
    poly = theta2 * poly + cam.radial[2];
    poly = theta2 * poly + cam.radial[1];
    poly = theta2 * poly + cam.radial[0];
    const float delta = (theta * (poly * theta2 + 1.0f)) / rho;
    ox = cam.fx * x * delta + cam.cx;
    oy = cam.fy * y * delta + cam.cy;
    const float mx0 = cam.res_x * tol, my0 = cam.res_y * tol;
    return (theta < cam.max_angle) && (ox > -mx0) && (oy > -my0) && (ox < cam.res_x + mx0) && (oy < cam.res_y + my0);
}

// f-theta projection of a sensor-space point (cameraProjections.cuh:148-198: 6-coefficient polynomials, 3 Newton iterations)
template <int N>
__device__ __forceinline__ float horner(const float* c, float x) {  // evalPolyHorner<N>, :38-48
    float y = c[N - 1];
#pragma unroll
    for (int i = N - 2; i >= 0; --i) y = x * y + c[i];
    return y;
}

__device__ __forceinline__ bool project_ftheta(const FrameCamera& cam, float tol, float x, float y, float z, float& ox, float& oy) {
    const float ax = fabsf(x), ay = fabsf(y);
    const float mn = fminf(ax, ay), mx = fmaxf(ax, ay);
    float rho = 0.f;
    if (mx > 0.f) {
        const float ratio = mn / mx;
        rho = mx * sqrtf(1.f + ratio * ratio);
    }
    if (rho <= 0.f) rho = 1.1920929e-07f;  // FLT_EPSILON
    const float theta_full = atan2f(rho, z);
    const float theta = fminf(theta_full, cam.max_angle);
    float delta = horner<6>(cam.ft_fw, theta);
    if (cam.ft_reference_poly == 0) {  // invert the backward polynomial, started from the forward one
        float dpoly[5];
#pragma unroll
        for (int i = 1; i < 6; ++i) dpoly[i - 1] = i * cam.ft_bw[i];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const float dfdx = horner<5>(dpoly, delta);
            const float residual = horner<6>(cam.ft_bw, delta) - theta;
            delta -= residual / dfdx;
        }
    }
    const float s = delta / rho;
    ox = s * (cam.ft_cde[0] * x + cam.ft_cde[1] * y);
    oy = s * (cam.ft_cde[2] * x + y);
    ox += cam.cx + .5f;  // image coordinate origin = centre of the first pixel
    oy += cam.cy + .5f;
    const float mx0 = cam.res_x * tol, my0 = cam.res_y * tol;
    return (theta < cam.max_angle) && (ox > -mx0) && (oy > -my0) && (ox < cam.res_x + mx0) && (oy < cam.res_y + my0);
}

__device__ __forceinline__ bool project_sensor(const FrameCamera& cam, float tol, float sx, float sy, float sz, float& ox, float& oy) {
    if (cam.model == 1) return project_fisheye(cam, tol, sx, sy, sz, ox, oy);
    if (cam.model == 2) return project_ftheta(cam, tol, sx, sy, sz, ox, oy);
    return project_pinhole(cam, tol, sx, sy, sz, ox, oy);
}

// column-major rotation (m[c*3+r]) applied like tcnn's tmat * tvec (vec.h:595-605), then the translation
__device__ __forceinline__ bool project_with_rotation(const FrameCamera& cam, float tol, const float* rot, const float* t, float px, float py,
                                                      float pz, float& ox, float& oy) {
    float s[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        float acc = 0.f;
        acc += rot[0 * 3 + j] * px;
        acc += rot[1 * 3 + j] * py;
        acc += rot[2 * 3 + j] * pz;
        s[j] = acc + t[j];
    }
    return project_sensor(cam, tol, s[0], s[1], s[2], ox, oy);
}

// tcnn::to_mat3 (vec.h:1185-1199), column major
__device__ __forceinline__ void quat_to_mat3(float w, float x, float y, float z, float* m) {
    const float qxx = x * x, qyy = y * y, qzz = z * z;
    const float qxz = x * z, qxy = x * y, qyz = y * z;
    const float qwx = w * x, qwy = w * y, qwz = w * z;
    m[0] = 1.f - 2.f * (qyy + qzz); m[1] = 2.f * (qxy + qwz); m[2] = 2.f * (qxz - qwy);
    m[3] = 2.f * (qxy - qwz); m[4] = 1.f - 2.f * (qxx + qzz); m[5] = 2.f * (qyz + qwx);
    m[6] = 2.f * (qxz + qwy); m[7] = 2.f * (qyz - qwx); m[8] = 1.f - 2.f * (qxx + qyy);
}

// pose at relative exposure time alpha: tcnn::slerp (vec.h:1146-1167) + tcnn::mix (vec.h:183), then project
__device__ __noinline__ bool project_at_time(const FrameCamera& cam, float tol, float alpha, float px, float py, float pz, float& ox, float& oy) {
    const float* a = cam.q_start;
    float zw = cam.q_end[0], zx = cam.q_end[1], zy = cam.q_end[2], zz = cam.q_end[3];
    float c = (a[0] * zw + a[1] * zx) + (a[2] * zy + a[3] * zz);
    if (c < 0.f) {
        zw = -zw; zx = -zx; zy = -zy; zz = -zz;
        c = -c;
    }
    float qw, qx, qy, qz;
    if (c > 1.f - 1.1920929e-07f) {
        const float k = 1.f - alpha;
        qw = a[0] * k + zw * alpha; qx = a[1] * k + zx * alpha; qy = a[2] * k + zy * alpha; qz = a[3] * k + zz * alpha;
    } else {
        const float ang = acosf(c);
        const float s0 = sinf((1.f - alpha) * ang), s1 = sinf(alpha * ang), sd = sinf(ang);
        qw = (s0 * a[0] + s1 * zw) / sd; qx = (s0 * a[1] + s1 * zx) / sd; qy = (s0 * a[2] + s1 * zy) / sd; qz = (s0 * a[3] + s1 * zz) / sd;
    }
    float rot[9], t[3];
    quat_to_mat3(qw, qx, qy, qz, rot);
#pragma unroll
    for (int k = 0; k < 3; ++k) t[k] = cam.t_start[k] * (1.f - alpha) + cam.t_end[k] * alpha;
    return project_with_rotation(cam, tol, rot, t, px, py, pz, ox, oy);
}

// relativeShutterTime (cameraProjections.cuh:50-65)
__device__ __forceinline__ float relative_shutter_time(const FrameCamera& cam, float x, float y) {
    switch (cam.rolling_shutter) {
        case 1: return floorf(y) / (cam.res_y - 1.f);
        case 2: return floorf(x) / (cam.res_x - 1.f);
        case 3: return (cam.res_y - ceilf(y)) / (cam.res_y - 1.f);
        case 4: return (cam.res_x - ceilf(x)) / (cam.res_x - 1.f);
        default: return 0.5f;
    }
}

// world point -> pixel: projectPointWithShutter (cameraProjections.cuh:218-257).  Global shutter: the shutter-open pose only.
template <bool ROLLING>
__device__ __forceinline__ bool project_world(const FrameCamera& cam, float tol, float px, float py, float pz, float& ox, float& oy) {
    bool valid = project_with_rotation(cam, tol, cam.rot_start, cam.t_start, px, py, pz, ox, oy);
    if (!ROLLING || cam.rolling_shutter == 0) return valid;
    if (!valid) {
        float rot[9];
        quat_to_mat3(cam.q_end[0], cam.q_end[1], cam.q_end[2], cam.q_end[3], rot);
        valid = project_with_rotation(cam, tol, rot, cam.t_end, px, py, pz, ox, oy);
        if (!valid) return false;
    }
    for (int i = 0; i < cam.rs_iterations; ++i) valid = project_at_time(cam, tol, relative_shutter_time(cam, ox, oy), px, py, pz, ox, oy);
    return valid;
}

constexpr float kC0 = 0.28209479177387814f;
constexpr float kC1 = 0.4886025119029199f;
__constant__ float kC2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f, -1.0925484305920792f,
                             0.5462742152960396f};
__constant__ float kC3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f, 0.3731763325901154f,
                             -0.4570457994644658f, 1.445305721320277f,  -0.5900435899266435f};

// unclamped view-dependent radiance of one particle (radianceFromSpH, models/gaussianParticles.cuh:68-100)
__device__ __forceinline__ void sph_radiance(int deg, const float* __restrict__ c, float x, float y, float z, float out[3]) {
    float cf[48];
    const float4* c4 = reinterpret_cast<const float4*>(c);
#pragma unroll
    for (int i = 0; i < 12; ++i) {
        const float4 v = __ldg(c4 + i);
        cf[i * 4 + 0] = v.x;
        cf[i * 4 + 1] = v.y;
        cf[i * 4 + 2] = v.z;
        cf[i * 4 + 3] = v.w;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
#define CF(i) cf[(i)*3 + k]
        float rad = kC0 * CF(0);
        if (deg > 0) {
            rad = rad - kC1 * y * CF(1) + kC1 * z * CF(2) - kC1 * x * CF(3);
            if (deg > 1) {
                const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                rad = rad + kC2[0] * xy * CF(4) + kC2[1] * yz * CF(5) + kC2[2] * (2.0f * zz - xx - yy) * CF(6) + kC2[3] * xz * CF(7) +
                      kC2[4] * (xx - yy) * CF(8);
                if (deg > 2) {
                    rad = rad + kC3[0] * y * (3.0f * xx - yy) * CF(9) + kC3[1] * xy * z * CF(10) +
                          kC3[2] * y * (4.0f * zz - xx - yy) * CF(11) + kC3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * CF(12) +
                          kC3[4] * x * (4.0f * zz - xx - yy) * CF(13) + kC3[5] * z * (xx - yy) * CF(14) +
                          kC3[6] * x * (xx - 3.0f * yy) * CF(15);
                }
            }
        }
#undef CF
        out[k] = rad + 0.5f;
    }
}

// G1: one thread per particle (projectOnTiles -> GUTProjector::eval, gutProjector.cuh:217-322)
// ROLLING = false is the global-shutter instantiation (no pose interpolation code, no stack frame); RGB = false skips the SH -> radiance
// work (NHT features are evaluated per hit in gut_render_nht.cu) and leaves `rgb` and `sph` untouched
template <bool ROLLING, bool RGB>
__global__ void __launch_bounds__(kProjThreads) project_kernel(FrameCamera cam, FrameConfig cfg, int64_t n,
                                                               const float* __restrict__ particles,
                                                               const float* __restrict__ sph, int sph_degree,
                                                               uint32_t* __restrict__ tiles_count, ProjRecord* __restrict__ proj,
                                                               float* __restrict__ depth, float* __restrict__ rgb,
                                                               float* __restrict__ visibility, uint32_t* __restrict__ tile_hist) {
    __shared__ __align__(128) float4 s_rec[kProjThreads * 3];
    __shared__ __align__(8) uint64_t s_bar;

    const int64_t base = static_cast<int64_t>(blockIdx.x) * kProjThreads;
    const int count = static_cast<int>(min(static_cast<int64_t>(kProjThreads), n - base));
    if (threadIdx.x == 0) {
        mbar_init(&s_bar, 1);
        fence_proxy_async();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t bytes = static_cast<uint32_t>(count) * 48u;
        mbar_expect_tx(&s_bar, bytes);
        tma_bulk_g2s(s_rec, particles + base * 12, bytes, &s_bar);
    }
    mbar_wait(&s_bar, 0);

    const int64_t i = base + threadIdx.x;
    const bool in_range = i < n;  // out-of-range lanes stay alive: the warp-cooperative tile count below needs every lane
    const int slot = in_range ? threadIdx.x : 0;

    const float4 r0 = s_rec[slot * 3 + 0];  // pos.xyz, density
    const float4 r1 = s_rec[slot * 3 + 1];  // quat wxyz
    const float4 r2 = s_rec[slot * 3 + 2];  // scale.xyz, pad
    const float px = r0.x, py = r0.y, pz = r0.z, opacity = r0.w;

    // rows of quaternionWXYZToMatrix == columns of R (models/gaussianParticles.cuh:39-59)
    float rot[3][3];
    {
        const float r = r1.x, x = r1.y, y = r1.z, z = r1.w;
        const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, xz = x * z, yz = y * z;
        const float rx = r * x, ry = r * y, rz = r * z;
        rot[0][0] = 1.f - 2.f * (yy + zz); rot[0][1] = 2.f * (xy + rz); rot[0][2] = 2.f * (xz - ry);
        rot[1][0] = 2.f * (xy - rz); rot[1][1] = 1.f - 2.f * (xx + zz); rot[1][2] = 2.f * (yz + rx);
        rot[2][0] = 2.f * (xz + ry); rot[2][1] = 2.f * (yz - rx); rot[2][2] = 1.f - 2.f * (xx + yy);
    }
    const float scl[3] = {r2.x, r2.y, r2.z};

    bool valid_proj = false, valid_conic = false;
    float pcx = 0.f, pcy = 0.f, cov0 = 0.f, cov1 = 0.f, cov2 = 0.f;
    const float zc = px * cam.view[0 * 3 + 2] + py * cam.view[1 * 3 + 2] + pz * cam.view[2 * 3 + 2] + cam.view[3 * 3 + 2];

    // unscentedParticleProjection (gutProjector.cuh:118-215): 7 sigma points, lambda = 0
    if (in_range && !(opacity < cfg.min_alpha) && !(zc < 0.2f)) {
        float spx[7], spy[7];
        int nvalid = 0;
        nvalid += project_world<ROLLING>(cam, cfg.ut_margin, px, py, pz, spx[0], spy[0]) ? 1 : 0;
        pcx = spx[0] * cfg.w0_mean;
        pcy = spy[0] * cfg.w0_mean;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float f = cfg.ut_delta * scl[k];
            const float dx = rot[k][0] * f, dy = rot[k][1] * f, dz = rot[k][2] * f;
            nvalid += project_world<ROLLING>(cam, cfg.ut_margin, px + dx, py + dy, pz + dz, spx[k + 1], spy[k + 1]) ? 1 : 0;
            pcx += cfg.wi * spx[k + 1];
            pcy += cfg.wi * spy[k + 1];
            nvalid += project_world<ROLLING>(cam, cfg.ut_margin, px - dx, py - dy, pz - dz, spx[k + 4], spy[k + 4]) ? 1 : 0;
            pcx += cfg.wi * spx[k + 4];
            pcy += cfg.wi * spy[k + 4];
        }
        if (nvalid != 0) {
            {
                const float ex = spx[0] - pcx, ey = spy[0] - pcy;
                cov0 = cfg.w0_cov * (ex * ex);
                cov1 = cfg.w0_cov * (ex * ey);
                cov2 = cfg.w0_cov * (ey * ey);
            }
#pragma unroll
            for (int k = 0; k < 6; ++k) {
                const float ex = spx[k + 1] - pcx, ey = spy[k + 1] - pcy;
                cov0 += cfg.wi * (ex * ex);
                cov1 += cfg.wi * (ex * ey);
                cov2 += cfg.wi * (ey * ey);
            }
            valid_proj = true;
        }
    }

    // computeProjectedExtentConicOpacity (gutProjector.cuh:81-116)
    float ex = 0.f, ey = 0.f, ca = 0.f, cb = 0.f, cc = 0.f, op = 0.f, maxpow = 0.f;
    if (valid_proj) {
        const float dcx = cov0 + 0.3f, dcy = cov1, dcz = cov2 + 0.3f;
        const float ddet = dcx * dcz - dcy * dcy;
        if (ddet != 0.0f) {
            ca = dcz / ddet;
            cb = -dcy / ddet;
            cc = dcx / ddet;
            const float cdet = cov0 * cov2 - cov1 * cov1;
            op = opacity * sqrtf(fmaxf(0.000025f, cdet / ddet));
            if (!(op < cfg.min_alpha)) {
                maxpow = logf(op / cfg.min_alpha);
                const float ef = cfg.tight_opacity_bounding ? fminf(3.33f, sqrtf(2.0f * maxpow)) : 3.33f;
                const float mid = 0.5f * (dcx + dcz);
                const float lam = mid + sqrtf(fmaxf(0.01f, mid * mid - ddet));
                const float radius = ef * sqrtf(lam);
                if (cfg.rect_bounding) {
                    ex = fminf(ef * sqrtf(dcx), radius);
                    ey = fminf(ef * sqrtf(dcz), radius);
                } else {
                    ex = radius;
                    ey = radius;
                }
                valid_conic = radius > 0.f;
            }
        }
    }

    const bool visible = valid_proj && valid_conic;
    // the reference stores int 1 into this float tensor (gutProjector.cuh:275, splatRaster.cpp:215,249);
    // consumers only test it for non-zero, we store the same bit pattern.
    if (in_range) visibility[i] = __int_as_float(visible ? 1 : 0);

    // tile count with per-tile culling (gutProjector.cuh:279-293).  Footprints of up to kSmallBox tiles are counted by the
    // owning lane; larger ones are counted by the whole warp, 32 tiles per step, so one big splat does not serialise its warp.
    uint32_t ntiles = 0;
    TileBox bb = {0, 0, 0, 0};
    int cells = 0;
    if (visible) {
        bb = tile_box(cam.grid_x, cam.grid_y, pcx, pcy, ex, ey);
        cells = (bb.x1 - bb.x0) * (bb.y1 - bb.y0);
        if (!cfg.tile_culling) {
            ntiles = static_cast<uint32_t>(cells);
            for (int y = bb.y0; y < bb.y1; ++y)
                for (int x = bb.x0; x < bb.x1; ++x) atomicAdd(&tile_hist[(y * cam.grid_x + x) * kTileSubs + (static_cast<int>(i) & (kTileSubs - 1))], 1u);
            cells = 0;
        } else if (cells <= kSmallBox) {
            for (int y = bb.y0; y < bb.y1; ++y)
                for (int x = bb.x0; x < bb.x1; ++x)
                    if (tile_min_power(static_cast<float>(x), static_cast<float>(y), ca, cb, cc, pcx, pcy) < maxpow) {
                        ntiles++;
                        atomicAdd(&tile_hist[(y * cam.grid_x + x) * kTileSubs + (static_cast<int>(i) & (kTileSubs - 1))], 1u);  // list length (tile_scan)
                    }
            cells = 0;
        }
    }
    {
        const unsigned lane = threadIdx.x & 31;
        unsigned big = __ballot_sync(0xFFFFFFFFu, cells > kSmallBox);
        while (big) {
            const int src = __ffs(big) - 1;
            big &= big - 1;
            const int bx0 = __shfl_sync(0xFFFFFFFFu, bb.x0, src), by0 = __shfl_sync(0xFFFFFFFFu, bb.y0, src);
            const int bw = __shfl_sync(0xFFFFFFFFu, bb.x1, src) - bx0, nc = __shfl_sync(0xFFFFFFFFu, cells, src);
            const float qa = __shfl_sync(0xFFFFFFFFu, ca, src), qb = __shfl_sync(0xFFFFFFFFu, cb, src), qc = __shfl_sync(0xFFFFFFFFu, cc, src);
            const float qx = __shfl_sync(0xFFFFFFFFu, pcx, src), qy = __shfl_sync(0xFFFFFFFFu, pcy, src), qp = __shfl_sync(0xFFFFFFFFu, maxpow, src);
            const int qsub = static_cast<int>(base + (threadIdx.x & ~31u) + src) & (kTileSubs - 1);  // sub-counter of the owning particle
            uint32_t total = 0;
            for (int c0 = 0; c0 < nc; c0 += 32) {
                const int c = c0 + static_cast<int>(lane);
                bool pass = false;
                if (c < nc) {
                    const int y = by0 + c / bw, x = bx0 + c % bw;
                    pass = tile_min_power(static_cast<float>(x), static_cast<float>(y), qa, qb, qc, qx, qy) < qp;
                    if (pass) atomicAdd(&tile_hist[(y * cam.grid_x + x) * kTileSubs + qsub], 1u);
                }
                total += __popc(__ballot_sync(0xFFFFFFFFu, pass));
            }
            if (static_cast<int>(lane) == src) ntiles = total;
        }
    }
    if (!in_range) return;
    tiles_count[i] = ntiles;

    ProjRecord pr;
    float zdepth = 0.f, col[3] = {0.f, 0.f, 0.f};
    if (ntiles == 0) {
        pr.cx = pr.cy = pr.ex = pr.ey = pr.ca = pr.cb = pr.cc = pr.op = 0.f;
    } else {
        const float sx = px - cam.cam_pos[0], sy = py - cam.cam_pos[1], sz = pz - cam.cam_pos[2];
        const float dist = sqrtf(sx * sx + sy * sy + sz * sz);
        if (RGB) sph_radiance(sph_degree, sph + i * 48, sx / dist, sy / dist, sz / dist, col);
        pr.cx = pcx; pr.cy = pcy; pr.ex = ex; pr.ey = ey;
        pr.ca = ca; pr.cb = cb; pr.cc = cc; pr.op = op;
        zdepth = cfg.global_z_order ? zc : dist;
    }
    proj[i] = pr;
    depth[i] = zdepth;
    if (!RGB) return;
    rgb[i * 3 + 0] = col[0];
    rgb[i * 3 + 1] = col[1];
    rgb[i * 3 + 2] = col[2];
}

// G3: emit (tile, particle) for every surviving tile (GUTProjector::expand, gutProjector.cuh:324-388).
// The reference emits 64-bit (tile << 32 | depth) keys in particle order and radix-sorts 44 bits of them (6 passes over
// 12 bytes per entry).  Here every pair goes straight into ITS TILE's slice of the key buffer (ranges from tile_scan) at a slot
// claimed with one atomic on the tile's fill counter, as the key (depth bits << 32 | particle index); tile_sort (gut_binning.cu) then
// orders each slice on chip.  The tile walk is the reference's (row-major, same culling arithmetic as project_kernel).
__global__ void __launch_bounds__(256) expand_place_kernel(FrameCamera cam, FrameConfig cfg, int64_t n, const ProjRecord* __restrict__ proj,
                                                           const float* __restrict__ depth, const uint32_t* __restrict__ tile_hist,
                                                           const uint32_t* __restrict__ sub_base, const uint32_t* __restrict__ totals,
                                                           uint32_t capacity, uint32_t* __restrict__ fill,
                                                           unsigned long long* __restrict__ keys) {
    if (totals[1] != 0u) return;  // capacity exceeded: the host grows the key buffer and launches again
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const bool in_range = i < n;
    ProjRecord pr;
    pr.ex = 0.f;
    if (in_range) pr = proj[i];
    const bool active = in_range && !(pr.ex <= 1e-06f);
    TileBox bb = {0, 0, 0, 0};
    float maxpow = 0.f;
    int cells = 0;
    unsigned long long key = 0ull;
    auto place = [&](int tile, unsigned long long k) {   // sub-bucket = low bits of the particle index (low word of the key)
        const size_t at = static_cast<size_t>(tile) * kTileSubs + (static_cast<uint32_t>(k) & (kTileSubs - 1));
        const uint32_t slot = atomicAdd(&fill[at], 1u);
        const uint32_t pos = sub_base[at] + slot;
        if (slot < tile_hist[at] && pos < capacity) keys[pos] = k;
    };
    if (active) {
        key = (static_cast<unsigned long long>(__float_as_uint(depth[i])) << 32) | static_cast<unsigned long long>(static_cast<uint32_t>(i));
        bb = tile_box(cam.grid_x, cam.grid_y, pr.cx, pr.cy, pr.ex, pr.ey);
        cells = (bb.x1 - bb.x0) * (bb.y1 - bb.y0);
        if (!cfg.tile_culling) {
            for (int y = bb.y0; y < bb.y1; ++y)
                for (int x = bb.x0; x < bb.x1; ++x) place(y * cam.grid_x + x, key);
            cells = 0;
        } else {
            maxpow = logf(pr.op / cfg.min_alpha);
            if (cells <= kSmallBox) {
                for (int y = bb.y0; y < bb.y1; ++y)
                    for (int x = bb.x0; x < bb.x1; ++x)
                        if (tile_min_power(static_cast<float>(x), static_cast<float>(y), pr.ca, pr.cb, pr.cc, pr.cx, pr.cy) < maxpow)
                            place(y * cam.grid_x + x, key);
                cells = 0;
            }
        }
    }
    const unsigned lane = threadIdx.x & 31;
    unsigned big = __ballot_sync(0xFFFFFFFFu, cells > kSmallBox);
    while (big) {
        const int src = __ffs(big) - 1;
        big &= big - 1;
        const int bx0 = __shfl_sync(0xFFFFFFFFu, bb.x0, src), by0 = __shfl_sync(0xFFFFFFFFu, bb.y0, src);
        const int bw = __shfl_sync(0xFFFFFFFFu, bb.x1, src) - bx0, nc = __shfl_sync(0xFFFFFFFFu, cells, src);
        const float qa = __shfl_sync(0xFFFFFFFFu, pr.ca, src), qb = __shfl_sync(0xFFFFFFFFu, pr.cb, src), qc = __shfl_sync(0xFFFFFFFFu, pr.cc, src);
        const float qx = __shfl_sync(0xFFFFFFFFu, pr.cx, src), qy = __shfl_sync(0xFFFFFFFFu, pr.cy, src), qp = __shfl_sync(0xFFFFFFFFu, maxpow, src);
        const unsigned long long qk = __shfl_sync(0xFFFFFFFFu, key, src);
        for (int c0 = 0; c0 < nc; c0 += 32) {
            const int c = c0 + static_cast<int>(lane);
            if (c < nc) {
                const int y = by0 + c / bw, x = bx0 + c % bw;
                if (tile_min_power(static_cast<float>(x), static_cast<float>(y), qa, qb, qc, qx, qy) < qp) place(y * cam.grid_x + x, qk);
            }
        }
    }
}

}  // namespace

void launch_project(cudaStream_t s, const FrameCamera& cam, const FrameConfig& cfg, int64_t n, const float* particles,
                    const float* sph, int sph_degree, uint32_t* tiles_count, ProjRecord* proj, float* depth, float* rgb,
                    float* visibility, uint32_t* tile_hist, bool radiance) {
    if (n <= 0) return;
    const unsigned blocks = static_cast<unsigned>((n + kProjThreads - 1) / kProjThreads);
#define GUT_PROJ(ROLLING_, RGB_) project_kernel<ROLLING_, RGB_><<<blocks, kProjThreads, 0, s>>>(cam, cfg, n, particles, sph, sph_degree, tiles_count, proj, depth, rgb, visibility, tile_hist)
    if (cam.rolling_shutter != 0) {
        if (radiance) GUT_PROJ(true, true); else GUT_PROJ(true, false);
    } else {
        if (radiance) GUT_PROJ(false, true); else GUT_PROJ(false, false);
    }
#undef GUT_PROJ
}

void launch_expand_place(cudaStream_t s, const FrameCamera& cam, const FrameConfig& cfg, int64_t n, const ProjRecord* proj, const float* depth,
                         const uint32_t* tile_hist, const uint32_t* sub_base, const uint32_t* totals, uint32_t capacity, uint32_t* fill,
                         unsigned long long* keys) {
    if (n <= 0) return;
    const unsigned blocks = static_cast<unsigned>((n + 255) / 256);
    expand_place_kernel<<<blocks, 256, 0, s>>>(cam, cfg, n, proj, depth, tile_hist, sub_base, totals, capacity, fill, keys);
}

}  // namespace gutb200
