/*
 * oracle/gut_oracle.c -- TEST INFRASTRUCTURE ONLY (see gut_oracle.h).
 *
 * CPU restatement of the reference 3DGUT path, fp32, operation order as written in the
 * reference sources (compile with -ffp-contract=off).  Citations are relative to
 * /root/reference/threedgut_tracer/ unless prefixed otherwise.
 *
 * Differences from the reference that are deliberate and documented in DESIGN.md:
 *  - IEEE division / sqrt / libm logf,expf instead of the -use_fast_math approximations;
 *  - per-particle gradient sums are accumulated in double (a more accurate sum than the
 *    reference's fp32 atomics; the per-(pixel,particle) terms are fp32 as in the reference);
 *  - `visibility` is defined as (valid projection && valid conic); the reference evaluates
 *    the conic test on an uninitialised covariance when the projection was rejected
 *    (include/3dgut/kernels/cuda/renderers/gutProjector.cuh:245-275).
 */
#include "gut_oracle.h"

#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define TILE 16
#define INVALID_U32 0xFFFFFFFFu

/* `real` is float in the oracle proper.  Building with -DORACLE_F64 (libgut_oracle_f64.so) evaluates the
 * per-ray compositing maths in double on the SAME fp32 inputs and sorted lists: that is the "ground truth" the
 * tests use to size the fp32 tolerance (how far two valid fp32 evaluation orders may drift apart). */
#ifdef ORACLE_F64
typedef double real;
#define R_SQRT sqrt
#define R_EXP exp
#define R_FMAX fmax
#define R_FMIN fmin
#else
typedef float real;
#define R_SQRT sqrtf
#define R_EXP expf
#define R_FMAX fmaxf
#define R_FMIN fminf
#endif

typedef struct { real x, y, z; } v3;

static inline v3 V3(real x, real y, real z) { v3 r = {x, y, z}; return r; }
static inline v3 add3(v3 a, v3 b) { return V3(a.x + b.x, a.y + b.y, a.z + b.z); }
static inline v3 sub3(v3 a, v3 b) { return V3(a.x - b.x, a.y - b.y, a.z - b.z); }
static inline v3 mul3(v3 a, v3 b) { return V3(a.x * b.x, a.y * b.y, a.z * b.z); }
static inline v3 scl3(v3 a, real s) { return V3(a.x * s, a.y * s, a.z * s); }
static inline real dot3(v3 a, v3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
static inline v3 cross3(v3 a, v3 b) {
    return V3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}

void gut_oracle_default_config(gut_oracle_config* c) {
    /* configs/render/3dgut.yaml + include/3dgut/threedgut.cuh:54-66 */
    c->kernel_degree = 2;
    c->min_kernel_density = 0.0113f;
    c->min_alpha = 1.0f / 255.0f;
    c->max_alpha = 0.99f;
    c->min_transmittance = 0.0001f;
    c->ut_alpha = 1.0f;
    c->ut_beta = 2.0f;
    c->ut_kappa = 0.0f;
    c->ut_delta = (float)1.7320508075688772;
    c->ut_margin = 0.1f;
    c->rect_bounding = 1;
    c->tight_opacity_bounding = 1;
    c->tile_culling = 1;
    c->global_z_order = 1;
    c->n_rolling_shutter_iterations = 5;
}

/* ------------------------------------------------------------------------------------------ */
/* quaternion / pose helpers: thirdparty/tiny-cuda-nn/include/tiny-cuda-nn/vec.h:1076-1199     */

typedef struct { float w, x, y, z; } quat;
/* column-major 3x3: m[c][r] */
typedef struct { float m[3][3]; } mat3c;

static mat3c quat_to_mat3(quat q) { /* vec.h:1185-1195 */
    float qxx = q.x * q.x, qyy = q.y * q.y, qzz = q.z * q.z;
    float qxz = q.x * q.z, qxy = q.x * q.y, qyz = q.y * q.z;
    float qwx = q.w * q.x, qwy = q.w * q.y, qwz = q.w * q.z;
    mat3c r;
    r.m[0][0] = 1.f - 2.f * (qyy + qzz); r.m[0][1] = 2.f * (qxy + qwz); r.m[0][2] = 2.f * (qxz - qwy);
    r.m[1][0] = 2.f * (qxy - qwz); r.m[1][1] = 1.f - 2.f * (qxx + qzz); r.m[1][2] = 2.f * (qyz + qwx);
    r.m[2][0] = 2.f * (qxz + qwy); r.m[2][1] = 2.f * (qyz - qwx); r.m[2][2] = 1.f - 2.f * (qxx + qyy);
    return r;
}

static quat mat3_to_quat(mat3c a) { /* vec.h:1079-1108 */
    float (*m)[3] = a.m;
    quat q;
    float tr = m[0][0] + m[1][1] + m[2][2];
    if (tr > 0.f) {
        float S = sqrtf(tr + 1.f) * 2.f;
        q.w = 0.25f * S;
        q.x = (m[1][2] - m[2][1]) / S;
        q.y = (m[2][0] - m[0][2]) / S;
        q.z = (m[0][1] - m[1][0]) / S;
    } else if (m[0][0] > m[1][1] && m[0][0] > m[2][2]) {
        float S = sqrtf(1.f + m[0][0] - m[1][1] - m[2][2]) * 2.f;
        q.w = (m[1][2] - m[2][1]) / S;
        q.x = 0.25f * S;
        q.y = (m[1][0] + m[0][1]) / S;
        q.z = (m[2][0] + m[0][2]) / S;
    } else if (m[1][1] > m[2][2]) {
        float S = sqrtf(1.f + m[1][1] - m[0][0] - m[2][2]) * 2.f;
        q.w = (m[2][0] - m[0][2]) / S;
        q.x = (m[1][0] + m[0][1]) / S;
        q.y = 0.25f * S;
        q.z = (m[2][1] + m[1][2]) / S;
    } else {
        float S = sqrtf(1.f + m[2][2] - m[0][0] - m[1][1]) * 2.f;
        q.w = (m[0][1] - m[1][0]) / S;
        q.x = (m[2][0] + m[0][2]) / S;
        q.y = (m[2][1] + m[1][2]) / S;
        q.z = 0.25f * S;
    }
    return q;
}

static quat quat_slerp(quat x, quat y, float t) { /* vec.h:1146-1167 */
    quat z = y;
    float c = (x.w * y.w + x.x * y.x) + (x.y * y.y + x.z * y.z);
    if (c < 0.f) {
        z.w = -y.w; z.x = -y.x; z.y = -y.y; z.z = -y.z;
        c = -c;
    }
    quat r;
    if (c > 1.f - FLT_EPSILON) {
        float a = 1.f - t;
        r.w = x.w * a + z.w * t; r.x = x.x * a + z.x * t; r.y = x.y * a + z.y * t; r.z = x.z * a + z.z * t;
    } else {
        float ang = acosf(c);
        float s0 = sinf((1.f - t) * ang), s1 = sinf(t * ang), sd = sinf(ang);
        r.w = (s0 * x.w + s1 * z.w) / sd; r.x = (s0 * x.x + s1 * z.x) / sd;
        r.y = (s0 * x.y + s1 * z.y) / sd; r.z = (s0 * x.z + s1 * z.z) / sd;
    }
    return r;
}

/* tcnn tmat * tvec (vec.h:595-605): result[j] = ((0 + m[0][j] v0) + m[1][j] v1) + m[2][j] v2 */
static inline v3 mat3c_mul(const mat3c* a, v3 v) {
    float r[3];
    for (int j = 0; j < 3; ++j) {
        float acc = 0.f;
        acc += a->m[0][j] * v.x;
        acc += a->m[1][j] * v.y;
        acc += a->m[2][j] * v.z;
        r[j] = acc;
    }
    return V3(r[0], r[1], r[2]);
}

typedef struct { float t[3]; quat q; } pose;

static pose pose_from7(const float p[7]) { /* sensors.h:33: t.xyz, q.xyzw */
    pose r;
    r.t[0] = p[0]; r.t[1] = p[1]; r.t[2] = p[2];
    r.q.w = p[6]; r.q.x = p[3]; r.q.y = p[4]; r.q.z = p[5];
    return r;
}

static pose pose_interp(pose a, pose b, float t) { /* sensors.h:53-66 */
    pose r;
    r.q = quat_slerp(a.q, b.q, t);
    for (int i = 0; i < 3; ++i) r.t[i] = a.t[i] * (1.f - t) + b.t[i] * t;
    return r;
}

static pose pose_inverse(pose p) { /* sensors.h:44-51 */
    mat3c r = quat_to_mat3(p.q), inv;
    for (int c = 0; c < 3; ++c)
        for (int k = 0; k < 3; ++k) inv.m[c][k] = r.m[k][c];
    pose o;
    o.q = mat3_to_quat(inv);
    mat3c neg;
    for (int c = 0; c < 3; ++c)
        for (int k = 0; k < 3; ++k) neg.m[c][k] = -1.0f * inv.m[c][k];
    v3 t = mat3c_mul(&neg, V3(p.t[0], p.t[1], p.t[2]));
    o.t[0] = t.x; o.t[1] = t.y; o.t[2] = t.z;
    return o;
}

static void pose_to_cols(pose p, float cols[12]) { /* sensors.h:68-73 */
    mat3c r = quat_to_mat3(p.q);
    for (int c = 0; c < 3; ++c)
        for (int k = 0; k < 3; ++k) cols[c * 3 + k] = r.m[c][k];
    cols[9] = p.t[0]; cols[10] = p.t[1]; cols[11] = p.t[2];
}

void gut_oracle_sensor_matrices(const gut_oracle_camera* cam, float view_cols[12], float inv_cols[12],
                                float cam_pos_world[3]) {
    /* src/gutRenderer.cu:266-267,282-284 */
    pose mid = pose_interp(pose_from7(cam->pose_start), pose_from7(cam->pose_end), 0.5f);
    pose inv = pose_inverse(mid);
    pose_to_cols(mid, view_cols);
    pose_to_cols(inv, inv_cols);
    cam_pos_world[0] = inv.t[0]; cam_pos_world[1] = inv.t[1]; cam_pos_world[2] = inv.t[2];
}

uint32_t gut_oracle_higher_msb(uint32_t n) { /* src/gutRenderer.cu:79-94 */
    uint32_t msb = sizeof(n) * 4;
    uint32_t step = msb;
    while (step > 1) {
        step /= 2;
        if (n >> msb) msb += step; else msb -= step;
    }
    if (n >> msb) msb++;
    return msb;
}

/* ------------------------------------------------------------------------------------------ */
/* particle record helpers: include/3dgut/kernels/cuda/models/gaussianParticles.cuh:24-59       */

typedef struct {
    v3 pos; real dns; real qw, qx, qy, qz; v3 scl;
    v3 rot[3]; /* rows of quaternionWXYZToMatrix == columns of the standard rotation R */
} particle;

static particle load_particle(const float* p) {
    particle g;
    g.pos = V3(p[0], p[1], p[2]);
    g.dns = p[3];
    g.qw = p[4]; g.qx = p[5]; g.qy = p[6]; g.qz = p[7];
    g.scl = V3(p[8], p[9], p[10]);
    const real r = g.qw, x = g.qx, y = g.qy, z = g.qz;
    const real xx = x * x, yy = y * y, zz = z * z, xy = x * y, xz = x * z, yz = y * z;
    const real rx = r * x, ry = r * y, rz = r * z;
    g.rot[0] = V3(1.f - 2.f * (yy + zz), 2.f * (xy + rz), 2.f * (xz - ry));
    g.rot[1] = V3(2.f * (xy - rz), 1.f - 2.f * (xx + zz), 2.f * (yz + rx));
    g.rot[2] = V3(2.f * (xz + ry), 2.f * (yz - rx), 1.f - 2.f * (xx + yy));
    return g;
}

/* v * M  (mathUtils.cuh:447-449): (M[0].v, M[1].v, M[2].v) = R^T v */
static inline v3 vecmat(v3 v, const v3 m[3]) { return V3(dot3(m[0], v), dot3(m[1], v), dot3(m[2], v)); }

/* ------------------------------------------------------------------------------------------ */
/* spherical harmonics: models/gaussianParticles.cuh:61-100                                    */

static const float SH_C0 = 0.28209479177387814f;
static const float SH_C1 = 0.4886025119029199f;
static const float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                               -1.0925484305920792f, 0.5462742152960396f};
static const float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f, 0.3731763325901154f,
                               -0.4570457994644658f, 1.445305721320277f, -0.5900435899266435f};

static void sh_basis(int deg, v3 d, real b[16]) {
    const real x = d.x, y = d.y, z = d.z;
    for (int i = 0; i < 16; ++i) b[i] = 0.f;
    b[0] = SH_C0;
    if (deg > 0) {
        b[1] = -SH_C1 * y; b[2] = SH_C1 * z; b[3] = -SH_C1 * x;
        if (deg > 1) {
            const real xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            b[4] = SH_C2[0] * xy; b[5] = SH_C2[1] * yz; b[6] = SH_C2[2] * (2.0f * zz - xx - yy);
            b[7] = SH_C2[3] * xz; b[8] = SH_C2[4] * (xx - yy);
            if (deg > 2) {
                b[9] = SH_C3[0] * y * (3.0f * xx - yy);
                b[10] = SH_C3[1] * xy * z;
                b[11] = SH_C3[2] * y * (4.0f * zz - xx - yy);
                b[12] = SH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy);
                b[13] = SH_C3[4] * x * (4.0f * zz - xx - yy);
                b[14] = SH_C3[5] * z * (xx - yy);
                b[15] = SH_C3[6] * x * (xx - 3.0f * yy);
            }
        }
    }
}

void gut_oracle_sph_eval(int32_t deg, const float c[48], const float dir[3], float out[3]) {
    /* radianceFromSpH(deg, coeffs, dir, clamped=false): same association order as the reference */
    const float x = dir[0], y = dir[1], z = dir[2];
    for (int k = 0; k < 3; ++k) {
#define CF(i) c[(i) * 3 + k]
        float rad = SH_C0 * CF(0);
        if (deg > 0) {
            rad = rad - SH_C1 * y * CF(1) + SH_C1 * z * CF(2) - SH_C1 * x * CF(3);
            if (deg > 1) {
                const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                rad = rad + SH_C2[0] * xy * CF(4) + SH_C2[1] * yz * CF(5) + SH_C2[2] * (2.0f * zz - xx - yy) * CF(6) +
                      SH_C2[3] * xz * CF(7) + SH_C2[4] * (xx - yy) * CF(8);
                if (deg > 2) {
                    rad = rad + SH_C3[0] * y * (3.0f * xx - yy) * CF(9) + SH_C3[1] * xy * z * CF(10) +
                          SH_C3[2] * y * (4.0f * zz - xx - yy) * CF(11) +
                          SH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * CF(12) +
                          SH_C3[4] * x * (4.0f * zz - xx - yy) * CF(13) + SH_C3[5] * z * (xx - yy) * CF(14) +
                          SH_C3[6] * x * (xx - 3.0f * yy) * CF(15);
                }
            }
        }
#undef CF
        out[k] = rad + 0.5f;
    }
}

/* ------------------------------------------------------------------------------------------ */
/* pinhole projection: include/3dgut/kernels/cuda/sensors/cameraProjections.cuh:67-118,218-233 */

static int within_resolution(float rx, float ry, float tol, float px, float py) {
    const float mx = rx * tol, my = ry * tol;
    return (px > -mx) && (py > -my) && (px < rx + mx) && (py < ry + my);
}

static int project_pinhole(const gut_oracle_camera* cam, v3 p, float tol, float out[2]) {
    if (p.z <= 0.f) {
        out[0] = 0.f; out[1] = 0.f;
        return 0;
    }
    const float u = p.x / p.z, v = p.y / p.z;
    const float uu = u * u, vv = v * v;
    const float r2 = uu + vv;
    const float a1 = 2.f * u * v;
    const float a2 = r2 + 2.f * uu;
    const float a3 = r2 + 2.f * vv;
    const float* k = cam->radial;
    const float num = 1.f + r2 * (k[0] + r2 * (k[1] + r2 * k[2]));
    const float den = 1.f + r2 * (k[3] + r2 * (k[4] + r2 * k[5]));
    const float icd = num / den;
    const float* t = cam->tangential;
    const float* s = cam->thin_prism;
    const float dx = t[0] * a1 + t[1] * a2 + r2 * (s[0] + r2 * s[1]);
    const float dy = t[0] * a3 + t[1] * a1 + r2 * (s[2] + r2 * s[3]);
    const float ndx = icd * u + dx, ndy = icd * v + dy;
    const int valid_radial = (icd > 0.8f) && (icd < 1.2f);
    if (valid_radial) {
        out[0] = ndx * cam->focal[0] + cam->principal[0];
        out[1] = ndy * cam->focal[1] + cam->principal[1];
    } else {
        const float clip = hypotf((float)cam->width, (float)cam->height);
        const float f = clip / sqrtf(r2);
        out[0] = f * u + cam->principal[0];
        out[1] = f * v + cam->principal[1];
    }
    return valid_radial && within_resolution((float)cam->width, (float)cam->height, tol, out[0], out[1]);
}

/* OpenCV fisheye projection: cameraProjections.cuh:25-35 (stableNorm2), 38-48 (evalPolyHorner), 120-146 */
static float stable_norm2(float x, float y) {
    const float ax = fabsf(x), ay = fabsf(y);
    const float mn = fminf(ax, ay), mx = fmaxf(ax, ay);
    if (mx <= 0.f) return 0.f;
    const float ratio = mn / mx;
    return mx * sqrtf(1.f + ratio * ratio);
}

static int project_fisheye(const gut_oracle_camera* cam, v3 p, float tol, float out[2]) {
    const float px = (float)p.x, py = (float)p.y, pz = (float)p.z;
    float rho = stable_norm2(px, py);
    if (rho <= 0.f) rho = FLT_EPSILON;
    const float theta_full = atan2f(rho, pz);
    const float theta = fminf(theta_full, cam->max_angle);   /* FOV-clamped projections are marked invalid below */
    const float theta2 = theta * theta;
    const float* k = cam->radial;
    float poly = k[3];
    poly = theta2 * poly + k[2];
    poly = theta2 * poly + k[1];
    poly = theta2 * poly + k[0];
    const float delta = (theta * (poly * theta2 + 1.0f)) / rho;
    out[0] = cam->focal[0] * px * delta + cam->principal[0];
    out[1] = cam->focal[1] * py * delta + cam->principal[1];
    return (theta < cam->max_angle) && within_resolution((float)cam->width, (float)cam->height, tol, out[0], out[1]);
}

/* f-theta projection: cameraProjections.cuh:148-198 (PolynomialDegree = 6 coefficients, 3 Newton iterations) */
static float horner(const float* c, int n, float x) { /* evalPolyHorner<N>, :38-48 */
    float y = c[n - 1];
    for (int i = n - 2; i >= 0; --i) y = x * y + c[i];
    return y;
}

static int project_ftheta(const gut_oracle_camera* cam, v3 p, float tol, float out[2]) {
    const float px = (float)p.x, py = (float)p.y, pz = (float)p.z;
    float rho = stable_norm2(px, py);
    if (rho <= 0.f) rho = FLT_EPSILON;
    const float theta_full = atan2f(rho, pz);
    const float theta = fminf(theta_full, cam->max_angle);
    float delta = 0.f;
    if (cam->ftheta_reference_poly == 0) {
        /* the backward polynomial is the reference: invert it with Newton iterations started from the forward polynomial */
        delta = horner(cam->ftheta_fw, 6, theta);
        float dpoly[5];
        for (int i = 1; i < 6; ++i) dpoly[i - 1] = i * cam->ftheta_bw[i];
        for (int i = 0; i < 3; ++i) {
            const float dfdx = horner(dpoly, 5, delta);
            const float residual = horner(cam->ftheta_bw, 6, delta) - theta;
            delta -= residual / dfdx;
        }
    } else {
        delta = horner(cam->ftheta_fw, 6, theta);
    }
    const float* cde = cam->ftheta_cde;
    const float s = delta / rho;
    out[0] = s * (cde[0] * px + cde[1] * py);
    out[1] = s * (cde[2] * px + py);
    /* the image coordinate origin of the f-theta model is the centre of the first pixel */
    out[0] += cam->principal[0] + .5f;
    out[1] += cam->principal[1] + .5f;
    return (theta < cam->max_angle) && within_resolution((float)cam->width, (float)cam->height, tol, out[0], out[1]);
}

static int project_sensor_point(const gut_oracle_camera* cam, v3 s, float tol, float out[2]) { /* projectPoint(TSensorModel), :200-216 */
    if (cam->model == 1) return project_fisheye(cam, s, tol, out);
    if (cam->model == 2) return project_ftheta(cam, s, tol, out);
    return project_pinhole(cam, s, tol, out);
}

static int project_with_pose(const gut_oracle_camera* cam, quat q, const float t[3], v3 p, float tol, float out[2]) {
    const mat3c r = quat_to_mat3(q);
    v3 s = mat3c_mul(&r, p);
    s = V3(s.x + t[0], s.y + t[1], s.z + t[2]);
    return project_sensor_point(cam, s, tol, out);
}

/* relativeShutterTime (cameraProjections.cuh:50-65) */
static float relative_shutter_time(const gut_oracle_camera* cam, const float pos[2]) {
    const float rx = (float)cam->width, ry = (float)cam->height;
    switch (cam->rolling_shutter) {
        case 1: return floorf(pos[1]) / (ry - 1.f);
        case 2: return floorf(pos[0]) / (rx - 1.f);
        case 3: return (ry - ceilf(pos[1])) / (ry - 1.f);
        case 4: return (rx - ceilf(pos[0])) / (rx - 1.f);
        default: return 0.5f;
    }
}

/* projectPointWithShutter (cameraProjections.cuh:218-257): start pose; for a rolling shutter fall back to the end pose when the
 * start pose fails, then iterate pose(time of the projected row / column) -> projection */
static int project_world_point(const gut_oracle_camera* cam, int iterations, const pose* ps, const pose* pe, v3 p, float tol,
                               float out[2]) {
    int valid = project_with_pose(cam, ps->q, ps->t, p, tol, out);
    if (cam->rolling_shutter == 0) return valid;
    if (!valid) {
        valid = project_with_pose(cam, pe->q, pe->t, p, tol, out);
        if (!valid) return 0;
    }
    for (int i = 0; i < iterations; ++i) {
        const float alpha = relative_shutter_time(cam, out);
        const quat q = quat_slerp(ps->q, pe->q, alpha);
        float t[3];
        for (int k = 0; k < 3; ++k) t[k] = ps->t[k] * (1.f - alpha) + pe->t[k] * alpha;  /* tcnn::mix (vec.h:183) */
        valid = project_with_pose(cam, q, t, p, tol, out);
    }
    return valid;
}

/* ------------------------------------------------------------------------------------------ */
/* tile helpers: renderers/gutProjector.cuh:32-78                                              */

typedef struct { int x0, y0, x1, y1; } bbox2;

static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int imax(int a, int b) { return a > b ? a : b; }

static bbox2 tile_bbox(int gx, int gy, float cx, float cy, float ex, float ey) {
    bbox2 b;
    b.x0 = imin(gx, imax(0, (int)floorf((cx - 0.5f - ex) / (float)TILE)));
    b.y0 = imin(gy, imax(0, (int)floorf((cy - 0.5f - ey) / (float)TILE)));
    b.x1 = imin(gx, imax(0, (int)ceilf((cx - 0.5f + ex) / (float)TILE)));
    b.y1 = imin(gy, imax(0, (int)ceilf((cy - 0.5f + ey) / (float)TILE)));
    return b;
}

static inline float saturatef(float x) { return fminf(fmaxf(x, 0.f), 1.f); }

static float tile_min_power(float tx, float ty, const float co[4], float mx, float my) {
    const float ts = (float)TILE;
    const float tminx = ts * tx, tminy = ts * ty;
    const float tmaxx = ts + tminx, tmaxy = ts + tminy;
    const float mox = tminx - mx, moy = tminy - my;
    const float lax = mox > 0.0f ? 1.f : 0.f, lay = moy > 0.0f ? 1.f : 0.f;
    const float nrx = lax + (mx > tmaxx ? 1.f : 0.f);
    const float nry = lay + (my > tmaxy ? 1.f : 0.f);
    if ((nrx + nry) > 0.0f) {
        /* tcnn::mix(tileMax, tileMin, leftAbove) = a*(1-c) + b*c */
        const float px = tmaxx * (1.f - lax) + tminx * lax;
        const float py = tmaxy * (1.f - lay) + tminy * lay;
        const float dxx = copysignf(ts, mox), dxy = copysignf(ts, moy);
        const float dfx = mx - px, dfy = my - py;
        const float rcx = 1.0f / (ts * ts * co[0]);
        const float rcy = 1.0f / (ts * ts * co[2]);
        const float tx_ = nry * saturatef((dxx * co[0] * dfx + dxx * co[1] * dfy) * rcx);
        const float ty_ = nrx * saturatef((dxy * co[1] * dfx + dxy * co[2] * dfy) * rcy);
        const float mdx = mx - (px + tx_ * dxx);
        const float mdy = my - (py + ty_ * dxy);
        return 0.5f * (co[0] * mdx * mdx + co[2] * mdy * mdy) + co[1] * mdx * mdy;
    }
    return 0.f;
}

/* ------------------------------------------------------------------------------------------ */
/* G1 projectOnTiles                                                                            */

void gut_oracle_project(const gut_oracle_config* cfg, const gut_oracle_camera* cam, int64_t n, const float* particles,
                        const float* sph, int32_t sph_degree, uint32_t* tiles_count, float* proj_pos,
                        float* conic_opacity, float* extent, float* depth, float* rgb, int32_t* visibility) {
    float view[12], inv[12], campos[3];
    gut_oracle_sensor_matrices(cam, view, inv, campos);
    const pose ps = pose_from7(cam->pose_start), pe = pose_from7(cam->pose_end);
    const int rs_iters = cfg->n_rolling_shutter_iterations;
    const int gx = (cam->width + TILE - 1) / TILE, gy = (cam->height + TILE - 1) / TILE;
    const float D = 3.f;
    const float lambda = cfg->ut_alpha * cfg->ut_alpha * (D + cfg->ut_kappa) - D;
    const float w0m = lambda / (D + lambda);
    const float wi = 1.f / (2.f * (D + lambda));
    const float w0c = lambda / (D + lambda) + (1.f - cfg->ut_alpha * cfg->ut_alpha + cfg->ut_beta);

#pragma omp parallel for schedule(dynamic, 1024)
    for (int64_t i = 0; i < n; ++i) {
        const particle g = load_particle(particles + i * 12);
        int valid_proj = 0, valid_conic = 0;
        float pc[2] = {0.f, 0.f}, cov[3] = {0.f, 0.f, 0.f};
        v3 sray = V3(0.f, 0.f, 0.f);
        float opacity = g.dns;
        /* unscentedParticleProjection (gutProjector.cuh:118-215) */
        do {
            if (opacity < cfg->min_alpha) break;
            const float zc = g.pos.x * view[0 * 3 + 2] + g.pos.y * view[1 * 3 + 2] + g.pos.z * view[2 * 3 + 2] + view[3 * 3 + 2];
            if (zc < 0.2f) break;
            sray = sub3(g.pos, V3(campos[0], campos[1], campos[2]));
            float sp[7][2];
            int nvalid = 0;
            nvalid += project_world_point(cam, rs_iters, &ps, &pe, g.pos, cfg->ut_margin, sp[0]);
            pc[0] = sp[0][0] * w0m;
            pc[1] = sp[0][1] * w0m;
            const float sc[3] = {g.scl.x, g.scl.y, g.scl.z};
            for (int k = 0; k < 3; ++k) {
                const v3 delta = scl3(g.rot[k], cfg->ut_delta * sc[k]);
                nvalid += project_world_point(cam, rs_iters, &ps, &pe, add3(g.pos, delta), cfg->ut_margin, sp[k + 1]);
                pc[0] += wi * sp[k + 1][0];
                pc[1] += wi * sp[k + 1][1];
                nvalid += project_world_point(cam, rs_iters, &ps, &pe, sub3(g.pos, delta), cfg->ut_margin, sp[k + 4]);
                pc[0] += wi * sp[k + 4][0];
                pc[1] += wi * sp[k + 4][1];
            }
            if (nvalid == 0) break;
            {
                const float cx = sp[0][0] - pc[0], cy = sp[0][1] - pc[1];
                cov[0] = w0c * (cx * cx);
                cov[1] = w0c * (cx * cy);
                cov[2] = w0c * (cy * cy);
            }
            for (int k = 0; k < 6; ++k) {
                const float cx = sp[k + 1][0] - pc[0], cy = sp[k + 1][1] - pc[1];
                cov[0] += wi * (cx * cx);
                cov[1] += wi * (cx * cy);
                cov[2] += wi * (cy * cy);
            }
            valid_proj = 1;
        } while (0);

        /* computeProjectedExtentConicOpacity (gutProjector.cuh:81-116) */
        float ext[2] = {0.f, 0.f}, co[4] = {0.f, 0.f, 0.f, 0.f}, maxpow = 0.f;
        if (valid_proj) do {
            const float dcx = cov[0] + 0.3f, dcy = cov[1], dcz = cov[2] + 0.3f;
            const float ddet = dcx * dcz - dcy * dcy;
            if (ddet == 0.0f) break;
            co[0] = dcz / ddet;
            co[1] = -dcy / ddet;
            co[2] = dcx / ddet;
            const float cdet = cov[0] * cov[2] - cov[1] * cov[1];
            const float conv = sqrtf(fmaxf(0.000025f, cdet / ddet));
            co[3] = opacity * conv;
            if (co[3] < cfg->min_alpha) break;
            maxpow = logf(co[3] / cfg->min_alpha);
            const float ef = cfg->tight_opacity_bounding ? fminf(3.33f, sqrtf(2.0f * maxpow)) : 3.33f;
            const float mid = 0.5f * (dcx + dcz);
            const float lam = mid + sqrtf(fmaxf(0.01f, mid * mid - ddet));
            const float radius = ef * sqrtf(lam);
            if (cfg->rect_bounding) {
                ext[0] = fminf(ef * sqrtf(dcx), radius);
                ext[1] = fminf(ef * sqrtf(dcz), radius);
            } else {
                ext[0] = radius; ext[1] = radius;
            }
            valid_conic = radius > 0.f;
        } while (0);

        visibility[i] = (valid_proj && valid_conic) ? 1 : 0;
        uint32_t ntiles = 0;
        if (valid_proj && valid_conic) {
            const bbox2 bb = tile_bbox(gx, gy, pc[0], pc[1], ext[0], ext[1]);
            if (cfg->tile_culling) {
                for (int y = bb.y0; y < bb.y1; ++y)
                    for (int x = bb.x0; x < bb.x1; ++x)
                        if (tile_min_power((float)x, (float)y, co, pc[0], pc[1]) < maxpow) ntiles++;
            } else {
                ntiles = (uint32_t)((bb.x1 - bb.x0) * (bb.y1 - bb.y0));
            }
        }
        tiles_count[i] = ntiles;
        if (ntiles == 0) {
            proj_pos[i * 2] = proj_pos[i * 2 + 1] = 0.f;
            conic_opacity[i * 4] = conic_opacity[i * 4 + 1] = conic_opacity[i * 4 + 2] = conic_opacity[i * 4 + 3] = 0.f;
            extent[i * 2] = extent[i * 2 + 1] = 0.f;
            depth[i] = 0.f;
            rgb[i * 3] = rgb[i * 3 + 1] = rgb[i * 3 + 2] = 0.f; /* reference leaves this slot stale */
            continue;
        }
        const float dist = sqrtf(sray.x * sray.x + sray.y * sray.y + sray.z * sray.z);
        const float dir[3] = {sray.x / dist, sray.y / dist, sray.z / dist};
        gut_oracle_sph_eval(sph_degree, sph + i * 48, dir, rgb + i * 3);
        proj_pos[i * 2] = pc[0]; proj_pos[i * 2 + 1] = pc[1];
        memcpy(conic_opacity + i * 4, co, sizeof(co));
        extent[i * 2] = ext[0]; extent[i * 2 + 1] = ext[1];
        if (cfg->global_z_order) {
            depth[i] = g.pos.x * view[0 * 3 + 2] + g.pos.y * view[1 * 3 + 2] + g.pos.z * view[2 * 3 + 2] + view[3 * 3 + 2];
        } else {
            depth[i] = dist;
        }
    }
}

/* ------------------------------------------------------------------------------------------ */
/* G2-G5 scan / expand / sort / ranges                                                          */

static void radix_sort_pairs(uint64_t* k0, uint32_t* v0, uint64_t* k1, uint32_t* v1, int64_t n, int end_bit) {
    /* stable LSD radix sort, 8-bit digits, on bits [0,end_bit) -- semantics of
     * cub::DeviceRadixSort::SortPairs(begin_bit=0,end_bit) (src/gutRenderer.cu:356-365). Result ends in k1/v1. */
    uint64_t* ks = k0; uint32_t* vs = v0; uint64_t* kd = k1; uint32_t* vd = v1;
    int passes = (end_bit + 7) / 8;
    for (int p = 0; p < passes; ++p) {
        const int shift = p * 8;
        const int bits = (end_bit - shift) < 8 ? (end_bit - shift) : 8;
        const uint64_t mask = (1ull << bits) - 1;
        int64_t hist[257];
        memset(hist, 0, sizeof(hist));
        for (int64_t i = 0; i < n; ++i) hist[((ks[i] >> shift) & mask) + 1]++;
        for (int d = 0; d < 256; ++d) hist[d + 1] += hist[d];
        for (int64_t i = 0; i < n; ++i) {
            const int64_t dst = hist[(ks[i] >> shift) & mask]++;
            kd[dst] = ks[i];
            vd[dst] = vs[i];
        }
        uint64_t* tk = ks; ks = kd; kd = tk;
        uint32_t* tv = vs; vs = vd; vd = tv;
    }
    if (ks != k1) {
        memcpy(k1, ks, (size_t)n * sizeof(uint64_t));
        memcpy(v1, vs, (size_t)n * sizeof(uint32_t));
    }
}

int64_t gut_oracle_bin(const gut_oracle_config* cfg, const gut_oracle_camera* cam, int64_t n,
                       const uint32_t* tiles_count, const float* proj_pos, const float* conic_opacity,
                       const float* extent, const float* depth, uint64_t* ukeys, uint32_t* uvals, uint64_t* skeys,
                       uint32_t* svals, uint32_t* ranges) {
    const int gx = (cam->width + TILE - 1) / TILE, gy = (cam->height + TILE - 1) / TILE;
    /* inclusive scan (src/gutRenderer.cu:303) */
    uint32_t* offs = (uint32_t*)malloc((size_t)(n > 0 ? n : 1) * sizeof(uint32_t));
    uint32_t run = 0;
    for (int64_t i = 0; i < n; ++i) { run += tiles_count[i]; offs[i] = run; }
    const int64_t total = run;
    /* expand (gutProjector.cuh:324-388) */
    for (int64_t i = 0; i < n; ++i) {
        const float ex = extent[i * 2], ey = extent[i * 2 + 1];
        if (ex <= 1e-06f) continue;
        uint32_t dkey;
        memcpy(&dkey, &depth[i], 4);
        uint32_t off = (i == 0) ? 0 : offs[i - 1];
        const uint32_t maxoff = offs[i];
        const float cx = proj_pos[i * 2], cy = proj_pos[i * 2 + 1];
        const bbox2 bb = tile_bbox(gx, gy, cx, cy, ex, ey);
        if (cfg->tile_culling) {
            const float* co = conic_opacity + i * 4;
            const float maxpow = logf(co[3] / cfg->min_alpha);
            for (int y = bb.y0; (y < bb.y1) && (off < maxoff); ++y)
                for (int x = bb.x0; (x < bb.x1) && (off < maxoff); ++x)
                    if (tile_min_power((float)x, (float)y, co, cx, cy) < maxpow) {
                        ukeys[off] = ((uint64_t)(uint32_t)(y * gx + x) << 32) | dkey;
                        uvals[off] = (uint32_t)i;
                        off++;
                    }
            for (; off < maxoff; ++off) {
                const float fm = 3.4028235e+38f;
                uint32_t fb;
                memcpy(&fb, &fm, 4);
                ukeys[off] = ((uint64_t)INVALID_U32 << 32) | fb;
                uvals[off] = INVALID_U32;
            }
        } else {
            for (int y = bb.y0; y < bb.y1; ++y)
                for (int x = bb.x0; x < bb.x1; ++x) {
                    ukeys[off] = ((uint64_t)(uint32_t)(y * gx + x) << 32) | dkey;
                    uvals[off] = (uint32_t)i;
                    off++;
                }
        }
    }
    free(offs);
    /* sort */
    const int end_bit = 32 + (int)gut_oracle_higher_msb((uint32_t)(gx * gy));
    if (total > 0) {
        uint64_t* tk = (uint64_t*)malloc((size_t)total * sizeof(uint64_t));
        uint32_t* tv = (uint32_t*)malloc((size_t)total * sizeof(uint32_t));
        memcpy(tk, ukeys, (size_t)total * sizeof(uint64_t));
        memcpy(tv, uvals, (size_t)total * sizeof(uint32_t));
        uint64_t* tk2 = (uint64_t*)malloc((size_t)total * sizeof(uint64_t));
        uint32_t* tv2 = (uint32_t*)malloc((size_t)total * sizeof(uint32_t));
        radix_sort_pairs(tk, tv, tk2, tv2, total, end_bit);
        memcpy(skeys, tk2, (size_t)total * sizeof(uint64_t));
        memcpy(svals, tv2, (size_t)total * sizeof(uint32_t));
        free(tk); free(tv); free(tk2); free(tv2);
    }
    /* ranges (src/gutRenderer.cu:46-76); buffer zeroed first (:161) */
    memset(ranges, 0, (size_t)gx * gy * 2 * sizeof(uint32_t));
    for (int64_t k = 0; k < total; ++k) {
        const uint32_t tile = (uint32_t)(skeys[k] >> 32);
        const int valid = tile != INVALID_U32;
        if (k == 0) {
            if (valid) ranges[tile * 2] = (uint32_t)k;
        } else {
            const uint32_t prev = (uint32_t)(skeys[k - 1] >> 32);
            if (prev != tile) {
                if (prev != INVALID_U32) ranges[prev * 2 + 1] = (uint32_t)k;
                if (valid) ranges[tile * 2] = (uint32_t)k;
            }
        }
        if (valid && (k == total - 1)) ranges[tile * 2 + 1] = (uint32_t)total;
    }
    return total;
}

/* ------------------------------------------------------------------------------------------ */
/* ray setup: kernels/cuda/common/rayPayload.cuh:76-108, utils/bounding_box.h:89-134            */

static void aabb_intersect(v3 o, v3 d, real* tmin_o, real* tmax_o) {
    const real lo = -1e06f, hi = 1e06f; /* src/splatRaster.cpp:240 */
    real tmin = (lo - o.x) / d.x, tmax = (hi - o.x) / d.x, t;
    if (tmin > tmax) { t = tmin; tmin = tmax; tmax = t; }
    real tymin = (lo - o.y) / d.y, tymax = (hi - o.y) / d.y;
    if (tymin > tymax) { t = tymin; tymin = tymax; tymax = t; }
    if (tmin > tymax || tymin > tmax) { *tmin_o = FLT_MAX; *tmax_o = FLT_MAX; return; }
    if (tymin > tmin) tmin = tymin;
    if (tymax < tmax) tmax = tymax;
    real tzmin = (lo - o.z) / d.z, tzmax = (hi - o.z) / d.z;
    if (tzmin > tzmax) { t = tzmin; tzmin = tzmax; tzmax = t; }
    if (tmin > tzmax || tzmin > tmax) { *tmin_o = FLT_MAX; *tmax_o = FLT_MAX; return; }
    if (tzmin > tmin) tmin = tzmin;
    if (tzmax < tmax) tmax = tzmax;
    *tmin_o = tmin; *tmax_o = tmax;
}

typedef struct { v3 o, d; real tmin, tmax; int alive; } ray_t;

static ray_t init_ray(const float inv[12], const float* ro, const float* rd) {
    ray_t r;
    real o[3], d[3];
    for (int j = 0; j < 3; ++j) {
        real acc = 0.f;
        acc += inv[0 * 3 + j] * ro[0];
        acc += inv[1 * 3 + j] * ro[1];
        acc += inv[2 * 3 + j] * ro[2];
        acc += inv[3 * 3 + j] * 1.0f;
        o[j] = acc;
        real acd = 0.f;
        acd += inv[0 * 3 + j] * rd[0];
        acd += inv[1 * 3 + j] * rd[1];
        acd += inv[2 * 3 + j] * rd[2];
        d[j] = acd;
    }
    r.o = V3(o[0], o[1], o[2]);
    r.d = V3(d[0], d[1], d[2]);
    aabb_intersect(r.o, r.d, &r.tmin, &r.tmax);
    r.tmin = R_FMAX(r.tmin, 0.0f);
    r.alive = r.tmax > r.tmin;
    return r;
}

/* ------------------------------------------------------------------------------------------ */
/* per-hit math: slang/models/gaussianParticles.slang:96-274 (forward), CUDA twin
 * models/gaussianParticles.cuh:350-422                                                         */

static inline real kernel_response(int degree, real gray) {
    switch (degree) { /* models/gaussianParticles.cuh:267-308 */
    case 8: { const real g2 = gray * gray; return R_EXP(-0.000685871056241f * g2 * g2); }
    case 5: return R_EXP(-0.0185185185185f * gray * gray * R_SQRT(gray));
    case 4: return R_EXP(-0.0555555555556f * gray * gray);
    case 3: return R_EXP(-0.166666666667f * gray * R_SQRT(gray));
    case 1: return R_EXP(-1.5f * R_SQRT(gray));
    case 0: return R_FMAX(1.f + -0.329630334487f * R_SQRT(gray), 0.f);
    default: return R_EXP(-0.5f * gray);
    }
}

static inline v3 safe_normalize(v3 v) { /* mathUtils.cuh:380-383 */
    const real l = v.x * v.x + v.y * v.y + v.z * v.z;
    return l > 0.0f ? scl3(v, 1.0f / R_SQRT(l)) : v;
}

typedef struct { v3 giscl, gposc, gposcr, gro, rayDirR, grdu, grd, gcrod; real gray, gres, galpha; int accept; } hit_t;

static hit_t eval_hit(const gut_oracle_config* cfg, const particle* g, v3 ro, v3 rd) {
    hit_t h;
    h.giscl = V3(1 / g->scl.x, 1 / g->scl.y, 1 / g->scl.z);
    h.gposc = sub3(ro, g->pos);
    h.gposcr = vecmat(h.gposc, g->rot);
    h.gro = mul3(h.giscl, h.gposcr);
    h.rayDirR = vecmat(rd, g->rot);
    h.grdu = mul3(h.giscl, h.rayDirR);
    h.grd = safe_normalize(h.grdu);
    h.gcrod = cross3(h.grd, h.gro);
    h.gray = dot3(h.gcrod, h.gcrod);
    h.gres = kernel_response(cfg->kernel_degree, h.gray);
    h.galpha = R_FMIN(cfg->max_alpha, h.gres * g->dns);
    h.accept = (h.gres > cfg->min_kernel_density) && (h.galpha > cfg->min_alpha);
    return h;
}

static inline real hit_distance(const particle* g, const hit_t* h) {
    const v3 grds = mul3(g->scl, scl3(h->grd, dot3(h->grd, scl3(h->gro, -1.f))));
    return R_SQRT(dot3(grds, grds));
}

int gut_oracle_hit_forward(const gut_oracle_config* cfg, const float ro[3], const float rd[3], const float p[12],
                           float* alpha, float* hit_t_out) {
    const particle g = load_particle(p);
    const hit_t h = eval_hit(cfg, &g, V3(ro[0], ro[1], ro[2]), V3(rd[0], rd[1], rd[2]));
    *alpha = (float)h.galpha;
    *hit_t_out = h.accept ? (float)hit_distance(&g, &h) : 0.f;
    return h.accept;
}

/* bench-only: process every k-th tile in the render loops (bounded CPU sample of a full-size frame) */
static int g_tile_stride = 1;
void gut_oracle_set_tile_stride(int k) { g_tile_stride = k > 0 ? k : 1; }

/* G6 */
void gut_oracle_render_forward(const gut_oracle_config* cfg, const gut_oracle_camera* cam, const float* rays_o,
                               const float* rays_d, const float* particles, const float* rgb,
                               const uint32_t* svals, const uint32_t* ranges, float* out_rgba, float* out_dist,
                               float* out_hits) {
    float view[12], inv[12], campos[3];
    gut_oracle_sensor_matrices(cam, view, inv, campos);
    const int W = cam->width, H = cam->height;
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
#pragma omp parallel for schedule(dynamic, 1)
    for (int tile = 0; tile < gx * gy; ++tile) {
        if (tile % g_tile_stride) continue;
        const int tx = tile % gx, ty = tile / gx;
        const uint32_t b = ranges[tile * 2], e = ranges[tile * 2 + 1];
        for (int py = ty * TILE; py < imin(H, (ty + 1) * TILE); ++py)
            for (int px = tx * TILE; px < imin(W, (tx + 1) * TILE); ++px) {
                const int64_t pix = px + (int64_t)W * py;
                ray_t r = init_ray(inv, rays_o + pix * 3, rays_d + pix * 3);
                /* outputs keep their initial values for invalid rays (src/splatRaster.cpp:212-215) */
                out_rgba[pix * 4] = out_rgba[pix * 4 + 1] = out_rgba[pix * 4 + 2] = out_rgba[pix * 4 + 3] = 0.f;
                out_dist[pix] = 1e06f;
                out_hits[pix] = 0.f;
                if (!r.alive) continue;
                real T = 1.f, cr = 0.f, cg = 0.f, cb = 0.f, dist = 0.f;
                uint32_t hits = 0;
                for (uint32_t k = b; k < e; ++k) {
                    const uint32_t idx = svals[k];
                    if (idx == INVALID_U32) break;
                    const particle g = load_particle(particles + (int64_t)idx * 12);
                    const hit_t h = eval_hit(cfg, &g, r.o, r.d);
                    if (!h.accept) continue;
                    const real t = hit_distance(&g, &h);
                    if (!(t > r.tmin && t < r.tmax)) continue;
                    const real w = h.galpha * T;
                    dist += t * w;
                    T *= (1 - h.galpha);
                    if (w > 0.0f) {
                        cr += R_FMAX(rgb[idx * 3], 0.f) * w;
                        cg += R_FMAX(rgb[idx * 3 + 1], 0.f) * w;
                        cb += R_FMAX(rgb[idx * 3 + 2], 0.f) * w;
                        hits++;
                    }
                    if (T < cfg->min_transmittance) break;
                }
                out_rgba[pix * 4] = cr; out_rgba[pix * 4 + 1] = cg; out_rgba[pix * 4 + 2] = cb;
                out_rgba[pix * 4 + 3] = 1.0f - T;
                out_dist[pix] = dist;
                out_hits[pix] = (real)hits;
            }
    }
}

/* G6 with a k-buffer (GAUSSIAN_K_BUFFER_SIZE = K > 0, "sorted" 3DGUT: renderers/gutKBufferRenderer.cuh:62-112 insert / closestHit,
 * :150-225 processHitParticle forward branch, :274-352 evalKBuffer).  Hits enter a per-ray buffer of the K farthest-so-far hits sorted
 * by hit distance; when it is full the closest one is composited before the new hit is inserted; the rest is composited in order at the
 * end.  The CUDA twin is 3dgrut_b200/csrc/gut_render_kbuffer.cu (walk in kbuffer_walk.cuh); tests/test_kbuffer_gpu.py compares the two. */
typedef struct { int idx; real t, alpha; } khit_t;

void gut_oracle_render_forward_kbuffer(const gut_oracle_config* cfg, const gut_oracle_camera* cam, int32_t K, const float* rays_o,
                                       const float* rays_d, const float* particles, const float* rgb, const uint32_t* svals,
                                       const uint32_t* ranges, float* out_rgba, float* out_dist, float* out_hits) {
    float view[12], inv[12], campos[3];
    gut_oracle_sensor_matrices(cam, view, inv, campos);
    const int W = cam->width, H = cam->height;
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    if (K < 1 || K > 64) return;
#pragma omp parallel for schedule(dynamic, 1)
    for (int tile = 0; tile < gx * gy; ++tile) {
        if (tile % g_tile_stride) continue;
        const int tx = tile % gx, ty = tile / gx;
        const uint32_t b = ranges[tile * 2], e = ranges[tile * 2 + 1];
        for (int py = ty * TILE; py < imin(H, (ty + 1) * TILE); ++py)
            for (int px = tx * TILE; px < imin(W, (tx + 1) * TILE); ++px) {
                const int64_t pix = px + (int64_t)W * py;
                ray_t r = init_ray(inv, rays_o + pix * 3, rays_d + pix * 3);
                out_rgba[pix * 4] = out_rgba[pix * 4 + 1] = out_rgba[pix * 4 + 2] = out_rgba[pix * 4 + 3] = 0.f;
                out_dist[pix] = 1e06f;
                out_hits[pix] = 0.f;
                if (!r.alive) continue;
                real T = 1.f, cr = 0.f, cg = 0.f, cb = 0.f, dist = 0.f;
                uint32_t hits = 0;
                int alive = 1, num = 0;
                khit_t kb[64];
                for (int i = 0; i < K; ++i) { kb[i].idx = -1; kb[i].t = -1.0f; kb[i].alpha = 0.f; }  /* InvalidHitT = -1 (:31) */
#define KB_PROCESS(HIT)                                                                         \
    do {                                                                                        \
        const khit_t hp_ = (HIT);                                                               \
        const real w_ = hp_.alpha * T;                                                          \
        dist += hp_.t * w_;                                                                     \
        T *= (1 - hp_.alpha);                                                                   \
        if (w_ > 0.0f) {                                                                        \
            cr += R_FMAX(rgb[hp_.idx * 3], 0.f) * w_;                                           \
            cg += R_FMAX(rgb[hp_.idx * 3 + 1], 0.f) * w_;                                       \
            cb += R_FMAX(rgb[hp_.idx * 3 + 2], 0.f) * w_;                                       \
            hits++;                                                                             \
        }                                                                                       \
        if (T < cfg->min_transmittance) alive = 0;                                              \
    } while (0)
                for (uint32_t k = b; alive && k < e; ++k) {
                    const uint32_t idx = svals[k];
                    if (idx == INVALID_U32) break;
                    const particle g = load_particle(particles + (int64_t)idx * 12);
                    const hit_t h = eval_hit(cfg, &g, r.o, r.d);
                    if (!h.accept) continue;
                    const real t = hit_distance(&g, &h);
                    if (!(t > r.tmin && t < r.tmax)) continue;
                    khit_t hp = {(int)idx, t, h.galpha};
                    const int full = (num == K);
                    if (full) KB_PROCESS(kb[0]);          /* closestHit (:101-103) */
                    /* insert (:78-92): when full the closest entry is overwritten, else the count grows; bubble towards the far end */
                    if (full) kb[0].t = -1.0f; else num++;
                    for (int i = K - 1; i >= 0; --i)
                        if (hp.t > kb[i].t) { const khit_t tmp = kb[i]; kb[i] = hp; hp = tmp; }
                }
                for (int i = 0; alive && i < num; ++i) KB_PROCESS(kb[K - num + i]);   /* :337-345 */
#undef KB_PROCESS
                out_rgba[pix * 4] = cr; out_rgba[pix * 4 + 1] = cg; out_rgba[pix * 4 + 2] = cb;
                out_rgba[pix * 4 + 3] = 1.0f - T;
                out_dist[pix] = dist;
                out_hits[pix] = (real)hits;
            }
    }
}

/* ------------------------------------------------------------------------------------------ */
/* G7 processHitBwd<degree,false,false> (models/gaussianParticles.cuh:484-751)                  */

static inline real response_grad(int degree, real gray, real gres, real gresGrd) {
    switch (degree) { /* models/gaussianParticles.cuh:223-265 */
    case 8: { const real s = (real)(-0.000685871056241 * (0.5f * 8)); return s * (gray * gray) * gray * gres * gresGrd; }
    case 5: { const real s = (real)(-0.0185185185185 * (0.5f * 5)); return s * gray * R_SQRT(gray) * gres * gresGrd; }
    case 4: { const real s = (real)(-0.0555555555556 * (0.5f * 4)); return s * gray * gres * gresGrd; }
    case 3: { const real s = (real)(-0.166666666667 * (0.5f * 3)); return s * R_SQRT(gray) * gres * gresGrd; }
    case 1: { const real s = -1.5f * (0.5f * 1); return s * R_SQRT(gray) * gres * gresGrd; }
    case 0: { const real s = -0.329630334487f; return gres > 0.f ? (0.5f * s * (1.0f / R_SQRT(gray))) * gresGrd : 0.f; }
    default: return -0.5f * gres * gresGrd;
    }
}

static inline v3 safe_normalize_bw(v3 v, v3 d) { /* mathUtils.cuh:410-420 */
    const real l = v.x * v.x + v.y * v.y + v.z * v.z;
    if (l > 0.0f) {
        const real il = 1.0f / R_SQRT(l);
        const real il3 = il * il * il;
        const v3 a = scl3(d, il);
        const v3 b = V3(d.x * (v.x * v.x) + d.y * (v.y * v.x) + d.z * (v.z * v.x),
                        d.x * (v.x * v.y) + d.y * (v.y * v.y) + d.z * (v.z * v.y),
                        d.x * (v.x * v.z) + d.y * (v.y * v.z) + d.z * (v.z * v.z));
        return sub3(a, scl3(b, il3));
    }
    return V3(0.f, 0.f, 0.f);
}

static inline v3 matmul_bw_vec(const v3 m[3], v3 g) { /* mathUtils.cuh:451-456 */
    return V3(g.x * m[0].x + g.y * m[1].x + g.z * m[2].x, g.x * m[0].y + g.y * m[1].y + g.z * m[2].y,
              g.x * m[0].z + g.y * m[1].z + g.z * m[2].z);
}

static inline void matmul_bw_quat(v3 p, v3 g, real r, real x, real y, real z, real out[4]) {
    /* mathUtils.cuh:458-523 */
    const v3 d0 = scl3(p, g.x), d1 = scl3(p, g.y), d2 = scl3(p, g.z);
    real dr = 0, dx = 0, dy = 0, dz = 0;
    dy += -4 * y * d0.x; dz += -4 * z * d0.x;
    dr += 2 * z * d0.y; dx += 2 * y * d0.y; dy += 2 * x * d0.y; dz += 2 * r * d0.y;
    dr += -2 * y * d0.z; dx += 2 * z * d0.z; dy += -2 * r * d0.z; dz += 2 * x * d0.z;
    dr += -2 * z * d1.x; dx += 2 * y * d1.x; dy += 2 * x * d1.x; dz += -2 * r * d1.x;
    dx += -4 * x * d1.y; dz += -4 * z * d1.y;
    dr += 2 * x * d1.z; dx += 2 * r * d1.z; dy += 2 * z * d1.z; dz += 2 * y * d1.z;
    dr += 2 * y * d2.x; dx += 2 * z * d2.x; dy += 2 * r * d2.x; dz += 2 * x * d2.x;
    dr += -2 * x * d2.y; dx += -2 * r * d2.y; dy += 2 * z * d2.y; dz += 2 * y * d2.y;
    dx += -4 * x * d2.z; dy += -4 * y * d2.z;
    out[0] = dr; out[1] = dx; out[2] = dy; out[3] = dz;
}

/* One accepted/rejected hit of the backward replay.  Returns 1 if accepted and fills grads
 * (pos3,dns1,quat4,scl3) and rgbgrad3; advances T, C (radiance), Dp (depth). */
static int hit_backward(const gut_oracle_config* cfg, const particle* g, v3 ro, v3 rd, const real prgb[3],
                        real Tint, real* T, real Tgrad, const real Cint[3], real C[3], const real Cgrad[3],
                        real Dint, real* Dp, real Dgrad, real grad[11], real rgbgrad[3]) {
    const hit_t h = eval_hit(cfg, g, ro, rd);
    if (!h.accept) return 0;
    const v3 gscl = g->scl;
    const v3 grdd = scl3(h.grd, dot3(h.grd, scl3(h.gro, -1.f)));
    const v3 grds = mul3(gscl, grdd);
    const real gsqdist = dot3(grds, grds);
    const real gdist = R_SQRT(gsqdist);
    const real trm = *T;
    const real weight = h.galpha * trm;
    const real nextT = (1 - h.galpha) * trm;

    *Dp += weight * gdist;
    const real resHitT = R_FMAX((nextT <= cfg->min_transmittance ? 0 : (Dint - *Dp) / nextT), 0);
    const real galphaRayHitGrd = (gdist - resHitT) * trm * Dgrad;
    const v3 grdsRayHitGrd = gsqdist > 0.0f ? scl3(scl3(scl3(grds, 2 * weight), 1.0f / (2 * gdist)), Dgrad) : V3(0, 0, 0);
    const v3 gsclRayHitGrd = mul3(grdd, grdsRayHitGrd);
    const real grdScaledDot = dot3(mul3(grdsRayHitGrd, gscl), h.grd);
    const v3 grdRayHitGrd = sub3(scl3(mul3(gscl, grdsRayHitGrd), dot3(h.grd, scl3(h.gro, -1.f))), scl3(h.gro, grdScaledDot));
    const v3 groRayHitGrd = scl3(scl3(h.grd, -1.f), grdScaledDot);

    const real resTrm = h.galpha < 0.999999f ? Tint / (1 - h.galpha) : trm;
    const real galphaRayDnsGrd = resTrm * -Tgrad;

    const real gr[3] = {prgb[0], prgb[1], prgb[2]}; /* already clamped (gutKBufferRenderer.cuh:658) */
    rgbgrad[0] = Cgrad[0] * weight; rgbgrad[1] = Cgrad[1] * weight; rgbgrad[2] = Cgrad[2] * weight;
    real resC[3];
    for (int k = 0; k < 3; ++k) {
        C[k] += weight * gr[k];
        resC[k] = R_FMAX((nextT <= cfg->min_transmittance ? 0.f : (Cint[k] - C[k]) / nextT), 0.f);
    }
    const real common = galphaRayHitGrd + galphaRayDnsGrd + trm * (gr[0] - resC[0]) * Cgrad[0] +
                         trm * (gr[1] - resC[1]) * Cgrad[1] + trm * (gr[2] - resC[2]) * Cgrad[2];
    grad[3] = h.gres * common;
    const real gresGrd = g->dns * common;
    const real grayGrd = response_grad(cfg->kernel_degree, h.gray, h.gres, gresGrd);

    const v3 gcrodGrd = scl3(scl3(h.gcrod, 2.f), grayGrd);
    const v3 grdGrd = V3(gcrodGrd.z * h.gro.y - gcrodGrd.y * h.gro.z, gcrodGrd.x * h.gro.z - gcrodGrd.z * h.gro.x,
                         gcrodGrd.y * h.gro.x - gcrodGrd.x * h.gro.y);
    const v3 groGrd = V3(gcrodGrd.y * h.grd.z - gcrodGrd.z * h.grd.y, gcrodGrd.z * h.grd.x - gcrodGrd.x * h.grd.z,
                         gcrodGrd.x * h.grd.y - gcrodGrd.y * h.grd.x);

    const v3 groTot = add3(groGrd, groRayHitGrd);
    const v3 gsclGrdGro = mul3(V3(-h.gposcr.x / (gscl.x * gscl.x), -h.gposcr.y / (gscl.y * gscl.y), -h.gposcr.z / (gscl.z * gscl.z)), groTot);
    const v3 gposcrGrd = mul3(h.giscl, groTot);
    const v3 gposcGrd = matmul_bw_vec(g->rot, gposcrGrd);
    real qa[4], qb[4];
    matmul_bw_quat(h.gposc, gposcrGrd, g->qw, g->qx, g->qy, g->qz, qa);
    grad[0] = -gposcGrd.x; grad[1] = -gposcGrd.y; grad[2] = -gposcGrd.z;

    const v3 grduGrd = safe_normalize_bw(h.grdu, add3(grdGrd, grdRayHitGrd));
    const v3 t3 = mul3(V3(-h.rayDirR.x / (gscl.x * gscl.x), -h.rayDirR.y / (gscl.y * gscl.y), -h.rayDirR.z / (gscl.z * gscl.z)), grduGrd);
    const v3 sg = add3(add3(gsclRayHitGrd, gsclGrdGro), t3);
    grad[8] = sg.x; grad[9] = sg.y; grad[10] = sg.z;
    const v3 rayDirRGrd = mul3(h.giscl, grduGrd);
    matmul_bw_quat(rd, rayDirRGrd, g->qw, g->qx, g->qy, g->qz, qb);
    grad[4] = qa[0] + qb[0]; grad[5] = qa[1] + qb[1]; grad[6] = qa[2] + qb[2]; grad[7] = qa[3] + qb[3];
    *T = nextT;
    return 1;
}

/* d(rgb_c)/d(dir) for the SH polynomial of gut_oracle_sph_eval (closed form of what Slang's
 * bwd_diff(sphericalHarmonics.decode) generates; slang/common/sphericalHarmonics.slang:21-64) */
static void sh_dir_jacobian(int deg, const float* c, v3 d, real drgb_dx[3], real drgb_dy[3], real drgb_dz[3]) {
    const real x = d.x, y = d.y, z = d.z;
    for (int k = 0; k < 3; ++k) {
#define CF(i) c[(i) * 3 + k]
        real gx = 0.f, gy = 0.f, gz = 0.f;
        if (deg > 0) {
            gx += -SH_C1 * CF(3); gy += -SH_C1 * CF(1); gz += SH_C1 * CF(2);
            if (deg > 1) {
                gx += SH_C2[0] * y * CF(4) + SH_C2[2] * (-2.f * x) * CF(6) + SH_C2[3] * z * CF(7) + SH_C2[4] * (2.f * x) * CF(8);
                gy += SH_C2[0] * x * CF(4) + SH_C2[1] * z * CF(5) + SH_C2[2] * (-2.f * y) * CF(6) + SH_C2[4] * (-2.f * y) * CF(8);
                gz += SH_C2[1] * y * CF(5) + SH_C2[2] * (4.f * z) * CF(6) + SH_C2[3] * x * CF(7);
                if (deg > 2) {
                    const real xx = x * x, yy = y * y, zz = z * z;
                    gx += SH_C3[0] * (6.f * x * y) * CF(9) + SH_C3[1] * (y * z) * CF(10) + SH_C3[2] * (-2.f * x * y) * CF(11) +
                          SH_C3[3] * (-6.f * x * z) * CF(12) + SH_C3[4] * (4.f * zz - 3.f * xx - yy) * CF(13) +
                          SH_C3[5] * (2.f * x * z) * CF(14) + SH_C3[6] * (3.f * xx - 3.f * yy) * CF(15);
                    gy += SH_C3[0] * (3.f * xx - 3.f * yy) * CF(9) + SH_C3[1] * (x * z) * CF(10) +
                          SH_C3[2] * (4.f * zz - xx - 3.f * yy) * CF(11) + SH_C3[3] * (-6.f * y * z) * CF(12) +
                          SH_C3[4] * (-2.f * x * y) * CF(13) + SH_C3[5] * (-2.f * y * z) * CF(14) + SH_C3[6] * (-6.f * x * y) * CF(15);
                    gz += SH_C3[1] * (x * y) * CF(10) + SH_C3[2] * (8.f * y * z) * CF(11) +
                          SH_C3[3] * (6.f * zz - 3.f * xx - 3.f * yy) * CF(12) + SH_C3[4] * (8.f * x * z) * CF(13) +
                          SH_C3[5] * (xx - yy) * CF(14);
                }
            }
        }
#undef CF
        drgb_dx[k] = gx; drgb_dy[k] = gy; drgb_dz[k] = gz;
    }
}

static void render_backward_impl(const gut_oracle_config* cfg, const gut_oracle_camera* cam, int32_t K, int64_t n,
                                 const float* rays_o, const float* rays_d, const float* particles, const float* sph,
                                 int32_t sph_degree, const float* rgb, const uint32_t* tiles_count,
                                 const uint32_t* svals, const uint32_t* ranges, const float* out_rgba,
                                 const float* out_dist, const float* d_rgba, const float* d_dist, float* d_particles,
                                 float* d_sph) {
    float view[12], inv[12], campos[3];
    gut_oracle_sensor_matrices(cam, view, inv, campos);
    const int W = cam->width, H = cam->height;
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    int nthreads = 1;
#ifdef _OPENMP
    nthreads = omp_get_max_threads();
#endif
    const size_t stride = (size_t)n * 14; /* 11 density-record grads + 3 rgb grads */
    double* acc = (double*)calloc((size_t)nthreads * stride, sizeof(double));

#pragma omp parallel for schedule(dynamic, 1)
    for (int tile = 0; tile < gx * gy; ++tile) {
        int tid = 0;
#ifdef _OPENMP
        tid = omp_get_thread_num();
#endif
        double* a = acc + (size_t)tid * stride;
        if (tile % g_tile_stride) continue;
        const int tx = tile % gx, ty = tile / gx;
        const uint32_t b = ranges[tile * 2], e = ranges[tile * 2 + 1];
        for (int py = ty * TILE; py < imin(H, (ty + 1) * TILE); ++py)
            for (int px = tx * TILE; px < imin(W, (tx + 1) * TILE); ++px) {
                const int64_t pix = px + (int64_t)W * py;
                ray_t r = init_ray(inv, rays_o + pix * 3, rays_d + pix * 3);
                if (!r.alive) continue;
                /* initializeBackwardRay (common/rayPayloadBackward.cuh:31-73) */
                const real Cint[3] = {out_rgba[pix * 4], out_rgba[pix * 4 + 1], out_rgba[pix * 4 + 2]};
                const real Cgrad[3] = {d_rgba[pix * 4], d_rgba[pix * 4 + 1], d_rgba[pix * 4 + 2]};
                const real Tint = 1.f - out_rgba[pix * 4 + 3];
                const real Tgrad = -1.f * d_rgba[pix * 4 + 3];
                const real Dint = out_dist[pix], Dgrad = d_dist[pix];
                real T = 1.f, C[3] = {0.f, 0.f, 0.f}, Dp = 0.f;
#define BWD_PROCESS(IDX)                                                                                                          \
    do {                                                                                                                          \
        const uint32_t id_ = (IDX);                                                                                               \
        const particle g_ = load_particle(particles + (int64_t)id_ * 12);                                                         \
        const real prgb_[3] = {R_FMAX(rgb[id_ * 3], 0.f), R_FMAX(rgb[id_ * 3 + 1], 0.f), R_FMAX(rgb[id_ * 3 + 2], 0.f)};          \
        real grad_[11], rg_[3];                                                                                                   \
        if (hit_backward(cfg, &g_, r.o, r.d, prgb_, Tint, &T, Tgrad, Cint, C, Cgrad, Dint, &Dp, Dgrad, grad_, rg_)) {             \
            double* ai_ = a + (size_t)id_ * 14;                                                                                   \
            for (int q = 0; q < 11; ++q) ai_[q] += (double)grad_[q];                                                              \
            for (int q = 0; q < 3; ++q) ai_[11 + q] += (double)rg_[q];                                                            \
        }                                                                                                                         \
    } while (0)
                if (K == 0) {
                    for (uint32_t k = b; k < e; ++k) {
                        const uint32_t idx = svals[k];
                        if (idx == INVALID_U32) break;
                        BWD_PROCESS(idx);
                        if (T < cfg->min_transmittance) break;
                    }
                } else {
                    /* sorted variant: the same traversal as gut_oracle_render_forward_kbuffer, the per-hit adjoint applied in the
                     * buffer's processing order (the exact gradient of that forward; the reference gets it from Slang autodiff,
                     * gutKBufferRenderer.cuh:158-199) */
                    khit_t kb[64];
                    int num = 0, alive = 1;
                    for (int i = 0; i < K; ++i) { kb[i].idx = -1; kb[i].t = -1.0f; kb[i].alpha = 0.f; }
                    for (uint32_t k = b; alive && k < e; ++k) {
                        const uint32_t idx = svals[k];
                        if (idx == INVALID_U32) break;
                        const particle g = load_particle(particles + (int64_t)idx * 12);
                        const hit_t h = eval_hit(cfg, &g, r.o, r.d);
                        if (!h.accept) continue;
                        const real t = hit_distance(&g, &h);
                        if (!(t > r.tmin && t < r.tmax)) continue;
                        khit_t hp = {(int)idx, t, h.galpha};
                        const int full = (num == K);
                        if (full) {
                            BWD_PROCESS((uint32_t)kb[0].idx);
                            if (T < cfg->min_transmittance) alive = 0;
                        }
                        if (full) kb[0].t = -1.0f; else num++;
                        for (int i = K - 1; i >= 0; --i)
                            if (hp.t > kb[i].t) { const khit_t tmp = kb[i]; kb[i] = hp; hp = tmp; }
                    }
                    for (int i = 0; alive && i < num; ++i) {
                        BWD_PROCESS((uint32_t)kb[K - num + i].idx);
                        if (T < cfg->min_transmittance) alive = 0;
                    }
                }
#undef BWD_PROCESS
            }
    }

    /* reduce thread-private sums; then G8 projectBackward (gutProjector.cuh:390-430) */
    memset(d_particles, 0, (size_t)n * 12 * sizeof(float));
    memset(d_sph, 0, (size_t)n * 48 * sizeof(float));
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        double s[14];
        for (int q = 0; q < 14; ++q) s[q] = 0.0;
        for (int t = 0; t < nthreads; ++t)
            for (int q = 0; q < 14; ++q) s[q] += acc[(size_t)t * stride + (size_t)i * 14 + q];
        float* dp = d_particles + i * 12;
        for (int q = 0; q < 11; ++q) dp[q] = (real)s[q];
        if (tiles_count[i] == 0) continue;
        const real frg[3] = {(real)s[11], (real)s[12], (real)s[13]};
        const float* p = particles + i * 12;
        const v3 vraw = V3(p[0] - campos[0], p[1] - campos[1], p[2] - campos[2]);
        const real len = R_SQRT(dot3(vraw, vraw));
        const v3 dir = len > 0.f ? scl3(vraw, 1.0f / len) : V3(1.f, 0.f, 0.f);
        real basis[16];
        sh_basis(sph_degree, dir, basis);
        real mg[3];
        for (int k = 0; k < 3; ++k) mg[k] = (rgb[i * 3 + k] > 0.0f) ? frg[k] : 0.f; /* clamp mask of max(f+0.5,0) */
        for (int j = 0; j < 16; ++j)
            for (int k = 0; k < 3; ++k) d_sph[i * 48 + j * 3 + k] = basis[j] * mg[k];
        real jx[3], jy[3], jz[3];
        sh_dir_jacobian(sph_degree, sph + i * 48, dir, jx, jy, jz);
        const v3 ddir = V3(jx[0] * mg[0] + jx[1] * mg[1] + jx[2] * mg[2], jy[0] * mg[0] + jy[1] * mg[1] + jy[2] * mg[2],
                           jz[0] * mg[0] + jz[1] * mg[1] + jz[2] * mg[2]);
        /* normalize(pos - cam) adjoint: (ddir - dir (dir.ddir)) / len   (gaussianParticles.slang:545-558) */
        if (len > 0.f) {
            const real dd = dot3(dir, ddir);
            dp[0] += (ddir.x - dir.x * dd) / len;
            dp[1] += (ddir.y - dir.y * dd) / len;
            dp[2] += (ddir.z - dir.z * dd) / len;
        }
    }
    free(acc);
}

void gut_oracle_render_backward(const gut_oracle_config* cfg, const gut_oracle_camera* cam, int64_t n,
                                const float* rays_o, const float* rays_d, const float* particles, const float* sph,
                                int32_t sph_degree, const float* rgb, const uint32_t* tiles_count,
                                const uint32_t* svals, const uint32_t* ranges, const float* out_rgba,
                                const float* out_dist, const float* d_rgba, const float* d_dist, float* d_particles,
                                float* d_sph) {
    render_backward_impl(cfg, cam, 0, n, rays_o, rays_d, particles, sph, sph_degree, rgb, tiles_count, svals, ranges, out_rgba, out_dist,
                         d_rgba, d_dist, d_particles, d_sph);
}

void gut_oracle_render_backward_kbuffer(const gut_oracle_config* cfg, const gut_oracle_camera* cam, int32_t K, int64_t n,
                                        const float* rays_o, const float* rays_d, const float* particles, const float* sph,
                                        int32_t sph_degree, const float* rgb, const uint32_t* tiles_count,
                                        const uint32_t* svals, const uint32_t* ranges, const float* out_rgba,
                                        const float* out_dist, const float* d_rgba, const float* d_dist, float* d_particles,
                                        float* d_sph) {
    if (K < 1 || K > 64) return;
    render_backward_impl(cfg, cam, K, n, rays_o, rays_d, particles, sph, sph_degree, rgb, tiles_count, svals, ranges, out_rgba, out_dist,
                         d_rgba, d_dist, d_particles, d_sph);
}

/* single-hit backward exposed for pinning against processHitBwd compiled from the reference (oracle/ref_gut.cpp) */
int gut_oracle_hit_backward(const gut_oracle_config* cfg, const float ro[3], const float rd[3], const float p[12],
                            const float prgb[3], float Tint, float* T, float Tgrad, const float Cint[3], float C[3],
                            const float Cgrad[3], float Dint, float* D, float Dgrad, float grad[11], float rgbgrad[3]) {
    const particle g = load_particle(p);
    const real prgb_[3] = {prgb[0], prgb[1], prgb[2]}, Cint_[3] = {Cint[0], Cint[1], Cint[2]}, Cgrad_[3] = {Cgrad[0], Cgrad[1], Cgrad[2]};
    real T_ = *T, D_ = *D, C_[3] = {C[0], C[1], C[2]}, grad_[11], rg_[3] = {0, 0, 0};
    for (int q = 0; q < 11; ++q) grad_[q] = 0;
    const int acc = hit_backward(cfg, &g, V3(ro[0], ro[1], ro[2]), V3(rd[0], rd[1], rd[2]), prgb_, Tint, &T_, Tgrad, Cint_, C_, Cgrad_,
                                 Dint, &D_, Dgrad, grad_, rg_);
    *T = (float)T_; *D = (float)D_;
    for (int q = 0; q < 3; ++q) { C[q] = (float)C_[q]; rgbgrad[q] = (float)rg_[q]; }
    for (int q = 0; q < 11; ++q) grad[q] = (float)grad_[q];
    return acc;
}

/* ========================================================================================== */
/* 3DGRT (threedgrt_tracer/): brute-force restatement of the ordered ray tracer.               */
/* No BVH here: every ray tests every particle proxy, which is what "all AABB-overlapping      */
/* candidates reach the intersection program" means for OptiX (SURVEY.md section 8c).          */
/* ========================================================================================== */

#define GRT_K 16 /* PipelineParameters::MaxNumHitPerTrace (include/3dgrt/pipelineParameters.h:82) */

/* kernelScale (threedgrt_tracer/src/particlePrimitives.cu:27-51), generalized Gaussian branch */
static float grt_kernel_scale(float density, float min_response, int clamping, float degree) {
    const float modulation = clamping ? density : 1.0f;
    const float minr = fminf(min_response / modulation, 0.97f);
    const float b = degree;
    const float a = -4.5f / powf(3.0f, b);
    return powf(logf(minr) / a, 1.0f / b);
}

/* proxy of one particle: instance transform A = [R diag(kscl) | mu] (particlePrimitives.cu:543-610) */
void grt_oracle_proxies(const gut_oracle_config* cfg, int32_t clamping, int64_t n, const float* particles, float* kscl /*[N,3]*/,
                        float* scene_aabb /*[6] min xyz, max xyz*/) {
    float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int64_t i = 0; i < n; ++i) {
        const float* p = particles + i * 12;
        const float ks = grt_kernel_scale(p[3], cfg->min_kernel_density, clamping, (float)cfg->kernel_degree);
        const float k[3] = {ks * p[8], ks * p[9], ks * p[10]};
        kscl[i * 3] = k[0]; kscl[i * 3 + 1] = k[1]; kscl[i * 3 + 2] = k[2];
        /* rows of R (quaternionWXYZToMatrixTranspose, include/3dgrt/mathUtils.h) */
        const float r = p[4], x = p[5], y = p[6], z = p[7];
        const float R[3][3] = {{1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
                               {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
                               {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}};
        for (int c = 0; c < 8; ++c) {
            const float v[3] = {((c & 4) ? 1.f : -1.f) * k[0], ((c & 2) ? 1.f : -1.f) * k[1], ((c & 1) ? 1.f : -1.f) * k[2]};
            for (int a = 0; a < 3; ++a) {
                const float w = (R[a][0] * v[0] + R[a][1] * v[1] + R[a][2] * v[2]) + p[a];
                lo[a] = fminf(lo[a], w);
                hi[a] = fmaxf(hi[a], w);
            }
        }
    }
    for (int a = 0; a < 3; ++a) { scene_aabb[a] = lo[a]; scene_aabb[3 + a] = hi[a]; }
}

typedef struct { float t, t_out; uint32_t pid; } grt_cand;

static int grt_cand_cmp(const void* a, const void* b) {
    const grt_cand* x = (const grt_cand*)a; const grt_cand* y = (const grt_cand*)b;
    if (x->t < y->t) return -1;
    if (x->t > y->t) return 1;
    return (x->pid > y->pid) - (x->pid < y->pid);
}

/* Candidates of one ray on (tmin, tmax): the ray segment meets the proxy box (OptiX traversal), the custom
 * intersection accepts (intersectInstanceParticle, include/3dgrt/kernels/cuda/gaussianParticles.cuh:449-465). */
static int64_t grt_candidates(int64_t n, const float* particles, const float* kscl, const float o[3], const float d[3], float tmin,
                              float tmax, grt_cand* out) {
    int64_t m = 0;
    for (int64_t i = 0; i < n; ++i) {
        const float* p = particles + i * 12;
        const float r = p[4], x = p[5], y = p[6], z = p[7];
        /* rows of the inverse rotation = columns of R */
        const float Rt[3][3] = {{1.f - 2.f * (y * y + z * z), 2.f * (x * y + r * z), 2.f * (x * z - r * y)},
                                {2.f * (x * y - r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z + r * x)},
                                {2.f * (x * z + r * y), 2.f * (y * z - r * x), 1.f - 2.f * (x * x + y * y)}};
        const float v[3] = {o[0] - p[0], o[1] - p[1], o[2] - p[2]};
        float oi[3], di[3];
        for (int a = 0; a < 3; ++a) {
            oi[a] = (Rt[a][0] * v[0] + Rt[a][1] * v[1] + Rt[a][2] * v[2]) / kscl[i * 3 + a];
            di[a] = (Rt[a][0] * d[0] + Rt[a][1] * d[1] + Rt[a][2] * d[2]) / kscl[i * 3 + a];
        }
        /* unit-cube slab test on [tmin, tmax] */
        float tin = tmin, tout = tmax;
        for (int a = 0; a < 3; ++a) {
            const float t0 = (-1.f - oi[a]) / di[a], t1 = (1.f - oi[a]) / di[a];
            tin = fmaxf(tin, fminf(t0, t1));
            tout = fminf(tout, fmaxf(t0, t1));
        }
        if (!(tin <= tout)) continue;
        const float num = -(oi[0] * di[0] + oi[1] * di[1] + oi[2] * di[2]);
        const float den = 1.f / (di[0] * di[0] + di[1] * di[1] + di[2] * di[2]);
        const float t = num * den;
        if (!((t > tmin) && (t < tmax))) continue;
        const float l = di[0] * di[0] + di[1] * di[1] + di[2] * di[2];
        const float il = l > 0.f ? 1.0f / sqrtf(l) : 1.f;
        const float n0 = di[0] * il, n1 = di[1] * il, n2 = di[2] * il;
        const float c0 = n1 * oi[2] - n2 * oi[1], c1 = n2 * oi[0] - n0 * oi[2], c2 = n0 * oi[1] - n1 * oi[0];
        if (!((c0 * c0 + c1 * c1 + c2 * c2) * den < 9.f)) continue; /* hitMaxParticleSquaredDistance (pipelineParameters.h:69) */
        out[m].t = t; out[m].t_out = tout; out[m].pid = (uint32_t)i; m++;
    }
    qsort(out, (size_t)m, sizeof(grt_cand), grt_cand_cmp);
    return m;
}

static void grt_ray(const float* r2w /*[3,4] row major*/, const float* ro, const float* rd, float o[3], float d[3]) {
    /* rayWorldOrigin / rayWorldDirection (pipelineParameters.h:96-114) */
    for (int a = 0; a < 3; ++a) {
        o[a] = r2w[a * 4] * ro[0] + r2w[a * 4 + 1] * ro[1] + r2w[a * 4 + 2] * ro[2] + r2w[a * 4 + 3];
        d[a] = r2w[a * 4] * rd[0] + r2w[a * 4 + 1] * rd[1] + r2w[a * 4 + 2] * rd[2];
    }
}

static void grt_aabb(const float* bb, const float o[3], const float d[3], float* tmin, float* tmax) {
    /* intersectAABB (src/kernels/cuda/referenceOptix.cu:33-39) */
    float mn = -FLT_MAX, mx = FLT_MAX;
    for (int a = 0; a < 3; ++a) {
        const float t0 = (bb[a] - o[a]) / d[a], t1 = (bb[3 + a] - o[a]) / d[a];
        mn = fmaxf(mn, fminf(t0, t1));
        mx = fminf(mx, fmaxf(t0, t1));
    }
    *tmin = fmaxf(0.f, mn);
    *tmax = mx;
}

static void grt_sh_basis_f(int deg, const float d[3], float b[16]) {
    real br[16];
    sh_basis(deg, V3(d[0], d[1], d[2]), br);
    for (int k = 0; k < 16; ++k) b[k] = (float)br[k];
}

/* forward: __raygen__rg of referenceOptix.cu:103-186 */
void grt_oracle_trace(const gut_oracle_config* cfg, int32_t clamping, int64_t n, const float* particles, const float* sph,
                      int32_t sph_degree, int64_t n_rays, const float* rays_o, const float* rays_d, const float* ray_to_world,
                      float* out_rgb, float* out_alpha, float* out_dist /*[R,2]*/, float* out_hits, float* visibility) {
    float* kscl = (float*)malloc((size_t)(n > 0 ? n : 1) * 3 * sizeof(float));
    float bb[6];
    grt_oracle_proxies(cfg, clamping, n, particles, kscl, bb);
    memset(visibility, 0, (size_t)n * sizeof(float));
    const float eps = 1e-9f;
#pragma omp parallel
    {
        grt_cand* cand = (grt_cand*)malloc((size_t)(n > 0 ? n : 1) * sizeof(grt_cand));
#pragma omp for schedule(dynamic, 64)
        for (int64_t ri = 0; ri < n_rays; ++ri) {
            float o[3], d[3], t0, t1;
            grt_ray(ray_to_world, rays_o + ri * 3, rays_d + ri * 3, o, d);
            grt_aabb(bb, o, d, &t0, &t1);
            float last = fmaxf(0.0f, t0 - eps);
            real T = 1.f, C[3] = {0.f, 0.f, 0.f}, D = 0.f;
            float hits = 0.f;
            const int64_t m = (last <= t1) ? grt_candidates(n, particles, kscl, o, d, last + eps, t1 + eps, cand) : 0;
            int64_t cur = 0;
            while ((last <= t1) && (T > cfg->min_transmittance)) {
                const float tmin = last + eps;
                /* the (up to) 16 nearest candidates beyond tmin: one optixTrace of the reference */
                int64_t sel[GRT_K];
                int ns = 0;
                for (int64_t c = cur; c < m && ns < GRT_K; ++c)
                    if (cand[c].t > tmin && cand[c].t_out >= tmin) sel[ns++] = c;
                if (ns == 0) break;
                for (int s = 0; s < ns; ++s) {
                    if (!(T > cfg->min_transmittance)) continue;
                    const grt_cand h = cand[sel[s]];
                    const particle g = load_particle(particles + (int64_t)h.pid * 12);
                    const hit_t e = eval_hit(cfg, &g, V3(o[0], o[1], o[2]), V3(d[0], d[1], d[2]));
                    if (e.accept) {
                        const real w = e.galpha * T;
                        const real t = hit_distance(&g, &e);
                        float rad[3];
                        gut_oracle_sph_eval(sph_degree, sph + (int64_t)h.pid * 48, d, rad);
                        for (int k = 0; k < 3; ++k) C[k] += R_FMAX((real)rad[k], (real)0.f) * w;
                        T *= (1 - e.galpha);
                        D += t * w;
                        hits += 1.f;
#pragma omp atomic write
                        visibility[h.pid] = 1.0f;
                    }
                    last = fmaxf(last, h.t);
                }
                while (cur < m && cand[cur].t <= last) cur++;
            }
            out_rgb[ri * 3] = (float)C[0]; out_rgb[ri * 3 + 1] = (float)C[1]; out_rgb[ri * 3 + 2] = (float)C[2];
            out_alpha[ri] = (float)(1 - T);
            out_dist[ri * 2] = (float)D;
            out_dist[ri * 2 + 1] = last;
            out_hits[ri] = hits;
        }
        free(cand);
    }
    free(kscl);
}

/* backward: __raygen__rg of referenceBwdOptix.cu:103-170 */
void grt_oracle_trace_bwd(const gut_oracle_config* cfg, int32_t clamping, int64_t n, const float* particles, const float* sph,
                          int32_t sph_degree, int64_t n_rays, const float* rays_o, const float* rays_d, const float* ray_to_world,
                          const float* out_rgb, const float* out_alpha, const float* out_dist, const float* d_rgb,
                          const float* d_alpha, const float* d_dist, float* d_particles, float* d_sph) {
    float* kscl = (float*)malloc((size_t)(n > 0 ? n : 1) * 3 * sizeof(float));
    float bb[6];
    grt_oracle_proxies(cfg, clamping, n, particles, kscl, bb);
    const float eps = 1e-9f;
    int nthreads = 1;
#ifdef _OPENMP
    nthreads = omp_get_max_threads();
#endif
    const size_t stride = (size_t)n * 59; /* 11 density-record grads + 48 SH grads */
    double* acc = (double*)calloc((size_t)nthreads * (stride ? stride : 1), sizeof(double));
#pragma omp parallel
    {
        int tid = 0;
#ifdef _OPENMP
        tid = omp_get_thread_num();
#endif
        double* a = acc + (size_t)tid * stride;
        grt_cand* cand = (grt_cand*)malloc((size_t)(n > 0 ? n : 1) * sizeof(grt_cand));
#pragma omp for schedule(dynamic, 64)
        for (int64_t ri = 0; ri < n_rays; ++ri) {
            float o[3], d[3], t0, t1;
            grt_ray(ray_to_world, rays_o + ri * 3, rays_d + ri * 3, o, d);
            grt_aabb(bb, o, d, &t0, &t1);
            float start = fmaxf(0.0f, t0 - eps);
            const float end = fminf(out_dist[ri * 2 + 1], t1) + eps;
            const real Cint[3] = {out_rgb[ri * 3], out_rgb[ri * 3 + 1], out_rgb[ri * 3 + 2]};
            const real Cgrad[3] = {d_rgb[ri * 3], d_rgb[ri * 3 + 1], d_rgb[ri * 3 + 2]};
            const real Tint = 1.0f - out_alpha[ri], Tgrad = -1.0f * d_alpha[ri];
            const real Dint = out_dist[ri * 2], Dgrad = d_dist[ri];
            real T = 1.f, C[3] = {0.f, 0.f, 0.f}, Dp = 0.f;
            const int64_t m = (start < end) ? grt_candidates(n, particles, kscl, o, d, start + eps, end, cand) : 0;
            int64_t cur = 0;
            float basis[16];
            grt_sh_basis_f(sph_degree, d, basis);
            while (start < end) {
                const float tmin = start + eps;
                int64_t sel[GRT_K];
                int ns = 0;
                for (int64_t c = cur; c < m && ns < GRT_K; ++c)
                    if (cand[c].t > tmin && cand[c].t_out >= tmin) sel[ns++] = c;
                if (ns == 0) break;
                for (int s = 0; s < ns; ++s) {
                    const grt_cand h = cand[sel[s]];
                    const particle g = load_particle(particles + (int64_t)h.pid * 12);
                    float rad[3];
                    gut_oracle_sph_eval(sph_degree, sph + (int64_t)h.pid * 48, d, rad);
                    const real prgb[3] = {R_FMAX((real)rad[0], (real)0.f), R_FMAX((real)rad[1], (real)0.f), R_FMAX((real)rad[2], (real)0.f)};
                    real grad[11], rg[3];
                    if (hit_backward(cfg, &g, V3(o[0], o[1], o[2]), V3(d[0], d[1], d[2]), prgb, Tint, &T, Tgrad, Cint, C, Cgrad, Dint, &Dp, Dgrad, grad, rg)) {
                        double* ai = a + (size_t)h.pid * 59;
                        for (int q = 0; q < 11; ++q) ai[q] += (double)grad[q];
                        /* radianceFromSpHBwd<true> (gaussianParticles.cuh:101-177): coefficient grads, clamp mask on the unclamped radiance */
                        for (int j = 0; j < 16; ++j)
                            for (int k = 0; k < 3; ++k)
                                if (rad[k] > 0.0f) ai[11 + j * 3 + k] += (double)((real)basis[j] * rg[k]);
                    }
                    start = fmaxf(start, h.t);
                }
                while (cur < m && cand[cur].t <= start) cur++;
            }
        }
        free(cand);
    }
    for (int64_t i = 0; i < n; ++i) {
        double s[59];
        for (int q = 0; q < 59; ++q) s[q] = 0.0;
        for (int t = 0; t < nthreads; ++t)
            for (int q = 0; q < 59; ++q) s[q] += acc[(size_t)t * stride + (size_t)i * 59 + q];
        for (int q = 0; q < 11; ++q) d_particles[i * 12 + q] = (float)s[q];
        d_particles[i * 12 + 11] = 0.f;
        for (int q = 0; q < 48; ++q) d_sph[i * 48 + q] = (float)s[11 + q];
    }
    free(acc);
    free(kscl);
}
