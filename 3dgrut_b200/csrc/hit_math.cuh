// 3dgrut_b200/csrc/hit_math.cuh -- per-(ray, particle) response, compositing weight and hand-derived adjoint shared
// by the ray-traced path (grt.cu).  Same mathematics as the inline versions in gut_render.cu; restated from
// threedgrt_tracer/include/3dgrt/kernels/cuda/gaussianParticles.cuh:336-405 (processHit) and :467-733 (processHitBwd).
#pragma once
#include <cuda_runtime.h>

namespace gutb200 {

struct ParticleFrame {
    float r0x, r0y, r0z, r1x, r1y, r1z, r2x, r2y, r2z;  // rows of quaternionWXYZToMatrix = columns of R
    float px, py, pz;                                    // position
    float sx, sy, sz, isx, isy, isz;                     // scale and its reciprocal
    float qr, qx, qy, qz;                                // quaternion (w,x,y,z)
    float dns;
};

__device__ __forceinline__ ParticleFrame load_frame(const float* __restrict__ particles, uint32_t pid) {
    const float4* p4 = reinterpret_cast<const float4*>(particles) + static_cast<size_t>(pid) * 3;
    const float4 a = __ldg(p4), q = __ldg(p4 + 1), s = __ldg(p4 + 2);
    ParticleFrame f;
    const float r = q.x, x = q.y, y = q.z, z = q.w;
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, xz = x * z, yz = y * z;
    const float rx = r * x, ry = r * y, rz = r * z;
    f.r0x = 1.f - 2.f * (yy + zz); f.r0y = 2.f * (xy + rz); f.r0z = 2.f * (xz - ry);
    f.r1x = 2.f * (xy - rz); f.r1y = 1.f - 2.f * (xx + zz); f.r1z = 2.f * (yz + rx);
    f.r2x = 2.f * (xz + ry); f.r2y = 2.f * (yz - rx); f.r2z = 1.f - 2.f * (xx + yy);
    f.px = a.x; f.py = a.y; f.pz = a.z; f.dns = a.w;
    f.sx = s.x; f.sy = s.y; f.sz = s.z;
    f.isx = 1.0f / s.x; f.isy = 1.0f / s.y; f.isz = 1.0f / s.z;
    f.qr = r; f.qx = x; f.qy = y; f.qz = z;
    return f;
}

struct CanonicalHit {
    float pcx, pcy, pcz;      // gposc = o - mu
    float gox, goy, goz;      // gro
    float ux, uy, uz;         // grdu
    float l, il;              // |grdu|^2 and its rsqrt
    float gdx, gdy, gdz;      // grd
    float ccx, ccy, ccz;      // gcrod
    float gray, gres, alpha;
    bool accept;
};

template <int DEG>
__device__ __forceinline__ float response(float gray) {
    if (DEG == 4) return __expf(-0.0555555555556f * gray * gray);
    return __expf(-0.5f * gray);
}

template <int DEG>
__device__ __forceinline__ float response_grad(float gray, float gres, float gres_grad) {
    if (DEG == 4) return (-0.0555555555556f * 2.0f) * gray * gres * gres_grad;
    return -0.5f * gres * gres_grad;
}

template <int DEG>
__device__ __forceinline__ CanonicalHit canonical_hit(const ParticleFrame& f, float ox, float oy, float oz, float dx, float dy, float dz,
                                                      float min_response, float min_alpha, float max_alpha) {
    CanonicalHit h;
    h.pcx = ox - f.px; h.pcy = oy - f.py; h.pcz = oz - f.pz;
    h.gox = f.isx * (f.r0x * h.pcx + f.r0y * h.pcy + f.r0z * h.pcz);
    h.goy = f.isy * (f.r1x * h.pcx + f.r1y * h.pcy + f.r1z * h.pcz);
    h.goz = f.isz * (f.r2x * h.pcx + f.r2y * h.pcy + f.r2z * h.pcz);
    h.ux = f.isx * (f.r0x * dx + f.r0y * dy + f.r0z * dz);
    h.uy = f.isy * (f.r1x * dx + f.r1y * dy + f.r1z * dz);
    h.uz = f.isz * (f.r2x * dx + f.r2y * dy + f.r2z * dz);
    h.l = h.ux * h.ux + h.uy * h.uy + h.uz * h.uz;
    h.il = h.l > 0.f ? rsqrtf(h.l) : 1.f;
    h.gdx = h.ux * h.il; h.gdy = h.uy * h.il; h.gdz = h.uz * h.il;
    h.ccx = h.gdy * h.goz - h.gdz * h.goy;
    h.ccy = h.gdz * h.gox - h.gdx * h.goz;
    h.ccz = h.gdx * h.goy - h.gdy * h.gox;
    h.gray = h.ccx * h.ccx + h.ccy * h.ccy + h.ccz * h.ccz;
    h.gres = response<DEG>(h.gray);
    h.alpha = fminf(max_alpha, h.gres * f.dns);
    h.accept = (h.gres > min_response) && (h.alpha > min_alpha);
    return h;
}

__device__ __forceinline__ float hit_distance(const ParticleFrame& f, const CanonicalHit& h) {
    const float pd = -(h.gdx * h.gox + h.gdy * h.goy + h.gdz * h.goz);
    const float hx = f.sx * h.gdx * pd, hy = f.sy * h.gdy * pd, hz = f.sz * h.gdz * pd;
    return sqrtf(hx * hx + hy * hy + hz * hz);
}

// Adjoint of one accepted hit.  In/out: T (transmittance before -> after), C (radiance accumulated through this hit),
// D (distance accumulated through this hit).  g[0..10] = d(pos3, density, quat4, scale3); rg = d(radiance of the particle).
template <int DEG>
__device__ __forceinline__ void hit_adjoint(const ParticleFrame& f, const CanonicalHit& h, float dx, float dy, float dz, float cr,
                                            float cg, float cb, float min_transmittance, float Tint, float Tgrad, float Cix,
                                            float Ciy, float Ciz, float Cgx, float Cgy, float Cgz, float Dint, float Dgrad, float& T,
                                            float& Cx, float& Cy, float& Cz, float& D, float g[11], float rg[3]) {
    const float pd = -(h.gdx * h.gox + h.gdy * h.goy + h.gdz * h.goz);
    const float ddx = h.gdx * pd, ddy = h.gdy * pd, ddz = h.gdz * pd;
    const float hx = f.sx * ddx, hy = f.sy * ddy, hz = f.sz * ddz;
    const float gsq = hx * hx + hy * hy + hz * hz;
    const float gdist = sqrtf(gsq);
    const float weight = h.alpha * T;
    const float nextT = (1.f - h.alpha) * T;
    const float inv_next = nextT <= min_transmittance ? 0.f : 1.0f / nextT;
    D += weight * gdist;
    const float resD = fmaxf((Dint - D) * inv_next, 0.f);
    const float a_hit = (gdist - resD) * T * Dgrad;
    const float hs = gsq > 0.f ? (weight / gdist) * Dgrad : 0.f;
    const float hgx = hx * hs, hgy = hy * hs, hgz = hz * hs;
    const float sd = hgx * f.sx * h.gdx + hgy * f.sy * h.gdy + hgz * f.sz * h.gdz;
    const float resT = h.alpha < 0.999999f ? Tint / (1.f - h.alpha) : T;
    const float a_dns = resT * -Tgrad;
    rg[0] = Cgx * weight; rg[1] = Cgy * weight; rg[2] = Cgz * weight;
    Cx += weight * cr; Cy += weight * cg; Cz += weight * cb;
    const float rcx = fmaxf((Cix - Cx) * inv_next, 0.f);
    const float rcy = fmaxf((Ciy - Cy) * inv_next, 0.f);
    const float rcz = fmaxf((Ciz - Cz) * inv_next, 0.f);
    const float common = a_hit + a_dns + T * (cr - rcx) * Cgx + T * (cg - rcy) * Cgy + T * (cb - rcz) * Cgz;
    g[3] = h.gres * common;
    const float gray_g = response_grad<DEG>(h.gray, h.gres, f.dns * common);
    const float kx = 2.f * h.ccx * gray_g, ky = 2.f * h.ccy * gray_g, kz = 2.f * h.ccz * gray_g;
    const float gd_gx = kz * h.goy - ky * h.goz + (f.sx * hgx * pd - h.gox * sd);
    const float gd_gy = kx * h.goz - kz * h.gox + (f.sy * hgy * pd - h.goy * sd);
    const float gd_gz = ky * h.gox - kx * h.goy + (f.sz * hgz * pd - h.goz * sd);
    const float go_gx = ky * h.gdz - kz * h.gdy - h.gdx * sd;
    const float go_gy = kz * h.gdx - kx * h.gdz - h.gdy * sd;
    const float go_gz = kx * h.gdy - ky * h.gdx - h.gdz * sd;
    const float prg_x = f.isx * go_gx, prg_y = f.isy * go_gy, prg_z = f.isz * go_gz;
    float sgx = ddx * hgx - h.gox * prg_x;
    float sgy = ddy * hgy - h.goy * prg_y;
    float sgz = ddz * hgz - h.goz * prg_z;
    g[0] = -(prg_x * f.r0x + prg_y * f.r1x + prg_z * f.r2x);
    g[1] = -(prg_x * f.r0y + prg_y * f.r1y + prg_z * f.r2y);
    g[2] = -(prg_x * f.r0z + prg_y * f.r1z + prg_z * f.r2z);
    const float il3 = h.il * h.il * h.il;
    const float du = gd_gx * h.ux + gd_gy * h.uy + gd_gz * h.uz;
    const float ug_x = h.l > 0.f ? h.il * gd_gx - il3 * h.ux * du : 0.f;
    const float ug_y = h.l > 0.f ? h.il * gd_gy - il3 * h.uy * du : 0.f;
    const float ug_z = h.l > 0.f ? h.il * gd_gz - il3 * h.uz * du : 0.f;
    const float rdg_x = f.isx * ug_x, rdg_y = f.isy * ug_y, rdg_z = f.isz * ug_z;
    sgx -= h.ux * rdg_x;
    sgy -= h.uy * rdg_y;
    sgz -= h.uz * rdg_z;
    g[8] = sgx; g[9] = sgy; g[10] = sgz;
    const float m00 = prg_x * h.pcx + rdg_x * dx, m01 = prg_x * h.pcy + rdg_x * dy, m02 = prg_x * h.pcz + rdg_x * dz;
    const float m10 = prg_y * h.pcx + rdg_y * dx, m11 = prg_y * h.pcy + rdg_y * dy, m12 = prg_y * h.pcz + rdg_y * dz;
    const float m20 = prg_z * h.pcx + rdg_z * dx, m21 = prg_z * h.pcy + rdg_z * dy, m22 = prg_z * h.pcz + rdg_z * dz;
    g[4] = 2.f * (f.qz * (m01 - m10) + f.qy * (m20 - m02) + f.qx * (m12 - m21));
    g[5] = 2.f * (f.qy * (m01 + m10) + f.qz * (m02 + m20) + f.qr * (m12 - m21)) - 4.f * f.qx * (m11 + m22);
    g[6] = 2.f * (f.qx * (m01 + m10) + f.qr * (m20 - m02) + f.qz * (m12 + m21)) - 4.f * f.qy * (m00 + m22);
    g[7] = 2.f * (f.qr * (m01 - m10) + f.qx * (m02 + m20) + f.qy * (m12 + m21)) - 4.f * f.qz * (m00 + m11);
    T = nextT;
}

// Adjoint of one accepted hit in the form of the reference's Slang pipelines (gaussianParticles.slang hit() / processHitFromBuffer
// under bwd_diff), used for NHT features.  Differences from hit_adjoint:
//   * alpha = min(max_alpha, response density) is differentiated: a clamped hit passes no gradient through response or density;
//   * the radiance residual is replaced by the features': fg = sum_c f_c g_c of this hit, FiG = sum_c F_out,c g_c of the ray and the
//     running FG = sum_c F_acc,c g_c (in/out), so res = (FiG - FG) / T_next is peeled without a clamp;
//   * pg = dL/dP of the canonical hit point P = gro + grd pd (the features depend on it) flows into gro and grd:
//     groGrd += pg - grd s, grdGrd += pd pg - s gro with s = grd . pg; the normalize adjoint below is the general one.
// g[0..10] = d(pos3, density, quat4, scale3).
template <int DEG>
__device__ __forceinline__ void hit_adjoint_nht(const ParticleFrame& f, const CanonicalHit& h, float dx, float dy, float dz, float fg, float pgx,
                                                float pgy, float pgz, float min_transmittance, float Tint, float Tgrad, float FiG, float Dint,
                                                float Dgrad, float& T, float& FG, float& D, float g[11]) {
    const float pd = -(h.gdx * h.gox + h.gdy * h.goy + h.gdz * h.goz);
    const float ddx = h.gdx * pd, ddy = h.gdy * pd, ddz = h.gdz * pd;
    const float hx = f.sx * ddx, hy = f.sy * ddy, hz = f.sz * ddz;
    const float gsq = hx * hx + hy * hy + hz * hz;
    const float gdist = sqrtf(gsq);
    const float weight = h.alpha * T;
    const float nextT = (1.f - h.alpha) * T;
    const float inv_next = nextT <= min_transmittance ? 0.f : 1.0f / nextT;
    D += weight * gdist;
    const float resD = fmaxf((Dint - D) * inv_next, 0.f);
    const float a_hit = (gdist - resD) * T * Dgrad;
    const float hs = gsq > 0.f ? (weight / gdist) * Dgrad : 0.f;
    const float hgx = hx * hs, hgy = hy * hs, hgz = hz * hs;
    const float sd = hgx * f.sx * h.gdx + hgy * f.sy * h.gdy + hgz * f.sz * h.gdz;
    const float resT = h.alpha < 0.999999f ? Tint / (1.f - h.alpha) : T;
    const float a_dns = resT * -Tgrad;
    FG += weight * fg;
    const float res_g = (FiG - FG) * inv_next;
    float common = a_hit + a_dns + T * (fg - res_g);
    if (h.gres * f.dns > h.alpha) common = 0.f;  // clamped at max_alpha: d min(max_alpha, x) / dx = 0
    g[3] = h.gres * common;
    const float gray_g = response_grad<DEG>(h.gray, h.gres, f.dns * common);
    const float kx = 2.f * h.ccx * gray_g, ky = 2.f * h.ccy * gray_g, kz = 2.f * h.ccz * gray_g;
    const float ps = h.gdx * pgx + h.gdy * pgy + h.gdz * pgz;
    const float gd_gx = kz * h.goy - ky * h.goz + (f.sx * hgx * pd - h.gox * sd) + (pd * pgx - ps * h.gox);
    const float gd_gy = kx * h.goz - kz * h.gox + (f.sy * hgy * pd - h.goy * sd) + (pd * pgy - ps * h.goy);
    const float gd_gz = ky * h.gox - kx * h.goy + (f.sz * hgz * pd - h.goz * sd) + (pd * pgz - ps * h.goz);
    const float go_gx = ky * h.gdz - kz * h.gdy - h.gdx * sd + (pgx - h.gdx * ps);
    const float go_gy = kz * h.gdx - kx * h.gdz - h.gdy * sd + (pgy - h.gdy * ps);
    const float go_gz = kx * h.gdy - ky * h.gdx - h.gdz * sd + (pgz - h.gdz * ps);
    const float prg_x = f.isx * go_gx, prg_y = f.isy * go_gy, prg_z = f.isz * go_gz;
    float sgx = ddx * hgx - h.gox * prg_x;
    float sgy = ddy * hgy - h.goy * prg_y;
    float sgz = ddz * hgz - h.goz * prg_z;
    g[0] = -(prg_x * f.r0x + prg_y * f.r1x + prg_z * f.r2x);
    g[1] = -(prg_x * f.r0y + prg_y * f.r1y + prg_z * f.r2y);
    g[2] = -(prg_x * f.r0z + prg_y * f.r1z + prg_z * f.r2z);
    const float il3 = h.il * h.il * h.il;
    const float du = gd_gx * h.ux + gd_gy * h.uy + gd_gz * h.uz;
    const float ug_x = h.l > 0.f ? h.il * gd_gx - il3 * h.ux * du : 0.f;
    const float ug_y = h.l > 0.f ? h.il * gd_gy - il3 * h.uy * du : 0.f;
    const float ug_z = h.l > 0.f ? h.il * gd_gz - il3 * h.uz * du : 0.f;
    const float rdg_x = f.isx * ug_x, rdg_y = f.isy * ug_y, rdg_z = f.isz * ug_z;
    sgx -= h.ux * rdg_x;
    sgy -= h.uy * rdg_y;
    sgz -= h.uz * rdg_z;
    g[8] = sgx; g[9] = sgy; g[10] = sgz;
    const float m00 = prg_x * h.pcx + rdg_x * dx, m01 = prg_x * h.pcy + rdg_x * dy, m02 = prg_x * h.pcz + rdg_x * dz;
    const float m10 = prg_y * h.pcx + rdg_y * dx, m11 = prg_y * h.pcy + rdg_y * dy, m12 = prg_y * h.pcz + rdg_y * dz;
    const float m20 = prg_z * h.pcx + rdg_z * dx, m21 = prg_z * h.pcy + rdg_z * dy, m22 = prg_z * h.pcz + rdg_z * dz;
    g[4] = 2.f * (f.qz * (m01 - m10) + f.qy * (m20 - m02) + f.qx * (m12 - m21));
    g[5] = 2.f * (f.qy * (m01 + m10) + f.qz * (m02 + m20) + f.qr * (m12 - m21)) - 4.f * f.qx * (m11 + m22);
    g[6] = 2.f * (f.qx * (m01 + m10) + f.qr * (m20 - m02) + f.qz * (m12 + m21)) - 4.f * f.qy * (m00 + m22);
    g[7] = 2.f * (f.qr * (m01 - m10) + f.qx * (m02 + m20) + f.qy * (m12 + m21)) - 4.f * f.qz * (m00 + m11);
    T = nextT;
}

// 16 real SH basis values of a direction (radianceFromSpH, gaussianParticles.cuh:61-93)
__device__ __forceinline__ void sh_basis16(int deg, float x, float y, float z, float b[16]) {
#pragma unroll
    for (int k = 0; k < 16; ++k) b[k] = 0.f;
    b[0] = 0.28209479177387814f;
    if (deg > 0) {
        const float c1 = 0.4886025119029199f;
        b[1] = -c1 * y; b[2] = c1 * z; b[3] = -c1 * x;
        if (deg > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            b[4] = 1.0925484305920792f * xy; b[5] = -1.0925484305920792f * yz; b[6] = 0.31539156525252005f * (2.0f * zz - xx - yy);
            b[7] = -1.0925484305920792f * xz; b[8] = 0.5462742152960396f * (xx - yy);
            if (deg > 2) {
                b[9] = -0.5900435899266435f * y * (3.0f * xx - yy);
                b[10] = 2.890611442640554f * xy * z;
                b[11] = -0.4570457994644658f * y * (4.0f * zz - xx - yy);
                b[12] = 0.3731763325901154f * z * (2.0f * zz - 3.0f * xx - 3.0f * yy);
                b[13] = -0.4570457994644658f * x * (4.0f * zz - xx - yy);
                b[14] = 1.445305721320277f * z * (xx - yy);
                b[15] = -0.5900435899266435f * x * (xx - 3.0f * yy);
            }
        }
    }
}

}  // namespace gutb200
