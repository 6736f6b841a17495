/*
 * tests/host_emul/grt_icosahedron_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * The brute-force 3DGRT oracle (oracle/gut_oracle.c, compiled into this unit unchanged) extended to the reference's
 * `primitive_type: icosahedron` proxies.  Restated literally from the reference, NOT through the slab shortcut the GPU
 * uses, so that GPU-vs-oracle agreement also checks that the shortcut equals the reference's triangles:
 *  - 12 world-space vertices per particle, vrt = (V_i * kscl) * rot + pos with kscl = kernelScale * scale * icosaVrtScale
 *    (threedgrt_tracer/src/particlePrimitives.cu:435-494), and the 20 faces of that file;
 *  - optixTrace with OPTIX_RAY_FLAG_CULL_BACK_FACING_TRIANGLES (src/kernels/cuda/referenceOptix.cu:62): a face counts when
 *    its vertices appear counter-clockwise from the ray origin (OptiX's front face), t in (tmin, tmax);
 *  - the any-hit program keys a particle (primitiveIndex / 20) by that t (referenceOptix.cu:40-42,221-248); there is no
 *    intersection program, so intersectInstanceParticle's closest-approach test does not apply.  A particle's key is its
 *    smallest front-face t: a ray exactly through an edge may be reported twice by OptiX (measure zero), once here;
 *  - the scene box is the box of all vertices and clips every ray (referenceOptix.cu:33-39,122).
 * Hit processing (processHit / processHitBwd, the ordered integration and the re-trace of the backward) is the oracle's.
 * Triangles are intersected in `real` precision (double with -DORACLE_F64).
 */
#include "../../oracle/gut_oracle.c"

#define ICO_NV 12
#define ICO_NT 20

static const float ico_phi = 1.618033988749895f;                   /* goldenRatio   (particlePrimitives.cu:444) */
static const float ico_vrt_scale = (float)(0.5 * 1.323169076499215f); /* icosaVrtScale (:445-446) */

static void ico_table(float v[ICO_NV][3]) { /* icosaHedronVrt (:468-472) */
    const float p = ico_phi;
    const float t[ICO_NV][3] = {{-1, p, 0}, {1, p, 0}, {0, 1, -p}, {-p, 0, -1}, {-p, 0, 1}, {0, 1, p},
                                {p, 0, 1},  {0, -1, p}, {-1, -p, 0}, {0, -1, -p}, {p, 0, -1}, {1, -p, 0}};
    memcpy(v, t, sizeof(t));
}
static const int ico_tri[ICO_NT][3] = { /* icosaHedronTri (:481-486) */
    {0, 1, 2}, {0, 2, 3}, {0, 3, 4}, {0, 4, 5}, {0, 5, 1}, {6, 1, 5}, {6, 5, 7}, {6, 7, 11}, {6, 11, 10}, {6, 10, 1},
    {8, 4, 3}, {8, 3, 9}, {8, 9, 11}, {8, 11, 7}, {8, 7, 4}, {9, 3, 2}, {9, 2, 10}, {9, 10, 11}, {5, 4, 7}, {1, 10, 2}};

/* table geometry for the tests: vertices [12,3] (unscaled) and faces [20,3] */
void grt_ico_oracle_table(float* vrt, int32_t* tri) {
    float v[ICO_NV][3];
    ico_table(v);
    memcpy(vrt, v, sizeof(v));
    for (int f = 0; f < ICO_NT; ++f)
        for (int k = 0; k < 3; ++k) tri[f * 3 + k] = ico_tri[f][k];
}

/* world-space vertices [N,12,3] (computeGaussianEnclosingIcosaHedronKernel) and the scene box of all of them */
void grt_ico_oracle_proxies(const gut_oracle_config* cfg, int32_t clamping, int64_t n, const float* particles, float* vrt,
                            float* scene_aabb /*[6] min xyz, max xyz*/) {
    float V[ICO_NV][3];
    ico_table(V);
    float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int64_t i = 0; i < n; ++i) {
        const float* p = particles + i * 12;
        const float ks = grt_kernel_scale(p[3], cfg->min_kernel_density, clamping, (float)cfg->kernel_degree);
        const float k[3] = {ks * p[8] * ico_vrt_scale, ks * p[9] * ico_vrt_scale, ks * p[10] * ico_vrt_scale};
        /* rows of R (quaternionWXYZToMatrixTranspose, as grt_oracle_proxies) */
        const float r = p[4], x = p[5], y = p[6], z = p[7];
        const float R[3][3] = {{1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
                               {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
                               {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}};
        for (int c = 0; c < ICO_NV; ++c) {
            const float v[3] = {V[c][0] * k[0], V[c][1] * k[1], V[c][2] * k[2]};
            for (int a = 0; a < 3; ++a) {
                const float w = (R[a][0] * v[0] + R[a][1] * v[1] + R[a][2] * v[2]) + p[a];
                vrt[(i * ICO_NV + c) * 3 + a] = w;
                lo[a] = fminf(lo[a], w);
                hi[a] = fmaxf(hi[a], w);
            }
        }
    }
    for (int a = 0; a < 3; ++a) { scene_aabb[a] = lo[a]; scene_aabb[3 + a] = hi[a]; }
}

/* front-face-only ray / triangle test (Moeller-Trumbore); det > 0 <=> counter-clockwise seen from the ray origin */
static int ico_front_hit(v3 o, v3 d, const float* a, const float* b, const float* c, real* t) {
    const v3 va = V3(a[0], a[1], a[2]);
    const v3 e1 = sub3(V3(b[0], b[1], b[2]), va), e2 = sub3(V3(c[0], c[1], c[2]), va);
    const v3 pv = cross3(d, e2);
    const real det = dot3(e1, pv);
    if (!(det > 0)) return 0; /* back-facing (culled) or parallel */
    const v3 tv = sub3(o, va);
    const real u = dot3(tv, pv) / det;
    if (u < 0 || u > 1) return 0;
    const v3 qv = cross3(tv, e1);
    const real w = dot3(d, qv) / det;
    if (w < 0 || u + w > 1) return 0;
    *t = dot3(e2, qv) / det;
    return 1;
}

/* candidates of one ray on (tmin, tmax), sorted by their front-face t (t_out = t: nothing else bounds a triangle hit) */
static int64_t ico_candidates(int64_t n, const float* vrt, const float* sphere /*[N,4] centre, radius*/, const float o[3],
                              const float d[3], float tmin, float tmax, grt_cand* out) {
    const v3 ro = V3(o[0], o[1], o[2]), rd = V3(d[0], d[1], d[2]);
    const real dd = dot3(rd, rd);
    int64_t m = 0;
    for (int64_t i = 0; i < n; ++i) {
        /* conservative bounding-sphere reject (speed only: a ray that misses the sphere meets no face) */
        const v3 co = sub3(ro, V3(sphere[i * 4], sphere[i * 4 + 1], sphere[i * 4 + 2]));
        const v3 cr = cross3(co, rd);
        const real rr = (real)sphere[i * 4 + 3] * (real)1.001 + (real)1e-6;
        if (dot3(cr, cr) > rr * rr * dd) continue;
        const float* v = vrt + i * ICO_NV * 3;
        real best = 0;
        int found = 0;
        for (int f = 0; f < ICO_NT; ++f) {
            real t;
            if (!ico_front_hit(ro, rd, v + ico_tri[f][0] * 3, v + ico_tri[f][1] * 3, v + ico_tri[f][2] * 3, &t)) continue;
            if (!((t > tmin) && (t < tmax))) continue;
            if (!found || t < best) best = t;
            found = 1;
        }
        if (!found) continue;
        out[m].t = (float)best; out[m].t_out = (float)best; out[m].pid = (uint32_t)i; m++;
    }
    qsort(out, (size_t)m, sizeof(grt_cand), grt_cand_cmp);
    return m;
}

/* candidate keys of world-space rays [R] x particles [N]: the smallest front-face t on (tmin, +inf), +inf where there is none */
void grt_ico_oracle_entry(const gut_oracle_config* cfg, int32_t clamping, int64_t n, const float* particles, int64_t n_rays,
                          const float* rays_o, const float* rays_d, float tmin, float* t_out /*[R,N]*/) {
    float* vrt = (float*)malloc((size_t)(n > 0 ? n : 1) * ICO_NV * 3 * sizeof(float));
    float bb[6];
    grt_ico_oracle_proxies(cfg, clamping, n, particles, vrt, bb);
#pragma omp parallel for schedule(dynamic, 16)
    for (int64_t ri = 0; ri < n_rays; ++ri) {
        const v3 o = V3(rays_o[ri * 3], rays_o[ri * 3 + 1], rays_o[ri * 3 + 2]), d = V3(rays_d[ri * 3], rays_d[ri * 3 + 1], rays_d[ri * 3 + 2]);
        for (int64_t i = 0; i < n; ++i) {
            const float* v = vrt + i * ICO_NV * 3;
            real best = 0;
            int found = 0;
            for (int f = 0; f < ICO_NT; ++f) {
                real t;
                if (!ico_front_hit(o, d, v + ico_tri[f][0] * 3, v + ico_tri[f][1] * 3, v + ico_tri[f][2] * 3, &t) || !(t > tmin)) continue;
                if (!found || t < best) best = t;
                found = 1;
            }
            t_out[ri * n + i] = found ? (float)best : INFINITY;
        }
    }
    free(vrt);
}

static void ico_setup(const gut_oracle_config* cfg, int32_t clamping, int64_t n, const float* particles, float** vrt, float** sphere,
                      float bb[6]) {
    *vrt = (float*)malloc((size_t)(n > 0 ? n : 1) * ICO_NV * 3 * sizeof(float));
    *sphere = (float*)malloc((size_t)(n > 0 ? n : 1) * 4 * sizeof(float));
    grt_ico_oracle_proxies(cfg, clamping, n, particles, *vrt, bb);
    for (int64_t i = 0; i < n; ++i) {
        const float* p = particles + i * 12;
        double r2 = 0.0;
        for (int c = 0; c < ICO_NV; ++c) {
            double s = 0.0;
            for (int a = 0; a < 3; ++a) {
                const double e = (double)(*vrt)[(i * ICO_NV + c) * 3 + a] - p[a];
                s += e * e;
            }
            r2 = s > r2 ? s : r2;
        }
        (*sphere)[i * 4] = p[0]; (*sphere)[i * 4 + 1] = p[1]; (*sphere)[i * 4 + 2] = p[2];
        (*sphere)[i * 4 + 3] = (float)sqrt(r2);
    }
}

/* forward: __raygen__rg of referenceOptix.cu:103-186 with icosahedron candidates (same loop as grt_oracle_trace) */
void grt_ico_oracle_trace(const gut_oracle_config* cfg, int32_t clamping, int64_t n, const float* particles, const float* sph,
                          int32_t sph_degree, int64_t n_rays, const float* rays_o, const float* rays_d, const float* ray_to_world,
                          float* out_rgb, float* out_alpha, float* out_dist /*[R,2]*/, float* out_hits, float* visibility) {
    float *vrt, *sphere, bb[6];
    ico_setup(cfg, clamping, n, particles, &vrt, &sphere, bb);
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
            const int64_t m = (last <= t1) ? ico_candidates(n, vrt, sphere, o, d, last + eps, t1 + eps, cand) : 0;
            int64_t cur = 0;
            while ((last <= t1) && (T > cfg->min_transmittance)) {
                const float tmin = last + eps;
                int64_t sel[GRT_K];
                int ns = 0;
                for (int64_t c = cur; c < m && ns < GRT_K; ++c)
                    if (cand[c].t > tmin) sel[ns++] = c;
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
    free(vrt);
    free(sphere);
}

/* backward: __raygen__rg of referenceBwdOptix.cu:103-170 with icosahedron candidates (same loop as grt_oracle_trace_bwd) */
void grt_ico_oracle_trace_bwd(const gut_oracle_config* cfg, int32_t clamping, int64_t n, const float* particles, const float* sph,
                              int32_t sph_degree, int64_t n_rays, const float* rays_o, const float* rays_d, const float* ray_to_world,
                              const float* out_rgb, const float* out_alpha, const float* out_dist, const float* d_rgb,
                              const float* d_alpha, const float* d_dist, float* d_particles, float* d_sph) {
    float *vrt, *sphere, bb[6];
    ico_setup(cfg, clamping, n, particles, &vrt, &sphere, bb);
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
            const int64_t m = (start < end) ? ico_candidates(n, vrt, sphere, o, d, start + eps, end, cand) : 0;
            int64_t cur = 0;
            float basis[16];
            grt_sh_basis_f(sph_degree, d, basis);
            while (start < end) {
                const float tmin = start + eps;
                int64_t sel[GRT_K];
                int ns = 0;
                for (int64_t c = cur; c < m && ns < GRT_K; ++c)
                    if (cand[c].t > tmin) sel[ns++] = c;
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
    free(vrt);
    free(sphere);
}
