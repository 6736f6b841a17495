/*
 * tests/host_emul/grt_trace_lists.c -- TEST INFRASTRUCTURE ONLY.
 *
 * The hit lists of the brute-force 3DGRT oracle: per ray, the candidates that grt_oracle_trace (primitive `instances`) or
 * grt_ico_oracle_trace (`icosahedron`) process, in order, and the ray's `last` (largest processed t).  The oracle and its
 * icosahedron extension are compiled into this unit unchanged; the loop below is theirs without the radiance, so a consumer that
 * recomposites over these lists integrates exactly what they integrate (tests/test_grt_nht_oracle.py checks that).  The float64
 * NHT oracle (tests/grt_nht_oracle.py) composites features over them.
 */
#include "grt_icosahedron_oracle.c"

/* Per ray ri: count[ri] = number of processed candidates (may exceed cap: only the first cap are stored), and for slot s < cap:
 * pid[ri*cap+s], key[ri*cap+s] (the candidate's t), alpha[ri*cap+s] = min(max_alpha, response density) when the hit is accepted else 0,
 * depth[ri*cap+s] = hit distance when accepted else 0 (`real` precision, widened to double); last[ri] = the ray's last processed t. */
static void trace_lists(const gut_oracle_config* cfg, int32_t clamping, int ico, int64_t n, const float* particles, int64_t n_rays,
                        const float* rays_o, const float* rays_d, const float* ray_to_world, int32_t cap, int32_t* count, int32_t* pid,
                        float* key, double* alpha, double* depth, float* last_out) {
    float *kscl = NULL, *vrt = NULL, *sphere = NULL, bb[6];
    if (ico) {
        ico_setup(cfg, clamping, n, particles, &vrt, &sphere, bb);
    } else {
        kscl = (float*)malloc((size_t)(n > 0 ? n : 1) * 3 * sizeof(float));
        grt_oracle_proxies(cfg, clamping, n, particles, kscl, bb);
    }
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
            real T = 1.f;
            int32_t k = 0;
            int64_t m = 0;
            if (last <= t1)
                m = ico ? ico_candidates(n, vrt, sphere, o, d, last + eps, t1 + eps, cand)
                        : grt_candidates(n, particles, kscl, o, d, last + eps, t1 + eps, cand);
            int64_t cur = 0;
            while ((last <= t1) && (T > cfg->min_transmittance)) {
                const float tmin = last + eps;
                int64_t sel[GRT_K];
                int ns = 0;
                for (int64_t c = cur; c < m && ns < GRT_K; ++c)
                    if (cand[c].t > tmin && cand[c].t_out >= tmin) sel[ns++] = c; /* t_out = t for icosahedra */
                if (ns == 0) break;
                for (int s = 0; s < ns; ++s) {
                    if (!(T > cfg->min_transmittance)) continue;
                    const grt_cand h = cand[sel[s]];
                    const particle g = load_particle(particles + (int64_t)h.pid * 12);
                    const hit_t e = eval_hit(cfg, &g, V3(o[0], o[1], o[2]), V3(d[0], d[1], d[2]));
                    if (k < cap) {
                        const int64_t q = ri * cap + k;
                        pid[q] = (int32_t)h.pid;
                        key[q] = h.t;
                        alpha[q] = e.accept ? (double)e.galpha : 0.0;
                        depth[q] = e.accept ? (double)hit_distance(&g, &e) : 0.0;
                    }
                    k++;
                    if (e.accept) T *= (1 - e.galpha);
                    last = fmaxf(last, h.t);
                }
                while (cur < m && cand[cur].t <= last) cur++;
            }
            count[ri] = k;
            last_out[ri] = last;
        }
        free(cand);
    }
    free(kscl);
    free(vrt);
    free(sphere);
}

void grt_oracle_trace_lists(const gut_oracle_config* cfg, int32_t clamping, int64_t n, const float* particles, int64_t n_rays,
                            const float* rays_o, const float* rays_d, const float* ray_to_world, int32_t cap, int32_t* count, int32_t* pid,
                            float* key, double* alpha, double* depth, float* last) {
    trace_lists(cfg, clamping, 0, n, particles, n_rays, rays_o, rays_d, ray_to_world, cap, count, pid, key, alpha, depth, last);
}

void grt_ico_oracle_trace_lists(const gut_oracle_config* cfg, int32_t clamping, int64_t n, const float* particles, int64_t n_rays,
                                const float* rays_o, const float* rays_d, const float* ray_to_world, int32_t cap, int32_t* count,
                                int32_t* pid, float* key, double* alpha, double* depth, float* last) {
    trace_lists(cfg, clamping, 1, n, particles, n_rays, rays_o, rays_d, ray_to_world, cap, count, pid, key, alpha, depth, last);
}
