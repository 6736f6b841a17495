// 3dgrut_b200/csrc/gut_render.cu -- per-tile compositing (G6), its adjoint (G7) and the per-particle
// spherical-harmonics adjoint (G8) of the 3DGUT path.
//
// Reference semantics restated (not copied) from
//   G6  threedgut_tracer/include/3dgut/kernels/cuda/renderers/gutKBufferRenderer.cuh:274-352 (k-buffer = 0)
//       + kernels/slang/models/gaussianParticles.slang:96-274 (canonical ray, response, integrate)
//   G7  gutKBufferRenderer.cuh:642-716 + kernels/cuda/models/gaussianParticles.cuh:484-751 (hand-written adjoint)
//   G8  kernels/cuda/renderers/gutProjector.cuh:390-430 + slang/common/sphericalHarmonics.slang:21-64
//
// Design (DESIGN.md section 4; sub-tile culling: see the section comment below): one CTA per 16x16 tile (the tile id is part of the sort key, so the tile
// shape is fixed by parity), 256 threads = 256 pixels, sorted particle lists consumed in batches staged in
// shared memory as render-ready records (scale folded into the rotation rows once per staged particle
// instead of once per pixel test).  Both kernels are FP32/SFU-issue bound, not HBM bound.
// G7 sums the 16 canonical per-particle sums (+ 3 depth slots; section comment "G7 backward") over a quarter of the warp through a
// per-warp shared-memory scratch and lands each 16-byte column with one vector RED into a [N,20] accumulator that G8 maps to the
// final gradients and re-zeroes.
#include "gut_common.cuh"
#include "hit_math.cuh"
#include "render_tile.cuh"
#include "subtile_cull.cuh"
#include "tma.cuh"

namespace gutb200 {

namespace {

constexpr int kBatch = 256;

// ----------------------------------------------------------------------------------------------------------
// Sub-tile culling (ours; the reference runs the full test on all 256 pixels of a tile for every entry of the tile's list).
//
// For rays with a common origin o the accept test of a (pixel, particle) pair,
//     |normalize(M d) x g|^2 < r^2,   M = S^-1 R^T, g = M (o - mu),  r^2 = r^2(min response, min alpha / density),
// is a quadratic inequality in the projective coordinates (u, v) of the ray in a local frame (e1, e2, e3), d ~ e3 + u e1 + v e2:
//     f(u,v) = |c3 + u c1 + v c2|^2 - r^2 |a3 + u a1 + v a2|^2 < 0,   a_i = M e_i,  c_i = a_i x g
// (same cross-product formulation as the exact test, hence the same conditioning).  Each warp owns an 8x4 pixel block; before it
// walks a chunk of 32 list entries, LANE k decides for ENTRY k whether {f < 0} can meet the block's (u, v) rectangle at all --
// the minimum of the convex quadratic over the rectangle, with r^2 inflated and a bound of the fp32 evaluation error subtracted,
// so the decision is a NECESSARY condition of the exact test.  The warp then runs the exact test only on the entries whose
// ballot bit is set (48 % of the warp iterations on C2).  Pairs dropped could never be accepted: outputs are bit-identical with
// the switch on and off (tests/test_gut_parity_gpu.py::test_subtile_culling_is_bit_identical).

// ----------------------------------------------------------------------------------------------------------
// G6 forward
// staged record, 5 x float4: rows of M = diag(1/s) R^T with the particle position in .w, then (s, density), (rgb)

struct FwdSmem {
    float4 m0[kBatch], m1[kBatch], m2[kBatch], sd[kBatch], col[kBatch];
};

// exact test + compositing of one (pixel, staged entry j) pair; returns whether the accept test passed (before the t-range test:
// the reference's backward does not re-apply the range test, DESIGN.md section 5)
template <int DEG, bool UNIFORM>
__device__ __forceinline__ bool forward_pair(const FrameConfig& cfg, const FwdSmem& sm, int j, const Ray& ray, bool& alive, float& T, float& cr,
                                             float& cg, float& cb, float& dist, uint32_t& hits) {
    const float4 m0 = sm.m0[j], m1 = sm.m1[j], m2 = sm.m2[j];
    float gox, goy, goz;
    if (UNIFORM) {
        gox = m0.w; goy = m1.w; goz = m2.w;
    } else {
        const float vx = ray.ox - m0.w, vy = ray.oy - m1.w, vz = ray.oz - m2.w;
        gox = m0.x * vx + m0.y * vy + m0.z * vz;
        goy = m1.x * vx + m1.y * vy + m1.z * vz;
        goz = m2.x * vx + m2.y * vy + m2.z * vz;
    }
    const float ax = m0.x * ray.dx + m0.y * ray.dy + m0.z * ray.dz;
    const float ay = m1.x * ray.dx + m1.y * ray.dy + m1.z * ray.dz;
    const float az = m2.x * ray.dx + m2.y * ray.dy + m2.z * ray.dz;
    const float l = ax * ax + ay * ay + az * az;
    const float il = l > 0.f ? rsqrtf(l) : 1.f;
    const float gdx = ax * il, gdy = ay * il, gdz = az * il;
    const float ccx = gdy * goz - gdz * goy, ccy = gdz * gox - gdx * goz, ccz = gdx * goy - gdy * gox;
    const float gray = ccx * ccx + ccy * ccy + ccz * ccz;
    const float gres = kernel_response<DEG>(gray);
    const float4 sd = sm.sd[j];
    const float alpha = fminf(cfg.max_alpha, gres * sd.w);
    const bool accept = (gres > cfg.min_kernel_density) && (alpha > cfg.min_alpha);
    if (accept) {
        const float pd = -(gdx * gox + gdy * goy + gdz * goz);
        const float hx = sd.x * gdx * pd, hy = sd.y * gdy * pd, hz = sd.z * gdz * pd;
        const float t = sqrtf(hx * hx + hy * hy + hz * hz);
        if ((t > ray.tmin) && (t < ray.tmax)) {
            const float w = alpha * T;
            dist += t * w;
            T *= (1.f - alpha);
            if (w > 0.f) {
                const float4 c = sm.col[j];
                cr += c.x * w;
                cg += c.y * w;
                cb += c.z * w;
                hits++;
            }
            if (T < cfg.min_transmittance) alive = false;
        }
    }
    return accept;
}

// Work counters (debug entry point gutb200_debug_work_counters; COUNT instantiations never run on the product path).
//   0 tests_ref   (pixel, entry) pairs the reference's loop evaluates: every live pixel tests every entry of its tile list
//   1 tests_exec  lane-level exact tests our forward executes after sub-tile culling
//   2 hits        accepted pairs (the set the backward's adjoint runs on)
//   3 fwd_iters   warp iterations of the forward's exact test     4 hit_iters  warp iterations with >= 1 accepting lane (= backward's iterations)
//   5 screens     lane-level sub-tile culling screens             6 bwd_lanes  live lanes summed over hit_iters (lane-level tests of the backward)
//   7 iters16 / 8 iters8   backward iterations when half-warps (4x4 pixels) / quarter-warps (4x2) walk their own entries in lockstep
//   9 sub16_hits / 10 sub8_hits   (half-warp, entry) / (quarter-warp, entry) pairs with >= 1 accepting lane (= gradient rows flushed)
struct WorkCounters {
    unsigned long long v[16];
};


template <int DEG, bool UNIFORM, bool COUNT>
__device__ __forceinline__ void forward_tile(const FrameConfig& cfg, FwdSmem& sm, const WarpFrame& wf, const Ray& ray, float o0x, float o0y,
                                             float o0z, int tid, uint32_t begin, uint32_t end, const float* __restrict__ particles,
                                             const float* __restrict__ rgb, const uint32_t* __restrict__ sorted_values,
                                             uint32_t* __restrict__ hit_words, bool& alive, float& T, float& cr, float& cg, float& cb,
                                             float& dist, uint32_t& hits, WorkCounters* __restrict__ ctr) {
    const int lane = tid & 31;
    unsigned long long c_ref = 0, c_exec = 0, c_hits = 0, c_iters = 0, c_hit_iters = 0, c_screens = 0, c_bwd_lanes = 0;
    unsigned long long c_iters16 = 0, c_iters8 = 0, c_sub16 = 0, c_sub8 = 0;
    for (uint32_t base = begin; base < end; base += kBatch) {
        if (__syncthreads_and(!alive)) break;
        const uint32_t k = base + tid;
        if (k < end) {
            const uint32_t idx = sorted_values[k];
            const float4* p4 = reinterpret_cast<const float4*>(particles) + static_cast<size_t>(idx) * 3;
            const float4 a = __ldg(p4), q = __ldg(p4 + 1), s = __ldg(p4 + 2);
            const float r = q.x, x = q.y, y = q.z, z = q.w;
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, xz = x * z, yz = y * z;
            const float rx = r * x, ry = r * y, rz = r * z;
            const float isx = 1.0f / s.x, isy = 1.0f / s.y, isz = 1.0f / s.z;
            float4 m0 = make_float4(isx * (1.f - 2.f * (yy + zz)), isx * (2.f * (xy + rz)), isx * (2.f * (xz - ry)), a.x);
            float4 m1 = make_float4(isy * (2.f * (xy - rz)), isy * (1.f - 2.f * (xx + zz)), isy * (2.f * (yz + rx)), a.y);
            float4 m2 = make_float4(isz * (2.f * (xz + ry)), isz * (2.f * (yz - rx)), isz * (1.f - 2.f * (xx + yy)), a.z);
            if (UNIFORM) {  // .w carries the canonical origin instead of the particle position
                const float vx = o0x - a.x, vy = o0y - a.y, vz = o0z - a.z;
                m0.w = m0.x * vx + m0.y * vy + m0.z * vz;
                m1.w = m1.x * vx + m1.y * vy + m1.z * vz;
                m2.w = m2.x * vx + m2.y * vy + m2.z * vz;
            }
            sm.m0[tid] = m0;
            sm.m1[tid] = m1;
            sm.m2[tid] = m2;
            sm.sd[tid] = make_float4(s.x, s.y, s.z, a.w);
            sm.col[tid] = make_float4(fmaxf(rgb[idx * 3 + 0], 0.f), fmaxf(rgb[idx * 3 + 1], 0.f), fmaxf(rgb[idx * 3 + 2], 0.f), 0.f);
        }
        __syncthreads();
        const int count = min(kBatch, static_cast<int>(end - base));
        // this warp's hit words of the batch: bit e of word c/32 = "some pixel of the warp's 8x4 block accepted entry c + e" -- the backward
        // walks only those entries (a necessary condition of its own exact test, so it drops nothing it would have accepted)
        uint32_t* words = hit_words + (static_cast<size_t>(base - begin) >> 5) * kWordsPerChunk + (tid >> 5) * 4;
        const int quarter = lane_quarter(lane);
        const unsigned my_quarter = quarter_lanes(quarter);
        const bool writer = (lane & 0x0B) == 0;  // lanes 0, 4, 16, 20: one per quarter
        if (UNIFORM) {
            // chunks of 32 entries: lane k screens entry k against the warp's pixel block, the warp walks the survivors
            for (int c = 0; c < count; c += 32) {
                if (!__any_sync(kFull, alive)) break;
                const int e = c + lane;
                bool cand = e < count;
                if (wf.on && cand) {
                    const float4 m0 = sm.m0[e], m1 = sm.m1[e], m2 = sm.m2[e];
                    cand = block_candidate<DEG>(cfg, wf, m0.x, m0.y, m0.z, m1.x, m1.y, m1.z, m2.x, m2.y, m2.z, m0.w, m1.w, m2.w, sm.sd[e].w);
                    if (COUNT) c_screens++;
                }
                unsigned todo = __ballot_sync(kFull, cand);
                uint32_t word = 0;
                int prev = c;
                while (todo) {
                    const int b = __ffs(todo) - 1;
                    const int j = c + b;
                    todo &= todo - 1;
                    int live_n = 0;
                    if (COUNT) {
                        live_n = __popc(__ballot_sync(kFull, alive));
                        c_ref += static_cast<unsigned long long>(live_n) * (j - prev + 1);
                        prev = j + 1;
                        c_iters++;
                        if (alive) c_exec++;
                    }
                    bool acc = false;
                    if (alive) acc = forward_pair<DEG, true>(cfg, sm, j, ray, alive, T, cr, cg, cb, dist, hits);
                    const unsigned accs = __ballot_sync(kFull, acc);
                    if (accs & my_quarter) word |= 1u << b;  // this lane's quarter (4x2 pixels) accepted entry j
                    if (COUNT && accs) {
                        c_hit_iters++;
                        c_bwd_lanes += live_n;
                        c_hits += acc ? 1 : 0;
                    }
                }
                if (COUNT) {
                    const unsigned live = __ballot_sync(kFull, alive);
                    c_ref += static_cast<unsigned long long>(__popc(live)) * (min(c + 32, count) - prev);
                    // lockstep iteration counts of the sub-block walks: halves split by b2, quarters by (b2, b4)
                    const uint32_t wq = word, wh = word | __shfl_xor_sync(kFull, word, 16);
                    const int p16 = __popc(wh), p8 = __popc(wq);
                    const int m16 = max(p16, __shfl_xor_sync(kFull, p16, 4));
                    int m8 = max(p8, __shfl_xor_sync(kFull, p8, 4));
                    m8 = max(m8, __shfl_xor_sync(kFull, m8, 16));
                    c_iters16 += m16;
                    c_iters8 += m8;
                    c_sub16 += p16 + __shfl_xor_sync(kFull, p16, 4);
                    int s8 = p8 + __shfl_xor_sync(kFull, p8, 4);
                    s8 += __shfl_xor_sync(kFull, s8, 16);
                    c_sub8 += s8;
                }
                if (writer) words[(c >> 5) * kWordsPerChunk + quarter] = word;
            }
        } else {
            // per-pixel origins: no warp-level screening; the backward gets all-ones words for these tiles
            if (writer)
                for (int c = 0; c < count; c += 32) words[(c >> 5) * kWordsPerChunk + quarter] = 0xFFFFFFFFu;
            for (int j = 0; alive && j < count; ++j) {
                const bool acc = forward_pair<DEG, false>(cfg, sm, j, ray, alive, T, cr, cg, cb, dist, hits);
                if (COUNT) {
                    c_exec++;
                    c_hits += acc ? 1 : 0;
                }
            }
        }
    }
    if (COUNT) {
        // c_ref, c_iters, c_hit_iters are warp-uniform (lane 0 reports); the others are per lane
        if (!UNIFORM) c_ref = 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            c_exec += __shfl_xor_sync(kFull, c_exec, o);
            c_hits += __shfl_xor_sync(kFull, c_hits, o);
            c_screens += __shfl_xor_sync(kFull, c_screens, o);
        }
        if (lane == 0) {
            if (!UNIFORM) c_ref = c_exec;
            atomicAdd(&ctr->v[0], c_ref);
            atomicAdd(&ctr->v[1], c_exec);
            atomicAdd(&ctr->v[2], c_hits);
            atomicAdd(&ctr->v[3], c_iters);
            atomicAdd(&ctr->v[4], c_hit_iters);
            atomicAdd(&ctr->v[5], c_screens);
            atomicAdd(&ctr->v[6], c_bwd_lanes);
            atomicAdd(&ctr->v[7], c_iters16);
            atomicAdd(&ctr->v[8], c_iters8);
            atomicAdd(&ctr->v[9], c_sub16);
            atomicAdd(&ctr->v[10], c_sub8);
        }
    }
}

template <int DEG, bool COUNT>
__global__ void __launch_bounds__(kTilePixels) render_forward_kernel(FrameCamera cam, FrameConfig cfg,
                                                                     const float* __restrict__ rays_o,
                                                                     const float* __restrict__ rays_d,
                                                                     const float* __restrict__ particles,
                                                                     const float* __restrict__ rgb,
                                                                     const uint32_t* __restrict__ sorted_values,
                                                                     const uint32_t* __restrict__ ranges,
                                                                     const uint32_t* __restrict__ tile_order,
                                                                     const uint32_t* __restrict__ chunk_base, uint32_t* __restrict__ hit_words,
                                                                     float* __restrict__ out_rgba, float* __restrict__ out_dist,
                                                                     float* __restrict__ out_hits, WorkCounters* __restrict__ ctr) {
    __shared__ FwdSmem sm;
    const int tile = tile_order[blockIdx.x];  // heaviest tiles first (tile_scan_kernel's order): shortens the tail of the grid
    const int tid = threadIdx.x;
    int px, py;
    tile_pixel(tile, cam.grid_x, tid, px, py);
    const bool inside = (px < cam.width) && (py < cam.height);
    const int64_t pix = static_cast<int64_t>(py) * cam.width + px;

    Ray ray;
    ray.alive = false;
    if (inside) ray = make_ray(cam, rays_o, rays_d, pix);
    const bool valid = inside && ray.alive;
    float o0x, o0y, o0z;
    const bool uniform = tile_common_origin(cam, rays_o, tile, inside, pix, o0x, o0y, o0z);
    const WarpFrame wf = make_warp_frame(cam, ray, valid, uniform && (cfg.subtile_culling & 2), tid & 31);

    float T = 1.f, cr = 0.f, cg = 0.f, cb = 0.f, dist = 0.f;
    uint32_t hits = 0;
    bool alive = valid;
    const uint32_t begin = ranges[tile * 2], end = ranges[tile * 2 + 1];
    uint32_t* words = hit_words + static_cast<size_t>(chunk_base[tile]) * kWordsPerChunk;
    if (uniform)
        forward_tile<DEG, true, COUNT>(cfg, sm, wf, ray, o0x, o0y, o0z, tid, begin, end, particles, rgb, sorted_values, words, alive, T, cr, cg, cb, dist, hits, ctr);
    else
        forward_tile<DEG, false, COUNT>(cfg, sm, wf, ray, o0x, o0y, o0z, tid, begin, end, particles, rgb, sorted_values, words, alive, T, cr, cg, cb, dist, hits, ctr);
    if (COUNT) return;  // the counting pass leaves the frame's outputs alone

    if (valid) {  // finalizeRay (rayPayload.cuh:160-193); invalid rays keep the initial buffer values
        reinterpret_cast<float4*>(out_rgba)[pix] = make_float4(cr, cg, cb, 1.0f - T);
        out_dist[pix] = dist;
        out_hits[pix] = static_cast<float>(hits);
    } else if (inside) {
        reinterpret_cast<float4*>(out_rgba)[pix] = make_float4(0.f, 0.f, 0.f, 0.f);
        out_dist[pix] = 1e06f;  // torch::ones(...)*1e6 (splatRaster.cpp:213)
        out_hits[pix] = 0.f;
    }
}

// ----------------------------------------------------------------------------------------------------------
// G7 backward
//
// What is summed per particle, and where (DESIGN.md section 4): with gro = S^-1 R (o - mu) and grdu = S^-1 R d the hand adjoint
// (gaussianParticles.cuh:684-747) ends in terms that are LINEAR in per-particle constants once the ray origin is fixed:
//     d pos   = -R^T (S^-1 groGrd)
//     d scale_i = <depth part>_i - grdu_i (S^-1 grduGrd)_i - gro_i (S^-1 groGrd)_i
//     d quat  = J(q)^T vec( (S^-1 groGrd) (o - mu)^T + (S^-1 grduGrd) d^T )
// and grdu_i = (R d)_i / s_i, so both the scale term and the quaternion term are contractions of the 3x3 matrix
//     W = sum over the particle's (pixel, hit) pairs of  grduGrd (x) d   (+ groGrd (x) (o - o_f) for pixels off the frame origin):
//     d scale_i -= (R_i . W_i) / s_i^2,      d quat = J(q)^T vec( S^-1 (W + G (o_f - mu)^T) ).
// The kernel therefore accumulates, per particle, the canonical sums  G = sum groGrd (slots 0..2), W (slots 4..12, row-major) and the
// depth branch's direct scale part (slots 16..18; only warps whose pixels carry a distance gradient touch them), all relative to the
// FRAME origin o_f = origin of the frame's first ray; G8 (project_backward_kernel<.., CANON = true>) applies the linear maps once per
// particle instead of once per (pixel, particle).  Pixels whose origin differs from o_f (GENERAL tiles: per-pixel origins) add the
// exact correction terms, so the result is the reference's gradient for any ray bundle.
// Without a distance gradient the adjoint of normalize() collapses: grdGrd = gro x k and groGrd = k x grd with k parallel to grd x gro
// give  grduGrd = (-(grd . gro) / |grdu|) groGrd  exactly, so the cross product, the dot product and the three-term normalisation
// adjoint of (:684-731) are one multiply; the terms that cancel analytically there (grd |gro|^2) are never formed.
//
// staged record, 6 x float4:
//   r0, r1, r2 = rows of quaternionWXYZToMatrix (columns of R); .w = canonical frame origin S^-1 R (o_f - mu) (FAST) | position (GENERAL)
//   sc = scale.xyz, density     is = 1/scale.xyz, _     cl = clamped rgb, particle index bits
// The rotation rows are kept apart from 1/scale (the forward stages M = S^-1 R^T): the backward's accept test applies 1/s after the
// rotation, as the reference's adjoint does.  With the forward's record the test moves by the last bits, borderline pairs flip, and
// on a 500-Gaussian scene the gradients drifted from 4.7e-4 to 1.8e-3 relative to the CPU restatement of the reference.
//
// The gradient rows of one lockstep iteration are summed through a per-warp scratch:
//   every lane stores its row (g[0..15], the depth slots 16..18 when the warp carries a distance gradient; zeros without a hit) as
//   float4 at a stride of kGradRow floats -- 8 consecutive lanes then hit 8 distinct 16-byte bank groups, so the stores are
//   conflict-free --, and lane r (r < 5, or < 4 without depth slots) of each sub-block sums float4 column r over the sub-block's
//   rows and lands it with one 16-byte vector RED.  For SUBL 8 and 16 the readers of one lane octet read two rows 4 lanes apart,
//   columns 0..3: 16-byte groups 5 row + r and 5 row + 20 + r are again 8 distinct ones.
// This replaced a transposing butterfly over the sub-block (14 SHFL + 14 FADD + ~28 SEL per lane, 3 more 5-level sums for the depth
// slots and a second RED): 5 STS.128 + SUBL LDS.128 on the summing lanes, 5 REDs per flushed row instead of 9 (4 instead of 8 without
// the depth slots).  render_backward on C2 (H100 80GB HBM3, 700 W, 1980 MHz, three runs each): 0.454-0.460 -> 0.417-0.422 ms; with the rgb / opacity
// loss (no depth slots) unchanged at 0.354-0.358 ms.

struct BwdSmem {
    float4 r0[kBatch], r1[kBatch], r2[kBatch], sc[kBatch], is[kBatch], cl[kBatch];
    uint32_t hw[(kBatch / 32) * kWordsPerChunk];        // the forward's hit words of this batch, [chunk][warp][quarter]
    float4 rows[kTilePixels / 32][32 * kGradRow / 4];  // gradient rows of one lockstep iteration, [warp][lane * 5 + column]
};

// Sub-blocks of SUBL lanes (32: the warp, 16: half = 4x4 pixels, 8: quarter = 4x2 pixels): the sub-block id uses lane bits b2 (and
// b4), the lanes within it the others.  sub_lane = the i-th lane of the sub-block whose lowest lane is `first`, sub_rank = its inverse.
template <int SUBL>
__device__ __forceinline__ int sub_first(int lane) { return SUBL == 32 ? 0 : SUBL == 16 ? (lane & 4) : (lane & 20); }

template <int SUBL>
__device__ __forceinline__ int sub_lane(int first, int i) {
    if (SUBL == 32) return i;
    if (SUBL == 16) return first | (i & 3) | ((i & 12) << 1);
    return first | (i & 3) | ((i & 4) << 1);
}

template <int SUBL>
__device__ __forceinline__ int sub_rank(int lane) {
    if (SUBL == 32) return lane;
    if (SUBL == 16) return (lane & 3) | ((lane >> 1) & 12);
    return (lane & 3) | ((lane >> 1) & 4);
}


// exact test + adjoint of one (pixel, staged entry j) pair (processHitBwd, gaussianParticles.cuh:484-751); fills g[] and returns true on a hit
template <int DEG, bool FAST>
__device__ __forceinline__ bool backward_pair(const FrameConfig& cfg, const BwdSmem& sm, int j, const Ray& ray, float dox, float doy, float doz,
                                              bool depth_grads, BwdRay& st, bool& alive, float (&g)[16], float (&ex)[3]) {
    const float4 r0 = sm.r0[j], r1 = sm.r1[j], r2 = sm.r2[j], sc = sm.sc[j], is = sm.is[j];
    float gox, goy, goz;                                                                          // gro
    float pcx = 0.f, pcy = 0.f, pcz = 0.f;
    if (FAST) {
        gox = r0.w; goy = r1.w; goz = r2.w;
    } else {
        pcx = ray.ox - r0.w; pcy = ray.oy - r1.w; pcz = ray.oz - r2.w;                              // gposc
        gox = is.x * (r0.x * pcx + r0.y * pcy + r0.z * pcz);
        goy = is.y * (r1.x * pcx + r1.y * pcy + r1.z * pcz);
        goz = is.z * (r2.x * pcx + r2.y * pcy + r2.z * pcz);
    }
    const float drx = r0.x * ray.dx + r0.y * ray.dy + r0.z * ray.dz;                                // rayDirR
    const float dry = r1.x * ray.dx + r1.y * ray.dy + r1.z * ray.dz;
    const float drz = r2.x * ray.dx + r2.y * ray.dy + r2.z * ray.dz;
    const float ux = is.x * drx, uy = is.y * dry, uz = is.z * drz;                                  // grdu
    const float l = ux * ux + uy * uy + uz * uz;
    const float il = l > 0.f ? rsqrtf(l) : 1.f;
    const float gdx = ux * il, gdy = uy * il, gdz = uz * il;                                        // grd
    const float ccx = gdy * goz - gdz * goy, ccy = gdz * gox - gdx * goz, ccz = gdx * goy - gdy * gox;  // gcrod
    const float gray = ccx * ccx + ccy * ccy + ccz * ccz;
    const float gres = kernel_response<DEG>(gray);
    const float dns = sc.w;
    const float alpha = fminf(cfg.max_alpha, gres * dns);
    if (!((gres > cfg.min_kernel_density) && (alpha > cfg.min_alpha))) return false;

    const float4 cl = sm.cl[j];
    const float T = st.T;
    const float weight = alpha * T;
    const float nextT = (1.f - alpha) * T;
    const bool last = nextT <= cfg.min_transmittance;
    const float inv_next = last ? 0.f : 1.0f / nextT;
    const float pd = -(gdx * gox + gdy * goy + gdz * goz);

    // depth branch (:545-580); skipped by warps whose pixels carry no distance gradient (an RGB-only loss)
    float a_hit = 0.f, sd = 0.f, hgx = 0.f, hgy = 0.f, hgz = 0.f, ddx = 0.f, ddy = 0.f, ddz = 0.f;
    if (depth_grads) {
        ddx = gdx * pd; ddy = gdy * pd; ddz = gdz * pd;                                             // grdd
        const float hx = sc.x * ddx, hy = sc.y * ddy, hz = sc.z * ddz;                              // grds
        const float gsq = hx * hx + hy * hy + hz * hz;
        const float gdist = sqrtf(gsq);
        st.D += weight * gdist;
        const float resD = fmaxf((st.Dint - st.D) * inv_next, 0.f);
        a_hit = (gdist - resD) * T * st.Dgrad;
        const float hs = gsq > 0.f ? (weight / gdist) * st.Dgrad : 0.f;
        hgx = hx * hs; hgy = hy * hs; hgz = hz * hs;                                                // grdsRayHitGrd
        sd = hgx * sc.x * gdx + hgy * sc.y * gdy + hgz * sc.z * gdz;                                // grdScaledDot
    }
    // opacity branch (:586-587)
    const float resT = alpha < 0.999999f ? st.Tint / (1.f - alpha) : T;
    const float a_dns = resT * -st.Tgrad;
    // radiance branch (:602-612)
    g[13] = st.Cgx * weight; g[14] = st.Cgy * weight; g[15] = st.Cgz * weight;
    st.Cx += weight * cl.x; st.Cy += weight * cl.y; st.Cz += weight * cl.z;
    const float rcx = fmaxf((st.Cix - st.Cx) * inv_next, 0.f);
    const float rcy = fmaxf((st.Ciy - st.Cy) * inv_next, 0.f);
    const float rcz = fmaxf((st.Ciz - st.Cz) * inv_next, 0.f);
    const float common = a_hit + a_dns + T * ((cl.x - rcx) * st.Cgx + (cl.y - rcy) * st.Cgy + (cl.z - rcz) * st.Cgz);
    g[3] = gres * common;                                                                           // d density (:624-627)
    const float gray_g = kernel_response_grad<DEG>(gray, gres, dns * common);                       // (:639-648)
    // gray = |grd x gro|^2  (:684-702)
    const float kx = 2.f * ccx * gray_g, ky = 2.f * ccy * gray_g, kz = 2.f * ccz * gray_g;          // gcrodGrd
    float go_gx = ky * gdz - kz * gdy, go_gy = kz * gdx - kx * gdz, go_gz = kx * gdy - ky * gdx;    // groGrd
    float ug_x, ug_y, ug_z;                                                                         // grduGrd
    if (depth_grads) {
        // + grdRayHitGrd = S grdsRayHitGrd pd - gro sd, groRayHitGrd = -grd sd (:560-580), then grd = normalize(grdu) (:729-731): with
        // P = k x grd (the groGrd above) the projection (I - grd grd^T) of grdGrd = gro x k + S hg pd - gro sd is, term by term,
        // pd P,  pd (S hg - grd sd)  and  -sd (gro + pd grd), i.e.  grduGrd = (pd (P + S hg - 2 sd grd) - sd gro) / |grdu|
        const float sd2 = 2.f * sd;
        const float vx = (go_gx + sc.x * hgx) - sd2 * gdx, vy = (go_gy + sc.y * hgy) - sd2 * gdy, vz = (go_gz + sc.z * hgz) - sd2 * gdz;
        ug_x = il * (pd * vx - sd * gox); ug_y = il * (pd * vy - sd * goy); ug_z = il * (pd * vz - sd * goz);
        go_gx -= gdx * sd; go_gy -= gdy * sd; go_gz -= gdz * sd;
        ex[0] = ddx * hgx; ex[1] = ddy * hgy; ex[2] = ddz * hgz;                                     // gsclRayHitGrd (:705-713)
    } else {  // the same chain in closed form (section comment): grduGrd = (pd / |grdu|) groGrd
        const float tq = pd * il;
        ug_x = tq * go_gx; ug_y = tq * go_gy; ug_z = tq * go_gz;
    }
    g[0] = go_gx; g[1] = go_gy; g[2] = go_gz;          // canonical: G8 turns the sums into d pos, the gro part of d scale and of d quat
    // W rows: grduGrd_i * d  (+ groGrd_i * (o - o_f) for pixels off the frame origin); G8 scales row i by 1/s_i (rayDirRGrd, gposcrGrd)
    // and contracts it with R for d scale (:733-738) and with the quaternion Jacobian for d quat (matmul_bw_quat, :719-747)
    g[4] = ug_x * ray.dx; g[5] = ug_x * ray.dy; g[6] = ug_x * ray.dz;
    g[7] = ug_y * ray.dx; g[8] = ug_y * ray.dy; g[9] = ug_y * ray.dz;
    g[10] = ug_z * ray.dx; g[11] = ug_z * ray.dy; g[12] = ug_z * ray.dz;
    if (!FAST) {
        g[4] += go_gx * dox; g[5] += go_gx * doy; g[6] += go_gx * doz;
        g[7] += go_gy * dox; g[8] += go_gy * doy; g[9] += go_gy * doz;
        g[10] += go_gz * dox; g[11] += go_gz * doy; g[12] += go_gz * doz;
    }
    st.T = nextT;
    if (nextT < cfg.min_transmittance) alive = false;
    return true;
}

template <int DEG, bool FAST, int SUBL>
__device__ __forceinline__ void backward_tile(const FrameConfig& cfg, BwdSmem& sm, const Ray& ray, float ofx, float ofy, float ofz, int tid,
                                              int lane, uint32_t begin, uint32_t end, const float* __restrict__ particles,
                                              const float* __restrict__ rgb, const uint32_t* __restrict__ sorted_values,
                                              const uint32_t* __restrict__ hit_words, bool use_words, bool alive, BwdRay& st,
                                              float* __restrict__ grad_acc) {
    const float dox = ray.ox - ofx, doy = ray.oy - ofy, doz = ray.oz - ofz;   // zero in FAST tiles
    const bool depth_grads = __any_sync(kFull, alive && (st.Dgrad != 0.f));
    const int quarter = lane_quarter(lane);
    // lanes of this lane's sub-block, and the float4 column of the gradient row this lane sums (columns >= 5 / 4: none)
    const unsigned sub_lanes = SUBL == 32 ? kFull : SUBL == 16 ? (quarter_lanes(quarter & 1) | quarter_lanes((quarter & 1) | 2)) : quarter_lanes(quarter);
    const int first = sub_first<SUBL>(lane);
    const int col = sub_rank<SUBL>(lane);
    const int cols = depth_grads ? 5 : 4;
    float4* rows = sm.rows[tid >> 5];
    for (uint32_t base = begin; base < end; base += kBatch) {
        if (__syncthreads_and(!alive)) break;
        const uint32_t k = base + tid;
        {   // 8 chunks x 8 warps x 4 quarters = one word per thread
            const uint32_t chunk = (base - begin) / 32 + (tid >> 5);
            const bool in_list = base + (tid >> 5) * 32 < end;
            sm.hw[tid] = (use_words && in_list) ? hit_words[static_cast<size_t>(chunk) * kWordsPerChunk + (tid & 31)] : 0xFFFFFFFFu;
        }
        if (k < end) {
            const uint32_t idx = sorted_values[k];
            const float4* p4 = reinterpret_cast<const float4*>(particles) + static_cast<size_t>(idx) * 3;
            const float4 a = __ldg(p4), q = __ldg(p4 + 1), s = __ldg(p4 + 2);
            const float r = q.x, x = q.y, y = q.z, z = q.w;
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, xz = x * z, yz = y * z;
            const float rx = r * x, ry = r * y, rz = r * z;
            float4 t0 = make_float4(1.f - 2.f * (yy + zz), 2.f * (xy + rz), 2.f * (xz - ry), a.x);
            float4 t1 = make_float4(2.f * (xy - rz), 1.f - 2.f * (xx + zz), 2.f * (yz + rx), a.y);
            float4 t2 = make_float4(2.f * (xz + ry), 2.f * (yz - rx), 1.f - 2.f * (xx + yy), a.z);
            if (FAST) {  // .w carries the canonical frame origin instead of the particle position
                const float vx = ofx - a.x, vy = ofy - a.y, vz = ofz - a.z;
                t0.w = (t0.x * vx + t0.y * vy + t0.z * vz) / s.x;
                t1.w = (t1.x * vx + t1.y * vy + t1.z * vz) / s.y;
                t2.w = (t2.x * vx + t2.y * vy + t2.z * vz) / s.z;
            }
            sm.r0[tid] = t0;
            sm.r1[tid] = t1;
            sm.r2[tid] = t2;
            sm.sc[tid] = make_float4(s.x, s.y, s.z, a.w);
            sm.is[tid] = make_float4(1.0f / s.x, 1.0f / s.y, 1.0f / s.z, 0.f);
            sm.cl[tid] = make_float4(fmaxf(rgb[idx * 3 + 0], 0.f), fmaxf(rgb[idx * 3 + 1], 0.f), fmaxf(rgb[idx * 3 + 2], 0.f),
                                     __uint_as_float(idx));
        }
        __syncthreads();
        const int count = min(kBatch, static_cast<int>(end - base));
        // chunks of 32 entries.  Every sub-block of the warp walks ITS OWN entries -- those some pixel of the sub-block accepted in the
        // forward (hit words) -- in lockstep with the other sub-blocks: one pass of the adjoint serves up to 32 / SUBL particles, and
        // the reduction tree is log2(SUBL) levels deep.
        for (int c = 0; c < count; c += 32) {
            if (__all_sync(kFull, !alive)) break;
            const uint32_t* hw = sm.hw + (c >> 5) * kWordsPerChunk + (tid >> 5) * 4;
            unsigned todo;
            if (SUBL == 32) todo = hw[0] | hw[1] | hw[2] | hw[3];
            else if (SUBL == 16) todo = hw[quarter & 1] | hw[(quarter & 1) | 2];
            else todo = hw[quarter];
            if (count - c < 32) todo &= (1u << (count - c)) - 1u;
            while (__any_sync(kFull, todo != 0u)) {
                const bool act = todo != 0u;
                const int j = act ? c + __ffs(todo) - 1 : c;
                todo &= todo - 1;
                float g[16], ex[3];
#pragma unroll
                for (int i = 0; i < 16; ++i) g[i] = 0.f;
                ex[0] = ex[1] = ex[2] = 0.f;
                bool hit = false;
                if (act && alive) hit = backward_pair<DEG, FAST>(cfg, sm, j, ray, dox, doy, doz, depth_grads, st, alive, g, ex);
                const unsigned hits = __ballot_sync(kFull, hit);
                if (hits) {
                    float4* mine = rows + lane * (kGradRow / 4);
                    mine[0] = make_float4(g[0], g[1], g[2], g[3]);
                    mine[1] = make_float4(g[4], g[5], g[6], g[7]);
                    mine[2] = make_float4(g[8], g[9], g[10], g[11]);
                    mine[3] = make_float4(g[12], g[13], g[14], g[15]);
                    if (depth_grads) mine[4] = make_float4(ex[0], ex[1], ex[2], 0.f);  // warp-uniform
                    __syncwarp();
                    if ((hits & sub_lanes) && col < cols) {  // this sub-block's particle received something
                        float4 s = rows[sub_lane<SUBL>(first, 0) * (kGradRow / 4) + col];
#pragma unroll
                        for (int i = 1; i < SUBL; ++i) {
                            const float4 v = rows[sub_lane<SUBL>(first, i) * (kGradRow / 4) + col];
                            s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
                        }
                        atomicAdd(reinterpret_cast<float4*>(grad_acc + static_cast<size_t>(__float_as_uint(sm.cl[j].w)) * kGradRow) + col, s);
                    }
                    __syncwarp();  // the next iteration overwrites the rows
                    if (__all_sync(kFull, !alive)) break;
                }
            }
        }
    }
}

// 3 CTAs per SM (72-80 registers, 45 KB of shared memory per CTA; 24 warps per SM).  4 CTAs would fit in shared memory but cap the
// kernel at 64 registers, where every instantiation spills (36 B stores, 64 B loads per thread).  Measured at C2 on an H100 80GB HBM3
// (700 W), bench.py --steps 50, three runs each, render_backward: 3 -> 0.417-0.422 ms, 4 (with the spills) -> 0.413-0.414 ms.
template <int DEG, int SUBL>
__global__ void __launch_bounds__(kTilePixels, 3) render_backward_kernel(FrameCamera cam, FrameConfig cfg,
                                                                      const float* __restrict__ rays_o,
                                                                      const float* __restrict__ rays_d,
                                                                      const float* __restrict__ particles,
                                                                      const float* __restrict__ rgb,
                                                                      const uint32_t* __restrict__ sorted_values,
                                                                      const uint32_t* __restrict__ ranges,
                                                                      const uint32_t* __restrict__ tile_order,
                                                                      const uint32_t* __restrict__ chunk_base,
                                                                      const uint32_t* __restrict__ hit_words,
                                                                      const float* __restrict__ out_rgba, const float* __restrict__ d_rgba,
                                                                      const float* __restrict__ out_dist, const float* __restrict__ d_dist,
                                                                      float* __restrict__ grad_acc) {
    __shared__ BwdSmem sm;
    const int tile = tile_order[blockIdx.x];
    const int tid = threadIdx.x;
    const int lane = tid & 31;
    int px, py;
    tile_pixel(tile, cam.grid_x, tid, px, py);
    const bool inside = (px < cam.width) && (py < cam.height);
    const int64_t pix = static_cast<int64_t>(py) * cam.width + px;

    Ray ray;
    ray.alive = false;
    if (inside) ray = make_ray(cam, rays_o, rays_d, pix);
    const bool alive = inside && ray.alive;

    BwdRay st;
    st.Cix = st.Ciy = st.Ciz = st.Cgx = st.Cgy = st.Cgz = 0.f;
    st.Tint = 1.f; st.Tgrad = 0.f; st.Dint = 0.f; st.Dgrad = 0.f;
    st.T = 1.f; st.Cx = st.Cy = st.Cz = st.D = 0.f;
    if (alive) {
        const float4 o = reinterpret_cast<const float4*>(out_rgba)[pix];
        const float4 g = reinterpret_cast<const float4*>(d_rgba)[pix];
        st.Cix = o.x; st.Ciy = o.y; st.Ciz = o.z;
        st.Cgx = g.x; st.Cgy = g.y; st.Cgz = g.z;
        st.Tint = 1.f - o.w;
        st.Tgrad = -1.f * g.w;
        st.Dint = out_dist[pix];
        st.Dgrad = d_dist[pix];
    }

    float ofx, ofy, ofz;
    const bool fast = frame_common_origin(cam, rays_o, inside, pix, ofx, ofy, ofz);
    const uint32_t begin = ranges[tile * 2], end = ranges[tile * 2 + 1];
    const uint32_t* words = hit_words + static_cast<size_t>(chunk_base[tile]) * kWordsPerChunk;
    const bool use_words = (cfg.subtile_culling & 4) != 0;
    if (fast)
        backward_tile<DEG, true, SUBL>(cfg, sm, ray, ofx, ofy, ofz, tid, lane, begin, end, particles, rgb, sorted_values, words, use_words, alive, st, grad_acc);
    else
        backward_tile<DEG, false, SUBL>(cfg, sm, ray, ofx, ofy, ofz, tid, lane, begin, end, particles, rgb, sorted_values, words, use_words, alive, st, grad_acc);
}

// ----------------------------------------------------------------------------------------------------------
// G8 per-particle SH adjoint + emission of the final gradient rows; re-zeroes the accumulator for the next frame.

constexpr float kC0 = 0.28209479177387814f;
constexpr float kC1 = 0.4886025119029199f;
__constant__ float kC2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f, -1.0925484305920792f,
                             0.5462742152960396f};
__constant__ float kC3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f, 0.3731763325901154f,
                             -0.4570457994644658f, 1.445305721320277f,  -0.5900435899266435f};

// Block of 128 particles, all global traffic through TMA bulk copies (cp.async.bulk + mbarrier): one copy brings the block's
// accumulator rows, one 192-byte copy per VISIBLE particle brings its SH coefficients, and three bulk stores write the
// d_sph rows, the d_particles rows and the re-zeroed accumulator rows (every output row is written, zeros for invisible
// particles, so the caller needs no memset).  Threads only touch shared memory, with 128-bit accesses.
constexpr int kPbThreads = 128;
constexpr int kAccVec = kGradRow / 4;          // float4 per accumulator row
constexpr uint32_t kAccBytes = kGradRow * 4;  // bytes per accumulator row

// COMPACT (view-parallel training): instead of the [N,48] SH gradient row the kernel emits the masked radiance gradient (3 floats) the
// row is the outer product of -- d_sph[j][c] = basis_j(direction) * g[c] -- so ranks exchange 16 instead of 192 bytes per particle and
// rebuild the summed rows with sph_from_views_kernel.
// CANON: the accumulator rows (kGradRow = 20 floats) hold G7's canonical sums (see the G7 section comment): slots 0..2 = G = sum groGrd,
// 3 = d density, 4..12 = W (row-major), 13..15 = d rgb, 16..18 = the depth branch's direct part of d scale; the per-particle linear maps
// are applied here.  (The sorted k-buffer kernels still accumulate final gradients: CANON = false, slots 0..10 + rgb in 12..14.)
// SPH = false (NHT features, gut_render_nht.cu): no radiance and no SH adjoint; sph, rgb and d_sph are not touched.
template <bool COMPACT, bool CANON, bool SPH>
__global__ void __launch_bounds__(kPbThreads) project_backward_kernel(FrameCamera cam, int64_t n, const float* __restrict__ particles,
                                                                      const float* __restrict__ sph, int deg, const float* __restrict__ rgb,
                                                                      const uint32_t* __restrict__ tiles_count, const float* __restrict__ rays_o,
                                                                      float* __restrict__ grad_acc, float* __restrict__ d_particles,
                                                                      float* __restrict__ d_sph) {
    __shared__ __align__(128) float4 s_acc[kPbThreads * kAccVec];   // in: accumulator rows, out: zeros
    __shared__ __align__(128) float4 s_sh[kPbThreads * 12];   // in: SH coefficients, out: d_sph rows
    __shared__ __align__(128) float4 s_dp[kPbThreads * 3];    // out: d_particles rows
    __shared__ __align__(8) uint64_t s_bar;
    const int tid = threadIdx.x;
    const int64_t base = static_cast<int64_t>(blockIdx.x) * kPbThreads;
    const int cnt = static_cast<int>(min(static_cast<int64_t>(kPbThreads), n - base));
    if (tid == 0) {
        mbar_init(&s_bar, kPbThreads);
        fence_proxy_async();
    }
    __syncthreads();
    const int64_t i = base + tid;
    const bool in_range = tid < cnt;
    const bool vis = in_range && (tiles_count[i] != 0u);
    const bool want_sh = SPH && vis && (deg > 0);
    mbar_expect_tx(&s_bar, (tid == 0 ? static_cast<uint32_t>(cnt) * kAccBytes : 0u) + (want_sh ? 192u : 0u));
    if (tid == 0) tma_bulk_g2s(s_acc, grad_acc + base * kGradRow, static_cast<uint32_t>(cnt) * kAccBytes, &s_bar);
    if (want_sh) tma_bulk_g2s(s_sh + tid * 12, sph + i * 48, 192u, &s_bar);
    // overlap the remaining scalar loads with the bulk copies
    float4 p = make_float4(0.f, 0.f, 0.f, 0.f), pq = p, ps = p;
    float c0 = 0.f, c1 = 0.f, c2 = 0.f;
    if (vis) {
        p = __ldg(reinterpret_cast<const float4*>(particles + i * 12));
        if (CANON) {
            pq = __ldg(reinterpret_cast<const float4*>(particles + i * 12) + 1);
            ps = __ldg(reinterpret_cast<const float4*>(particles + i * 12) + 2);
        }
        if (SPH) { c0 = rgb[i * 3 + 0]; c1 = rgb[i * 3 + 1]; c2 = rgb[i * 3 + 2]; }
    }
    float ofx = 0.f, ofy = 0.f, ofz = 0.f;
    if (CANON) {  // world-space origin of the frame's first ray, as G7 computes it (frame_common_origin)
        const float ax = rays_o[0], ay = rays_o[1], az = rays_o[2];
        const float* m = cam.s2w;
        ofx = m[0] * ax + m[3] * ay + m[6] * az + m[9];
        ofy = m[1] * ax + m[4] * ay + m[7] * az + m[10];
        ofz = m[2] * ax + m[5] * ay + m[8] * az + m[11];
    }
    mbar_wait(&s_bar, 0);

    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    if (in_range) {
        float4 a0 = s_acc[tid * kAccVec + 0], a1 = s_acc[tid * kAccVec + 1], a2 = s_acc[tid * kAccVec + 2];
        float4 a3 = s_acc[tid * kAccVec + 3];
        const float4 a4 = s_acc[tid * kAccVec + 4];
#pragma unroll
        for (int k = 0; k < kAccVec; ++k) s_acc[tid * kAccVec + k] = zero;
        if (CANON) {
            const float w00 = a1.x, w01 = a1.y, w02 = a1.z, w10 = a1.w, w11 = a2.x, w12 = a2.y, w20 = a2.z, w21 = a2.w, w22 = a3.x;
            a3 = make_float4(a3.y, a3.z, a3.w, 0.f);                                            // d rgb to the legacy position
            a1 = zero;
            a2 = zero;
            if (vis) {
                const float r = pq.x, x = pq.y, y = pq.z, z = pq.w;
                const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, xz = x * z, yz = y * z;
                const float rx = r * x, ry = r * y, rz = r * z;
                const float r0x = 1.f - 2.f * (yy + zz), r0y = 2.f * (xy + rz), r0z = 2.f * (xz - ry);
                const float r1x = 2.f * (xy - rz), r1y = 1.f - 2.f * (xx + zz), r1z = 2.f * (yz + rx);
                const float r2x = 2.f * (xz + ry), r2y = 2.f * (yz - rx), r2z = 1.f - 2.f * (xx + yy);
                const float isx = 1.0f / ps.x, isy = 1.0f / ps.y, isz = 1.0f / ps.z;
                const float pcx = ofx - p.x, pcy = ofy - p.y, pcz = ofz - p.z;                      // gposc of the frame origin
                const float gox = isx * (r0x * pcx + r0y * pcy + r0z * pcz);                        // gro of the frame origin
                const float goy = isy * (r1x * pcx + r1y * pcy + r1z * pcz);
                const float goz = isz * (r2x * pcx + r2y * pcy + r2z * pcz);
                const float prx = isx * a0.x, pry = isy * a0.y, prz = isz * a0.z;                   // gposcrGrd = S^-1 sum groGrd
                a0.x = -(prx * r0x + pry * r1x + prz * r2x);                                        // gposcr = R gposc  (gaussianParticles.cuh:715-726)
                a0.y = -(prx * r0y + pry * r1y + prz * r2y);
                a0.z = -(prx * r0z + pry * r1z + prz * r2z);
                // d scale: depth part - grdu_i rayDirRGrd_i (= (R_i . W_i) / s_i^2, :733-738) - gro_i gposcrGrd_i (gposcr/s^2 = gro/s, :705-713)
                a2.x = a4.x - isx * isx * (r0x * w00 + r0y * w01 + r0z * w02) - gox * prx;
                a2.y = a4.y - isy * isy * (r1x * w10 + r1y * w11 + r1z * w12) - goy * pry;
                a2.z = a4.z - isz * isz * (r2x * w20 + r2y * w21 + r2z * w22) - goz * prz;
                // rotation rows receive  rayDirRGrd_i d + gposcrGrd_i (o - mu) = (W_i + G_i (o_f - mu)) / s_i;  matmul_bw_quat (:719-747)
                const float m00 = isx * w00 + prx * pcx, m01 = isx * w01 + prx * pcy, m02 = isx * w02 + prx * pcz;
                const float m10 = isy * w10 + pry * pcx, m11 = isy * w11 + pry * pcy, m12 = isy * w12 + pry * pcz;
                const float m20 = isz * w20 + prz * pcx, m21 = isz * w21 + prz * pcy, m22 = isz * w22 + prz * pcz;
                a1.x = 2.f * (z * (m01 - m10) + y * (m20 - m02) + x * (m12 - m21));
                a1.y = 2.f * (y * (m01 + m10) + z * (m02 + m20) + r * (m12 - m21)) - 4.f * x * (m11 + m22);
                a1.z = 2.f * (x * (m01 + m10) + r * (m20 - m02) + z * (m12 + m21)) - 4.f * y * (m00 + m22);
                a1.w = 2.f * (r * (m01 - m10) + x * (m02 + m20) + y * (m12 + m21)) - 4.f * z * (m00 + m11);
            }
        }
        float dpx = a0.x, dpy = a0.y, dpz = a0.z;
        float4* row = s_sh + tid * 12;
        if (!SPH) {
        } else if (!vis) {
#pragma unroll
            for (int k = 0; k < 12; ++k) row[k] = zero;
        } else {
            // incident direction = normalize(position - sensor position) (gutProjector.cuh:418)
            const float vx = p.x - cam.cam_pos[0], vy = p.y - cam.cam_pos[1], vz = p.z - cam.cam_pos[2];
            const float len = sqrtf(vx * vx + vy * vy + vz * vz);
            const float inv_len = len > 0.f ? 1.0f / len : 0.f;
            const float x = len > 0.f ? vx * inv_len : 1.f, y = vy * inv_len, z = vz * inv_len;
            // clamp mask of max(f + 0.5, 0) (sphericalHarmonics.slang:63); rgb holds the unclamped f + 0.5
            const float mgr = c0 > 0.f ? a3.x : 0.f, mgg = c1 > 0.f ? a3.y : 0.f, mgb = c2 > 0.f ? a3.z : 0.f;
            float bs[16];
            sh_basis16(deg, x, y, z, bs);
            if (deg > 0 && len > 0.f) {
                // s[j] = sum_c coeff[j][c] * masked_grad[c]; then d(rgb)/d(direction) . grad, then through normalize
                // (gaussianParticles.slang:545-558)
                float cf[48];
#pragma unroll
                for (int k = 0; k < 12; ++k) {
                    const float4 v = row[k];
                    cf[k * 4] = v.x; cf[k * 4 + 1] = v.y; cf[k * 4 + 2] = v.z; cf[k * 4 + 3] = v.w;
                }
                float sc[16];
#pragma unroll
                for (int k = 0; k < 16; ++k) sc[k] = cf[k * 3] * mgr + cf[k * 3 + 1] * mgg + cf[k * 3 + 2] * mgb;
                const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                float gx = -kC1 * sc[3], gy = -kC1 * sc[1], gz = kC1 * sc[2];
                if (deg > 1) {
                    gx += kC2[0] * y * sc[4] + kC2[2] * (-2.f * x) * sc[6] + kC2[3] * z * sc[7] + kC2[4] * (2.f * x) * sc[8];
                    gy += kC2[0] * x * sc[4] + kC2[1] * z * sc[5] + kC2[2] * (-2.f * y) * sc[6] + kC2[4] * (-2.f * y) * sc[8];
                    gz += kC2[1] * y * sc[5] + kC2[2] * (4.f * z) * sc[6] + kC2[3] * x * sc[7];
                    if (deg > 2) {
                        gx += kC3[0] * (6.f * xy) * sc[9] + kC3[1] * yz * sc[10] + kC3[2] * (-2.f * xy) * sc[11] + kC3[3] * (-6.f * xz) * sc[12] +
                              kC3[4] * (4.f * zz - 3.f * xx - yy) * sc[13] + kC3[5] * (2.f * xz) * sc[14] + kC3[6] * (3.f * xx - 3.f * yy) * sc[15];
                        gy += kC3[0] * (3.f * xx - 3.f * yy) * sc[9] + kC3[1] * xz * sc[10] + kC3[2] * (4.f * zz - xx - 3.f * yy) * sc[11] +
                              kC3[3] * (-6.f * yz) * sc[12] + kC3[4] * (-2.f * xy) * sc[13] + kC3[5] * (-2.f * yz) * sc[14] +
                              kC3[6] * (-6.f * xy) * sc[15];
                        gz += kC3[1] * xy * sc[10] + kC3[2] * (8.f * yz) * sc[11] + kC3[3] * (6.f * zz - 3.f * xx - 3.f * yy) * sc[12] +
                              kC3[4] * (8.f * xz) * sc[13] + kC3[5] * (xx - yy) * sc[14];
                    }
                }
                const float dd = x * gx + y * gy + z * gz;
                dpx += (gx - x * dd) * inv_len;
                dpy += (gy - y * dd) * inv_len;
                dpz += (gz - z * dd) * inv_len;
            }
            if (COMPACT) {
                row[0] = make_float4(mgr, mgg, mgb, 0.f);
            } else {
                float o[48];  // d SH = basis x masked gradient
#pragma unroll
                for (int k = 0; k < 16; ++k) {
                    o[k * 3 + 0] = bs[k] * mgr;
                    o[k * 3 + 1] = bs[k] * mgg;
                    o[k * 3 + 2] = bs[k] * mgb;
                }
#pragma unroll
                for (int k = 0; k < 12; ++k) row[k] = make_float4(o[k * 4], o[k * 4 + 1], o[k * 4 + 2], o[k * 4 + 3]);
            }
        }
        s_dp[tid * 3 + 0] = make_float4(dpx, dpy, dpz, a0.w);
        s_dp[tid * 3 + 1] = a1;
        s_dp[tid * 3 + 2] = make_float4(a2.x, a2.y, a2.z, 0.f);
    }
    if (SPH && COMPACT) {  // pack the 16-byte radiance gradients of the block contiguously (front of s_sh) for one bulk store
        const float4 mine = in_range ? s_sh[tid * 12] : zero;
        __syncthreads();
        s_sh[tid] = mine;
    }
    fence_proxy_async();  // our shared-memory writes must be visible to the TMA engine
    __syncthreads();
    if (tid == 0) {
        if (SPH && COMPACT)
            tma_bulk_s2g(d_sph + base * 4, s_sh, static_cast<uint32_t>(cnt) * 16u);
        else if (SPH)
            tma_bulk_s2g(d_sph + base * 48, s_sh, static_cast<uint32_t>(cnt) * 192u);
        tma_bulk_s2g(d_particles + base * 12, s_dp, static_cast<uint32_t>(cnt) * 48u);
        tma_bulk_s2g(grad_acc + base * kGradRow, s_acc, static_cast<uint32_t>(cnt) * kAccBytes);
        tma_commit_group();
        tma_wait_group_read0();  // shared memory must stay valid until the engine has read it
    }
}

// d_sph[p] = sum over views v of basis(direction of particle p seen from view v) x radiance gradient of view v (the rows the
// non-compact G8 of each view would have written, summed in view order -- the same order on every rank).
struct ViewPositions {
    float pos[64][3];
};

__global__ void __launch_bounds__(128) sph_from_views_kernel(int64_t n, const float* __restrict__ particles, int deg, int views, ViewPositions vp,
                                                              const float4* __restrict__ d_radiance_all, float4* __restrict__ d_sph) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = __ldg(reinterpret_cast<const float4*>(particles + i * 12));
    float o[48];
#pragma unroll
    for (int k = 0; k < 48; ++k) o[k] = 0.f;
    for (int v = 0; v < views; ++v) {
        const float4 g = __ldg(d_radiance_all + static_cast<int64_t>(v) * n + i);
        if (g.x == 0.f && g.y == 0.f && g.z == 0.f) continue;  // invisible in that view (or clamped): a zero row
        const float vx = p.x - vp.pos[v][0], vy = p.y - vp.pos[v][1], vz = p.z - vp.pos[v][2];
        const float len = sqrtf(vx * vx + vy * vy + vz * vz);
        const float inv_len = len > 0.f ? 1.0f / len : 0.f;
        const float x = len > 0.f ? vx * inv_len : 1.f, y = vy * inv_len, z = vz * inv_len;
        float bs[16];
        sh_basis16(deg, x, y, z, bs);
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            o[k * 3 + 0] += bs[k] * g.x;
            o[k * 3 + 1] += bs[k] * g.y;
            o[k * 3 + 2] += bs[k] * g.z;
        }
    }
    float4* row = d_sph + i * 12;
#pragma unroll
    for (int k = 0; k < 12; ++k) row[k] = make_float4(o[k * 4], o[k * 4 + 1], o[k * 4 + 2], o[k * 4 + 3]);
}

}  // namespace

void launch_render_forward(cudaStream_t s, const FrameCamera& cam, const FrameConfig& cfg, const float* rays_o,
                           const float* rays_d, const float* particles, const float* rgb, const uint32_t* sorted_values,
                           const uint32_t* ranges, const uint32_t* tile_order, const uint32_t* chunk_base, uint32_t* hit_words, float* out_rgba,
                           float* out_dist, float* out_hits) {
    const unsigned grid = cam.grid_x * cam.grid_y;
    if (cfg.kernel_degree == 4)
        render_forward_kernel<4, false><<<grid, kTilePixels, 0, s>>>(cam, cfg, rays_o, rays_d, particles, rgb, sorted_values, ranges, tile_order, chunk_base, hit_words, out_rgba, out_dist, out_hits, nullptr);
    else
        render_forward_kernel<2, false><<<grid, kTilePixels, 0, s>>>(cam, cfg, rays_o, rays_d, particles, rgb, sorted_values, ranges, tile_order, chunk_base, hit_words, out_rgba, out_dist, out_hits, nullptr);
}

// debug: the forward's list walk with work counters (see WorkCounters); writes no image, rewrites the same hit words
void launch_count_work(cudaStream_t s, const FrameCamera& cam, const FrameConfig& cfg, const float* rays_o, const float* rays_d,
                       const float* particles, const float* rgb, const uint32_t* sorted_values, const uint32_t* ranges,
                       const uint32_t* tile_order, const uint32_t* chunk_base, uint32_t* hit_words, unsigned long long* counters8) {
    const unsigned grid = cam.grid_x * cam.grid_y;
    WorkCounters* ctr = reinterpret_cast<WorkCounters*>(counters8);
    if (cfg.kernel_degree == 4)
        render_forward_kernel<4, true><<<grid, kTilePixels, 0, s>>>(cam, cfg, rays_o, rays_d, particles, rgb, sorted_values, ranges, tile_order, chunk_base, hit_words, nullptr, nullptr, nullptr, ctr);
    else
        render_forward_kernel<2, true><<<grid, kTilePixels, 0, s>>>(cam, cfg, rays_o, rays_d, particles, rgb, sorted_values, ranges, tile_order, chunk_base, hit_words, nullptr, nullptr, nullptr, ctr);
}

void launch_render_backward(cudaStream_t s, const FrameCamera& cam, const FrameConfig& cfg, const float* rays_o,
                            const float* rays_d, const float* particles, const float* rgb, const uint32_t* sorted_values,
                            const uint32_t* ranges, const uint32_t* tile_order, const uint32_t* chunk_base, const uint32_t* hit_words,
                            const float* out_rgba, const float* d_rgba, const float* out_dist, const float* d_dist, float* grad_acc) {
    const unsigned grid = cam.grid_x * cam.grid_y;
    // sub-block width of the backward walk: bits 4..5 of the switch (0 = default quarter-warps, 1 = half-warps, 2 = whole warp;
    // check_args rejects 3)
    const int sub = (cfg.subtile_culling >> 4) & 3;
#define GUT_BWD(DEG_, SUB_) render_backward_kernel<DEG_, SUB_><<<grid, kTilePixels, 0, s>>>(cam, cfg, rays_o, rays_d, particles, rgb, sorted_values, ranges, tile_order, chunk_base, hit_words, out_rgba, d_rgba, out_dist, d_dist, grad_acc)
    if (cfg.kernel_degree == 4) {
        if (sub == 2) GUT_BWD(4, 32); else if (sub == 1) GUT_BWD(4, 16); else GUT_BWD(4, 8);
    } else {
        if (sub == 2) GUT_BWD(2, 32); else if (sub == 1) GUT_BWD(2, 16); else GUT_BWD(2, 8);
    }
#undef GUT_BWD
}

void launch_project_backward(cudaStream_t s, const FrameCamera& cam, int64_t n, const float* particles, const float* sph,
                             int sph_degree, const float* rgb, const uint32_t* tiles_count, const float* rays_o, float* grad_acc,
                             float* d_particles, float* d_sph, bool compact, bool canon, bool radiance) {
    if (n <= 0) return;
    const unsigned blocks = static_cast<unsigned>((n + kPbThreads - 1) / kPbThreads);
    if (!radiance)
        project_backward_kernel<false, true, false><<<blocks, kPbThreads, 0, s>>>(cam, n, particles, nullptr, 0, nullptr, tiles_count, rays_o, grad_acc, d_particles, nullptr);
    else if (compact && canon)
        project_backward_kernel<true, true, true><<<blocks, kPbThreads, 0, s>>>(cam, n, particles, sph, sph_degree, rgb, tiles_count, rays_o, grad_acc, d_particles, d_sph);
    else if (compact)
        project_backward_kernel<true, false, true><<<blocks, kPbThreads, 0, s>>>(cam, n, particles, sph, sph_degree, rgb, tiles_count, rays_o, grad_acc, d_particles, d_sph);
    else if (canon)
        project_backward_kernel<false, true, true><<<blocks, kPbThreads, 0, s>>>(cam, n, particles, sph, sph_degree, rgb, tiles_count, rays_o, grad_acc, d_particles, d_sph);
    else
        project_backward_kernel<false, false, true><<<blocks, kPbThreads, 0, s>>>(cam, n, particles, sph, sph_degree, rgb, tiles_count, rays_o, grad_acc, d_particles, d_sph);
}

void launch_sph_from_views(cudaStream_t s, int64_t n, const float* particles, int sph_degree, int views, const float* view_positions /*host [views,3]*/,
                           const float* d_radiance_all, float* d_sph) {
    if (n <= 0) return;
    ViewPositions vp;
    for (int v = 0; v < views; ++v)
        for (int k = 0; k < 3; ++k) vp.pos[v][k] = view_positions[v * 3 + k];
    const unsigned blocks = static_cast<unsigned>((n + 127) / 128);
    sph_from_views_kernel<<<blocks, 128, 0, s>>>(n, particles, sph_degree, views, vp, reinterpret_cast<const float4*>(d_radiance_all),
                                                 reinterpret_cast<float4*>(d_sph));
}

}  // namespace gutb200
