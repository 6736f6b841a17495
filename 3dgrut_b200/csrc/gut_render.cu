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
// G6 forward: the shared walk (render_tile.cuh) with the radiance payload.
// staged record, 5 x float4: FwdRecords (rows of M = diag(1/s) R^T with the particle position in .w, then (s, density)), then (rgb)

struct FwdSmem : FwdRecords<kBatch> {
    float4 col[kBatch];
};

struct RadiancePayload {
    float4* col;
    const float* __restrict__ rgb;
    float cr = 0.f, cg = 0.f, cb = 0.f;
    __device__ __forceinline__ void entry(int slot, uint32_t idx) {
        col[slot] = make_float4(fmaxf(rgb[idx * 3 + 0], 0.f), fmaxf(rgb[idx * 3 + 1], 0.f), fmaxf(rgb[idx * 3 + 2], 0.f), 0.f);
    }
    __device__ __forceinline__ void batch(const uint32_t* __restrict__, uint32_t, int, int) {}
    __device__ __forceinline__ void add(int j, float w, float, float, float) {
        const float4 c = col[j];
        cr += c.x * w;
        cg += c.y * w;
        cb += c.z * w;
    }
};

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
    const int tid = threadIdx.x;
    const TileRay tr = tile_ray(cam, rays_o, rays_d, tile_order, tid);
    RadiancePayload pay{sm.col, rgb};
    float T = 1.f, dist = 0.f;
    uint32_t hits = 0;
    forward_list<DEG, COUNT>(cam, cfg, sm, pay, tr, tid, rays_o, particles, sorted_values, ranges, chunk_base, hit_words, T, dist, hits, ctr);
    if (COUNT) return;  // the counting pass leaves the frame's outputs alone

    const int64_t pix = tr.pix;
    if (tr.valid) {  // finalizeRay (rayPayload.cuh:160-193); invalid rays keep the initial buffer values
        reinterpret_cast<float4*>(out_rgba)[pix] = make_float4(pay.cr, pay.cg, pay.cb, 1.0f - T);
        out_dist[pix] = dist;
        out_hits[pix] = static_cast<float>(hits);
    } else if (tr.inside) {
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
// staged record, 6 x float4: BwdRecords (r0, r1, r2, sc, is; render_tile.cuh), then cl = clamped rgb, particle index bits.
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

struct BwdSmem : BwdRecords<kBatch> {
    float4 cl[kBatch];
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


// per-pixel backward state (initializeBackwardRay, kernels/cuda/common/rayPayloadBackward.cuh:31-73)
struct BwdRay {
    float Cix, Ciy, Ciz, Cgx, Cgy, Cgz, Tint, Tgrad, Dint, Dgrad;
    float T, Cx, Cy, Cz, D;
};

// the radiance terms of backward_pair (render_tile.cuh): g[13..15] = d rgb, depth slots 16..18
struct RadianceHit {
    static constexpr int kDepthSlot = 16;
    static constexpr bool kHitPoint = false;
    float4 cl;
    __device__ __forceinline__ void at_hit(const BwdSmem& sm, int j, const BwdRay&, float, float, float, float, float (&)[19]) { cl = sm.cl[j]; }
    // radiance branch (:602-612)
    __device__ __forceinline__ float common(const FrameConfig&, BwdRay& st, float T, float weight, float inv_next, float, float partial,
                                            float (&g)[19]) {
        g[13] = st.Cgx * weight; g[14] = st.Cgy * weight; g[15] = st.Cgz * weight;
        st.Cx += weight * cl.x; st.Cy += weight * cl.y; st.Cz += weight * cl.z;
        const float rcx = fmaxf((st.Cix - st.Cx) * inv_next, 0.f);
        const float rcy = fmaxf((st.Ciy - st.Cy) * inv_next, 0.f);
        const float rcz = fmaxf((st.Ciz - st.Cz) * inv_next, 0.f);
        return partial + T * ((cl.x - rcx) * st.Cgx + (cl.y - rcy) * st.Cgy + (cl.z - rcz) * st.Cgz);
    }
};

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
    backward_batches<FAST>(sm, sm.hw, ofx, ofy, ofz, tid, begin, end, particles, sorted_values, hit_words, use_words, alive,
        [&](uint32_t idx) {
            sm.cl[tid] = make_float4(fmaxf(rgb[idx * 3 + 0], 0.f), fmaxf(rgb[idx * 3 + 1], 0.f), fmaxf(rgb[idx * 3 + 2], 0.f), __uint_as_float(idx));
        },
        [](uint32_t, int) {},
        [&](int count) {
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
                float g[19];
#pragma unroll
                for (int i = 0; i < 19; ++i) g[i] = 0.f;
                bool hit = false;
                if (act && alive) hit = backward_pair<DEG, FAST, RadianceHit>(cfg, sm, j, ray, dox, doy, doz, depth_grads, st, alive, g);
                const unsigned hits = __ballot_sync(kFull, hit);
                if (hits) {
                    float4* mine = rows + lane * (kGradRow / 4);
                    mine[0] = make_float4(g[0], g[1], g[2], g[3]);
                    mine[1] = make_float4(g[4], g[5], g[6], g[7]);
                    mine[2] = make_float4(g[8], g[9], g[10], g[11]);
                    mine[3] = make_float4(g[12], g[13], g[14], g[15]);
                    if (depth_grads) mine[4] = make_float4(g[16], g[17], g[18], 0.f);  // warp-uniform
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
    });
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
    const int tid = threadIdx.x;
    const TileRay tr = tile_ray(cam, rays_o, rays_d, tile_order, tid);
    const int64_t pix = tr.pix;

    BwdRay st;
    st.Cix = st.Ciy = st.Ciz = st.Cgx = st.Cgy = st.Cgz = 0.f;
    st.Tint = 1.f; st.Tgrad = 0.f; st.Dint = 0.f; st.Dgrad = 0.f;
    st.T = 1.f; st.Cx = st.Cy = st.Cz = st.D = 0.f;
    if (tr.valid) {
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
    const bool fast = frame_common_origin(cam, rays_o, tr.inside, pix, ofx, ofy, ofz);
    const uint32_t begin = ranges[tr.tile * 2], end = ranges[tr.tile * 2 + 1];
    const uint32_t* words = hit_words + static_cast<size_t>(chunk_base[tr.tile]) * kWordsPerChunk;
    const bool use_words = (cfg.subtile_culling & 4) != 0;
    if (fast)
        backward_tile<DEG, true, SUBL>(cfg, sm, tr.ray, ofx, ofy, ofz, tid, tid & 31, begin, end, particles, rgb, sorted_values, words, use_words, tr.valid, st, grad_acc);
    else
        backward_tile<DEG, false, SUBL>(cfg, sm, tr.ray, ofx, ofy, ofz, tid, tid & 31, begin, end, particles, rgb, sorted_values, words, use_words, tr.valid, st, grad_acc);
}

// ----------------------------------------------------------------------------------------------------------
// G8 per-particle SH adjoint + emission of the final gradient rows; re-zeroes the accumulator for the next frame.

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
                // rotation_rows (render_tile.cuh) written out: routed through the helper this kernel compiles to different SASS
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
