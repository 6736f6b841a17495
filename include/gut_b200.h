/*
 * include/gut_b200.h -- C ABI of the H100-native (sm_90a) 3DGUT renderer (lib: 3dgrut_b200/libgut_b200.so).
 *
 * Drop-in boundary.  The reference's FFI for this path is pybind11 + ATen, not extern "C"
 * (threedgut_tracer/bindings.cpp:103-109): class SplatRaster{trace, trace_bwd, collect_times}.
 * This header is the raw-pointer core a maintainer binds instead (see INTEGRATION.md): every entry
 * point takes plain device/host pointers, sizes and a cudaStream_t passed as void*; no torch types.
 *
 *   gutb200_create / destroy      <- SplatRaster::SplatRaster / ~SplatRaster   (threedgut_tracer/src/splatRaster.cpp:163-182)
 *   gutb200_forward               <- SplatRaster::trace                         (src/splatRaster.cpp:184-262) -> GUTRenderer::renderForward (src/gutRenderer.cu:241-421)
 *   gutb200_backward              <- SplatRaster::traceBwd                      (src/splatRaster.cpp:264-350) -> GUTRenderer::renderBackward (src/gutRenderer.cu:423-519)
 *   gutb200_collect_times         <- SplatRaster::collectTimes                  (src/splatRaster.cpp:352-382)
 *   gutb200_forward_host/_backward_host : same calls with HOST buffers (copies inside), used for the e2e metric.
 *   gutb200_backward_compact / gutb200_sph_grad_from_views / gutb200_camera_position : view-parallel training (no reference twin).
 *   gutb200_debug_copy            : test-only read-back of the binning artefacts (tile counts, sort keys, ranges).
 *
 * Data layouts (all fp32 unless noted; identical to the reference tensors):
 *   particles [N,12] = pos3, density, quat(w,x,y,z), scale3, pad     (threedgut_tracer/tracer.py:176-178)
 *   sph       [N,48] = 16 SH coefficients x rgb                       (gaussianParticles.cuh:208-221)
 *   rays_o/d  [H,W,3] sensor space                                    (tracer.py:317-330)
 *   out_rgba  [H,W,4], out_dist [H,W], out_hits [H,W], visibility [N] (src/splatRaster.cpp:212-216)
 *   d_particles [N,12], d_sph [N,48]                                  (src/splatRaster.cpp:291-293)
 * Errors: every call returns 0 on success, non-zero on failure; gutb200_last_error() gives the message
 * (the reference logs and drops its Status codes, src/splatRaster.cpp:242,254; we surface them).  Given NULL, it gives the message of
 * the last failed call on this thread that takes no context and records one (gutb200_image_loss), else "null context".
 */
#ifndef GUT_B200_H
#define GUT_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* OpenCV pinhole + global shutter (CameraModelParameters, include/3dgut/sensors/cameraModels.h:22-72).
 * Poses are world->sensor [t.xyz, q.xyzw] at shutter open / close (include/3dgut/sensors/sensors.h:33-42). */
typedef struct gutb200_camera {
    int32_t width, height;
    float principal[2];
    float focal[2];
    float radial[6];
    float tangential[2];
    float thin_prism[4];
    float pose_start[7];
    float pose_end[7];
    int32_t model;      /* TSensorModel::ModelType (sensors/cameraModels.h:59-72): 0 = OpenCV pinhole (radial[6], tangential, thin prism),
                         * 1 = OpenCV fisheye (radial[0..3] = k1..k4, max_angle; bindings.cpp:68-84), 2 = f-theta (fields below). */
    float max_angle;    /* OpenCVFisheyeProjectionParameters::maxAngle (cameraModels.h:30-35) / FThetaProjectionParameters::maxAngle */
    /* model 2 = f-theta (FThetaProjectionParameters, cameraModels.h:37-47; bindings.cpp:86-101); principal point = principal[] */
    int32_t ftheta_reference_poly;  /* 0 PIXELDIST_TO_ANGLE, 1 ANGLE_TO_PIXELDIST */
    float ftheta_bw[6];             /* pixeldist_to_angle_poly (backward) */
    float ftheta_fw[6];             /* angle_to_pixeldist_poly (forward)  */
    float ftheta_cde[3];            /* linear_cde */
    int32_t rolling_shutter;        /* 0 global shutter; 1..4 = CameraModelParameters::ShutterType + 1 (cameraModels.h:49-57): rolling
                                     * top-to-bottom, left-to-right, bottom-to-top, right-to-left.  Affects the projection only
                                     * (projectPointWithShutter, cameraProjections.cuh:218-257); rays use the mid-exposure pose like the
                                     * reference (gutRenderer.cu:266-267,406). */
} gutb200_camera;

/* Render configuration == the reference's compile-time -D constants (threedgut_tracer/setup_3dgut.py:64-95). */
typedef struct gutb200_config {
    int32_t kernel_degree;    /* GAUSSIAN_PARTICLE_KERNEL_DEGREE: 2 (3DGUT default) or 4          */
    float min_kernel_density; /* GAUSSIAN_PARTICLE_MIN_KERNEL_DENSITY                              */
    float min_alpha;          /* GAUSSIAN_PARTICLE_MIN_ALPHA                                       */
    float max_alpha;          /* GAUSSIAN_PARTICLE_MAX_ALPHA                                       */
    float min_transmittance;  /* GAUSSIAN_MIN_TRANSMITTANCE_THRESHOLD                               */
    float ut_alpha, ut_beta, ut_kappa, ut_delta;
    float ut_margin;          /* GAUSSIAN_UT_IN_IMAGE_MARGIN_FACTOR                                */
    int32_t rect_bounding, tight_opacity_bounding, tile_culling;
    int32_t global_z_order;
    int32_t enable_timings;   /* render.enable_kernel_timings (src/splatRaster.cpp:168-169); 2 = also per-stage events */
    int32_t n_rolling_shutter_iterations; /* GAUSSIAN_N_ROLLING_SHUTTER_ITERATIONS (configs/render/3dgut.yaml:18): 5 */
    int32_t k_buffer_size;    /* GAUSSIAN_K_BUFFER_SIZE (render.splat.k_buffer_size): 0 = unsorted (default), 1..16 = sorted 3DGUT */
    int32_t subtile_culling;  /* ours (no reference twin), bit mask, default 7: bit 1 = exact-conservative sub-tile screens in render,
                               * bit 2 = renderBackward walks only the list entries some pixel of a sub-block accepted in the forward
                               * ("hit words"; the sub-blocks are quarter-warps, 4x2 pixels); bits 4..5 must be 0; bit 0 unused.
                               * Forward results are bit-identical with bit 1 on or off. */
} gutb200_config;

typedef struct gutb200_ctx gutb200_ctx;

void gutb200_default_config(gutb200_config* cfg);
int gutb200_create(const gutb200_config* cfg, int device, gutb200_ctx** out);
void gutb200_destroy(gutb200_ctx* ctx);
const char* gutb200_last_error(const gutb200_ctx* ctx);
const char* gutb200_version(void);

int gutb200_forward(gutb200_ctx* ctx, void* stream, const gutb200_camera* cam, int64_t n, const float* particles,
                    const float* sph, int32_t sph_degree, const float* rays_o, const float* rays_d, float* out_rgba,
                    float* out_dist, float* out_hits, float* visibility);

int gutb200_backward(gutb200_ctx* ctx, void* stream, const gutb200_camera* cam, int64_t n, const float* particles,
                     const float* sph, int32_t sph_degree, const float* rays_o, const float* rays_d,
                     const float* out_rgba, const float* d_rgba, const float* out_dist, const float* d_dist,
                     float* d_particles, float* d_sph);

/* Neural Harmonic Texture (NHT) features instead of SH radiance (model.feature_type: nht; neuralHarmonicFeaturesParticle.slang).
 * features [N,feature_dim] per particle: 4 tetrahedron vertices x 12 features, fp32 (features_half = 0) or fp16 (features_half = 1,
 * render.particle_feature_half), 16-byte aligned.  Built: feature_dim 48, barycentric interpolation, sincos activation with 1 frequency
 * -> 24 ray features.  out_features_alpha [H,W,25] = 24 features then the opacity, fp32; out_dist / out_hits / visibility as
 * gutb200_forward.  The backward replays the forward of the same camera and stream, which must be gutb200_forward_nht (and SH forwards
 * only take gutb200_backward); d_particles [N,12] as gutb200_backward, d_features [N,48] fp32 whatever the feature precision.  Every row of
 * both is written.  k_buffer_size > 0 is refused. */
int gutb200_forward_nht(gutb200_ctx* ctx, void* stream, const gutb200_camera* cam, int64_t n, const float* particles, const void* features,
                        int32_t feature_dim, int32_t features_half, const float* rays_o, const float* rays_d, float* out_features_alpha,
                        float* out_dist, float* out_hits, float* visibility);
int gutb200_backward_nht(gutb200_ctx* ctx, void* stream, const gutb200_camera* cam, int64_t n, const float* particles, const void* features,
                         int32_t feature_dim, int32_t features_half, const float* rays_o, const float* rays_d, const float* out_features_alpha,
                         const float* d_features_alpha, const float* out_dist, const float* d_dist, float* d_particles, float* d_features);

/* Host-buffer variants: pinned or pageable host pointers; H2D/D2H copies happen inside on the context's stream. */
/* View-parallel training (ours, no reference twin -- the reference is single-GPU): the [N,48] SH gradient row of a view is the outer
 * product basis16(direction particle <- sensor) x g, g = masked dL/d(radiance) of the particle in that view.  gutb200_backward_compact
 * emits g ([N,4], .w = 0) instead of the row; ranks all-gather the g's and all-reduce d_particles (16 + 48 instead of 240 bytes per
 * particle on the wire), then gutb200_sph_grad_from_views rebuilds sum_v basis(direction_v) x g_v on every rank in view order.
 * view_positions_host: [views,3] sensor positions from gutb200_camera_position (host pointers); d_radiance_all: [views,N,4] device. */
int gutb200_backward_compact(gutb200_ctx* ctx, void* stream, const gutb200_camera* cam, int64_t n, const float* particles,
                             const float* sph, int32_t sph_degree, const float* rays_o, const float* rays_d, const float* out_rgba,
                             const float* d_rgba, const float* out_dist, const float* d_dist, float* d_particles, float* d_radiance);
int gutb200_sph_grad_from_views(gutb200_ctx* ctx, void* stream, int64_t n, const float* particles, int32_t sph_degree, int32_t views,
                                const float* view_positions_host, const float* d_radiance_all, float* d_sph);
int gutb200_camera_position(const gutb200_camera* cam, float* pos3);

/* Optimizer step (SURVEY.md 8f row 2).  No context: plain launches on `stream` of the current device; 0 on success.
 * gutb200_selective_adam_update replaces selective_adam_update of the reference's optimizer plugin
 * (threedgrut/optimizers/optimizers.cu:49-108, optimizers.cpp): param/grad/exp_avg/exp_avg_sq [n,m] fp32, visibility [n] bytes
 * (bool), Adam without bias correction on the visible rows.  visibility == NULL updates every row.
 * gutb200_gaussian_adam_step (ours) updates the six raw parameter tensors of the SH model in ONE launch from the renderer's
 * gradients: params6 / exp_avg6 / exp_avg_sq6 = {positions [n,3], density [n,1], rotation [n,4], scale [n,3], features_albedo [n,3],
 * features_specular [n,45]} (device pointers in a host array), lr6 their learning rates, d_particles [n,12] and d_sph [n,48] the
 * gradients w.r.t. the ACTIVATED values as gutb200_backward writes them; the activation chain rule (sigmoid / exp / normalize,
 * threedgrut/model/model.py:102-118) is applied inside.  selective = 0: torch.optim.Adam with bias correction at `step` (>= 1,
 * model.py:807-810); selective = 1: the plugin's rule on rows with visibility != 0 (visibility = the renderer's [n] float output). */
int gutb200_selective_adam_update(void* stream, float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                                  const uint8_t* visibility, float lr, float b1, float b2, float eps, int64_t n, int64_t m);
int gutb200_gaussian_adam_step(void* stream, int64_t n, float* const* params6, float* const* exp_avg6, float* const* exp_avg_sq6,
                               const float* lr6, float b1, float b2, float eps, int64_t step, int32_t selective, const float* d_particles,
                               const float* d_sph, const float* visibility);
/* The same step with the opacity and scale regularisers of the reference loss (threedgrut/trainer.py:722-736): reg_density =
 * lambda_opacity / n is added to every d density and reg_scale = lambda_scale / (3 n) to every d scale (w.r.t. the activated values)
 * before the chain rule.  Both zero: exactly gutb200_gaussian_adam_step.  The selective rule still skips invisible rows. */
int gutb200_gaussian_adam_step_reg(void* stream, int64_t n, float* const* params6, float* const* exp_avg6, float* const* exp_avg_sq6,
                                   const float* lr6, float b1, float b2, float eps, int64_t step, int32_t selective, const float* d_particles,
                                   const float* d_sph, const float* visibility, float reg_density, float reg_scale);
/* gutb200_nht_adam_step (ours): the same one-launch step for the NHT model plus its feature decoder.  params6 / exp_avg6 / exp_avg_sq6 =
 * {positions [n,3], density [n,1], rotation [n,4], scale [n,3], features [n,48], decoder params [n_decoder]}; lr6 their learning rates;
 * steps6 each group's own Adam step count (>= 1 where bias-corrected).  The four geometry groups take the chain rule of
 * gutb200_gaussian_adam_step from d_particles [n,12]; features are raw, their gradient is d_features [n,48]; the decoder's gradient is
 * d_decoder [n_decoder] plus decoder_weight_decay x param (torch.optim.Adam weight_decay), with decoder_b1 / decoder_b2 / decoder_eps and
 * never the selective rule.  Bit k of frozen_mask freezes group k: it launches no block and its parameters and moments are not touched
 * (their pointers and gradients may then be NULL).  reg_density / reg_scale as in gutb200_gaussian_adam_step_reg (0 = none). */
int gutb200_nht_adam_step(void* stream, int64_t n, int64_t n_decoder, float* const* params6, float* const* exp_avg6,
                          float* const* exp_avg_sq6, const float* lr6, const int64_t* steps6, float b1, float b2, float eps, int32_t selective,
                          float decoder_b1, float decoder_b2, float decoder_eps, float decoder_weight_decay, int32_t frozen_mask,
                          const float* d_particles, const float* d_features, const float* d_decoder, const float* visibility, float reg_density,
                          float reg_scale);

/* Image loss of the training step and its gradient (SURVEY.md 8f row 3): loss = lambda_l1 mean|x - y| + lambda_ssim (1 - SSIM(x, y))
 * (threedgrut/trainer.py:698-739, model/losses.py:20-33 -> fused_ssim(..., padding="valid"), third-party fused-ssim @ 1272e21), on the
 * prediction composited onto a background, post-processed and multiplied by a mask (model/background.py:80-93, trainer.py:691-694,
 * 1165-1172): x = s(c) m, c = rgb + bg (1 - alpha), y = target m; d rgb = m s'(c) dL/dx, d alpha = -sum_c bg_c m s'(c_c) dL/dx_c.
 * layout 4: pred [H,W,4] rgba (the renderer's output) and d_pred [H,W,4] = d_rgba, 16-byte aligned (directly the d_rgba of
 * gutb200_backward); pred_alpha / d_alpha unused.  layout 3: pred [H,W,3] rgb + pred_alpha [H,W] and d_pred [H,W,3] = d_rgb + d_alpha
 * [H,W] (grtb200_trace's out_rgb / out_alpha and the d_rgb / d_alpha of grtb200_trace_bwd); pred_alpha is needed only with a background,
 * d_alpha only with a background, a mask or post-processing (otherwise it is zeroed when given).  background_rgb: 3 host floats or NULL
 * (black); background_image: [H,W,3] device floats or NULL (used instead of background_rgb).  mask: [H,W] device floats or NULL.
 * post_processing (post_processing.method, threedgrut/utils/post_processing_linear_to_srgb.py): 0 = none (s = identity), 1 =
 * linear-to-sRGB, s(c) = 1.055 max(c, 1e-8)^(1/2.4) - 0.055 above c = 0.0031308, 12.92 c at or below it (no clamp).
 * A black background with no mask and no post-processing is the plain loss: zero alpha gradient, and layout 3's rgb gradient is
 * bit-identical to layout 4's on the [H,W,4] concatenation of rgb and alpha.
 * sums2 [2] device floats = (sum |x - y|, sum of the SSIM map over the valid region): l1 = sums2[0] / (3 H W), ssim = sums2[1] / (3 (H-10)
 * (W-10)).  scratch: gutb200_image_loss_scratch_bytes(H, W) device bytes.  Two launches on `stream`; returns 0, 1 for bad arguments, 3 for
 * a misaligned d_pred (layout 4), 2 for a launch error, and gutb200_last_error(NULL) then names the cause. */
size_t gutb200_image_loss_scratch_bytes(int32_t height, int32_t width);
int gutb200_image_loss(void* stream, int32_t height, int32_t width, int32_t layout, const float* pred, const float* pred_alpha,
                       const float* target_rgb, const float* background_rgb, const float* background_image, const float* mask,
                       float lambda_l1, float lambda_ssim, void* scratch, float* d_pred, float* d_alpha, float* sums2, int32_t post_processing);

/* Test-set metrics of one rendered frame as the reference evaluator computes them (threedgrut/render.py:294-369, trainer.py:641-657,
 * 1350-1364), with the pixel loads of gutb200_image_loss and no mask: x = s(rgb + bg (1 - alpha)) against the target y [H,W,3].
 *   psnr = 10 log10(1 / mean (x - y)^2) over 3HW (x unclipped; +inf when x == y).  ssim: the 11-tap Gaussian window (sigma 1.5), C1 =
 *   0.01^2, C2 = 0.03^2, both variances clamped at 0, mean over the (H-10)(W-10) 3 interior (torchmetrics' SSIM with data_range 1:
 *   reflect pad 5, crop 5).  a, b per channel (threedgrut/utils/color_correct.py:96-145) from fp64 moments over all HW pixels: var =
 *   max(E[y^2] - E[y]^2, 1e-8), a = (E[xy] - E[x] E[y]) / var, b = E[x] - a E[y], then a = 1 where |a| < 1e-8; cc_psnr / cc_ssim are psnr
 *   / ssim of x_cc = clip((x - b) / a, 0, 1) (fp32, IEEE division) against y.  l1 = mean |x - y|.  hits [H,W] int32 or NULL: mean,
 *   unbiased std, min, max (NaN without hits).
 * layout, pred, pred_alpha, background_rgb and post_processing as in gutb200_image_loss (a background image is not taken: evaluation
 * composites a constant colour, and a random training background evaluates as black).  pred_u8 / target_u8: [H,W,3] device bytes or
 * NULL, x and y quantised as torchvision.utils.save_image does: trunc(clamp(fl(fl(v 255) + 0.5), 0, 255)).
 * out: GUTB200_METRICS_K device doubles in the order of the enum below.  scratch: gutb200_image_metrics_scratch_bytes(H, W) device bytes,
 * 8-byte aligned.  Four launches on `stream` (pass, finalise, colour-corrected pass, finalise), no synchronisation, no atomics: the same
 * inputs give the same bits.  Returns 0, 1 for bad arguments (H or W below 11 among them), 2 for a launch error; gutb200_last_error(NULL)
 * then names the cause. */
enum {
    GUTB200_METRIC_PSNR = 0,
    GUTB200_METRIC_SSIM = 1,
    GUTB200_METRIC_CC_PSNR = 2,
    GUTB200_METRIC_CC_SSIM = 3,
    GUTB200_METRIC_L1 = 4,
    GUTB200_METRIC_HITS_MEAN = 5,
    GUTB200_METRIC_HITS_STD = 6,
    GUTB200_METRIC_HITS_MIN = 7,
    GUTB200_METRIC_HITS_MAX = 8,
    GUTB200_METRIC_A = 9,  /* a[3] */
    GUTB200_METRIC_B = 12, /* b[3] */
    GUTB200_METRICS_K = 15
};
size_t gutb200_image_metrics_scratch_bytes(int32_t height, int32_t width);
int gutb200_image_metrics(void* stream, int32_t height, int32_t width, int32_t layout, const float* pred, const float* pred_alpha,
                          const float* target_rgb, const float* background_rgb, int32_t post_processing, const int32_t* hits, void* scratch,
                          double* out, uint8_t* pred_u8, uint8_t* target_u8);

/* 3DGRUT hybrid (ours; hybrid.py's mirror_rays and render_hybrid as device code for train_step_hybrid): primary rays through 3DGUT, one
 * mirror bounce off a plane through 3DGRT.  No context: one launch each on `stream` of the current device, no synchronisation; 0 on success.
 * gutb200_hybrid_rays: rays_o / rays_d [pixels,3] in camera space, T_to_world_host the 12 floats of the camera-to-world [R | t] (row-major
 * 3x4, host), plane_point_host / plane_normal_host 3 host floats each (unit normal) -> out_o / out_d [pixels,3] world-space secondary rays
 * and out_hit [pixels] (1 where the ray meets the plane in front of it from its front side, else 0; a ray that misses keeps its own world
 * origin and direction).  gutb200_hybrid_composite: out_rgb [pixels,3] = primary rgb + reflectivity (1 - primary alpha) hit secondary_rgb
 * from primary_rgba [pixels,4] (gutb200_forward's out_rgba, 16-byte aligned) and secondary_rgb [pixels,3] (grtb200_trace's out_rgb).
 * gutb200_hybrid_composite_bwd: from d_rgb [pixels,3] and d_alpha [pixels] (NULL = 0; the loss's gradient on the primary alpha) writes every
 * element of d_primary_rgba [pixels,4] (16-byte aligned; rgb = d_rgb, alpha = d_alpha - reflectivity hit <d_rgb, secondary_rgb>) and
 * d_secondary_rgb [pixels,3] = reflectivity (1 - primary alpha) hit d_rgb. */
int gutb200_hybrid_rays(void* stream, int64_t pixels, const float* rays_o, const float* rays_d, const float* T_to_world_host,
                        const float* plane_point_host, const float* plane_normal_host, float* out_o, float* out_d, float* out_hit);
int gutb200_hybrid_composite(void* stream, int64_t pixels, const float* primary_rgba, const float* secondary_rgb, const float* hit,
                             float reflectivity, float* out_rgb);
int gutb200_hybrid_composite_bwd(void* stream, int64_t pixels, const float* primary_rgba, const float* secondary_rgb, const float* hit,
                                 float reflectivity, const float* d_rgb, const float* d_alpha, float* d_primary_rgba, float* d_secondary_rgb);

/* Exact k nearest neighbours (ours; the initial Gaussian scales of initialization.py, DESIGN.md section 19).  targets [n_targets,3] and
 * queries [n_queries,3] float32 device arrays; queries NULL: the targets query themselves (n_queries must equal n_targets) and query i
 * excludes target i, and only it (duplicates are neighbours at distance 0).  Row q of out_idx [n_queries,k] int32 holds the k targets with
 * the smallest float32 squared distance (qx-px)^2 + (qy-py)^2 + (qz-pz)^2, ascending, ties broken by the lower target index; out_dist
 * [n_queries,k] (NULL: not written) those squared distances.  Exact and deterministic: the same inputs give the same bits on every run.
 * No context: launches on `stream` of the current device, no synchronisation.  workspace: gutb200_knn_workspace_bytes(n_targets) device
 * bytes (0 for n_targets outside 1..INT32_MAX).  Returns 1, with the message in gutb200_last_error(NULL), for k outside 1..4, fewer
 * than k + 1 targets with self-exclusion or k without, sizes above INT32_MAX, a NULL array or a workspace that is too small. */
size_t gutb200_knn_workspace_bytes(int64_t n_targets);
int gutb200_knn(void* stream, int64_t n_targets, const float* targets, int64_t n_queries, const float* queries, int32_t k, void* workspace,
                size_t workspace_bytes, int32_t* out_idx, float* out_dist);

int gutb200_forward_host(gutb200_ctx* ctx, const gutb200_camera* cam, int64_t n, const float* particles,
                         const float* sph, int32_t sph_degree, const float* rays_o, const float* rays_d,
                         float* out_rgba, float* out_dist, float* out_hits, float* visibility);
int gutb200_backward_host(gutb200_ctx* ctx, const gutb200_camera* cam, int64_t n, const float* particles,
                          const float* sph, int32_t sph_degree, const float* rays_o, const float* rays_d,
                          const float* out_rgba, const float* d_rgba, const float* out_dist, const float* d_dist,
                          float* d_particles, float* d_sph);

/* Statistics of the last forward: N, I (= particle/tile intersections), V (= particles with tiles_count>0), T tiles. */
int gutb200_last_stats(gutb200_ctx* ctx, int64_t* n, int64_t* num_intersections, int64_t* num_visible, int64_t* num_tiles);

/* Test-only read-back (synchronises).  `what`: */
enum {
    GUTB200_DBG_TILES_COUNT = 0,   /* u32 [N]   */
    GUTB200_DBG_SORTED_KEYS = 1,   /* u64 [I]   */
    GUTB200_DBG_SORTED_VALUES = 2, /* u32 [I]   */
    GUTB200_DBG_TILE_RANGES = 3,   /* u32 [T,2] */
    GUTB200_DBG_DEPTH = 4,         /* f32 [N]   */
    GUTB200_DBG_RGB = 5,           /* f32 [N,3] (unclamped precomputed radiance) */
    GUTB200_DBG_PROJ = 6           /* f32 [N,8] = centre2, extent2, conic3, opacity */
};
int gutb200_debug_copy(gutb200_ctx* ctx, int what, void* host_dst, size_t bytes);

/* Mean device time (ms) of the forward / backward calls since the last collect (needs enable_timings). */
int gutb200_collect_times(gutb200_ctx* ctx, float* forward_ms, float* backward_ms);

/* Change the timing level of a live context: 0 off, 1 forward/backward events, 2 also per-stage events. */
int gutb200_set_timings(gutb200_ctx* ctx, int level);

/* Mean device time (ms) per stage since the last collect (needs enable_timings >= 2); order:
 * project, scan, expand, sort, tile_ranges, render, render_backward, project_backward. */
int gutb200_collect_stage_times(gutb200_ctx* ctx, float* mean_ms /*[8]*/);

/* Measurement helpers (debug, synchronise; never on the render path).
 * work counters of the last forward (unsorted path): counters16 = { tests_ref: (pixel, entry) pairs the reference's per-pixel loop
 * evaluates, tests_exec: lane-level exact tests our forward ran after sub-tile screening, hits: accepted pairs (the adjoint's work),
 * fwd_iters / hit_iters: warp iterations of the forward / of the backward, screens: lane-level sub-tile screens, bwd_lanes: live lanes
 * summed over those, iters16 / iters8: backward iterations when half- / quarter-warps walk their own entries in lockstep, sub16_hits /
 * sub8_hits: (half- / quarter-warp, entry) pairs with a hit = gradient rows flushed, 0... }.  particles / rays_* are the device pointers
 * the forward was called with. */
int gutb200_debug_work_counters(gutb200_ctx* ctx, const float* particles, const float* rays_o, const float* rays_d, uint64_t* counters16);
/* FP32 FMA throughput of the device in TFLOP/s (micro-benchmark, best of `repeats` launches): the roofline_fp32 denominator. */
int gutb200_debug_fma_peak(gutb200_ctx* ctx, int repeats, float* tflops);

/* Number of kernels this library launched since the context was created (bench.py's gpu_launches). */
int64_t gutb200_launch_count(const gutb200_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif
