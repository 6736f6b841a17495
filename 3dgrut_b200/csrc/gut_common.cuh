// 3dgrut_b200/csrc/gut_common.cuh -- shared device/host declarations of the 3DGUT renderer.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/gut_b200.h"

namespace gutb200 {

constexpr int kTile         = 16;   // GUTParameters::Tiling::BlockX/Y (gutRendererParameters.h:22-25): part of the key format
constexpr int kTilePixels   = kTile * kTile;
constexpr uint32_t kInvalid = 0xFFFFFFFFu;

// Per-frame camera block handed to every kernel by value (lives in the constant bank of the launch).
struct FrameCamera {
    int width, height, grid_x, grid_y;
    float fx, fy, cx, cy;
    float radial[6], tangential[2], thin_prism[4];
    float rot_start[9];   // column-major world->sensor rotation at shutter open (cameraProjections.cuh:225-229)
    float t_start[3];
    float view[12];       // world->sensor at mid exposure, 4 columns x 3 (gutRenderer.cu:266,284)
    float s2w[12];        // sensor->world at mid exposure (gutRenderer.cu:267,406)
    float cam_pos[3];     // sensor position in world space (gutRenderer.cu:282)
    float res_x, res_y;   // float copies of width/height
    int has_distortion;   // any radial / tangential / thin-prism coefficient non-zero
    int model;            // 0 OpenCV pinhole, 1 OpenCV fisheye (radial[0..3] = k1..k4), 2 f-theta
    float max_angle;      // fisheye / f-theta: half-angle of the valid cone
    int ft_reference_poly;          // f-theta (model 2): 0 backward polynomial is the reference, 1 forward
    float ft_bw[6], ft_fw[6], ft_cde[3];
    // rolling shutter (projectPointWithShutter, cameraProjections.cuh:218-257): 0 global, 1..4 = readout top-to-bottom, left-to-right,
    // bottom-to-top, right-to-left; poses at shutter open / close as quaternion (wxyz) + translation
    int rolling_shutter, rs_iterations;
    float q_start[4], q_end[4], t_end[3];
};

struct FrameConfig {
    int kernel_degree;
    float min_kernel_density, min_alpha, max_alpha, min_transmittance;
    float ut_delta, ut_margin;
    float w0_mean, wi, w0_cov;   // unscented-transform weights (gutProjector.cuh:150,163,201)
    int rect_bounding, tight_opacity_bounding, tile_culling, global_z_order;
    int subtile_culling;   // ours: conservative per-warp / per-pixel conic pre-test in the render kernels (gut_render.cu)
    int k_buffer_size;     // GAUSSIAN_K_BUFFER_SIZE: 0 (default) or 1..16 = sorted 3DGUT (gut_render_kbuffer.cu)
};

// Projection result of one particle consumed by the expand kernel: centre, extent, conic, opacity (32 B).
struct __align__(16) ProjRecord {
    float cx, cy, ex, ey;
    float ca, cb, cc, op;
};

// Gradient accumulator row (80 B), filled with vector REDs by G7 and consumed + re-zeroed by G8.
//   unsorted 3DGUT (canonical sums, gut_render.cu "G7 backward"): 0..2 sum groGrd, 3 density, 4..12 W (3x3 row-major), 13..15 rgb,
//                                                                  16..18 depth branch's direct scale part, 19 pad
//   sorted k-buffer (final gradients): 0..2 pos, 3 density, 4..7 quat(wxyz), 8..10 scale, 11 pad, 12..14 rgb, 15..19 pad
constexpr int kGradRow = 20;

void launch_project(cudaStream_t s, const FrameCamera& cam, const FrameConfig& cfg, int64_t n, const float* particles,
                    const float* sph, int sph_degree, uint32_t* tiles_count, ProjRecord* proj, float* depth, float* rgb,
                    float* visibility, uint32_t* tile_hist, bool radiance = true);
void launch_expand_place(cudaStream_t s, const FrameCamera& cam, const FrameConfig& cfg, int64_t n, const ProjRecord* proj, const float* depth,
                         const uint32_t* tile_hist, const uint32_t* sub_base, const uint32_t* totals, uint32_t capacity, uint32_t* fill,
                         unsigned long long* keys);
// gut_binning.cu: tile ranges / order / hit-word slices from the per-tile histogram, per-tile on-chip sort of the 64-bit keys
constexpr int kTileSubs = 16;  // sub-counters per tile (a particle uses sub-counter `particle & 15`): spreads the atomics of hot tiles
size_t tile_scan_parts_words(int num_tiles);  // size of the scan's per-CTA partials (`parts`) in 32-bit words
void launch_tile_scan(cudaStream_t s, int num_tiles, const uint32_t* counts, uint32_t capacity, uint32_t* ranges, uint32_t* sub_base,
                      uint32_t* chunk_base, uint32_t* order, uint32_t* fill, uint32_t* totals, uint32_t* parts);
cudaError_t launch_tile_sort(cudaStream_t s, int num_tiles, const uint32_t* order, const uint32_t* ranges, const uint32_t* totals,
                             unsigned long long* keys, unsigned long long* keys_alt, uint32_t* sorted_values);
void launch_synth_tile_keys(cudaStream_t s, int num_tiles, const uint32_t* ranges, const uint32_t* vals, const float* depth, uint64_t* out);

// hit words: one 32-bit word per (32-entry chunk of a tile list, warp of the tile's CTA, quarter of the warp's 8x4 pixel block);
// tile t's slice starts at chunk_base[t] * 32 words
inline size_t hit_words_capacity(int64_t num_isect, int64_t tiles) { return (static_cast<size_t>(num_isect) / 32 + static_cast<size_t>(tiles) + 1) * 32; }
void launch_render_forward(cudaStream_t s, const FrameCamera& cam, const FrameConfig& cfg, const float* rays_o,
                           const float* rays_d, const float* particles, const float* rgb, const uint32_t* sorted_values,
                           const uint32_t* ranges, const uint32_t* tile_order, const uint32_t* chunk_base, uint32_t* hit_words, float* out_rgba,
                           float* out_dist, float* out_hits);
void launch_count_work(cudaStream_t s, const FrameCamera& cam, const FrameConfig& cfg, const float* rays_o, const float* rays_d,
                       const float* particles, const float* rgb, const uint32_t* sorted_values, const uint32_t* ranges,
                       const uint32_t* tile_order, const uint32_t* chunk_base, uint32_t* hit_words, unsigned long long* counters8);
void launch_render_backward(cudaStream_t s, const FrameCamera& cam, const FrameConfig& cfg, const float* rays_o,
                            const float* rays_d, const float* particles, const float* rgb, const uint32_t* sorted_values,
                            const uint32_t* ranges, const uint32_t* tile_order, const uint32_t* chunk_base, const uint32_t* hit_words,
                            const float* out_rgba, const float* d_rgba, const float* out_dist, const float* d_dist, float* grad_acc);
// gut_render_nht.cu: Neural Harmonic Texture features (48 per particle, barycentric, sincos) -> [H,W,25] features + opacity, and the
// adjoint: canonical sums into grad_acc (G8 with radiance = false maps them) and the feature gradient into d_features (zeroed by the caller)
void launch_render_forward_nht(cudaStream_t s, const FrameCamera& cam, const FrameConfig& cfg, const float* rays_o, const float* rays_d,
                               const float* particles, const void* features, bool half, const uint32_t* sorted_values, const uint32_t* ranges,
                               const uint32_t* tile_order, const uint32_t* chunk_base, uint32_t* hit_words, float* out_features_alpha,
                               float* out_dist, float* out_hits);
cudaError_t launch_render_backward_nht(cudaStream_t s, const FrameCamera& cam, const FrameConfig& cfg, const float* rays_o, const float* rays_d,
                                       const float* particles, const void* features, bool half, const uint32_t* sorted_values,
                                       const uint32_t* ranges, const uint32_t* tile_order, const uint32_t* chunk_base, const uint32_t* hit_words,
                                       const float* out_features_alpha, const float* d_features_alpha, const float* out_dist, const float* d_dist,
                                       float* grad_acc, float* d_features);
void launch_fma_peak(cudaStream_t s, int blocks, int iters, float* sink);
void launch_render_forward_kbuffer(cudaStream_t s, const FrameCamera& cam, const FrameConfig& cfg, int K, const float* rays_o, const float* rays_d,
                                   const float* particles, const float* rgb, const uint32_t* sorted_values, const uint32_t* ranges,
                                   float* out_rgba, float* out_dist, float* out_hits);
void launch_render_backward_kbuffer(cudaStream_t s, const FrameCamera& cam, const FrameConfig& cfg, int K, const float* rays_o, const float* rays_d,
                                    const float* particles, const float* rgb, const uint32_t* sorted_values, const uint32_t* ranges,
                                    const float* out_rgba, const float* d_rgba, const float* out_dist, const float* d_dist, float* grad_acc);
void launch_project_backward(cudaStream_t s, const FrameCamera& cam, int64_t n, const float* particles, const float* sph,
                             int sph_degree, const float* rgb, const uint32_t* tiles_count, const float* rays_o, float* grad_acc,
                             float* d_particles, float* d_sph, bool compact, bool canon, bool radiance = true);
void launch_sph_from_views(cudaStream_t s, int64_t n, const float* particles, int sph_degree, int views, const float* view_positions,
                           const float* d_radiance_all, float* d_sph);

// CUB-backed helpers (scan + radix sort), gut_sort.cu
size_t sort32_temp_bytes(int64_t n);
void run_sort32_pairs(cudaStream_t s, void* temp, size_t temp_bytes, const uint32_t* kin, uint32_t* kout, const uint32_t* vin,
                      uint32_t* vout, int64_t n, int end_bit);

}  // namespace gutb200
