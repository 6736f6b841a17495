/*
 * include/nht_b200.h -- C ABI of the H100-native (sm_90a) Neural Harmonic Texture feature decoder (lib: 3dgrut_b200/libgut_b200.so).
 *
 * The network is tiny-cuda-nn's NetworkWithInputEncoding as the reference's FeatureDecoder configures it
 * (threedgrut/model/feature_decoder.py:69-97):
 *   encoding  Composite[Identity(F), SphericalHarmonics(degree d)] of [features, (dir * sh_scale + 1) / 2], fp16.  The encoded row is
 *             [features (F), ones (P), SH(3 dir * sh_scale) (d^2)] with P the padding up to a multiple of 16: tcnn's Composite pads its
 *             last nested encoding, and the SH encoding writes its padding lanes (value 1, the bias of the bias-free net) first.
 *   MLP       bias-free FullyFusedMLP, width 128, n_hidden_layers >= 1, ReLU, output padded to 16 rows, output activation; only outputs
 *             0..2 are returned.
 *   params    fp32, tcnn's order and layout: W_0 [128][K0] (K0 = F + P + d^2), n_hidden_layers - 1 matrices [128][128], W_out [16][128],
 *             each row-major [out][in].  A tcnn checkpoint's `params` loads unchanged.
 * Built: width 128, n_hidden_layers >= 1 (while the fp16 weights fit in shared memory), SH degree 1..4, F + d^2 <= 128.  Anything else
 * returns NHTB200_UNSUPPORTED.
 *
 * Conventions as in gut_b200.h: raw device pointers, the cudaStream_t passed as void*, caller-allocated outputs, no hidden synchronisation;
 * every call returns 0 on success and non-zero on failure, nhtb200_last_error() gives the message.
 * Features [n,F], directions [n,3], outputs [n,3], d_features [n,F]: fp32, row-major, contiguous.  Any n >= 0.
 */
#ifndef NHT_B200_H
#define NHT_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { NHTB200_ACT_NONE = 0, NHTB200_ACT_RELU = 1, NHTB200_ACT_SIGMOID = 2 };
enum { NHTB200_OK = 0, NHTB200_UNSUPPORTED = 1, NHTB200_BAD_ARGUMENT = 2, NHTB200_CUDA_ERROR = 3 };

typedef struct nhtb200_config {
    int32_t n_features;         /* F, ray_feature_dim */
    int32_t sh_degree;          /* d: d^2 SH coefficients (tcnn "degree") */
    int32_t n_hidden_layers;    /* tcnn n_hidden_layers (FeatureDecoder num_layers) */
    int32_t width;              /* n_neurons: 128 */
    int32_t output_activation;  /* NHTB200_ACT_* */
    float sh_scale;             /* directions enter the encoding as (dir * sh_scale + 1) / 2 */
} nhtb200_config;

const char* nhtb200_last_error(void);
/* Length of the flat params vector (tcnn's n_params), or -1 if the configuration is not built. */
int64_t nhtb200_n_params(const nhtb200_config* cfg);
/* Device bytes of the workspace nhtb200_backward needs for n rows. */
size_t nhtb200_backward_workspace_bytes(const nhtb200_config* cfg, int64_t n);
/* out [n,3] = decoder(features, dirs).  Writes nothing but out: the backward recomputes the activations, so the same call serves training
 * and inference. */
int nhtb200_forward(const nhtb200_config* cfg, void* stream, int64_t n, const float* features, const float* dirs, const float* params,
                    float* out);
/* d_out [n,3] -> d_features [n,F] and d_params [n_params] (summed over all rows, overwritten).  Directions get no gradient.
 * Deterministic: the parameter gradient is reduced in a fixed order, without atomics. */
int nhtb200_backward(const nhtb200_config* cfg, void* stream, int64_t n, const float* features, const float* dirs, const float* params,
                     const float* d_out, float* d_features, float* d_params, void* workspace);

#ifdef __cplusplus
}
#endif
#endif
