// Neural Harmonic Texture feature decoder (include/nht_b200.h): tcnn's NetworkWithInputEncoding with a Composite[Identity, SH] encoding
// and a bias-free width-128 MLP, on the H100's tensor cores.
//
// Every matrix product is mma.sync.m16n8k16 with fp16 operands and fp32 accumulation.  A warp owns 16 rows; the weights of all layers
// are resident in shared memory for the life of a persistent CTA (row stride in + 8 halves, so ldmatrix is conflict-free).  The
// encoding is staged per warp in shared memory and read as the first layer's A operand; after that the accumulator of one layer, after
// ReLU and packing to fp16, is the next layer's A fragment in registers.
//
// Backward: no activations are kept from the forward.  nht_bwd recomputes the forward of its 16 rows, backpropagates the output
// gradient through the layers (delta_{m-1} = (delta_m W_m) * [h_m > 0]), writes d_features, and stores each matrix's fp16 input
// activations A_m and output gradients D_m to the workspace.  nht_dw then forms dW_m = D_m^T A_m per fixed chunk of rows with the same
// mma, and nht_dw_reduce sums the chunks in a fixed order: the parameter gradient is deterministic.  The output gradient is scaled by a
// power of two that brings its largest magnitude to 1 before it becomes an fp16 operand (the role of tcnn's loss scale, but exact and
// chosen from the data); the scale is divided out of d_features and d_params.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <string>

#include "../../include/nht_b200.h"

namespace {

constexpr int WIDTH = 128;
constexpr int OUT_PAD = 16;
constexpr int MAXM = 16;          // matrices (n_hidden_layers + 1) a config may have
constexpr int DW_ROWS = 64;       // rows per shared-memory tile of nht_dw
constexpr int DW_CHUNKS = 256;    // fixed row chunks of the parameter-gradient reduction (independent of the device: deterministic)

thread_local std::string g_err;

struct Net {
    int F, D, K0, n_mats, act;
    float sh_scale;
    int in[MAXM], out[MAXM];
    int woff[MAXM];       // smem offset of W_m, halves (row stride in[m] + 8)
    int64_t poff[MAXM];   // offset of W_m in params
    int64_t n_params;
    int w_halves;         // smem halves of all weights
};

struct Work {  // nht_bwd -> nht_dw: per matrix, input activations A_m [n_pad][in] and output gradients D_m [n_pad][out], fp16
    __half* A[MAXM];
    __half* Dg[MAXM];
    float* partial;       // [DW_CHUNKS][n_params]
    unsigned* amax;       // bits of max |d_out|
    int64_t n_pad;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void ldsm4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(smem_u32(p)));
}

__device__ __forceinline__ void ldsm4t(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(smem_u32(p)));
}

__device__ __forceinline__ void mma(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint32_t pack(float lo, float hi) {
    __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&h);
}

// tcnn's SH polynomials (common_device.h sh_enc), degree <= 4, evaluated where tcnn evaluates them: at (u * 2 - 1) with
// u = (dir * sh_scale + 1) * 0.5 computed in fp32 as the reference's FeatureDecoder computes it.
__device__ __forceinline__ void sh_enc(int degree, float x, float y, float z, float* o) {
    float xy = x * y, xz = x * z, yz = y * z, x2 = x * x, y2 = y * y, z2 = z * z;
    o[0] = 0.28209479177387814f;
    if (degree <= 1) return;
    o[1] = -0.48860251190291987f * y;
    o[2] = 0.48860251190291987f * z;
    o[3] = -0.48860251190291987f * x;
    if (degree <= 2) return;
    o[4] = 1.0925484305920792f * xy;
    o[5] = -1.0925484305920792f * yz;
    o[6] = 0.94617469575755997f * z2 - 0.31539156525251999f;
    o[7] = -1.0925484305920792f * xz;
    o[8] = 0.54627421529603959f * x2 - 0.54627421529603959f * y2;
    if (degree <= 3) return;
    o[9] = 0.59004358992664352f * y * (-3.0f * x2 + y2);
    o[10] = 2.8906114426405538f * xy * z;
    o[11] = 0.45704579946446572f * y * (1.0f - 5.0f * z2);
    o[12] = 0.3731763325901154f * z * (5.0f * z2 - 3.0f);
    o[13] = 0.45704579946446572f * x * (1.0f - 5.0f * z2);
    o[14] = 1.4453057213202769f * z * (x2 - y2);
    o[15] = 0.59004358992664352f * x * (-x2 + 3.0f * y2);
}

// Weights of all matrices to shared memory as fp16, W_m at woff[m], row stride in[m] + 8.
__device__ void load_weights(const Net& net, const float* __restrict__ params, __half* w) {
    for (int m = 0; m < net.n_mats; ++m) {
        const int in = net.in[m], n = net.out[m] * in;
        const float* p = params + net.poff[m];
        __half* d = w + net.woff[m];
        for (int i = threadIdx.x; i < n; i += blockDim.x) d[(i / in) * (in + 8) + i % in] = __float2half_rn(p[i]);
    }
}

// The encoded rows [row0, row0 + 16) as fp16 in st[16][K0 + 8]; rows >= n encode zero features and a zero direction.
__device__ void encode_tile(const Net& net, int64_t row0, int64_t n, const float* __restrict__ feat, const float* __restrict__ dirs,
                            __half* st) {
    const int lane = threadIdx.x & 31, F = net.F, S = net.K0 + 8;
    for (int i = lane; i < 16 * F; i += 32) {
        const int r = i / F, j = i - r * F;
        const int64_t row = row0 + r;
        st[r * S + j] = __float2half_rn(row < n ? feat[row0 * F + i] : 0.0f);
    }
    if (lane < 16) {
        const int64_t row = row0 + lane;
        float d[3] = {0.f, 0.f, 0.f};
        if (row < n) d[0] = dirs[row * 3], d[1] = dirs[row * 3 + 1], d[2] = dirs[row * 3 + 2];
        float c[3];
        for (int k = 0; k < 3; ++k) c[k] = __fsub_rn(__fmul_rn(__fmul_rn(__fadd_rn(__fmul_rn(d[k], net.sh_scale), 1.0f), 0.5f), 2.0f), 1.0f);
        float sh[16];
        const int degree = net.D == 1 ? 1 : net.D == 4 ? 2 : net.D == 9 ? 3 : 4;
        sh_enc(degree, c[0], c[1], c[2], sh);
        __half* o = st + lane * S;
        for (int j = F; j < net.K0 - net.D; ++j) o[j] = __float2half_rn(1.0f);
        for (int j = 0; j < net.D; ++j) o[net.K0 - net.D + j] = __float2half_rn(sh[j]);
    }
    __syncwarp();
}

// acc[16 rows][128] = A (ldmatrix from st[16][K0+8]) x W_0^T
__device__ __forceinline__ void layer0(const Net& net, const __half* st, const __half* w, float (&acc)[16][4]) {
    const int lane = threadIdx.x & 31, S = net.K0 + 8, WS = net.K0 + 8;
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
    const __half* W = w + net.woff[0];
#pragma unroll 1
    for (int kt = 0; kt < net.K0 / 16; ++kt) {
        uint32_t a[4];
        ldsm4(a[0], a[1], a[2], a[3], st + ((lane & 7) + ((lane >> 3) & 1) * 8) * S + kt * 16 + (lane >> 4) * 8);
#pragma unroll
        for (int p = 0; p < 8; ++p) {
            uint32_t b0, b1, b2, b3;
            ldsm4(b0, b1, b2, b3, W + (p * 16 + (lane >> 4) * 8 + (lane & 7)) * WS + kt * 16 + ((lane >> 3) & 1) * 8);
            mma(acc[2 * p], a, b0, b1);
            mma(acc[2 * p + 1], a, b2, b3);
        }
    }
}

// acc[16 rows][NT*8] = a (registers, 8 k-tiles of 16) x W^T, W [NT*8][128] at stride 136
template <int NT>
__device__ __forceinline__ void layer_reg(const uint32_t (&a)[8][4], const __half* W, float (&acc)[16][4]) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int j = 0; j < NT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
#pragma unroll
    for (int kt = 0; kt < 8; ++kt) {
#pragma unroll
        for (int p = 0; p < NT / 2; ++p) {
            uint32_t b0, b1, b2, b3;
            ldsm4(b0, b1, b2, b3, W + (p * 16 + (lane >> 4) * 8 + (lane & 7)) * (WIDTH + 8) + kt * 16 + ((lane >> 3) & 1) * 8);
            mma(acc[2 * p], a[kt], b0, b1);
            mma(acc[2 * p + 1], a[kt], b2, b3);
        }
    }
}

// ReLU, fp16, and the accumulator layout reread as the A fragments of the next layer
__device__ __forceinline__ void relu_pack(const float (&acc)[16][4], uint32_t (&a)[8][4]) {
#pragma unroll
    for (int kt = 0; kt < 8; ++kt) {
        a[kt][0] = pack(fmaxf(acc[2 * kt][0], 0.f), fmaxf(acc[2 * kt][1], 0.f));
        a[kt][1] = pack(fmaxf(acc[2 * kt][2], 0.f), fmaxf(acc[2 * kt][3], 0.f));
        a[kt][2] = pack(fmaxf(acc[2 * kt + 1][0], 0.f), fmaxf(acc[2 * kt + 1][1], 0.f));
        a[kt][3] = pack(fmaxf(acc[2 * kt + 1][2], 0.f), fmaxf(acc[2 * kt + 1][3], 0.f));
    }
}

__device__ __forceinline__ float activate(int act, float x) {
    return act == NHTB200_ACT_SIGMOID ? 1.0f / (1.0f + __expf(-x)) : act == NHTB200_ACT_RELU ? fmaxf(x, 0.f) : x;
}

__device__ __forceinline__ float activate_grad(int act, float x) {
    if (act == NHTB200_ACT_SIGMOID) {
        const float y = 1.0f / (1.0f + __expf(-x));
        return y * (1.0f - y);
    }
    return act == NHTB200_ACT_RELU ? (x > 0.f ? 1.f : 0.f) : 1.f;
}

// forward of 16 rows up to the output layer's pre-activation; h_m (m = 1..L) also go to hs[m-1] (fp16 [16][136]) when hs != nullptr
__device__ __forceinline__ void forward_tile(const Net& net, const __half* st, const __half* w, float (&acc)[16][4], uint32_t (&a)[8][4],
                                             __half* hs) {
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    layer0(net, st, w, acc);
    for (int m = 1; m < net.n_mats; ++m) {
        relu_pack(acc, a);
        if (hs) {
            __half* h = hs + (m - 1) * 16 * (WIDTH + 8);
#pragma unroll
            for (int kt = 0; kt < 8; ++kt) {
                *reinterpret_cast<uint32_t*>(h + g * (WIDTH + 8) + kt * 16 + 2 * t) = a[kt][0];
                *reinterpret_cast<uint32_t*>(h + (g + 8) * (WIDTH + 8) + kt * 16 + 2 * t) = a[kt][1];
                *reinterpret_cast<uint32_t*>(h + g * (WIDTH + 8) + kt * 16 + 8 + 2 * t) = a[kt][2];
                *reinterpret_cast<uint32_t*>(h + (g + 8) * (WIDTH + 8) + kt * 16 + 8 + 2 * t) = a[kt][3];
            }
        }
        if (m + 1 < net.n_mats) layer_reg<16>(a, w + net.woff[m], acc);
        else layer_reg<2>(a, w + net.woff[m], acc);
    }
}

// Per-warp shared-memory halves: the encoded tile, plus (backward) one [16][136] tile per hidden layer.
__host__ __device__ inline int warp_halves(const Net& net, bool bwd) { return 16 * (net.K0 + 8) + (bwd ? (net.n_mats - 1) * 16 * (WIDTH + 8) : 0); }

__global__ void __launch_bounds__(256) nht_fwd(Net net, int64_t n, const float* __restrict__ feat, const float* __restrict__ dirs,
                                               const float* __restrict__ params, float* __restrict__ out) {
    extern __shared__ __align__(16) __half smem[];
    load_weights(net, params, smem);
    __syncthreads();
    const int warp = threadIdx.x >> 5, nw = blockDim.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    __half* st = smem + net.w_halves + warp * warp_halves(net, false);
    const int64_t tiles = (n + 15) / 16;
    float acc[16][4];
    uint32_t a[8][4];
    for (int64_t tile = (int64_t)blockIdx.x * nw + warp; tile < tiles; tile += (int64_t)gridDim.x * nw) {
        const int64_t row0 = tile * 16;
        encode_tile(net, row0, n, feat, dirs, st);
        forward_tile(net, st, smem, acc, a, nullptr);
        __syncwarp();  // st is rewritten by the next tile
        if (t < 2) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int64_t row = row0 + g + 8 * h;
                if (row < n) {
                    out[row * 3 + 2 * t] = activate(net.act, acc[0][2 * h]);
                    if (t == 0) out[row * 3 + 1] = activate(net.act, acc[0][2 * h + 1]);
                }
            }
        }
    }
}

// [16][w] fp16 tile (row stride w + 8) -> rows [row0, row0 + 16) of a [*, w] global array
__device__ __forceinline__ void store_tile(const __half* s, int w, __half* __restrict__ gdst, int64_t row0) {
    const int lane = threadIdx.x & 31, v = w / 8;
    for (int i = lane; i < 16 * v; i += 32) {
        const int r = i / v, c = (i - r * v) * 8;
        *reinterpret_cast<uint4*>(gdst + (row0 + r) * w + c) = *reinterpret_cast<const uint4*>(s + r * (w + 8) + c);
    }
}

__global__ void nht_amax(int64_t n3, const float* __restrict__ d_out, unsigned* amax) {
    float m = 0.f;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n3; i += (int64_t)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(d_out[i]));
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(amax, __float_as_uint(m));  // non-negative floats order as their bits
}

// power of two that brings max |d_out| to (0.5, 1]
__device__ __forceinline__ float grad_scale(const unsigned* amax) {
    const float m = __uint_as_float(*amax);
    return (m > 0.f && isfinite(m)) ? exp2f(-ceilf(log2f(m))) : 1.0f;
}

__global__ void __launch_bounds__(256) nht_bwd(Net net, Work wk, int64_t n, const float* __restrict__ feat, const float* __restrict__ dirs,
                                               const float* __restrict__ params, const float* __restrict__ d_out,
                                               float* __restrict__ d_feat) {
    extern __shared__ __align__(16) __half smem[];
    load_weights(net, params, smem);
    __syncthreads();
    const int warp = threadIdx.x >> 5, nw = blockDim.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    __half* st = smem + net.w_halves + warp * warp_halves(net, true);
    __half* hs = st + 16 * (net.K0 + 8);
    const float scale = grad_scale(wk.amax), inv_scale = 1.0f / scale;
    const int L = net.n_mats - 1;
    const int64_t tiles = wk.n_pad / 16;
    float acc[16][4];
    uint32_t a[8][4];
    for (int64_t tile = (int64_t)blockIdx.x * nw + warp; tile < tiles; tile += (int64_t)gridDim.x * nw) {
        const int64_t row0 = tile * 16;
        encode_tile(net, row0, n, feat, dirs, st);
        forward_tile(net, st, smem, acc, a, hs);
        __syncwarp();
        store_tile(st, net.K0, wk.A[0], row0);
        for (int m = 1; m <= L; ++m) store_tile(hs + (m - 1) * 16 * (WIDTH + 8), WIDTH, wk.A[m], row0);

        // delta_L = d_out * act'(z) * scale on the 3 live outputs, 0 on the padded ones and on rows >= n
        uint32_t da[8][4];
        {
            float dl[2][4];
#pragma unroll
            for (int j = 0; j < 2; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int col = j * 8 + 2 * t + (e & 1);
                    const int64_t row = row0 + g + 8 * (e >> 1);
                    dl[j][e] = (col < 3 && row < n) ? d_out[row * 3 + col] * activate_grad(net.act, acc[j][e]) * scale : 0.f;
                }
            da[0][0] = pack(dl[0][0], dl[0][1]);
            da[0][1] = pack(dl[0][2], dl[0][3]);
            da[0][2] = pack(dl[1][0], dl[1][1]);
            da[0][3] = pack(dl[1][2], dl[1][3]);
            __half* D = wk.Dg[L];
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                *reinterpret_cast<uint32_t*>(D + (row0 + g) * OUT_PAD + j * 8 + 2 * t) = da[0][2 * j];
                *reinterpret_cast<uint32_t*>(D + (row0 + g + 8) * OUT_PAD + j * 8 + 2 * t) = da[0][2 * j + 1];
            }
        }
        // delta_{m-1} = (delta_m W_m) * [h_m > 0], m = L..1; W_m [out][in] read transposed as B[k = out][n = in]
        for (int m = L; m >= 1; --m) {
            const __half* W = smem + net.woff[m];
            const int WS = net.in[m] + 8, kts = net.out[m] / 16;
#pragma unroll
            for (int j = 0; j < 16; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
#pragma unroll
            for (int kt = 0; kt < 8; ++kt) {
                if (kt < kts) {
#pragma unroll
                    for (int p = 0; p < 8; ++p) {
                        uint32_t b0, b1, b2, b3;
                        ldsm4t(b0, b1, b2, b3, W + (kt * 16 + ((lane >> 3) & 1) * 8 + (lane & 7)) * WS + p * 16 + (lane >> 4) * 8);
                        mma(acc[2 * p], da[kt], b0, b1);
                        mma(acc[2 * p + 1], da[kt], b2, b3);
                    }
                }
            }
            __half* h = hs + (m - 1) * 16 * (WIDTH + 8);
#pragma unroll
            for (int j = 0; j < 16; ++j)
#pragma unroll
                for (int e = 0; e < 4; e += 2) {
                    __half2* p = reinterpret_cast<__half2*>(h + (g + 4 * e) * (WIDTH + 8) + j * 8 + 2 * t);
                    const __half2 hv = *p;
                    const float v0 = __low2float(hv) > 0.f ? acc[j][e] : 0.f, v1 = __high2float(hv) > 0.f ? acc[j][e + 1] : 0.f;
                    acc[j][e] = v0, acc[j][e + 1] = v1;
                    *p = __floats2half2_rn(v0, v1);
                }
#pragma unroll
            for (int kt = 0; kt < 8; ++kt) {
                da[kt][0] = pack(acc[2 * kt][0], acc[2 * kt][1]);
                da[kt][1] = pack(acc[2 * kt][2], acc[2 * kt][3]);
                da[kt][2] = pack(acc[2 * kt + 1][0], acc[2 * kt + 1][1]);
                da[kt][3] = pack(acc[2 * kt + 1][2], acc[2 * kt + 1][3]);
            }
            __syncwarp();
            store_tile(h, WIDTH, wk.Dg[m - 1], row0);
        }
        // d_features = (delta_0 W_0)[:, :F] / scale
        {
            const __half* W = smem + net.woff[0];
            const int WS = net.K0 + 8, np = net.K0 / 16;
#pragma unroll
            for (int j = 0; j < 16; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
#pragma unroll
            for (int kt = 0; kt < 8; ++kt) {
#pragma unroll
                for (int p = 0; p < 8; ++p) {
                    if (p < np) {
                        uint32_t b0, b1, b2, b3;
                        ldsm4t(b0, b1, b2, b3, W + (kt * 16 + ((lane >> 3) & 1) * 8 + (lane & 7)) * WS + p * 16 + (lane >> 4) * 8);
                        mma(acc[2 * p], da[kt], b0, b1);
                        mma(acc[2 * p + 1], da[kt], b2, b3);
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < 16; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int col = j * 8 + 2 * t + (e & 1);
                    const int64_t row = row0 + g + 8 * (e >> 1);
                    if (col < net.F && row < n) d_feat[row * net.F + col] = acc[j][e] * inv_scale;
                }
        }
        __syncwarp();  // the smem tiles are rewritten by the next tile
    }
}

// partial[chunk][W_m] = sum over the chunk's rows of D_m^T A_m; blockIdx.y = m.  8 warps; warp tile 16 (out) x nwc (in).
__global__ void __launch_bounds__(256) nht_dw(Net net, Work wk) {
    __shared__ __align__(16) __half sD[DW_ROWS * (WIDTH + 8)];
    __shared__ __align__(16) __half sA[DW_ROWS * (WIDTH + 8)];
    const int m = blockIdx.y, out = net.out[m], in = net.in[m];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    // out = 128: warp w owns out rows [16w, 16w+16) and every input column; out = 16: every warp owns a 16-column slice of in = 128
    const int mbase = out == WIDTH ? warp * 16 : 0;
    const int nwc = out == WIDTH ? in : in / 8, nbase = out == WIDTH ? 0 : warp * nwc;
    const int64_t tiles = wk.n_pad / DW_ROWS, per = (tiles + DW_CHUNKS - 1) / DW_CHUNKS;
    const int64_t t0 = blockIdx.x * per, t1 = min(tiles, t0 + per);
    const __half* Dg = wk.Dg[m];
    const __half* Ag = wk.A[m];
    float acc[16][4];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
    for (int64_t tile = t0; tile < t1; ++tile) {
        const int64_t r0 = tile * DW_ROWS;
        for (int i = threadIdx.x; i < DW_ROWS * out / 8; i += blockDim.x) {
            const int r = i / (out / 8), c = (i - r * (out / 8)) * 8;
            *reinterpret_cast<uint4*>(sD + r * (out + 8) + c) = *reinterpret_cast<const uint4*>(Dg + (r0 + r) * out + c);
        }
        for (int i = threadIdx.x; i < DW_ROWS * in / 8; i += blockDim.x) {
            const int r = i / (in / 8), c = (i - r * (in / 8)) * 8;
            *reinterpret_cast<uint4*>(sA + r * (in + 8) + c) = *reinterpret_cast<const uint4*>(Ag + (r0 + r) * in + c);
        }
        __syncthreads();
#pragma unroll
        for (int kt = 0; kt < DW_ROWS / 16; ++kt) {
            uint32_t a[4];  // A[m = out][k = row] from sD[row][out], transposed
            ldsm4t(a[0], a[1], a[2], a[3], sD + (kt * 16 + (lane >> 4) * 8 + (lane & 7)) * (out + 8) + mbase + ((lane >> 3) & 1) * 8);
#pragma unroll
            for (int p = 0; p < 8; ++p) {
                if (p < nwc / 16) {
                    uint32_t b0, b1, b2, b3;  // B[k = row][n = in] from sA[row][in], transposed
                    ldsm4t(b0, b1, b2, b3, sA + (kt * 16 + ((lane >> 3) & 1) * 8 + (lane & 7)) * (in + 8) + nbase + p * 16 + (lane >> 4) * 8);
                    mma(acc[2 * p], a, b0, b1);
                    mma(acc[2 * p + 1], a, b2, b3);
                }
            }
        }
        __syncthreads();
    }
    float* dst = wk.partial + (int64_t)blockIdx.x * net.n_params + net.poff[m];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        if (j < nwc / 8) {
            const int col = nbase + j * 8 + 2 * t;
            *reinterpret_cast<float2*>(dst + (mbase + g) * in + col) = make_float2(acc[j][0], acc[j][1]);
            *reinterpret_cast<float2*>(dst + (mbase + g + 8) * in + col) = make_float2(acc[j][2], acc[j][3]);
        }
    }
}

__global__ void nht_dw_reduce(int64_t n_params, const float* __restrict__ partial, const unsigned* amax, float* __restrict__ d_params) {
    const float inv_scale = 1.0f / grad_scale(amax);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_params; i += (int64_t)gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int c = 0; c < DW_CHUNKS; ++c) s += partial[(int64_t)c * n_params + i];
        d_params[i] = s * inv_scale;
    }
}

int fail(int code, const std::string& msg) {
    g_err = msg;
    return code;
}

// NHTB200_OK and a filled Net, or NHTB200_UNSUPPORTED / NHTB200_BAD_ARGUMENT with g_err set
int make_net(const nhtb200_config* cfg, Net& net) {
    if (!cfg) return fail(NHTB200_BAD_ARGUMENT, "null config");
    if (cfg->width != WIDTH) return fail(NHTB200_UNSUPPORTED, "width " + std::to_string(cfg->width) + " is not built (only 128)");
    if (cfg->sh_degree < 1 || cfg->sh_degree > 4)
        return fail(NHTB200_UNSUPPORTED, "SH degree " + std::to_string(cfg->sh_degree) + " is not built (1..4)");
    if (cfg->n_hidden_layers < 1 || cfg->n_hidden_layers >= MAXM)
        return fail(NHTB200_UNSUPPORTED, "n_hidden_layers " + std::to_string(cfg->n_hidden_layers) + " is not built");
    if (cfg->output_activation < NHTB200_ACT_NONE || cfg->output_activation > NHTB200_ACT_SIGMOID)
        return fail(NHTB200_UNSUPPORTED, "output activation " + std::to_string(cfg->output_activation) + " is not built");
    const int D = cfg->sh_degree * cfg->sh_degree;
    if (cfg->n_features < 1 || cfg->n_features + D > WIDTH)
        return fail(NHTB200_UNSUPPORTED, "n_features + sh_degree^2 must lie in 2..128, got " + std::to_string(cfg->n_features + D));
    net.F = cfg->n_features;
    net.D = D;
    net.K0 = (cfg->n_features + D + 15) / 16 * 16;
    net.n_mats = cfg->n_hidden_layers + 1;
    net.act = cfg->output_activation;
    net.sh_scale = cfg->sh_scale;
    int64_t p = 0;
    int wo = 0;
    for (int m = 0; m < net.n_mats; ++m) {
        net.in[m] = m == 0 ? net.K0 : WIDTH;
        net.out[m] = m + 1 == net.n_mats ? OUT_PAD : WIDTH;
        net.poff[m] = p;
        net.woff[m] = wo;
        p += (int64_t)net.in[m] * net.out[m];
        wo += net.out[m] * (net.in[m] + 8);
    }
    net.n_params = p;
    net.w_halves = wo;
    return NHTB200_OK;
}

// Largest of 8, 4, 2, 1 warps whose shared memory fits the device; 0 if none does.
int pick_warps(const Net& net, bool bwd, size_t& smem) {
    int dev = 0, optin = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    for (int w = 8; w >= 1; w >>= 1) {
        smem = (size_t)(net.w_halves + w * warp_halves(net, bwd)) * sizeof(__half);
        if (smem <= (size_t)optin) return w;
    }
    return 0;
}

template <typename K>
int grid_for(K kernel, int warps, size_t smem, int64_t warp_tiles) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, warps * 32, smem);
    const int64_t need = (warp_tiles + warps - 1) / warps;
    return (int)std::max<int64_t>(1, std::min<int64_t>(need, (int64_t)sms * std::max(per_sm, 1)));
}

size_t align256(size_t b) { return (b + 255) / 256 * 256; }

// workspace layout: amax | A_0, D_0, A_1, D_1, ... | partial
size_t workspace_layout(const Net& net, int64_t n, Work* wk, char* base) {
    const int64_t n_pad = (n + DW_ROWS - 1) / DW_ROWS * DW_ROWS;
    size_t off = 256;
    for (int m = 0; m < net.n_mats; ++m) {
        if (wk) wk->A[m] = reinterpret_cast<__half*>(base + off);
        off += align256((size_t)n_pad * net.in[m] * sizeof(__half));
        if (wk) wk->Dg[m] = reinterpret_cast<__half*>(base + off);
        off += align256((size_t)n_pad * net.out[m] * sizeof(__half));
    }
    if (wk) {
        wk->partial = reinterpret_cast<float*>(base + off);
        wk->amax = reinterpret_cast<unsigned*>(base);
        wk->n_pad = n_pad;
    }
    off += align256((size_t)DW_CHUNKS * net.n_params * sizeof(float));
    return off;
}

int cuda_check(const char* what) {
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? NHTB200_OK : fail(NHTB200_CUDA_ERROR, std::string(what) + ": " + cudaGetErrorString(e));
}

}  // namespace

extern "C" {

const char* nhtb200_last_error(void) { return g_err.c_str(); }

int64_t nhtb200_n_params(const nhtb200_config* cfg) {
    Net net;
    return make_net(cfg, net) == NHTB200_OK ? net.n_params : -1;
}

size_t nhtb200_backward_workspace_bytes(const nhtb200_config* cfg, int64_t n) {
    Net net;
    if (make_net(cfg, net) != NHTB200_OK || n < 0) return 0;
    return workspace_layout(net, n, nullptr, nullptr);
}

int nhtb200_forward(const nhtb200_config* cfg, void* stream, int64_t n, const float* features, const float* dirs, const float* params,
                    float* out) {
    Net net;
    if (int rc = make_net(cfg, net)) return rc;
    if (n < 0) return fail(NHTB200_BAD_ARGUMENT, "n < 0");
    if (n == 0) return NHTB200_OK;
    if (!features || !dirs || !params || !out) return fail(NHTB200_BAD_ARGUMENT, "null pointer");
    size_t smem = 0;
    const int warps = pick_warps(net, false, smem);
    if (!warps) return fail(NHTB200_UNSUPPORTED, "the weights of this network do not fit in shared memory");
    const int grid = grid_for(nht_fwd, warps, smem, (n + 15) / 16);
    nht_fwd<<<grid, warps * 32, smem, (cudaStream_t)stream>>>(net, n, features, dirs, params, out);
    return cuda_check("nht_fwd");
}

int nhtb200_backward(const nhtb200_config* cfg, void* stream, int64_t n, const float* features, const float* dirs, const float* params,
                     const float* d_out, float* d_features, float* d_params, void* workspace) {
    Net net;
    if (int rc = make_net(cfg, net)) return rc;
    if (n < 0) return fail(NHTB200_BAD_ARGUMENT, "n < 0");
    if (!params || !d_params || !workspace || (n > 0 && (!features || !dirs || !d_out || !d_features)))
        return fail(NHTB200_BAD_ARGUMENT, "null pointer");
    const cudaStream_t s = (cudaStream_t)stream;
    Work wk;
    workspace_layout(net, n, &wk, static_cast<char*>(workspace));
    size_t smem = 0;
    const int warps = pick_warps(net, true, smem);
    if (!warps) return fail(NHTB200_UNSUPPORTED, "the weights of this network do not fit in shared memory");
    cudaMemsetAsync(wk.amax, 0, sizeof(unsigned), s);
    if (n > 0) {
        nht_amax<<<264, 256, 0, s>>>(n * 3, d_out, wk.amax);
        const int grid = grid_for(nht_bwd, warps, smem, wk.n_pad / 16);
        nht_bwd<<<grid, warps * 32, smem, s>>>(net, wk, n, features, dirs, params, d_out, d_features);
    }
    nht_dw<<<dim3(DW_CHUNKS, net.n_mats), 256, 0, s>>>(net, wk);
    nht_dw_reduce<<<(int)std::min<int64_t>((net.n_params + 255) / 256, 1024), 256, 0, s>>>(net.n_params, wk.partial, wk.amax, d_params);
    return cuda_check("nhtb200_backward");
}

}  // extern "C"
