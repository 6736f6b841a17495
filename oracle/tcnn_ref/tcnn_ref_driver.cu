// oracle/tcnn_ref/tcnn_ref_driver.cu -- TEST / BASELINE INFRASTRUCTURE ONLY (never linked into the product).
//
// extern "C" driver (our code) around the reference's tiny-cuda-nn `NetworkWithInputEncoding`, configured the way the reference's
// `FeatureDecoder` configures it: Composite[Identity(F), SphericalHarmonics(degree)] -> FullyFusedMLP(width 128, ReLU,
// n_hidden_layers, output activation), fp16 network precision, 3 outputs.  tiny-cuda-nn is compiled in place from the reference tree by
// oracle/tcnn_ref/Makefile; nothing is copied into this repository.  The driver does what the tcnn torch binding does
// (bindings/torch/tinycudann/modules.py): fp32 params are rounded to the fp16 parameter buffer, the batch is padded to a multiple of
// 256 with zero rows, the output gradient is multiplied by the default fp16 loss scale (128) before the backward and the input and
// parameter gradients are divided by it afterwards.  Uses: the golden fixture tests/golden/nht_decoder_tcnn.npz
// (tests/golden/make_tcnn_golden.py), the live tcnn check of tests/test_nht_decoder_gpu.py and the tcnn baseline of
// scripts/bench_nht_decoder.py.
#include <tiny-cuda-nn/common.h>
#include <tiny-cuda-nn/encoding.h>
#include <tiny-cuda-nn/gpu_matrix.h>
#include <tiny-cuda-nn/gpu_memory.h>
#include <tiny-cuda-nn/network.h>
#include <tiny-cuda-nn/network_with_input_encoding.h>
#include <tiny-cuda-nn/rtc_kernel.h>

#include <cstdio>
#include <memory>
#include <string>

using namespace tcnn;
using T = __half;

// Built without runtime compilation (no TCNN_RTC), src/rtc_kernel.cu leaves CudaRtcKernel::set undefined although the header's inline
// launch helper refers to it.  The CudaRtcKernel constructor throws in that build, so no object ever reaches this definition.
void tcnn::CudaRtcKernel::set(CUfunction_attribute, int) { throw std::runtime_error{"tiny-cuda-nn was built without RTC"}; }

namespace {

constexpr float LOSS_SCALE = 128.0f;
constexpr uint32_t GRANULARITY = 256;

struct Ref {
    uint32_t n_input = 0;  // F + 3
    std::unique_ptr<NetworkWithInputEncoding<T>> net;
    GPUMemory<T> params, grads;
    GPUMemory<float> in_pad, din_pad;  // [n_pad, F+3]
    GPUMemory<T> out, dout;            // [n_pad, 16]
    std::unique_ptr<Context> ctx;
    uint32_t n_pad = 0;
};

__global__ void to_half(uint32_t n, const float* __restrict__ a, T* __restrict__ b) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) b[i] = __float2half(a[i]);
}

__global__ void to_float(uint32_t n, float scale, const T* __restrict__ a, float* __restrict__ b) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) b[i] = __half2float(a[i]) * scale;
}

__global__ void scale_float(uint32_t n, float scale, const float* __restrict__ a, float* __restrict__ b) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) b[i] = a[i] * scale;
}

// [n, 3] fp32 rows <-> [n_pad, 16] fp16 rows (padded lanes and rows stay zero)
__global__ void out_to_float(uint32_t n, const T* __restrict__ a, float* __restrict__ b) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n * 3) b[i] = __half2float(a[(i / 3) * 16 + i % 3]);
}

__global__ void dout_to_half(uint32_t n, const float* __restrict__ a, T* __restrict__ b) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n * 3) b[(i / 3) * 16 + i % 3] = __float2half(a[i] * LOSS_SCALE);
}

void resize(Ref& r, uint32_t n, cudaStream_t s) {
    uint32_t n_pad = (n + GRANULARITY - 1) / GRANULARITY * GRANULARITY;
    if (n_pad != r.n_pad) {
        r.in_pad.resize((size_t)n_pad * r.n_input);
        r.din_pad.resize((size_t)n_pad * r.n_input);
        r.out.resize((size_t)n_pad * 16);
        r.dout.resize((size_t)n_pad * 16);
        r.n_pad = n_pad;
    }
    cudaMemsetAsync(r.in_pad.data(), 0, r.in_pad.get_bytes(), s);
}

}  // namespace

extern "C" {

int tcnnref_create(int n_features, int sh_degree, int n_hidden_layers, const char* output_activation, void** out) {
    try {
        json enc = {{"otype", "Composite"},
                    {"nested", json::array({json{{"otype", "Identity"}, {"n_dims_to_encode", n_features}},
                                            json{{"otype", "SphericalHarmonics"}, {"degree", sh_degree}, {"n_dims_to_encode", 3}}})}};
        json net = {{"otype", "FullyFusedMLP"}, {"activation", "ReLU"}, {"output_activation", std::string(output_activation)},
                    {"n_neurons", 128}, {"n_hidden_layers", n_hidden_layers}};
        auto* r = new Ref;
        r->n_input = (uint32_t)n_features + 3;
        r->net = std::make_unique<NetworkWithInputEncoding<T>>(r->n_input, 3u, enc, net);
        r->params.resize(r->net->n_params());
        r->grads.resize(r->net->n_params());
        r->params.memset(0);
        r->grads.memset(0);
        r->net->set_params(r->params.data(), r->params.data(), r->grads.data());
        *out = r;
        return 0;
    } catch (const std::exception& e) {
        fprintf(stderr, "tcnnref_create: %s\n", e.what());
        return 1;
    }
}

void tcnnref_destroy(void* h) { delete static_cast<Ref*>(h); }

int64_t tcnnref_n_params(void* h) { return (int64_t) static_cast<Ref*>(h)->net->n_params(); }

int tcnnref_padded_input_width(void* h) { return (int)static_cast<Ref*>(h)->net->num_encoded_dims(); }

// params: device fp32 [n_params], rounded into tcnn's fp16 parameter buffer
int tcnnref_set_params(void* h, void* stream, const float* params) {
    auto& r = *static_cast<Ref*>(h);
    uint32_t n = (uint32_t)r.net->n_params();
    to_half<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(n, params, r.params.data());
    return cudaGetLastError() != cudaSuccess;
}

// input: device fp32 [n, F+3] (features, then directions already mapped to the unit cube); out: device fp32 [n, 3].
// training != 0 keeps the forward context for tcnnref_backward; otherwise the inference path runs.
int tcnnref_forward(void* h, void* stream, int64_t n, const float* input, float* out, int training) {
    try {
        auto& r = *static_cast<Ref*>(h);
        auto s = (cudaStream_t)stream;
        resize(r, (uint32_t)n, s);
        cudaMemcpyAsync(r.in_pad.data(), input, (size_t)n * r.n_input * sizeof(float), cudaMemcpyDeviceToDevice, s);
        GPUMatrixDynamic<float> in(r.in_pad.data(), r.n_input, r.n_pad, CM);
        GPUMatrixDynamic<T> o(r.out.data(), 16, r.n_pad, CM);
        if (training) {
            r.ctx = r.net->forward(s, in, &o, false, true);
        } else {
            r.net->inference_mixed_precision(s, in, o, false);
        }
        out_to_float<<<((uint32_t)n * 3 + 255) / 256, 256, 0, s>>>((uint32_t)n, r.out.data(), out);
        return cudaGetLastError() != cudaSuccess;
    } catch (const std::exception& e) {
        fprintf(stderr, "tcnnref_forward: %s\n", e.what());
        return 1;
    }
}

// After a training forward on the same input: d_out device fp32 [n, 3] -> d_input [n, F+3] fp32, d_params [n_params] fp32.
int tcnnref_backward(void* h, void* stream, int64_t n, const float* d_out, float* d_input, float* d_params) {
    try {
        auto& r = *static_cast<Ref*>(h);
        auto s = (cudaStream_t)stream;
        if (!r.ctx) return 2;
        cudaMemsetAsync(r.dout.data(), 0, r.dout.get_bytes(), s);
        dout_to_half<<<((uint32_t)n * 3 + 255) / 256, 256, 0, s>>>((uint32_t)n, d_out, r.dout.data());
        GPUMatrixDynamic<float> in(r.in_pad.data(), r.n_input, r.n_pad, CM);
        GPUMatrixDynamic<T> o(r.out.data(), 16, r.n_pad, CM);
        GPUMatrixDynamic<T> dout(r.dout.data(), 16, r.n_pad, CM);
        GPUMatrixDynamic<float> din(r.din_pad.data(), r.n_input, r.n_pad, CM);
        r.net->backward(s, *r.ctx, in, o, dout, &din, false, GradientMode::Overwrite);
        uint32_t np = (uint32_t)r.net->n_params();
        to_float<<<(np + 255) / 256, 256, 0, s>>>(np, 1.0f / LOSS_SCALE, r.grads.data(), d_params);
        uint32_t ni = (uint32_t)n * r.n_input;
        scale_float<<<(ni + 255) / 256, 256, 0, s>>>(ni, 1.0f / LOSS_SCALE, r.din_pad.data(), d_input);
        return cudaGetLastError() != cudaSuccess;
    } catch (const std::exception& e) {
        fprintf(stderr, "tcnnref_backward: %s\n", e.what());
        return 1;
    }
}

}  // extern "C"
