// wvn-b200: internal interface of effnet_kernels.cu (the non-GEMM kernels of the EfficientNet-B0 backbone).
#pragma once

#include <cuda_runtime.h>

namespace wvn {

// Output pixels whose pool sums one depthwise CTA reduces: partial sums are [batch, depthwise_pool_blocks(ho, wo), pitch].
constexpr int kDwPoolPixels = 64;
inline int depthwise_pool_blocks(int ho, int wo) { return (ho * wo + kDwPoolPixels - 1) / kDwPoolPixels; }

// k x k depthwise convolution (k in {3, 5}, stride in {1, 2}, zero padding (k - 1) / 2) of the NHWC bf16 map
// in [batch, h, w, pitch] (pitch % 8 == 0) -> out [batch, ho, wo, pitch] = bf16(SiLU(conv + bias)), with fp32 weights
// [k, k, pitch] (channel fastest) and bias [pitch].  partial [batch, depthwise_pool_blocks(ho, wo), pitch] receives, per
// block of kDwPoolPixels consecutive output pixels, the per-channel sums of the bf16-rounded outputs (the values the
// squeeze-excitation's average pool reads), each added in a fixed order.
int depthwise_silu(const void* in, int batch, int h, int w, int pitch, int k, int stride, const float* weight,
                   const float* bias, void* out, float* partial, cudaStream_t stream);

// Squeeze-excitation gates of each frame: mean = (sum over the nblk partial rows, in order) / hw, then
// gates[b, c] = sigmoid(fc2(SiLU(fc1(mean)))) for c < channels and 0 for c in [channels, pitch).
// fc1: weight [squeeze, pitch] (columns past `channels` zero), bias [squeeze]; fc2: weight [pitch, squeeze], bias [pitch].
int se_gates(const float* partial, int batch, int nblk, int hw, int channels, int pitch, const float* fc1_w,
             const float* fc1_b, int squeeze, const float* fc2_w, const float* fc2_b, float* gates, cudaStream_t stream);

// In place: x[b, p, c] = bf16(x[b, p, c] * gates[b, c]) for the NHWC bf16 map x [batch, hw, pitch] (pitch % 8 == 0).
int channel_scale(void* x, int batch, long long hw, int pitch, const float* gates, cudaStream_t stream);

}  // namespace wvn
