// wvn-b200: the non-GEMM kernels of the EfficientNet-B0 feature backbone (torchvision efficientnet_b0 behind
// TorchVisionInterface): the depthwise convolution of each MBConv block with its folded batch norm and SiLU, and the
// squeeze-excitation (average pool, fc1, SiLU, fc2, sigmoid, channel multiply).
//
// Activations are NHWC bf16 at a channel pitch that is a multiple of 64 (the GEMM's narrowest tile); the pad channels
// hold zeros, which every kernel here keeps at zero (zero weights and bias, SiLU(0) = 0, gate 0).
#include <cuda_bf16.h>

#include <algorithm>

#include "common.cuh"
#include "effnet_kernels.h"
#include "host_common.h"

namespace wvn {

namespace {

constexpr int kDwThreads = 256;
constexpr int kSeThreads = 256;

// as the GEMM's ACT_SILU epilogue
__device__ __forceinline__ float silu(float v) { return __fdividef(v, 1.f + __expf(-v)); }

// One CTA per (block of kDwPoolPixels output pixels, group of up to 32 x 8 channels, frame).  Thread (tx, ty) owns the
// 8 channels of group tx and the block's pixels ty, ty + lanes, ...; it accumulates the window in fp32 in (ky, kx)
// order, stores bf16(SiLU(acc + bias)) and adds that rounded value to its pool sums in pixel order.  The CTA then adds
// the lanes' sums in lane order, so the partial sums do not depend on scheduling.
template <int K>
__global__ void __launch_bounds__(kDwThreads)
depthwise_silu_kernel(const uint4* __restrict__ in, int h, int w, int c8, int stride, int ho, int wo,
                      const float* __restrict__ weight, const float* __restrict__ bias, uint4* __restrict__ out,
                      float* __restrict__ partial, int nblk) {
  __shared__ float red[kDwThreads * 8];
  const int cg = min(c8, 32), lanes = kDwThreads / cg;
  const int tx = threadIdx.x % cg, ty = threadIdx.x / cg;
  const int g = blockIdx.y * cg + tx;
  const int b = blockIdx.z, pb = blockIdx.x;
  const int pitch = c8 * 8, pad = (K - 1) / 2;
  const int hw = ho * wo;
  float sum[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) sum[j] = 0.f;
  if (ty < lanes && g < c8) {
    float bs[8];
    {
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + g * 8));
      const float4 b1 = __ldg(reinterpret_cast<const float4*>(bias + g * 8 + 4));
      bs[0] = b0.x; bs[1] = b0.y; bs[2] = b0.z; bs[3] = b0.w; bs[4] = b1.x; bs[5] = b1.y; bs[6] = b1.z; bs[7] = b1.w;
    }
    const uint4* inb = in + static_cast<long long>(b) * h * w * c8;
    const int p_end = min((pb + 1) * kDwPoolPixels, hw);
    for (int p = pb * kDwPoolPixels + ty; p < p_end; p += lanes) {
      const int oy = p / wo, ox = p - oy * wo;
      float acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
      for (int ky = 0; ky < K; ++ky) {
        const int iy = oy * stride - pad + ky;
        if (iy < 0 || iy >= h) continue;
#pragma unroll
        for (int kx = 0; kx < K; ++kx) {
          const int ix = ox * stride - pad + kx;
          if (ix < 0 || ix >= w) continue;
          const uint4 v = inb[(static_cast<long long>(iy) * w + ix) * c8 + g];
          const float* wp = weight + (ky * K + kx) * pitch + g * 8;
          const float4 w0 = __ldg(reinterpret_cast<const float4*>(wp));
          const float4 w1 = __ldg(reinterpret_cast<const float4*>(wp + 4));
          const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
          const uint32_t xv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            acc[2 * q] = fmaf(bf16_lo(xv[q]), wv[2 * q], acc[2 * q]);
            acc[2 * q + 1] = fmaf(bf16_hi(xv[q]), wv[2 * q + 1], acc[2 * q + 1]);
          }
        }
      }
      uint32_t o[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const __nv_bfloat16 lo = __float2bfloat16_rn(silu(acc[2 * q] + bs[2 * q]));
        const __nv_bfloat16 hi = __float2bfloat16_rn(silu(acc[2 * q + 1] + bs[2 * q + 1]));
        sum[2 * q] += __bfloat162float(lo);
        sum[2 * q + 1] += __bfloat162float(hi);
        o[q] = static_cast<uint32_t>(__bfloat16_as_ushort(lo)) | (static_cast<uint32_t>(__bfloat16_as_ushort(hi)) << 16);
      }
      out[(static_cast<long long>(b) * hw + p) * c8 + g] = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[threadIdx.x * 8 + j] = sum[j];
  __syncthreads();
  // thread t < cg * 8 adds channel t of the CTA's group over the lanes, lane 0 first
  if (static_cast<int>(threadIdx.x) < cg * 8) {
    const int txr = threadIdx.x >> 3, j = threadIdx.x & 7;
    const int gr = blockIdx.y * cg + txr;
    if (gr < c8) {
      float s = 0.f;
      for (int l = 0; l < lanes; ++l) s += red[(l * cg + txr) * 8 + j];
      partial[(static_cast<long long>(b) * nblk + pb) * pitch + gr * 8 + j] = s;
    }
  }
}

// One CTA per frame.  The fc1 dot products are one warp each, lanes striding the channels and combined by a fixed
// butterfly, so every step has a fixed order.
__global__ void __launch_bounds__(kSeThreads)
se_gates_kernel(const float* __restrict__ partial, int nblk, float hw, int channels, int pitch,
                const float* __restrict__ fc1_w, const float* __restrict__ fc1_b, int squeeze,
                const float* __restrict__ fc2_w, const float* __restrict__ fc2_b, float* __restrict__ gates) {
  extern __shared__ float sm[];  // [pitch] means, then [squeeze] hidden
  float* mean = sm;
  float* hid = sm + pitch;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* pb = partial + static_cast<long long>(b) * nblk * pitch;
  for (int c = tid; c < pitch; c += kSeThreads) {
    float s = 0.f;
    for (int q = 0; q < nblk; ++q) s += pb[static_cast<long long>(q) * pitch + c];
    mean[c] = s / hw;
  }
  __syncthreads();
  for (int j = warp; j < squeeze; j += kSeThreads / 32) {
    float s = 0.f;
    for (int c = lane; c < pitch; c += 32) s = fmaf(__ldg(fc1_w + static_cast<long long>(j) * pitch + c), mean[c], s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) hid[j] = silu(s + __ldg(fc1_b + j));
  }
  __syncthreads();
  for (int c = tid; c < pitch; c += kSeThreads) {
    float g = 0.f;
    if (c < channels) {
      float z = __ldg(fc2_b + c);
      for (int j = 0; j < squeeze; ++j) z = fmaf(__ldg(fc2_w + static_cast<long long>(c) * squeeze + j), hid[j], z);
      g = 1.f / (1.f + __expf(-z));
    }
    gates[static_cast<long long>(b) * pitch + c] = g;
  }
}

__global__ void __launch_bounds__(256)
channel_scale_kernel(uint4* __restrict__ x, long long hw, int c8, const float* __restrict__ gates, long long total) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % c8);
    const long long b = i / c8 / hw;
    const float* gp = gates + b * c8 * 8 + g * 8;
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gp));
    const float4 g1 = __ldg(reinterpret_cast<const float4*>(gp + 4));
    const float gv[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    uint4 v = x[i];
    uint32_t* w = reinterpret_cast<uint32_t*>(&v);
#pragma unroll
    for (int q = 0; q < 4; ++q) w[q] = pack_bf16x2(bf16_lo(w[q]) * gv[2 * q], bf16_hi(w[q]) * gv[2 * q + 1]);
    x[i] = v;
  }
}

}  // namespace

int depthwise_silu(const void* in, int batch, int h, int w, int pitch, int k, int stride, const float* weight,
                   const float* bias, void* out, float* partial, cudaStream_t stream) {
  WVN_REQUIRE(in && weight && bias && out && partial && batch > 0 && h > 0 && w > 0,
              "depthwise: bad arguments (batch=%d h=%d w=%d)", batch, h, w);
  WVN_REQUIRE(pitch > 0 && pitch % 8 == 0, "depthwise: channel pitch %d must be a positive multiple of 8", pitch);
  WVN_REQUIRE((k == 3 || k == 5) && (stride == 1 || stride == 2), "depthwise: k=%d stride=%d (k 3 or 5, stride 1 or 2)",
              k, stride);
  WVN_REQUIRE(batch <= 65535, "depthwise: batch %d", batch);
  const int pad = (k - 1) / 2;
  const int ho = (h + 2 * pad - k) / stride + 1, wo = (w + 2 * pad - k) / stride + 1;
  const int c8 = pitch / 8, cg = std::min(c8, 32);
  const int nblk = depthwise_pool_blocks(ho, wo);
  const dim3 grid(nblk, (c8 + cg - 1) / cg, batch);
  auto kern = k == 3 ? depthwise_silu_kernel<3> : depthwise_silu_kernel<5>;
  kern<<<grid, kDwThreads, 0, stream>>>(reinterpret_cast<const uint4*>(in), h, w, c8, stride, ho, wo, weight, bias,
                                        reinterpret_cast<uint4*>(out), partial, nblk);
  WVN_CHECK_LAUNCH("depthwise_silu_kernel");
  return WVN_OK;
}

int se_gates(const float* partial, int batch, int nblk, int hw, int channels, int pitch, const float* fc1_w,
             const float* fc1_b, int squeeze, const float* fc2_w, const float* fc2_b, float* gates, cudaStream_t stream) {
  WVN_REQUIRE(partial && fc1_w && fc1_b && fc2_w && fc2_b && gates && batch > 0 && nblk > 0 && hw > 0,
              "se_gates: bad arguments (batch=%d nblk=%d hw=%d)", batch, nblk, hw);
  WVN_REQUIRE(channels > 0 && channels <= pitch && squeeze > 0 && squeeze <= 1024,
              "se_gates: channels=%d pitch=%d squeeze=%d", channels, pitch, squeeze);
  const size_t smem = (static_cast<size_t>(pitch) + squeeze) * sizeof(float);
  WVN_REQUIRE(smem <= 48 * 1024, "se_gates: pitch %d is too wide", pitch);
  se_gates_kernel<<<batch, kSeThreads, smem, stream>>>(partial, nblk, static_cast<float>(hw), channels, pitch, fc1_w,
                                                       fc1_b, squeeze, fc2_w, fc2_b, gates);
  WVN_CHECK_LAUNCH("se_gates_kernel");
  return WVN_OK;
}

int channel_scale(void* x, int batch, long long hw, int pitch, const float* gates, cudaStream_t stream) {
  WVN_REQUIRE(x && gates && batch > 0 && hw > 0 && pitch > 0 && pitch % 8 == 0,
              "channel_scale: bad arguments (batch=%d hw=%lld pitch=%d)", batch, hw, pitch);
  const long long total = static_cast<long long>(batch) * hw * (pitch / 8);
  const int blocks = static_cast<int>(std::max(1ll, std::min<long long>((total + 255) / 256, 65536)));
  channel_scale_kernel<<<blocks, 256, 0, stream>>>(reinterpret_cast<uint4*>(x), hw, pitch / 8, gates, total);
  WVN_CHECK_LAUNCH("channel_scale_kernel");
  return WVN_OK;
}

}  // namespace wvn
