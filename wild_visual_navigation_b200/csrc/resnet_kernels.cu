// wvn-b200: the non-GEMM kernels of the ResNet feature backbone (torchvision ResNet-18 / ResNet-50 behind
// TorchVisionInterface, reference feature_extractor/torchvision_interface.py) and its multiscale segment pooling
// (FeatureExtractor.sparsify_features' feature-pyramid branch, feature_extractor.py:314-366).
//
// Activations are NHWC bf16.  A convolution is an im2col pass (when it is not 1 x 1 / stride 1) followed by the wgmma
// GEMM, whose rows are the output pixels and whose columns are the output channels; batch norm is folded into the
// GEMM's weights and bias on the host.
#include <cuda_bf16.h>

#include <algorithm>

#include "common.cuh"
#include "host_common.h"
#include "resnet_kernels.h"

namespace wvn {

namespace {

inline int grid_for(long long n, int threads) {
  return static_cast<int>(std::max(1ll, std::min<long long>((n + threads - 1) / threads, 65536)));
}

// one thread moves 8 channels (16 bytes) of one window position of one output row
__global__ void __launch_bounds__(256)
im2col_nhwc_kernel(const uint4* __restrict__ in, int batch, int h, int w, int c8, int k, int stride, int pad, int ho,
                   int wo, uint4* __restrict__ out, long long pitch8) {
  const long long per_row = static_cast<long long>(k) * k * c8;
  const long long total = static_cast<long long>(batch) * ho * wo * per_row;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / per_row;
    const int col = static_cast<int>(i - row * per_row);
    const int ch = col % c8, kk = col / c8;
    const int kx = kk % k, ky = kk / k;
    const int ox = static_cast<int>(row % wo);
    const long long t = row / wo;
    const int oy = static_cast<int>(t % ho);
    const int b = static_cast<int>(t / ho);
    const int iy = oy * stride - pad + ky, ix = ox * stride - pad + kx;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (iy >= 0 && iy < h && ix >= 0 && ix < w) v = in[((static_cast<long long>(b) * h + iy) * w + ix) * c8 + ch];
    out[row * pitch8 + col] = v;
  }
}

// one thread writes one element; consecutive threads walk a row's (ky, kx, channel) columns
__global__ void __launch_bounds__(256)
im2col_image_kernel(const float* __restrict__ img, int batch, int h, int w, int k, int stride, int pad, int ho, int wo,
                    __nv_bfloat16* __restrict__ out, long long pitch) {
  const int K = k * k * 3;
  const long long total = static_cast<long long>(batch) * ho * wo * K;
  // torchvision Normalize(mean, std): (x - mean) / std
  const float mean[3] = {0.485f, 0.456f, 0.406f}, sd[3] = {0.229f, 0.224f, 0.225f};
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / K;
    const int col = static_cast<int>(i - row * K);
    const int ch = col % 3, kk = col / 3;
    const int kx = kk % k, ky = kk / k;
    const int ox = static_cast<int>(row % wo);
    const long long t = row / wo;
    const int oy = static_cast<int>(t % ho);
    const int b = static_cast<int>(t / ho);
    const int iy = oy * stride - pad + ky, ix = ox * stride - pad + kx;
    float v = 0.f;  // zero padding of the normalised image (the padding is applied after Normalize)
    if (iy >= 0 && iy < h && ix >= 0 && ix < w)
      v = (__ldg(img + ((static_cast<long long>(b) * 3 + ch) * h + iy) * w + ix) - mean[ch]) / sd[ch];
    out[row * pitch + col] = __float2bfloat16_rn(v);
  }
}

__global__ void __launch_bounds__(256)
maxpool3s2_kernel(const uint4* __restrict__ in, int batch, int h, int w, int c8, int ho, int wo, uint4* __restrict__ out) {
  const long long total = static_cast<long long>(batch) * ho * wo * c8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ch = static_cast<int>(i % c8);
    const long long pix = i / c8;
    const int ox = static_cast<int>(pix % wo);
    const long long t = pix / wo;
    const int oy = static_cast<int>(t % ho);
    const int b = static_cast<int>(t / ho);
    const __nv_bfloat162 ninf = __float2bfloat162_rn(-INFINITY);
    __nv_bfloat162 m[4] = {ninf, ninf, ninf, ninf};
    for (int dy = 0; dy < 3; ++dy) {
      const int iy = 2 * oy - 1 + dy;
      if (iy < 0 || iy >= h) continue;
      for (int dx = 0; dx < 3; ++dx) {
        const int ix = 2 * ox - 1 + dx;
        if (ix < 0 || ix >= w) continue;
        const uint4 v = in[((static_cast<long long>(b) * h + iy) * w + ix) * c8 + ch];
        const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
        for (int j = 0; j < 4; ++j) m[j] = __hmax2(m[j], p[j]);
      }
    }
    out[i] = *reinterpret_cast<const uint4*>(m);
  }
}

constexpr int kPoolThreads = 256;
constexpr int kPoolMaxChannelsPerThread = 8;  // channels up to 2048 (ResNet-50's trunk output)

// One CTA per (segment, frame).  For each level the CTA scans the level's cells in chunks of 256, compacts the cells
// whose nearest-downsampled id equals the segment into shared memory in cell order, and sums their channels in that
// order (one thread per channel), so the result does not depend on scheduling.
__global__ void __launch_bounds__(kPoolThreads)
segment_pool_pyramid_kernel(const long long* __restrict__ seg, const float* __restrict__ centers, PyramidArgs a,
                            float* __restrict__ out) {
  __shared__ int list[kPoolThreads];
  __shared__ int warp_cnt[kPoolThreads / 32];
  const int s = blockIdx.x, b = blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int D = 0;
  for (int l = 0; l < a.levels; ++l) D += a.tc[l];
  float* orow = out + (static_cast<long long>(b) * a.smax + s) * D;
  const long long* segb = seg + static_cast<long long>(b) * a.h * a.w;
  const float cx = centers[(static_cast<long long>(b) * a.smax + s) * 2 + 0];
  const float cy = centers[(static_cast<long long>(b) * a.smax + s) * 2 + 1];
  int off = 0;
  for (int l = 0; l < a.levels; ++l) {
    const int th = a.th[l], tw = a.tw[l], C = a.tc[l], P = a.tp[l];
    const int sy = a.h / th, sx = a.w / tw;  // seg_l[i, j] = seg[i * H / h_l, j * W / w_l]
    const int cells = th * tw;
    const __nv_bfloat16* map = reinterpret_cast<const __nv_bfloat16*>(a.taps[l]) + static_cast<long long>(b) * cells * P;
    float acc[kPoolMaxChannelsPerThread];
#pragma unroll
    for (int j = 0; j < kPoolMaxChannelsPerThread; ++j) acc[j] = 0.f;
    int total = 0;
    for (int base = 0; base < cells; base += kPoolThreads) {
      const int cell = base + tid;
      bool m = false;
      if (cell < cells) {
        const int i = cell / tw, j = cell - i * tw;
        m = segb[static_cast<long long>(i) * sy * a.w + static_cast<long long>(j) * sx] == s;
      }
      const unsigned bal = __ballot_sync(0xffffffffu, m);
      if (lane == 0) warp_cnt[warp] = __popc(bal);
      __syncthreads();
      int pos = 0, n = 0;
#pragma unroll
      for (int wi = 0; wi < kPoolThreads / 32; ++wi) {
        if (wi < warp) pos += warp_cnt[wi];
        n += warp_cnt[wi];
      }
      if (m) list[pos + __popc(bal & ((1u << lane) - 1u))] = cell;
      __syncthreads();
      for (int q = 0; q < n; ++q) {
        const __nv_bfloat16* src = map + static_cast<long long>(list[q]) * P;
#pragma unroll
        for (int j = 0; j < kPoolMaxChannelsPerThread; ++j) {
          const int c = tid + j * kPoolThreads;
          if (c < C) acc[j] += __bfloat162float(src[c]);
        }
      }
      total += n;
      __syncthreads();  // list / warp_cnt are rewritten by the next chunk
    }
    if (total > 0) {
      const float inv = static_cast<float>(total);
#pragma unroll
      for (int j = 0; j < kPoolMaxChannelsPerThread; ++j) {
        const int c = tid + j * kPoolThreads;
        if (c < C) orow[off + c] = acc[j] / inv;
      }
    } else {
      // no cell of this level carries the segment: the cell under its centroid (floor(row * h_l / H), exact because
      // H / h_l is an integer); a segment without pixels has a NaN centroid and gets a NaN row, like the plain pooling
      const bool empty = !(cx == cx) || !(cy == cy);
      const int i = empty ? 0 : min(max(static_cast<int>(floorf(cy / static_cast<float>(sy))), 0), th - 1);
      const int j = empty ? 0 : min(max(static_cast<int>(floorf(cx / static_cast<float>(sx))), 0), tw - 1);
      const __nv_bfloat16* src = map + (static_cast<long long>(i) * tw + j) * P;
      for (int c = tid; c < C; c += kPoolThreads) orow[off + c] = empty ? __int_as_float(0x7fc00000) : __bfloat162float(src[c]);
    }
    off += C;
  }
}

}  // namespace

int im2col_nhwc(const void* in, int batch, int h, int w, int c, int k, int stride, int pad, void* out, long long pitch,
                cudaStream_t stream) {
  WVN_REQUIRE(in && out && batch > 0 && h > 0 && w > 0 && k > 0 && stride > 0 && pad >= 0,
              "im2col: bad arguments (batch=%d h=%d w=%d k=%d stride=%d pad=%d)", batch, h, w, k, stride, pad);
  WVN_REQUIRE(c > 0 && c % 8 == 0, "im2col: channels %d must be a positive multiple of 8", c);
  WVN_REQUIRE(pitch >= static_cast<long long>(k) * k * c && pitch % 8 == 0, "im2col: pitch %lld", pitch);
  const int ho = (h + 2 * pad - k) / stride + 1, wo = (w + 2 * pad - k) / stride + 1;
  WVN_REQUIRE(ho > 0 && wo > 0, "im2col: empty output");
  const long long total = static_cast<long long>(batch) * ho * wo * k * k * (c / 8);
  im2col_nhwc_kernel<<<grid_for(total, 256), 256, 0, stream>>>(reinterpret_cast<const uint4*>(in), batch, h, w, c / 8, k,
                                                               stride, pad, ho, wo, reinterpret_cast<uint4*>(out), pitch / 8);
  WVN_CHECK_LAUNCH("im2col_nhwc_kernel");
  return WVN_OK;
}

int im2col_image(const float* img, int batch, int h, int w, int k, int stride, int pad, void* out, long long pitch,
                 cudaStream_t stream) {
  WVN_REQUIRE(img && out && batch > 0 && h > 0 && w > 0 && k > 0 && stride > 0 && pad >= 0,
              "im2col_image: bad arguments (batch=%d h=%d w=%d k=%d stride=%d pad=%d)", batch, h, w, k, stride, pad);
  WVN_REQUIRE(pitch >= 3ll * k * k && pitch % 8 == 0, "im2col_image: pitch %lld", pitch);
  const int ho = (h + 2 * pad - k) / stride + 1, wo = (w + 2 * pad - k) / stride + 1;
  WVN_REQUIRE(ho > 0 && wo > 0, "im2col_image: empty output");
  const long long total = static_cast<long long>(batch) * ho * wo * k * k * 3;
  im2col_image_kernel<<<grid_for(total, 256), 256, 0, stream>>>(img, batch, h, w, k, stride, pad, ho, wo,
                                                                reinterpret_cast<__nv_bfloat16*>(out), pitch);
  WVN_CHECK_LAUNCH("im2col_image_kernel");
  return WVN_OK;
}

int maxpool3s2_nhwc(const void* in, int batch, int h, int w, int c, void* out, cudaStream_t stream) {
  WVN_REQUIRE(in && out && batch > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0,
              "maxpool: bad arguments (batch=%d h=%d w=%d c=%d)", batch, h, w, c);
  const int ho = (h - 1) / 2 + 1, wo = (w - 1) / 2 + 1;  // (h + 2 - 3) / 2 + 1
  const long long total = static_cast<long long>(batch) * ho * wo * (c / 8);
  maxpool3s2_kernel<<<grid_for(total, 256), 256, 0, stream>>>(reinterpret_cast<const uint4*>(in), batch, h, w, c / 8, ho,
                                                              wo, reinterpret_cast<uint4*>(out));
  WVN_CHECK_LAUNCH("maxpool3s2_kernel");
  return WVN_OK;
}

int segment_pool_pyramid(const long long* seg, const float* centers, const PyramidArgs& a, float* out,
                         cudaStream_t stream) {
  WVN_REQUIRE(seg && centers && out && a.batch > 0 && a.h > 0 && a.w > 0 && a.smax > 0,
              "segment_pool_pyramid: bad arguments (batch=%d h=%d w=%d smax=%d)", a.batch, a.h, a.w, a.smax);
  WVN_REQUIRE(a.batch <= 65535, "segment_pool_pyramid: batch %d", a.batch);
  WVN_REQUIRE(a.levels >= 1 && a.levels <= kPyramidMaxLevels, "segment_pool_pyramid: %d levels (1 .. %d)", a.levels,
              kPyramidMaxLevels);
  for (int l = 0; l < a.levels; ++l) {
    WVN_REQUIRE(a.taps[l] && a.th[l] > 0 && a.tw[l] > 0 && a.h % a.th[l] == 0 && a.w % a.tw[l] == 0,
                "segment_pool_pyramid: level %d is %dx%d, which must divide the %dx%d segmentation", l, a.th[l], a.tw[l],
                a.h, a.w);
    WVN_REQUIRE(a.tc[l] > 0 && a.tc[l] <= kPoolThreads * kPoolMaxChannelsPerThread,
                "segment_pool_pyramid: level %d has %d channels (1 .. %d)", l, a.tc[l],
                kPoolThreads * kPoolMaxChannelsPerThread);
    WVN_REQUIRE(a.tp[l] >= a.tc[l], "segment_pool_pyramid: level %d has pitch %d < %d channels", l, a.tp[l], a.tc[l]);
  }
  segment_pool_pyramid_kernel<<<dim3(a.smax, a.batch), kPoolThreads, 0, stream>>>(seg, centers, a, out);
  WVN_CHECK_LAUNCH("segment_pool_pyramid_kernel");
  return WVN_OK;
}

}  // namespace wvn
