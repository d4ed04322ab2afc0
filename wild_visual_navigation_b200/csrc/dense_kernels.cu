// wvn-b200: kernels between the ViT token grid and image resolution (sm_90a).
//
//   upsample_tokens_dense : F.interpolate(features, (H,H), "bilinear", align_corners=True)
//                           (reference: dino_interface.py:87-90, stego_interface.py:107) —
//                           only launched when a caller insists on the materialised
//                           (B, D, H, H) tensor (`return_dense_features=True`).
//   interp_pixel_rows     : the same interpolation, but emitted as bf16 rows [pixels, D] that
//                           feed the per-pixel traversability MLP GEMMs (replaces
//                           `dense_feat[0].permute(1,2,0).reshape(-1, D)`,
//                           wvn_feature_extractor_node.py:320-322) for a range of pixels.
//   logits_argmax         : bilinear (align_corners=False) upsampling of per-patch class
//                           logits + per-pixel argmax -> segment ids (STEGO postprocess,
//                           SURVEY.md §8 a4 [EXTERNAL-RECALLED]); exact because the cluster /
//                           linear probes are affine in the code and argmax ignores the
//                           positive per-pixel normalisation.
#include "common.cuh"
#include "dense_kernels.h"

#include <algorithm>
#include "host_common.h"

namespace wvn {

namespace {

// align_corners=True source coordinate: src = dst * (in - 1) / (out - 1)
__device__ __forceinline__ void ac_true_coord(int dst, float scale, int in_size, int& i0, int& i1, float& w1) {
  const float s = dst * scale;
  i0 = min(static_cast<int>(s), in_size - 1);
  i1 = min(i0 + 1, in_size - 1);
  w1 = s - static_cast<float>(i0);
}

// align_corners=False: src = max((dst + 0.5) * in/out - 0.5, 0)
__device__ __forceinline__ void ac_false_coord(int dst, float scale, int in_size, int& i0, int& i1, float& w1) {
  float s = (dst + 0.5f) * scale - 0.5f;
  s = fmaxf(s, 0.f);
  i0 = min(static_cast<int>(s), in_size - 1);
  i1 = min(i0 + 1, in_size - 1);
  w1 = s - static_cast<float>(i0);
}

// grid: (out_h, ceil(C/32), B); block: 256 threads.  Stages the two source token rows for 32
// channels in shared memory, then writes 32 channel rows of out_w pixels, coalesced along x.
__global__ void __launch_bounds__(256)
upsample_tokens_dense_kernel(const float* __restrict__ tok, float* __restrict__ out, DenseArgs a) {
  extern __shared__ float sm[];  // [2][grid_w][33]
  const int y = blockIdx.x, c0 = blockIdx.y * 32, b = blockIdx.z;
  int y0, y1;
  float wy;
  ac_true_coord(y, a.scale_y, a.grid_h, y0, y1, wy);
  const float* base = tok + static_cast<long long>(b) * a.grid_h * a.grid_w * a.dim;
  for (int i = threadIdx.x; i < 2 * a.grid_w * 32; i += blockDim.x) {
    const int c = i & 31;
    const int gx = (i >> 5) % a.grid_w;
    const int r = (i >> 5) / a.grid_w;
    const int gy = r == 0 ? y0 : y1;
    sm[(r * a.grid_w + gx) * 33 + c] =
        (c0 + c < a.dim) ? base[(static_cast<long long>(gy) * a.grid_w + gx) * a.dim + c0 + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 32 * a.out_w; i += blockDim.x) {
    const int x = i % a.out_w;
    const int c = i / a.out_w;
    if (c0 + c >= a.dim) continue;
    int x0, x1;
    float wx;
    ac_true_coord(x, a.scale_x, a.grid_w, x0, x1, wx);
    const float v00 = sm[(x0)*33 + c], v01 = sm[(x1)*33 + c];
    const float v10 = sm[(a.grid_w + x0) * 33 + c], v11 = sm[(a.grid_w + x1) * 33 + c];
    // same operation order as ATen's upsample_bilinear2d: blend x within each row, then y
    const float top = (1.f - wx) * v00 + wx * v01;
    const float bot = (1.f - wx) * v10 + wx * v11;
    out[((static_cast<long long>(b) * a.dim + c0 + c) * a.out_h + y) * a.out_w + x] = (1.f - wy) * top + wy * bot;
  }
}

// One warp per pixel; lanes stride the feature dimension in float4s.
__global__ void __launch_bounds__(256)
interp_pixel_rows_kernel(const float* __restrict__ tok, __nv_bfloat16* __restrict__ out, DenseArgs a,
                         long long pix0, long long npix) {
  const int lane = threadIdx.x & 31;
  const long long warp_global = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const long long warps_total = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const int vecs = a.dim >> 2;
  for (long long i = warp_global; i < npix; i += warps_total) {
    const long long p = pix0 + i;
    const int x = static_cast<int>(p % a.out_w);
    const int y = static_cast<int>((p / a.out_w) % a.out_h);
    const long long b = p / (static_cast<long long>(a.out_w) * a.out_h);
    int x0, x1, y0, y1;
    float wx, wy;
    ac_true_coord(x, a.scale_x, a.grid_w, x0, x1, wx);
    ac_true_coord(y, a.scale_y, a.grid_h, y0, y1, wy);
    const float* base = tok + b * a.grid_h * a.grid_w * a.dim;
    const float4* r00 = reinterpret_cast<const float4*>(base + (static_cast<long long>(y0) * a.grid_w + x0) * a.dim);
    const float4* r01 = reinterpret_cast<const float4*>(base + (static_cast<long long>(y0) * a.grid_w + x1) * a.dim);
    const float4* r10 = reinterpret_cast<const float4*>(base + (static_cast<long long>(y1) * a.grid_w + x0) * a.dim);
    const float4* r11 = reinterpret_cast<const float4*>(base + (static_cast<long long>(y1) * a.grid_w + x1) * a.dim);
    __nv_bfloat16* dst = out + i * a.ld_out;
    if (a.dim & 3) {  // rows are not 16-byte aligned (the 90-d STEGO code): scalar channels
      const float* s00 = reinterpret_cast<const float*>(r00);
      const float* s01 = reinterpret_cast<const float*>(r01);
      const float* s10 = reinterpret_cast<const float*>(r10);
      const float* s11 = reinterpret_cast<const float*>(r11);
      for (int c = lane; c < a.dim; c += 32)
        dst[c] = __float2bfloat16_rn((1.f - wy) * ((1.f - wx) * __ldg(s00 + c) + wx * __ldg(s01 + c)) +
                                     wy * ((1.f - wx) * __ldg(s10 + c) + wx * __ldg(s11 + c)));
      continue;
    }
    for (int v = lane; v < vecs; v += 32) {
      const float4 a00 = __ldg(r00 + v), a01 = __ldg(r01 + v), a10 = __ldg(r10 + v), a11 = __ldg(r11 + v);
      float4 o;
      o.x = (1.f - wy) * ((1.f - wx) * a00.x + wx * a01.x) + wy * ((1.f - wx) * a10.x + wx * a11.x);
      o.y = (1.f - wy) * ((1.f - wx) * a00.y + wx * a01.y) + wy * ((1.f - wx) * a10.y + wx * a11.y);
      o.z = (1.f - wy) * ((1.f - wx) * a00.z + wx * a01.z) + wy * ((1.f - wx) * a10.z + wx * a11.z);
      o.w = (1.f - wy) * ((1.f - wx) * a00.w + wx * a01.w) + wy * ((1.f - wx) * a10.w + wx * a11.w);
      *reinterpret_cast<uint2*>(dst + 4 * v) = make_uint2(pack_bf16x2(o.x, o.y), pack_bf16x2(o.z, o.w));
    }
  }
}

// One thread per output pixel: bilinear blend of the class logits of the 4 neighbouring patches
// (float4 loads), running argmax (first maximum wins, like torch.argmax).  Up to two logit ranges
// (STEGO cluster probe and linear probe) are resolved in the same pass.
__global__ void __launch_bounds__(256)
logits_argmax_kernel(const float* __restrict__ logits, long long* __restrict__ seg_a, long long* __restrict__ seg_b,
                     LogitsArgs a) {
  const long long total = static_cast<long long>(a.batch) * a.out_h * a.out_w;
  for (long long p = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; p < total;
       p += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(p % a.out_w);
    const int y = static_cast<int>((p / a.out_w) % a.out_h);
    const long long b = p / (static_cast<long long>(a.out_w) * a.out_h);
    int x0, x1, y0, y1;
    float wx, wy;
    ac_false_coord(x, a.scale_x, a.grid_w, x0, x1, wx);
    ac_false_coord(y, a.scale_y, a.grid_h, y0, y1, wy);
    const float w00 = (1.f - wy) * (1.f - wx), w01 = (1.f - wy) * wx, w10 = wy * (1.f - wx), w11 = wy * wx;
    // token row of patch (gy, gx) in the padded activation layout: b*npad + 1 + gy*gw + gx
    const float* base = logits + (b * a.npad + 1) * a.ld;
    const float* r00 = base + (static_cast<long long>(y0) * a.grid_w + x0) * a.ld;
    const float* r01 = base + (static_cast<long long>(y0) * a.grid_w + x1) * a.ld;
    const float* r10 = base + (static_cast<long long>(y1) * a.grid_w + x0) * a.ld;
    const float* r11 = base + (static_cast<long long>(y1) * a.grid_w + x1) * a.ld;
#pragma unroll
    for (int range = 0; range < 2; ++range) {
      const int col0 = range == 0 ? a.col0 : a.col0_b;
      const int classes = range == 0 ? a.classes : a.classes_b;
      long long* out = range == 0 ? seg_a : seg_b;
      if (out == nullptr || classes <= 0) continue;
      float best = -INFINITY;
      int arg = 0;
      for (int k4 = 0; k4 < classes; k4 += 4) {
        const float4 a00 = __ldg(reinterpret_cast<const float4*>(r00 + col0 + k4));
        const float4 a01 = __ldg(reinterpret_cast<const float4*>(r01 + col0 + k4));
        const float4 a10 = __ldg(reinterpret_cast<const float4*>(r10 + col0 + k4));
        const float4 a11 = __ldg(reinterpret_cast<const float4*>(r11 + col0 + k4));
        // same grouping as ATen: blend x inside each row, then y  ((1-wy)*((1-wx)a+wx b) + wy*(...))
        const float v[4] = {
            (1.f - wy) * ((1.f - wx) * a00.x + wx * a01.x) + wy * ((1.f - wx) * a10.x + wx * a11.x),
            (1.f - wy) * ((1.f - wx) * a00.y + wx * a01.y) + wy * ((1.f - wx) * a10.y + wx * a11.y),
            (1.f - wy) * ((1.f - wx) * a00.z + wx * a01.z) + wy * ((1.f - wx) * a10.z + wx * a11.z),
            (1.f - wy) * ((1.f - wx) * a00.w + wx * a01.w) + wy * ((1.f - wx) * a10.w + wx * a11.w)};
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (k4 + i < classes && v[i] > best) { best = v[i]; arg = k4 + i; }
      }
      out[p] = arg;
    }
    (void)w00; (void)w01; (void)w10; (void)w11;
  }
}

}  // namespace

int upsample_tokens_dense(const float* tokens, float* out, const DenseArgs& a, cudaStream_t stream) {
  WVN_REQUIRE(a.batch > 0 && a.dim > 0 && a.grid_h > 0 && a.grid_w > 0, "upsample: empty problem");
  dim3 grid(a.out_h, (a.dim + 31) / 32, a.batch);
  const size_t smem = static_cast<size_t>(2) * a.grid_w * 33 * sizeof(float);
  upsample_tokens_dense_kernel<<<grid, 256, smem, stream>>>(tokens, out, a);
  WVN_CHECK_LAUNCH("upsample_tokens_dense_kernel");
  return WVN_OK;
}

int interp_pixel_rows(const float* tokens, void* out_bf16, const DenseArgs& a, long long pix0, long long npix,
                      cudaStream_t stream) {
  WVN_REQUIRE(a.dim > 0 && a.ld_out >= a.dim && a.ld_out % 4 == 0, "interp_pixel_rows: bad dims");
  if (npix <= 0) return WVN_OK;
  long long blocks = (npix * 32 + 255) / 256;
  const long long max_blocks = static_cast<long long>(sm_count()) * 16;
  if (blocks > max_blocks) blocks = max_blocks;
  interp_pixel_rows_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
      tokens, reinterpret_cast<__nv_bfloat16*>(out_bf16), a, pix0, npix);
  WVN_CHECK_LAUNCH("interp_pixel_rows_kernel");
  return WVN_OK;
}

int logits_argmax(const float* logits, long long* seg, long long* seg_b, const LogitsArgs& a, cudaStream_t stream) {
  WVN_REQUIRE(a.classes > 0 && a.batch > 0, "logits_argmax: empty problem");
  WVN_REQUIRE(a.col0 % 4 == 0 && a.col0_b % 4 == 0 && a.ld % 4 == 0, "logits_argmax: columns must be float4-aligned");
  const long long total = static_cast<long long>(a.batch) * a.out_h * a.out_w;
  long long blocks = (total + 255) / 256;
  const long long max_blocks = static_cast<long long>(sm_count()) * 16;
  if (blocks > max_blocks) blocks = max_blocks;
  logits_argmax_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(logits, seg, seg_b, a);
  WVN_CHECK_LAUNCH("logits_argmax_kernel");
  return WVN_OK;
}

namespace {
__global__ void __launch_bounds__(256)
flip_average_kernel(float* __restrict__ head, int batch, int npad, int grid, long long ld) {
  const long long per_frame = static_cast<long long>(npad) * ld;
  const long long total = batch * per_frame;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long b = i / per_frame, rem = i - b * per_frame;
    const int row = static_cast<int>(rem / ld), c = static_cast<int>(rem - static_cast<long long>(row) * ld);
    const int p = row - 1;
    float v = 0.f;
    if (p >= 0 && p < grid * grid) {
      const int y = p / grid, x = p - y * grid;
      const long long mirrored = (static_cast<long long>(batch + b) * npad + 1 + y * grid + (grid - 1 - x)) * ld + c;
      v = 0.5f * (head[i] + head[mirrored]);   // the flipped pass's rows are only read
    }
    head[i] = v;
  }
}
}  // namespace

int flip_average(float* head, int batch, int npad, int grid, long long ld, cudaStream_t stream) {
  WVN_REQUIRE(head && batch > 0 && npad > grid * grid && ld > 0, "flip_average: bad arguments");
  const long long total = static_cast<long long>(batch) * npad * ld;
  const int blocks = static_cast<int>(std::min<long long>((total + 255) / 256, static_cast<long long>(sm_count()) * 16));
  flip_average_kernel<<<blocks, 256, 0, stream>>>(head, batch, npad, grid, ld);
  WVN_CHECK_LAUNCH("flip_average_kernel");
  return WVN_OK;
}

}  // namespace wvn
