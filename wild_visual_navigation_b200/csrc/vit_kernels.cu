// wvn-b200: memory-bound helper kernels of the ViT forward pass (sm_90a).
//
//   image_to_patches   : NEAREST resize + center crop + ImageNet normalisation + im2col -> bf16
//                        (reference: dino_interface.py:52-59,81 transform, then the DINO
//                         PatchEmbed Conv2d(3, D, p, p) expressed as a GEMM — SURVEY.md K1).
//                        Source is either the float CHW tensor the reference hands to the interface or
//                        (SURVEY.md §8f rank 1) the camera's uint8 HWC frame itself: ToTensor's `/ 255`
//                        (ros_converter.py:113-126) and ImageProjector.resize_image's NEAREST resize +
//                        center crop (image_projector.py:55-59,199-200) happen inside the loader.
//   init_token_rows    : CLS row (cls_token + pos_embed[0]) and zeroed padding rows
//   layernorm_rows     : LayerNorm(D, eps) over the fp32 residual stream -> bf16 GEMM operand
//                        (optionally also the fp32 patch-token output, CLS dropped — K2/K7)
#include "common.cuh"
#include "host_common.h"
#include "vit_kernels.h"

namespace wvn {

namespace {

// One thread produces G consecutive K-elements of one patch row of one channel (G = 8 for p = 8 / 16, a whole row of
// 14 for p = 14): reads G floats that are contiguous in the source row when no resize happens.  Output rows are
// patch_pitch(p) elements apart; the pad columns [3 p p, pitch) are never written (the GEMM does not read them).
template <bool U8_HWC, int G>
__global__ void image_to_patches_kernel(const void* __restrict__ img_raw, __nv_bfloat16* __restrict__ out,
                                        ImagePatchArgs a) {
  const float* img = reinterpret_cast<const float*>(img_raw);
  const unsigned char* img8 = reinterpret_cast<const unsigned char*>(img_raw);
  const int ps = a.patch;
  const int k_total = 3 * ps * ps;
  const int pitch = patch_pitch(ps);
  const int groups_per_row = k_total / G;
  const long long total = static_cast<long long>(a.batch) * a.grid_h * a.grid_w * groups_per_row;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(idx % groups_per_row);
    const long long prow = idx / groups_per_row;  // patch row index in [0, B*P)
    const int pw = static_cast<int>(prow % a.grid_w);
    const int ph = static_cast<int>((prow / a.grid_w) % a.grid_h);
    const int b = static_cast<int>(prow / (static_cast<long long>(a.grid_w) * a.grid_h));
    const int k0 = g * G;  // k = c*ps*ps + ky*ps + kx
    const int c = k0 / (ps * ps);
    const int ky = (k0 / ps) % ps;
    const int kx0 = k0 % ps;
    // destination pixel in the cropped (size x size) image
    const int y = ph * ps + ky;
    // torch 'nearest': src = min(floor(dst * scale), in - 1), scale = in / out in fp32
    const int sy = min(static_cast<int>(floorf((y + a.crop_top) * a.scale_y)), a.in_h - 1);
    const float mean = a.mean[c], inv_std = a.inv_std[c];
    const int gb = a.frame0 + b;
    const bool flip = gb >= a.flip_from;
    const int sb = gb % a.src_frames;
    const float* src_row = img + ((static_cast<long long>(sb) * 3 + c) * a.in_h + sy) * a.in_w;
    const unsigned char* src_row8 = img8 + (static_cast<long long>(sb) * a.in_h + sy) * a.in_w * 3 + c;
    float v[G];
#pragma unroll
    for (int i = 0; i < G; ++i) {
      const int xo = pw * ps + kx0 + i;
      // the flip mirrors the whole crop: when patch does not divide it, the patches of the flipped image do not cover
      // its last crop - grid_w * ps columns, which are the first columns of the straight image
      const int x = flip ? a.crop - 1 - xo : xo;
      const int sx = min(static_cast<int>(floorf((x + a.crop_left) * a.scale_x)), a.in_w - 1);
      // uint8: the same IEEE division torchvision's ToTensor performs, so both sources give identical patches
      const float px = U8_HWC ? static_cast<float>(__ldg(src_row8 + 3 * sx)) / 255.f : __ldg(src_row + sx);
      v[i] = (px - mean) * inv_std;
    }
    __nv_bfloat16* dst = out + prow * pitch + k0;
    if (G == 8) {
      st_global_v4(dst, pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]),
                   pack_bf16x2(v[6], v[7]));
    } else {
      // 14 elements at a 28-byte offset inside the row: 4-byte aligned pairs
#pragma unroll
      for (int i = 0; i < G; i += 2) *reinterpret_cast<uint32_t*>(dst + i) = pack_bf16x2(v[i], v[i + 1]);
    }
  }
}

__global__ void init_token_rows_kernel(float* __restrict__ x, const float* __restrict__ cls,
                                       const float* __restrict__ pos, const float* __restrict__ reg, int registers,
                                       int batch, int npad, int n_valid, int dim) {
  // rows handled per frame: row 0 (CLS), rows [1, 1 + registers) (register tokens, no position embedding) and rows
  // [n_valid, npad) (padding)
  const int head_rows = 1 + registers;
  const int rows_per_frame = head_rows + (npad - n_valid);
  const long long total = static_cast<long long>(batch) * rows_per_frame * dim;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int d = static_cast<int>(idx % dim);
    const long long r = idx / dim;
    const int rr = static_cast<int>(r % rows_per_frame);
    const int b = static_cast<int>(r / rows_per_frame);
    const int row = (rr < head_rows) ? rr : (n_valid + rr - head_rows);
    const float v = (rr == 0) ? (cls[d] + pos[d]) : (rr < head_rows ? reg[static_cast<long long>(rr - 1) * dim + d] : 0.f);
    x[(static_cast<long long>(b) * npad + row) * dim + d] = v;
  }
}

// One warp per row, D = 128 * VEC_ITERS (384 -> 3, 768 -> 6, 1024 -> 8, 1536 -> 12).  Two-pass statistics in
// registers (mean, then centred variance) — the same arithmetic order class as torch's LN.
template <int ITERS>
__global__ void __launch_bounds__(256)
layernorm_rows_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                      __nv_bfloat16* __restrict__ out_bf16, float* __restrict__ out_f32, LayerNormArgs a) {
  constexpr int D = 128 * ITERS;
  const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int warps_total = (gridDim.x * blockDim.x) >> 5;
  for (long long r = warp_global; r < a.rows; r += warps_total) {
    const long long row = a.reverse ? a.rows - 1 - r : r;
    const float4* src = reinterpret_cast<const float4*>(x + row * D);
    float4 v[ITERS];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < ITERS; ++i) {
      v[i] = src[lane + 32 * i];
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
    const float mean = warp_sum(s) * (1.f / D);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < ITERS; ++i) {
      const float dx = v[i].x - mean, dy = v[i].y - mean, dz = v[i].z - mean, dw = v[i].w - mean;
      q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
    }
    const float rstd = rsqrtf(warp_sum(q) * (1.f / D) + a.eps);
    // optional fp32 output: only real patch tokens (CLS, register and padding rows dropped)
    long long f32_row = -1;
    if (out_f32 != nullptr) {
      const int tok = static_cast<int>(row % a.npad);
      const long long frame = row / a.npad;
      if (tok >= a.row0 && tok < a.n_valid) f32_row = frame * (a.n_valid - a.row0) + (tok - a.row0);
    }
#pragma unroll
    for (int i = 0; i < ITERS; ++i) {
      const int c4 = lane + 32 * i;
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + c4);
      const float4 bt = __ldg(reinterpret_cast<const float4*>(beta) + c4);
      float4 y;
      y.x = (v[i].x - mean) * rstd * g.x + bt.x;
      y.y = (v[i].y - mean) * rstd * g.y + bt.y;
      y.z = (v[i].z - mean) * rstd * g.z + bt.z;
      y.w = (v[i].w - mean) * rstd * g.w + bt.w;
      if (out_bf16 != nullptr) {
        uint2 p = make_uint2(pack_bf16x2(y.x, y.y), pack_bf16x2(y.z, y.w));
        *reinterpret_cast<uint2*>(out_bf16 + row * D + 4 * c4) = p;
      }
      if (f32_row >= 0) reinterpret_cast<float4*>(out_f32 + f32_row * D)[c4] = y;
    }
  }
}


// ---- parity-debug attention (SURVEY.md §7 "an fp32 mode kept for debugging parity"; $WVN_VIT_PRECISE=1) ----------------
// softmax(q k^T * scale) v in fp32 CUDA-core arithmetic on the fp32 QKV projections: no bf16 rounding of q, k, v, of the
// scores or of P.  One thread = one query row (q and the output accumulator in registers), K / V tiles of 64 keys staged
// in shared memory, online softmax per 16-key chunk.  ~40x slower than the wgmma kernel; it exists to separate
// "kernel bug" from "bf16 rounding of peaked attention logits" (tests/test_path_gpu.py::test_vit_base_default_std...).
__global__ void __launch_bounds__(128)
attention_f32_debug_kernel(const float* __restrict__ qkv, __nv_bfloat16* __restrict__ out, int npad, int n_valid, int heads,
                           int dim, float scale) {
  __shared__ float ks[64][65];
  __shared__ float vs[64][65];
  const int h = blockIdx.y, b = blockIdx.z;
  const int qi = blockIdx.x * 128 + threadIdx.x;
  const long long row0 = static_cast<long long>(b) * npad;
  const int ld = 3 * dim;
  float q[64], o[64];
  const bool active = qi < npad;
#pragma unroll
  for (int d = 0; d < 64; ++d) {
    q[d] = active ? qkv[(row0 + qi) * ld + h * 64 + d] * scale : 0.f;
    o[d] = 0.f;
  }
  float m = -INFINITY, l = 0.f;
  for (int k0 = 0; k0 < n_valid; k0 += 64) {
    __syncthreads();
    for (int i = threadIdx.x; i < 64 * 64; i += 128) {
      const int kk = i >> 6, d = i & 63;
      const bool ok = k0 + kk < n_valid;
      ks[kk][d] = ok ? qkv[(row0 + k0 + kk) * ld + dim + h * 64 + d] : 0.f;
      vs[kk][d] = ok ? qkv[(row0 + k0 + kk) * ld + 2 * dim + h * 64 + d] : 0.f;
    }
    __syncthreads();
    for (int c0 = 0; c0 < 64; c0 += 16) {
      float sc[16], cmax = -INFINITY;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float acc = 0.f;
#pragma unroll
        for (int d = 0; d < 64; ++d) acc = fmaf(q[d], ks[c0 + j][d], acc);
        sc[j] = (k0 + c0 + j < n_valid) ? acc : -INFINITY;
        cmax = fmaxf(cmax, sc[j]);
      }
      if (cmax == -INFINITY) continue;
      const float m_new = fmaxf(m, cmax);
      const float alpha = expf(m - m_new);   // exp(-inf) = 0 on the first chunk
      l *= alpha;
#pragma unroll
      for (int d = 0; d < 64; ++d) o[d] *= alpha;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float p = expf(sc[j] - m_new);
        l += p;
#pragma unroll
        for (int d = 0; d < 64; ++d) o[d] = fmaf(p, vs[c0 + j][d], o[d]);
      }
      m = m_new;
    }
  }
  if (active) {
    const float inv = 1.f / l;
    __nv_bfloat16* dst = out + (row0 + qi) * dim + h * 64;
#pragma unroll
    for (int d = 0; d < 64; ++d) dst[d] = __float2bfloat16_rn(o[d] * inv);
  }
}

}  // namespace

int image_patch_args(int batch, int in_h, int in_w, int resized_h, int resized_w, int image_size, int patch, int frame0,
                     int src_frames, int flip_from, ImagePatchArgs* a) {
  WVN_REQUIRE(a != nullptr, "image_patch_args: null argument");
  WVN_REQUIRE(patch == 8 || patch == 14 || patch == 16, "image_to_patches: patch size %d unsupported", patch);
  WVN_REQUIRE(batch > 0 && in_h > 0 && in_w > 0 && image_size >= patch, "image_to_patches: empty problem");
  WVN_REQUIRE(resized_h >= image_size && resized_w >= image_size,
              "image_to_patches: resized image %dx%d smaller than the crop %d", resized_h, resized_w, image_size);
  WVN_REQUIRE(frame0 >= 0 && src_frames > 0, "image_to_patches: frame0 %d, src_frames %d", frame0, src_frames);
  ImagePatchArgs r;
  r.batch = batch;
  r.in_h = in_h; r.in_w = in_w; r.patch = patch;
  r.grid_h = r.grid_w = image_size / patch;
  r.crop = image_size;
  // torchvision CenterCrop: top = int(round((H - size) / 2.0)); lrintf rounds half to even, as Python's round does
  r.crop_top = static_cast<int>(lrintf((resized_h - image_size) / 2.0f));
  r.crop_left = static_cast<int>(lrintf((resized_w - image_size) / 2.0f));
  // torch 'nearest' with an output size: scale = (float)in / out
  r.scale_y = static_cast<float>(in_h) / static_cast<float>(resized_h);
  r.scale_x = static_cast<float>(in_w) / static_cast<float>(resized_w);
  r.frame0 = frame0; r.src_frames = src_frames; r.flip_from = flip_from;
  *a = r;
  return WVN_OK;
}

int image_to_patches(const void* img, bool u8_hwc, void* out_bf16, const ImagePatchArgs& a, cudaStream_t stream) {
  WVN_REQUIRE(a.patch == 8 || a.patch == 14 || a.patch == 16, "image_to_patches: patch size %d unsupported", a.patch);
  const int group = a.patch == 14 ? 14 : 8;
  const long long total = static_cast<long long>(a.batch) * a.grid_h * a.grid_w * (3 * a.patch * a.patch / group);
  const int threads = 256;
  long long blocks = (total + threads - 1) / threads;
  const long long max_blocks = static_cast<long long>(sm_count()) * 16;
  if (blocks > max_blocks) blocks = max_blocks;
  __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(out_bf16);
  const unsigned nb = static_cast<unsigned>(blocks);
  if (group == 14) {
    if (u8_hwc) image_to_patches_kernel<true, 14><<<nb, threads, 0, stream>>>(img, out, a);
    else image_to_patches_kernel<false, 14><<<nb, threads, 0, stream>>>(img, out, a);
  } else {
    if (u8_hwc) image_to_patches_kernel<true, 8><<<nb, threads, 0, stream>>>(img, out, a);
    else image_to_patches_kernel<false, 8><<<nb, threads, 0, stream>>>(img, out, a);
  }
  WVN_CHECK_LAUNCH("image_to_patches_kernel");
  return WVN_OK;
}

int init_token_rows(float* x, const float* cls, const float* pos, const float* reg, int registers, int batch, int npad,
                    int n_valid, int dim, cudaStream_t stream) {
  WVN_REQUIRE(registers >= 0 && (registers == 0 || reg != nullptr), "init_token_rows: %d registers without their weights",
              registers);
  const long long total = static_cast<long long>(batch) * (1 + registers + npad - n_valid) * dim;
  const int threads = 256;
  long long blocks = (total + threads - 1) / threads;
  if (blocks > 4096) blocks = 4096;
  init_token_rows_kernel<<<static_cast<unsigned>(blocks), threads, 0, stream>>>(x, cls, pos, reg, registers, batch, npad,
                                                                                n_valid, dim);
  WVN_CHECK_LAUNCH("init_token_rows_kernel");
  return WVN_OK;
}

int layernorm_rows(const float* x, const float* gamma, const float* beta, void* out_bf16, float* out_f32,
                   const LayerNormArgs& a, cudaStream_t stream) {
  WVN_REQUIRE(a.dim == 384 || a.dim == 768 || a.dim == 1024 || a.dim == 1536,
              "layernorm: dim %d unsupported (384, 768, 1024 or 1536)", a.dim);
  const int threads = 256;
  long long blocks = (a.rows * 32 + threads - 1) / threads;
  const long long max_blocks = static_cast<long long>(sm_count()) * 8;
  if (blocks > max_blocks) blocks = max_blocks;
  if (a.dim == 384)
    layernorm_rows_kernel<3><<<static_cast<unsigned>(blocks), threads, 0, stream>>>(
        x, gamma, beta, reinterpret_cast<__nv_bfloat16*>(out_bf16), out_f32, a);
  else if (a.dim == 768)
    layernorm_rows_kernel<6><<<static_cast<unsigned>(blocks), threads, 0, stream>>>(
        x, gamma, beta, reinterpret_cast<__nv_bfloat16*>(out_bf16), out_f32, a);
  else if (a.dim == 1024)
    layernorm_rows_kernel<8><<<static_cast<unsigned>(blocks), threads, 0, stream>>>(
        x, gamma, beta, reinterpret_cast<__nv_bfloat16*>(out_bf16), out_f32, a);
  else
    layernorm_rows_kernel<12><<<static_cast<unsigned>(blocks), threads, 0, stream>>>(
        x, gamma, beta, reinterpret_cast<__nv_bfloat16*>(out_bf16), out_f32, a);
  WVN_CHECK_LAUNCH("layernorm_rows_kernel");
  return WVN_OK;
}

int attention_f32_debug(const float* qkv, void* out_bf16, int batch, int heads, int npad, int n_valid, int dim, float scale,
                        cudaStream_t stream) {
  WVN_REQUIRE(dim == heads * 64, "attention_f32_debug: head dim must be 64");
  dim3 grid((npad + 127) / 128, heads, batch);
  attention_f32_debug_kernel<<<grid, 128, 0, stream>>>(qkv, reinterpret_cast<__nv_bfloat16*>(out_bf16), npad, n_valid, heads,
                                                      dim, scale);
  WVN_CHECK_LAUNCH("attention_f32_debug_kernel");
  return WVN_OK;
}

}  // namespace wvn
