// wvn-b200: internal interface of the memory-bound ViT helper kernels (vit_kernels.cu).
#pragma once

#include <cuda_runtime.h>

namespace wvn {

struct ImagePatchArgs {
  int batch = 0;
  int in_h = 0, in_w = 0;        // source image size
  int patch = 8;
  int grid_h = 0, grid_w = 0;    // patches per column / row of the cropped image
  int crop = 0;                  // side of the (square) cropped image; grid * patch < crop when patch does not divide it
  int crop_top = 0, crop_left = 0;  // center-crop offsets in the (virtually) resized image
  float scale_y = 1.f, scale_x = 1.f;  // in / resized (torch 'nearest' source index scale)
  // Test-time-augmentation passes: output frame f reads source frame (frame0 + f) % src_frames, and frames with
  // frame0 + f >= flip_from are the horizontal flip of the TRANSFORMED (resized + cropped) image, as Stego.get_code
  // flips its already-transformed input: column x of the flipped image is column crop - 1 - x of the crop (the whole
  // crop, not just the grid * patch columns the patches cover).  Defaults = identity.
  int frame0 = 0, src_frames = 1 << 30, flip_from = 1 << 30;
  float mean[3] = {0.485f, 0.456f, 0.406f};
  float inv_std[3] = {1.f / 0.229f, 1.f / 0.224f, 1.f / 0.225f};
};

// The patch loader's arguments for `batch` frames of an in_h x in_w image, NEAREST-resized to resized_h x resized_w and
// center-cropped to image_size (torchvision CenterCrop: offset int(round((resized - image_size) / 2)), half to even),
// cut into image_size / patch patches per side (conv-floor semantics), with the TTA fields above.  The ViT forward and
// the testing entry wvn_image_to_patches both derive their arguments here.
int image_patch_args(int batch, int in_h, int in_w, int resized_h, int resized_w, int image_size, int patch, int frame0,
                     int src_frames, int flip_from, ImagePatchArgs* a);

struct LayerNormArgs {
  long long rows = 0;
  int dim = 0;
  float eps = 1e-6f;
  // only used when an fp32 output is requested: keeps rows [row0, n_valid) of each npad-row frame (drops CLS, register
  // and padding rows); row0 = 1 + register tokens
  int npad = 0, n_valid = 0, row0 = 1;
  int reverse = 0;  // walk the rows last-to-first (start where the producer kernel finished: those rows are still in L2)
};

// Row pitch (elements) of a patch row of 3 * p * p K-elements in (c, ky, kx) order: rounded up to the 16 bytes TMA
// needs (p = 14: 588 -> 592; p = 8 / 16: 192 / 768, unpadded).  The patch-embed weight is stored at the same pitch.
__host__ __device__ inline int patch_pitch(int p) { return (3 * p * p + 7) / 8 * 8; }

// img: [batch, 3, in_h, in_w] fp32 in [0,1], or (u8_hwc) [batch, in_h, in_w, 3] uint8 RGB
// out_bf16: [batch * grid_h * grid_w, patch_pitch(patch)] bf16; patch in {8, 14, 16}
int image_to_patches(const void* img, bool u8_hwc, void* out_bf16, const ImagePatchArgs& a, cudaStream_t stream);
// Per frame: row 0 = cls + pos[0], rows [1, 1 + registers) = reg (no position embedding), rows [n_valid, npad) = 0;
// the patch rows [1 + registers, n_valid) are left to the patch-embed GEMM.
int init_token_rows(float* x, const float* cls, const float* pos, const float* reg, int registers, int batch, int npad,
                    int n_valid, int dim, cudaStream_t stream);
int layernorm_rows(const float* x, const float* gamma, const float* beta, void* out_bf16, float* out_f32,
                   const LayerNormArgs& a, cudaStream_t stream);

// Parity-debug attention in fp32 ($WVN_VIT_PRECISE=1): qkv [batch*npad, 3*dim] fp32 -> out [batch*npad, dim] bf16.
int attention_f32_debug(const float* qkv, void* out_bf16, int batch, int heads, int npad, int n_valid, int dim, float scale,
                        cudaStream_t stream);

}  // namespace wvn
