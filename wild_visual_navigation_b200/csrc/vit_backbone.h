// wvn-b200: the ViT backbone handle (wvn_vit_*) — internal interface of vit_backbone.cu.
#pragma once

#include <cuda_runtime.h>

#include "../../include/wvn_b200.h"

namespace wvn {

// ffn: WVN_VIT_FFN_MLP or WVN_VIT_FFN_SWIGLU
int vit_create(const wvn_vit_config* cfg, int ffn, wvn_vit** out);
void vit_destroy(wvn_vit* h);
int vit_set_weight(wvn_vit* h, const char* name, const float* data, long long numel);
// img: [batch, 3, in_h, in_w] fp32, or (u8_hwc) [batch, in_h, in_w, 3] uint8.  flip_tta: the `batch` source frames are
// run twice, frames [batch, 2 batch) on the horizontally flipped transformed images.  tokens_out may be null.
int vit_forward_impl(wvn_vit* h, const void* img, bool u8_hwc, int batch, int in_h, int in_w, int resized_h,
                     int resized_w, float* tokens_out, bool flip_tta, cudaStream_t s);
int vit_stego_head(wvn_vit* h, int batch, float* out, cudaStream_t s);

// The bf16 tokens the last forward left in the handle: `batch` frames of `npad` rows of `dim` elements, the grid x grid
// patch tokens of a frame starting at row t0.  batch is 0 before the first forward.
struct VitTokens {
  const void* tok_bf16 = nullptr;
  int batch = 0, npad = 0, t0 = 0, grid = 0, dim = 0;
};
VitTokens vit_tokens(const wvn_vit* h);

}  // namespace wvn
