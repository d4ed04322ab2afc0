// wvn-b200: internal interface of the fused wgmma attention kernel (attention_wgmma.cu).
#pragma once

#include <cuda_runtime.h>

namespace wvn {

struct AttnArgs {
  int batch = 0, heads = 0;
  int npad = 0;        // padded tokens per frame (multiple of 128)
  int n_valid = 0;     // real tokens per frame (CLS + patches); keys >= n_valid are masked
  float scale_log2 = 0.f;  // head_dim^-0.5 * log2(e)
  void* out = nullptr;     // [batch, npad, ldo] bf16, head h occupies columns [64h, 64h+64)
  long long ldo = 0;
  int reverse = 0;     // walk (frame, head, q-tile) last-to-first: start on what the QKV GEMM wrote last (L2 hits)
};

// q, k: [batch*heads, npad, 64] bf16; vt: [batch*heads, 64, npad] bf16.
int attention_bf16(const AttnArgs& args, const void* q, const void* k, const void* vt, cudaStream_t stream);

}  // namespace wvn
