// wvn-b200: STEGO's dense CRF (permutohedral-lattice mean field), the wvn_crf_* handle — internal interface of
// dense_crf.cu.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>

#include "../../include/wvn_b200.h"

namespace wvn {

struct CrfInput {
  const void* img = nullptr;       // [batch, 3, in_h, in_w] fp32 in [0, 1], or (u8_hwc) [batch, in_h, in_w, 3] uint8 RGB
  int u8_hwc = 0;
  int batch = 0, in_h = 0, in_w = 0, resized_h = 0, resized_w = 0;
  const float* head = nullptr;     // STEGO head output [batch * npad, ld]; patch p of frame b at row b * npad + 1 + p
  long long ld = 0;
  int npad = 0, grid = 0;
  int col0 = 0, classes = 0;       // logit columns
  int code_col = 0, code_dim = 0;  // code_dim > 0: cluster probe (logits / |upsampled code| * logit_scale)
  float logit_scale = 1.f;
};

// size: side S of the transformed image; max_classes <= 64; chunk: frames whose lattices are built and refined together.
int crf_create(int size, int max_classes, int chunk, int iterations, wvn_crf** out);
void crf_destroy(wvn_crf* h);
size_t crf_workspace_bytes(const wvn_crf* h);
// labels [batch, S, S] int64 (argmax of Q); q_out (optional) [batch, S*S, classes] fp32.
int crf_run(wvn_crf* h, const CrfInput& in, long long* labels, float* q_out, cudaStream_t s);
// Testing: build both lattices of frames [0, batch <= chunk) of `in` (only the image fields are read); filter `values`
// [batch*S*S, v] through lattice `which` (0: spatial, 1: bilateral) without normalisation; export a lattice.
int crf_build(wvn_crf* h, const CrfInput& in, cudaStream_t s);
int crf_filter(wvn_crf* h, int which, const float* values, int v, float* out, cudaStream_t s);
int crf_export(wvn_crf* h, int which, unsigned long long* keys, int* counts, int* offsets, float* bary, int* m,
               cudaStream_t s);

}  // namespace wvn
