// wvn-b200: the traversability MLP inference handle (wvn_mlp_infer_*) — internal interface of mlp_infer.cu.
#pragma once

#include <cuda_runtime.h>

#include "../../include/wvn_b200.h"

namespace wvn {

// double_layout: a DoubleMLP of two nets of widths h1 / h2 (its shape checked by the caller), else a SimpleMLP.
int mlp_infer_create(int dim, int h1, int h2, int chunk_rows, int double_layout, wvn_mlp_infer** out);
void mlp_infer_destroy(wvn_mlp_infer* h);
int mlp_infer_reserve(wvn_mlp_infer* h, int tokens_per_frame);
int mlp_infer_set_params(wvn_mlp_infer* h, const float* params, cudaStream_t s);
// Per-pixel maps from the tokens the ViT's last forward left in `vit` (fused head only).
int mlp_infer_pixels_vit(wvn_mlp_infer* h, const wvn_vit* vit, int batch, int out_h, int out_w, const float* cg_mean,
                         const float* cg_std, float std_factor, float* trav, float* conf, cudaStream_t s);
int mlp_infer_pixels(wvn_mlp_infer* h, const float* tokens, int batch, int gh, int gw, int out_h, int out_w,
                     const float* cg_mean, const float* cg_std, float std_factor, float* trav, float* conf,
                     cudaStream_t s);
int mlp_infer_rows(wvn_mlp_infer* h, const float* x, long long rows, const float* cg_mean, const float* cg_std,
                   float std_factor, float* trav, float* conf, cudaStream_t s);
int mlp_infer_rows_padded(wvn_mlp_infer* h, const float* x, int groups, int rows_per_group, const int* n_rows,
                          const float* cg_mean, const float* cg_std, float std_factor, float* trav, float* conf,
                          cudaStream_t s);

}  // namespace wvn
