// wvn-b200: internal interface of the fused per-pixel traversability head (pixel_head.cu).
#pragma once

#include <cuda_runtime.h>

#include "mlp_train.h"

namespace wvn {

constexpr int kPixelHeadN = 320;  // columns of the per-token GEMM: 256 G | 32 U | cT_hi | cT_lo | pad

// Weight-only constants (fp32), copied to shared memory by every CTA.
struct PixelHeadConsts {
  float b2[32];      // layers.2.bias
  float w0[32];      // row 0 of layers.4.weight (traversability logit)
  float tv[32];      // 2 * R^T c
  float m[32 * 32];  // R^T R, upper-triangular with doubled off-diagonals
  float b0;          // layers.4.bias[0]
  float cc;          // c . c
  float pad[2];
  float b2r[32];     // layer 2's bias of the reconstruction network (DoubleMLP: networks.1.2.bias; SimpleMLP: b2)
};

struct PixelHeadArgs {
  const float* gu = nullptr;     // [batch * gh*gw, ldg] fp32 per-token (G | U | cT) rows
  long long ldg = 0;
  const float* gram = nullptr;   // [batch * gh*gw, 5] fp32 token Gram entries
  const PixelHeadConsts* consts = nullptr;
  const float* cg_mean = nullptr;
  const float* cg_std = nullptr;
  float std_factor = 0.5f;
  float* trav = nullptr;         // [batch, H, W]
  float* conf = nullptr;
  float* loss_reco = nullptr;    // optional
  int batch = 0, gh = 0, gw = 0, H = 0, W = 0;
  float sy = 0.f, sx = 0.f;      // (gh-1)/(H-1), (gw-1)/(W-1)
  int ww = 0;                    // token-window columns per tile (from pixel_head_supported)
  int feat = 0;                  // D
  long long frame_rows = 0;      // rows of gu / gram between two frames (0 = gh*gw): the ViT's own token buffer keeps
  int row0 = 0;                  // npad rows per frame with the patch tokens starting at row 1
};

// Returns the token-window width if the fused kernel supports this geometry, else 0.
int pixel_head_supported(int h1, int h2, int gh, int gw, int H, int W);
int pixel_head_pack(const float* params, const MlpShape& s, int dim_p, void* wcat_bf16, float* bias,
                    PixelHeadConsts* consts, cudaStream_t stream);
int token_gram(const void* tok_bf16, float* gram, int batch, int gh, int gw, int dim, long long frame_rows, int row0,
               cudaStream_t stream);
int pixel_head(const PixelHeadArgs& a, const void* w2_bf16, int w2_ld, cudaStream_t stream);

// The DoubleMLP head (net widths h1 in {64, 128}, h2 = 32): per-token GEMM columns G_0 | G_1 | U | cT_hi | cT_lo, padded
// to pixel_head_columns(2 h1) (192 / 320); U / cT from networks.1.4, the logit from networks.0.4.  w2_bf16: the packed
// block-diagonal layer 2 [64 rows][w2_ld] (rows 0..31 net 0 on channels [0, h1), rows 32..63 net 1 on [h1, 2 h1)).
bool pixel_head_double_shape(int h1, int h2);
int pixel_head_supported_double(int h1, int h2, int gh, int gw, int H, int W);
int pixel_head_columns(int g_channels);
int pixel_head_pack_double(const float* params, const MlpShape& net, int dim_p, void* wcat_bf16, float* bias,
                           PixelHeadConsts* consts, cudaStream_t stream);
int pixel_head_double(const PixelHeadArgs& a, int h1, const void* w2_bf16, int w2_ld, cudaStream_t stream);

}  // namespace wvn
