// wvn-b200: internal interface of the wgmma GEMM family (see gemm_wgmma.cu).
#pragma once

#include <cuda_runtime.h>

namespace wvn {

enum GemmEpilogue : int {
  EPI_BF16 = 0,       // out(bf16)[row, col]  = act(acc + bias)
  EPI_F32 = 1,        // out(f32)[row, col]   = acc + bias
  EPI_RESID_F32 = 2,  // out(f32)[row, col] += acc + bias            (residual stream, in place)
  EPI_PATCH = 3,      // out(f32)[frame*npad + 1 + registers + tok, col] = acc + bias + pos[1 + tok, col]
  EPI_QKV = 4,        // scatter to Q/K [b,h,npad,64] and V^T [b,h,64,npad] (bf16)
  EPI_MLP_HEAD = 5,   // last layer of the traversability MLP fused with its consumers:
                      //   cols [0,feat) reconstruct x -> loss_reco = mean((out - x)^2) -> confidence,
                      //   col feat = traversability logit -> sigmoid.  Nothing of [M,N] is stored.
  EPI_BF16_RESID = 6, // out(bf16)[row, col]  = act(acc + bias + residual(bf16)[row, col])  (a residual block's last conv)
  EPI_SWIGLU = 7,     // block_n 256 only, W and bias in swiglu_packed_row order: tile t's columns [0, 128) are gate
                      //   columns, [128, 256) the matching value columns;
                      //   out(bf16)[row, 128 t + j] = silu(acc_g + b_g) * (acc_v + b_v), N / 2 columns
};

// The SwiGLU FFN's w12 = [gate rows (H); value rows (H)] as EPI_SWIGLU reads it: packed row p of the 2H rows holds
// checkpoint row swiglu_packed_row(p, 2H), so that each 256-row tile is 128 gate rows followed by their 128 value rows.
// Needs H % 128 == 0.
inline long long swiglu_packed_row(long long p, long long rows) {
  const long long t = p / 256, j = p % 256;
  return j < 128 ? t * 128 + j : rows / 2 + t * 128 + (j - 128);
}

enum GemmAct : int { ACT_NONE = 0, ACT_RELU = 1, ACT_GELU = 2, ACT_SILU = 3 /* EPI_BF16 only */ };

struct GemmArgs {
  int M = 0, N = 0, K = 0;
  int epi = EPI_BF16, act = ACT_NONE;
  const float* bias = nullptr;  // [N] fp32 or null
  void* out = nullptr;          // primary output (see GemmEpilogue)
  long long ldo = 0;            // leading dimension of `out` (elements)
  // EPI_PATCH
  const float* pos = nullptr;   // [1 + tokens_in, ldo] positional embedding (row 0 = CLS)
  int tokens_in = 0;            // patches per frame (rows of A per frame)
  int registers = 0;            // register tokens between CLS and the first patch row (no position embedding)
  // EPI_PATCH / EPI_QKV
  int npad = 0;                 // padded tokens per frame in the activation layout
  // EPI_QKV
  int dim = 0, heads = 0;
  void* q = nullptr;
  void* k = nullptr;
  void* vt = nullptr;
  // EPI_MLP_HEAD
  int feat = 0;                 // feature dimension D: output columns [0, feat) reconstruct x
  int trav_col = 0;             // output column holding the traversability logit (multiple of 32, >= feat)
  const void* x = nullptr;      // [M, ldx] bf16 MLP input rows (reconstruction target)
  long long ldx = 0;
  float* trav = nullptr;        // [M]
  float* conf = nullptr;        // [M]
  float* loss_reco = nullptr;   // [M] optional
  const float* cg_mean = nullptr;  // device scalars of the ConfidenceGenerator
  const float* cg_std = nullptr;
  float cg_std_factor = 0.5f;
  // EPI_BF16_RESID
  const void* residual = nullptr;  // [M, ldr] bf16
  long long ldr = 0;
  // launch control
  int max_ctas = 0;             // 0 = one CTA per SM
  int reverse_m = 0;            // walk the m-blocks last-to-first (start on the rows the producer kernel wrote last: L2 hits)
};

int pick_block_n(int N);

// Row pitch (elements) of the W operand: K rounded up to 8, the 16-byte multiple TMA needs (K itself when K % 64 == 0).
inline long long gemm_w_pitch(int K) { return (static_cast<long long>(K) + 7) / 8 * 8; }

// Any K >= 1.  A: [M, K] bf16 with row pitch lda >= K (elements, a multiple of 8); W: [N, K] bf16 at row pitch
// gemm_w_pitch(K).  Columns past K of either operand are never read.
int gemm_bf16(const GemmArgs& args, const void* A, long long lda, const void* W, int block_n, cudaStream_t stream);

}  // namespace wvn
