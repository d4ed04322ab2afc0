// wvn-b200: the traversability MLP inference handle — SimpleMLP / DoubleMLP rows through the bf16 GEMM chain, and
// per-pixel maps through the fused head (pixel_head.cu) or interpolated pixel rows.
#include "mlp_infer.h"

#include <cuda_bf16.h>

#include <stdlib.h>

#include <algorithm>
#include <string>

#include "dense_kernels.h"
#include "double_mlp_train.h"
#include "gemm.h"
#include "host_common.h"
#include "mlp_train.h"
#include "pixel_head.h"
#include "vit_backbone.h"

using namespace wvn;

struct wvn_mlp_infer {
  int dim, h1, h2;
  int dim_p, h1_p, h2_p, n3, n3_p, bn3, trav_col;
  int chunk_rows;
  DevBuf w1, b1, w2, b2, w3, b3;  // bf16 weights (padded / permuted), fp32 biases
  DevBuf x, a1, a2;               // bf16 activations of one chunk
  // fused per-pixel head (pixel_head.cu): per-token GEMM operands + workspaces for kFusedFrames frames
  DevBuf wcat, bias_cat, head_consts, tok_bf16, gu, gram;
  int fused_tokens = 0;           // token rows the fused workspaces are sized for (grown on demand)
  int head_n = 0;                 // columns of the per-token GEMM (G | U | cT); 0: no fused head for this handle
  int force_unfused = 0;          // debugging / A-B knob ($WVN_PIXEL_HEAD=unfused)
  // DoubleMLP layout (wvn_mlp_infer_create_double): the two nets packed as one block-structured SimpleMLP with
  // h1 = 2 net_h1, h2 = 2 net_h2; the unfused GEMM chain and its EPI_MLP_HEAD epilogue run it unchanged, and for
  // net_h1 in {64, 128}, net_h2 = 32 the fused head's DoubleMLP instantiation (pixel_head_double) takes the fused
  // geometries
  int double_layout = 0, net_h1 = 0, net_h2 = 0;
  bool loaded = false;
};

static constexpr int kFusedFrames = 8;

namespace {

// Pack the flat fp32 state-dict parameters into the padded bf16 operands of the three GEMMs.
// Layer 3 rows are permuted: reconstruction rows first (so output column j reconstructs x[j]),
// the traversability row at column trav_col.
__global__ void pack_mlp_kernel(const float* __restrict__ p, MlpOffsets o, int dim, int h1, int h2, int dim_p, int h1_p,
                                int h2_p, int n3_p, int trav_col, __nv_bfloat16* w1, float* b1, __nv_bfloat16* w2,
                                float* b2, __nv_bfloat16* w3, float* b3) {
  const long long n1 = static_cast<long long>(h1_p) * dim_p, n2 = static_cast<long long>(h2_p) * h1_p,
                  n3 = static_cast<long long>(n3_p) * h2_p;
  const long long total = n1 + n2 + n3 + h1_p + h2_p + n3_p;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    long long j = i;
    if (j < n1) {
      const int r = static_cast<int>(j / dim_p), c = static_cast<int>(j % dim_p);
      w1[j] = __float2bfloat16_rn((r < h1 && c < dim) ? p[o.w1 + static_cast<long long>(r) * dim + c] : 0.f);
      continue;
    }
    j -= n1;
    if (j < n2) {
      const int r = static_cast<int>(j / h1_p), c = static_cast<int>(j % h1_p);
      w2[j] = __float2bfloat16_rn((r < h2 && c < h1) ? p[o.w2 + static_cast<long long>(r) * h1 + c] : 0.f);
      continue;
    }
    j -= n2;
    if (j < n3) {
      const int r = static_cast<int>(j / h2_p), c = static_cast<int>(j % h2_p);
      int src = -1;
      if (r < dim) src = 1 + r; else if (r == trav_col) src = 0;
      w3[j] = __float2bfloat16_rn((src >= 0 && c < h2) ? p[o.w3 + static_cast<long long>(src) * h2 + c] : 0.f);
      continue;
    }
    j -= n3;
    if (j < h1_p) { b1[j] = j < h1 ? p[o.b1 + j] : 0.f; continue; }
    j -= h1_p;
    if (j < h2_p) { b2[j] = j < h2 ? p[o.b2 + j] : 0.f; continue; }
    j -= h2_p;
    {
      int src = -1;
      if (j < dim) src = 1 + static_cast<int>(j); else if (j == trav_col) src = 0;
      b3[j] = src >= 0 ? p[o.b3 + src] : 0.f;
    }
  }
}

// The DoubleMLP's flat parameters as the block-structured SimpleMLP the GEMM chain runs (h1 = 2 h, h2 = 2 k for nets of
// widths h / k): W1 = [W1_0; W1_1], W2 = diag(W2_0, W2_1), layer 3's reconstruction rows [0 | W3_1] first and its
// traversability row [w3_0 | 0] at trav_col; the biases stacked the same way.  Padding is zero.
__global__ void pack_double_mlp_kernel(const float* __restrict__ p, DoubleOffsets o, int dim, int h, int k, int dim_p,
                                       int h1_p, int h2_p, int n3_p, int trav_col, __nv_bfloat16* w1, float* b1,
                                       __nv_bfloat16* w2, float* b2, __nv_bfloat16* w3, float* b3) {
  const long long n1 = static_cast<long long>(h1_p) * dim_p, n2 = static_cast<long long>(h2_p) * h1_p,
                  n3 = static_cast<long long>(n3_p) * h2_p;
  const long long total = n1 + n2 + n3 + h1_p + h2_p + n3_p;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    long long j = i;
    float v = 0.f;
    if (j < n1) {
      const int r = static_cast<int>(j / dim_p), c = static_cast<int>(j % dim_p), net = r < h ? 0 : 1;
      if (r < 2 * h && c < dim) v = p[o.w1[net] + static_cast<long long>(r - net * h) * dim + c];
      w1[j] = __float2bfloat16_rn(v);
      continue;
    }
    j -= n1;
    if (j < n2) {
      const int r = static_cast<int>(j / h1_p), c = static_cast<int>(j % h1_p), net = r < k ? 0 : 1;
      if (r < 2 * k && c >= net * h && c < (net + 1) * h) v = p[o.w2[net] + static_cast<long long>(r - net * k) * h + c - net * h];
      w2[j] = __float2bfloat16_rn(v);
      continue;
    }
    j -= n2;
    if (j < n3) {
      const int r = static_cast<int>(j / h2_p), c = static_cast<int>(j % h2_p);
      if (r < dim && c >= k && c < 2 * k) v = p[o.w3[1] + static_cast<long long>(r) * k + c - k];
      else if (r == trav_col && c < k) v = p[o.w3[0] + c];
      w3[j] = __float2bfloat16_rn(v);
      continue;
    }
    j -= n3;
    if (j < h1_p) { b1[j] = j < 2 * h ? p[(j < h ? o.b1[0] : o.b1[1] - h) + j] : 0.f; continue; }
    j -= h1_p;
    if (j < h2_p) { b2[j] = j < 2 * k ? p[(j < k ? o.b2[0] : o.b2[1] - k) + j] : 0.f; continue; }
    j -= h2_p;
    b3[j] = j < dim ? p[o.b3[1] + j] : (j == trav_col ? p[o.b3[0]] : 0.f);
  }
}

int mlp_infer_chunk(wvn_mlp_infer* h, long long rows, long long row0, const float* cg_mean, const float* cg_std,
                    float std_factor, float* trav, float* conf, cudaStream_t s) {
  GemmArgs g1;
  g1.M = static_cast<int>(rows); g1.N = h->h1_p; g1.K = h->dim_p; g1.epi = EPI_BF16; g1.act = ACT_RELU;
  g1.bias = reinterpret_cast<float*>(h->b1.p); g1.out = h->a1.p; g1.ldo = h->h1_p;
  WVN_PROPAGATE(gemm_bf16(g1, h->x.p, h->dim_p, h->w1.p, 0, s));
  GemmArgs g2;
  g2.M = static_cast<int>(rows); g2.N = h->h2_p; g2.K = h->h1_p; g2.epi = EPI_BF16; g2.act = ACT_RELU;
  g2.bias = reinterpret_cast<float*>(h->b2.p); g2.out = h->a2.p; g2.ldo = h->h2_p;
  WVN_PROPAGATE(gemm_bf16(g2, h->a1.p, h->h1_p, h->w2.p, 0, s));
  GemmArgs g3;
  g3.M = static_cast<int>(rows); g3.N = h->n3_p; g3.K = h->h2_p; g3.epi = EPI_MLP_HEAD;
  g3.bias = reinterpret_cast<float*>(h->b3.p); g3.feat = h->dim; g3.trav_col = h->trav_col; g3.x = h->x.p;
  g3.ldx = h->dim_p; g3.trav = trav + row0; g3.conf = conf + row0; g3.cg_mean = cg_mean; g3.cg_std = cg_std;
  g3.cg_std_factor = std_factor;
  WVN_PROPAGATE(gemm_bf16(g3, h->a2.p, h->h2_p, h->w3.p, h->bn3, s));
  return WVN_OK;
}

// Rows [r0, r0 + rows) of groups padded to rpg rows each -> bf16 at pitch ld.  A padding row (r >= n_rows[g]) is not
// read: it is written as zeros, so the GEMM chain sees finite values there.
__global__ void cast_rows_padded_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long r0,
                                        long long rows, int rpg, const int* __restrict__ n_rows, int dim, long long ld) {
  const long long n = rows * dim;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / dim, pr = r0 + r, g = pr / rpg;
    const int c = static_cast<int>(i - r * dim);
    const bool live = pr - g * rpg < n_rows[g];
    dst[r * ld + c] = __float2bfloat16_rn(live ? src[pr * dim + c] : 0.f);
  }
}

// trav / conf of every padding row -> NaN (conf may be null)
__global__ void nan_padding_rows_kernel(float* __restrict__ trav, float* __restrict__ conf, long long rows, int rpg,
                                        const int* __restrict__ n_rows) {
  for (long long r = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; r < rows;
       r += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long g = r / rpg;
    if (r - g * rpg >= n_rows[g]) {
      trav[r] = __int_as_float(0x7fc00000);
      if (conf) conf[r] = __int_as_float(0x7fc00000);
    }
  }
}

}  // namespace

namespace wvn {

int mlp_infer_create(int dim, int h1, int h2, int chunk_rows, int double_layout, wvn_mlp_infer** out) {
  WVN_REQUIRE(out && dim > 0 && h1 > 0 && h2 > 0, "wvn_mlp_infer_create: bad arguments");
  WVN_PROPAGATE(wvn_check_device());
  wvn_mlp_infer* h = new wvn_mlp_infer();
  h->double_layout = double_layout;
  if (double_layout) {
    h->net_h1 = h1; h->net_h2 = h2;
    h1 *= 2; h2 *= 2;
  }
  h->dim = dim; h->h1 = h1; h->h2 = h2;
  h->dim_p = round_up(dim, 64); h->h1_p = round_up(h1, 64); h->h2_p = round_up(h2, 64);
  h->trav_col = round_up(dim, 32);
  h->n3 = h->trav_col + 1;
  // pick the layer-3 tile width with the least padding (ties -> wider tile)
  int best_bn = 64, best_n = round_up(h->n3, 64);
  for (int bn : {128, 192, 224, 256}) {
    const int n = round_up(h->n3, bn);
    if (n <= best_n) { best_n = n; best_bn = bn; }
  }
  h->bn3 = best_bn; h->n3_p = best_n;
  h->chunk_rows = chunk_rows > 0 ? round_up(chunk_rows, 128) : sm_count() * 128 * 3;  // three waves of 128-row tiles
  int rc = WVN_OK;
  auto alloc = [&](DevBuf& b, size_t bytes) { if (rc == WVN_OK) rc = b.alloc(bytes); };
  alloc(h->w1, static_cast<size_t>(h->h1_p) * h->dim_p * 2);
  alloc(h->b1, static_cast<size_t>(h->h1_p) * 4);
  alloc(h->w2, static_cast<size_t>(h->h2_p) * h->h1_p * 2);
  alloc(h->b2, static_cast<size_t>(h->h2_p) * 4);
  alloc(h->w3, static_cast<size_t>(h->n3_p) * h->h2_p * 2);
  alloc(h->b3, static_cast<size_t>(h->n3_p) * 4);
  alloc(h->x, static_cast<size_t>(h->chunk_rows) * h->dim_p * 2);
  alloc(h->a1, static_cast<size_t>(h->chunk_rows) * h->h1_p * 2);
  alloc(h->a2, static_cast<size_t>(h->chunk_rows) * h->h2_p * 2);
  if (!double_layout)
    h->head_n = kPixelHeadN;
  else if (pixel_head_double_shape(h->net_h1, h->net_h2))
    h->head_n = pixel_head_columns(2 * h->net_h1);
  if (h->head_n > 0) {
    alloc(h->wcat, static_cast<size_t>(h->head_n) * h->dim_p * 2);
    alloc(h->bias_cat, static_cast<size_t>(h->head_n) * 4);
    alloc(h->head_consts, sizeof(PixelHeadConsts));
  }
  {
    const char* e = getenv("WVN_PIXEL_HEAD");
    h->force_unfused = (e && std::string(e) == "unfused") ? 1 : 0;
  }
  if (rc != WVN_OK) {
    delete h;
    return rc;
  }
  *out = h;
  return WVN_OK;
}

void mlp_infer_destroy(wvn_mlp_infer* h) { delete h; }

int mlp_infer_reserve(wvn_mlp_infer* h, int tokens_per_frame) {
  const int P = tokens_per_frame;
  if (h->head_n == 0 || h->fused_tokens >= kFusedFrames * P) return WVN_OK;   // no fused head: nothing to size
  WVN_PROPAGATE(h->tok_bf16.alloc(static_cast<size_t>(kFusedFrames) * P * h->dim_p * 2));
  WVN_PROPAGATE(h->gu.alloc(static_cast<size_t>(kFusedFrames) * P * h->head_n * 4));
  WVN_PROPAGATE(h->gram.alloc(static_cast<size_t>(kFusedFrames) * P * 5 * 4));
  h->fused_tokens = kFusedFrames * P;
  return WVN_OK;
}

int mlp_infer_set_params(wvn_mlp_infer* h, const float* params, cudaStream_t s) {
  MlpShape sh;
  sh.dim = h->dim; sh.h1 = h->h1; sh.h2 = h->h2;
  if (h->double_layout) {
    MlpShape net;
    net.dim = h->dim; net.h1 = h->net_h1; net.h2 = h->net_h2;
    pack_double_mlp_kernel<<<256, 256, 0, s>>>(
        params, double_mlp_offsets(net), h->dim, net.h1, net.h2, h->dim_p, h->h1_p, h->h2_p, h->n3_p, h->trav_col,
        reinterpret_cast<__nv_bfloat16*>(h->w1.p), reinterpret_cast<float*>(h->b1.p),
        reinterpret_cast<__nv_bfloat16*>(h->w2.p), reinterpret_cast<float*>(h->b2.p),
        reinterpret_cast<__nv_bfloat16*>(h->w3.p), reinterpret_cast<float*>(h->b3.p));
    WVN_CHECK_LAUNCH("pack_double_mlp_kernel");
    if (h->head_n > 0)
      WVN_PROPAGATE(pixel_head_pack_double(params, net, h->dim_p, h->wcat.p, reinterpret_cast<float*>(h->bias_cat.p),
                                           reinterpret_cast<PixelHeadConsts*>(h->head_consts.p), s));
    h->loaded = true;
    return WVN_OK;
  }
  pack_mlp_kernel<<<256, 256, 0, s>>>(
      params, mlp_offsets(sh), h->dim, h->h1, h->h2, h->dim_p, h->h1_p, h->h2_p, h->n3_p, h->trav_col,
      reinterpret_cast<__nv_bfloat16*>(h->w1.p), reinterpret_cast<float*>(h->b1.p),
      reinterpret_cast<__nv_bfloat16*>(h->w2.p), reinterpret_cast<float*>(h->b2.p),
      reinterpret_cast<__nv_bfloat16*>(h->w3.p), reinterpret_cast<float*>(h->b3.p));
  WVN_CHECK_LAUNCH("pack_mlp_kernel");
  if (h->h1 == 256 && h->h2 == 32)
    WVN_PROPAGATE(pixel_head_pack(params, sh, h->dim_p, h->wcat.p, reinterpret_cast<float*>(h->bias_cat.p),
                                  reinterpret_cast<PixelHeadConsts*>(h->head_consts.p), s));
  h->loaded = true;
  return WVN_OK;
}

// Token-window width of the fused head for this handle and geometry, 0 when the fused head does not take it.
static int fused_window(const wvn_mlp_infer* h, int gh, int gw, int out_h, int out_w) {
  if (h->double_layout) return h->head_n > 0 ? pixel_head_supported_double(h->net_h1, h->net_h2, gh, gw, out_h, out_w) : 0;
  return pixel_head_supported(h->h1, h->h2, gh, gw, out_h, out_w);
}

// Fused per-pixel head over frames [b0, b0 + nb): per-token GEMM (G | U | cT) + token Gram + one pixel kernel.
// tok_bf16: the frames' bf16 tokens, frame_rows rows per frame with the patch tokens starting at row row0.
static int pixels_fused_chunk(wvn_mlp_infer* h, const void* tok_bf16, long long frame_rows, int row0, int b0, int nb,
                              int gh, int gw, int out_h, int out_w, int ww, const float* cg_mean, const float* cg_std,
                              float std_factor, float* trav, float* conf, cudaStream_t s) {
  const long long rows = static_cast<long long>(nb) * frame_rows;
  GemmArgs g;
  g.M = static_cast<int>(rows); g.N = h->head_n; g.K = h->dim_p; g.epi = EPI_F32;
  g.bias = reinterpret_cast<float*>(h->bias_cat.p); g.out = h->gu.p; g.ldo = h->head_n;
  WVN_PROPAGATE(gemm_bf16(g, tok_bf16, h->dim_p, h->wcat.p, 64, s));
  WVN_PROPAGATE(token_gram(tok_bf16, reinterpret_cast<float*>(h->gram.p), nb, gh, gw, h->dim_p, frame_rows, row0, s));
  PixelHeadArgs a;
  a.gu = reinterpret_cast<float*>(h->gu.p); a.ldg = h->head_n; a.gram = reinterpret_cast<float*>(h->gram.p);
  a.consts = reinterpret_cast<PixelHeadConsts*>(h->head_consts.p);
  a.cg_mean = cg_mean; a.cg_std = cg_std; a.std_factor = std_factor;
  a.trav = trav + static_cast<long long>(b0) * out_h * out_w;
  a.conf = conf + static_cast<long long>(b0) * out_h * out_w;
  a.batch = nb; a.gh = gh; a.gw = gw; a.H = out_h; a.W = out_w;
  a.sy = static_cast<float>(gh - 1) / static_cast<float>(out_h - 1);
  a.sx = static_cast<float>(gw - 1) / static_cast<float>(out_w - 1);
  a.ww = ww; a.feat = h->dim;
  a.frame_rows = frame_rows; a.row0 = row0;
  if (h->double_layout) WVN_PROPAGATE(pixel_head_double(a, h->net_h1, h->w2.p, h->h1_p, s));
  else WVN_PROPAGATE(pixel_head(a, h->w2.p, h->h1_p, s));
  return WVN_OK;
}

int mlp_infer_pixels_vit(wvn_mlp_infer* h, const wvn_vit* vit_h, int batch, int out_h, int out_w, const float* cg_mean,
                         const float* cg_std, float std_factor, float* trav, float* conf, cudaStream_t s) {
  if (!h->loaded) return set_error(WVN_ERR_STATE, "wvn_mlp_infer_pixels_vit: parameters were never set");
  const VitTokens vit = vit_tokens(vit_h);
  if (vit.batch == 0 || batch > vit.batch)
    return set_error(WVN_ERR_STATE, "wvn_mlp_infer_pixels_vit: the backbone holds the tokens of %d frames, %d asked",
                     vit.batch, batch);
  WVN_REQUIRE(h->dim == vit.dim && h->dim_p == vit.dim, "wvn_mlp_infer_pixels_vit: the MLP takes %d-d features, "
              "the backbone's tokens are %d-d", h->dim, vit.dim);
  const int g = vit.grid;
  const int ww = fused_window(h, g, g, out_h, out_w);
  WVN_REQUIRE(ww > 0, "wvn_mlp_infer_pixels_vit: geometry outside the fused per-pixel head (use wvn_mlp_infer_pixels)");
  if (h->fused_tokens < kFusedFrames * vit.npad) WVN_PROPAGATE(mlp_infer_reserve(h, vit.npad));
  for (int b0 = 0; b0 < batch; b0 += kFusedFrames) {
    const int nb = std::min(kFusedFrames, batch - b0);
    const __nv_bfloat16* tok = reinterpret_cast<const __nv_bfloat16*>(vit.tok_bf16) +
                               static_cast<long long>(b0) * vit.npad * vit.dim;
    WVN_PROPAGATE(pixels_fused_chunk(h, tok, vit.npad, vit.t0, b0, nb, g, g, out_h, out_w, ww, cg_mean, cg_std, std_factor, trav,
                                     conf, s));
  }
  return WVN_OK;
}

int mlp_infer_pixels(wvn_mlp_infer* h, const float* tokens, int batch, int gh, int gw, int out_h, int out_w,
                     const float* cg_mean, const float* cg_std, float std_factor, float* trav, float* conf,
                     cudaStream_t s) {
  if (!h->loaded) return set_error(WVN_ERR_STATE, "wvn_mlp_infer_pixels: parameters were never set");
  // any feature width works (the 90-d STEGO code is zero-padded to 128 columns in the bf16 operands)
  const int ww = h->force_unfused ? 0 : fused_window(h, gh, gw, out_h, out_w);
  if (ww > 0) {
    // ---- fused path: per-token GEMM (G | U | cT) + token Gram, then one kernel per chunk of frames
    const int P = gh * gw;
    // workspaces are sized by wvn_mlp_infer_reserve (called by the owner right after create); a larger token grid
    // than reserved grows them here once
    if (h->fused_tokens < kFusedFrames * P) WVN_PROPAGATE(mlp_infer_reserve(h, P));
    for (int b0 = 0; b0 < batch; b0 += kFusedFrames) {
      const int nb = std::min(kFusedFrames, batch - b0);
      const long long rows = static_cast<long long>(nb) * P;
      WVN_PROPAGATE(cast_rows_to_bf16(tokens + static_cast<long long>(b0) * P * h->dim, h->tok_bf16.p, rows, h->dim,
                                      h->dim_p, 8192, s));
      WVN_PROPAGATE(pixels_fused_chunk(h, h->tok_bf16.p, P, 0, b0, nb, gh, gw, out_h, out_w, ww, cg_mean, cg_std,
                                       std_factor, trav, conf, s));
    }
    return WVN_OK;
  }
  DenseArgs d;
  d.batch = batch; d.dim = h->dim; d.grid_h = gh; d.grid_w = gw; d.out_h = out_h; d.out_w = out_w;
  d.scale_y = out_h > 1 ? static_cast<float>(gh - 1) / static_cast<float>(out_h - 1) : 0.f;
  d.scale_x = out_w > 1 ? static_cast<float>(gw - 1) / static_cast<float>(out_w - 1) : 0.f;
  d.ld_out = h->dim_p;
  const long long total = static_cast<long long>(batch) * out_h * out_w;
  for (long long p0 = 0; p0 < total; p0 += h->chunk_rows) {
    const long long n = std::min<long long>(h->chunk_rows, total - p0);
    WVN_PROPAGATE(interp_pixel_rows(tokens, h->x.p, d, p0, n, s));
    WVN_PROPAGATE(mlp_infer_chunk(h, n, p0, cg_mean, cg_std, std_factor, trav, conf, s));
  }
  return WVN_OK;
}

int mlp_infer_rows(wvn_mlp_infer* h, const float* x, long long rows, const float* cg_mean, const float* cg_std,
                   float std_factor, float* trav, float* conf, cudaStream_t s) {
  if (!h->loaded) return set_error(WVN_ERR_STATE, "wvn_mlp_infer_rows: parameters were never set");
  for (long long r0 = 0; r0 < rows; r0 += h->chunk_rows) {
    const long long n = std::min<long long>(h->chunk_rows, rows - r0);
    WVN_PROPAGATE(cast_rows_to_bf16(x + r0 * h->dim, h->x.p, n, h->dim, h->dim_p, 8192, s));
    WVN_PROPAGATE(mlp_infer_chunk(h, n, r0, cg_mean, cg_std, std_factor, trav, conf, s));
  }
  return WVN_OK;
}

// The padded form runs the same chunks over all groups * rows_per_group rows: the GEMMs' tile shapes depend on N and K
// only (BM is fixed, block_n follows N), so each live row goes through exactly the arithmetic of wvn_mlp_infer_rows.
int mlp_infer_rows_padded(wvn_mlp_infer* h, const float* x, int groups, int rows_per_group, const int* n_rows,
                          const float* cg_mean, const float* cg_std, float std_factor, float* trav, float* conf,
                          cudaStream_t s) {
  WVN_REQUIRE(groups >= 0 && rows_per_group >= 0, "wvn_mlp_infer_rows_padded: bad geometry (groups=%d rows=%d)", groups,
              rows_per_group);
  if (!h->loaded) return set_error(WVN_ERR_STATE, "wvn_mlp_infer_rows_padded: parameters were never set");
  const long long rows = static_cast<long long>(groups) * rows_per_group;
  if (rows == 0) return WVN_OK;
  for (long long r0 = 0; r0 < rows; r0 += h->chunk_rows) {
    const long long n = std::min<long long>(h->chunk_rows, rows - r0);
    const long long elems = n * h->dim;
    int blocks = static_cast<int>(std::min<long long>((elems + 255) / 256, 8192));
    cast_rows_padded_kernel<<<blocks, 256, 0, s>>>(x, reinterpret_cast<__nv_bfloat16*>(h->x.p), r0, n, rows_per_group,
                                                   n_rows, h->dim, h->dim_p);
    WVN_CHECK_LAUNCH("cast_rows_padded_kernel");
    WVN_PROPAGATE(mlp_infer_chunk(h, n, r0, cg_mean, cg_std, std_factor, trav, conf, s));
  }
  const int blocks = static_cast<int>(std::min<long long>((rows + 255) / 256, 4096));
  nan_padding_rows_kernel<<<blocks, 256, 0, s>>>(trav, conf, rows, rows_per_group, n_rows);
  WVN_CHECK_LAUNCH("nan_padding_rows_kernel");
  return WVN_OK;
}

}  // namespace wvn
