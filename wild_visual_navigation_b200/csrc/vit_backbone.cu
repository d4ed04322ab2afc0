// wvn-b200: the ViT backbone handle — DINO / DINOv2 ViT-S / B / L / g token forward and STEGO's segmentation head.
#include "vit_backbone.h"

#include <cuda_bf16.h>

#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "attention.h"
#include "gemm.h"
#include "host_common.h"
#include "vit_kernels.h"

using namespace wvn;

namespace {

// One transformer block's parameters, resolved from the weight store at create (the storage never moves).  With the
// SwiGLU FFN, fc1 is w12 (its rows and bias in swiglu_packed_row order) and fc2 is w3.
struct VitBlock {
  const float *norm1_w, *norm1_b, *qkv_b, *proj_b, *norm2_w, *norm2_b, *fc1_b, *fc2_b;
  const void *qkv_w, *proj_w, *fc1_w, *fc2_w;
};

}  // namespace

struct wvn_vit {
  wvn_vit_config cfg;
  int ffn = WVN_VIT_FFN_MLP;
  // t0: first patch row of a frame (1 + register tokens); rows [t0, n_valid) are the P patches
  int grid = 0, P = 0, t0 = 1, n_valid = 0, npad = 0, kpe = 0, kpe_ld = 0, chunk = 0;
  WeightStore weights;
  std::vector<VitBlock> blocks;
  const float *cls = nullptr, *pos = nullptr, *reg = nullptr, *pe_b = nullptr, *norm_w = nullptr, *norm_b = nullptr;
  const void* pe_w = nullptr;
  const float *hidden_b = nullptr, *head_a_b = nullptr;  // STEGO head (head_out > 0)
  const void *hidden_w = nullptr, *head_a_w = nullptr, *head_b_w = nullptr;
  // workspaces (per chunk)
  DevBuf x, xn, q, k, vt, attn, hid, ape;
  // per max_batch
  DevBuf tok_bf16, head_hidden;
  DevBuf qkv_f32;        // only with $WVN_VIT_PRECISE=1 at create: fp32 QKV projections of one chunk (parity-debug attention)
  bool precise = false;
  int last_batch = 0;    // frames of the last forward, 0 before the first
};

namespace wvn {

int vit_create(const wvn_vit_config* cfg, int ffn, wvn_vit** out) {
  WVN_REQUIRE(cfg->dim == 384 || cfg->dim == 768 || cfg->dim == 1024 || cfg->dim == 1536,
              "vit: dim %d unsupported (384, 768, 1024, 1536)", cfg->dim);
  WVN_REQUIRE(ffn == WVN_VIT_FFN_MLP || ffn == WVN_VIT_FFN_SWIGLU, "vit: ffn %d unsupported (0 = GELU MLP, 1 = SwiGLU)",
              ffn);
  // SwiGLU: w12's 2 mlp_dim rows pack into 256-row tiles of 128 gate + 128 value rows (EPI_SWIGLU)
  WVN_REQUIRE(ffn != WVN_VIT_FFN_SWIGLU || cfg->mlp_dim % 128 == 0,
              "vit: the SwiGLU FFN needs mlp_dim %% 128 == 0 (got %d)", cfg->mlp_dim);
  WVN_REQUIRE(cfg->heads * 64 == cfg->dim, "vit: heads*64 must equal dim");
  WVN_REQUIRE(cfg->patch_size == 8 || cfg->patch_size == 14 || cfg->patch_size == 16, "vit: patch size %d unsupported",
              cfg->patch_size);
  WVN_REQUIRE(cfg->image_size >= cfg->patch_size, "vit: image size too small");
  WVN_REQUIRE(cfg->mlp_dim % 64 == 0 && cfg->depth > 0 && cfg->max_batch > 0, "vit: bad mlp_dim/depth/max_batch");
  WVN_REQUIRE(cfg->head_out % 64 == 0, "vit: head_out must be a multiple of 64");
  WVN_REQUIRE(cfg->registers >= 0, "vit: registers must be >= 0");
  // the STEGO head's consumers (wvn_flip_average, wvn_logits_argmax, wvn_stego_kmeans) read patch p at row 1 + p
  WVN_REQUIRE(cfg->registers == 0 || cfg->head_out == 0, "vit: register tokens and a STEGO head cannot be combined");
  wvn_vit* h = new wvn_vit();
  h->cfg = *cfg;
  h->ffn = ffn;
  if (h->cfg.ln_eps <= 0.f) h->cfg.ln_eps = 1e-6f;
  h->grid = cfg->image_size / cfg->patch_size;  // conv-floor semantics for non-divisible sizes
  h->P = h->grid * h->grid;
  h->t0 = 1 + cfg->registers;
  h->n_valid = h->t0 + h->P;
  h->npad = round_up(h->n_valid, 128);
  h->kpe = 3 * cfg->patch_size * cfg->patch_size;
  h->kpe_ld = patch_pitch(cfg->patch_size);  // == gemm_w_pitch(kpe): patch rows and weight rows share one pitch
  h->chunk = cfg->chunk > 0 ? cfg->chunk : 8;
  if (h->chunk > cfg->max_batch) h->chunk = cfg->max_batch;
  const int D = cfg->dim;
  int rc = WVN_OK;
  // adds a weight and returns its storage, which the forward reads through the pointers kept here
  auto add = [&](const std::string& n, long long rows, int cols, bool bf) -> float* {
    if (rc == WVN_OK) rc = h->weights.add(n, rows, cols, bf);
    return rc == WVN_OK ? h->weights.ptr<float>(n) : nullptr;
  };
  h->cls = add("cls_token", 1, D, false);
  h->pos = add("pos_embed", 1 + h->P, D, false);
  if (cfg->registers > 0) h->reg = add("register_tokens", cfg->registers, D, false);
  h->pe_w = add("patch_embed.proj.weight", D, h->kpe, true);
  h->pe_b = add("patch_embed.proj.bias", 1, D, false);
  for (int i = 0; i < cfg->depth; ++i) {
    const std::string b = "blocks." + std::to_string(i) + ".";
    VitBlock k;
    k.norm1_w = add(b + "norm1.weight", 1, D, false);
    k.norm1_b = add(b + "norm1.bias", 1, D, false);
    k.qkv_w = add(b + "attn.qkv.weight", 3 * D, D, true);
    k.qkv_b = add(b + "attn.qkv.bias", 1, 3 * D, false);
    k.proj_w = add(b + "attn.proj.weight", D, D, true);
    k.proj_b = add(b + "attn.proj.bias", 1, D, false);
    k.norm2_w = add(b + "norm2.weight", 1, D, false);
    k.norm2_b = add(b + "norm2.bias", 1, D, false);
    if (ffn == WVN_VIT_FFN_SWIGLU) {
      // the bias as 2 mlp_dim rows of one element, so that vit_set_weight packs it row by row as it packs the weight
      k.fc1_w = add(b + "mlp.w12.weight", 2LL * cfg->mlp_dim, D, true);
      k.fc1_b = add(b + "mlp.w12.bias", 2LL * cfg->mlp_dim, 1, false);
      k.fc2_w = add(b + "mlp.w3.weight", D, cfg->mlp_dim, true);
      k.fc2_b = add(b + "mlp.w3.bias", 1, D, false);
    } else {
      k.fc1_w = add(b + "mlp.fc1.weight", cfg->mlp_dim, D, true);
      k.fc1_b = add(b + "mlp.fc1.bias", 1, cfg->mlp_dim, false);
      k.fc2_w = add(b + "mlp.fc2.weight", D, cfg->mlp_dim, true);
      k.fc2_b = add(b + "mlp.fc2.bias", 1, D, false);
    }
    h->blocks.push_back(k);
  }
  h->norm_w = add("norm.weight", 1, D, false);
  h->norm_b = add("norm.bias", 1, D, false);
  if (cfg->head_out > 0) {
    h->head_a_w = add("stego.head_a.weight", cfg->head_out, D, true);
    h->head_a_b = add("stego.head_a.bias", 1, cfg->head_out, false);
    h->hidden_w = add("stego.hidden.weight", D, D, true);
    h->hidden_b = add("stego.hidden.bias", 1, D, false);
    h->head_b_w = add("stego.head_b.weight", cfg->head_out, D, true);
  }
  const size_t rows = static_cast<size_t>(h->chunk) * h->npad;
  const size_t bh = static_cast<size_t>(h->chunk) * cfg->heads;
  auto alloc = [&](DevBuf& b, size_t bytes) { if (rc == WVN_OK) rc = b.alloc(bytes); };
  alloc(h->x, rows * D * 4);
  alloc(h->xn, rows * D * 2);
  alloc(h->q, bh * h->npad * 64 * 2);
  alloc(h->k, bh * h->npad * 64 * 2);
  alloc(h->vt, bh * 64 * h->npad * 2);
  alloc(h->attn, rows * D * 2);
  alloc(h->hid, rows * cfg->mlp_dim * 2);
  alloc(h->ape, static_cast<size_t>(h->chunk) * h->P * h->kpe_ld * 2);
  alloc(h->tok_bf16, static_cast<size_t>(cfg->max_batch) * h->npad * D * 2);
  if (cfg->head_out > 0) alloc(h->head_hidden, static_cast<size_t>(cfg->max_batch) * h->npad * D * 2);
  {
    // parity-debug mode (SURVEY.md §7): Q K^T, softmax and P V in fp32 on fp32 projections, ~40x slower attention
    const char* e = getenv("WVN_VIT_PRECISE");
    h->precise = e && atoi(e) == 1;
    if (h->precise) alloc(h->qkv_f32, rows * 3 * D * 4);
  }
  if (rc != WVN_OK) {
    delete h;
    return rc;
  }
  *out = h;
  return WVN_OK;
}

void vit_destroy(wvn_vit* h) { delete h; }

namespace {
bool ends_with(const char* s, const char* suffix) {
  const size_t n = strlen(s), m = strlen(suffix);
  return n >= m && strcmp(s + n - m, suffix) == 0;
}
}  // namespace

int vit_set_weight(wvn_vit* h, const char* name, const float* data, long long numel) {
  // w12 arrives in the checkpoint's row order [gate; value] and is stored in EPI_SWIGLU's packed order
  if (h->ffn == WVN_VIT_FFN_SWIGLU && (ends_with(name, ".mlp.w12.weight") || ends_with(name, ".mlp.w12.bias")))
    return h->weights.set(name, data, numel, swiglu_packed_row);
  return h->weights.set(name, data, numel);
}

VitTokens vit_tokens(const wvn_vit* h) {
  return {h->tok_bf16.p, h->last_batch, h->npad, h->t0, h->grid, h->cfg.dim};
}

constexpr int kDefaultSubAttn = 1 << 30;  // frames per (LN1, QKV, attention) pass: one pass over the whole chunk

// flip_tta: `batch` source frames are run twice — frames [batch, 2*batch) of the activation layout / tokens_out are
// the backbone's output on the horizontally flipped TRANSFORMED images (Stego.get_code's second pass).
int vit_forward_impl(wvn_vit* h, const void* img, bool u8_hwc, int src_batch, int in_h, int in_w, int resized_h, int resized_w,
                     float* tokens_out, bool flip_tta, cudaStream_t s) {
  const int batch = flip_tta ? 2 * src_batch : src_batch;
  WVN_REQUIRE(h && img, "wvn_vit_forward: null argument");
  WVN_REQUIRE(batch > 0 && batch <= h->cfg.max_batch, "wvn_vit_forward: batch %d outside (0, %d]", batch, h->cfg.max_batch);
  WVN_REQUIRE(resized_h >= h->cfg.image_size && resized_w >= h->cfg.image_size,
              "wvn_vit_forward: resized image %dx%d smaller than the crop %d", resized_h, resized_w, h->cfg.image_size);
  WVN_PROPAGATE(h->weights.check_loaded("vit", "stego."));
  const wvn_vit_config& c = h->cfg;
  const int D = c.dim;

  for (int b0 = 0; b0 < batch; b0 += h->chunk) {
    const int nb = std::min(h->chunk, batch - b0);
    const int rows = nb * h->npad;
    float* x = reinterpret_cast<float*>(h->x.p);
    ImagePatchArgs ia;
    WVN_PROPAGATE(image_patch_args(nb, in_h, in_w, resized_h, resized_w, c.image_size, c.patch_size, b0, src_batch,
                                   flip_tta ? src_batch : (1 << 30), &ia));
    WVN_PROPAGATE(image_to_patches(img, u8_hwc, h->ape.p, ia, s));
    WVN_PROPAGATE(init_token_rows(x, h->cls, h->pos, h->reg, c.registers, nb, h->npad, h->n_valid, D, s));
    {
      GemmArgs g;
      g.M = nb * h->P; g.N = D; g.K = h->kpe; g.epi = EPI_PATCH; g.bias = h->pe_b;
      g.out = x; g.ldo = D; g.pos = h->pos; g.tokens_in = h->P; g.npad = h->npad;
      g.registers = c.registers;
      WVN_PROPAGATE(gemm_bf16(g, h->ape.p, h->kpe_ld, h->pe_w, 0, s));
    }
    LayerNormArgs la;
    la.rows = rows; la.dim = D; la.eps = c.ln_eps; la.npad = h->npad; la.n_valid = h->n_valid; la.row0 = h->t0;
    // GEMMs / LayerNorms can run over sub-chunks of `sub` frames ($WVN_VIT_SUBCHUNK) to keep xn / hid / x
    // L2-resident between producer and consumer.  Smaller GEMMs lose to wave quantisation what they gain in L2
    // hits, which the snake order below already collects for the rows written last — default off.
    static int sub_env = -1;
    if (sub_env < 0) {
      const char* e = getenv("WVN_VIT_SUBCHUNK");
      sub_env = e ? atoi(e) : (1 << 30);
      if (sub_env < 1) sub_env = 1 << 30;
    }
    const int sub = std::min(sub_env, nb);
    // "Snake" order: every kernel of the chain walks its rows in the opposite direction to its producer, so it
    // starts on the rows that were written last and are still in the 50 MB L2 ($WVN_VIT_SNAKE=0 disables).
    static int snake = -1;
    if (snake < 0) { const char* e = getenv("WVN_VIT_SNAKE"); snake = (e && atoi(e) == 0) ? 0 : 1; }
    int dir = 0;  // the patch-embed GEMM above ran first-to-last
    auto next_dir = [&]() { dir = snake ? dir ^ 1 : 0; return dir; };
    __nv_bfloat16* xn = reinterpret_cast<__nv_bfloat16*>(h->xn.p);
    __nv_bfloat16* attn = reinterpret_cast<__nv_bfloat16*>(h->attn.p);
    // The attention half of a block (LN1 -> QKV -> attention) can additionally run over `sub_a` frames at a time
    // ($WVN_VIT_SUB_ATTN): Q / K / V^T of a half-chunk (118 MB at 16 frames) are consumed while still in L2.
    static int sub_attn_env = -1;
    if (sub_attn_env < 0) {
      const char* e = getenv("WVN_VIT_SUB_ATTN");
      sub_attn_env = e ? atoi(e) : kDefaultSubAttn;
      if (sub_attn_env < 1) sub_attn_env = 1 << 30;
    }
    const int sub_a = std::min(sub_attn_env, nb);   // independent of `sub`: attention wants the whole chunk (8.1 waves of CTAs)
    for (int l = 0; l < c.depth; ++l) {
      const VitBlock& b = h->blocks[l];
      for (int s0 = 0; s0 < nb; s0 += sub_a) {
        const int ns = std::min(sub_a, nb - s0);
        const long long roff = static_cast<long long>(s0) * h->npad;
        LayerNormArgs ls = la;
        ls.rows = static_cast<long long>(ns) * h->npad;
        ls.reverse = next_dir();
        WVN_PROPAGATE(layernorm_rows(x + roff * D, b.norm1_w, b.norm1_b,
                                     xn + roff * D, nullptr, ls, s));
        if (h->precise) {
          GemmArgs g;
          float* qkv = reinterpret_cast<float*>(h->qkv_f32.p) + roff * 3 * D;
          g.M = ns * h->npad; g.N = 3 * D; g.K = D; g.epi = EPI_F32; g.bias = b.qkv_b;
          g.out = qkv; g.ldo = 3 * D;
          WVN_PROPAGATE(gemm_bf16(g, xn + roff * D, D, b.qkv_w, 0, s));
          WVN_PROPAGATE(attention_f32_debug(qkv, attn + roff * D, ns, c.heads, h->npad, h->n_valid, D, 0.125f, s));
          continue;
        }
        GemmArgs g;
        g.M = ns * h->npad; g.N = 3 * D; g.K = D; g.epi = EPI_QKV; g.bias = b.qkv_b;
        g.npad = h->npad; g.dim = D; g.heads = c.heads;
        const long long hoff = static_cast<long long>(s0) * c.heads * h->npad * 64;  // frames are outermost in q / k / vt
        g.q = reinterpret_cast<__nv_bfloat16*>(h->q.p) + hoff;
        g.k = reinterpret_cast<__nv_bfloat16*>(h->k.p) + hoff;
        g.vt = reinterpret_cast<__nv_bfloat16*>(h->vt.p) + hoff;
        g.reverse_m = next_dir();
        WVN_PROPAGATE(gemm_bf16(g, xn + roff * D, D, b.qkv_w, 0, s));
        AttnArgs a;
        a.batch = ns; a.heads = c.heads; a.npad = h->npad; a.n_valid = h->n_valid;
        a.scale_log2 = 0.125f * 1.4426950408889634f;  // head_dim 64: 64^-0.5 * log2(e)
        a.out = attn + roff * D; a.ldo = D;
        a.reverse = next_dir();
        WVN_PROPAGATE(attention_bf16(a, g.q, g.k, g.vt, s));
      }
      for (int s0 = 0; s0 < nb; s0 += sub) {
        const int ns = std::min(sub, nb - s0);
        const long long roff = static_cast<long long>(s0) * h->npad;
        const int srows = ns * h->npad;
        LayerNormArgs ls = la;
        ls.rows = srows;
        {
          GemmArgs g;
          g.M = srows; g.N = D; g.K = D; g.epi = EPI_RESID_F32; g.bias = b.proj_b;
          g.out = x + roff * D; g.ldo = D;
          g.reverse_m = next_dir();
          WVN_PROPAGATE(gemm_bf16(g, attn + roff * D, D, b.proj_w, 0, s));
        }
        ls.reverse = next_dir();
        WVN_PROPAGATE(layernorm_rows(x + roff * D, b.norm2_w, b.norm2_b,
                                     xn + roff * D, nullptr, ls, s));
        {
          GemmArgs g;
          g.M = srows; g.N = c.mlp_dim; g.K = D; g.epi = EPI_BF16; g.act = ACT_GELU;
          g.bias = b.fc1_b; g.out = h->hid.p; g.ldo = c.mlp_dim;  // hid is reused per sub-chunk
          if (h->ffn == WVN_VIT_FFN_SWIGLU) {
            // w12 -> silu(gate) * value, the 2 mlp_dim products never stored
            g.N = 2 * c.mlp_dim; g.epi = EPI_SWIGLU; g.act = ACT_NONE;
          }
          g.reverse_m = next_dir();
          WVN_PROPAGATE(gemm_bf16(g, xn + roff * D, D, b.fc1_w, 0, s));
        }
        {
          GemmArgs g;
          g.M = srows; g.N = D; g.K = c.mlp_dim; g.epi = EPI_RESID_F32; g.bias = b.fc2_b;
          g.out = x + roff * D; g.ldo = D;
          g.reverse_m = next_dir();
          WVN_PROPAGATE(gemm_bf16(g, h->hid.p, c.mlp_dim, b.fc2_w, 0, s));
        }
      }
    }
    __nv_bfloat16* tok_bf = reinterpret_cast<__nv_bfloat16*>(h->tok_bf16.p) + static_cast<long long>(b0) * h->npad * D;
    float* tok_f = tokens_out ? tokens_out + static_cast<long long>(b0) * h->P * D : nullptr;
    la.reverse = next_dir();
    WVN_PROPAGATE(layernorm_rows(x, h->norm_w, h->norm_b, tok_bf, tok_f, la, s));
  }
  h->last_batch = batch;
  return WVN_OK;
}

int vit_stego_head(wvn_vit* h, int batch, float* out, cudaStream_t s) {
  WVN_REQUIRE(h->cfg.head_out > 0, "wvn_vit_stego_head: handle was created without a head");
  WVN_REQUIRE(h->last_batch > 0 && batch == h->last_batch, "wvn_vit_stego_head: call wvn_vit_forward with the same batch first");
  WVN_PROPAGATE(h->weights.check_loaded("vit"));
  const int D = h->cfg.dim, rows = batch * h->npad, HO = h->cfg.head_out;
  GemmArgs g;
  g.M = rows; g.N = D; g.K = D; g.epi = EPI_BF16; g.act = ACT_RELU; g.bias = h->hidden_b;
  g.out = h->head_hidden.p; g.ldo = D;
  WVN_PROPAGATE(gemm_bf16(g, h->tok_bf16.p, D, h->hidden_w, 0, s));
  GemmArgs a;
  a.M = rows; a.N = HO; a.K = D; a.epi = EPI_F32; a.bias = h->head_a_b; a.out = out; a.ldo = HO;
  WVN_PROPAGATE(gemm_bf16(a, h->tok_bf16.p, D, h->head_a_w, 0, s));
  GemmArgs b;
  b.M = rows; b.N = HO; b.K = D; b.epi = EPI_RESID_F32; b.bias = nullptr; b.out = out; b.ldo = HO;
  WVN_PROPAGATE(gemm_bf16(b, h->head_hidden.p, D, h->head_b_w, 0, s));
  return WVN_OK;
}

}  // namespace wvn
