// wvn-b200: the C ABI (include/wvn_b200.h) — handles, composite forward passes, primitives.
#include <cuda_bf16.h>

#include <stdio.h>
#include <stdlib.h>

#include <map>
#include <string>
#include <vector>

#include "../../include/wvn_b200.h"
#include "attention.h"
#include "dense_crf.h"
#include "dense_kernels.h"
#include "effnet_kernels.h"
#include "double_mlp_train.h"
#include "gcn_train.h"
#include "gemm.h"
#include "host_common.h"
#include "mlp_train.h"
#include "mission_graph.h"
#include "mlp_train_fused.h"
#include "pixel_head.h"
#include "resnet_kernels.h"
#include "segment_kernels.h"
#include "flow_train.h"
#include "footprint_kernels.h"
#include "slic_kernels.h"
#include "stego_kmeans.h"
#include "train_core.h"
#include "vit_kernels.h"

using namespace wvn;

namespace {

inline cudaStream_t S(void* s) { return reinterpret_cast<cudaStream_t>(s); }
inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

__global__ void cast_f32_to_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    dst[i] = __float2bfloat16_rn(src[i]);
}

// fp32 rows [rows, dim] -> bf16 rows [rows, ld] (padding columns left untouched = zero)
__global__ void cast_rows_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long rows, int dim,
                                 long long ld) {
  const long long n = rows * dim;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / dim;
    const int c = static_cast<int>(i - r * dim);
    dst[r * ld + c] = __float2bfloat16_rn(src[i]);
  }
}

int cast_to_bf16(const float* src, void* dst, long long n, cudaStream_t s) {
  if (n <= 0) return WVN_OK;
  int blocks = static_cast<int>(std::min<long long>((n + 255) / 256, 4096));
  cast_f32_to_bf16_kernel<<<blocks, 256, 0, s>>>(src, reinterpret_cast<__nv_bfloat16*>(dst), n);
  WVN_CHECK_LAUNCH("cast_f32_to_bf16_kernel");
  return WVN_OK;
}

struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  int alloc(size_t n) {
    bytes = n;
    WVN_CHECK_CUDA(cudaMalloc(&p, n ? n : 1));
    WVN_CHECK_CUDA(cudaMemset(p, 0, n ? n : 1));
    return WVN_OK;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
  }
};

struct Weight {
  void* p = nullptr;   // device storage (fp32 or bf16)
  long long numel = 0;
  bool bf16 = false;
  bool loaded = false;
  int cols = 0, ld = 0;  // bf16 rows of `cols` elements stored `ld` apart (0: dense)
};

}  // namespace

// ============================================================================================
// ViT handle
// ============================================================================================
struct wvn_vit {
  wvn_vit_config cfg;
  // t0: first patch row of a frame (1 + register tokens); rows [t0, n_valid) are the P patches
  int grid = 0, P = 0, t0 = 1, n_valid = 0, npad = 0, kpe = 0, kpe_ld = 0, chunk = 0;
  std::map<std::string, Weight> w;
  std::vector<DevBuf> owned;
  // workspaces (per chunk)
  DevBuf x, xn, q, k, vt, attn, hid, ape, stage;
  // per max_batch
  DevBuf tok_bf16, head_hidden;
  DevBuf qkv_f32;        // only with $WVN_VIT_PRECISE=1 at create: fp32 QKV projections of one chunk (parity-debug attention)
  bool precise = false;
  bool forwarded = false;
  int last_batch = 0;

  // cols / ld: a bf16 matrix whose rows of `cols` elements are stored `ld` apart (the pad columns stay zero)
  int add_weight(const std::string& name, long long numel, bool bf16, int cols = 0, int ld = 0) {
    DevBuf b;
    const long long stored = cols > 0 ? numel / cols * ld : numel;
    WVN_PROPAGATE(b.alloc(static_cast<size_t>(stored) * (bf16 ? 2 : 4)));
    owned.push_back(b);
    Weight wt;
    wt.p = b.p; wt.numel = numel; wt.bf16 = bf16; wt.cols = cols; wt.ld = ld;
    w[name] = wt;
    return WVN_OK;
  }
  template <class T>
  T* wp(const std::string& name) { return reinterpret_cast<T*>(w[name].p); }
};

extern "C" {

const char* wvn_last_error(void) { return last_error(); }
int wvn_version(void) { return 108; }

int wvn_check_device(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) return set_error(WVN_ERR_NO_DEVICE, "no CUDA device visible");
  int dev = 0;
  cudaGetDevice(&dev);
  int major = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  int minor = 0;
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (major != 9 || minor != 0)
    return set_error(WVN_ERR_NO_DEVICE, "device %d has compute capability %d.%d, need 9.0 (sm_90a)", dev, major, minor);
  return WVN_OK;
}

long long wvn_launch_count(void) { return launch_count(); }
void wvn_profile_enable(int category_mask) { prof_enable(category_mask); }
int wvn_profile_collect(float* host_ms, long long* host_launches) {
  WVN_REQUIRE(host_ms && host_launches, "wvn_profile_collect: null argument");
  return prof_collect(host_ms, host_launches);
}

// -------------------------------------------------------------------------------- primitives
int wvn_gemm_bf16(const void* a, long long lda, const void* w, const float* bias, void* out, long long ldo, int m, int n,
                  int k, int out_kind, int act, int block_n, void* stream) {
  GemmArgs g;
  g.M = m; g.N = n; g.K = k;
  g.epi = out_kind == 0 ? EPI_BF16 : (out_kind == 1 ? EPI_F32 : EPI_RESID_F32);
  WVN_REQUIRE(out_kind >= 0 && out_kind <= 2, "wvn_gemm_bf16: out_kind %d", out_kind);
  g.act = act; g.bias = bias; g.out = out; g.ldo = ldo;
  return gemm_bf16(g, a, lda, w, block_n, S(stream));
}

int wvn_gemm_bf16_ex(const wvn_gemm_ex_args* x, void* stream) {
  WVN_REQUIRE(x, "wvn_gemm_bf16_ex: null argument");
  GemmArgs g;
  g.M = x->m; g.N = x->n; g.K = x->k; g.epi = x->epi; g.act = x->act;
  g.bias = x->bias; g.out = x->out; g.ldo = x->ldo;
  g.pos = x->pos; g.tokens_in = x->tokens_in; g.npad = x->npad;
  g.dim = x->dim; g.heads = x->heads; g.q = x->q_out; g.k = x->k_out; g.vt = x->vt_out;
  g.feat = x->feat; g.trav_col = x->trav_col; g.x = x->x; g.ldx = x->ldx; g.trav = x->trav; g.conf = x->conf;
  g.loss_reco = x->loss_reco; g.cg_mean = x->cg_mean; g.cg_std = x->cg_std; g.cg_std_factor = x->cg_std_factor;
  g.reverse_m = x->reverse_m; g.registers = x->registers;
  g.residual = x->residual; g.ldr = x->ldr;
  return gemm_bf16(g, x->a, x->lda, x->w, x->block_n, S(stream));
}

int wvn_attention_bf16(const void* q, const void* k, const void* vt, void* out, int batch, int heads, int npad,
                       int n_valid, float scale, void* stream) {
  AttnArgs a;
  a.batch = batch; a.heads = heads; a.npad = npad; a.n_valid = n_valid;
  a.scale_log2 = scale * 1.4426950408889634f;
  a.out = out; a.ldo = static_cast<long long>(heads) * 64;
  return attention_bf16(a, q, k, vt, S(stream));
}

int wvn_layernorm(const float* x, const float* gamma, const float* beta, void* out_bf16, long long rows, int dim,
                  float eps, void* stream) {
  return wvn_layernorm_ex(x, gamma, beta, out_bf16, nullptr, rows, dim, eps, 0, 0, 1, 0, stream);
}

// -------------------------------------------------------------------------------- ViT primitives, exposed for testing
int wvn_image_to_patches(const void* img, int u8_hwc, int batch, int in_h, int in_w, int resized_h, int resized_w,
                         int image_size, int patch, int frame0, int src_frames, int flip_from, void* out_bf16,
                         void* stream) {
  WVN_REQUIRE(img && out_bf16, "wvn_image_to_patches: null argument");
  ImagePatchArgs a;
  WVN_PROPAGATE(image_patch_args(batch, in_h, in_w, resized_h, resized_w, image_size, patch, frame0, src_frames, flip_from,
                                 &a));
  return image_to_patches(img, u8_hwc != 0, out_bf16, a, S(stream));
}

int wvn_init_token_rows(float* x, const float* cls, const float* pos, const float* reg, int registers, int batch, int npad,
                        int n_valid, int dim, void* stream) {
  WVN_REQUIRE(x && cls && pos, "wvn_init_token_rows: null argument");
  WVN_REQUIRE(batch > 0 && dim > 0 && n_valid >= 1 + registers && npad >= n_valid,
              "wvn_init_token_rows: bad geometry (batch %d, npad %d, n_valid %d, registers %d)", batch, npad, n_valid,
              registers);
  return init_token_rows(x, cls, pos, reg, registers, batch, npad, n_valid, dim, S(stream));
}

int wvn_layernorm_ex(const float* x, const float* gamma, const float* beta, void* out_bf16, float* out_f32,
                     long long rows, int dim, float eps, int npad, int n_valid, int row0, int reverse, void* stream) {
  WVN_REQUIRE(x && gamma && beta && (out_bf16 || out_f32), "wvn_layernorm_ex: null argument");
  WVN_REQUIRE(out_f32 == nullptr || (npad > 0 && rows % npad == 0 && 0 <= row0 && row0 <= n_valid && n_valid <= npad),
              "wvn_layernorm_ex: fp32 output needs rows %% npad == 0 and 0 <= row0 <= n_valid <= npad");
  LayerNormArgs a;
  a.rows = rows; a.dim = dim; a.eps = eps; a.npad = npad; a.n_valid = n_valid; a.row0 = row0; a.reverse = reverse != 0;
  return layernorm_rows(x, gamma, beta, out_bf16, out_f32, a, S(stream));
}

int wvn_attention_f32_debug(const float* qkv, void* out_bf16, int batch, int heads, int npad, int n_valid, int dim,
                            float scale, void* stream) {
  WVN_REQUIRE(qkv && out_bf16, "wvn_attention_f32_debug: null argument");
  WVN_REQUIRE(batch > 0 && heads > 0 && 0 < n_valid && n_valid <= npad, "wvn_attention_f32_debug: bad geometry");
  return attention_f32_debug(qkv, out_bf16, batch, heads, npad, n_valid, dim, scale, S(stream));
}

// -------------------------------------------------------------------------------- ViT
int wvn_vit_create(const wvn_vit_config* cfg, wvn_vit_t** out) {
  WVN_REQUIRE(cfg && out, "wvn_vit_create: null argument");
  WVN_PROPAGATE(wvn_check_device());
  WVN_REQUIRE(cfg->dim == 384 || cfg->dim == 768, "vit: dim %d unsupported (384, 768)", cfg->dim);
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
  auto add = [&](const std::string& n, long long numel, bool bf) { if (rc == WVN_OK) rc = h->add_weight(n, numel, bf); };
  add("cls_token", D, false);
  add("pos_embed", static_cast<long long>(1 + h->P) * D, false);
  if (cfg->registers > 0) add("register_tokens", static_cast<long long>(cfg->registers) * D, false);
  if (rc == WVN_OK) rc = h->add_weight("patch_embed.proj.weight", static_cast<long long>(D) * h->kpe, true, h->kpe, h->kpe_ld);
  add("patch_embed.proj.bias", D, false);
  for (int i = 0; i < cfg->depth; ++i) {
    const std::string b = "blocks." + std::to_string(i) + ".";
    add(b + "norm1.weight", D, false);
    add(b + "norm1.bias", D, false);
    add(b + "attn.qkv.weight", 3ll * D * D, true);
    add(b + "attn.qkv.bias", 3 * D, false);
    add(b + "attn.proj.weight", static_cast<long long>(D) * D, true);
    add(b + "attn.proj.bias", D, false);
    add(b + "norm2.weight", D, false);
    add(b + "norm2.bias", D, false);
    add(b + "mlp.fc1.weight", static_cast<long long>(cfg->mlp_dim) * D, true);
    add(b + "mlp.fc1.bias", cfg->mlp_dim, false);
    add(b + "mlp.fc2.weight", static_cast<long long>(D) * cfg->mlp_dim, true);
    add(b + "mlp.fc2.bias", D, false);
  }
  add("norm.weight", D, false);
  add("norm.bias", D, false);
  if (cfg->head_out > 0) {
    add("stego.head_a.weight", static_cast<long long>(cfg->head_out) * D, true);
    add("stego.head_a.bias", cfg->head_out, false);
    add("stego.hidden.weight", static_cast<long long>(D) * D, true);
    add("stego.hidden.bias", D, false);
    add("stego.head_b.weight", static_cast<long long>(cfg->head_out) * D, true);
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
  alloc(h->stage, 8u << 20);
  alloc(h->tok_bf16, static_cast<size_t>(cfg->max_batch) * h->npad * D * 2);
  if (cfg->head_out > 0) alloc(h->head_hidden, static_cast<size_t>(cfg->max_batch) * h->npad * D * 2);
  {
    // parity-debug mode (SURVEY.md §7): Q K^T, softmax and P V in fp32 on fp32 projections, ~40x slower attention
    const char* e = getenv("WVN_VIT_PRECISE");
    h->precise = e && atoi(e) == 1;
    if (h->precise) alloc(h->qkv_f32, rows * 3 * D * 4);
  }
  if (rc != WVN_OK) {
    wvn_vit_destroy(h);
    return rc;
  }
  *out = h;
  return WVN_OK;
}

void wvn_vit_destroy(wvn_vit_t* h) {
  if (!h) return;
  for (auto& b : h->owned) b.release();
  for (DevBuf* b : {&h->x, &h->xn, &h->q, &h->k, &h->vt, &h->attn, &h->hid, &h->ape, &h->stage, &h->tok_bf16,
                    &h->head_hidden, &h->qkv_f32})
    b->release();
  delete h;
}

int wvn_vit_npad(const wvn_vit_t* h) { return h ? h->npad : 0; }

// Copies fp32 `data` (host or device) into a handle's weight: fp32 storage as is, bf16 storage cast on the device (through
// the `stage` buffer when the source is host memory), pitched rows into their padded rows.
static int load_weight(Weight& wt, DevBuf& stage, const char* name, const float* data, long long numel) {
  WVN_REQUIRE(wt.numel == numel, "set_weight: '%s' expects %lld elements, got %lld", name, wt.numel, numel);
  cudaPointerAttributes attr;
  bool on_device = false;
  if (cudaPointerGetAttributes(&attr, data) == cudaSuccess)
    on_device = (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged);
  else
    cudaGetLastError();
  // fp32 destination: copy straight in; bf16 destination: stage (if host) + cast on device
  if (!wt.bf16) {
    WVN_CHECK_CUDA(cudaMemcpy(wt.p, data, numel * 4, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
  } else if (wt.cols > 0) {
    // pitched rows: stage whole rows, cast each into its row of the padded storage
    const long long chunk_rows = static_cast<long long>(stage.bytes / 4) / wt.cols;
    const long long rows = numel / wt.cols;
    for (long long r0 = 0; r0 < rows; r0 += chunk_rows) {
      const long long n = std::min(chunk_rows, rows - r0);
      const float* src = data + r0 * wt.cols;
      if (!on_device) {
        WVN_CHECK_CUDA(cudaMemcpy(stage.p, src, n * wt.cols * 4, cudaMemcpyHostToDevice));
        src = reinterpret_cast<const float*>(stage.p);
      }
      const int blocks = static_cast<int>(std::min<long long>((n * wt.cols + 255) / 256, 4096));
      cast_rows_kernel<<<blocks, 256, 0, 0>>>(src, reinterpret_cast<__nv_bfloat16*>(wt.p) + r0 * wt.ld, n, wt.cols, wt.ld);
      WVN_CHECK_LAUNCH("cast_rows_kernel");
      WVN_CHECK_CUDA(cudaStreamSynchronize(0));
    }
  } else {
    const long long chunk_elems = static_cast<long long>(stage.bytes / 4);
    for (long long off = 0; off < numel; off += chunk_elems) {
      const long long n = std::min(chunk_elems, numel - off);
      const float* src = data + off;
      if (!on_device) {
        WVN_CHECK_CUDA(cudaMemcpy(stage.p, src, n * 4, cudaMemcpyHostToDevice));
        src = reinterpret_cast<const float*>(stage.p);
      }
      WVN_PROPAGATE(cast_to_bf16(src, reinterpret_cast<__nv_bfloat16*>(wt.p) + off, n, 0));
      WVN_CHECK_CUDA(cudaStreamSynchronize(0));
    }
  }
  wt.loaded = true;
  return WVN_OK;
}


int wvn_vit_set_weight(wvn_vit_t* h, const char* name, const float* data, long long numel) {
  WVN_REQUIRE(h && name && data, "wvn_vit_set_weight: null argument");
  auto it = h->w.find(name);
  WVN_REQUIRE(it != h->w.end(), "wvn_vit_set_weight: unknown weight '%s'", name);
  return load_weight(it->second, h->stage, name, data, numel);
}

static int vit_check_loaded(wvn_vit* h, bool need_head) {
  for (auto& kv : h->w) {
    const bool is_head = kv.first.rfind("stego.", 0) == 0;
    if (is_head && !need_head) continue;
    if (!kv.second.loaded) return set_error(WVN_ERR_STATE, "vit: weight '%s' was never set", kv.first.c_str());
  }
  return WVN_OK;
}

constexpr int kDefaultSubAttn = 1 << 30;  // frames per (LN1, QKV, attention) pass: one pass over the whole chunk

namespace {
int vit_forward_impl(wvn_vit_t* h, const void* img, bool u8_hwc, int batch, int in_h, int in_w, int resized_h, int resized_w,
                     float* tokens_out, void* stream, bool flip_tta = false);
}

int wvn_vit_forward_tta(wvn_vit_t* h, const float* img, int batch, int in_h, int in_w, int resized_h, int resized_w,
                        float* tokens_out, void* stream) {
  return vit_forward_impl(h, img, false, batch, in_h, in_w, resized_h, resized_w, tokens_out, stream, true);
}

int wvn_vit_forward(wvn_vit_t* h, const float* img, int batch, int in_h, int in_w, int resized_h, int resized_w,
                    float* tokens_out, void* stream) {
  return vit_forward_impl(h, img, false, batch, in_h, in_w, resized_h, resized_w, tokens_out, stream);
}

int wvn_vit_forward_u8(wvn_vit_t* h, const unsigned char* img_hwc, int batch, int in_h, int in_w, int resized_h,
                       int resized_w, float* tokens_out, void* stream) {
  return vit_forward_impl(h, img_hwc, true, batch, in_h, in_w, resized_h, resized_w, tokens_out, stream);
}

namespace {
// flip_tta: `batch` source frames are run twice — frames [batch, 2*batch) of the activation layout / tokens_out are
// the backbone's output on the horizontally flipped TRANSFORMED images (Stego.get_code's second pass).
int vit_forward_impl(wvn_vit_t* h, const void* img, bool u8_hwc, int src_batch, int in_h, int in_w, int resized_h, int resized_w,
                     float* tokens_out, void* stream, bool flip_tta) {
  const int batch = flip_tta ? 2 * src_batch : src_batch;
  WVN_REQUIRE(h && img, "wvn_vit_forward: null argument");
  WVN_REQUIRE(batch > 0 && batch <= h->cfg.max_batch, "wvn_vit_forward: batch %d outside (0, %d]", batch, h->cfg.max_batch);
  WVN_REQUIRE(resized_h >= h->cfg.image_size && resized_w >= h->cfg.image_size,
              "wvn_vit_forward: resized image %dx%d smaller than the crop %d", resized_h, resized_w, h->cfg.image_size);
  WVN_PROPAGATE(vit_check_loaded(h, false));
  cudaStream_t s = S(stream);
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
    const float* reg = c.registers > 0 ? h->wp<float>("register_tokens") : nullptr;
    WVN_PROPAGATE(init_token_rows(x, h->wp<float>("cls_token"), h->wp<float>("pos_embed"), reg, c.registers, nb, h->npad,
                                  h->n_valid, D, s));
    {
      GemmArgs g;
      g.M = nb * h->P; g.N = D; g.K = h->kpe; g.epi = EPI_PATCH; g.bias = h->wp<float>("patch_embed.proj.bias");
      g.out = x; g.ldo = D; g.pos = h->wp<float>("pos_embed"); g.tokens_in = h->P; g.npad = h->npad;
      g.registers = c.registers;
      WVN_PROPAGATE(gemm_bf16(g, h->ape.p, h->kpe_ld, h->wp<void>("patch_embed.proj.weight"), 0, s));
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
      const std::string b = "blocks." + std::to_string(l) + ".";
      for (int s0 = 0; s0 < nb; s0 += sub_a) {
        const int ns = std::min(sub_a, nb - s0);
        const long long roff = static_cast<long long>(s0) * h->npad;
        LayerNormArgs ls = la;
        ls.rows = static_cast<long long>(ns) * h->npad;
        ls.reverse = next_dir();
        WVN_PROPAGATE(layernorm_rows(x + roff * D, h->wp<float>(b + "norm1.weight"), h->wp<float>(b + "norm1.bias"),
                                     xn + roff * D, nullptr, ls, s));
        if (h->precise) {
          GemmArgs g;
          float* qkv = reinterpret_cast<float*>(h->qkv_f32.p) + roff * 3 * D;
          g.M = ns * h->npad; g.N = 3 * D; g.K = D; g.epi = EPI_F32; g.bias = h->wp<float>(b + "attn.qkv.bias");
          g.out = qkv; g.ldo = 3 * D;
          WVN_PROPAGATE(gemm_bf16(g, xn + roff * D, D, h->wp<void>(b + "attn.qkv.weight"), 0, s));
          WVN_PROPAGATE(attention_f32_debug(qkv, attn + roff * D, ns, c.heads, h->npad, h->n_valid, D, 0.125f, s));
          continue;
        }
        GemmArgs g;
        g.M = ns * h->npad; g.N = 3 * D; g.K = D; g.epi = EPI_QKV; g.bias = h->wp<float>(b + "attn.qkv.bias");
        g.npad = h->npad; g.dim = D; g.heads = c.heads;
        const long long hoff = static_cast<long long>(s0) * c.heads * h->npad * 64;  // frames are outermost in q / k / vt
        g.q = reinterpret_cast<__nv_bfloat16*>(h->q.p) + hoff;
        g.k = reinterpret_cast<__nv_bfloat16*>(h->k.p) + hoff;
        g.vt = reinterpret_cast<__nv_bfloat16*>(h->vt.p) + hoff;
        g.reverse_m = next_dir();
        WVN_PROPAGATE(gemm_bf16(g, xn + roff * D, D, h->wp<void>(b + "attn.qkv.weight"), 0, s));
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
          g.M = srows; g.N = D; g.K = D; g.epi = EPI_RESID_F32; g.bias = h->wp<float>(b + "attn.proj.bias");
          g.out = x + roff * D; g.ldo = D;
          g.reverse_m = next_dir();
          WVN_PROPAGATE(gemm_bf16(g, attn + roff * D, D, h->wp<void>(b + "attn.proj.weight"), 0, s));
        }
        ls.reverse = next_dir();
        WVN_PROPAGATE(layernorm_rows(x + roff * D, h->wp<float>(b + "norm2.weight"), h->wp<float>(b + "norm2.bias"),
                                     xn + roff * D, nullptr, ls, s));
        {
          GemmArgs g;
          g.M = srows; g.N = c.mlp_dim; g.K = D; g.epi = EPI_BF16; g.act = ACT_GELU;
          g.bias = h->wp<float>(b + "mlp.fc1.bias"); g.out = h->hid.p; g.ldo = c.mlp_dim;  // hid is reused per sub-chunk
          g.reverse_m = next_dir();
          WVN_PROPAGATE(gemm_bf16(g, xn + roff * D, D, h->wp<void>(b + "mlp.fc1.weight"), 0, s));
        }
        {
          GemmArgs g;
          g.M = srows; g.N = D; g.K = c.mlp_dim; g.epi = EPI_RESID_F32; g.bias = h->wp<float>(b + "mlp.fc2.bias");
          g.out = x + roff * D; g.ldo = D;
          g.reverse_m = next_dir();
          WVN_PROPAGATE(gemm_bf16(g, h->hid.p, c.mlp_dim, h->wp<void>(b + "mlp.fc2.weight"), 0, s));
        }
      }
    }
    __nv_bfloat16* tok_bf = reinterpret_cast<__nv_bfloat16*>(h->tok_bf16.p) + static_cast<long long>(b0) * h->npad * D;
    float* tok_f = tokens_out ? tokens_out + static_cast<long long>(b0) * h->P * D : nullptr;
    la.reverse = next_dir();
    WVN_PROPAGATE(layernorm_rows(x, h->wp<float>("norm.weight"), h->wp<float>("norm.bias"), tok_bf, tok_f, la, s));
  }
  h->forwarded = true;
  h->last_batch = batch;
  return WVN_OK;
}
}  // namespace

int wvn_vit_stego_head(wvn_vit_t* h, int batch, float* out, void* stream) {
  WVN_REQUIRE(h && out, "wvn_vit_stego_head: null argument");
  WVN_REQUIRE(h->cfg.head_out > 0, "wvn_vit_stego_head: handle was created without a head");
  WVN_REQUIRE(h->forwarded && batch == h->last_batch, "wvn_vit_stego_head: call wvn_vit_forward with the same batch first");
  WVN_PROPAGATE(vit_check_loaded(h, true));
  cudaStream_t s = S(stream);
  const int D = h->cfg.dim, rows = batch * h->npad, HO = h->cfg.head_out;
  GemmArgs g;
  g.M = rows; g.N = D; g.K = D; g.epi = EPI_BF16; g.act = ACT_RELU; g.bias = h->wp<float>("stego.hidden.bias");
  g.out = h->head_hidden.p; g.ldo = D;
  WVN_PROPAGATE(gemm_bf16(g, h->tok_bf16.p, D, h->wp<void>("stego.hidden.weight"), 0, s));
  GemmArgs a;
  a.M = rows; a.N = HO; a.K = D; a.epi = EPI_F32; a.bias = h->wp<float>("stego.head_a.bias"); a.out = out; a.ldo = HO;
  WVN_PROPAGATE(gemm_bf16(a, h->tok_bf16.p, D, h->wp<void>("stego.head_a.weight"), 0, s));
  GemmArgs b;
  b.M = rows; b.N = HO; b.K = D; b.epi = EPI_RESID_F32; b.bias = nullptr; b.out = out; b.ldo = HO;
  WVN_PROPAGATE(gemm_bf16(b, h->head_hidden.p, D, h->wp<void>("stego.head_b.weight"), 0, s));
  return WVN_OK;
}

// -------------------------------------------------------------------------------- dense
int wvn_upsample_dense(const float* tokens, float* out, int batch, int dim, int gh, int gw, int out_h, int out_w,
                       void* stream) {
  DenseArgs a;
  a.batch = batch; a.dim = dim; a.grid_h = gh; a.grid_w = gw; a.out_h = out_h; a.out_w = out_w;
  a.scale_y = out_h > 1 ? static_cast<float>(gh - 1) / static_cast<float>(out_h - 1) : 0.f;
  a.scale_x = out_w > 1 ? static_cast<float>(gw - 1) / static_cast<float>(out_w - 1) : 0.f;
  return upsample_tokens_dense(tokens, out, a, S(stream));
}

int wvn_logits_argmax(const float* logits, long long ld, int col0, int classes, int col0_b, int classes_b, int batch,
                      int npad, int gh, int gw, int out_h, int out_w, long long* seg, long long* seg_b, void* stream) {
  LogitsArgs a;
  a.batch = batch; a.classes = classes; a.grid_h = gh; a.grid_w = gw; a.out_h = out_h; a.out_w = out_w;
  a.scale_y = static_cast<float>(gh) / static_cast<float>(out_h);
  a.scale_x = static_cast<float>(gw) / static_cast<float>(out_w);
  a.npad = npad; a.ld = ld; a.col0 = col0; a.col0_b = col0_b; a.classes_b = classes_b;
  return logits_argmax(logits, seg, seg_b, a, S(stream));
}

int wvn_flip_average(float* head, int batch, int npad, int grid, long long ld, void* stream) {
  return flip_average(head, batch, npad, grid, ld, S(stream));
}

size_t wvn_stego_kmeans_workspace_bytes(int batch, int k, int code_dim) { return stego_kmeans_workspace_bytes(batch, k, code_dim); }

int wvn_stego_kmeans(float* rows, long long ld, int batch, int npad, int patches, int code_col, int code_dim, int logit_col,
                     int k, int iters, float* centroids_out, void* workspace, void* stream) {
  KmeansArgs a;
  a.batch = batch; a.npad = npad; a.patches = patches; a.ld = ld; a.code_col = code_col; a.code_dim = code_dim;
  a.logit_col = logit_col; a.k = k; a.iters = iters; a.centroids_out = centroids_out;
  return stego_kmeans(rows, a, reinterpret_cast<float*>(workspace), S(stream));
}

// -------------------------------------------------------------------------------- segments
static void seg_ws_layout(int batch, int smax, int gh, int gw, size_t& off_w, size_t& off_adj, size_t& total) {
  const size_t stats = static_cast<size_t>(batch) * smax * 3 * sizeof(unsigned long long);
  off_w = (stats + 255) / 256 * 256;
  const size_t wbytes = static_cast<size_t>(batch) * smax * gh * gw * sizeof(float);
  off_adj = off_w + (wbytes + 255) / 256 * 256;
  total = off_adj + static_cast<size_t>(batch) * smax * ((smax + 31) / 32) * sizeof(unsigned int);
}

size_t wvn_segment_workspace_bytes(int batch, int smax, int gh, int gw) {
  size_t a, b, t;
  seg_ws_layout(batch, smax, gh, gw, a, b, t);
  return t;
}

int wvn_segment_reduce(const long long* seg, int batch, int h, int w, int smax, const float* tokens, int gh, int gw,
                       int dim, float* feat, float* centers, long long* edges, int* n_edges, int max_edges,
                       void* workspace, void* stream) {
  WVN_REQUIRE(seg && workspace, "wvn_segment_reduce: null argument");
  WVN_REQUIRE(feat == nullptr || tokens != nullptr, "wvn_segment_reduce: feat requested without tokens");
  WVN_REQUIRE((edges == nullptr) == (n_edges == nullptr), "wvn_segment_reduce: edges and n_edges go together");
  // dense features exist on (h, h) only (dino_interface.py:87-88): pixels with x >= h have no feature — the reference
  // raises an index error there, so do we
  WVN_REQUIRE(feat == nullptr || w <= h, "wvn_segment_reduce: segment map %dx%d is wider than the (h, h) feature map", h, w);
  size_t off_w, off_adj, total;
  seg_ws_layout(batch, smax, gh, gw, off_w, off_adj, total);
  char* ws = reinterpret_cast<char*>(workspace);
  unsigned long long* stats = reinterpret_cast<unsigned long long*>(ws);
  float* wseg = feat ? reinterpret_cast<float*>(ws + off_w) : nullptr;
  unsigned int* adj = edges ? reinterpret_cast<unsigned int*>(ws + off_adj) : nullptr;
  SegmentArgs a;
  a.batch = batch; a.h = h; a.w = w; a.smax = smax; a.grid_h = gh; a.grid_w = gw; a.dim = dim;
  // dense features are upsampled to (h, h) in the reference (dino_interface.py:87-88)
  a.scale_y = h > 1 ? static_cast<float>(gh - 1) / static_cast<float>(h - 1) : 0.f;
  a.scale_x = h > 1 ? static_cast<float>(gw - 1) / static_cast<float>(h - 1) : 0.f;
  WVN_PROPAGATE(segment_accumulate(seg, a, stats, wseg, adj, S(stream)));
  if (feat || centers) WVN_PROPAGATE(segment_pool(wseg, tokens, stats, feat, centers, a, S(stream)));
  if (edges) WVN_PROPAGATE(adjacency_emit(adj, edges, n_edges, batch, smax, max_edges, S(stream)));
  return WVN_OK;
}

int wvn_segment_relabel(long long* seg, int batch, long long pix_per_frame, int num_labels, int* scratch, int* counts,
                        void* stream) {
  return relabel_compact(seg, scratch, counts, batch, pix_per_frame, num_labels, S(stream));
}

int wvn_segment_maps(const void* seg, int seg_is_int64, int batch, long long hw, const float* trav, const float* conf,
                     int smax, const int* n_rows, float* trav_map, float* conf_map, void* stream) {
  return segment_maps(seg, seg_is_int64 != 0, batch, hw, trav, conf, smax, n_rows, trav_map, conf_map, S(stream));
}

int wvn_supervision_pool(const long long* seg, const float* mask, int batch, int channels, int h, int w, int smax,
                         float* y, unsigned char* y_valid, float* count_ws, void* stream) {
  WVN_REQUIRE(seg && mask && y && y_valid && count_ws, "wvn_supervision_pool: null argument");
  return supervision_pool(seg, mask, batch, channels, h, w, smax, y, y_valid, count_ws, S(stream));
}

void wvn_slic_tables(int* g256, int* m9, int* f4096) { slic_tables(g256, m9, f4096); }

int wvn_slic_geometry(int h, int w, int num_components, int* grid_interval, int* nx, int* ny) {
  WVN_REQUIRE(h > 0 && w > 0 && num_components > 0 && grid_interval && nx && ny, "wvn_slic_geometry: bad argument");
  slic_geometry(h, w, num_components, grid_interval, nx, ny);
  return WVN_OK;
}

struct wvn_crf {
  DenseCrf* crf = nullptr;
};

int wvn_crf_create(int size, int max_classes, int chunk, int iterations, wvn_crf_t** out) {
  WVN_REQUIRE(out, "wvn_crf_create: null argument");
  WVN_PROPAGATE(wvn_check_device());
  DenseCrf* c = nullptr;
  WVN_PROPAGATE(crf_create(size, max_classes, chunk, iterations, &c));
  *out = new wvn_crf{c};
  return WVN_OK;
}

void wvn_crf_destroy(wvn_crf_t* h) {
  if (!h) return;
  crf_destroy(h->crf);
  delete h;
}

size_t wvn_crf_workspace_bytes(const wvn_crf_t* h) { return h ? crf_workspace_bytes(h->crf) : 0; }

static CrfInput crf_input(const void* img, int u8_hwc, int batch, int in_h, int in_w, int resized_h, int resized_w) {
  CrfInput in;
  in.img = img; in.u8_hwc = u8_hwc; in.batch = batch; in.in_h = in_h; in.in_w = in_w;
  in.resized_h = resized_h; in.resized_w = resized_w;
  return in;
}

int wvn_crf_run(wvn_crf_t* h, const void* img, int u8_hwc, int batch, int in_h, int in_w, int resized_h, int resized_w,
                const float* head, long long ld, int npad, int grid, int col0, int classes, int code_col, int code_dim,
                float logit_scale, long long* labels, float* q_out, void* stream) {
  WVN_REQUIRE(h, "wvn_crf_run: null handle");
  CrfInput in = crf_input(img, u8_hwc, batch, in_h, in_w, resized_h, resized_w);
  in.head = head; in.ld = ld; in.npad = npad; in.grid = grid; in.col0 = col0; in.classes = classes;
  in.code_col = code_col; in.code_dim = code_dim; in.logit_scale = logit_scale;
  return crf_run(h->crf, in, labels, q_out, S(stream));
}

int wvn_crf_build(wvn_crf_t* h, const void* img, int u8_hwc, int batch, int in_h, int in_w, int resized_h, int resized_w,
                  void* stream) {
  WVN_REQUIRE(h, "wvn_crf_build: null handle");
  return crf_build(h->crf, crf_input(img, u8_hwc, batch, in_h, in_w, resized_h, resized_w), S(stream));
}

int wvn_crf_filter(wvn_crf_t* h, int which, const float* values, int v, float* out, void* stream) {
  WVN_REQUIRE(h, "wvn_crf_filter: null handle");
  return crf_filter(h->crf, which, values, v, out, S(stream));
}

int wvn_crf_export(wvn_crf_t* h, int which, unsigned long long* keys, int* counts, int* offsets, float* bary, int* m,
                   void* stream) {
  WVN_REQUIRE(h, "wvn_crf_export: null handle");
  return crf_export(h->crf, which, keys, counts, offsets, bary, m, S(stream));
}

size_t wvn_slic_workspace_bytes(int batch, int h, int w, int num_components) {
  return slic_workspace_bytes(batch, h, w, num_components);
}

int wvn_slic(const float* img, int batch, int h, int w, int num_components, float compactness, int iters,
             const int* lut_g, const int* lut_m, const int* lut_f, long long* labels, void* workspace, void* stream) {
  WVN_REQUIRE(img && lut_g && lut_m && lut_f && labels && workspace, "wvn_slic: null argument");
  return slic_segment(img, batch, h, w, num_components, compactness, iters, lut_g, lut_m, lut_f, labels, workspace,
                      S(stream));
}

int wvn_project_and_render(const float* K, const float* pose_camera_in_world, const float* points, const float* colors,
                           int color_batched, int batch, int n_points, int h, int w, const float* traversability,
                           float* masks, float* projected, unsigned char* valid, float* supervision_inout, void* stream) {
  WVN_REQUIRE(K && pose_camera_in_world && points, "wvn_project_and_render: null argument");
  WVN_REQUIRE(colors || (!masks && !supervision_inout), "wvn_project_and_render: colors are required to render");
  FootprintArgs a;
  a.batch = batch; a.n_points = n_points; a.h = h; a.w = w; a.color_batched = color_batched;
  return footprint_render(a, K, pose_camera_in_world, points, colors, traversability, masks, projected, valid,
                          supervision_inout, S(stream));
}

size_t wvn_mission_propagate_workspace_bytes(int max_slots, int smax) {
  return mission_propagate_workspace_bytes(max_slots, smax);
}

int wvn_mission_propagate(const int* slots, const unsigned char* restart, int n_slots, const float* K,
                          const float* pose_cam_in_world, const float* points, int n_points, const float* traversability,
                          const int* seg, float* mask, int h, int w, int smax, float* y, unsigned char* y_valid,
                          int* slot_valid, void* workspace, void* stream) {
  WVN_REQUIRE(slots && K && pose_cam_in_world && points && traversability && seg && mask && y && y_valid && workspace,
              "wvn_mission_propagate: null argument");
  MissionPropagateArgs a;
  a.n_slots = n_slots; a.n_points = n_points; a.h = h; a.w = w; a.smax = smax;
  return mission_propagate(a, slots, restart, K, pose_cam_in_world, points, traversability, seg, mask, y, y_valid,
                           slot_valid, workspace, S(stream));
}

// ============================================================================================
// Convolutional trunks (torchvision ResNet-18 / ResNet-50 and EfficientNet-B0; reference torchvision_interface.py)
// ============================================================================================
}  // extern "C"

namespace {

constexpr int kTrunkRoles = 5;  // activation workspaces a trunk's walk may name

// What a convolutional trunk handle owns: its weights, the host staging buffer of set_weight, the im2col rows and the
// activation workspaces, all sized at create.
struct ConvTrunk {
  std::map<std::string, Weight> w;
  std::vector<DevBuf> owned;
  DevBuf stage, col;
  DevBuf act[kTrunkRoles];

  int add_weight(const std::string& name, long long rows, int cols, bool bf16) {
    // bf16: rows of `cols` elements at the GEMM's W pitch; fp32: dense
    const long long ld = bf16 ? gemm_w_pitch(cols) : cols;
    DevBuf b;
    WVN_PROPAGATE(b.alloc(static_cast<size_t>(rows * ld) * (bf16 ? 2 : 4)));
    owned.push_back(b);
    Weight wt;
    wt.p = b.p; wt.numel = rows * cols; wt.bf16 = bf16;
    if (bf16) { wt.cols = cols; wt.ld = static_cast<int>(ld); }
    w[name] = wt;
    return WVN_OK;
  }
  template <class T>
  T* wp(const std::string& name) { return reinterpret_cast<T*>(w[name].p); }
  int set_weight(const char* name, const float* data, long long numel) {
    auto it = w.find(name);
    WVN_REQUIRE(it != w.end(), "set_weight: unknown weight '%s'", name);
    return load_weight(it->second, stage, name, data, numel);
  }
  int check_loaded(const char* what) const {
    for (auto& kv : w)
      if (!kv.second.loaded) return set_error(WVN_ERR_STATE, "%s: weight '%s' was never set", what, kv.first.c_str());
    return WVN_OK;
  }
  size_t workspace_bytes() const {
    size_t n = col.bytes;
    for (const auto& b : act) n += b.bytes;
    return n;
  }
  void release() {
    for (auto& b : owned) b.release();
    stage.release();
    col.release();
    for (auto& b : act) b.release();
  }
};

enum TrunkPass { RN_REGISTER, RN_SIZE, RN_RUN };

// One walk of a trunk: the same code registers the weights (RN_REGISTER), sizes the workspaces for a batch (RN_SIZE)
// and enqueues the forward (RN_RUN), so the three can never disagree.
struct TrunkRun {
  ConvTrunk* t;
  TrunkPass pass;
  int batch;
  cudaStream_t s;
  size_t need_col = 0, need_act[kTrunkRoles] = {0, 0, 0, 0, 0};
  int rc = WVN_OK;

  void need(int role, size_t bytes) {
    if (role >= 0) need_act[role] = std::max(need_act[role], bytes);
  }

  // k x k convolution of the NHWC map `in` [batch, H, W, C] (batch norm folded in) -> `out` [batch, Ho, Wo, Cout];
  // `role` is the workspace buffer the output lives in (-1: a caller's tap buffer), `residual` is added before the
  // activation.  C and Cout are channel pitches: the rows of `in` and `out` are C and Cout elements apart.
  void conv(const std::string& name, const void* in, int H, int W, int C, int k, int stride, int pad, int Cout,
            void* out, int role, int act, const void* residual, int* Ho_, int* Wo_, const float* img = nullptr,
            bool stem = false) {
    const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
    *Ho_ = Ho; *Wo_ = Wo;
    if (rc != WVN_OK) return;
    const int K = k * k * C;
    const long long M = static_cast<long long>(batch) * Ho * Wo;
    const bool direct = k == 1 && stride == 1 && !stem;
    const long long pitch = gemm_w_pitch(K);
    if (pass == RN_REGISTER) {
      if ((rc = t->add_weight(name + ".weight", Cout, K, true)) != WVN_OK) return;
      rc = t->add_weight(name + ".bias", 1, Cout, false);
      return;
    }
    if (pass == RN_SIZE) {
      if (!direct) need_col = std::max(need_col, static_cast<size_t>(M * pitch * 2));
      need(role, static_cast<size_t>(M * Cout * 2));
      return;
    }
    const void* A = in;
    long long lda = C;
    if (!direct) {
      rc = stem ? im2col_image(img, batch, H, W, k, stride, pad, t->col.p, pitch, s)
               : im2col_nhwc(in, batch, H, W, C, k, stride, pad, t->col.p, pitch, s);
      if (rc != WVN_OK) return;
      A = t->col.p;
      lda = pitch;
    }
    if (M > 0x7fffffff) {
      rc = set_error(WVN_ERR_INVALID, "trunk: %lld output rows", M);
      return;
    }
    GemmArgs g;
    g.M = static_cast<int>(M); g.N = Cout; g.K = K;
    g.epi = residual ? EPI_BF16_RESID : EPI_BF16;
    g.act = act;
    g.bias = t->wp<const float>(name + ".bias");
    g.out = out; g.ldo = Cout;
    g.residual = residual; g.ldr = Cout;
    rc = gemm_bf16(g, A, lda, t->wp<void>(name + ".weight"), 0, s);
  }

  // allocates the workspaces the RN_SIZE walk asked for
  int alloc_workspaces() const {
    WVN_PROPAGATE(t->stage.alloc(8u << 20));
    WVN_PROPAGATE(t->col.alloc(need_col));
    for (int i = 0; i < kTrunkRoles; ++i)
      if (need_act[i] > 0) WVN_PROPAGATE(t->act[i].alloc(need_act[i]));
    return WVN_OK;
  }
};

// Blocks per stage of the two supported depths (torchvision resnet18 / resnet50)
const int kBlocks18[4] = {2, 2, 2, 2};
const int kBlocks50[4] = {3, 4, 6, 3};

}  // namespace

struct wvn_resnet : ConvTrunk {
  wvn_resnet_config cfg;
  int bottleneck = 0;
};

namespace {

struct ResnetRun : TrunkRun {
  wvn_resnet* h;
  ResnetRun(wvn_resnet* h_, TrunkPass p, int b, cudaStream_t st) : TrunkRun{h_, p, b, st}, h(h_) {}

  // The whole trunk; in RN_RUN the four taps are written to taps[0..3] (NHWC bf16).  Buffers: 0 / 1 block input and
  // output (alternating), 2 conv1 out, 3 conv2 out, 4 downsample out.
  void walk(const float* img, void* const* taps) {
    const int S = h->cfg.image_size;
    const bool bn = h->bottleneck != 0;
    const int* blocks = bn ? kBlocks50 : kBlocks18;
    void* A[5];
    for (int i = 0; i < 5; ++i) A[i] = h->act[i].p;
    void* T[4] = {nullptr, nullptr, nullptr, nullptr};
    if (taps) for (int i = 0; i < 4; ++i) T[i] = taps[i];
    int Ho, Wo;
    // stem: conv1 7x7/2 + bn1 + relu (output in buffer 2), max-pool 3x3/2 into buffer 0
    conv("conv1", nullptr, S, S, 3, 7, 2, 3, 64, A[2], 2, ACT_RELU, nullptr, &Ho, &Wo, img, true);
    int H = (Ho - 1) / 2 + 1, W = (Wo - 1) / 2 + 1, C = 64;
    if (pass == RN_SIZE) need(0, static_cast<size_t>(batch) * H * W * C * 2);
    if (pass == RN_RUN && rc == WVN_OK) rc = maxpool3s2_nhwc(A[2], batch, Ho, Wo, 64, A[0], s);
    const void* cur = A[0];
    int cur_role = 0;
    for (int L = 1; L <= 4; ++L) {
      const int planes = 64 << (L - 1), out_c = bn ? planes * 4 : planes;
      for (int blk = 0; blk < blocks[L - 1]; ++blk) {
        const std::string p = "layer" + std::to_string(L) + "." + std::to_string(blk) + ".";
        const int stride = (blk == 0 && L > 1) ? 2 : 1;
        const int out_role = cur_role == 0 ? 1 : 0;
        const bool out_tap = bn ? (L == 4 && blk == blocks[3] - 1) : (blk == blocks[L - 1] - 1);
        void* out = out_tap ? T[bn ? 3 : L - 1] : A[out_role];
        int h1, w1, h2, w2, hd, wd;
        const void* res = cur;
        if (blk == 0 && (stride != 1 || C != out_c)) {
          conv(p + "downsample", cur, H, W, C, 1, stride, 0, out_c, A[4], 4, ACT_NONE, nullptr, &hd, &wd);
          res = A[4];
        }
        if (bn) {
          // taps feat1..feat3: layer{2,3,4}.0.relu, the ReLU after bn1 of each stage's first block
          const bool t1_tap = blk == 0 && L >= 2;
          void* t1 = t1_tap ? T[L - 2] : A[2];
          conv(p + "conv1", cur, H, W, C, 1, 1, 0, planes, t1, t1_tap ? -1 : 2, ACT_RELU, nullptr, &h1, &w1);
          conv(p + "conv2", t1, h1, w1, planes, 3, stride, 1, planes, A[3], 3, ACT_RELU, nullptr, &h2, &w2);
          conv(p + "conv3", A[3], h2, w2, planes, 1, 1, 0, out_c, out, out_tap ? -1 : out_role, ACT_RELU, res, &H, &W);
        } else {
          conv(p + "conv1", cur, H, W, C, 3, stride, 1, planes, A[2], 2, ACT_RELU, nullptr, &h1, &w1);
          conv(p + "conv2", A[2], h1, w1, planes, 3, 1, 1, out_c, out, out_tap ? -1 : out_role, ACT_RELU, res, &H, &W);
        }
        C = out_c;
        cur = out;
        cur_role = out_tap ? -1 : out_role;
      }
    }
  }
};

}  // namespace

extern "C" {

int wvn_resnet_create(const wvn_resnet_config* cfg, wvn_resnet_t** out) {
  WVN_REQUIRE(cfg && out, "wvn_resnet_create: null argument");
  WVN_PROPAGATE(wvn_check_device());
  WVN_REQUIRE(cfg->depth == 18 || cfg->depth == 50, "resnet: depth %d unsupported (18, 50)", cfg->depth);
  WVN_REQUIRE(cfg->image_size >= 32 && cfg->image_size % 32 == 0, "resnet: image size %d must be a multiple of 32",
              cfg->image_size);
  WVN_REQUIRE(cfg->max_batch > 0, "resnet: max_batch must be positive");
  wvn_resnet* h = new wvn_resnet();
  h->cfg = *cfg;
  h->bottleneck = cfg->depth == 50;
  ResnetRun reg(h, RN_REGISTER, cfg->max_batch, 0);
  reg.walk(nullptr, nullptr);
  ResnetRun size(h, RN_SIZE, cfg->max_batch, 0);
  size.walk(nullptr, nullptr);
  int rc = reg.rc;
  if (rc == WVN_OK) rc = size.alloc_workspaces();
  if (rc != WVN_OK) {
    wvn_resnet_destroy(h);
    return rc;
  }
  *out = h;
  return WVN_OK;
}

void wvn_resnet_destroy(wvn_resnet_t* h) {
  if (!h) return;
  h->release();
  delete h;
}

size_t wvn_resnet_workspace_bytes(const wvn_resnet_t* h) { return h ? h->workspace_bytes() : 0; }

int wvn_resnet_set_weight(wvn_resnet_t* h, const char* name, const float* data, long long numel) {
  WVN_REQUIRE(h && name && data, "wvn_resnet_set_weight: null argument");
  return h->set_weight(name, data, numel);
}

int wvn_resnet_forward(wvn_resnet_t* h, const float* img, int batch, void* const* taps, void* stream) {
  WVN_REQUIRE(h && img && taps, "wvn_resnet_forward: null argument");
  WVN_REQUIRE(batch > 0 && batch <= h->cfg.max_batch, "wvn_resnet_forward: batch %d outside (0, %d]", batch,
              h->cfg.max_batch);
  for (int i = 0; i < 4; ++i) WVN_REQUIRE(taps[i], "wvn_resnet_forward: tap %d is null", i);
  WVN_PROPAGATE(h->check_loaded("resnet"));
  ResnetRun run(h, RN_RUN, batch, S(stream));
  run.walk(img, taps);
  return run.rc;
}

}  // extern "C"

// -------------------------------------------------------------------------------- EfficientNet-B0
struct wvn_effnet : ConvTrunk {
  wvn_effnet_config cfg;
  DevBuf partial, gates;  // the depthwise convs' pool sums and the squeeze-excitation gates
};

namespace {

inline int pitch64(int c) { return round_up(c, 64); }

// torchvision efficientnet_b0's stages: (expand ratio, kernel, stride, output channels, blocks)
const int kB0Stages[7][5] = {{1, 3, 1, 16, 1}, {6, 3, 2, 24, 2}, {6, 5, 2, 40, 2}, {6, 3, 2, 80, 3},
                             {6, 5, 1, 112, 3}, {6, 5, 2, 192, 4}, {6, 3, 1, 320, 1}};
// taps feat1..feat4: the expand convs (features.{2,3,4,6}.0.block.0) of these stages' first blocks
const int kB0TapStage[4] = {2, 3, 4, 6};

struct EffnetRun : TrunkRun {
  wvn_effnet* h;
  size_t need_partial = 0, need_gates = 0;
  EffnetRun(wvn_effnet* h_, TrunkPass p, int b, cudaStream_t st) : TrunkRun{h_, p, b, st}, h(h_) {}

  // depthwise k x k conv + folded batch norm + SiLU of `in` [batch, H, W, P] -> buffer 3, with the pool sums
  void depthwise(const std::string& name, const void* in, int H, int W, int P, int k, int stride, int* Ho, int* Wo) {
    const int pad = (k - 1) / 2;
    *Ho = (H + 2 * pad - k) / stride + 1;
    *Wo = (W + 2 * pad - k) / stride + 1;
    if (rc != WVN_OK) return;
    if (pass == RN_REGISTER) {
      if ((rc = t->add_weight(name + ".weight", 1, k * k * P, false)) != WVN_OK) return;
      rc = t->add_weight(name + ".bias", 1, P, false);
      return;
    }
    if (pass == RN_SIZE) {
      need(3, static_cast<size_t>(batch) * *Ho * *Wo * P * 2);
      need_partial = std::max(need_partial, static_cast<size_t>(batch) * depthwise_pool_blocks(*Ho, *Wo) * P * 4);
      return;
    }
    rc = depthwise_silu(in, batch, H, W, P, k, stride, t->wp<const float>(name + ".weight"),
                        t->wp<const float>(name + ".bias"), h->act[3].p, reinterpret_cast<float*>(h->partial.p), s);
  }

  // squeeze-excitation of buffer 3 [batch, Ho, Wo, P] (C real channels, `squeeze` hidden), in place
  void squeeze_excite(const std::string& name, int Ho, int Wo, int C, int P, int squeeze) {
    if (rc != WVN_OK) return;
    if (pass == RN_REGISTER) {
      if ((rc = t->add_weight(name + ".fc1.weight", squeeze, P, false)) != WVN_OK) return;
      if ((rc = t->add_weight(name + ".fc1.bias", 1, squeeze, false)) != WVN_OK) return;
      if ((rc = t->add_weight(name + ".fc2.weight", P, squeeze, false)) != WVN_OK) return;
      rc = t->add_weight(name + ".fc2.bias", 1, P, false);
      return;
    }
    if (pass == RN_SIZE) {
      need_gates = std::max(need_gates, static_cast<size_t>(batch) * P * 4);
      return;
    }
    float* gates = reinterpret_cast<float*>(h->gates.p);
    rc = se_gates(reinterpret_cast<const float*>(h->partial.p), batch, depthwise_pool_blocks(Ho, Wo), Ho * Wo, C, P,
                  t->wp<const float>(name + ".fc1.weight"), t->wp<const float>(name + ".fc1.bias"), squeeze,
                  t->wp<const float>(name + ".fc2.weight"), t->wp<const float>(name + ".fc2.bias"), gates, s);
    if (rc == WVN_OK) rc = channel_scale(h->act[3].p, batch, static_cast<long long>(Ho) * Wo, P, gates, s);
  }

  // The whole trunk at channel pitches rounded up to 64 (pad channels stay zero); in RN_RUN the five taps are written
  // to taps[0..4].  Buffers: 0 / 1 block input and output (alternating), 2 expand out, 3 depthwise out.
  void walk(const float* img, void* const* taps) {
    const int S = h->cfg.image_size;
    void* A[4];
    for (int i = 0; i < 4; ++i) A[i] = h->act[i].p;
    void* T[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    if (taps) for (int i = 0; i < 5; ++i) T[i] = taps[i];
    int H, W;
    // stem: 3 x 3 / 2 conv + bn + SiLU, 32 channels
    conv("features.0", nullptr, S, S, 3, 3, 2, 1, pitch64(32), A[0], 0, ACT_SILU, nullptr, &H, &W, img, true);
    const void* cur = A[0];
    int cur_role = 0, cin = 32, tap = 0;
    for (int st = 0; st < 7; ++st) {
      const int ratio = kB0Stages[st][0], k = kB0Stages[st][1], cout = kB0Stages[st][3];
      for (int blk = 0; blk < kB0Stages[st][4]; ++blk) {
        const std::string p = "features." + std::to_string(st + 1) + "." + std::to_string(blk) + ".block.";
        const int stride = blk == 0 ? kB0Stages[st][2] : 1;
        const int cexp = cin * ratio, pin = pitch64(cin), pexp = pitch64(cexp), pout = pitch64(cout);
        int j = 0, Ho, Wo, h1, w1;
        const void* x = cur;
        if (ratio != 1) {
          const bool is_tap = blk == 0 && tap < 4 && kB0TapStage[tap] == st + 1;
          void* e = is_tap ? T[tap++] : A[2];
          conv(p + "0", cur, H, W, pin, 1, 1, 0, pexp, e, is_tap ? -1 : 2, ACT_SILU, nullptr, &h1, &w1);
          x = e;
          j = 1;
        }
        depthwise(p + std::to_string(j), x, H, W, pexp, k, stride, &Ho, &Wo);
        squeeze_excite(p + std::to_string(j + 1), Ho, Wo, cexp, pexp, std::max(1, cin / 4));
        const int out_role = cur_role == 0 ? 1 : 0;
        const void* res = stride == 1 && cin == cout ? cur : nullptr;
        conv(p + std::to_string(j + 2), A[3], Ho, Wo, pexp, 1, 1, 0, pout, A[out_role], out_role, ACT_NONE, res, &H, &W);
        cur = A[out_role];
        cur_role = out_role;
        cin = cout;
      }
    }
    // head: 1 x 1 conv 320 -> 1280 + bn + SiLU (features.8), the fifth tap
    int h5, w5;
    conv("features.8", cur, H, W, pitch64(cin), 1, 1, 0, 1280, T[4], -1, ACT_SILU, nullptr, &h5, &w5);
  }
};

}  // namespace

extern "C" {

int wvn_effnet_create(const wvn_effnet_config* cfg, wvn_effnet_t** out) {
  WVN_REQUIRE(cfg && out, "wvn_effnet_create: null argument");
  WVN_PROPAGATE(wvn_check_device());
  WVN_REQUIRE(cfg->image_size >= 32 && cfg->image_size % 32 == 0, "effnet: image size %d must be a multiple of 32",
              cfg->image_size);
  WVN_REQUIRE(cfg->max_batch > 0 && cfg->max_batch <= 65535, "effnet: max_batch %d outside (0, 65535]", cfg->max_batch);
  wvn_effnet* h = new wvn_effnet();
  h->cfg = *cfg;
  EffnetRun reg(h, RN_REGISTER, cfg->max_batch, 0);
  reg.walk(nullptr, nullptr);
  EffnetRun size(h, RN_SIZE, cfg->max_batch, 0);
  size.walk(nullptr, nullptr);
  int rc = reg.rc;
  if (rc == WVN_OK) rc = size.alloc_workspaces();
  if (rc == WVN_OK) rc = h->partial.alloc(size.need_partial);
  if (rc == WVN_OK) rc = h->gates.alloc(size.need_gates);
  if (rc != WVN_OK) {
    wvn_effnet_destroy(h);
    return rc;
  }
  *out = h;
  return WVN_OK;
}

void wvn_effnet_destroy(wvn_effnet_t* h) {
  if (!h) return;
  h->release();
  h->partial.release();
  h->gates.release();
  delete h;
}

size_t wvn_effnet_workspace_bytes(const wvn_effnet_t* h) {
  return h ? h->workspace_bytes() + h->partial.bytes + h->gates.bytes : 0;
}

int wvn_effnet_set_weight(wvn_effnet_t* h, const char* name, const float* data, long long numel) {
  WVN_REQUIRE(h && name && data, "wvn_effnet_set_weight: null argument");
  return h->set_weight(name, data, numel);
}

int wvn_effnet_forward(wvn_effnet_t* h, const float* img, int batch, void* const* taps, void* stream) {
  WVN_REQUIRE(h && img && taps, "wvn_effnet_forward: null argument");
  WVN_REQUIRE(batch > 0 && batch <= h->cfg.max_batch, "wvn_effnet_forward: batch %d outside (0, %d]", batch,
              h->cfg.max_batch);
  for (int i = 0; i < 5; ++i) WVN_REQUIRE(taps[i], "wvn_effnet_forward: tap %d is null", i);
  WVN_PROPAGATE(h->check_loaded("effnet"));
  EffnetRun run(h, RN_RUN, batch, S(stream));
  run.walk(img, taps);
  return run.rc;
}

int wvn_depthwise_silu_bf16_nhwc(const void* in, int batch, int h, int w, int pitch, int k, int stride,
                                 const float* weight, const float* bias, void* out, float* partial, void* stream) {
  return depthwise_silu(in, batch, h, w, pitch, k, stride, weight, bias, out, partial, S(stream));
}

int wvn_depthwise_pool_blocks(int ho, int wo) { return depthwise_pool_blocks(ho, wo); }

int wvn_se_gates(const float* partial, int batch, int nblk, int hw, int channels, int pitch, const float* fc1_w,
                 const float* fc1_b, int squeeze, const float* fc2_w, const float* fc2_b, float* gates, void* stream) {
  return se_gates(partial, batch, nblk, hw, channels, pitch, fc1_w, fc1_b, squeeze, fc2_w, fc2_b, gates, S(stream));
}

int wvn_channel_scale_bf16_nhwc(void* x, int batch, long long hw, int pitch, const float* gates, void* stream) {
  return channel_scale(x, batch, hw, pitch, gates, S(stream));
}

int wvn_im2col_bf16_nhwc(const void* in, int batch, int h, int w, int c, int k, int stride, int pad, void* out,
                         long long pitch, void* stream) {
  return im2col_nhwc(in, batch, h, w, c, k, stride, pad, out, pitch, S(stream));
}

int wvn_im2col_image(const float* img, int batch, int h, int w, int k, int stride, int pad, void* out, long long pitch,
                     void* stream) {
  return im2col_image(img, batch, h, w, k, stride, pad, out, pitch, S(stream));
}

int wvn_maxpool3s2_bf16_nhwc(const void* in, int batch, int h, int w, int c, void* out, void* stream) {
  return maxpool3s2_nhwc(in, batch, h, w, c, out, S(stream));
}

int wvn_segment_pool_levels(const long long* seg, int batch, int h, int w, int smax, const float* centers, int levels,
                            void* const* taps, const int* tap_h, const int* tap_w, const int* tap_c, const int* tap_pitch,
                            float* out, void* stream) {
  WVN_REQUIRE(taps && tap_h && tap_w && tap_c && tap_pitch, "wvn_segment_pool_levels: null argument");
  WVN_REQUIRE(levels >= 1 && levels <= kPyramidMaxLevels, "wvn_segment_pool_levels: %d levels (1 .. %d)", levels,
              kPyramidMaxLevels);
  PyramidArgs a;
  a.batch = batch; a.h = h; a.w = w; a.smax = smax; a.levels = levels;
  for (int l = 0; l < levels; ++l) {
    a.taps[l] = taps[l]; a.th[l] = tap_h[l]; a.tw[l] = tap_w[l]; a.tc[l] = tap_c[l]; a.tp[l] = tap_pitch[l];
  }
  return segment_pool_pyramid(seg, centers, a, out, S(stream));
}

int wvn_segment_pool_pyramid(const long long* seg, int batch, int h, int w, int smax, const float* centers,
                             void* const* taps, const int* tap_h, const int* tap_w, const int* tap_c, float* out,
                             void* stream) {
  WVN_REQUIRE(tap_c, "wvn_segment_pool_pyramid: null argument");
  return wvn_segment_pool_levels(seg, batch, h, w, smax, centers, 4, taps, tap_h, tap_w, tap_c, tap_c, out, stream);
}

}  // extern "C"

// ============================================================================================
// Traversability MLP inference handle
// ============================================================================================
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

extern "C" {

static int mlp_infer_create(int dim, int h1, int h2, int chunk_rows, int double_layout, wvn_mlp_infer_t** out) {
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
    wvn_mlp_infer_destroy(h);
    return rc;
  }
  *out = h;
  return WVN_OK;
}

int wvn_mlp_infer_create(int dim, int h1, int h2, int chunk_rows, wvn_mlp_infer_t** out) {
  return mlp_infer_create(dim, h1, h2, chunk_rows, 0, out);
}

int wvn_mlp_infer_create_double(int dim, int h1, int h2, int chunk_rows, wvn_mlp_infer_t** out) {
  MlpShape s;
  s.dim = dim; s.h1 = h1; s.h2 = h2;
  WVN_PROPAGATE(double_mlp_check_shape(s, "wvn_mlp_infer_create_double"));
  return mlp_infer_create(dim, h1, h2, chunk_rows, 1, out);
}

void wvn_mlp_infer_destroy(wvn_mlp_infer_t* h) {
  if (!h) return;
  for (DevBuf* b : {&h->w1, &h->b1, &h->w2, &h->b2, &h->w3, &h->b3, &h->x, &h->a1, &h->a2, &h->wcat, &h->bias_cat,
                    &h->head_consts, &h->tok_bf16, &h->gu, &h->gram})
    b->release();
  delete h;
}

int wvn_mlp_infer_reserve(wvn_mlp_infer_t* h, int tokens_per_frame) {
  WVN_REQUIRE(h && tokens_per_frame > 0, "wvn_mlp_infer_reserve: bad arguments");
  const int P = tokens_per_frame;
  if (h->head_n == 0 || h->fused_tokens >= kFusedFrames * P) return WVN_OK;   // no fused head: nothing to size
  for (DevBuf* b : {&h->tok_bf16, &h->gu, &h->gram}) b->release();
  WVN_PROPAGATE(h->tok_bf16.alloc(static_cast<size_t>(kFusedFrames) * P * h->dim_p * 2));
  WVN_PROPAGATE(h->gu.alloc(static_cast<size_t>(kFusedFrames) * P * h->head_n * 4));
  WVN_PROPAGATE(h->gram.alloc(static_cast<size_t>(kFusedFrames) * P * 5 * 4));
  h->fused_tokens = kFusedFrames * P;
  return WVN_OK;
}

int wvn_mlp_infer_set_params(wvn_mlp_infer_t* h, const float* params, void* stream) {
  WVN_REQUIRE(h && params, "wvn_mlp_infer_set_params: null argument");
  MlpShape sh;
  sh.dim = h->dim; sh.h1 = h->h1; sh.h2 = h->h2;
  if (h->double_layout) {
    MlpShape net;
    net.dim = h->dim; net.h1 = h->net_h1; net.h2 = h->net_h2;
    pack_double_mlp_kernel<<<256, 256, 0, S(stream)>>>(
        params, double_mlp_offsets(net), h->dim, net.h1, net.h2, h->dim_p, h->h1_p, h->h2_p, h->n3_p, h->trav_col,
        reinterpret_cast<__nv_bfloat16*>(h->w1.p), reinterpret_cast<float*>(h->b1.p),
        reinterpret_cast<__nv_bfloat16*>(h->w2.p), reinterpret_cast<float*>(h->b2.p),
        reinterpret_cast<__nv_bfloat16*>(h->w3.p), reinterpret_cast<float*>(h->b3.p));
    WVN_CHECK_LAUNCH("pack_double_mlp_kernel");
    if (h->head_n > 0)
      WVN_PROPAGATE(pixel_head_pack_double(params, net, h->dim_p, h->wcat.p, reinterpret_cast<float*>(h->bias_cat.p),
                                           reinterpret_cast<PixelHeadConsts*>(h->head_consts.p), S(stream)));
    h->loaded = true;
    return WVN_OK;
  }
  pack_mlp_kernel<<<256, 256, 0, S(stream)>>>(
      params, mlp_offsets(sh), h->dim, h->h1, h->h2, h->dim_p, h->h1_p, h->h2_p, h->n3_p, h->trav_col,
      reinterpret_cast<__nv_bfloat16*>(h->w1.p), reinterpret_cast<float*>(h->b1.p),
      reinterpret_cast<__nv_bfloat16*>(h->w2.p), reinterpret_cast<float*>(h->b2.p),
      reinterpret_cast<__nv_bfloat16*>(h->w3.p), reinterpret_cast<float*>(h->b3.p));
  WVN_CHECK_LAUNCH("pack_mlp_kernel");
  if (h->h1 == 256 && h->h2 == 32)
    WVN_PROPAGATE(pixel_head_pack(params, sh, h->dim_p, h->wcat.p, reinterpret_cast<float*>(h->bias_cat.p),
                                  reinterpret_cast<PixelHeadConsts*>(h->head_consts.p), S(stream)));
  h->loaded = true;
  return WVN_OK;
}

// Token-window width of the fused head for this handle and geometry, 0 when the fused head does not take it.
static int fused_window(const wvn_mlp_infer_t* h, int gh, int gw, int out_h, int out_w) {
  if (h->double_layout) return h->head_n > 0 ? pixel_head_supported_double(h->net_h1, h->net_h2, gh, gw, out_h, out_w) : 0;
  return pixel_head_supported(h->h1, h->h2, gh, gw, out_h, out_w);
}

// Fused per-pixel head over frames [b0, b0 + nb): per-token GEMM (G | U | cT) + token Gram + one pixel kernel.
// tok_bf16: the frames' bf16 tokens, frame_rows rows per frame with the patch tokens starting at row row0.
static int pixels_fused_chunk(wvn_mlp_infer_t* h, const void* tok_bf16, long long frame_rows, int row0, int b0, int nb,
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

int wvn_mlp_infer_pixels_vit(wvn_mlp_infer_t* h, wvn_vit_t* vit, int batch, int out_h, int out_w, const float* cg_mean,
                             const float* cg_std, float std_factor, float* trav, float* conf, void* stream) {
  WVN_REQUIRE(h && vit && trav && conf && cg_mean && cg_std, "wvn_mlp_infer_pixels_vit: null argument");
  if (!h->loaded) return set_error(WVN_ERR_STATE, "wvn_mlp_infer_pixels_vit: parameters were never set");
  if (!vit->forwarded || batch > vit->last_batch)
    return set_error(WVN_ERR_STATE, "wvn_mlp_infer_pixels_vit: the backbone holds the tokens of %d frames, %d asked",
                     vit->forwarded ? vit->last_batch : 0, batch);
  WVN_REQUIRE(h->dim == vit->cfg.dim && h->dim_p == vit->cfg.dim, "wvn_mlp_infer_pixels_vit: the MLP takes %d-d features, "
              "the backbone's tokens are %d-d", h->dim, vit->cfg.dim);
  const int g = vit->grid;
  const int ww = fused_window(h, g, g, out_h, out_w);
  WVN_REQUIRE(ww > 0, "wvn_mlp_infer_pixels_vit: geometry outside the fused per-pixel head (use wvn_mlp_infer_pixels)");
  if (h->fused_tokens < kFusedFrames * vit->npad) WVN_PROPAGATE(wvn_mlp_infer_reserve(h, vit->npad));
  for (int b0 = 0; b0 < batch; b0 += kFusedFrames) {
    const int nb = std::min(kFusedFrames, batch - b0);
    const __nv_bfloat16* tok = reinterpret_cast<const __nv_bfloat16*>(vit->tok_bf16.p) +
                               static_cast<long long>(b0) * vit->npad * vit->cfg.dim;
    WVN_PROPAGATE(pixels_fused_chunk(h, tok, vit->npad, vit->t0, b0, nb, g, g, out_h, out_w, ww, cg_mean, cg_std, std_factor, trav,
                                     conf, S(stream)));
  }
  return WVN_OK;
}

int wvn_mlp_infer_pixels(wvn_mlp_infer_t* h, const float* tokens, int batch, int gh, int gw, int out_h, int out_w,
                         const float* cg_mean, const float* cg_std, float std_factor, float* trav, float* conf,
                         void* stream) {
  WVN_REQUIRE(h && tokens && trav && conf && cg_mean && cg_std, "wvn_mlp_infer_pixels: null argument");
  if (!h->loaded) return set_error(WVN_ERR_STATE, "wvn_mlp_infer_pixels: parameters were never set");
  cudaStream_t s = S(stream);
  // any feature width works (the 90-d STEGO code is zero-padded to 128 columns in the bf16 operands)
  const int ww = h->force_unfused ? 0 : fused_window(h, gh, gw, out_h, out_w);
  if (ww > 0) {
    // ---- fused path: per-token GEMM (G | U | cT) + token Gram, then one kernel per chunk of frames
    const int P = gh * gw;
    // workspaces are sized by wvn_mlp_infer_reserve (called by the owner right after create); a larger token grid
    // than reserved grows them here once
    if (h->fused_tokens < kFusedFrames * P) WVN_PROPAGATE(wvn_mlp_infer_reserve(h, P));
    for (int b0 = 0; b0 < batch; b0 += kFusedFrames) {
      const int nb = std::min(kFusedFrames, batch - b0);
      const long long rows = static_cast<long long>(nb) * P;
      const long long elems = rows * h->dim;
      int blocks = static_cast<int>(std::min<long long>((elems + 255) / 256, 8192));
      cast_rows_kernel<<<blocks, 256, 0, s>>>(tokens + static_cast<long long>(b0) * P * h->dim,
                                             reinterpret_cast<__nv_bfloat16*>(h->tok_bf16.p), rows, h->dim, h->dim_p);
      WVN_CHECK_LAUNCH("cast_rows_kernel");
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

int wvn_mlp_infer_rows(wvn_mlp_infer_t* h, const float* x, long long rows, const float* cg_mean, const float* cg_std,
                       float std_factor, float* trav, float* conf, void* stream) {
  WVN_REQUIRE(h && x && trav && conf && cg_mean && cg_std, "wvn_mlp_infer_rows: null argument");
  if (!h->loaded) return set_error(WVN_ERR_STATE, "wvn_mlp_infer_rows: parameters were never set");
  cudaStream_t s = S(stream);
  for (long long r0 = 0; r0 < rows; r0 += h->chunk_rows) {
    const long long n = std::min<long long>(h->chunk_rows, rows - r0);
    const long long elems = n * h->dim;
    int blocks = static_cast<int>(std::min<long long>((elems + 255) / 256, 8192));
    cast_rows_kernel<<<blocks, 256, 0, s>>>(x + r0 * h->dim, reinterpret_cast<__nv_bfloat16*>(h->x.p), n, h->dim,
                                           h->dim_p);
    WVN_CHECK_LAUNCH("cast_rows_kernel");
    WVN_PROPAGATE(mlp_infer_chunk(h, n, r0, cg_mean, cg_std, std_factor, trav, conf, s));
  }
  return WVN_OK;
}

// The padded form runs the same chunks over all groups * rows_per_group rows: the GEMMs' tile shapes depend on N and K
// only (BM is fixed, block_n follows N), so each live row goes through exactly the arithmetic of wvn_mlp_infer_rows.
int wvn_mlp_infer_rows_padded(wvn_mlp_infer_t* h, const float* x, int groups, int rows_per_group, const int* n_rows,
                              const float* cg_mean, const float* cg_std, float std_factor, float* trav, float* conf,
                              void* stream) {
  WVN_REQUIRE(h && x && n_rows && trav && conf && cg_mean && cg_std, "wvn_mlp_infer_rows_padded: null argument");
  WVN_REQUIRE(groups >= 0 && rows_per_group >= 0, "wvn_mlp_infer_rows_padded: bad geometry (groups=%d rows=%d)", groups,
              rows_per_group);
  if (!h->loaded) return set_error(WVN_ERR_STATE, "wvn_mlp_infer_rows_padded: parameters were never set");
  cudaStream_t s = S(stream);
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

// -------------------------------------------------------------------------------- training
static MlpShape shape_of(int dim, int h1, int h2) {
  MlpShape s;
  s.dim = dim; s.h1 = h1; s.h2 = h2;
  return s;
}
static LossCfg loss_of(const wvn_train_config* c) {
  LossCfg l;
  l.w_trav = c->w_trav; l.w_reco = c->w_reco; l.std_factor = c->std_factor; l.anomaly_balanced = c->anomaly_balanced;
  return l;
}
static AdamCfg adam_of(const wvn_train_config* c) {
  AdamCfg a;
  a.lr = c->lr; a.beta1 = c->beta1; a.beta2 = c->beta2; a.eps = c->eps;
  return a;
}

size_t wvn_mlp_param_count(int dim, int h1, int h2) { return mlp_param_count(shape_of(dim, h1, h2)); }
size_t wvn_mlp_train_workspace_bytes(int dim, int h1, int h2, int max_rows) {
  return mlp_train_workspace_floats(shape_of(dim, h1, h2), max_rows) * sizeof(float);
}
size_t wvn_mlp_train_scalars_bytes(void) { return sizeof(TrainScalars); }

int wvn_mlp_train_forward_stats(int dim, int h1, int h2, const float* params, const float* x, const float* y,
                                const unsigned char* y_valid, int rows, int max_rows, void* workspace, void* scalars,
                                void* stream) {
  WVN_REQUIRE(params && x && y && y_valid && workspace && scalars, "wvn_mlp_train_forward_stats: null argument");
  return mlp_train_forward_stats(shape_of(dim, h1, h2), params, x, y, y_valid, rows, max_rows,
                                 reinterpret_cast<float*>(workspace), reinterpret_cast<TrainScalars*>(scalars), S(stream));
}

int wvn_mlp_train_backward(int dim, int h1, int h2, const float* params, const float* x, const float* y,
                           const unsigned char* y_valid, int rows, int max_rows, long long n_total,
                           const wvn_train_config* cfg, void* workspace, void* scalars, float* cg_mean, float* cg_std,
                           float* grads, float* confidence_out, void* stream) {
  WVN_REQUIRE(params && x && y && y_valid && workspace && scalars && cfg && grads && confidence_out,
              "wvn_mlp_train_backward: null argument");
  return mlp_train_backward(shape_of(dim, h1, h2), params, x, y, y_valid, rows, max_rows, n_total, loss_of(cfg),
                            reinterpret_cast<float*>(workspace), reinterpret_cast<TrainScalars*>(scalars), cg_mean,
                            cg_std, grads, confidence_out, S(stream));
}

int wvn_mlp_train_apply(int dim, int h1, int h2, float* params, const float* grads, float* exp_avg, float* exp_avg_sq,
                        long long* step_counter, long long n_total, const wvn_train_config* cfg, void* scalars,
                        void* stream) {
  WVN_REQUIRE(params && grads && exp_avg && exp_avg_sq && step_counter && cfg && scalars,
              "wvn_mlp_train_apply: null argument");
  const long long n = static_cast<long long>(mlp_param_count(shape_of(dim, h1, h2)));
  WVN_PROPAGATE(mlp_train_finalize(reinterpret_cast<TrainScalars*>(scalars), grads, n, n_total, loss_of(cfg), S(stream)));
  return mlp_adam_step(params, grads, exp_avg, exp_avg_sq, n, adam_of(cfg), step_counter, S(stream));
}

__global__ void read_metrics_kernel(const TrainScalars* sc, float* out) {
  out[0] = sc->loss_total; out[1] = sc->loss_trav; out[2] = sc->loss_reco; out[3] = sc->loss_trav_conf;
  out[4] = sc->mean; out[5] = sc->std;
}

int wvn_mlp_train_read_metrics(const void* scalars, float* metrics_out, void* stream) {
  WVN_REQUIRE(scalars && metrics_out, "wvn_mlp_train_read_metrics: null argument");
  read_metrics_kernel<<<1, 1, 0, S(stream)>>>(reinterpret_cast<const TrainScalars*>(scalars), metrics_out);
  WVN_CHECK_LAUNCH("read_metrics_kernel");
  return WVN_OK;
}

int wvn_mlp_forward_f32(int dim, int h1, int h2, const float* params, const float* x, int rows, float* h1_buf,
                        float* h2_buf, float* out, void* stream) {
  WVN_REQUIRE(params && x && h1_buf && h2_buf && out && rows > 0, "wvn_mlp_forward_f32: bad argument");
  return mlp_forward_f32(shape_of(dim, h1, h2), params, x, rows, h1_buf, h2_buf, out, S(stream));
}


// -------------------------------------------------------------------------------- trainers
// A wvn_trainer_t is the address of the learner's Trainer base (train_core.h).
static Trainer* impl(wvn_trainer_t* h) { return reinterpret_cast<Trainer*>(h); }
static wvn_trainer_t* handle_of(Trainer* t) { return reinterpret_cast<wvn_trainer_t*>(t); }

void wvn_trainer_destroy(wvn_trainer_t* t) { delete impl(t); }

int wvn_trainer_set_confidence(wvn_trainer_t* t, int method, float* var, double* running_n, double* running_sum,
                               double* running_sum_of_squares, float kf_proc_cov, float kf_meas_cov) {
  WVN_REQUIRE(t, "wvn_trainer_set_confidence: null trainer");
  return trainer_conf_bind(&impl(t)->conf, method, var, running_n, running_sum, running_sum_of_squares, kf_proc_cov,
                           kf_meas_cov);
}

int wvn_trainer_copy_confidence(wvn_trainer_t* dst, const wvn_trainer_t* src, void* stream) {
  WVN_REQUIRE(dst && src, "wvn_trainer_copy_confidence: null trainer");
  const Trainer* from = reinterpret_cast<const Trainer*>(src);
  WVN_PROPAGATE(trainer_check(from, impl(dst)->kind, "wvn_trainer_copy_confidence"));
  return trainer_conf_copy(&impl(dst)->conf, &from->conf, S(stream));
}

int wvn_comm_unique_id(void* id128) { return comm_unique_id(id128); }

int wvn_trainer_init_comm(wvn_trainer_t* t, const void* id128, int rank, int world) {
  WVN_REQUIRE(t, "wvn_trainer_init_comm: null trainer");
  return trainer_comm_init(&impl(t)->comm, id128, rank, world);
}

double* wvn_trainer_stats(wvn_trainer_t* t, int* n_doubles) {
  if (n_doubles) *n_doubles = t ? impl(t)->n_stats : 0;
  return t ? impl(t)->stats : nullptr;
}

// -------------------------------------------------------------------------------- fused train step
size_t wvn_mlp_trainer_scalars_bytes(void) { return sizeof(FusedScalars); }

int wvn_mlp_trainer_create(int dim, int h1, int h2, int max_rows, const wvn_train_config* cfg, void* scalars, float* grads,
                           wvn_trainer_t** out) {
  WVN_REQUIRE(cfg && out, "wvn_mlp_trainer_create: null argument");
  WVN_PROPAGATE(wvn_check_device());
  Trainer* t = nullptr;
  WVN_PROPAGATE(fused_trainer_create(shape_of(dim, h1, h2), max_rows, loss_of(cfg), adam_of(cfg), scalars, grads, &t));
  *out = handle_of(t);
  return WVN_OK;
}

int wvn_mlp_train_step(wvn_trainer_t* t, float* params, float* exp_avg, float* exp_avg_sq, long long* step_counter,
                       const float* x, int groups, int rows_per_group, const int* n_rows, const float* y,
                       const unsigned char* y_valid, float* cg_mean, float* cg_std, float* confidence_out,
                       float* metrics_out, int phase_mask, void* stream) {
  return fused_train_step(impl(t), params, exp_avg, exp_avg_sq, step_counter, x, groups, rows_per_group, n_rows, y,
                          y_valid, cg_mean, cg_std, confidence_out, metrics_out, phase_mask, S(stream));
}

}  // extern "C"

// ============================================================================================
// DoubleMLP learner: fp32 row forward and online train step (double_mlp_train.cu)
// ============================================================================================
extern "C" {

size_t wvn_double_mlp_param_count(int dim, int h1, int h2) { return double_mlp_param_count(shape_of(dim, h1, h2)); }

int wvn_double_mlp_forward_f32(int dim, int h1, int h2, const float* params, const float* x, int rows, float* a1_buf,
                               float* a2_buf, float* out, void* stream) {
  return double_mlp_forward_f32(shape_of(dim, h1, h2), params, x, rows, a1_buf, a2_buf, out, S(stream));
}

int wvn_double_mlp_trainer_create(int dim, int h1, int h2, int max_rows, const wvn_train_config* cfg, float* grads,
                                  wvn_trainer_t** out) {
  WVN_REQUIRE(cfg && out, "wvn_double_mlp_trainer_create: null argument");
  WVN_PROPAGATE(wvn_check_device());
  Trainer* t = nullptr;
  WVN_PROPAGATE(double_trainer_create(shape_of(dim, h1, h2), max_rows, loss_of(cfg), adam_of(cfg), grads, &t));
  *out = handle_of(t);
  return WVN_OK;
}

int wvn_double_mlp_train_step_padded(wvn_trainer_t* t, float* params, float* exp_avg, float* exp_avg_sq,
                                     long long* step_counter, const float* x, int groups, int rows_per_group,
                                     const int* n_rows, const float* y, const unsigned char* y_valid, float* cg_mean,
                                     float* cg_std, float* confidence_out, float* metrics_out, int phase_mask,
                                     void* stream) {
  return double_train_step_padded(impl(t), params, exp_avg, exp_avg_sq, step_counter, x, groups, rows_per_group, n_rows,
                                  y, y_valid, cg_mean, cg_std, confidence_out, metrics_out, phase_mask, S(stream));
}

}  // extern "C"

// ============================================================================================
// SimpleGCN learner: graph build, row forward and online train step (gcn_train.cu)
// ============================================================================================
extern "C" {

size_t wvn_gcn_param_count(int dim, int h1, int h2) { return gcn_param_count(shape_of(dim, h1, h2)); }

int wvn_gcn_trainer_create(int dim, int h1, int h2, int max_rows, int max_edges, const wvn_train_config* cfg,
                           float* grads, wvn_trainer_t** out) {
  WVN_REQUIRE(cfg && out, "wvn_gcn_trainer_create: null argument");
  WVN_PROPAGATE(wvn_check_device());
  Trainer* t = nullptr;
  WVN_PROPAGATE(gcn_trainer_create(shape_of(dim, h1, h2), max_rows, max_edges, loss_of(cfg), adam_of(cfg), grads, &t));
  *out = handle_of(t);
  return WVN_OK;
}

int wvn_gcn_train_step_padded(wvn_trainer_t* t, float* params, float* exp_avg, float* exp_avg_sq,
                              long long* step_counter, const float* x, int groups, int rows_per_group,
                              const int* n_rows, const long long* edges, int edges_per_group, const int* n_edges,
                              const float* y, const unsigned char* y_valid, float* cg_mean, float* cg_std,
                              float* confidence_out, float* metrics_out, int phase_mask, void* stream) {
  return gcn_train_step_padded(impl(t), params, exp_avg, exp_avg_sq, step_counter, x, groups, rows_per_group, n_rows,
                               edges, edges_per_group, n_edges, y, y_valid, cg_mean, cg_std, confidence_out,
                               metrics_out, phase_mask, S(stream));
}

int wvn_gcn_infer_rows(wvn_trainer_t* t, const float* params, const float* x, int groups, int rows_per_group,
                       const int* n_rows, const long long* edges, int edges_per_group, const int* n_edges,
                       const float* cg_mean, const float* cg_std, float std_factor, float* out, float* trav,
                       float* confidence, void* stream) {
  return gcn_infer_rows(impl(t), params, x, groups, rows_per_group, n_rows, edges, edges_per_group, n_edges, cg_mean,
                        cg_std, std_factor, out, trav, confidence, S(stream));
}

}  // extern "C"

// ============================================================================================
// LinearRnvp flow: fp32 row forward and online train step (flow_train.cu)
// ============================================================================================
// inference only: the fp32 row forward (forward workspaces only) and the per-pixel wgmma path
struct wvn_flow_infer {
  Trainer* rows = nullptr;
  FlowPixels* pix = nullptr;
};

namespace {
FlowBuffers buffers_of(const wvn_flow_buffers* b) {
  FlowBuffers f;
  if (b) {
    f.mask0 = b->mask0; f.mask1 = b->mask1; f.p1 = b->p1; f.invp1 = b->invp1; f.p3 = b->p3; f.invp3 = b->invp3;
  }
  return f;
}
}  // namespace

extern "C" {

size_t wvn_flow_param_count(int dim, int hidden) {
  FlowShape s;
  s.dim = dim; s.hidden = hidden;
  return flow_param_count(s);
}

int wvn_flow_trainer_create(int dim, int hidden, int max_rows, const wvn_train_config* cfg, float* grads,
                            wvn_trainer_t** out) {
  WVN_REQUIRE(cfg && out, "wvn_flow_trainer_create: null argument");
  WVN_PROPAGATE(wvn_check_device());
  FlowShape s;
  s.dim = dim; s.hidden = hidden;
  Trainer* t = nullptr;
  WVN_PROPAGATE(flow_trainer_create(s, max_rows, cfg->std_factor, adam_of(cfg), grads, false, &t));
  *out = handle_of(t);
  return WVN_OK;
}

int wvn_flow_train_step(wvn_trainer_t* t, float* params, float* exp_avg, float* exp_avg_sq, long long* step_counter,
                        const wvn_flow_buffers* buffers, const float* x, int rows, const unsigned char* y_valid,
                        float* cg_mean, float* cg_std, float* confidence_out, float* metrics_out, int phase_mask,
                        void* stream) {
  WVN_REQUIRE(buffers, "wvn_flow_train_step: null argument");
  return flow_train_step(impl(t), params, exp_avg, exp_avg_sq, step_counter, buffers_of(buffers), x, rows, y_valid,
                         cg_mean, cg_std, confidence_out, metrics_out, phase_mask, S(stream));
}

int wvn_flow_train_step_padded(wvn_trainer_t* t, float* params, float* exp_avg, float* exp_avg_sq,
                               long long* step_counter, const wvn_flow_buffers* buffers, const float* x, int groups,
                               int rows_per_group, const int* n_rows, const unsigned char* y_valid, float* cg_mean,
                               float* cg_std, float* confidence_out, float* metrics_out, int phase_mask, void* stream) {
  WVN_REQUIRE(buffers, "wvn_flow_train_step_padded: null argument");
  return flow_train_step_padded(impl(t), params, exp_avg, exp_avg_sq, step_counter, buffers_of(buffers), x, groups,
                                rows_per_group, n_rows, y_valid, cg_mean, cg_std, confidence_out, metrics_out,
                                phase_mask, S(stream));
}

int wvn_flow_infer_create(int dim, int hidden, int max_rows, int chunk_pixels, wvn_flow_infer_t** out) {
  WVN_REQUIRE(out && max_rows > 0, "wvn_flow_infer_create: bad arguments");
  WVN_PROPAGATE(wvn_check_device());
  FlowShape s;
  s.dim = dim; s.hidden = hidden;
  wvn_flow_infer* h = new wvn_flow_infer();
  int rc = flow_trainer_create(s, max_rows, 0.5f, AdamCfg(), nullptr, true, &h->rows);
  if (rc == WVN_OK) rc = flow_pixels_create(s, chunk_pixels, &h->pix);
  if (rc != WVN_OK) {
    wvn_flow_infer_destroy(h);
    return rc;
  }
  *out = h;
  return WVN_OK;
}

void wvn_flow_infer_destroy(wvn_flow_infer_t* h) {
  if (!h) return;
  delete h->rows;
  flow_pixels_destroy(h->pix);
  delete h;
}

int wvn_flow_infer_set_params(wvn_flow_infer_t* h, const float* params, void* stream) {
  WVN_REQUIRE(h, "wvn_flow_infer_set_params: null handle");
  return flow_pixels_set_params(h->pix, params, S(stream));
}

int wvn_flow_infer_rows(wvn_flow_infer_t* h, const float* params, const wvn_flow_buffers* buffers, const float* x, int rows,
                        float* z, float* log_det, float* logprob, const float* cg_mean, const float* cg_std,
                        float std_factor, float* trav, void* stream) {
  WVN_REQUIRE(h && buffers, "wvn_flow_infer_rows: null argument");
  return flow_forward_rows(h->rows, params, buffers_of(buffers), x, rows, z, log_det, logprob, cg_mean, cg_std,
                           std_factor, trav, S(stream));
}

int wvn_flow_infer_rows_padded(wvn_flow_infer_t* h, const float* params, const wvn_flow_buffers* buffers, const float* x,
                               int groups, int rows_per_group, const int* n_rows, const float* cg_mean,
                               const float* cg_std, float std_factor, float* trav, void* stream) {
  WVN_REQUIRE(h && buffers, "wvn_flow_infer_rows_padded: null argument");
  return flow_forward_rows_padded(h->rows, params, buffers_of(buffers), x, groups, rows_per_group, n_rows, cg_mean,
                                  cg_std, std_factor, trav, S(stream));
}

int wvn_flow_infer_pixels(wvn_flow_infer_t* h, const wvn_flow_buffers* buffers, const float* tokens, int batch, int gh,
                          int gw, int out_h, int out_w, const float* cg_mean, const float* cg_std, float std_factor,
                          float* trav, float* nll, void* stream) {
  WVN_REQUIRE(h && buffers, "wvn_flow_infer_pixels: null argument");
  return flow_pixels_run(h->pix, buffers_of(buffers), tokens, batch, gh, gw, out_h, out_w, cg_mean, cg_std, std_factor,
                         trav, nll, S(stream));
}

}  // extern "C"
