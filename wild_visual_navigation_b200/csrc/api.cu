// wvn-b200: the C ABI (include/wvn_b200.h) — argument checks and calls into the modules that own each handle, and
// the stateless primitives.
#include "../../include/wvn_b200.h"
#include "attention.h"
#include "conv_trunk.h"
#include "dense_crf.h"
#include "dense_kernels.h"
#include "effnet_kernels.h"
#include "double_mlp_train.h"
#include "gcn_train.h"
#include "gemm.h"
#include "host_common.h"
#include "mlp_infer.h"
#include "mlp_train.h"
#include "mission_graph.h"
#include "mlp_train_fused.h"
#include "resnet_kernels.h"
#include "segment_kernels.h"
#include "flow_train.h"
#include "footprint_kernels.h"
#include "slic_kernels.h"
#include "stego_kmeans.h"
#include "train_core.h"
#include "vit_backbone.h"
#include "vit_kernels.h"

using namespace wvn;

namespace {

inline cudaStream_t S(void* s) { return reinterpret_cast<cudaStream_t>(s); }
MlpShape shape_of(int dim, int h1, int h2) {
  MlpShape s;
  s.dim = dim; s.h1 = h1; s.h2 = h2;
  return s;
}

}  // namespace

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

// -------------------------------------------------------------------------------- ViT (vit_backbone.cu)
int wvn_vit_create(const wvn_vit_config* cfg, wvn_vit_t** out) {
  WVN_REQUIRE(cfg && out, "wvn_vit_create: null argument");
  WVN_PROPAGATE(wvn_check_device());
  return vit_create(cfg, out);
}

void wvn_vit_destroy(wvn_vit_t* h) { vit_destroy(h); }
int wvn_vit_npad(const wvn_vit_t* h) { return h ? vit_tokens(h).npad : 0; }

int wvn_vit_set_weight(wvn_vit_t* h, const char* name, const float* data, long long numel) {
  WVN_REQUIRE(h && name && data, "wvn_vit_set_weight: null argument");
  return vit_set_weight(h, name, data, numel);
}

int wvn_vit_forward(wvn_vit_t* h, const float* img, int batch, int in_h, int in_w, int resized_h, int resized_w,
                    float* tokens_out, void* stream) {
  return vit_forward_impl(h, img, false, batch, in_h, in_w, resized_h, resized_w, tokens_out, false, S(stream));
}

int wvn_vit_forward_tta(wvn_vit_t* h, const float* img, int batch, int in_h, int in_w, int resized_h, int resized_w,
                        float* tokens_out, void* stream) {
  return vit_forward_impl(h, img, false, batch, in_h, in_w, resized_h, resized_w, tokens_out, true, S(stream));
}

int wvn_vit_forward_u8(wvn_vit_t* h, const unsigned char* img_hwc, int batch, int in_h, int in_w, int resized_h,
                       int resized_w, float* tokens_out, void* stream) {
  return vit_forward_impl(h, img_hwc, true, batch, in_h, in_w, resized_h, resized_w, tokens_out, false, S(stream));
}

int wvn_vit_stego_head(wvn_vit_t* h, int batch, float* out, void* stream) {
  WVN_REQUIRE(h && out, "wvn_vit_stego_head: null argument");
  return vit_stego_head(h, batch, out, S(stream));
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

int wvn_crf_create(int size, int max_classes, int chunk, int iterations, wvn_crf_t** out) {
  WVN_REQUIRE(out, "wvn_crf_create: null argument");
  WVN_PROPAGATE(wvn_check_device());
  return crf_create(size, max_classes, chunk, iterations, out);
}

void wvn_crf_destroy(wvn_crf_t* h) { crf_destroy(h); }
size_t wvn_crf_workspace_bytes(const wvn_crf_t* h) { return crf_workspace_bytes(h); }

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
  return crf_run(h, in, labels, q_out, S(stream));
}

int wvn_crf_build(wvn_crf_t* h, const void* img, int u8_hwc, int batch, int in_h, int in_w, int resized_h, int resized_w,
                  void* stream) {
  WVN_REQUIRE(h, "wvn_crf_build: null handle");
  return crf_build(h, crf_input(img, u8_hwc, batch, in_h, in_w, resized_h, resized_w), S(stream));
}

int wvn_crf_filter(wvn_crf_t* h, int which, const float* values, int v, float* out, void* stream) {
  WVN_REQUIRE(h, "wvn_crf_filter: null handle");
  return crf_filter(h, which, values, v, out, S(stream));
}

int wvn_crf_export(wvn_crf_t* h, int which, unsigned long long* keys, int* counts, int* offsets, float* bary, int* m,
                   void* stream) {
  WVN_REQUIRE(h, "wvn_crf_export: null handle");
  return crf_export(h, which, keys, counts, offsets, bary, m, S(stream));
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

// -------------------------------------------------------------------------------- conv trunks (conv_trunk.cu)
int wvn_resnet_create(const wvn_resnet_config* cfg, wvn_resnet_t** out) {
  WVN_REQUIRE(cfg && out, "wvn_resnet_create: null argument");
  WVN_PROPAGATE(wvn_check_device());
  return resnet_create(cfg, out);
}

void wvn_resnet_destroy(wvn_resnet_t* h) { resnet_destroy(h); }
size_t wvn_resnet_workspace_bytes(const wvn_resnet_t* h) { return h ? resnet_workspace_bytes(h) : 0; }

int wvn_resnet_set_weight(wvn_resnet_t* h, const char* name, const float* data, long long numel) {
  WVN_REQUIRE(h && name && data, "wvn_resnet_set_weight: null argument");
  return resnet_set_weight(h, name, data, numel);
}

int wvn_resnet_forward(wvn_resnet_t* h, const float* img, int batch, void* const* taps, void* stream) {
  WVN_REQUIRE(h && img && taps, "wvn_resnet_forward: null argument");
  return resnet_forward(h, img, batch, taps, S(stream));
}

int wvn_effnet_create(const wvn_effnet_config* cfg, wvn_effnet_t** out) {
  WVN_REQUIRE(cfg && out, "wvn_effnet_create: null argument");
  WVN_PROPAGATE(wvn_check_device());
  return effnet_create(cfg, out);
}

void wvn_effnet_destroy(wvn_effnet_t* h) { effnet_destroy(h); }
size_t wvn_effnet_workspace_bytes(const wvn_effnet_t* h) { return h ? effnet_workspace_bytes(h) : 0; }

int wvn_effnet_set_weight(wvn_effnet_t* h, const char* name, const float* data, long long numel) {
  WVN_REQUIRE(h && name && data, "wvn_effnet_set_weight: null argument");
  return effnet_set_weight(h, name, data, numel);
}

int wvn_effnet_forward(wvn_effnet_t* h, const float* img, int batch, void* const* taps, void* stream) {
  WVN_REQUIRE(h && img && taps, "wvn_effnet_forward: null argument");
  return effnet_forward(h, img, batch, taps, S(stream));
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

// -------------------------------------------------------------------------------- MLP inference (mlp_infer.cu)
int wvn_mlp_infer_create(int dim, int h1, int h2, int chunk_rows, wvn_mlp_infer_t** out) {
  return mlp_infer_create(dim, h1, h2, chunk_rows, 0, out);
}

int wvn_mlp_infer_create_double(int dim, int h1, int h2, int chunk_rows, wvn_mlp_infer_t** out) {
  WVN_PROPAGATE(double_mlp_check_shape(shape_of(dim, h1, h2), "wvn_mlp_infer_create_double"));
  return mlp_infer_create(dim, h1, h2, chunk_rows, 1, out);
}

void wvn_mlp_infer_destroy(wvn_mlp_infer_t* h) { mlp_infer_destroy(h); }

int wvn_mlp_infer_reserve(wvn_mlp_infer_t* h, int tokens_per_frame) {
  WVN_REQUIRE(h && tokens_per_frame > 0, "wvn_mlp_infer_reserve: bad arguments");
  return mlp_infer_reserve(h, tokens_per_frame);
}

int wvn_mlp_infer_set_params(wvn_mlp_infer_t* h, const float* params, void* stream) {
  WVN_REQUIRE(h && params, "wvn_mlp_infer_set_params: null argument");
  return mlp_infer_set_params(h, params, S(stream));
}

int wvn_mlp_infer_pixels_vit(wvn_mlp_infer_t* h, wvn_vit_t* vit, int batch, int out_h, int out_w, const float* cg_mean,
                             const float* cg_std, float std_factor, float* trav, float* conf, void* stream) {
  WVN_REQUIRE(h && vit && trav && conf && cg_mean && cg_std, "wvn_mlp_infer_pixels_vit: null argument");
  return mlp_infer_pixels_vit(h, vit, batch, out_h, out_w, cg_mean, cg_std, std_factor, trav, conf, S(stream));
}

int wvn_mlp_infer_pixels(wvn_mlp_infer_t* h, const float* tokens, int batch, int gh, int gw, int out_h, int out_w,
                         const float* cg_mean, const float* cg_std, float std_factor, float* trav, float* conf,
                         void* stream) {
  WVN_REQUIRE(h && tokens && trav && conf && cg_mean && cg_std, "wvn_mlp_infer_pixels: null argument");
  return mlp_infer_pixels(h, tokens, batch, gh, gw, out_h, out_w, cg_mean, cg_std, std_factor, trav, conf, S(stream));
}

int wvn_mlp_infer_rows(wvn_mlp_infer_t* h, const float* x, long long rows, const float* cg_mean, const float* cg_std,
                       float std_factor, float* trav, float* conf, void* stream) {
  WVN_REQUIRE(h && x && trav && conf && cg_mean && cg_std, "wvn_mlp_infer_rows: null argument");
  return mlp_infer_rows(h, x, rows, cg_mean, cg_std, std_factor, trav, conf, S(stream));
}

int wvn_mlp_infer_rows_padded(wvn_mlp_infer_t* h, const float* x, int groups, int rows_per_group, const int* n_rows,
                              const float* cg_mean, const float* cg_std, float std_factor, float* trav, float* conf,
                              void* stream) {
  WVN_REQUIRE(h && x && n_rows && trav && conf && cg_mean && cg_std, "wvn_mlp_infer_rows_padded: null argument");
  return mlp_infer_rows_padded(h, x, groups, rows_per_group, n_rows, cg_mean, cg_std, std_factor, trav, conf,
                               S(stream));
}

// -------------------------------------------------------------------------------- training
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
// LinearRnvp flow: fp32 row forward, online train step and the inference handle (flow_train.cu)
// ============================================================================================
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
  return flow_infer_create(s, max_rows, chunk_pixels, out);
}

void wvn_flow_infer_destroy(wvn_flow_infer_t* h) { flow_infer_destroy(h); }

int wvn_flow_infer_set_params(wvn_flow_infer_t* h, const float* params, void* stream) {
  WVN_REQUIRE(h, "wvn_flow_infer_set_params: null handle");
  return flow_infer_set_params(h, params, S(stream));
}

int wvn_flow_infer_rows(wvn_flow_infer_t* h, const float* params, const wvn_flow_buffers* buffers, const float* x, int rows,
                        float* z, float* log_det, float* logprob, const float* cg_mean, const float* cg_std,
                        float std_factor, float* trav, void* stream) {
  WVN_REQUIRE(h && buffers, "wvn_flow_infer_rows: null argument");
  return flow_forward_rows(flow_infer_trainer(h), params, buffers_of(buffers), x, rows, z, log_det, logprob, cg_mean,
                           cg_std, std_factor, trav, S(stream));
}

int wvn_flow_infer_rows_padded(wvn_flow_infer_t* h, const float* params, const wvn_flow_buffers* buffers, const float* x,
                               int groups, int rows_per_group, const int* n_rows, const float* cg_mean,
                               const float* cg_std, float std_factor, float* trav, void* stream) {
  WVN_REQUIRE(h && buffers, "wvn_flow_infer_rows_padded: null argument");
  return flow_forward_rows_padded(flow_infer_trainer(h), params, buffers_of(buffers), x, groups, rows_per_group, n_rows,
                                  cg_mean, cg_std, std_factor, trav, S(stream));
}

int wvn_flow_infer_pixels(wvn_flow_infer_t* h, const wvn_flow_buffers* buffers, const float* tokens, int batch, int gh,
                          int gw, int out_h, int out_w, const float* cg_mean, const float* cg_std, float std_factor,
                          float* trav, float* nll, void* stream) {
  WVN_REQUIRE(h && buffers, "wvn_flow_infer_pixels: null argument");
  return flow_infer_pixels(h, buffers_of(buffers), tokens, batch, gh, gw, out_h, out_w, cg_mean, cg_std, std_factor,
                           trav, nll, S(stream));
}

}  // extern "C"
