/* wvn-b200 — C ABI of libwvn_b200.so
 *
 * H100-native (sm_90a) implementation of the Wild Visual Navigation per-frame hot path:
 * DINO ViT forward -> STEGO segmentation head / per-segment feature gather -> traversability
 * MLP (per-pixel inference with confidence, and the online train step).
 *
 * The reference (leggedrobotics/wild_visual_navigation @ 8b9caf9) is pure Python and has no
 * FFI for this path (SURVEY.md §8b): its boundary is the Python class surface
 * (FeatureExtractor / DinoInterface / StegoInterface / SegmentExtractor / SimpleMLP /
 * TraversabilityLoss / ConfidenceGenerator / TraversabilityEstimator).  The entry points
 * below are what a ctypes binding inside those classes calls; each cites the reference
 * code it replaces (paths relative to the reference repository root).  INTEGRATION.md shows
 * the reference-side stub.
 *
 * Conventions
 *  - every pointer is a DEVICE pointer unless named host_*; tensors are dense, row-major;
 *  - `stream` is a cudaStream_t passed as void* (0 = legacy default stream);
 *  - functions return 0 on success, a negative wvn_status otherwise; wvn_last_error() gives
 *    the message for the calling thread;
 *  - no ownership transfer; handles own their weights and workspaces (allocated at create,
 *    nothing is allocated on the per-frame path);
 *  - a handle must not be used from two host threads at once (the reference serialises
 *    frames through its Scheduler and training through `_learning_lock`).
 */
#ifndef WVN_B200_H_
#define WVN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  WVN_STATUS_OK = 0,
  WVN_STATUS_INVALID = -1,   /* bad argument / unsupported shape */
  WVN_STATUS_CUDA = -2,      /* CUDA error, see wvn_last_error() */
  WVN_STATUS_NO_DEVICE = -3, /* no sm_90 device visible */
  WVN_STATUS_STATE = -4      /* handle not ready (e.g. a weight was never set) */
} wvn_status;

const char* wvn_last_error(void);
/* 0 if device 0..n has compute capability 9.0, WVN_STATUS_NO_DEVICE otherwise. */
int wvn_check_device(void);
/* ABI version.  101: wvn_vit_config and wvn_gemm_ex_args gained a trailing `int registers` (0 = the layout of 100), so
 * callers that fill these structs by layout (ctypes mirrors, code compiled against an older header) must add the field.
 * 102: adds wvn_mlp_trainer_copy_confidence; no layout change.
 * 103: wvn_gemm_ex_args gained trailing `residual` / `ldr` (epi 6); adds the ResNet handle, the im2col / max-pool
 * primitives and wvn_segment_pool_pyramid.
 * 104: adds the LinearRnvp flow handles, their functions wvn_flow_* and the struct wvn_flow_buffers; no layout change.
 * 106: adds the padded, phased and data-parallel DoubleMLP and flow steps (wvn_double_mlp_train_step_padded,
 * wvn_double_mlp_trainer_init_comm, wvn_double_mlp_trainer_stats, wvn_flow_train_step_padded, wvn_flow_init_comm,
 * wvn_flow_stats); no layout change.
 * 107: adds wvn_mission_propagate and wvn_mission_propagate_workspace_bytes (the mission graph's label propagation);
 * no layout change.  The SimpleGCN learner's functions (wvn_gcn_*) were added later under the same version number:
 * they add symbols only.  A caller that binds every declared symbol at load (the Python package does) needs a library
 * that exports them.
 * 108: the four learners' trainers share one handle type, wvn_trainer_t, and five entry points (wvn_trainer_destroy,
 * wvn_trainer_set_confidence, wvn_trainer_copy_confidence, wvn_trainer_init_comm, wvn_trainer_stats) in place of
 * each learner's own; wvn_flow_create is renamed wvn_flow_trainer_create and wvn_double_mlp_train_step is removed (its
 * padded form with one group is the same step).  A learner's entry point refuses another learner's handle.
 * Later additions under 108 add symbols only: the dense CRF (wvn_crf_*), the EfficientNet-B0 handle (wvn_effnet_*)
 * with its primitives, GEMM activation 3 (SiLU), wvn_segment_pool_levels, and the segment-wise inference entries
 * wvn_segment_maps, wvn_mlp_infer_rows_padded and wvn_flow_infer_rows_padded, and the ViT primitives
 * wvn_image_to_patches, wvn_init_token_rows, wvn_layernorm_ex and wvn_attention_f32_debug. */
int wvn_version(void);
/* Number of kernel launches this library has issued in this process (bench.py's gpu_launches). */
long long wvn_launch_count(void);
/* Optional CUDA-event timing of the dominant kernels inside real steps (bench.py roofline):
 * category 0 = fused attention, 1 = wgmma GEMMs; category_mask bit c enables category c (0 = off, 1 = the
 * roofline kernel only — 24 event pairs per step —, 3 = attention + the ~280 GEMM launches per step).
 * collect() synchronises and writes the summed milliseconds / launch counts per category into HOST arrays of
 * length 2 and clears the records. */
void wvn_profile_enable(int category_mask);
int wvn_profile_collect(float* host_ms, long long* host_launches);

/* ------------------------------------------------------------------------------------------
 * Primitive: bf16 tensor-core GEMM  C = A[M,K] * W[N,K]^T  (wgmma, fp32 accumulate)
 * Replaces every nn.Linear / 1x1-conv call of the path (cuBLAS in the reference).
 * out_kind: 0 = bf16 out[M,ldo] = act(acc + bias); 1 = fp32 out = acc + bias;
 *           2 = fp32 out += acc + bias (residual).   act: 0 none, 1 ReLU, 2 GELU(erf), 3 SiLU (out_kind 0 only).
 * Any K >= 1: lda >= K and a multiple of 8, and W's rows are round_up(K, 8) elements apart (== K whenever K % 8 == 0);
 * columns past K of either operand are never read (the last 64-wide k-block is zero-filled past K).
 * N % block_n == 0, block_n in {0 (auto), 64, 128, 192, 224, 256}.
 * ---------------------------------------------------------------------------------------- */
int wvn_gemm_bf16(const void* a_bf16, long long lda, const void* w_bf16, const float* bias, void* out, long long ldo,
                  int m, int n, int k, int out_kind, int act, int block_n, void* stream);

/* Testing and diagnostics entry: runs the same GEMM with any of its fused epilogues, including the three the
 * handles use internally (patch-embed scatter, Q / K / V^T scatter, traversability-MLP head), so that each can be
 * checked on its own.  The fields mirror the library's internal GEMM arguments; the shape and geometry checks are the
 * GEMM's own.  epi: 0 = bf16 out[m,ldo] = act(acc + bias); 1 = fp32 out = acc + bias; 2 = fp32 out += acc + bias;
 *   3 = patch embed: fp32 out[frame*npad + 1 + registers + tok, :] = acc + bias + pos[1 + tok, :] (frame = row / tokens_in;
 *       rows [frame*npad, frame*npad + 1 + registers) — CLS and register tokens — are not written);
 *   4 = QKV: bf16 q_out, k_out [m/npad*heads, npad, 64] and vt_out [m/npad*heads, 64, npad] from the columns of [q | k | v];
 *   5 = MLP head: columns [0, feat) reconstruct x -> loss_reco = mean((out - x)^2) -> conf, column trav_col ->
 *       trav = sigmoid; nothing of [m, n] is stored;
 *   6 = residual: bf16 out[m,ldo] = act(acc + bias + residual[m,ldr]) (residual bf16, ldr even and >= n; act 0 or 1).
 * reverse_m = 1 walks the 64-row blocks last-to-first (the result must not change). */
typedef struct {
  int m, n, k;
  int epi, act;
  int block_n;              /* 0 = auto */
  const void* a;            /* [m, lda] bf16 */
  long long lda;
  const void* w;            /* [n, k] bf16, rows round_up(k, 8) elements apart (any k >= 1, see wvn_gemm_bf16) */
  const float* bias;        /* [n] or NULL */
  void* out;                /* epi 0-3 */
  long long ldo;
  const float* pos;         /* epi 3: [1 + tokens_in, ldo] */
  int tokens_in, npad;      /* epi 3 (npad also epi 4) */
  int dim, heads;           /* epi 4 */
  void* q_out;
  void* k_out;
  void* vt_out;
  int feat, trav_col;       /* epi 5 */
  const void* x;            /* [m, ldx] bf16 */
  long long ldx;
  float* trav;
  float* conf;
  float* loss_reco;         /* or NULL */
  const float* cg_mean;     /* device scalars */
  const float* cg_std;
  float cg_std_factor;
  int reverse_m;
  int registers;            /* epi 3: register tokens between CLS and the first patch row (0 = DINO / DINOv2 layout) */
  const void* residual;     /* epi 6: [m, ldr] bf16 */
  long long ldr;
} wvn_gemm_ex_args;
int wvn_gemm_bf16_ex(const wvn_gemm_ex_args* args, void* stream);

/* ------------------------------------------------------------------------------------------
 * Primitive: fused multi-head attention, head dim 64, non-causal.
 * Replaces `softmax(q @ k.transpose(-2,-1) * scale) @ v` of the DINO ViT block
 * ([EXTERNAL] stego/backbones/dino/vision_transformer.py Attention.forward; SURVEY.md §8 a3).
 * q,k: [batch*heads, npad, 64] bf16; vt: [batch*heads, 64, npad] bf16;
 * out: [batch, npad, heads*64] bf16.  Keys >= n_valid are masked.  npad % 128 == 0.
 * ---------------------------------------------------------------------------------------- */
int wvn_attention_bf16(const void* q, const void* k, const void* vt, void* out, int batch, int heads, int npad,
                       int n_valid, float scale, void* stream);

/* LayerNorm over fp32 rows -> bf16 rows; dim in {384, 768}.  The same as wvn_layernorm_ex without an fp32 output. */
int wvn_layernorm(const float* x, const float* gamma, const float* beta, void* out_bf16, long long rows, int dim,
                  float eps, void* stream);

/* ------------------------------------------------------------------------------------------
 * ViT primitives, exposed for testing: the memory-bound kernels the ViT handle runs around its GEMMs and attention.
 * ---------------------------------------------------------------------------------------- */
/* The patch loader: img [src_frames, 3, in_h, in_w] fp32 in [0, 1], or (u8_hwc = 1) [src_frames, in_h, in_w, 3]
 * uint8 RGB (px = u8 / 255), NEAREST-resized to resized_h x resized_w (torch 'nearest', fp32 scale in / resized),
 * center-cropped to image_size (offset int(round((resized - image_size) / 2)), half to even), ImageNet-normalised
 * ((px - mean) * (1 / std) in fp32) and cut into g = image_size / patch patches per side (conv-floor semantics).
 * out_bf16 [batch * g * g, pitch] bf16, pitch = round_up(3 * patch * patch, 8), row (f, py, px) in (c, ky, kx) order;
 * columns [3 * patch * patch, pitch) are never written.  Output frame f reads source frame (frame0 + f) % src_frames;
 * frames with frame0 + f >= flip_from are the horizontal flip of the whole image_size-wide crop.  patch in {8, 14, 16};
 * the same derivation of crop, scales and frames as wvn_vit_forward / wvn_vit_forward_tta / wvn_vit_forward_u8. */
int wvn_image_to_patches(const void* img, int u8_hwc, int batch, int in_h, int in_w, int resized_h, int resized_w,
                         int image_size, int patch, int frame0, int src_frames, int flip_from, void* out_bf16,
                         void* stream);
/* x [batch, npad, dim] fp32, per frame: row 0 = cls + pos[0, :], rows [1, 1 + registers) = reg (no position
 * embedding), rows [n_valid, npad) = 0; every other row is left as it is.  cls [dim], pos [>= 1, dim],
 * reg [registers, dim] (NULL when registers == 0). */
int wvn_init_token_rows(float* x, const float* cls, const float* pos, const float* reg, int registers, int batch, int npad,
                        int n_valid, int dim, void* stream);
/* LayerNorm(dim, eps) of fp32 rows x [rows, dim] (biased variance, eps inside the square root), dim in {384, 768}:
 * out_bf16 [rows, dim] bf16 (or NULL) and out_f32 (or NULL) fp32, which receives only rows [row0, n_valid) of each
 * npad-row frame, compacted: frame f's row t lands at f * (n_valid - row0) + t - row0 (rows % npad == 0).
 * reverse = 1 walks the rows last-to-first; the result does not change. */
int wvn_layernorm_ex(const float* x, const float* gamma, const float* beta, void* out_bf16, float* out_f32,
                     long long rows, int dim, float eps, int npad, int n_valid, int row0, int reverse, void* stream);
/* The parity-debug attention of $WVN_VIT_PRECISE=1: fp32 qkv [batch * npad, 3 * dim] (columns [q | k | v], head h at
 * columns h * 64 of each) -> out_bf16 [batch * npad, dim] = softmax(q k^T * scale) v over keys [0, n_valid), in fp32
 * CUDA-core arithmetic; every row of [0, npad) is written.  dim = heads * 64. */
int wvn_attention_f32_debug(const float* qkv, void* out_bf16, int batch, int heads, int npad, int n_valid, int dim,
                            float scale, void* stream);

/* ------------------------------------------------------------------------------------------
 * ViT backbone handle — replaces DinoInterface.__init__/inference's backbone
 * (wild_visual_navigation/feature_extractor/dino_interface.py:16-59, :70-92 and the
 *  [EXTERNAL] stego.backbones.backbone.get_backbone -> DINO VisionTransformer).
 * ---------------------------------------------------------------------------------------- */
typedef struct wvn_vit wvn_vit_t;

typedef struct {
  int image_size;   /* side of the (square) network input after resize + center crop, e.g. 448 */
  int patch_size;   /* 8 or 16 (DINO), 14 (DINOv2) */
  int dim;          /* 384 (vit_small) or 768 (vit_base) */
  int depth;        /* 12 */
  int heads;        /* dim / 64 */
  int mlp_dim;      /* 4 * dim */
  int max_batch;    /* largest batch a single forward call may carry */
  int chunk;        /* frames processed together (activations stay L2-resident); 0 = default */
  float ln_eps;     /* 1e-6 */
  int head_out;     /* columns of the STEGO head output matrix (multiple of 64), 0 = no head */
  int registers;    /* register tokens R (DINOv2 *_reg: 4), 0 = none.  Token rows of a frame: [CLS, reg_0 .. reg_{R-1},
                       patch_0 ..], so patch p sits in row 1 + R + p and n_valid = 1 + R + P.  R > 0 needs head_out == 0
                       (the STEGO consumers below address patch p as row 1 + p). */
} wvn_vit_config;

int wvn_vit_create(const wvn_vit_config* cfg, wvn_vit_t** out);
void wvn_vit_destroy(wvn_vit_t* h);

/* Weights use the DINO state-dict names (fp32, host or device memory):
 *   cls_token [dim], pos_embed [(1+P), dim] (CLS + patches, already interpolated to this token grid),
 *   register_tokens [registers, dim] (only when registers > 0; they get no position embedding),
 *   patch_embed.proj.weight [dim, 3*p*p] (the Conv2d weight as given; the library keeps it at its own padded pitch),
 *   patch_embed.proj.bias [dim],
 *   blocks.{i}.norm1.{weight,bias}, blocks.{i}.attn.qkv.{weight [3dim,dim],bias},
 *   blocks.{i}.attn.proj.{weight,bias}, blocks.{i}.norm2.{weight,bias},
 *   blocks.{i}.mlp.fc1.{weight [mlp,dim],bias}, blocks.{i}.mlp.fc2.{weight [dim,mlp],bias},
 *   norm.{weight,bias}
 * and for the STEGO head (see wvn_vit_stego_head):
 *   stego.head_a.weight [head_out, dim], stego.head_a.bias [head_out],
 *   stego.hidden.weight [dim, dim], stego.hidden.bias [dim], stego.head_b.weight [head_out, dim]. */
int wvn_vit_set_weight(wvn_vit_t* h, const char* name, const float* data, long long numel);

/* img: [batch, 3, in_h, in_w] fp32 in [0,1].  Applies the interface's transform
 * (Resize(image_size, NEAREST) + CenterCrop(image_size) + ImageNet Normalize,
 *  dino_interface.py:52-59) inside the patch loader, runs the backbone, and writes the final
 * LayerNorm output of the patch tokens (CLS and register tokens dropped): tokens_out [batch, P, dim] fp32.
 * resized_h/resized_w: size after the virtual NEAREST resize (== in_h/in_w when no resize). */
int wvn_vit_forward(wvn_vit_t* h, const float* img, int batch, int in_h, int in_w, int resized_h, int resized_w,
                    float* tokens_out, void* stream);

/* Flip test-time augmentation of STEGO ([EXTERNAL] Stego.get_code, called at stego_interface.py:91): the `batch`
 * frames are run twice, the second time on the horizontal flip of the TRANSFORMED (resized + cropped + normalised)
 * image; tokens_out [2*batch, P, dim] (second half = flipped pass) and the activation layout hold 2*batch frames,
 * so 2*batch <= max_batch. */
int wvn_vit_forward_tta(wvn_vit_t* h, const float* img, int batch, int in_h, int in_w, int resized_h, int resized_w,
                        float* tokens_out, void* stream);

/* Same as wvn_vit_forward, from the camera frame itself: img_hwc [batch, in_h, in_w, 3] uint8 RGB.  Folds into the patch loader the
 * two steps that precede the interface in the reference's node (SURVEY.md §8f rank 1):
 *   ros_image_to_torch  — torchvision ToTensor: HWC uint8 -> CHW float / 255   (ros_converter.py:113-126)
 *   ImageProjector.resize_image — Resize(h, NEAREST) + CenterCrop(h)            (image_projector.py:55-59,199-200)
 * followed by the interface's own transform as in wvn_vit_forward; with network_input_image_height == image_size
 * (the shipped configuration) the two NEAREST resizes are one, expressed by resized_h / resized_w. */
int wvn_vit_forward_u8(wvn_vit_t* h, const unsigned char* img_hwc, int batch, int in_h, int in_w, int resized_h,
                       int resized_w, float* tokens_out, void* stream);

/* STEGO segmentation head on the tokens of the last forward
 * (stego_interface.py:91-100; [EXTERNAL] stego.stego.Stego.forward / cluster & linear probes):
 *   out[row, :] = head_a(t) + head_b(relu(hidden(t)))           out: [batch*npad, head_out] fp32
 * where the caller stacks code / cluster-probe / linear-probe rows into head_a / head_b.
 * Row b*npad + 1 + p holds patch p of frame b (row b*npad is the CLS token). */
int wvn_vit_stego_head(wvn_vit_t* h, int batch, float* out, void* stream);
int wvn_vit_npad(const wvn_vit_t* h);

/* ------------------------------------------------------------------------------------------
 * ResNet backbone handle — replaces TorchVisionInterface's model (wild_visual_navigation/feature_extractor/
 * torchvision_interface.py:22-101: torchvision resnet18 / resnet50 behind create_feature_extractor).
 * Activations are NHWC bf16 with fp32 accumulation; every conv is one wgmma GEMM over its output pixels (1 x 1 /
 * stride 1 convs straight on the activation rows, the others after an im2col pass whose rows are round_up(K, 8)
 * elements apart), with bias, residual and ReLU in the GEMM's epilogue.
 * ---------------------------------------------------------------------------------------- */
typedef struct wvn_resnet wvn_resnet_t;

typedef struct {
  int image_size;   /* side of the square input, a multiple of 32 (e.g. 448) */
  int depth;        /* 18 (BasicBlock [2,2,2,2]) or 50 (Bottleneck [3,4,6,3]) */
  int max_batch;    /* largest batch a forward call may carry; the workspaces are sized for it at create */
} wvn_resnet_config;

int wvn_resnet_create(const wvn_resnet_config* cfg, wvn_resnet_t** out);
void wvn_resnet_destroy(wvn_resnet_t* h);
/* Bytes of activation and im2col workspace the handle allocated at create. */
size_t wvn_resnet_workspace_bytes(const wvn_resnet_t* h);
/* Weights use the torchvision state-dict names of the convolutions, with eval-mode batch norm already folded in
 * (w * gamma / sqrt(var + eps) per output channel, bias = beta - mean * gamma / sqrt(var + eps)), fp32, host or device:
 *   conv1.{weight,bias}, layer{L}.{B}.conv{1,2[,3]}.{weight,bias}, layer{L}.0.downsample.{weight,bias}
 * (the downsample conv + its batch norm, where the block has one).  A weight is given in (out, ky, kx, in) order —
 * torch's [out, in, ky, kx] tensor permuted to (0, 2, 3, 1) — and a bias has `out` elements. */
int wvn_resnet_set_weight(wvn_resnet_t* h, const char* name, const float* data, long long numel);
/* img: [batch, 3, image_size, image_size] fp32 in [0, 1]; ImageNet Normalize is applied in the stem's loader, before
 * the zero padding.  taps: host array of four device pointers, each an NHWC bf16 map [batch, h_l, w_l, c_l]:
 *   depth 18: layer{1,2,3,4}.1.relu_1 (the stage outputs): 64 @ S/4, 128 @ S/8, 256 @ S/16, 512 @ S/32;
 *   depth 50: layer{2,3,4}.0.relu (after bn1 of each stage's first block): 128 @ S/4, 256 @ S/8, 512 @ S/16,
 *             and layer4.2.relu_2 (the trunk output): 2048 @ S/32. */
int wvn_resnet_forward(wvn_resnet_t* h, const float* img, int batch, void* const* taps, void* stream);

/* The ResNet path's primitives, exposed for testing.  im2col rows of an NHWC bf16 map [batch, h, w, c] (c % 8 == 0):
 * row (b, oy, ox) holds the k x k window at (oy * stride - pad, ox * stride - pad) in (ky, kx, channel) order, zero
 * outside the map; rows are `pitch` elements apart and columns [k*k*c, pitch) are left as they are.
 * wvn_im2col_image: the same rows (k*k*3 columns) from the fp32 NCHW image [batch, 3, h, w] after ImageNet Normalize.
 * wvn_maxpool3s2_bf16_nhwc: 3 x 3 / stride 2 / pad 1 max-pool with -inf padding, out [batch, (h+1)/2, (w+1)/2, c]. */
int wvn_im2col_bf16_nhwc(const void* in, int batch, int h, int w, int c, int k, int stride, int pad, void* out,
                         long long pitch, void* stream);
int wvn_im2col_image(const float* img, int batch, int h, int w, int k, int stride, int pad, void* out, long long pitch,
                     void* stream);
int wvn_maxpool3s2_bf16_nhwc(const void* in, int batch, int h, int w, int c, void* out, void* stream);

/* ------------------------------------------------------------------------------------------
 * EfficientNet-B0 backbone handle — replaces TorchVisionInterface's model for model_type "efficientnet_b0"
 * (torchvision efficientnet_b0 in eval mode behind create_feature_extractor).  NHWC bf16 activations at channel
 * pitches rounded up to 64 (the pad channels are zero throughout), fp32 accumulation.  The stem (3 x 3 / 2, after an
 * im2col pass of K = 27), every expand and project 1 x 1 conv and the head are wgmma GEMMs with batch norm folded in,
 * SiLU or the residual add in the epilogue; each MBConv block's depthwise conv (+ batch norm + SiLU) is a SIMT kernel
 * that also emits the squeeze-excitation's pool sums, then one kernel per frame computes the gates and one pass
 * multiplies them in.  Nothing is allocated after create and forward never synchronises with the host.
 * ---------------------------------------------------------------------------------------- */
typedef struct wvn_effnet wvn_effnet_t;

typedef struct {
  int image_size;   /* side of the square input, a multiple of 32 (e.g. 448) */
  int max_batch;    /* largest batch a forward call may carry; the workspaces are sized for it at create */
} wvn_effnet_config;

int wvn_effnet_create(const wvn_effnet_config* cfg, wvn_effnet_t** out);
void wvn_effnet_destroy(wvn_effnet_t* h);
/* Bytes of activation, im2col, pool-sum and gate workspace the handle allocated at create. */
size_t wvn_effnet_workspace_bytes(const wvn_effnet_t* h);
/* Weights are named after torchvision's modules, batch norm folded in (as for wvn_resnet_set_weight), fp32, host or
 * device, zero-padded to the channel pitches P(c) = round_up(c, 64):
 *   features.0.{weight [64, 27] (out, ky, kx, in), bias [64]}                                  the stem
 *   features.{s}.{i}.block.{j}.{weight [P(out), P(in)], bias [P(out)]}                         expand / project 1 x 1
 *   features.{s}.{i}.block.{j}.{weight [k, k, P(c)] (channel fastest), bias [P(c)]}           depthwise k x k
 *   features.{s}.{i}.block.{j}.fc1.{weight [sq, P(c)], bias [sq]}, .fc2.{weight [P(c), sq], bias [P(c)]}
 *                                                                                            squeeze-excitation
 *   features.8.{weight [1280, 320], bias [1280]}                                               the head
 * with j counted as torchvision does (stage 1 has no expand conv: its depthwise is block.0). */
int wvn_effnet_set_weight(wvn_effnet_t* h, const char* name, const float* data, long long numel);
/* img: [batch, 3, image_size, image_size] fp32 in [0, 1] (ImageNet Normalize in the stem's loader).  taps: host array
 * of five device pointers, each an NHWC bf16 map [batch, h_l, w_l, P(c_l)] (channels [c_l, P(c_l)) come out zero):
 *   features.2.0.block.0  96 @ S/2,  features.3.0.block.0 144 @ S/4,  features.4.0.block.0 240 @ S/8,
 *   features.6.0.block.0 672 @ S/16, features.8 1280 @ S/32. */
int wvn_effnet_forward(wvn_effnet_t* h, const float* img, int batch, void* const* taps, void* stream);

/* The EfficientNet path's primitives, exposed for testing.  NHWC bf16 maps at a channel pitch that is a multiple of 8.
 * wvn_depthwise_silu_bf16_nhwc: out [batch, ho, wo, pitch] = bf16(SiLU(depthwise k x k conv (k 3 or 5, stride 1 or 2,
 *   zero padding (k-1)/2) + bias)), weight [k, k, pitch] fp32, bias [pitch]; partial
 *   [batch, wvn_depthwise_pool_blocks(ho, wo), pitch] fp32 receives the per-channel sums of the bf16-ROUNDED outputs
 *   over consecutive blocks of 64 output pixels, each added in a fixed order (no atomics).
 * wvn_se_gates: gates [batch, pitch] = sigmoid(fc2(SiLU(fc1(mean)))), mean = (sum of the frame's partial rows in row
 *   order) / hw; fc1 [squeeze, pitch], fc2 [pitch, squeeze]; channels [channels, pitch) get gate 0.
 * wvn_channel_scale_bf16_nhwc: in place x[b, p, c] = bf16(x[b, p, c] * gates[b, c]), x [batch, hw, pitch]. */
int wvn_depthwise_silu_bf16_nhwc(const void* in, int batch, int h, int w, int pitch, int k, int stride,
                                 const float* weight, const float* bias, void* out, float* partial, void* stream);
int wvn_depthwise_pool_blocks(int ho, int wo);
int wvn_se_gates(const float* partial, int batch, int nblk, int hw, int channels, int pitch, const float* fc1_w,
                 const float* fc1_b, int squeeze, const float* fc2_w, const float* fc2_b, float* gates, void* stream);
int wvn_channel_scale_bf16_nhwc(void* x, int batch, long long hw, int pitch, const float* gates, void* stream);

/* ------------------------------------------------------------------------------------------
 * Token grid -> image resolution
 * ---------------------------------------------------------------------------------------- */
/* F.interpolate(features, (out,out), "bilinear", align_corners=True) (dino_interface.py:87-90).
 * tokens: [batch, gh*gw, dim] fp32 -> out: [batch, dim, out_h, out_w] fp32. */
int wvn_upsample_dense(const float* tokens, float* out, int batch, int dim, int gh, int gw, int out_h, int out_w,
                       void* stream);
/* bilinear (align_corners=False) upsampling of per-patch logits + argmax -> int64 segment ids
 * (STEGO postprocess + stego_interface.py:108-109).  logits: [batch*npad, ld] fp32.  Two logit
 * column ranges (cluster probe -> seg, linear probe -> seg_b; seg_b may be NULL) share one pass.
 * Columns are read in float4s: col0, col0_b and ld are multiples of 4 and col0 + round_up(classes, 4) <= ld (likewise
 * for the second range when it is used). */
int wvn_logits_argmax(const float* logits, long long ld, int col0, int classes, int col0_b, int classes_b, int batch,
                      int npad, int gh, int gw, int out_h, int out_w, long long* seg, long long* seg_b, void* stream);

/* Per-image k-means of the STEGO code (run_clustering=True — the reference's default for stego segmentation,
 * feature_extractor.py:47-53; [EXTERNAL] Stego.postprocess(image_clustering=True), stego_interface.py:91-100).
 * rows: the head-output matrix [batch*npad, ld] fp32 (row 0 of every frame = CLS), code in columns
 * [code_col, code_col+code_dim).  Lloyd iterations (Euclidean, `iters` fixed, evenly spaced deterministic init) over the
 * `patches` code rows of each frame; the per-patch nearest-centroid scores <x,c_k> - |c_k|^2/2 are written to columns
 * [logit_col, logit_col+k) so that wvn_logits_argmax yields the per-pixel labels of the upsampled code.
 * centroids_out: optional [batch, k, code_dim]; workspace: wvn_stego_kmeans_workspace_bytes(batch, k, code_dim) bytes of device
 * memory (partial sums of the 8 CTAs that share a frame; no initialisation needed).  One launch for all frames and iterations. */
/* STEGO's flip test-time augmentation (Stego.get_code: the code of the image and of its horizontal flip are averaged):
 * head [2*batch*npad, ld] holds the head output of the straight pass (frames [0, batch)) and of the pass over the flipped
 * transformed images (frames [batch, 2*batch), see wvn_vit_forward_tta).  In place: rows of the straight pass become
 * 0.5 * (own + mirrored row of the flipped pass); CLS / padding rows are zeroed. */
int wvn_flip_average(float* head, int batch, int npad, int grid, long long ld, void* stream);
size_t wvn_stego_kmeans_workspace_bytes(int batch, int k, int code_dim);
int wvn_stego_kmeans(float* rows, long long ld, int batch, int npad, int patches, int code_col, int code_dim, int logit_col,
                     int k, int iters, float* centroids_out, void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------
 * STEGO's dense CRF (run_crf=True; [EXTERNAL-RECALLED] stego crf.py dense_crf on pydensecrf, restated in
 * oracle/dense_crf.py): DenseCRF2D with a Gaussian (sxy 1, Potts weight 3) and a bilateral (sxy 67, srgb 3, weight 4)
 * kernel on permutohedral lattices, symmetric normalisation, `iterations` mean-field updates from
 * U = -log(clip(softmax(logits), 1e-5, 1)).  The handle owns every workspace, sized at create for the worst case of
 * `chunk` frames of size x size pixels; a run allocates nothing and never synchronises with the host.
 * ---------------------------------------------------------------------------------------- */
typedef struct wvn_crf wvn_crf_t;
/* size: side S of the transformed (square) image; max_classes in [1, 64]; chunk: frames refined together. */
int wvn_crf_create(int size, int max_classes, int chunk, int iterations, wvn_crf_t** out);
void wvn_crf_destroy(wvn_crf_t* h);
size_t wvn_crf_workspace_bytes(const wvn_crf_t* h);
/* img: the frames the patch loader read ([batch, 3, in_h, in_w] fp32 in [0, 1], or u8_hwc [batch, in_h, in_w, 3] uint8
 * RGB), resized (nearest) to resized_h x resized_w and center-cropped to S x S as in wvn_vit_forward.
 * head: the STEGO head output [batch*npad, ld] fp32 (patch p of frame b at row b*npad + 1 + p, grid x grid patches).
 * Logits: columns [col0, col0+classes) upsampled bilinearly (align_corners=False) to S x S; with code_dim > 0 they are
 * divided by the norm of the upsampled code (columns [code_col, code_col+code_dim)) and multiplied by logit_scale (the
 * cluster probe: logit_scale 2).  labels: [batch, S, S] int64 argmax of Q; q_out (optional): [batch, S*S, classes]. */
int wvn_crf_run(wvn_crf_t* h, const void* img, int u8_hwc, int batch, int in_h, int in_w, int resized_h, int resized_w,
                const float* head, long long ld, int npad, int grid, int col0, int classes, int code_col, int code_dim,
                float logit_scale, long long* labels, float* q_out, void* stream);
/* Testing.  wvn_crf_build: the two lattices (0: spatial, 1: bilateral) of frames [0, batch <= chunk).
 * wvn_crf_filter: values [batch*S*S, v] through lattice `which`, unnormalised (splat, blur, slice) -> out.
 * wvn_crf_export: vertex keys (packed as in oracle/dense_crf.py, ascending) and pixel counts, each pixel's d+1 vertex
 * indices and barycentric weights ([batch*S*S, d+1]) and the vertex count m (device int). */
int wvn_crf_build(wvn_crf_t* h, const void* img, int u8_hwc, int batch, int in_h, int in_w, int resized_h, int resized_w,
                  void* stream);
int wvn_crf_filter(wvn_crf_t* h, int which, const float* values, int v, float* out, void* stream);
int wvn_crf_export(wvn_crf_t* h, int which, unsigned long long* keys, int* counts, int* offsets, float* bary, int* m,
                   void* stream);

/* ------------------------------------------------------------------------------------------
 * Segment reductions — replace SegmentExtractor.adjacency_list / .centers
 * (feature_extractor/segment_extractor.py:40-92), FeatureExtractor.sparsify_features
 * (feature_extractor.py:389-396) and the relabel loop of segment_stego (:245-246).
 * ---------------------------------------------------------------------------------------- */
size_t wvn_segment_workspace_bytes(int batch, int smax, int gh, int gw);
/* seg: [batch, h, w] int64 with ids in [0, smax) (others ignored).
 * feat: [batch, smax, dim] fp32 or NULL (needs tokens [batch, gh*gw, dim] fp32);
 * centers: [batch, smax, 2] fp32 (x=col, y=row) or NULL;
 * edges: [batch, max_edges, 2] int64 (le, ri) sorted like torch.unique of the reference's keys,
 * n_edges: [batch] int32; both NULL to skip. */
int wvn_segment_reduce(const long long* seg, int batch, int h, int w, int smax, const float* tokens, int gh, int gw,
                       int dim, float* feat, float* centers, long long* edges, int* n_edges, int max_edges,
                       void* workspace, void* stream);
/* Multiscale segment pooling — replaces the feature-pyramid branch of FeatureExtractor.sparsify_features
 * (feature_extractor.py:314-366).  seg: [batch, h, w] int64 (ids outside [0, smax) ignored); taps: host array of four
 * device pointers to NHWC bf16 maps [batch, tap_h[l], tap_w[l], tap_c[l]] (host int arrays), each level dividing h x w;
 * centers: [batch, smax, 2] fp32 (col, row) as wvn_segment_reduce returns them.  out: [batch, smax, sum(tap_c)] fp32 —
 * per level, the mean of the level's cells whose nearest-downsampled id seg[i*h/tap_h, j*w/tap_w] is the segment;
 * a segment with no such cell takes the cell (clamp(floor(row*tap_h/h)), clamp(floor(col*tap_w/w))) under its centroid
 * (the reference raises AttributeError there); a segment without pixels gets a NaN row, as wvn_segment_reduce's feat. */
int wvn_segment_pool_pyramid(const long long* seg, int batch, int h, int w, int smax, const float* centers,
                             void* const* taps, const int* tap_h, const int* tap_w, const int* tap_c, float* out,
                             void* stream);
/* The same pooling over 1 to 5 levels whose maps are [batch, tap_h[l], tap_w[l], tap_pitch[l]] with the first tap_c[l]
 * channels pooled (tap_pitch[l] >= tap_c[l]); out [batch, smax, sum(tap_c)].  wvn_segment_pool_pyramid is this call
 * with four levels and tap_pitch = tap_c. */
int wvn_segment_pool_levels(const long long* seg, int batch, int h, int w, int smax, const float* centers, int levels,
                            void* const* taps, const int* tap_h, const int* tap_w, const int* tap_c, const int* tap_pitch,
                            float* out, void* stream);
/* Segment-wise maps — replaces the per-pixel lookup of the node's segment-wise mode
 * (wvn_feature_extractor_node.py:323-338, prediction_per_pixel False): map[b, p] = v[b, seg[b, p]] for every frame at once.
 * seg: [batch, hw] int64 (seg_is_int64 != 0) or int32; trav / conf: [batch, smax] fp32 per-segment values (conf may be
 * NULL); n_rows: [batch] int32 on the device.  trav_map / conf_map: [batch, hw] fp32 (conf_map NULL when conf is).  A
 * pixel whose id is outside [0, min(n_rows[b], smax)) gets NaN; no padding row is read. */
int wvn_segment_maps(const void* seg, int seg_is_int64, int batch, long long hw, const float* trav, const float* conf,
                     int smax, const int* n_rows, float* trav_map, float* conf_map, void* stream);
/* In-place relabel of each frame to 0..S-1; scratch: [batch*num_labels] int32; counts: [batch] int32. */
int wvn_segment_relabel(long long* seg, int batch, long long pix_per_frame, int num_labels, int* scratch, int* counts,
                        void* stream);

/* Supervision label pooling — replaces MissionNode.update_supervision_signal (traversability_estimator/nodes.py:400-440):
 *   signal = supervision_mask.nanmean(0);  per segment s: mean of signal over the segment's non-NaN pixels,
 *   nan_to_num(0);  valid = signal_mean > 0
 * without the reference's (H, W, S) one-hot expansion.  seg: [batch, h, w] int64 (ids outside [0, smax) ignored);
 * mask: [batch, channels, h, w] fp32 with NaN = unlabelled; y: [batch, smax] fp32; y_valid: [batch, smax] uint8;
 * count_ws: [batch, smax] fp32 scratch. */
int wvn_supervision_pool(const long long* seg, const float* mask, int batch, int channels, int h, int w, int smax,
                         float* y, unsigned char* y_valid, float* count_ws, void* stream);

/* SLIC superpixels — replaces fast_slic's Slic(num_components, compactness).iterate(np.uint8(img * 255)) behind
 * FeatureExtractor(segmentation_type="slic") (feature_extractor/feature_extractor.py:88-95, 221-225).  fast-slic is an
 * un-vendored C++ dependency; the algorithm is restated in all-integer form (oracle/slic.py is the definition; the labels
 * of this kernel are bit-identical to it).  img: [batch,3,h,w] fp32 in [0,1]; labels: [batch,h,w] int64 cluster ids in
 * [0, nx*ny) (empty clusters are possible: compact with wvn_segment_relabel); lut_*: device copies of the host tables
 * wvn_slic_tables() fills (256 / 9 / 4096 ints); workspace: wvn_slic_workspace_bytes(). */
void wvn_slic_tables(int* g256, int* m9, int* f4096);
int wvn_slic_geometry(int h, int w, int num_components, int* grid_interval, int* nx, int* ny);
size_t wvn_slic_workspace_bytes(int batch, int h, int w, int num_components);
int wvn_slic(const float* img, int batch, int h, int w, int num_components, float compactness, int iters,
             const int* lut_g, const int* lut_m, const int* lut_f, long long* labels, void* workspace, void* stream);

/* Footprint projection + rasterisation — replaces ImageProjector.project_and_render
 * (image_projector/image_projector.py:152-197; its kornia calls transform_points, PinholeCamera.project and
 * draw_convex_polygon are restated, see oracle/image_projector.py) and, when supervision_inout != NULL, the mask update of
 * TraversabilityEstimator.add_supervision_node (traversability_estimator/traversability_estimator.py:281-284):
 *   supervision = fmin(supervision, mask * traversability).
 * K: [batch,4,4] SCALED camera matrices (ImageProjector.__init__ :61-75); pose_camera_in_world: [batch,4,4];
 * points: [batch,n_points,3] convex polygon in the world frame; colors: [batch,3] (color_batched) or [3];
 * traversability: device scalar or NULL (= 1).  Outputs (each may be NULL): masks [batch,3,h,w] fp32 with NaN outside the
 * polygon (and where the colour is 0, as `masks[masks == 0] = nan`); projected [batch,n_points,2] pixel coordinates
 * (NaN for points behind the camera); valid [batch,n_points] uint8 (check_validity :103-124). */
int wvn_project_and_render(const float* K, const float* pose_camera_in_world, const float* points, const float* colors,
                           int color_batched, int batch, int n_points, int h, int w, const float* traversability,
                           float* masks, float* projected, unsigned char* valid, float* supervision_inout, void* stream);

/* Mission-graph label propagation — one supervision event into every in-range mission node
 * (TraversabilityEstimator.add_supervision_node, traversability_estimator.py:257-289, then each node's
 * MissionNode.update_supervision_signal, nodes.py:400-440), in one pass over each slot's h x w.  For list entry i and
 * slot s = slots[i] (distinct slots; any order, e.g. a wrapped ring range):
 *   mask[s] = fmin(restart[i] ? 0 : mask[s], render(points, K[s], pose_cam_in_world[s]) * traversability)
 *   y[s][k] = nan_to_num(mean of mask[s] over the pixels of segment k that are not NaN), y_valid[s][k] = y[s][k] > 0,
 *   slot_valid[s] = any(y_valid[s])
 * The footprint is projected and rasterised exactly as wvn_project_and_render does it (shared device code) with colour 1;
 * the mask has one channel (the reference's three are identical).  restart (nullable): per list entry, nonzero = the
 * node's mask was dropped (clear_debug_data), so the event starts it from a zero mask as the reference does.
 * slots [n_slots] int32, restart [n_slots] uint8, points [n_points,3] world frame, traversability: device scalar — all on
 * the device.  Per slot: K [cap,4,4] SCALED camera matrices, pose_cam_in_world [cap,4,4], seg [cap,h,w] int32 (ids outside
 * [0, smax) ignored), mask [cap,h,w] fp32 (NaN = unlabelled), y [cap,smax] fp32, y_valid [cap,smax] uint8, slot_valid
 * [cap] int32 (nullable).  Slots not in the list are not touched.  1 <= smax <= 4096, 1 <= n_points <= 1024.
 * workspace: wvn_mission_propagate_workspace_bytes(>= n_slots, smax) bytes that are zero before the first call; each call
 * leaves them zero again.  No allocation, no host synchronisation: everything is enqueued on `stream`. */
size_t wvn_mission_propagate_workspace_bytes(int max_slots, int smax);
int wvn_mission_propagate(const int* slots, const unsigned char* restart, int n_slots, const float* K,
                          const float* pose_cam_in_world, const float* points, int n_points, const float* traversability,
                          const int* seg, float* mask, int h, int w, int smax, float* y, unsigned char* y_valid,
                          int* slot_valid, void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------
 * Traversability MLP inference over every pixel — replaces
 *   x = dense_feat[0].permute(1,2,0).reshape(-1, D); prediction = model.forward(Data(x));
 *   out_trav = prediction[...,0]; loss_reco = mse(prediction[:,1:], x).mean(1);
 *   confidence = confidence_generator.inference_without_update(loss_reco)
 * (wild_visual_navigation_ros/scripts/wvn_feature_extractor_node.py:319-370,
 *  model/simple_mlp.py:33-39, utils/confidence_generator.py:182-193).
 * ---------------------------------------------------------------------------------------- */
typedef struct wvn_mlp_infer wvn_mlp_infer_t;
int wvn_mlp_infer_create(int dim, int h1, int h2, int chunk_rows, wvn_mlp_infer_t** out);
void wvn_mlp_infer_destroy(wvn_mlp_infer_t* h);
/* Sizes the per-pixel path's workspaces for a token grid of `tokens_per_frame` patches, so that wvn_mlp_infer_pixels
 * never allocates (call once after create; a later call with a larger grid grows them). */
int wvn_mlp_infer_reserve(wvn_mlp_infer_t* h, int tokens_per_frame);
/* params: flat fp32 buffer in state_dict order layers.0.weight, layers.0.bias, layers.2.weight,
 * layers.2.bias, layers.4.weight, layers.4.bias (device memory). */
int wvn_mlp_infer_set_params(wvn_mlp_infer_t* h, const float* params, void* stream);
/* tokens: [batch, gh*gw, dim] fp32; trav, conf: [batch, out_h, out_w] fp32;
 * cg_mean, cg_std: device scalars of the ConfidenceGenerator. */
int wvn_mlp_infer_pixels(wvn_mlp_infer_t* h, const float* tokens, int batch, int gh, int gw, int out_h, int out_w,
                         const float* cg_mean, const float* cg_std, float std_factor, float* trav, float* conf,
                         void* stream);
/* The same maps straight from the backbone's own bf16 token buffer (the tokens of the last wvn_vit_forward* call, frames
 * [0, batch)): no fp32 -> bf16 re-cast of the tokens; patch p of a frame is read from row 1 + registers + p.  Needs
 * dim == the backbone's width and the fused geometry. */
int wvn_mlp_infer_pixels_vit(wvn_mlp_infer_t* h, wvn_vit_t* vit, int batch, int out_h, int out_w, const float* cg_mean,
                             const float* cg_std, float std_factor, float* trav, float* conf, void* stream);
/* Same arithmetic on explicit rows x: [rows, dim] fp32 (segment-wise prediction mode). */
int wvn_mlp_infer_rows(wvn_mlp_infer_t* h, const float* x, long long rows, const float* cg_mean,
                       const float* cg_std, float std_factor, float* trav, float* conf, void* stream);
/* The same on rows padded per frame: x [groups, rows_per_group, dim] fp32, n_rows [groups] int32 on the device (row r of
 * group g is live when r < n_rows[g]).  trav / conf: [groups, rows_per_group]; padding rows are NaN and their features
 * are never read (the loader writes zeros in their place).  A live row's values are bit-identical to
 * wvn_mlp_infer_rows on the compacted rows: the GEMM chain's tiles do not depend on the row count.  No host
 * synchronisation, no allocation. */
int wvn_mlp_infer_rows_padded(wvn_mlp_infer_t* h, const float* x, int groups, int rows_per_group, const int* n_rows,
                              const float* cg_mean, const float* cg_std, float std_factor, float* trav, float* conf,
                              void* stream);
/* The same handle for a DoubleMLP(dim, [h1, h2, 1]) (bounds of wvn_double_mlp_trainer_create): set_params takes its
 * flat parameters (networks.0.{0,2,4}.{weight,bias}, then networks.1's) and packs the two nets as one block-structured
 * MLP of widths 2 h1 / 2 h2 — layer 1 [W1_0; W1_1], layer 2 diag(W2_0, W2_1), layer 3 [w3_0 | 0] for traversability and
 * [0 | W3_1] for the reconstruction — so pixels / rows compute sigmoid(net0(x)), the reconstruction error of net1(x)
 * and its confidence with the GEMM chain above.  For h1 in {64, 128} and h2 = 32, pixels and pixels_vit take the fused
 * per-pixel head at its geometries (per-token GEMM columns G_0 | G_1 | U | cT, layer 2 as one wgmma chain per network);
 * other shapes and geometries take the unfused path, and pixels_vit then fails. */
int wvn_mlp_infer_create_double(int dim, int h1, int h2, int chunk_rows, wvn_mlp_infer_t** out);

/* ------------------------------------------------------------------------------------------
 * Online train step (fp32) — replaces the body of TraversabilityEstimator.train()
 * (traversability_estimator/traversability_estimator.py:464-477): SimpleMLP.forward,
 * TraversabilityLoss.forward (utils/loss.py:93-160) with the ConfidenceGenerator
 * "latest_measurement" update (utils/confidence_generator.py:78-82), backward, Adam.
 * Three phases so a data-parallel caller can all-reduce between them:
 *   forward_stats -> [all-reduce scalars[0..4] (5 doubles)] -> backward
 *   -> [all-reduce grads (n_params + 1 floats)] -> finalize + adam.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  float w_trav, w_reco, std_factor;
  int anomaly_balanced;
  float lr, beta1, beta2, eps;
} wvn_train_config;

size_t wvn_mlp_param_count(int dim, int h1, int h2);
size_t wvn_mlp_train_workspace_bytes(int dim, int h1, int h2, int max_rows);
size_t wvn_mlp_train_scalars_bytes(void);
int wvn_mlp_train_forward_stats(int dim, int h1, int h2, const float* params, const float* x, const float* y,
                                const unsigned char* y_valid, int rows, int max_rows, void* workspace, void* scalars,
                                void* stream);
int wvn_mlp_train_backward(int dim, int h1, int h2, const float* params, const float* x, const float* y,
                           const unsigned char* y_valid, int rows, int max_rows, long long n_total,
                           const wvn_train_config* cfg, void* workspace, void* scalars, float* cg_mean, float* cg_std,
                           float* grads, float* confidence_out, void* stream);
int wvn_mlp_train_apply(int dim, int h1, int h2, float* params, const float* grads, float* exp_avg, float* exp_avg_sq,
                        long long* step_counter, long long n_total, const wvn_train_config* cfg, void* scalars,
                        void* stream);
/* metrics_out (device, 6 floats): loss_total, loss_trav, loss_reco, loss_trav_confidence, cg_mean, cg_std */
int wvn_mlp_train_read_metrics(const void* scalars, float* metrics_out, void* stream);
/* fp32 forward only: out [rows, 1+dim] (column 0 through the sigmoid), SimpleMLP.forward. */
int wvn_mlp_forward_f32(int dim, int h1, int h2, const float* params, const float* x, int rows, float* h1_buf,
                        float* h2_buf, float* out, void* stream);

/* ------------------------------------------------------------------------------------------
 * Trainers.  Every learner's train step (SimpleMLP, DoubleMLP, SimpleGCN, LinearRnvp) runs on a wvn_trainer_t made by
 * that learner's create function; the functions below work on any of them.  A learner's own entry points return
 * WVN_STATUS_INVALID, before they enqueue anything, when given another learner's handle.
 *
 * Data-parallel steps: each step has three phases (phase_mask 1, 2, 4; 7 = the whole step) with an exchange after the
 * first two.  With a communicator (wvn_trainer_init_comm) the step issues both all-reduces itself, between its kernels
 * on the caller's stream.  Without one, a data-parallel caller all-reduces, between the phases, the statistics block
 * (wvn_trainer_stats) — doubles 0..5 with SUM, and for moving_average double 6 with MIN and 7 with MAX — after phase 1,
 * and after phase 2 the gradient with SUM and, when the block has a ninth double, that double with SUM.
 * ---------------------------------------------------------------------------------------- */
typedef struct wvn_trainer wvn_trainer_t;
void wvn_trainer_destroy(wvn_trainer_t* t);
/* ConfidenceGenerator method of the step (utils/confidence_generator.py:49-76): 0 latest_measurement (default),
 * 1 running_mean (:94-115), 2 kalman_filter (:131-145 with utils/kalman_filter.py:78-111, D = 1, F = H = 1; kf_proc_cov /
 * kf_meas_cov = its Q / R), 3 moving_average (:117-129, window of 5 steps kept inside the trainer).  The state the
 * reference keeps in module parameters is read and updated in place through these device pointers — var (1,1) fp32;
 * running_n / running_sum / running_sum_of_squares (1,) fp64 — each may be NULL (the trainer then keeps a private copy). */
int wvn_trainer_set_confidence(wvn_trainer_t* t, int method, float* var, double* running_n, double* running_sum,
                               double* running_sum_of_squares, float kf_proc_cov, float kf_meas_cov);
/* Copies the confidence state src keeps itself (moving_average's window of 5 steps; var / running sums given as NULL to
 * set_confidence) into dst, ordered on `stream`.  For replacing a trainer by a larger one: create the new one, copy,
 * then destroy the old one; the generator continues as if nothing had changed.  Both must be the same learner's. */
int wvn_trainer_copy_confidence(wvn_trainer_t* dst, const wvn_trainer_t* src, void* stream);
/* Library-owned NCCL communicator (libnccl.so.2 is resolved from the running process): rank 0 fills a 128-byte id with
 * wvn_comm_unique_id, the caller broadcasts it by any means, every rank calls wvn_trainer_init_comm. */
int wvn_comm_unique_id(void* id128);
int wvn_trainer_init_comm(wvn_trainer_t* t, const void* id128, int rank, int world);
/* The trainer's statistics block (device doubles; *n_doubles receives their number, 8 or 9): sum and sum of squares of
 * the confidence input (loss_reco, or the NLL for LinearRnvp) over the labelled rows, sum of (trav - y)^2 (0 for
 * LinearRnvp), labelled and live row counts (LinearRnvp: labelled, then 0), a sixth sum (SimpleGCN: the overflow flag,
 * so its SUM tells every rank; else 0), the input's min and max; DoubleMLP and SimpleGCN add a ninth double, the
 * confidence-weighted traversability error summed over the live rows, written by phase 2.  For SimpleMLP the block is
 * the first 8 doubles of the trainer's scalars.  Valid until the trainer is destroyed. */
double* wvn_trainer_stats(wvn_trainer_t* t, int* n_doubles);

/* ------------------------------------------------------------------------------------------
 * Fused online train step — the same arithmetic as the three-phase entry points above in FOUR kernels, with the
 * row compaction (`feat[seg_mask]`, wvn_feature_extractor_node.py:324-327 / nodes.py:199-241) and, for data-parallel
 * runs, the two all-reduces inside the library (SURVEY.md §8b "wvn_mlp_train_step(..., ncclComm_t or NULL, ...)",
 * §8e).  No host synchronisation, no allocation after create.
 *   x: [groups, rows_per_group, dim] fp32, PADDED per group; n_rows: [groups] int32 (device) live rows per group, or
 *   NULL when every row is live;  y [fp32] / y_valid [uint8] / confidence_out [fp32] are indexed by the COMPACTED row
 *   number (live rows of group 0, then group 1, ...);  metrics_out (device, 6 floats, may be NULL): loss_total,
 *   loss_trav, loss_reco, loss_trav_confidence, cg_mean, cg_std.  params / exp_avg / exp_avg_sq: flat fp32 buffers in
 *   state_dict order (torch.optim.Adam state), step_counter: device int64.
 * phase_mask: 7 = whole step; 1 / 2 / 4 = forward+stats / backward+weight-gradients / metrics+Adam separately; the
 * gradient a caller without a communicator all-reduces has n_params + 1 floats.
 * ---------------------------------------------------------------------------------------- */
/* scalars: optional caller-owned device buffer of wvn_mlp_trainer_scalars_bytes(); grads: optional caller-owned device
 * buffer of n_params + 1 floats (NULL: the trainer allocates them with its workspace). */
size_t wvn_mlp_trainer_scalars_bytes(void);
int wvn_mlp_trainer_create(int dim, int h1, int h2, int max_rows, const wvn_train_config* cfg, void* scalars,
                           float* grads, wvn_trainer_t** out);
int wvn_mlp_train_step(wvn_trainer_t* t, float* params, float* exp_avg, float* exp_avg_sq, long long* step_counter,
                       const float* x, int groups, int rows_per_group, const int* n_rows, const float* y,
                       const unsigned char* y_valid, float* cg_mean, float* cg_std, float* confidence_out,
                       float* metrics_out, int phase_mask, void* stream);

/* ------------------------------------------------------------------------------------------
 * DoubleMLP learner (model/simple_mlp.py DoubleMLP, fp32): DoubleMLP(dim, [h1, h2, 1]) — networks.0 Linear(dim, h1)
 * ReLU Linear(h1, h2) ReLU Linear(h2, 1) through a sigmoid (traversability), networks.1 the same ending in
 * Linear(h2, dim) (reconstruction); output [rows, 1 + dim] = [sigmoid(net0(x)) | net1(x)], SimpleMLP's layout.
 * Bounds: 1 <= dim <= 1024, 4 <= h1 <= 256 and a multiple of 4, 1 <= h2 <= 32.  params / exp_avg / exp_avg_sq: flat
 * fp32 buffers of wvn_double_mlp_param_count floats in parameters() order (networks.0.{0,2,4}.{weight,bias}, then
 * networks.1's), i.e. torch.optim.Adam's state.  The trainer owns the workspaces for max_rows rows.
 * ---------------------------------------------------------------------------------------- */
size_t wvn_double_mlp_param_count(int dim, int h1, int h2);
/* DoubleMLP.forward on x [rows, dim] fp32: a1_buf [2, rows, h1], a2_buf [2, rows, h2] (net 0, then net 1) receive the
 * hidden activations, out [rows, 1 + dim] the output. */
int wvn_double_mlp_forward_f32(int dim, int h1, int h2, const float* params, const float* x, int rows, float* a1_buf,
                               float* a2_buf, float* out, void* stream);
/* cfg: the loss weights, anomaly_balanced, the generator's std_factor and Adam's lr / betas / eps; grads: optional
 * caller-owned device buffer of wvn_double_mlp_param_count floats (NULL: the trainer allocates it). */
int wvn_double_mlp_trainer_create(int dim, int h1, int h2, int max_rows, const wvn_train_config* cfg, float* grads,
                                  wvn_trainer_t** out);
/* One step of TraversabilityEstimator.train() with TraversabilityLoss on rows padded per group: forward, loss, the
 * ConfidenceGenerator update, backward, Adam; one fixed sequence of launches, no host synchronisation,
 * bit-reproducible.  x: [groups, rows_per_group, dim] fp32; n_rows: [groups] int32 (device) live rows per group, or NULL
 * when every row is live; y [fp32] / y_valid [uint8] / confidence_out are indexed by the COMPACTED row number (live rows
 * of group 0, then group 1, ...).  Padding rows may hold anything (NaN included): they are never read.
 * groups * rows_per_group <= max_rows.  metrics_out (device, 6 floats, may be NULL): loss_total, loss_trav, loss_reco,
 * loss_trav_confidence, cg_mean, cg_std.  phase_mask: 7 = whole step; 1 = forward + the statistic sums, 2 = generator
 * update + backward + weight gradients, 4 = metrics + Adam. */
int wvn_double_mlp_train_step_padded(wvn_trainer_t* t, float* params, float* exp_avg, float* exp_avg_sq,
                                     long long* step_counter, const float* x, int groups, int rows_per_group,
                                     const int* n_rows, const float* y, const unsigned char* y_valid, float* cg_mean,
                                     float* cg_std, float* confidence_out, float* metrics_out, int phase_mask,
                                     void* stream);

/* ------------------------------------------------------------------------------------------
 * SimpleGCN learner (model/simple_gcn.py, fp32): SimpleGCN(dim, True, [h1, h2, 1]) — GCNConv(dim, h1) ReLU
 * GCNConv(h1, h2) ReLU GCNConv(h2, 1 + dim), sigmoid on column 0; output [rows, 1 + dim], SimpleMLP's layout.  Each
 * GCNConv is torch_geometric 2.x's with its defaults: Z = D^-1/2 (A + I) D^-1/2 X W^T + b, A[i, j] the number of edges
 * j -> i once the input's self-loops are dropped, D = 1 + the in-degree.  Edges are directed as given (not symmetrised).
 * Bounds: 1 <= dim <= 1024, 1 <= h1, h2 <= 512.  params / exp_avg / exp_avg_sq: flat fp32 buffers of
 * wvn_gcn_param_count floats in parameters() order (layers.{0,1,2}: bias, then lin.weight [out, in]).
 * Rows come padded per frame: x [groups, rows_per_group, dim] fp32 with n_rows [groups] int32 (device; NULL: all) live
 * rows per frame, and the frame's graph as edges [groups, edges_per_group, 2] int64 (source, target) local row ids of
 * which the first n_edges[g] (device int32) are read.  Edges with an endpoint outside the frame's live rows are dropped.
 * The handle owns the workspaces for max_rows padded rows and max_edges padded edges (groups * edges_per_group).
 * ---------------------------------------------------------------------------------------- */
size_t wvn_gcn_param_count(int dim, int h1, int h2);
/* cfg: the loss weights, anomaly_balanced, the generator's std_factor and Adam's lr / betas / eps; grads: optional
 * caller-owned device buffer of wvn_gcn_param_count floats (NULL: the trainer allocates it). */
int wvn_gcn_trainer_create(int dim, int h1, int h2, int max_rows, int max_edges, const wvn_train_config* cfg,
                           float* grads, wvn_trainer_t** out);
/* One step of TraversabilityEstimator.train() with TraversabilityLoss on the padded frames and their graphs: graph
 * build, forward, loss, the ConfidenceGenerator update, backward, Adam; no host synchronisation, bit-reproducible.
 * y / y_valid / confidence_out are indexed by the COMPACTED row number (live rows of frame 0, then frame 1, ...).
 * metrics_out (device, 7 floats, may be NULL): loss_total, loss_trav, loss_reco, loss_trav_confidence, cg_mean, cg_std,
 * and 1 when some n_edges[g] was negative (the segment reducer's overflow flag; that frame's edges are not read), else 0.
 * phase_mask as wvn_double_mlp_train_step_padded. */
int wvn_gcn_train_step_padded(wvn_trainer_t* t, float* params, float* exp_avg, float* exp_avg_sq,
                              long long* step_counter, const float* x, int groups, int rows_per_group,
                              const int* n_rows, const long long* edges, int edges_per_group, const int* n_edges,
                              const float* y, const unsigned char* y_valid, float* cg_mean, float* cg_std,
                              float* confidence_out, float* metrics_out, int phase_mask, void* stream);
/* SimpleGCN.forward on the same padded input (a negative n_edges[g]: no edges for that frame), then per live row
 * traversability = out[:, 0] and the confidence of its reconstruction loss under the generator (mean / std device
 * scalars, std_factor; ConfidenceGenerator.inference_without_update).  out (may be NULL): [groups * rows_per_group,
 * 1 + dim], the live rows first in compacted order.  trav / confidence (may be NULL): [groups * rows_per_group] in
 * PADDED order; padding rows are not written. */
int wvn_gcn_infer_rows(wvn_trainer_t* t, const float* params, const float* x, int groups, int rows_per_group,
                       const int* n_rows, const long long* edges, int edges_per_group, const int* n_edges,
                       const float* cg_mean, const float* cg_std, float std_factor, float* out, float* trav,
                       float* confidence, void* stream);

/* ------------------------------------------------------------------------------------------
 * LinearRnvp anomaly-detection learner (model/linear_rnvp.py, fp32): LinearRnvp(dim, [hidden]) with flow_n = 2,
 * use_permutation = True — coupling 0, permutation 1, coupling 2, permutation 3; every coupling has nets s and t, each
 * Linear(dim, hidden) ReLU Linear(hidden, hidden) ReLU Linear(hidden, dim).  Bounds: 2 <= dim <= 4096, hidden <= 512
 * and a multiple of 8.  params / exp_avg / exp_avg_sq: flat fp32 buffers of wvn_flow_param_count floats in the
 * module's parameters() order (flows.0.s, flows.0.t, flows.2.s, flows.2.t; each net 0.weight, 0.bias, 2.weight,
 * 2.bias, 4.weight, 4.bias), i.e. torch.optim.Adam's state.  The masks and permutations are read from the model's
 * buffers on every call, so "odds" and "half" masks and a loaded permutation cost nothing.
 * The handle owns the workspaces for max_rows rows (allocated at create, nothing per call).
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  const float* mask0;       /* flows.0.mask [dim] fp32 */
  const float* mask1;       /* flows.2.mask [dim] fp32 */
  const long long* p1;      /* flows.1.p / flows.1.invp [dim] int64 */
  const long long* invp1;
  const long long* p3;      /* flows.3.p / flows.3.invp [dim] int64 */
  const long long* invp3;
} wvn_flow_buffers;
size_t wvn_flow_param_count(int dim, int hidden);
/* cfg: std_factor (the ConfidenceGenerator's) and Adam's lr / betas / eps are used; grads: optional caller-owned device
 * buffer of wvn_flow_param_count floats (NULL: the handle allocates it). */
int wvn_flow_trainer_create(int dim, int hidden, int max_rows, const wvn_train_config* cfg, float* grads,
                            wvn_trainer_t** out);
/* One step of TraversabilityEstimator.train() with AnomalyLoss on the rows of x [rows, dim] whose y_valid [rows] uint8
 * is set (NULL: every row): forward, loss -mean(sum(logprob) + log_det), the ConfidenceGenerator update with the
 * per-row NLL, backward, Adam.  No host synchronisation.  confidence_out [rows]: the labelled rows in order;
 * metrics_out (device, 6 floats, may be NULL): loss_total, loss_trav (0), loss_reco (0), labelled rows, cg_mean, cg_std.
 * phase_mask: 7 = whole step; 1 = forward + statistics + generator update, 2 = backward (gradient), 4 = Adam. */
int wvn_flow_train_step(wvn_trainer_t* t, float* params, float* exp_avg, float* exp_avg_sq, long long* step_counter,
                        const wvn_flow_buffers* buffers, const float* x, int rows, const unsigned char* y_valid,
                        float* cg_mean, float* cg_std, float* confidence_out, float* metrics_out, int phase_mask,
                        void* stream);
/* The same step on rows padded per group, data-parallel.  x: [groups, rows_per_group, dim] fp32; n_rows: [groups] int32
 * (device) live rows per group, or NULL; y_valid (NULL: all) is indexed by the COMPACTED row number and selects the
 * rows trained on; confidence_out: the selected rows in order.  Padding rows are never read.  phase_mask: 7 = whole step;
 * 1 = forward + the NLL sums, 2 = generator update + metrics + confidence + backward, 4 = Adam (note: phase 1 here
 * stops BEFORE the generator update, which needs the global sums).  The loss is the NLL's mean over the global labelled
 * count; a rank with no labelled row still takes part. */
int wvn_flow_train_step_padded(wvn_trainer_t* t, float* params, float* exp_avg, float* exp_avg_sq,
                               long long* step_counter, const wvn_flow_buffers* buffers, const float* x, int groups,
                               int rows_per_group, const int* n_rows, const unsigned char* y_valid, float* cg_mean,
                               float* cg_std, float* confidence_out, float* metrics_out, int phase_mask, void* stream);

/* Inference handle (no backward workspaces, no gradient buffer).  max_rows: rows of wvn_flow_infer_rows per call;
 * chunk_pixels: pixels per wgmma chunk of wvn_flow_infer_pixels (0 = 8192). */
typedef struct wvn_flow_infer wvn_flow_infer_t;
int wvn_flow_infer_create(int dim, int hidden, int max_rows, int chunk_pixels, wvn_flow_infer_t** out);
void wvn_flow_infer_destroy(wvn_flow_infer_t* h);
/* Packs the bf16 operands of the per-pixel path from the flat fp32 parameters: call again after they change. */
int wvn_flow_infer_set_params(wvn_flow_infer_t* h, const float* params, void* stream);
/* LinearRnvp.forward on x [rows, dim] fp32 in fp32 (rows <= max_rows): z / logprob [rows, dim], log_det [rows], each may
 * be NULL.  trav [rows] (may be NULL): ConfidenceGenerator.inference_without_update of the NLL
 * -(sum(logprob) + log_det) with the generator's mean / std (device scalars) and std_factor. */
int wvn_flow_infer_rows(wvn_flow_infer_t* h, const float* params, const wvn_flow_buffers* buffers, const float* x, int rows,
                        float* z, float* log_det, float* logprob, const float* cg_mean, const float* cg_std,
                        float std_factor, float* trav, void* stream);
/* The same trav on rows padded per frame: x [groups, rows_per_group, dim] fp32, n_rows [groups] int32 on the device
 * (groups * rows_per_group <= max_rows).  trav [groups, rows_per_group]: the live rows' values, NaN on padding rows,
 * which are neither read nor computed.  No host synchronisation, no allocation. */
int wvn_flow_infer_rows_padded(wvn_flow_infer_t* h, const float* params, const wvn_flow_buffers* buffers, const float* x,
                               int groups, int rows_per_group, const int* n_rows, const float* cg_mean,
                               const float* cg_std, float std_factor, float* trav, void* stream);
/* The per-pixel anomaly map (wvn_feature_extractor_node.py:332-338): tokens [batch, gh * gw, dim] fp32 are upsampled
 * bilinearly (align_corners = True) to out_h x out_w, every net layer runs as a wgmma GEMM (bf16 operands, fp32
 * accumulation), the coupling arithmetic in fp32.  trav [batch, out_h, out_w]: inference_without_update of the NLL;
 * nll (may be NULL): the per-pixel NLL.  Masks / permutations are read from `buffers` on every call. */
int wvn_flow_infer_pixels(wvn_flow_infer_t* h, const wvn_flow_buffers* buffers, const float* tokens, int batch, int gh,
                          int gw, int out_h, int out_w, const float* cg_mean, const float* cg_std, float std_factor,
                          float* trav, float* nll, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* WVN_B200_H_ */
