// wvn-b200: the convolutional trunk handles — torchvision ResNet-18 / ResNet-50 and EfficientNet-B0 (reference
// torchvision_interface.py).
#include "conv_trunk.h"

#include <algorithm>
#include <string>

#include "effnet_kernels.h"
#include "gemm.h"
#include "host_common.h"
#include "resnet_kernels.h"

using namespace wvn;

namespace {

constexpr int kTrunkRoles = 5;  // activation workspaces a trunk's walk may name

// What a convolutional trunk handle owns: its weights, the im2col rows and the activation workspaces, all sized at
// create.
struct ConvTrunk {
  WeightStore weights;
  DevBuf col;
  DevBuf act[kTrunkRoles];

  size_t workspace_bytes() const {
    size_t n = col.bytes;
    for (const auto& b : act) n += b.bytes;
    return n;
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
      if ((rc = t->weights.add(name + ".weight", Cout, K, true)) != WVN_OK) return;
      rc = t->weights.add(name + ".bias", 1, Cout, false);
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
    g.bias = t->weights.ptr<const float>(name + ".bias");
    g.out = out; g.ldo = Cout;
    g.residual = residual; g.ldr = Cout;
    rc = gemm_bf16(g, A, lda, t->weights.ptr<void>(name + ".weight"), 0, s);
  }

  // allocates the workspaces the RN_SIZE walk asked for
  int alloc_workspaces() const {
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

namespace wvn {

int resnet_create(const wvn_resnet_config* cfg, wvn_resnet** out) {
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
    delete h;
    return rc;
  }
  *out = h;
  return WVN_OK;
}

void resnet_destroy(wvn_resnet* h) { delete h; }

size_t resnet_workspace_bytes(const wvn_resnet* h) { return h->workspace_bytes(); }

int resnet_set_weight(wvn_resnet* h, const char* name, const float* data, long long numel) {
  return h->weights.set(name, data, numel);
}

int resnet_forward(wvn_resnet* h, const float* img, int batch, void* const* taps, cudaStream_t s) {
  WVN_REQUIRE(batch > 0 && batch <= h->cfg.max_batch, "wvn_resnet_forward: batch %d outside (0, %d]", batch,
              h->cfg.max_batch);
  for (int i = 0; i < 4; ++i) WVN_REQUIRE(taps[i], "wvn_resnet_forward: tap %d is null", i);
  WVN_PROPAGATE(h->weights.check_loaded("resnet"));
  ResnetRun run(h, RN_RUN, batch, s);
  run.walk(img, taps);
  return run.rc;
}

}  // namespace wvn

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
      if ((rc = t->weights.add(name + ".weight", 1, k * k * P, false)) != WVN_OK) return;
      rc = t->weights.add(name + ".bias", 1, P, false);
      return;
    }
    if (pass == RN_SIZE) {
      need(3, static_cast<size_t>(batch) * *Ho * *Wo * P * 2);
      need_partial = std::max(need_partial, static_cast<size_t>(batch) * depthwise_pool_blocks(*Ho, *Wo) * P * 4);
      return;
    }
    rc = depthwise_silu(in, batch, H, W, P, k, stride, t->weights.ptr<const float>(name + ".weight"),
                        t->weights.ptr<const float>(name + ".bias"), h->act[3].p, reinterpret_cast<float*>(h->partial.p), s);
  }

  // squeeze-excitation of buffer 3 [batch, Ho, Wo, P] (C real channels, `squeeze` hidden), in place
  void squeeze_excite(const std::string& name, int Ho, int Wo, int C, int P, int squeeze) {
    if (rc != WVN_OK) return;
    if (pass == RN_REGISTER) {
      if ((rc = t->weights.add(name + ".fc1.weight", squeeze, P, false)) != WVN_OK) return;
      if ((rc = t->weights.add(name + ".fc1.bias", 1, squeeze, false)) != WVN_OK) return;
      if ((rc = t->weights.add(name + ".fc2.weight", P, squeeze, false)) != WVN_OK) return;
      rc = t->weights.add(name + ".fc2.bias", 1, P, false);
      return;
    }
    if (pass == RN_SIZE) {
      need_gates = std::max(need_gates, static_cast<size_t>(batch) * P * 4);
      return;
    }
    float* gates = reinterpret_cast<float*>(h->gates.p);
    rc = se_gates(reinterpret_cast<const float*>(h->partial.p), batch, depthwise_pool_blocks(Ho, Wo), Ho * Wo, C, P,
                  t->weights.ptr<const float>(name + ".fc1.weight"), t->weights.ptr<const float>(name + ".fc1.bias"), squeeze,
                  t->weights.ptr<const float>(name + ".fc2.weight"), t->weights.ptr<const float>(name + ".fc2.bias"), gates, s);
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

namespace wvn {

int effnet_create(const wvn_effnet_config* cfg, wvn_effnet** out) {
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
    delete h;
    return rc;
  }
  *out = h;
  return WVN_OK;
}

void effnet_destroy(wvn_effnet* h) { delete h; }

size_t effnet_workspace_bytes(const wvn_effnet* h) { return h->workspace_bytes() + h->partial.bytes + h->gates.bytes; }

int effnet_set_weight(wvn_effnet* h, const char* name, const float* data, long long numel) {
  return h->weights.set(name, data, numel);
}

int effnet_forward(wvn_effnet* h, const float* img, int batch, void* const* taps, cudaStream_t s) {
  WVN_REQUIRE(batch > 0 && batch <= h->cfg.max_batch, "wvn_effnet_forward: batch %d outside (0, %d]", batch,
              h->cfg.max_batch);
  for (int i = 0; i < 5; ++i) WVN_REQUIRE(taps[i], "wvn_effnet_forward: tap %d is null", i);
  WVN_PROPAGATE(h->weights.check_loaded("effnet"));
  EffnetRun run(h, RN_RUN, batch, s);
  run.walk(img, taps);
  return run.rc;
}

}  // namespace wvn
