// wvn-b200: online traversability-MLP training step in fp32 (sm_90a, latency-bound).
//
// One call sequence = the body of TraversabilityEstimator.train()
// (traversability_estimator.py:464-477):
//   res  = SimpleMLP.forward(x)                      (model/simple_mlp.py:33-39)
//   loss = TraversabilityLoss(graph, res)            (utils/loss.py:93-160) incl. the
//          ConfidenceGenerator "latest_measurement" update (utils/confidence_generator.py:78-82)
//   loss.backward(); Adam.step()                     (torch.optim.Adam defaults, lr from params)
//
// The learner has 119 489 parameters and a few thousand rows per step: the reference spends
// its time in ~60 tiny eager launches and three .item() syncs.  Here the step is a fixed
// sequence of 13 small fp32 kernels with every scalar kept on the device, split in three
// phases so a data-parallel caller can all-reduce (a) the three confidence statistics and
// (b) the flat gradient between them (SURVEY.md §8e).  fp32 CUDA-core math on purpose: the
// work is ~2 GFLOP and the reference's arithmetic is fp32, so parity is tight (1e-5).
#include "common.cuh"
#include "host_common.h"
#include "mlp_train.h"

namespace wvn {

namespace {

constexpr int TS = 64;  // C tile
constexpr int TK = 16;

enum { SACT_NONE = 0, SACT_RELU = 1, SACT_SIGMOID_COL0 = 2 };

struct SgemmArgs {
  const float* A; long long sam, sak;   // A(m,k) = A[m*sam + k*sak]
  const float* B; long long sbk, sbn;   // B(k,n) = B[k*sbk + n*sbn]
  float* C; long long ldc;
  int M, N, K;
  const float* bias;                    // [N] or null
  int act;
  const float* relu_mask; long long ld_mask;  // multiply by (mask[m,n] > 0) or null
  int k_per_split;                      // K range per blockIdx.z; > 0 and < K => atomic accumulate into C
};

__global__ void __launch_bounds__(256)
sgemm_kernel(SgemmArgs a) {
  __shared__ float As[TK][TS + 1];
  __shared__ float Bs[TK][TS + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * TS, n0 = blockIdx.x * TS;
  const int kbeg = blockIdx.z * a.k_per_split;
  const int kend = min(a.K, kbeg + a.k_per_split);
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = kbeg; k0 < kend; k0 += TK) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int idx = threadIdx.x + 256 * r;  // 0..1023
      int m, k;
      if (a.sak == 1) { m = idx >> 4; k = idx & 15; } else { k = idx >> 6; m = idx & 63; }
      const int gm = m0 + m, gk = k0 + k;
      As[k][m] = (gm < a.M && gk < kend) ? a.A[gm * a.sam + gk * a.sak] : 0.f;
      int n, kk;
      if (a.sbk == 1) { n = idx >> 4; kk = idx & 15; } else { kk = idx >> 6; n = idx & 63; }
      const int gn = n0 + n, gk2 = k0 + kk;
      Bs[kk][n] = (gn < a.N && gk2 < kend) ? a.B[gk2 * a.sbk + gn * a.sbn] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TK; ++k) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) av[i] = As[k][ty + 16 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) bv[j] = Bs[k][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
  const bool atomic = a.k_per_split < a.K;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gm = m0 + ty + 16 * i;
    if (gm >= a.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx + 16 * j;
      if (gn >= a.N) continue;
      float v = acc[i][j];
      if (atomic) {
        atomicAdd(&a.C[gm * a.ldc + gn], v);
      } else {
        if (a.bias) v += a.bias[gn];
        if (a.act == SACT_RELU) v = fmaxf(v, 0.f);
        if (a.act == SACT_SIGMOID_COL0 && gn == 0) v = 1.f / (1.f + expf(-v));
        if (a.relu_mask) v = (a.relu_mask[gm * a.ld_mask + gn] > 0.f) ? v : 0.f;
        a.C[gm * a.ldc + gn] = v;
      }
    }
  }
}

int sgemm(const SgemmArgs& a, int splits, cudaStream_t s) {
  SgemmArgs b = a;
  if (splits < 1) splits = 1;
  b.k_per_split = ((a.K + splits - 1) / splits + TK - 1) / TK * TK;
  const int z = (a.K + b.k_per_split - 1) / b.k_per_split;
  if (z <= 1) b.k_per_split = a.K;
  dim3 grid((a.N + TS - 1) / TS, (a.M + TS - 1) / TS, z < 1 ? 1 : z);
  sgemm_kernel<<<grid, 256, 0, s>>>(b);
  WVN_CHECK_LAUNCH("sgemm_kernel");
  return WVN_OK;
}

// ---- per-row loss terms + global statistics -------------------------------------------------
// One warp per row: loss_reco_i = mean_d (out[i,1+d] - x[i,d])^2 ; raw_i = (out[i,0] - y_i)^2.
__global__ void __launch_bounds__(256)
loss_rows_kernel(const float* __restrict__ out, const float* __restrict__ x, const float* __restrict__ y,
                 const unsigned char* __restrict__ valid, float* __restrict__ loss_reco, float* __restrict__ raw,
                 TrainScalars* __restrict__ sc, int rows, int dim) {
  const int lane = threadIdx.x & 31;
  const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int warps_total = (gridDim.x * blockDim.x) >> 5;
  double s1 = 0.0, s2 = 0.0, sraw = 0.0, nv = 0.0;
  for (int r = warp_global; r < rows; r += warps_total) {
    const float* o = out + static_cast<long long>(r) * (dim + 1);
    const float* xr = x + static_cast<long long>(r) * dim;
    float acc = 0.f;
    for (int d = lane; d < dim; d += 32) {
      const float df = o[1 + d] - xr[d];
      acc = fmaf(df, df, acc);
    }
    acc = warp_sum(acc) / static_cast<float>(dim);
    if (lane == 0) {
      loss_reco[r] = acc;
      const float dt = o[0] - y[r];
      raw[r] = dt * dt;
      sraw += static_cast<double>(dt * dt);
      if (valid[r]) { s1 += acc; s2 += static_cast<double>(acc) * acc; nv += 1.0; }
    }
  }
  if (lane == 0 && (nv != 0.0 || sraw != 0.0)) {
    atomicAdd(&sc->sum_lr, s1);
    atomicAdd(&sc->sum_lr2, s2);
    atomicAdd(&sc->sum_raw, sraw);
    atomicAdd(&sc->n_valid, nv);
  }
}

// ConfidenceGenerator.update_latest_measurement: mean / unbiased std of the valid rows'
// loss_reco -> persisted into the generator's parameters.
__global__ void confidence_update_kernel(TrainScalars* sc, float* cg_mean, float* cg_std, float* cg_var) {
  const double n = sc->n_valid;
  const double mean = sc->sum_lr / n;                        // n == 0 -> NaN, like torch's mean of empty
  const double var = (sc->sum_lr2 - n * mean * mean) / (n - 1.0);  // n == 1 -> NaN, like torch.std
  const float sd = static_cast<float>(sqrt(fmax(var, 0.0)));
  const float m = static_cast<float>(mean);
  sc->mean = m;
  sc->std = (n > 1.0) ? sd : nanf("");
  if (cg_mean) *cg_mean = sc->mean;
  if (cg_std) *cg_std = sc->std;
  (void)cg_var;  // 'latest_measurement' leaves var untouched (confidence_generator.py:78-82)
}

// dOut + the scalar loss terms.  One warp per row.
__global__ void __launch_bounds__(256)
loss_grad_kernel(const float* __restrict__ out, const float* __restrict__ x, const float* __restrict__ y,
                 const unsigned char* __restrict__ valid, const float* __restrict__ loss_reco,
                 const float* __restrict__ raw, float* __restrict__ d_out, float* __restrict__ conf_out,
                 TrainScalars* __restrict__ sc, float* __restrict__ trav_w_sum, LossCfg cfg, int rows, int dim,
                 long long n_total) {
  const int lane = threadIdx.x & 31;
  const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int warps_total = (gridDim.x * blockDim.x) >> 5;
  const float mean = sc->mean, sd = sc->std;
  const float shifted = mean + sd * cfg.std_factor;
  const float lo = fmaxf(shifted - sd, 0.f);
  const float hi = shifted + sd;
  const float n_valid = static_cast<float>(sc->n_valid);
  const float g_reco = cfg.w_reco * 2.f / (n_valid * static_cast<float>(dim));
  const float g_trav = cfg.w_trav * 2.f / static_cast<float>(n_total);
  double s_trav = 0.0;
  for (int r = warp_global; r < rows; r += warps_total) {
    const float* o = out + static_cast<long long>(r) * (dim + 1);
    const float* xr = x + static_cast<long long>(r) * dim;
    float* g = d_out + static_cast<long long>(r) * (dim + 1);
    const bool v = valid[r] != 0;
    const float lr = loss_reco[r];
    const float xc = fminf(fmaxf(lr, lo), hi);
    const float conf = 1.f - (xc - lo) / (hi - lo);
    const float wgt = (v || !cfg.anomaly_balanced) ? 1.f : (1.f - conf);
    for (int d = lane; d < dim; d += 32) g[1 + d] = v ? g_reco * (o[1 + d] - xr[d]) : 0.f;
    if (lane == 0) {
      conf_out[r] = conf;
      const float t = o[0];
      g[0] = g_trav * wgt * (t - y[r]) * t * (1.f - t);  // through the sigmoid
      s_trav += static_cast<double>(raw[r] * wgt);
    }
  }
  // local sum of the confidence-weighted traversability errors rides at the end of the flat
  // gradient buffer, so the one gradient all-reduce of a data-parallel run also carries it
  if (lane == 0 && s_trav != 0.0) atomicAdd(trav_w_sum, static_cast<float>(s_trav));
}

__global__ void loss_finalize_kernel(TrainScalars* sc, const float* trav_w_sum, LossCfg cfg, long long n_total) {
  const double n = sc->n_valid;
  sc->loss_reco = static_cast<float>(sc->sum_lr / n);
  sc->loss_trav_conf = static_cast<float>(static_cast<double>(*trav_w_sum) / static_cast<double>(n_total));
  sc->loss_trav = static_cast<float>(sc->sum_raw / static_cast<double>(n_total));
  sc->loss_total = cfg.w_trav * sc->loss_trav_conf + cfg.w_reco * sc->loss_reco;  // + w_temp * 0
}

// column sums (bias gradients): grid (ceil(N/128), row_slices)
__global__ void __launch_bounds__(128)
colsum_kernel(const float* __restrict__ a, long long lda, int rows, int cols, float* __restrict__ out) {
  const int c = blockIdx.x * 128 + threadIdx.x;
  if (c >= cols) return;
  const int per = (rows + gridDim.y - 1) / gridDim.y;
  const int r0 = blockIdx.y * per, r1 = min(rows, r0 + per);
  float s = 0.f;
  for (int r = r0; r < r1; ++r) s += a[r * lda + c];
  atomicAdd(&out[c], s);
}

__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
            long long n, AdamCfg cfg, const long long* __restrict__ step_ptr) {
  // torch.optim.Adam (no amsgrad, no weight decay): step t counts from 1
  const double t = static_cast<double>(*step_ptr);
  const float bc1 = static_cast<float>(1.0 - pow(static_cast<double>(cfg.beta1), t));
  const float bc2_sqrt = static_cast<float>(sqrt(1.0 - pow(static_cast<double>(cfg.beta2), t)));
  const float step_size = cfg.lr / bc1;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float gi = g[i];
    const float mi = m[i] + (gi - m[i]) * (1.f - cfg.beta1);      // lerp form used by torch
    const float vi = v[i] * cfg.beta2 + (1.f - cfg.beta2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    const float denom = sqrtf(vi) / bc2_sqrt + cfg.eps;
    p[i] -= step_size * (mi / denom);
  }
}

__global__ void bump_step_kernel(long long* step) { *step += 1; }

}  // namespace

size_t mlp_param_count(const MlpShape& s) {
  return static_cast<size_t>(s.h1) * s.dim + s.h1 + static_cast<size_t>(s.h2) * s.h1 + s.h2 +
         static_cast<size_t>(s.dim + 1) * s.h2 + (s.dim + 1);
}

MlpOffsets mlp_offsets(const MlpShape& s) {
  MlpOffsets o;
  o.w1 = 0;
  o.b1 = o.w1 + static_cast<size_t>(s.h1) * s.dim;
  o.w2 = o.b1 + s.h1;
  o.b2 = o.w2 + static_cast<size_t>(s.h2) * s.h1;
  o.w3 = o.b2 + s.h2;
  o.b3 = o.w3 + static_cast<size_t>(s.dim + 1) * s.h2;
  o.total = o.b3 + (s.dim + 1);
  return o;
}

size_t mlp_train_workspace_floats(const MlpShape& s, int max_rows) {
  const size_t R = static_cast<size_t>(max_rows);
  // h1, h2, out, d_out, d_h2, d_h1, loss_reco, raw
  return R * s.h1 * 2 + R * s.h2 * 2 + R * (s.dim + 1) * 2 + R * 2;
}

namespace {
struct Ws {
  float *h1, *h2, *out, *d_out, *d_h2, *d_h1, *loss_reco, *raw;
};
Ws carve(float* ws, const MlpShape& s, int max_rows) {
  const size_t R = static_cast<size_t>(max_rows);
  Ws w;
  w.h1 = ws;
  w.h2 = w.h1 + R * s.h1;
  w.out = w.h2 + R * s.h2;
  w.d_out = w.out + R * (s.dim + 1);
  w.d_h2 = w.d_out + R * (s.dim + 1);
  w.d_h1 = w.d_h2 + R * s.h2;
  w.loss_reco = w.d_h1 + R * s.h1;
  w.raw = w.loss_reco + R;
  return w;
}
}  // namespace

int mlp_forward_f32(const MlpShape& s, const float* params, const float* x, int rows, float* h1, float* h2, float* out,
                    cudaStream_t stream) {
  const MlpOffsets o = mlp_offsets(s);
  SgemmArgs g{};
  g.A = x; g.sam = s.dim; g.sak = 1; g.B = params + o.w1; g.sbk = 1; g.sbn = s.dim; g.C = h1; g.ldc = s.h1;
  g.M = rows; g.N = s.h1; g.K = s.dim; g.bias = params + o.b1; g.act = SACT_RELU; g.relu_mask = nullptr; g.ld_mask = 0;
  WVN_PROPAGATE(sgemm(g, 1, stream));
  g.A = h1; g.sam = s.h1; g.B = params + o.w2; g.sbn = s.h1; g.C = h2; g.ldc = s.h2; g.N = s.h2; g.K = s.h1;
  g.bias = params + o.b2;
  WVN_PROPAGATE(sgemm(g, 1, stream));
  g.A = h2; g.sam = s.h2; g.B = params + o.w3; g.sbn = s.h2; g.C = out; g.ldc = s.dim + 1; g.N = s.dim + 1; g.K = s.h2;
  g.bias = params + o.b3; g.act = SACT_SIGMOID_COL0;
  WVN_PROPAGATE(sgemm(g, 1, stream));
  return WVN_OK;
}

int mlp_train_forward_stats(const MlpShape& s, const float* params, const float* x, const float* y,
                            const unsigned char* y_valid, int rows, int max_rows, float* workspace,
                            TrainScalars* scalars, cudaStream_t stream) {
  WVN_REQUIRE(rows > 0 && rows <= max_rows, "train: rows=%d outside (0, %d]", rows, max_rows);
  Ws w = carve(workspace, s, max_rows);
  WVN_CHECK_CUDA(cudaMemsetAsync(scalars, 0, sizeof(TrainScalars), stream));
  WVN_PROPAGATE(mlp_forward_f32(s, params, x, rows, w.h1, w.h2, w.out, stream));
  int blocks = (rows * 32 + 255) / 256;
  if (blocks > sm_count() * 4) blocks = sm_count() * 4;
  loss_rows_kernel<<<blocks, 256, 0, stream>>>(w.out, x, y, y_valid, w.loss_reco, w.raw, scalars, rows, s.dim);
  WVN_CHECK_LAUNCH("loss_rows_kernel");
  return WVN_OK;
}

int mlp_train_backward(const MlpShape& s, const float* params, const float* x, const float* y,
                       const unsigned char* y_valid, int rows, int max_rows, long long n_total, const LossCfg& cfg,
                       float* workspace, TrainScalars* scalars, float* cg_mean, float* cg_std, float* grads,
                       float* conf_out, cudaStream_t stream) {
  WVN_REQUIRE(rows > 0 && rows <= max_rows, "train: rows=%d outside (0, %d]", rows, max_rows);
  Ws w = carve(workspace, s, max_rows);
  const MlpOffsets o = mlp_offsets(s);
  confidence_update_kernel<<<1, 1, 0, stream>>>(scalars, cg_mean, cg_std, nullptr);
  WVN_CHECK_LAUNCH("confidence_update_kernel");
  int blocks = (rows * 32 + 255) / 256;
  if (blocks > sm_count() * 4) blocks = sm_count() * 4;
  WVN_CHECK_CUDA(cudaMemsetAsync(grads, 0, sizeof(float) * (o.total + 1), stream));
  loss_grad_kernel<<<blocks, 256, 0, stream>>>(w.out, x, y, y_valid, w.loss_reco, w.raw, w.d_out, conf_out, scalars,
                                               grads + o.total, cfg, rows, s.dim, n_total);
  WVN_CHECK_LAUNCH("loss_grad_kernel");

  const int nout = s.dim + 1;
  const int splits = rows >= 512 ? 16 : (rows >= 128 ? 4 : 1);
  SgemmArgs g{};
  // dW3[nout, h2] = dOut^T · H2
  g.A = w.d_out; g.sam = 1; g.sak = nout; g.B = w.h2; g.sbk = s.h2; g.sbn = 1; g.C = grads + o.w3; g.ldc = s.h2;
  g.M = nout; g.N = s.h2; g.K = rows; g.bias = nullptr; g.act = SACT_NONE; g.relu_mask = nullptr; g.ld_mask = 0;
  WVN_PROPAGATE(sgemm(g, splits, stream));
  colsum_kernel<<<dim3((nout + 127) / 128, 16), 128, 0, stream>>>(w.d_out, nout, rows, nout, grads + o.b3);
  WVN_CHECK_LAUNCH("colsum_kernel");
  // dH2[rows, h2] = (dOut · W3) * (H2 > 0)
  g.A = w.d_out; g.sam = nout; g.sak = 1; g.B = params + o.w3; g.sbk = s.h2; g.sbn = 1; g.C = w.d_h2; g.ldc = s.h2;
  g.M = rows; g.N = s.h2; g.K = nout; g.relu_mask = w.h2; g.ld_mask = s.h2;
  WVN_PROPAGATE(sgemm(g, 1, stream));
  // dW2[h2, h1] = dH2^T · H1
  g.A = w.d_h2; g.sam = 1; g.sak = s.h2; g.B = w.h1; g.sbk = s.h1; g.sbn = 1; g.C = grads + o.w2; g.ldc = s.h1;
  g.M = s.h2; g.N = s.h1; g.K = rows; g.relu_mask = nullptr; g.ld_mask = 0;
  WVN_PROPAGATE(sgemm(g, splits, stream));
  colsum_kernel<<<dim3((s.h2 + 127) / 128, 16), 128, 0, stream>>>(w.d_h2, s.h2, rows, s.h2, grads + o.b2);
  WVN_CHECK_LAUNCH("colsum_kernel");
  // dH1[rows, h1] = (dH2 · W2) * (H1 > 0)
  g.A = w.d_h2; g.sam = s.h2; g.sak = 1; g.B = params + o.w2; g.sbk = s.h1; g.sbn = 1; g.C = w.d_h1; g.ldc = s.h1;
  g.M = rows; g.N = s.h1; g.K = s.h2; g.relu_mask = w.h1; g.ld_mask = s.h1;
  WVN_PROPAGATE(sgemm(g, 1, stream));
  // dW1[h1, dim] = dH1^T · X
  g.A = w.d_h1; g.sam = 1; g.sak = s.h1; g.B = x; g.sbk = s.dim; g.sbn = 1; g.C = grads + o.w1; g.ldc = s.dim;
  g.M = s.h1; g.N = s.dim; g.K = rows; g.relu_mask = nullptr; g.ld_mask = 0;
  WVN_PROPAGATE(sgemm(g, splits, stream));
  colsum_kernel<<<dim3((s.h1 + 127) / 128, 16), 128, 0, stream>>>(w.d_h1, s.h1, rows, s.h1, grads + o.b1);
  WVN_CHECK_LAUNCH("colsum_kernel");
  return WVN_OK;
}

int mlp_train_finalize(TrainScalars* scalars, const float* grads, long long n_params, long long n_total,
                       const LossCfg& cfg, cudaStream_t stream) {
  loss_finalize_kernel<<<1, 1, 0, stream>>>(scalars, grads + n_params, cfg, n_total);
  WVN_CHECK_LAUNCH("loss_finalize_kernel");
  return WVN_OK;
}

int mlp_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n,
                  const AdamCfg& cfg, long long* step_counter, cudaStream_t stream) {
  bump_step_kernel<<<1, 1, 0, stream>>>(step_counter);
  WVN_CHECK_LAUNCH("bump_step_kernel");
  int blocks = static_cast<int>((n + 255) / 256);
  if (blocks > sm_count() * 4) blocks = sm_count() * 4;
  adam_kernel<<<blocks, 256, 0, stream>>>(params, grads, exp_avg, exp_avg_sq, n, cfg, step_counter);
  WVN_CHECK_LAUNCH("adam_kernel");
  return WVN_OK;
}

}  // namespace wvn
