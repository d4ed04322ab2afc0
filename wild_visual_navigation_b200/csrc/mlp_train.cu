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
#include "train_core.h"

namespace wvn {

namespace {

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
  GemmProblem g = gemm_problem(x, s.dim, 1, params + o.w1, 1, s.dim, h1, s.h1, rows, s.h1, s.dim);
  g.bias = params + o.b1; g.act = F32_RELU_FMAX;
  WVN_PROPAGATE(launch_gemms(&g, 1, nullptr, stream));
  g = gemm_problem(h1, s.h1, 1, params + o.w2, 1, s.h1, h2, s.h2, rows, s.h2, s.h1);
  g.bias = params + o.b2; g.act = F32_RELU_FMAX;
  WVN_PROPAGATE(launch_gemms(&g, 1, nullptr, stream));
  g = gemm_problem(h2, s.h2, 1, params + o.w3, 1, s.h2, out, s.dim + 1, rows, s.dim + 1, s.h2);
  g.bias = params + o.b3; g.act = F32_SIGMOID_COL0;
  WVN_PROPAGATE(launch_gemms(&g, 1, nullptr, stream));
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
  // dW3[nout, h2] = dOut^T · H2
  GemmProblem g = gemm_problem(w.d_out, 1, nout, w.h2, s.h2, 1, grads + o.w3, s.h2, nout, s.h2, rows);
  WVN_PROPAGATE(launch_gemms(&g, 1, nullptr, stream, splits));
  colsum_kernel<<<dim3((nout + 127) / 128, 16), 128, 0, stream>>>(w.d_out, nout, rows, nout, grads + o.b3);
  WVN_CHECK_LAUNCH("colsum_kernel");
  // dH2[rows, h2] = (dOut · W3) * (H2 > 0)
  g = gemm_problem(w.d_out, nout, 1, params + o.w3, s.h2, 1, w.d_h2, s.h2, rows, s.h2, nout);
  g.ref = w.h2; g.ld_ref = s.h2;
  WVN_PROPAGATE(launch_gemms(&g, 1, nullptr, stream));
  // dW2[h2, h1] = dH2^T · H1
  g = gemm_problem(w.d_h2, 1, s.h2, w.h1, s.h1, 1, grads + o.w2, s.h1, s.h2, s.h1, rows);
  WVN_PROPAGATE(launch_gemms(&g, 1, nullptr, stream, splits));
  colsum_kernel<<<dim3((s.h2 + 127) / 128, 16), 128, 0, stream>>>(w.d_h2, s.h2, rows, s.h2, grads + o.b2);
  WVN_CHECK_LAUNCH("colsum_kernel");
  // dH1[rows, h1] = (dH2 · W2) * (H1 > 0)
  g = gemm_problem(w.d_h2, s.h2, 1, params + o.w2, s.h1, 1, w.d_h1, s.h1, rows, s.h1, s.h2);
  g.ref = w.h1; g.ld_ref = s.h1;
  WVN_PROPAGATE(launch_gemms(&g, 1, nullptr, stream));
  // dW1[h1, dim] = dH1^T · X
  g = gemm_problem(w.d_h1, 1, s.h1, x, s.dim, 1, grads + o.w1, s.dim, s.h1, s.dim, rows);
  WVN_PROPAGATE(launch_gemms(&g, 1, nullptr, stream, splits));
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

}  // namespace wvn
