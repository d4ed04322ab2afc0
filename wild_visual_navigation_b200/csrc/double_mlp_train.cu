// wvn-b200: the DoubleMLP learner (model/simple_mlp.py DoubleMLP) in fp32 — the row forward and the online train step,
// the body of TraversabilityEstimator.train() (traversability_estimator.py:464-477) with TraversabilityLoss
// (utils/loss.py:93-160) on a DoubleMLP.
//
// Two networks read the same rows: net 0 (dim -> h1 -> h2 -> 1, sigmoid) gives traversability, net 1 (dim -> h1 -> h2
// -> dim) the reconstruction; out = [sigmoid(net0(x)) | net1(x)] has SimpleMLP's (rows, 1 + dim) layout, so the loss,
// its gradient and the confidence are SimpleMLP's.  The step is one fixed sequence of 15 launches with every scalar on
// the device (no host synchronisation), in three phases with a data-parallel exchange after the first two:
//   1: compaction of the padded rows (train_core) -> gather of the live rows -> forward: 3 batched GEMMs of two problems
//      each (one per net; bias + ReLU, then layer 3 writes column 0 through the sigmoid and columns 1..dim) -> per-row
//      loss terms -> this rank's statistic sums and loss_reco's extrema      [SUM of the sums, MIN / MAX of the extrema]
//   2: generator update (train_core.cuh) -> dLoss/dOut with the global row counts and per-row confidence -> 2 batched
//      data-gradient GEMMs (ReLU backward) -> ONE six-problem launch of every weight and bias gradient -> this rank's
//      confidence-weighted traversability error                             [SUM of the gradient and that error]
//   4: loss metrics from the global sums -> Adam (mlp_adam_step).
// Every launch after the compaction is bounded by the device count of live rows, so a padded batch and the same rows
// compacted run the same arithmetic.
// Training batches are small (~8 nodes x ~100 segments), so the step is latency-bound: the GEMMs are the training core's
// fp32 CUDA-core tiles, every output element and every sum is formed by one thread (or one fixed reduction tree) in a
// fixed order, with no atomics: two runs of the same step are bit-identical.
#include <stddef.h>
#include <string.h>

#include <algorithm>

#include "common.cuh"
#include "double_mlp_train.h"
#include "host_common.h"
#include "recon_loss.cuh"
#include "train_core.cuh"

namespace wvn {

// ------------------------------------------------------------------------------------------------ host side
DoubleOffsets double_mlp_offsets(const MlpShape& s) {
  const size_t D = s.dim, h1 = s.h1, h2 = s.h2;
  DoubleOffsets o;
  size_t off = 0;
  for (int k = 0; k < 2; ++k) {
    const size_t last = k == 0 ? 1 : D;
    o.w1[k] = off; off += h1 * D;
    o.b1[k] = off; off += h1;
    o.w2[k] = off; off += h2 * h1;
    o.b2[k] = off; off += h2;
    o.w3[k] = off; off += last * h2;
    o.b3[k] = off; off += last;
  }
  o.total = off;
  return o;
}

size_t double_mlp_param_count(const MlpShape& s) { return double_mlp_offsets(s).total; }

int double_mlp_check_shape(const MlpShape& s, const char* who) {
  WVN_REQUIRE(s.dim >= 1 && s.dim <= 1024 && s.h1 >= 4 && s.h1 <= 256 && s.h1 % 4 == 0 && s.h2 >= 1 && s.h2 <= 32,
              "%s: DoubleMLP(%d, [%d, %d, 1]) outside the kernels' range (1 <= dim <= 1024, 4 <= h1 <= 256 and a "
              "multiple of 4, 1 <= h2 <= 32)", who, s.dim, s.h1, s.h2);
  return WVN_OK;
}

namespace {

// The three forward launches; a1 / a2 hold net 0's block, then net 1's, `pitch` rows apart.  n_live (device, may be
// NULL): only the first *n_live of the `rows` rows are computed.
int forward_gemms(const MlpShape& s, const DoubleOffsets& o, const float* params, const float* x, int rows, long long pitch,
                  float* a1, float* a2, float* out, const int* n_live, cudaStream_t stream) {
  const int D = s.dim, h1 = s.h1, h2 = s.h2, live = n_live ? 1 : 0;
  GemmProblem ps[2];
  for (int k = 0; k < 2; ++k) {   // a1_k = ReLU(x W1_k^T + b1_k)
    ps[k] = gemm_problem(x, D, 1, params + o.w1[k], 1, D, a1 + k * pitch * h1, h1, rows, h1, D, live);
    ps[k].bias = params + o.b1[k]; ps[k].act = F32_RELU_FMAX;
  }
  WVN_PROPAGATE(launch_gemms(ps, 2, n_live, stream));
  for (int k = 0; k < 2; ++k) {   // a2_k = ReLU(a1_k W2_k^T + b2_k)
    ps[k] = gemm_problem(a1 + k * pitch * h1, h1, 1, params + o.w2[k], 1, h1, a2 + k * pitch * h2, h2, rows, h2, h1,
                         live);
    ps[k].bias = params + o.b2[k]; ps[k].act = F32_RELU_FMAX;
  }
  WVN_PROPAGATE(launch_gemms(ps, 2, n_live, stream));
  // column 0 = sigmoid(a2_0 w3_0 + b3_0), columns 1..dim = a2_1 W3_1^T + b3_1
  ps[0] = gemm_problem(a2, h2, 1, params + o.w3[0], 1, h2, out, D + 1, rows, 1, h2, live);
  ps[0].bias = params + o.b3[0]; ps[0].act = F32_SIGMOID_COL0;
  ps[1] = gemm_problem(a2 + pitch * h2, h2, 1, params + o.w3[1], 1, h2, out + 1, D + 1, rows, D, h2, live);
  ps[1].bias = params + o.b3[1];
  return launch_gemms(ps, 2, n_live, stream);
}

}  // namespace

int double_mlp_forward_f32(const MlpShape& s, const float* params, const float* x, int rows, float* a1, float* a2,
                           float* out, cudaStream_t stream) {
  WVN_PROPAGATE(double_mlp_check_shape(s, "double mlp forward"));
  WVN_REQUIRE(params && x && a1 && a2 && out && rows > 0, "double mlp forward: bad argument");
  return forward_gemms(s, double_mlp_offsets(s), params, x, rows, rows, a1, a2, out, nullptr, stream);
}

struct DoubleTrainer : Trainer {
  DoubleTrainer() : Trainer(TRAINER_DOUBLE_MLP) {}
  MlpShape s;
  DoubleOffsets o;
  DoubleScalars* sc = nullptr;
  int* comp = nullptr;     // compacted -> padded row map
  int* n_live = nullptr;   // this rank's live rows (device)
  float *xg = nullptr, *a1 = nullptr, *a2 = nullptr, *out = nullptr, *d_out = nullptr, *d2 = nullptr, *d1 = nullptr;
  float *loss_reco = nullptr, *raw = nullptr, *wraw = nullptr;
};

int double_trainer_create(const MlpShape& s, int max_rows, const LossCfg& loss, const AdamCfg& adam, float* grads_ext,
                          Trainer** out) {
  WVN_REQUIRE(out && max_rows > 0, "double mlp trainer: bad arguments");
  WVN_PROPAGATE(double_mlp_check_shape(s, "double mlp trainer"));
  DoubleTrainer* t = new DoubleTrainer();
  t->s = s; t->o = double_mlp_offsets(s); t->loss = loss; t->adam = adam;
  t->max_rows = max_rows;
  const size_t R = max_rows, D = s.dim, h1 = s.h1, h2 = s.h2;
  // a1 / d1 / a2 / d2 hold both nets, the second R rows after the first
  const int rc = trainer_alloc(t, [&](Carver& a) {
    t->sc = a.take<DoubleScalars>(1);
    t->n_live = a.take<int>(1);
    t->comp = a.take<int>(R);
    t->xg = a.take<float>(R * D);
    t->a1 = a.take<float>(2 * R * h1);
    t->d1 = a.take<float>(2 * R * h1);
    t->a2 = a.take<float>(2 * R * h2);
    t->d2 = a.take<float>(2 * R * h2);
    t->out = a.take<float>(R * (D + 1));
    t->d_out = a.take<float>(R * (D + 1));
    t->loss_reco = a.take<float>(R);
    t->raw = a.take<float>(R);
    t->wraw = a.take<float>(R);
    t->grads = grads_ext ? grads_ext : a.take<float>(t->o.total);
  }, "double mlp trainer");
  if (rc != WVN_OK) {
    delete t;
    return rc;
  }
  t->stats = &t->sc->sum_lr;
  t->n_stats = kStatDoubles + 1;
  *out = t;
  return WVN_OK;
}

int double_train_step_padded(Trainer* base, float* params, float* exp_avg, float* exp_avg_sq,
                             long long* step_counter, const float* x, int groups, int rows_per_group,
                             const int* n_rows, const float* y, const unsigned char* y_valid, float* cg_mean,
                             float* cg_std, float* conf_out, float* metrics, int phase_mask, cudaStream_t stream) {
  WVN_PROPAGATE(trainer_check(base, TRAINER_DOUBLE_MLP, "double mlp train step"));
  DoubleTrainer* t = static_cast<DoubleTrainer*>(base);
  WVN_REQUIRE(params && exp_avg && exp_avg_sq && step_counter && x && y && y_valid && conf_out,
              "double mlp train step: null argument");
  const long long cap = static_cast<long long>(groups) * rows_per_group;
  WVN_REQUIRE(groups > 0 && rows_per_group > 0 && cap <= t->max_rows,
              "double mlp train step: %d x %d rows outside (0, %d]", groups, rows_per_group, t->max_rows);
  const MlpShape& s = t->s;
  const DoubleOffsets& o = t->o;
  const int D = s.dim, h1 = s.h1, h2 = s.h2, n3 = D + 1, rows = static_cast<int>(cap);
  const long long R = t->max_rows;   // the per-net blocks of a1 / a2 / d1 / d2 are max_rows rows apart
  const int row_blocks = (rows * 32 + kRowThreads - 1) / kRowThreads;
  // every row loop, GEMM and reduction below is bounded by the device count *n_live: padding rows are never read
  if (phase_mask & 1) {   // live rows -> forward -> per-row loss terms -> this rank's statistic sums (-> all-reduce)
    WVN_PROPAGATE(compact_rows(groups, rows_per_group, n_rows, nullptr, t->comp, t->n_live, stream));
    double_gather_kernel<<<row_blocks, kRowThreads, 0, stream>>>(x, t->comp, t->n_live, D, t->xg);
    WVN_CHECK_LAUNCH("double_gather_kernel");
    WVN_PROPAGATE(forward_gemms(s, o, params, t->xg, rows, R, t->a1, t->a2, t->out, t->n_live, stream));
    double_loss_rows_kernel<<<row_blocks, kRowThreads, 0, stream>>>(t->out, t->xg, y, t->loss_reco, t->raw, t->n_live, D);
    WVN_CHECK_LAUNCH("double_loss_rows_kernel");
    double_stats_kernel<<<1, kStatThreads, 0, stream>>>(t->loss_reco, t->raw, y_valid, t->n_live, t->sc);
    WVN_CHECK_LAUNCH("double_stats_kernel");
    WVN_PROPAGATE(trainer_comm_stats(&t->comm, &t->sc->sum_lr, t->conf.cs.method == CONF_MOVING_AVERAGE, stream));
  }
  if (phase_mask & 2) {   // generator update -> dLoss/dOut + confidence -> backward -> gradients (-> all-reduce)
    double_conf_kernel<<<1, 32, 0, stream>>>(D, t->loss, t->conf.cs, cg_mean, cg_std, t->sc);
    WVN_CHECK_LAUNCH("double_conf_kernel");
    double_dout_kernel<<<row_blocks, kRowThreads, 0, stream>>>(t->out, t->xg, y, y_valid, t->loss_reco, t->raw, t->sc,
                                                               t->loss, t->conf.cs.method, t->d_out, conf_out, t->wraw,
                                                               t->n_live, D);
    WVN_CHECK_LAUNCH("double_dout_kernel");
    // data gradients: d2_k = (dOut_k W3_k) * (a2_k > 0), d1_k = (d2_k W2_k) * (a1_k > 0)
    GemmProblem ps[2];
    ps[0] = gemm_problem(t->d_out, n3, 1, params + o.w3[0], h2, 1, t->d2, h2, rows, h2, 1, 1);
    ps[1] = gemm_problem(t->d_out + 1, n3, 1, params + o.w3[1], h2, 1, t->d2 + R * h2, h2, rows, h2, D, 1);
    for (int k = 0; k < 2; ++k) { ps[k].ref = t->a2 + k * R * h2; ps[k].ld_ref = h2; }
    WVN_PROPAGATE(launch_gemms(ps, 2, t->n_live, stream));
    for (int k = 0; k < 2; ++k) {
      ps[k] = gemm_problem(t->d2 + k * R * h2, h2, 1, params + o.w2[k], h1, 1, t->d1 + k * R * h1, h1, rows, h1, h2, 1);
      ps[k].ref = t->a1 + k * R * h1; ps[k].ld_ref = h1;
    }
    WVN_PROPAGATE(launch_gemms(ps, 2, t->n_live, stream));
    // every weight gradient dW = dZ^T A and bias gradient db = column sums of dZ: one launch of six problems, the row
    // reduction (K) bounded by *n_live (a rank without live rows contributes zeros)
    GemmProblem wg[6];
    wg[0] = gemm_problem(t->d_out, 1, n3, t->a2, h2, 1, t->grads + o.w3[0], h2, 1, h2, rows, 2);
    wg[0].db = t->grads + o.b3[0];
    wg[1] = gemm_problem(t->d_out + 1, 1, n3, t->a2 + R * h2, h2, 1, t->grads + o.w3[1], h2, D, h2, rows, 2);
    wg[1].db = t->grads + o.b3[1];
    for (int k = 0; k < 2; ++k) {
      wg[2 + k] = gemm_problem(t->d2 + k * R * h2, 1, h2, t->a1 + k * R * h1, h1, 1, t->grads + o.w2[k], h1, h2, h1, rows,
                               2);
      wg[2 + k].db = t->grads + o.b2[k];
      wg[4 + k] = gemm_problem(t->d1 + k * R * h1, 1, h1, t->xg, D, 1, t->grads + o.w1[k], D, h1, D, rows, 2);
      wg[4 + k].db = t->grads + o.b1[k];
    }
    WVN_PROPAGATE(launch_gemms(wg, 6, t->n_live, stream));
    double_trav_w_kernel<<<1, kStatThreads, 0, stream>>>(t->wraw, t->n_live, t->sc);
    WVN_CHECK_LAUNCH("double_trav_w_kernel");
    WVN_PROPAGATE(trainer_comm_sum(&t->comm, t->grads, o.total, false, stream));
    WVN_PROPAGATE(trainer_comm_sum(&t->comm, &t->sc->trav_w, 1, true, stream));
  }
  if (phase_mask & 4) {   // loss metrics from the global sums, then Adam
    if (metrics) {
      double_finish_kernel<<<1, 32, 0, stream>>>(t->loss, t->sc, metrics);
      WVN_CHECK_LAUNCH("double_finish_kernel");
    }
    WVN_PROPAGATE(mlp_adam_step(params, t->grads, exp_avg, exp_avg_sq, static_cast<long long>(o.total), t->adam,
                                step_counter, stream));
  }
  return WVN_OK;
}

}  // namespace wvn
