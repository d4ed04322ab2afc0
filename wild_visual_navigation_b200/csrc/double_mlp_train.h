// wvn-b200: internal interface of the DoubleMLP learner's fp32 kernels (double_mlp_train.cu): the row forward and the
// online train step.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>

#include "mlp_train.h"
#include "train_core.h"

namespace wvn {

// DoubleMLP(input_size = dim, hidden_sizes = [h1, h2, 1]): two networks read the same rows,
//   networks.0: Linear(dim, h1) ReLU Linear(h1, h2) ReLU Linear(h2, 1)     -> sigmoid: traversability
//   networks.1: Linear(dim, h1) ReLU Linear(h1, h2) ReLU Linear(h2, dim)   -> reconstruction
// and the output is cat([sigmoid(net0(x)), net1(x)], 1): the (rows, 1 + dim) layout of SimpleMLP.
// The flat fp32 parameter buffer is in parameters() order: networks.0.{0,2,4}.{weight,bias}, then networks.1's.
struct DoubleOffsets {
  size_t w1[2], b1[2], w2[2], b2[2], w3[2], b3[2], total;
};
DoubleOffsets double_mlp_offsets(const MlpShape& s);
size_t double_mlp_param_count(const MlpShape& s);
// The shapes the kernels take: 1 <= dim <= 1024, 4 <= h1 <= 256 with h1 % 4 == 0, 1 <= h2 <= 32 (WVN_ERR_INVALID else).
int double_mlp_check_shape(const MlpShape& s, const char* who);

// DoubleMLP.forward on x [rows, dim]: a1 [2][rows, h1], a2 [2][rows, h2] (net 0's block, then net 1's) and
// out [rows, 1 + dim].  Three launches.
int double_mlp_forward_f32(const MlpShape& s, const float* params, const float* x, int rows, float* a1, float* a2,
                           float* out, cudaStream_t stream);

// grads_ext: caller-owned device buffer of double_mlp_param_count floats, or NULL (the trainer allocates it).
// The statistics block has 9 doubles: the kStatDoubles of train_core.h (sum and sum of squares of loss_reco over the
// labelled rows, sum of (trav - y)^2, labelled and live row counts, 0, loss_reco's min and max), then the
// confidence-weighted traversability error summed over the live rows (written by phase 2, all-reduced with the gradient).
int double_trainer_create(const MlpShape& s, int max_rows, const LossCfg& loss, const AdamCfg& adam, float* grads_ext,
                          Trainer** out);
// One TraversabilityEstimator.train() body on rows padded per group: x [groups, rows_per_group, dim] with n_rows[g]
// (device int32; NULL: all) live rows in group g; y / y_valid (uint8) / conf_out are indexed by the compacted row number.
// The live rows are gathered first, and every later launch is bounded by their device count, so padding (NaN included)
// is never read.  phase_mask: 1 = forward, per-row losses, the statistic sums (+ their all-reduce); 2 = generator update
// from the global sums, dLoss/dOut with the global row counts, backward, weight gradients (+ the gradient all-reduce);
// 4 = loss metrics from the global sums + Adam; 7 = the whole step.  metrics [6] (may be NULL): loss_total, loss_trav,
// loss_reco, loss_trav_conf, cg_mean, cg_std.
int double_train_step_padded(Trainer* t, float* params, float* exp_avg, float* exp_avg_sq,
                             long long* step_counter, const float* x, int groups, int rows_per_group,
                             const int* n_rows, const float* y, const unsigned char* y_valid, float* cg_mean,
                             float* cg_std, float* conf_out, float* metrics, int phase_mask, cudaStream_t stream);

}  // namespace wvn
