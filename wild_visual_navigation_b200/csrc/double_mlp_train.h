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

struct DoubleTrainer;
// grads_ext: caller-owned device buffer of double_mlp_param_count floats, or NULL (the trainer allocates it).
int double_trainer_create(const MlpShape& s, int max_rows, const LossCfg& loss, const AdamCfg& adam, float* grads_ext,
                          DoubleTrainer** out);
void double_trainer_destroy(DoubleTrainer* t);
// The trainer's ConfidenceGenerator (bound and copied with trainer_conf_bind / trainer_conf_copy).
TrainerConf* double_trainer_conf(DoubleTrainer* t);
// One TraversabilityEstimator.train() body on x [rows, dim], y [rows], y_valid [rows] (uint8): forward,
// TraversabilityLoss with the generator update, backward, Adam.  conf_out [rows]; metrics [6] (may be NULL):
// loss_total, loss_trav, loss_reco, loss_trav_conf, cg_mean, cg_std.
int double_train_step(DoubleTrainer* t, float* params, float* exp_avg, float* exp_avg_sq, long long* step_counter,
                      const float* x, int rows, const float* y, const unsigned char* y_valid, float* cg_mean,
                      float* cg_std, float* conf_out, float* metrics, cudaStream_t stream);

}  // namespace wvn
