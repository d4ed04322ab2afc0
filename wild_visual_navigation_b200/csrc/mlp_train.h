// wvn-b200: internal interface of the fp32 online-learning kernels (mlp_train.cu).
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>

namespace wvn {

struct MlpShape {
  int dim = 384;  // input features D; output is 1 + D (traversability + reconstruction)
  int h1 = 256;
  int h2 = 32;
};

// Offsets into the flat fp32 parameter / gradient / Adam-moment buffers, in the reference's
// state_dict order: layers.0.weight, layers.0.bias, layers.2.weight, layers.2.bias,
// layers.4.weight, layers.4.bias (model/simple_mlp.py:24-30).
struct MlpOffsets {
  size_t w1, b1, w2, b2, w3, b3, total;
};

struct LossCfg {
  float w_trav = 0.03f;
  float w_reco = 0.5f;
  float std_factor = 0.5f;
  int anomaly_balanced = 1;
};

// Device-resident scalars of one step.  The five leading doubles are plain sums so a
// data-parallel caller can all-reduce them in one call between the phases.
struct TrainScalars {
  double sum_lr;      // sum of loss_reco over valid rows
  double sum_lr2;     // sum of loss_reco^2 over valid rows
  double sum_raw;     // sum of (trav - y)^2 over all rows
  double n_valid;     // number of valid rows
  double reserved;
  float mean, std;    // ConfidenceGenerator state after the update
  float loss_total, loss_trav, loss_reco, loss_trav_conf;
};

size_t mlp_param_count(const MlpShape& s);
MlpOffsets mlp_offsets(const MlpShape& s);
size_t mlp_train_workspace_floats(const MlpShape& s, int max_rows);

int mlp_forward_f32(const MlpShape& s, const float* params, const float* x, int rows, float* h1, float* h2, float* out,
                    cudaStream_t stream);
// phase 1: forward + per-row losses + local statistic sums (scalars zeroed first)
int mlp_train_forward_stats(const MlpShape& s, const float* params, const float* x, const float* y,
                            const unsigned char* y_valid, int rows, int max_rows, float* workspace,
                            TrainScalars* scalars, cudaStream_t stream);
// phase 2: confidence update (from the — possibly all-reduced — sums), dLoss/dOut, backward.
// grads has total+1 floats: the last one is the local sum of confidence-weighted trav errors.
int mlp_train_backward(const MlpShape& s, const float* params, const float* x, const float* y,
                       const unsigned char* y_valid, int rows, int max_rows, long long n_total, const LossCfg& cfg,
                       float* workspace, TrainScalars* scalars, float* cg_mean, float* cg_std, float* grads,
                       float* conf_out, cudaStream_t stream);
// phase 3: loss metrics from the (possibly all-reduced) sums; then Adam (mlp_adam_step, train_core.h).
int mlp_train_finalize(TrainScalars* scalars, const float* grads, long long n_params, long long n_total,
                       const LossCfg& cfg, cudaStream_t stream);

}  // namespace wvn
