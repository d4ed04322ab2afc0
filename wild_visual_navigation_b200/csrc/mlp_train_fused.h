// wvn-b200: internal interface of the fused online train step (mlp_train_fused.cu).
#pragma once

#include <cuda_runtime.h>

#include "mlp_train.h"
#include "train_core.h"

namespace wvn {

// Device-resident scalars of one step.  The six leading doubles are plain sums (incl. the row count), so a
// data-parallel step all-reduces them in ONE call between the forward and the backward kernels.
struct FusedScalars {
  double sum_lr;    // sum of loss_reco over valid rows
  double sum_lr2;   // sum of loss_reco^2 over valid rows
  double sum_raw;   // sum of (trav - y)^2 over all live rows
  double n_valid;   // number of valid (labelled) rows
  double n_rows;    // number of live rows (the loss' N; global after the all-reduce)
  double reserved;
  // extrema of loss_reco over the live rows (moving_average's min-max normalisation): all-reduced with MIN / MAX.
  // x_min is reset to +inf / x_max to 0 by the step's last kernel, not by the step's memset.
  double x_min, x_max;
  float mean, std;  // ConfidenceGenerator state after the update
  float loss_total, loss_trav, loss_reco, loss_trav_conf;
  // what the row kernels need of the updated generator: latest_measurement / running_mean: the interval [lo, hi];
  // kalman_filter: mean and 1 / (std * std_factor) in lo / hi; moving_average: the clip interval and the clipped extrema
  float lo, hi, cmin, cmax, g_reco, g_trav;
};

// scalars_ext (sizeof(FusedScalars) bytes) / grads_ext (n_params + 1 floats): caller-owned device buffers, or NULL to
// let the trainer allocate them with the rest of its workspace (everything is allocated here, nothing per step).
// The statistics block is the scalars' first kStatDoubles.
int fused_trainer_create(const MlpShape& s, int max_rows, const LossCfg& loss, const AdamCfg& adam, void* scalars_ext,
                         float* grads_ext, Trainer** out);
// phase_mask: 1 = forward + statistics (+ their all-reduce), 2 = backward + weight gradients (+ gradient all-reduce),
// 4 = loss metrics + Adam; 7 = the whole step.
int fused_train_step(Trainer* t, float* params, float* exp_avg, float* exp_avg_sq, long long* step_counter,
                     const float* x, int groups, int rows_per_group, const int* n_rows, const float* y,
                     const unsigned char* y_valid, float* cg_mean, float* cg_std, float* conf_out, float* metrics,
                     int phase_mask, cudaStream_t stream);

}  // namespace wvn
