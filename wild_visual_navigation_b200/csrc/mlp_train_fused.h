// wvn-b200: internal interface of the fused online train step (mlp_train_fused.cu).
#pragma once

#include <cuda_runtime.h>

#include "mlp_train.h"

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

// ConfidenceGenerator methods (utils/confidence_generator.py:49-76)
enum ConfMethod : int { CONF_LATEST = 0, CONF_RUNNING_MEAN = 1, CONF_KALMAN = 2, CONF_MOVING_AVERAGE = 3 };
constexpr int kConfWindow = 5;   // moving_average's deque(maxlen=5)

// State the reference keeps in the ConfidenceGenerator module, updated in place on the device.
struct ConfState {
  int method = CONF_LATEST;
  float* var = nullptr;                                        // (1,1) fp32 parameter
  double *running_n = nullptr, *running_sum = nullptr, *running_sumsq = nullptr;   // (1,) fp64 parameters
  float kf_proc_cov = 0.2f, kf_meas_cov = 1.0f;                // the 1-D Kalman filter's Q and R (F = H = 1)
  double* ring = nullptr;                                      // trainer-owned: [kConfWindow][3] (n, sum, sum^2) + count
};

struct FusedTrainer;

// scalars_ext (sizeof(FusedScalars) bytes) / grads_ext (n_params + 1 floats): caller-owned device buffers, or NULL to
// let the trainer allocate them with the rest of its workspace (everything is allocated here, nothing per step).
int fused_trainer_create(const MlpShape& s, int max_rows, const LossCfg& loss, const AdamCfg& adam, void* scalars_ext,
                         float* grads_ext, FusedTrainer** out);
void fused_trainer_destroy(FusedTrainer* t);
int fused_comm_unique_id(void* id128);
int fused_trainer_init_comm(FusedTrainer* t, const void* id128, int rank, int world);
// method: ConfMethod; pointers may be null for methods that do not use them (the trainer then keeps private state).
int fused_trainer_set_confidence(FusedTrainer* t, int method, float* var, double* running_n, double* running_sum,
                                 double* running_sumsq, float kf_proc_cov, float kf_meas_cov);
// Copies src's private confidence state (moving_average's window; var / running sums not bound to caller buffers) into
// dst, on `stream`: a caller that replaces a trainer by a larger one keeps the generator where it was.
int fused_trainer_copy_confidence(FusedTrainer* dst, const FusedTrainer* src, cudaStream_t stream);
// phase_mask: 1 = forward + statistics (+ their all-reduce), 2 = backward + weight gradients (+ gradient all-reduce),
// 4 = loss metrics + Adam; 7 = the whole step.
int fused_train_step(FusedTrainer* t, float* params, float* exp_avg, float* exp_avg_sq, long long* step_counter,
                     const float* x, int groups, int rows_per_group, const int* n_rows, const float* y,
                     const unsigned char* y_valid, float* cg_mean, float* cg_std, float* conf_out, float* metrics,
                     int phase_mask, cudaStream_t stream);

}  // namespace wvn
