// wvn-b200: device code shared by the train steps (train_core.cu, mlp_train_fused.cu, flow_train.cu): the Adam update
// and the ConfidenceGenerator.  utils/confidence_generator.py: latest_measurement :78-82, running_mean :94-115,
// moving_average :117-129, kalman_filter :131-145 (+ KalmanFilter, utils/kalman_filter.py:78-111 with D = 1, F = H = 1).
#pragma once

#include <cuda_runtime.h>

#include "train_core.h"

namespace wvn {

// torch.optim.Adam (no amsgrad, no weight decay) over n parameters, grid-stride: step t = *step_ptr counts from 1
__device__ __forceinline__ void adam_update(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                            float* __restrict__ v, long long n, const AdamCfg& cfg,
                                            const long long* __restrict__ step_ptr) {
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

// The generator after one update, and what a row needs to turn its loss into a confidence:
// latest_measurement / running_mean: the interval [lo, hi]; kalman_filter: mean and 1 / (std * std_factor) in lo / hi;
// moving_average: the clip interval and the clipped extrema cmin / cmax.
struct ConfUpdate {
  float mean, std, lo, hi, cmin, cmax;
};

// One update from the sums over the positive set (n rows, sum s1, sum of squares s2) and the extrema of x.  Updates the
// state behind cs in place; the Kalman state is read from *cg_mean (0 when null).  One thread.
__device__ __forceinline__ ConfUpdate conf_generator_update(const ConfState& cs, float std_factor, double n, double s1,
                                                            double s2, double x_min, double x_max,
                                                            const float* cg_mean) {
  float m, sd;
  float lo, hi, cmin = 0.f, cmax = 0.f;
  if (cs.method == CONF_RUNNING_MEAN) {
    const double rn = *cs.running_n + n, rs = *cs.running_sum + s1, rq = *cs.running_sumsq + s2;
    *cs.running_n = rn; *cs.running_sum = rs; *cs.running_sumsq = rq;
    m = static_cast<float>(rs / rn);
    const float var = static_cast<float>(rq / rn - static_cast<double>(m * m));   // float64 - float32^2, stored as fp32
    sd = sqrtf(var);
    if (cs.var) *cs.var = var;
  } else if (cs.method == CONF_KALMAN) {
    float state = cg_mean ? *cg_mean : 0.f, cov = cs.var ? *cs.var : 1.f;
    if (n > 0.0) {
      const float meas = static_cast<float>(s1 / n);
      cov = cov + cs.kf_proc_cov;                      // prediction: F = 1
      const float gain = cov / (cov + cs.kf_meas_cov);
      state = state + gain * (meas - state);
      cov = (1.f - gain) * cov;
      if (cs.var) *cs.var = cov;
    }
    m = state;
    sd = sqrtf(cov);
  } else if (cs.method == CONF_MOVING_AVERAGE) {
    // the deque of the last kConfWindow positive sets, kept as (n, sum, sum of squares) per step
    double* ring = cs.ring;
    const int count = static_cast<int>(ring[3 * kConfWindow]);
    const int slot = count % kConfWindow;
    ring[3 * slot] = n; ring[3 * slot + 1] = s1; ring[3 * slot + 2] = s2;
    ring[3 * kConfWindow] = count + 1;
    double N = 0.0, S1 = 0.0, S2 = 0.0;
    for (int i = 0; i < (count + 1 < kConfWindow ? count + 1 : kConfWindow); ++i) { N += ring[3 * i]; S1 += ring[3 * i + 1]; S2 += ring[3 * i + 2]; }
    const double mean = S1 / N;
    m = static_cast<float>(mean);
    sd = N > 1.0 ? static_cast<float>(sqrt(fmax((S2 - N * mean * mean) / (N - 1.0), 0.0))) : nanf("");
  } else {
    const double mean = s1 / n;                                   // n == 0 -> NaN, like torch's mean of empty
    const double var = (s2 - n * mean * mean) / (n - 1.0);        // n == 1 -> NaN, like torch.std
    m = static_cast<float>(mean);
    sd = (n > 1.0) ? static_cast<float>(sqrt(fmax(var, 0.0))) : nanf("");
  }
  if (cs.method == CONF_KALMAN) {
    lo = m;
    hi = 1.f / (sd * std_factor);
  } else if (cs.method == CONF_MOVING_AVERAGE) {
    lo = m - 2.f * sd;
    hi = m + 2.f * sd;
    cmin = fminf(fmaxf(static_cast<float>(x_min), lo), hi);   // min / max of the clipped losses = clipped extrema
    cmax = fminf(fmaxf(static_cast<float>(x_max), lo), hi);
  } else {
    const float shifted = m + sd * std_factor;
    lo = fmaxf(shifted - sd, 0.f);
    hi = shifted + sd;
  }
  return ConfUpdate{m, sd, lo, hi, cmin, cmax};
}

// The confidence of one row's loss under the updated generator (the value ConfidenceGenerator.update returns for it).
__device__ __forceinline__ float row_confidence(int method, float lr, float lo, float hi, float cmin, float cmax) {
  if (method == CONF_KALMAN) {   // lo = mean, hi = 1 / (std * std_factor)
    const float z = (lr - lo) * hi;
    return lr < lo ? 1.f : expf(-(z * z) * 0.5f);
  }
  const float xc = fminf(fmaxf(lr, lo), hi);
  if (method == CONF_MOVING_AVERAGE) return (xc - cmin) / (cmax - cmin);
  return 1.f - (xc - lo) / (hi - lo);
}

}  // namespace wvn
