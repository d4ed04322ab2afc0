// wvn-b200: the TraversabilityLoss kernels of the learners whose output has SimpleMLP's (rows, 1 + dim) layout and whose
// step runs on the training core (double_mlp_train.cu, gcn_train.cu): the gather of the live rows, the per-row loss
// terms, the fp64 statistic sums and extrema, the ConfidenceGenerator update, dLoss/dOut with the per-row confidence,
// the confidence-weighted error sum and the loss metrics.  Every sum is formed by one thread or one fixed reduction
// tree, with no atomics.  Included by one translation unit per learner (internal linkage).
#pragma once

#include <stddef.h>

#include "common.cuh"
#include "mlp_train.h"
#include "train_core.cuh"

namespace wvn {

namespace {

constexpr int kRowThreads = 256;    // one warp per row
constexpr int kStatThreads = 256;   // the single-block reductions

// The step's scalars.  The first kStatDoubles are the statistics block every trainer exchanges (train_core.h): over
// the labelled rows the sum of loss_reco and of its square, over the live rows the sum of (trav - y)^2, the two row
// counts, then loss_reco's extrema.  trav_w: the confidence-weighted traversability error summed over the live rows.
struct DoubleScalars {
  double sum_lr, sum_lr2, sum_raw, n_valid, n_rows, reserved, x_min, x_max;
  double trav_w;
  float lo, hi, cmin, cmax, g_reco, g_trav;   // the updated generator and the loss-gradient scales
  float mean, std;
};
static_assert(offsetof(DoubleScalars, x_min) == kStatSums * sizeof(double) &&
              offsetof(DoubleScalars, trav_w) == kStatDoubles * sizeof(double), "statistics block layout");

// xg[i] = x[comp[i]]: the live rows, compacted (one warp per row)
__global__ void __launch_bounds__(kRowThreads)
double_gather_kernel(const float* __restrict__ x, const int* __restrict__ comp, const int* __restrict__ n_live, int dim,
                     float* __restrict__ xg) {
  const int lane = threadIdx.x & 31;
  const int r = (blockIdx.x * kRowThreads + threadIdx.x) >> 5;
  if (r >= *n_live) return;
  const float* src = x + static_cast<long long>(comp[r]) * dim;
  float* dst = xg + static_cast<long long>(r) * dim;
  for (int d = lane; d < dim; d += 32) dst[d] = src[d];
}

// loss_reco[r] = mean_d (out[r, 1 + d] - x[r, d])^2,  raw[r] = (out[r, 0] - y[r])^2
__global__ void __launch_bounds__(kRowThreads)
double_loss_rows_kernel(const float* __restrict__ out, const float* __restrict__ x, const float* __restrict__ y,
                        float* __restrict__ loss_reco, float* __restrict__ raw, const int* __restrict__ n_live,
                        int dim) {
  const int lane = threadIdx.x & 31;
  const int r = (blockIdx.x * kRowThreads + threadIdx.x) >> 5;
  if (r >= *n_live) return;
  const float* o = out + static_cast<long long>(r) * (dim + 1);
  const float* xr = x + static_cast<long long>(r) * dim;
  float acc = 0.f;
  for (int d = lane; d < dim; d += 32) {
    const float df = o[1 + d] - xr[d];
    acc = fmaf(df, df, acc);
  }
  acc = warp_sum(acc);
  if (lane == 0) {
    loss_reco[r] = acc / static_cast<float>(dim);
    const float dt = o[0] - y[r];
    raw[r] = dt * dt;
  }
}

// One block: this rank's statistic sums in fp64 (fixed reduction order) and loss_reco's extrema.  The extrema skip NaN
// rows (fminf / fmaxf).  The fused SimpleMLP step skips them too, except that a 32-row tile whose every live row is NaN
// makes its x_max NaN (mlp_train_fused.cu, atomicMax on the bits).
__global__ void __launch_bounds__(kStatThreads, 1)
double_stats_kernel(const float* __restrict__ loss_reco, const float* __restrict__ raw,
                    const unsigned char* __restrict__ y_valid, const int* __restrict__ n_live,
                    DoubleScalars* __restrict__ sc) {
  __shared__ double red[4][kStatThreads / 32];
  __shared__ float rmin[kStatThreads / 32], rmax[kStatThreads / 32];
  const int rows = *n_live, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  double s1 = 0.0, s2 = 0.0, sraw = 0.0, nv = 0.0;
  float mn = INFINITY, mx = 0.f;
  for (int i = t; i < rows; i += kStatThreads) {
    const float lr = loss_reco[i];
    sraw += static_cast<double>(raw[i]);
    mn = fminf(mn, lr);
    mx = fmaxf(mx, lr);
    if (y_valid[i]) { s1 += lr; s2 += static_cast<double>(lr) * lr; nv += 1.0; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    sraw += __shfl_xor_sync(0xffffffffu, sraw, o);
    nv += __shfl_xor_sync(0xffffffffu, nv, o);
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if (lane == 0) { red[0][warp] = s1; red[1][warp] = s2; red[2][warp] = sraw; red[3][warp] = nv; rmin[warp] = mn; rmax[warp] = mx; }
  __syncthreads();
  if (t != 0) return;
  double S1 = 0.0, S2 = 0.0, SR = 0.0, NV = 0.0;
  float MN = INFINITY, MX = 0.f;
  for (int w = 0; w < kStatThreads / 32; ++w) {
    S1 += red[0][w]; S2 += red[1][w]; SR += red[2][w]; NV += red[3][w];
    MN = fminf(MN, rmin[w]); MX = fmaxf(MX, rmax[w]);
  }
  sc->sum_lr = S1; sc->sum_lr2 = S2; sc->sum_raw = SR; sc->n_valid = NV; sc->n_rows = static_cast<double>(rows);
  sc->reserved = 0.0;
  sc->x_min = MN; sc->x_max = MX;
}

// One thread: the ConfidenceGenerator update from the (all-reduced) sums, and the loss-gradient scales over the global
// row counts.
__global__ void double_conf_kernel(int dim, LossCfg cfg, ConfState cs, float* __restrict__ cg_mean,
                                   float* __restrict__ cg_std, DoubleScalars* __restrict__ sc) {
  if (threadIdx.x != 0) return;
  const double NV = sc->n_valid;
  const ConfUpdate u = conf_generator_update(cs, cfg.std_factor, NV, sc->sum_lr, sc->sum_lr2, sc->x_min, sc->x_max,
                                             cg_mean);
  sc->lo = u.lo; sc->hi = u.hi; sc->cmin = u.cmin; sc->cmax = u.cmax;
  sc->g_reco = cfg.w_reco * 2.f / (static_cast<float>(NV) * static_cast<float>(dim));
  sc->g_trav = cfg.w_trav * 2.f / static_cast<float>(sc->n_rows);
  sc->mean = u.mean;
  sc->std = u.std;
  if (cg_mean) *cg_mean = u.mean;
  if (cg_std) *cg_std = u.std;
}

// dLoss/dOut of w_trav * L_trav + w_reco * L_reco (+ w_temp * 0), the confidence of each row under the updated
// generator (what ConfidenceGenerator.update returns) and each row's confidence-weighted traversability error.
__global__ void __launch_bounds__(kRowThreads)
double_dout_kernel(const float* __restrict__ out, const float* __restrict__ x, const float* __restrict__ y,
                   const unsigned char* __restrict__ y_valid, const float* __restrict__ loss_reco,
                   const float* __restrict__ raw, const DoubleScalars* __restrict__ sc, LossCfg cfg, int method,
                   float* __restrict__ d_out, float* __restrict__ conf_out, float* __restrict__ wraw,
                   const int* __restrict__ n_live, int dim) {
  const int lane = threadIdx.x & 31;
  const int r = (blockIdx.x * kRowThreads + threadIdx.x) >> 5;
  if (r >= *n_live) return;
  const float lo = sc->lo, hi = sc->hi, cmin = sc->cmin, cmax = sc->cmax, g_reco = sc->g_reco, g_trav = sc->g_trav;
  const bool v = y_valid[r] != 0;
  const float conf = row_confidence(method, loss_reco[r], lo, hi, cmin, cmax);
  const float wgt = (v || !cfg.anomaly_balanced) ? 1.f : (1.f - conf);
  const float* o = out + static_cast<long long>(r) * (dim + 1);
  const float* xr = x + static_cast<long long>(r) * dim;
  float* g = d_out + static_cast<long long>(r) * (dim + 1);
  for (int d = lane; d < dim; d += 32) g[1 + d] = v ? g_reco * (o[1 + d] - xr[d]) : 0.f;
  if (lane == 0) {
    const float tv = o[0];
    g[0] = g_trav * wgt * (tv - y[r]) * tv * (1.f - tv);   // through the sigmoid
    conf_out[r] = conf;
    wraw[r] = raw[r] * wgt;
  }
}

// This rank's confidence-weighted traversability error sum (one block, fixed reduction order).
__global__ void __launch_bounds__(kStatThreads, 1)
double_trav_w_kernel(const float* __restrict__ wraw, const int* __restrict__ n_live, DoubleScalars* __restrict__ sc) {
  __shared__ double red[kStatThreads / 32];
  const int rows = *n_live, t = threadIdx.x;
  double s = 0.0;
  for (int i = t; i < rows; i += kStatThreads) s += static_cast<double>(wraw[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((t & 31) == 0) red[t >> 5] = s;
  __syncthreads();
  if (t != 0) return;
  double S = 0.0;
  for (int w = 0; w < kStatThreads / 32; ++w) S += red[w];
  sc->trav_w = S;
}

// Loss metrics from the global sums; leaves them in metrics[6] for the host.
__global__ void double_finish_kernel(LossCfg cfg, const DoubleScalars* __restrict__ sc, float* __restrict__ metrics) {
  if (threadIdx.x != 0) return;
  const float loss_reco = static_cast<float>(sc->sum_lr / sc->n_valid);
  const float loss_trav_conf = static_cast<float>(sc->trav_w / sc->n_rows);
  metrics[0] = cfg.w_trav * loss_trav_conf + cfg.w_reco * loss_reco;
  metrics[1] = static_cast<float>(sc->sum_raw / sc->n_rows);
  metrics[2] = loss_reco;
  metrics[3] = loss_trav_conf;
  metrics[4] = sc->mean;
  metrics[5] = sc->std;
}

}  // namespace

}  // namespace wvn
