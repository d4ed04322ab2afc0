// wvn-b200: the online train step as FOUR kernels and (data-parallel) two in-library collectives.
//
// Same arithmetic as mlp_train.cu (the body of TraversabilityEstimator.train(), traversability_estimator.py:464-477:
// SimpleMLP.forward -> TraversabilityLoss.forward incl. the ConfidenceGenerator "latest_measurement" update ->
// backward -> Adam), restructured to remove what that version's launch list shows — some twenty short launches, two host
// synchronisations (a boolean-mask gather and an .item()) and three torch.distributed calls per step:
//
//   K1 train_fwd_rows   : per 32-row tile the three layers run back to back out of shared memory; per-row loss terms and
//                         the statistic sums (6 doubles, incl. the row count) leave the kernel
//   [all-reduce of the 6 doubles]                               (only with a communicator)
//   K2 train_bwd_rows   : confidence update, dLoss/dOut, dH2, dH1 per 32-row tile; bumps the Adam step counter
//   K3 train_wgrad      : dW3 | dW2 | dW1 (+ the three bias gradients) as ONE multi-problem split-K launch
//   [all-reduce of the flat gradient (+ the confidence-weighted error sum riding at its end)]
//   K4 train_apply      : loss metrics + Adam + metrics vector for the host
//
// Rows arrive PADDED, as the segment-pooling kernel leaves them: x [groups, rows_per_group, dim] with n_rows[g] live rows
// per group (device memory).  The compaction the reference does with a boolean mask (`feat[seg_mask]`) happens inside
// the kernels — labels y / y_valid are indexed by the compacted row number — so the step has no host synchronisation.
// The communicator is the training core's (train_core.h: NCCL, owned by the library, wvn_trainer_init_comm), so the
// collectives are issued from here on the caller's stream.
#include <string.h>

#include <algorithm>

#include "common.cuh"
#include "host_common.h"
#include "mlp_train.h"
#include "mlp_train_fused.h"
#include "train_core.cuh"

namespace wvn {

namespace {

constexpr int TR = 32;     // rows per CTA
constexpr int TRP = 33;    // padded row stride of transposed activation tiles
constexpr int KC = 32;     // layer-1 K chunk
constexpr int kThreads = 256;

// Compacted index of padded row r (group-major), -1 when the row is padding.
__device__ __forceinline__ int compact_index(const int* __restrict__ n_rows, int groups, int rpg, int r) {
  if (r >= groups * rpg) return -1;
  if (n_rows == nullptr) return r;
  const int g = r / rpg, s = r - g * rpg;
  if (s >= min(n_rows[g], rpg)) return -1;
  int base = 0;
  for (int i = 0; i < g; ++i) base += min(n_rows[i], rpg);
  return base + s;
}

// ------------------------------------------------------------------------------------------------ K1
// smem (floats): xt[dim][TR] | wbuf[max(KC*(h1+1), h1*33, ...)] | h1t[h1][TRP] | h2t[h2][TR] | red[TR] | rowinfo[TR]
__global__ void __launch_bounds__(kThreads)
train_fwd_rows_kernel(MlpShape s, MlpOffsets o, const float* __restrict__ params, const float* __restrict__ x,
                      const float* __restrict__ y, const unsigned char* __restrict__ y_valid,
                      const int* __restrict__ n_rows, int groups, int rpg, float* __restrict__ h1g,
                      float* __restrict__ h2g, float* __restrict__ outg, float* __restrict__ loss_reco,
                      float* __restrict__ raw, FusedScalars* __restrict__ sc, float* __restrict__ trav_w_sum) {
  // the confidence-weighted traversability sum of this step is accumulated by K2: start it from zero here (the flat
  // gradient itself is cleared by K2 before K3 accumulates into it, the statistic sums by the previous step's K4)
  if (blockIdx.x == 0 && threadIdx.x == 0) *trav_w_sum = 0.f;
  extern __shared__ __align__(16) float sm[];
  const int dim = s.dim, h1 = s.h1, h2 = s.h2, n3 = s.dim + 1;
  float* xt = sm;                               // [dim][TR]
  float* wbuf = xt + dim * TR;                  // scratch for weight tiles
  const int wbuf_floats = max(KC * (h1 + 1), h1 * TRP);  // W1 chunk [KC][h1+1]  |  W2^T [h1][33]
  float* h1t = wbuf + wbuf_floats;              // [h1][TRP]
  float* h2t = h1t + h1 * TRP;                  // [h2][TR]
  float* red = h2t + h2 * TR;                   // [TR]
  int* rinfo = reinterpret_cast<int*>(red + TR);  // [TR]

  const int t = threadIdx.x;
  const int r0 = blockIdx.x * TR;
  if (t < TR) {
    rinfo[t] = compact_index(n_rows, groups, rpg, r0 + t);
    red[t] = 0.f;
  }
  __syncthreads();
  // x tile, transposed; padding rows read as zeros
  for (int idx = t; idx < TR * dim; idx += kThreads) {
    const int row = idx / dim, k = idx - row * dim;
    xt[k * TR + row] = rinfo[row] >= 0 ? x[static_cast<long long>(r0 + row) * dim + k] : 0.f;
  }

  // ---- layer 1: h1 = relu(x W1^T + b1); thread -> cols cg + 64 j, rows 8 rg .. 8 rg + 7
  {
    const int cg = t & 63, rg = t >> 6;
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    const float* W1 = params + o.w1;
    const int ldw = h1 + 1;
    for (int k0 = 0; k0 < dim; k0 += KC) {
      __syncthreads();  // previous chunk consumed (and xt complete on the first pass)
      const int kc = min(KC, dim - k0);
      for (int idx = t; idx < h1 * KC; idx += kThreads) {
        const int n = idx / KC, kk = idx - n * KC;
        wbuf[kk * ldw + n] = kk < kc ? W1[static_cast<long long>(n) * dim + k0 + kk] : 0.f;
      }
      __syncthreads();
#pragma unroll 4
      for (int kk = 0; kk < KC; ++kk) {
        const float4 xa = *reinterpret_cast<const float4*>(&xt[(k0 + kk < dim ? k0 + kk : 0) * TR + 8 * rg]);
        const float4 xb = *reinterpret_cast<const float4*>(&xt[(k0 + kk < dim ? k0 + kk : 0) * TR + 8 * rg + 4]);
        const float xv[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
        float wv[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) wv[j] = (cg + 64 * j < h1) ? wbuf[kk * ldw + cg + 64 * j] : 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(xv[i], wv[j], acc[i][j]);
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = cg + 64 * j;
      if (n >= h1) continue;
      const float b = params[o.b1 + n];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int row = 8 * rg + i;
        const float v = fmaxf(acc[i][j] + b, 0.f);
        h1t[n * TRP + row] = v;
        if (rinfo[row] >= 0) h1g[static_cast<long long>(r0 + row) * h1 + n] = v;
      }
    }
  }
  __syncthreads();
  // ---- layer 2: h2 = relu(h1 W2^T + b2); thread -> col n = t & 31 (h2 <= 32), rows 4 rg .. 4 rg + 3
  {
    const float* W2 = params + o.w2;
    for (int idx = t; idx < h2 * h1; idx += kThreads) {
      const int n = idx / h1, k = idx - n * h1;
      wbuf[k * TRP + n] = W2[idx];
    }
    __syncthreads();
    const int n = t & 31, rg = t >> 5;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    if (n < h2) {
      for (int k = 0; k < h1; ++k) {
        const float w = wbuf[k * TRP + n];
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i] = fmaf(h1t[k * TRP + 4 * rg + i], w, acc[i]);
      }
      const float b = params[o.b2 + n];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int row = 4 * rg + i;
        const float v = fmaxf(acc[i] + b, 0.f);
        h2t[n * TR + row] = v;
        if (rinfo[row] >= 0) h2g[static_cast<long long>(r0 + row) * h2 + n] = v;
      }
    }
  }
  __syncthreads();
  // ---- layer 3 + per-row loss terms: thread -> output columns t, t + 256, ... for all 32 rows
  {
    const float* W3 = params + o.w3;
    const int lane = t & 31;
    for (int n = t; n < (n3 + kThreads - 1) / kThreads * kThreads; n += kThreads) {
      float part[TR];
#pragma unroll
      for (int i = 0; i < TR; ++i) part[i] = 0.f;
      if (n < n3) {
        float acc[TR];
#pragma unroll
        for (int i = 0; i < TR; ++i) acc[i] = 0.f;
        for (int k = 0; k < h2; ++k) {
          const float w = W3[static_cast<long long>(n) * h2 + k];
#pragma unroll
          for (int i4 = 0; i4 < TR / 4; ++i4) {
            const float4 hv = *reinterpret_cast<const float4*>(&h2t[k * TR + 4 * i4]);
            acc[4 * i4 + 0] = fmaf(hv.x, w, acc[4 * i4 + 0]);
            acc[4 * i4 + 1] = fmaf(hv.y, w, acc[4 * i4 + 1]);
            acc[4 * i4 + 2] = fmaf(hv.z, w, acc[4 * i4 + 2]);
            acc[4 * i4 + 3] = fmaf(hv.w, w, acc[4 * i4 + 3]);
          }
        }
        const float b = params[o.b3 + n];
#pragma unroll
        for (int i = 0; i < TR; ++i) {
          float v = acc[i] + b;
          if (n == 0) v = 1.f / (1.f + expf(-v));  // x[:, :1] = sigmoid(x[:, :1])  (simple_mlp.py:37)
          if (rinfo[i] >= 0) outg[static_cast<long long>(r0 + i) * n3 + n] = v;
          if (n > 0) {
            const float df = v - xt[(n - 1) * TR + i];
            part[i] = df * df;
          } else if (rinfo[i] >= 0) {
            const float dt = v - y[rinfo[i]];
            raw[r0 + i] = dt * dt;
          }
        }
      }
      // sum of squared reconstruction errors per row: warp shuffle, then one shared-memory atomic per warp and row
#pragma unroll
      for (int i = 0; i < TR; ++i) {
        const float v = warp_sum(part[i]);
        if (lane == 0) atomicAdd(&red[i], v);
      }
    }
  }
  __syncthreads();
  if (t < TR) {  // one warp: per-row results + the statistic sums of this tile
    const int ci = rinfo[t];
    double s1 = 0.0, s2 = 0.0, sraw = 0.0, nv = 0.0, nr = 0.0;
    if (ci >= 0) {
      const float lr = red[t] / static_cast<float>(dim);
      loss_reco[r0 + t] = lr;
      sraw = static_cast<double>(raw[r0 + t]);
      nr = 1.0;
      if (y_valid[ci]) { s1 = lr; s2 = static_cast<double>(lr) * lr; nv = 1.0; }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, off);
      s2 += __shfl_xor_sync(0xffffffffu, s2, off);
      sraw += __shfl_xor_sync(0xffffffffu, sraw, off);
      nv += __shfl_xor_sync(0xffffffffu, nv, off);
      nr += __shfl_xor_sync(0xffffffffu, nr, off);
    }
    // extrema of loss_reco over the live rows (non-negative doubles order like their bit patterns)
    double lmin = ci >= 0 ? static_cast<double>(red[t] / static_cast<float>(dim)) : __longlong_as_double(0x7ff0000000000000ll);
    double lmax = ci >= 0 ? static_cast<double>(red[t] / static_cast<float>(dim)) : 0.0;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      lmin = fmin(lmin, __shfl_xor_sync(0xffffffffu, lmin, off));
      lmax = fmax(lmax, __shfl_xor_sync(0xffffffffu, lmax, off));
    }
    if (t == 0 && nr > 0.0) {
      atomicMin(reinterpret_cast<unsigned long long*>(&sc->x_min), static_cast<unsigned long long>(__double_as_longlong(lmin)));
      atomicMax(reinterpret_cast<unsigned long long*>(&sc->x_max), static_cast<unsigned long long>(__double_as_longlong(lmax)));
      atomicAdd(&sc->sum_lr, s1);
      atomicAdd(&sc->sum_lr2, s2);
      atomicAdd(&sc->sum_raw, sraw);
      atomicAdd(&sc->n_valid, nv);
      atomicAdd(&sc->n_rows, nr);
    }
  }
}

// ------------------------------------------------------------------------------------------------ K1b
// ConfidenceGenerator.update from the (all-reduced) sums of this step: one thread (train_core.cuh).
__global__ void train_conf_kernel(LossCfg cfg, ConfState cs, int dim, FusedScalars* __restrict__ sc,
                                  float* __restrict__ cg_mean, float* __restrict__ cg_std,
                                  long long* __restrict__ step_counter) {
  if (threadIdx.x != 0) return;
  const double n = sc->n_valid;
  const ConfUpdate u = conf_generator_update(cs, cfg.std_factor, n, sc->sum_lr, sc->sum_lr2, sc->x_min, sc->x_max,
                                             cg_mean);
  const float m = u.mean, sd = u.std, lo = u.lo, hi = u.hi, cmin = u.cmin, cmax = u.cmax;
  sc->lo = lo; sc->hi = hi; sc->cmin = cmin; sc->cmax = cmax;
  sc->g_reco = cfg.w_reco * 2.f / (static_cast<float>(n) * static_cast<float>(dim));
  sc->g_trav = cfg.w_trav * 2.f / static_cast<float>(sc->n_rows);
  sc->mean = m;
  sc->std = sd;
  if (cg_mean) *cg_mean = m;
  if (cg_std) *cg_std = sd;
  *step_counter += 1;  // torch.optim.Adam counts from 1; K4 reads the bumped value
}

// ------------------------------------------------------------------------------------------------ K2
// smem (floats): dot[n3][TRP] | dh2t[h2][TR] | rowinfo[TR] | cst[8]
// conf_method == CONF_LATEST: the generator's update has no memory, so every block derives it from the sums itself
// (block 0 publishes it and bumps the step counter) and train_conf_kernel is not launched: the default step is 4 launches.
__global__ void __launch_bounds__(kThreads)
train_bwd_rows_kernel(MlpShape s, MlpOffsets o, LossCfg cfg, int conf_method, const float* __restrict__ params,
                      const float* __restrict__ x, const float* __restrict__ y,
                      const unsigned char* __restrict__ y_valid, const int* __restrict__ n_rows, int groups, int rpg,
                      const float* __restrict__ h1g, const float* __restrict__ h2g, const float* __restrict__ outg,
                      const float* __restrict__ loss_reco, const float* __restrict__ raw, float* __restrict__ d_out,
                      float* __restrict__ d_h2, float* __restrict__ d_h1, float* __restrict__ conf_out,
                      FusedScalars* __restrict__ sc, float* __restrict__ cg_mean, float* __restrict__ cg_std,
                      float* __restrict__ trav_w_sum, long long* __restrict__ step_counter,
                      float* __restrict__ grads_clear, long long n_clear) {
  for (long long i = blockIdx.x * static_cast<long long>(kThreads) + threadIdx.x; i < n_clear;
       i += static_cast<long long>(gridDim.x) * kThreads)
    grads_clear[i] = 0.f;   // K3 accumulates the weight gradients with atomics
  extern __shared__ __align__(16) float sm[];
  const int dim = s.dim, h1 = s.h1, h2 = s.h2, n3 = s.dim + 1;
  float* dot = sm;                                 // [n3][TRP]
  float* dh2t = dot + ((n3 * TRP + 3) & ~3);       // [h2][TR], 16-byte aligned for the float4 broadcasts
  int* rinfo = reinterpret_cast<int*>(dh2t + h2 * TR);
  const int t = threadIdx.x;
  const int r0 = blockIdx.x * TR;
  float* cst = reinterpret_cast<float*>(rinfo + TR);  // lo, hi, g_reco, g_trav
  if (t < TR) rinfo[t] = compact_index(n_rows, groups, rpg, r0 + t);
  if (t == 0) {
    if (conf_method == CONF_LATEST) {
      // ConfidenceGenerator.update_latest_measurement (confidence_generator.py:78-82) from the (all-reduced) sums
      const double n = sc->n_valid;
      const double mean = sc->sum_lr / n;                                  // n == 0 -> NaN, like torch's mean of empty
      const double var = (sc->sum_lr2 - n * mean * mean) / (n - 1.0);     // n == 1 -> NaN, like torch.std
      const float m = static_cast<float>(mean);
      const float sd = (n > 1.0) ? static_cast<float>(sqrt(fmax(var, 0.0))) : nanf("");
      const float shifted = m + sd * cfg.std_factor;
      cst[0] = fmaxf(shifted - sd, 0.f);
      cst[1] = shifted + sd;
      cst[2] = cfg.w_reco * 2.f / (static_cast<float>(n) * static_cast<float>(dim));
      cst[3] = cfg.w_trav * 2.f / static_cast<float>(sc->n_rows);
      cst[4] = cst[5] = 0.f;
      if (blockIdx.x == 0) {
        sc->mean = m;
        sc->std = sd;
        if (cg_mean) *cg_mean = m;
        if (cg_std) *cg_std = sd;
        *step_counter += 1;  // torch.optim.Adam counts from 1; K4 reads the bumped value
      }
    } else {
      cst[0] = sc->lo; cst[1] = sc->hi; cst[2] = sc->g_reco; cst[3] = sc->g_trav; cst[4] = sc->cmin; cst[5] = sc->cmax;
    }
  }
  __syncthreads();
  const float lo = cst[0], hi = cst[1], g_reco = cst[2], g_trav = cst[3], cmin = cst[4], cmax = cst[5];
  // ---- dOut (one warp per 4 rows), kept transposed in shared memory for the two products below
  {
    const int warp = t >> 5, lane = t & 31;
    double s_trav = 0.0;
    for (int i = 0; i < 4; ++i) {
      const int row = warp * 4 + i;
      const int ci = rinfo[row];
      const long long r = r0 + row;
      if (ci < 0) {
        for (int n = lane; n < n3; n += 32) dot[n * TRP + row] = 0.f;
        continue;
      }
      const bool v = y_valid[ci] != 0;
      const float lr = loss_reco[r];
      const float conf = row_confidence(conf_method, lr, lo, hi, cmin, cmax);
      const float wgt = (v || !cfg.anomaly_balanced) ? 1.f : (1.f - conf);
      const float* orow = outg + r * n3;
      const float* xr = x + r * dim;
      float* grow = d_out + r * n3;
      for (int n = lane; n < n3; n += 32) {
        float g;
        if (n == 0) {
          const float tv = orow[0];
          g = g_trav * wgt * (tv - y[ci]) * tv * (1.f - tv);  // through the sigmoid
        } else {
          g = v ? g_reco * (orow[n] - xr[n - 1]) : 0.f;
        }
        dot[n * TRP + row] = g;
        grow[n] = g;
      }
      if (lane == 0) {
        conf_out[ci] = conf;
        s_trav += static_cast<double>(raw[r] * wgt);
      }
    }
    if (lane == 0 && s_trav != 0.0) atomicAdd(trav_w_sum, static_cast<float>(s_trav));
  }
  __syncthreads();
  // ---- dH2 = (dOut W3) * (H2 > 0): thread -> col m = t & 31, rows 4 rg .. 4 rg + 3
  {
    const float* W3 = params + o.w3;
    const int m = t & 31, rg = t >> 5;
    if (m < h2) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int n = 0; n < n3; ++n) {
        const float w = W3[static_cast<long long>(n) * h2 + m];
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i] = fmaf(dot[n * TRP + 4 * rg + i], w, acc[i]);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int row = 4 * rg + i;
        const long long r = r0 + row;
        float v = 0.f;
        if (rinfo[row] >= 0) {
          v = h2g[r * h2 + m] > 0.f ? acc[i] : 0.f;
          d_h2[r * h2 + m] = v;
        }
        dh2t[m * TR + row] = v;
      }
    }
  }
  __syncthreads();
  // ---- dH1 = (dH2 W2) * (H1 > 0): thread -> columns t, t + 256, ... for all 32 rows
  {
    const float* W2 = params + o.w2;
    for (int j = t; j < h1; j += kThreads) {
      float acc[TR];
#pragma unroll
      for (int i = 0; i < TR; ++i) acc[i] = 0.f;
      for (int m = 0; m < h2; ++m) {
        const float w = W2[static_cast<long long>(m) * h1 + j];
#pragma unroll
        for (int i4 = 0; i4 < TR / 4; ++i4) {
          const float4 dv = *reinterpret_cast<const float4*>(&dh2t[m * TR + 4 * i4]);
          acc[4 * i4 + 0] = fmaf(dv.x, w, acc[4 * i4 + 0]);
          acc[4 * i4 + 1] = fmaf(dv.y, w, acc[4 * i4 + 1]);
          acc[4 * i4 + 2] = fmaf(dv.z, w, acc[4 * i4 + 2]);
          acc[4 * i4 + 3] = fmaf(dv.w, w, acc[4 * i4 + 3]);
        }
      }
#pragma unroll
      for (int i = 0; i < TR; ++i) {
        if (rinfo[i] < 0) continue;
        const long long r = r0 + i;
        d_h1[r * h1 + j] = h1g[r * h1 + j] > 0.f ? acc[i] : 0.f;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ K3
// Three weight-gradient products dW = dZ^T · A (reduction over the rows) + the bias gradients (column sums of dZ),
// one launch: blockIdx.x enumerates (problem, m tile, n tile, row split).  Padding rows are skipped via n_rows.
constexpr int TS = 64, TK = 16;
struct WgradProblem {
  const float* dz; int ldz; int m;   // dZ [rows, m]  -> gradient rows
  const float* a; int lda; int n;    // A  [rows, n]  -> gradient columns
  float* dw;                          // [m, n]
  float* db;                          // [m]
  int tiles_m, tiles_n, first_block;
};
struct WgradArgs {
  WgradProblem p[3];
  int splits, total_rows, rows_per_split;
  const int* n_rows; int groups, rpg;
};

__global__ void __launch_bounds__(256)
train_wgrad_kernel(WgradArgs a) {
  __shared__ float As[TK][TS + 1];  // dZ tile, [k = row][m]
  __shared__ float Bs[TK][TS + 1];  // A tile,  [k = row][n]
  __shared__ unsigned char live[TK];
  int pi = 0;
  if (blockIdx.x >= a.p[1].first_block) pi = 1;
  if (blockIdx.x >= a.p[2].first_block) pi = 2;
  const WgradProblem& p = a.p[pi];
  int rel = blockIdx.x - p.first_block;
  const int split = rel % a.splits;
  rel /= a.splits;
  const int tn = rel % p.tiles_n, tm = rel / p.tiles_n;
  const int m0 = tm * TS, n0 = tn * TS;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int kbeg = split * a.rows_per_split, kend = min(a.total_rows, kbeg + a.rows_per_split);
  float acc[4][4], bsum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = kbeg; k0 < kend; k0 += TK) {
    if (threadIdx.x < TK) {
      const int r = k0 + threadIdx.x;
      bool ok = r < kend;
      if (ok && a.n_rows) {
        const int g = r / a.rpg;
        ok = (r - g * a.rpg) < a.n_rows[g];
      }
      live[threadIdx.x] = ok;
    }
    __syncthreads();
#pragma unroll
    for (int rr = 0; rr < 4; ++rr) {
      const int idx = threadIdx.x + 256 * rr;  // 0..1023
      const int k = idx >> 6, c = idx & 63;    // consecutive threads -> consecutive columns of one row (coalesced)
      const long long r = k0 + k;
      As[k][c] = (live[k] && m0 + c < p.m) ? p.dz[r * p.ldz + m0 + c] : 0.f;
      Bs[k][c] = (live[k] && n0 + c < p.n) ? p.a[r * p.lda + n0 + c] : 0.f;
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
      for (int i = 0; i < 4; ++i) {
        bsum[i] += av[i];
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gm = m0 + ty + 16 * i;
    if (gm >= p.m) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx + 16 * j;
      if (gn < p.n) atomicAdd(&p.dw[static_cast<long long>(gm) * p.n + gn], acc[i][j]);
    }
    if (tn == 0 && tx == 0) atomicAdd(&p.db[gm], bsum[i]);
  }
}

// ------------------------------------------------------------------------------------------------ K4
__global__ void __launch_bounds__(256)
train_apply_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                   long long n, AdamCfg cfg, LossCfg lcfg, const long long* __restrict__ step_ptr,
                   FusedScalars* __restrict__ sc, float* __restrict__ metrics) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const double nv = sc->n_valid, nt = sc->n_rows;
    sc->loss_reco = static_cast<float>(sc->sum_lr / nv);
    sc->loss_trav_conf = static_cast<float>(static_cast<double>(g[n]) / nt);
    sc->loss_trav = static_cast<float>(sc->sum_raw / nt);
    sc->loss_total = lcfg.w_trav * sc->loss_trav_conf + lcfg.w_reco * sc->loss_reco;  // + w_temp * 0
    if (metrics) {
      metrics[0] = sc->loss_total; metrics[1] = sc->loss_trav; metrics[2] = sc->loss_reco;
      metrics[3] = sc->loss_trav_conf; metrics[4] = sc->mean; metrics[5] = sc->std;
    }
    // leave the accumulators clean for the next step (no memsets on the per-frame path)
    sc->x_min = __longlong_as_double(0x7ff0000000000000ll);   // +inf / 0: ready for atomicMin / atomicMax
    sc->x_max = 0.0;
    sc->sum_lr = sc->sum_lr2 = sc->sum_raw = sc->n_valid = sc->n_rows = sc->reserved = 0.0;
  }
  adam_update(p, g, m, v, n, cfg, step_ptr);
}

}  // namespace

struct FusedTrainer : Trainer {
  FusedTrainer() : Trainer(TRAINER_MLP) {}
  MlpShape s;
  MlpOffsets o;
  float *h1 = nullptr, *h2 = nullptr, *out = nullptr, *d_out = nullptr, *d_h2 = nullptr, *d_h1 = nullptr,
        *loss_reco = nullptr, *raw = nullptr;
  FusedScalars* sc = nullptr;
  size_t smem_fwd = 0, smem_bwd = 0;
};

int fused_trainer_create(const MlpShape& s, int max_rows, const LossCfg& loss, const AdamCfg& adam, void* scalars_ext,
                         float* grads_ext, Trainer** out) {
  WVN_REQUIRE(out && max_rows > 0, "trainer: bad arguments");
  WVN_REQUIRE(s.dim > 0 && s.dim <= 1024 && s.h1 > 0 && s.h1 <= 256 && s.h1 % 4 == 0 && s.h2 > 0 && s.h2 <= 32,
              "trainer: shape %d-%d-%d outside the fused kernels' range (dim <= 1024, h1 <= 256 and a multiple of 4, "
              "h2 <= 32)", s.dim, s.h1, s.h2);
  FusedTrainer* t = new FusedTrainer();
  t->s = s; t->o = mlp_offsets(s); t->loss = loss; t->adam = adam;
  t->max_rows = (max_rows + TR - 1) / TR * TR;
  const size_t R = t->max_rows, n3 = s.dim + 1;
  const int rc = trainer_alloc(t, [&](Carver& a) {
    t->sc = scalars_ext ? reinterpret_cast<FusedScalars*>(scalars_ext) : a.take<FusedScalars>(1);
    t->h1 = a.take<float>(R * s.h1);
    t->d_h1 = a.take<float>(R * s.h1);
    t->h2 = a.take<float>(R * s.h2);
    t->d_h2 = a.take<float>(R * s.h2);
    t->out = a.take<float>(R * n3);
    t->d_out = a.take<float>(R * n3);
    t->loss_reco = a.take<float>(R);
    t->raw = a.take<float>(R);
    t->grads = grads_ext ? grads_ext : a.take<float>(t->o.total + 1);   // + the confidence-weighted traversability sum
  }, "trainer");
  if (rc != WVN_OK) {
    delete t;
    return rc;
  }
  t->stats = &t->sc->sum_lr;
  {
    FusedScalars init;
    memset(&init, 0, sizeof(init));
    init.x_min = INFINITY;
    cudaMemcpy(t->sc, &init, sizeof(init), cudaMemcpyHostToDevice);
  }
  t->smem_fwd = sizeof(float) * (static_cast<size_t>(s.dim) * TR + std::max(KC * (s.h1 + 1), s.h1 * TRP) + s.h1 * TRP +
                                 s.h2 * TR + TR + TR);
  t->smem_bwd = sizeof(float) * (((n3 * TRP + 3) & ~size_t(3)) + s.h2 * TR + TR + 8);
  if (t->smem_fwd > 227 * 1024 || t->smem_bwd > 227 * 1024) {
    delete t;
    return set_error(WVN_ERR_INVALID, "trainer: shared memory need exceeds 227 KB");
  }
  cudaFuncSetAttribute(train_fwd_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(t->smem_fwd));
  cudaFuncSetAttribute(train_bwd_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(t->smem_bwd));
  *out = t;
  return WVN_OK;
}

int fused_train_step(Trainer* base, float* params, float* exp_avg, float* exp_avg_sq, long long* step_counter,
                     const float* x, int groups, int rpg, const int* n_rows, const float* y,
                     const unsigned char* y_valid, float* cg_mean, float* cg_std, float* conf_out, float* metrics,
                     int phase_mask, cudaStream_t stream) {
  WVN_PROPAGATE(trainer_check(base, TRAINER_MLP, "train step"));
  FusedTrainer* t = static_cast<FusedTrainer*>(base);
  WVN_REQUIRE(params && exp_avg && exp_avg_sq && step_counter && x && y && y_valid && conf_out,
              "train step: null argument");
  const long long rows = static_cast<long long>(groups) * rpg;
  WVN_REQUIRE(groups > 0 && rpg > 0 && rows <= t->max_rows, "train step: %d x %d rows exceed the trainer's capacity %d",
              groups, rpg, t->max_rows);
  const MlpShape& s = t->s;
  const int tiles = static_cast<int>((rows + TR - 1) / TR);
  const long long np = static_cast<long long>(t->o.total);
  if (phase_mask & 1) {
    // no memsets: the statistic sums were left clean by the previous step's K4 (by create for the first step)
    train_fwd_rows_kernel<<<tiles, kThreads, t->smem_fwd, stream>>>(s, t->o, params, x, y, y_valid, n_rows, groups, rpg,
                                                                   t->h1, t->h2, t->out, t->loss_reco, t->raw, t->sc,
                                                                   t->grads + np);
    WVN_CHECK_LAUNCH("train_fwd_rows_kernel");
    WVN_PROPAGATE(trainer_comm_stats(&t->comm, &t->sc->sum_lr, t->conf.cs.method == CONF_MOVING_AVERAGE, stream));
  }
  if (phase_mask & 2) {
    if (t->conf.cs.method != CONF_LATEST) {   // generators with memory: one thread updates the state once
      train_conf_kernel<<<1, 32, 0, stream>>>(t->loss, t->conf.cs, s.dim, t->sc, cg_mean, cg_std, step_counter);
      WVN_CHECK_LAUNCH("train_conf_kernel");
    }
    train_bwd_rows_kernel<<<tiles, kThreads, t->smem_bwd, stream>>>(
        s, t->o, t->loss, t->conf.cs.method, params, x, y, y_valid, n_rows, groups, rpg, t->h1, t->h2, t->out, t->loss_reco,
        t->raw, t->d_out, t->d_h2, t->d_h1, conf_out, t->sc, cg_mean, cg_std, t->grads + np, step_counter, t->grads, np);
    WVN_CHECK_LAUNCH("train_bwd_rows_kernel");
    WgradArgs w;
    const int n3 = s.dim + 1;
    w.p[0] = {t->d_out, n3, n3, t->h2, s.h2, s.h2, t->grads + t->o.w3, t->grads + t->o.b3, 0, 0, 0};
    w.p[1] = {t->d_h2, s.h2, s.h2, t->h1, s.h1, s.h1, t->grads + t->o.w2, t->grads + t->o.b2, 0, 0, 0};
    w.p[2] = {t->d_h1, s.h1, s.h1, x, s.dim, s.dim, t->grads + t->o.w1, t->grads + t->o.b1, 0, 0, 0};
    w.total_rows = static_cast<int>(rows);
    w.splits = rows >= 2048 ? 8 : (rows >= 512 ? 4 : (rows >= 128 ? 2 : 1));
    w.rows_per_split = ((w.total_rows + w.splits - 1) / w.splits + TK - 1) / TK * TK;
    w.n_rows = n_rows; w.groups = groups; w.rpg = rpg;
    int blocks = 0;
    for (int i = 0; i < 3; ++i) {
      w.p[i].tiles_m = (w.p[i].m + TS - 1) / TS;
      w.p[i].tiles_n = (w.p[i].n + TS - 1) / TS;
      w.p[i].first_block = blocks;
      blocks += w.p[i].tiles_m * w.p[i].tiles_n * w.splits;
    }
    train_wgrad_kernel<<<blocks, 256, 0, stream>>>(w);
    WVN_CHECK_LAUNCH("train_wgrad_kernel");
    WVN_PROPAGATE(trainer_comm_sum(&t->comm, t->grads, static_cast<size_t>(np + 1), false, stream));
  }
  if (phase_mask & 4) {
    int blocks = static_cast<int>((np + 255) / 256);
    if (blocks > sm_count() * 2) blocks = sm_count() * 2;
    train_apply_kernel<<<blocks, 256, 0, stream>>>(params, t->grads, exp_avg, exp_avg_sq, np, t->adam, t->loss,
                                                   step_counter, t->sc, metrics);
    WVN_CHECK_LAUNCH("train_apply_kernel");
  }
  return WVN_OK;
}

}  // namespace wvn
