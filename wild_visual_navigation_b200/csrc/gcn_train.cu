// wvn-b200: the SimpleGCN learner (model/simple_gcn.py) in fp32 — the graph build over each frame's segment adjacency,
// the forward on rows, and the online train step, the body of TraversabilityEstimator.train() with TraversabilityLoss
// on a SimpleGCN.
//
// Three GCNConv layers (torch_geometric 2.x defaults): Z = Â (X W^T) + b with Â = D^-1/2 (A + I) D^-1/2, A[i, j] the
// number of edges j -> i after dropping the input's self-loops, D = 1 + the in-degree.  The edges are kept as the
// segment reducer gives them (one directed pair per touching pair): a segment aggregates from its sources and itself.
// The output [sigmoid(Z3[:, 0]) | Z3[:, 1:]] has SimpleMLP's (rows, 1 + dim) layout, so the loss, its gradient and the
// confidence are the DoubleMLP step's kernels (recon_loss.cuh).  The step, with every scalar on the device:
//   1: compaction of the padded rows -> graph build (per frame: CSR by target and by source over the compacted rows,
//      with the edge weights d(j)^-1/2 d(i)^-1/2) -> gather of the live rows -> per layer one GEMM X W^T and one
//      aggregation (weighted CSR gather + self term + bias, then ReLU, or the sigmoid on column 0 for the last layer)
//      -> per-row loss terms -> this rank's statistic sums and extrema                [SUM of the sums, MIN / MAX]
//   2: generator update -> dLoss/dOut -> per layer the transposed aggregation Â^T dZ through the source CSR and the
//      data-gradient GEMM with ReLU's backward -> one launch of the three weight-gradient GEMMs -> one launch of the
//      three bias gradients (column sums of dZ) -> this rank's confidence-weighted error sum       [SUM of the gradient]
//   4: loss metrics -> Adam (mlp_adam_step).
// No edge crosses frames, so frames sharded across ranks give the global batch's step exactly.  Every output element
// and every sum is formed by one thread or one fixed reduction tree, with no atomics: two runs are bit-identical.
#include <stddef.h>
#include <string.h>

#include <algorithm>

#include "common.cuh"
#include "gcn_train.h"
#include "host_common.h"
#include "recon_loss.cuh"
#include "train_core.cuh"

namespace wvn {

namespace {

constexpr int kGraphThreads = 512;   // one block per frame
constexpr int kEdgeTile = 1024;      // edges staged in shared memory per pass
constexpr int kAggThreads = 128;     // one block per row, threads over the columns

// Per frame g (one block): the frame's first compacted row is the live-row count of the frames before it.  Valid edges
// are (s, d) with 0 <= s, d < n_rows[g] and s != d.  Both CSRs live in the frame's own slice [g * epg, (g + 1) * epg):
// the in-edges of a row are its slice's valid edges with that target, in edge order, after those with smaller targets
// (likewise the out-edges by source).  Each count and position is formed by one thread scanning the frame's edges.
__global__ void __launch_bounds__(kGraphThreads)
gcn_graph_kernel(const long long* __restrict__ edges, int epg, const int* __restrict__ n_edges,
                 const int* __restrict__ n_rows, int rpg, int* __restrict__ in_start, int* __restrict__ in_cnt,
                 int* __restrict__ out_start, int* __restrict__ out_cnt, int* __restrict__ in_src,
                 float* __restrict__ in_w, int* __restrict__ out_dst, float* __restrict__ out_w,
                 float* __restrict__ dinv, double* __restrict__ overflow) {
  __shared__ int2 tile[kEdgeTile];
  __shared__ int row0_s;
  const int g = blockIdx.x, t = threadIdx.x;
  auto live_rows = [&](int f) { return n_rows ? min(max(n_rows[f], 0), rpg) : rpg; };
  if (t == 0) {
    int r0 = 0;
    for (int f = 0; f < g; ++f) r0 += live_rows(f);
    row0_s = r0;
  }
  const int n = live_rows(g);
  int ne = n_edges[g];
  if (ne < 0) {
    if (t == 0) *overflow = 1.0;
    ne = 0;
  }
  ne = min(ne, epg);
  __syncthreads();
  const int row0 = row0_s;
  const long long* eg = edges + static_cast<long long>(g) * epg * 2;
  const long long slice = static_cast<long long>(g) * epg;
  auto load = [&](int e) {
    const long long s = eg[2 * e], d = eg[2 * e + 1];
    const bool ok = s >= 0 && s < n && d >= 0 && d < n && s != d;
    return ok ? make_int2(static_cast<int>(s), static_cast<int>(d)) : make_int2(-1, -1);
  };
  // pass 1: per row, in / out counts and the number of valid edges with a smaller target / source
  const int rows_per_thread = (n + kGraphThreads - 1) / kGraphThreads;
  int ci[4] = {0, 0, 0, 0}, cib[4] = {0, 0, 0, 0}, co[4] = {0, 0, 0, 0}, cob[4] = {0, 0, 0, 0};
  // this thread's rows t, t + 512, ..., four per pass over the frame's edges
  for (int base = 0; base < rows_per_thread; base += 4) {
    for (int k = 0; k < 4; ++k) ci[k] = cib[k] = co[k] = cob[k] = 0;
    for (int e0 = 0; e0 < ne; e0 += kEdgeTile) {
      const int m = min(kEdgeTile, ne - e0);
      __syncthreads();
      for (int e = t; e < m; e += kGraphThreads) tile[e] = load(e0 + e);
      __syncthreads();
      for (int e = 0; e < m; ++e) {
        const int2 v = tile[e];
        if (v.x < 0) continue;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int s = t + (base + k) * kGraphThreads;
          ci[k] += v.y == s; cib[k] += v.y < s;
          co[k] += v.x == s; cob[k] += v.x < s;
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int s = t + (base + k) * kGraphThreads;
      if (s >= n) continue;
      const int i = row0 + s;
      in_cnt[i] = ci[k]; in_start[i] = static_cast<int>(slice) + cib[k];
      out_cnt[i] = co[k]; out_start[i] = static_cast<int>(slice) + cob[k];
      dinv[i] = 1.f / sqrtf(static_cast<float>(1 + ci[k]));
    }
  }
  __syncthreads();   // dinv of every row of the frame is written (global memory, visible within the block)
  // pass 2: per valid edge, its position in the target-sorted and the source-sorted order (stable in edge order)
  for (int e = t; e - t < ne; e += kGraphThreads) {
    const int2 me = e < ne ? load(e) : make_int2(-1, -1);
    int pin = 0, pout = 0;
    for (int e0 = 0; e0 < ne; e0 += kEdgeTile) {
      const int m = min(kEdgeTile, ne - e0);
      __syncthreads();
      for (int k = t; k < m; k += kGraphThreads) tile[k] = load(e0 + k);
      __syncthreads();
      if (me.x >= 0) {
        for (int k = 0; k < m; ++k) {
          const int2 v = tile[k];
          if (v.x < 0) continue;
          const bool before = e0 + k < e;
          pin += v.y < me.y || (v.y == me.y && before);
          pout += v.x < me.x || (v.x == me.x && before);
        }
      }
    }
    if (me.x >= 0) {
      const float w = dinv[row0 + me.x] * dinv[row0 + me.y];
      in_src[slice + pin] = row0 + me.x;
      in_w[slice + pin] = w;
      out_dst[slice + pout] = row0 + me.y;
      out_w[slice + pout] = w;
    }
  }
}

// One side of the normalised adjacency: for row i, the rows it reads (nbr) with their weights, from start[i].
struct Csr {
  const int* start; const int* cnt; const int* nbr; const float* w; const float* dinv;
};

enum AggAct : int { AGG_LINEAR = 0, AGG_RELU = 1, AGG_SIGMOID_COL0 = 2 };

// out[i, c] = act( sum_{e in csr(i)} w_e y[nbr_e, c] + dinv[i]^2 y[i, c] + bias[c] ): the neighbours in CSR order,
// then the self-loop, then the bias.  Rows bounded by *n_live.  ReLU is fmaxf (NaN becomes 0).
__global__ void __launch_bounds__(kAggThreads)
gcn_aggregate_kernel(const float* __restrict__ y, int ncol, Csr csr, const float* __restrict__ bias, int act,
                     float* __restrict__ out, const int* __restrict__ n_live) {
  const int i = blockIdx.x;
  if (i >= *n_live) return;
  const int st = csr.start[i], cnt = csr.cnt[i];
  const float di = csr.dinv[i], self = di * di;
  const float* yi = y + static_cast<long long>(i) * ncol;
  float* o = out + static_cast<long long>(i) * ncol;
  for (int c = threadIdx.x; c < ncol; c += kAggThreads) {
    float acc = 0.f;
    for (int e = st; e < st + cnt; ++e) acc = fmaf(csr.w[e], y[static_cast<long long>(csr.nbr[e]) * ncol + c], acc);
    acc = fmaf(self, yi[c], acc);
    if (bias) acc += bias[c];
    if (act == AGG_RELU) acc = fmaxf(acc, 0.f);
    if (act == AGG_SIGMOID_COL0 && c == 0) acc = 1.f / (1.f + expf(-acc));
    o[c] = acc;
  }
}

// The bias gradients: out[c] = sum over the live rows of a[r, c], for up to three matrices (blockIdx.y).  32 columns
// per block; 8 row lanes each sum rows r = lane, lane + 8, ... in order, then lane 0 adds the 8 partial sums in order.
struct ColSum {
  const float* a; int ld, ncol; float* out;
};

__global__ void __launch_bounds__(256)
gcn_colsum_kernel(ColSum p0, ColSum p1, ColSum p2, const int* __restrict__ n_live) {
  __shared__ float red[8][33];
  const ColSum p = blockIdx.y == 0 ? p0 : (blockIdx.y == 1 ? p1 : p2);   // no dynamic index into the parameters
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5, c = blockIdx.x * 32 + tx, rows = *n_live;
  float acc = 0.f;
  if (c < p.ncol)
    for (int r = ty; r < rows; r += 8) acc += p.a[static_cast<long long>(r) * p.ld + c];
  red[ty][tx] = acc;
  __syncthreads();
  if (ty != 0 || c >= p.ncol) return;
  float s = red[0][tx];
  for (int k = 1; k < 8; ++k) s += red[k][tx];
  p.out[c] = s;
}

// Inference per live row (one warp): trav = out[r, 0], conf = inference_without_update(mean_d (out[r, 1 + d] - x)^2),
// written at the row's padded index.
__global__ void __launch_bounds__(kRowThreads)
gcn_infer_rows_kernel(const float* __restrict__ out, const float* __restrict__ x, const int* __restrict__ comp,
                      const int* __restrict__ n_live, int dim, const float* __restrict__ cg_mean,
                      const float* __restrict__ cg_std, float std_factor, float* __restrict__ trav,
                      float* __restrict__ conf) {
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
  if (lane != 0) return;
  const int p = comp[r];
  if (trav) trav[p] = o[0];
  if (conf) {
    const float m = *cg_mean, sd = *cg_std, shifted = m + sd * std_factor;
    conf[p] = row_confidence(CONF_LATEST, acc / static_cast<float>(dim), fmaxf(shifted - sd, 0.f), shifted + sd, 0.f,
                             0.f);
  }
}

// metrics[6]: 1 when some rank met a negative edge count (the statistics block's sixth sum, all-reduced with the others)
__global__ void gcn_overflow_metric_kernel(const DoubleScalars* __restrict__ sc, float* __restrict__ metrics) {
  if (threadIdx.x == 0) metrics[6] = sc->reserved > 0.0 ? 1.f : 0.f;
}

}  // namespace

// ------------------------------------------------------------------------------------------------ host side
GcnOffsets gcn_offsets(const MlpShape& s) {
  const size_t in[3] = {static_cast<size_t>(s.dim), static_cast<size_t>(s.h1), static_cast<size_t>(s.h2)};
  const size_t out[3] = {static_cast<size_t>(s.h1), static_cast<size_t>(s.h2), static_cast<size_t>(s.dim) + 1};
  GcnOffsets o;
  size_t off = 0;
  for (int l = 0; l < 3; ++l) {
    o.b[l] = off; off += out[l];
    o.w[l] = off; off += out[l] * in[l];
  }
  o.total = off;
  return o;
}

size_t gcn_param_count(const MlpShape& s) { return gcn_offsets(s).total; }

int gcn_check_shape(const MlpShape& s, const char* who) {
  WVN_REQUIRE(s.dim >= 1 && s.dim <= 1024 && s.h1 >= 1 && s.h1 <= 512 && s.h2 >= 1 && s.h2 <= 512,
              "%s: SimpleGCN(%d, True, [%d, %d, 1]) outside the kernels' range (1 <= dim <= 1024, 1 <= h1, h2 <= 512)",
              who, s.dim, s.h1, s.h2);
  return WVN_OK;
}

struct GcnTrainer : Trainer {
  GcnTrainer() : Trainer(TRAINER_GCN) {}
  MlpShape s;
  GcnOffsets o;
  int max_edges = 0;
  DoubleScalars* sc = nullptr;
  int* n_live = nullptr;
  double* overflow = nullptr;   // this rank's overflow flag, copied into the statistics block's sixth sum
  int* comp = nullptr;
  int *in_start = nullptr, *in_cnt = nullptr, *out_start = nullptr, *out_cnt = nullptr, *in_src = nullptr,
      *out_dst = nullptr;
  float *in_w = nullptr, *out_w = nullptr, *dinv = nullptr;
  // y_l = X_l W_l^T (forward), then Â^T dZ_l (backward); a_l = ReLU(Z_l); dz_l: dLoss/dZ_l (dz3 = d_out)
  float *xg = nullptr, *y1 = nullptr, *a1 = nullptr, *dz1 = nullptr, *y2 = nullptr, *a2 = nullptr, *dz2 = nullptr,
        *y3 = nullptr, *out = nullptr, *d_out = nullptr;
  float *loss_reco = nullptr, *raw = nullptr, *wraw = nullptr;
};

int gcn_trainer_create(const MlpShape& s, int max_rows, int max_edges, const LossCfg& loss, const AdamCfg& adam,
                       float* grads_ext, Trainer** out) {
  WVN_REQUIRE(out && max_rows > 0 && max_edges >= 0, "gcn trainer: bad arguments");
  WVN_PROPAGATE(gcn_check_shape(s, "gcn trainer"));
  GcnTrainer* t = new GcnTrainer();
  t->s = s; t->o = gcn_offsets(s); t->loss = loss; t->adam = adam;
  t->max_rows = max_rows;
  t->max_edges = max_edges;
  const size_t R = max_rows, E = std::max(max_edges, 1), D = s.dim, h1 = s.h1, h2 = s.h2, n3 = D + 1;
  const int rc = trainer_alloc(t, [&](Carver& a) {
    t->sc = a.take<DoubleScalars>(1);
    t->n_live = a.take<int>(1);
    t->overflow = a.take<double>(1);
    t->comp = a.take<int>(R);
    t->in_start = a.take<int>(R); t->in_cnt = a.take<int>(R);
    t->out_start = a.take<int>(R); t->out_cnt = a.take<int>(R);
    t->in_src = a.take<int>(E); t->out_dst = a.take<int>(E);
    t->dinv = a.take<float>(R);
    t->in_w = a.take<float>(E); t->out_w = a.take<float>(E);
    t->xg = a.take<float>(R * D);
    t->y1 = a.take<float>(R * h1); t->a1 = a.take<float>(R * h1); t->dz1 = a.take<float>(R * h1);
    t->y2 = a.take<float>(R * h2); t->a2 = a.take<float>(R * h2); t->dz2 = a.take<float>(R * h2);
    t->y3 = a.take<float>(R * n3); t->out = a.take<float>(R * n3); t->d_out = a.take<float>(R * n3);
    t->loss_reco = a.take<float>(R); t->raw = a.take<float>(R); t->wraw = a.take<float>(R);
    t->grads = grads_ext ? grads_ext : a.take<float>(t->o.total);
  }, "gcn trainer");
  if (rc != WVN_OK) {
    delete t;
    return rc;
  }
  t->stats = &t->sc->sum_lr;
  t->n_stats = kStatDoubles + 1;
  *out = t;
  return WVN_OK;
}

namespace {

int check_geometry(const GcnTrainer* t, int groups, int rows_per_group, const long long* edges, int epg,
                   const int* n_edges, const char* who) {
  const long long cap = static_cast<long long>(groups) * rows_per_group;
  WVN_REQUIRE(groups > 0 && rows_per_group > 0 && cap <= t->max_rows, "%s: %d x %d rows outside (0, %d]", who, groups,
              rows_per_group, t->max_rows);
  WVN_REQUIRE(epg >= 0 && static_cast<long long>(groups) * epg <= t->max_edges && n_edges && (edges || epg == 0),
              "%s: %d x %d edges outside [0, %d] or no edge counts", who, groups, epg, t->max_edges);
  return WVN_OK;
}

// compaction, graph build, gather and the three layers: out [live rows, 1 + dim]
int forward(GcnTrainer* t, const float* params, const float* x, int groups, int rows_per_group, const int* n_rows,
            const long long* edges, int epg, const int* n_edges, cudaStream_t stream) {
  const MlpShape& s = t->s;
  const GcnOffsets& o = t->o;
  const int D = s.dim, h1 = s.h1, h2 = s.h2, n3 = D + 1, rows = groups * rows_per_group;
  WVN_PROPAGATE(compact_rows(groups, rows_per_group, n_rows, nullptr, t->comp, t->n_live, stream));
  WVN_CHECK_CUDA(cudaMemsetAsync(t->overflow, 0, sizeof(double), stream));
  gcn_graph_kernel<<<groups, kGraphThreads, 0, stream>>>(edges, epg, n_edges, n_rows, rows_per_group, t->in_start,
                                                          t->in_cnt, t->out_start, t->out_cnt, t->in_src, t->in_w,
                                                          t->out_dst, t->out_w, t->dinv, t->overflow);
  WVN_CHECK_LAUNCH("gcn_graph_kernel");
  const int row_blocks = (rows * 32 + kRowThreads - 1) / kRowThreads;
  double_gather_kernel<<<row_blocks, kRowThreads, 0, stream>>>(x, t->comp, t->n_live, D, t->xg);
  WVN_CHECK_LAUNCH("double_gather_kernel");
  const Csr in{t->in_start, t->in_cnt, t->in_src, t->in_w, t->dinv};
  const float* xin[3] = {t->xg, t->a1, t->a2};
  float* y[3] = {t->y1, t->y2, t->y3};
  float* z[3] = {t->a1, t->a2, t->out};
  const int nin[3] = {D, h1, h2}, nout[3] = {h1, h2, n3};
  for (int l = 0; l < 3; ++l) {
    const GemmProblem p = gemm_problem(xin[l], nin[l], 1, params + o.w[l], 1, nin[l], y[l], nout[l], rows, nout[l],
                                       nin[l], 1);
    WVN_PROPAGATE(launch_gemms(&p, 1, t->n_live, stream));
    gcn_aggregate_kernel<<<rows, kAggThreads, 0, stream>>>(y[l], nout[l], in, params + o.b[l],
                                                            l == 2 ? AGG_SIGMOID_COL0 : AGG_RELU, z[l], t->n_live);
    WVN_CHECK_LAUNCH("gcn_aggregate_kernel");
  }
  return WVN_OK;
}

}  // namespace

int gcn_train_step_padded(Trainer* base, float* params, float* exp_avg, float* exp_avg_sq, long long* step_counter,
                          const float* x, int groups, int rows_per_group, const int* n_rows, const long long* edges,
                          int edges_per_group, const int* n_edges, const float* y, const unsigned char* y_valid,
                          float* cg_mean, float* cg_std, float* conf_out, float* metrics, int phase_mask,
                          cudaStream_t stream) {
  WVN_PROPAGATE(trainer_check(base, TRAINER_GCN, "gcn train step"));
  GcnTrainer* t = static_cast<GcnTrainer*>(base);
  WVN_REQUIRE(params && exp_avg && exp_avg_sq && step_counter && x && y && y_valid && conf_out,
              "gcn train step: null argument");
  WVN_PROPAGATE(check_geometry(t, groups, rows_per_group, edges, edges_per_group, n_edges, "gcn train step"));
  const MlpShape& s = t->s;
  const GcnOffsets& o = t->o;
  const int D = s.dim, h1 = s.h1, h2 = s.h2, n3 = D + 1, rows = groups * rows_per_group;
  const int row_blocks = (rows * 32 + kRowThreads - 1) / kRowThreads;
  if (phase_mask & 1) {
    WVN_PROPAGATE(forward(t, params, x, groups, rows_per_group, n_rows, edges, edges_per_group, n_edges, stream));
    double_loss_rows_kernel<<<row_blocks, kRowThreads, 0, stream>>>(t->out, t->xg, y, t->loss_reco, t->raw, t->n_live, D);
    WVN_CHECK_LAUNCH("double_loss_rows_kernel");
    double_stats_kernel<<<1, kStatThreads, 0, stream>>>(t->loss_reco, t->raw, y_valid, t->n_live, t->sc);
    WVN_CHECK_LAUNCH("double_stats_kernel");
    WVN_CHECK_CUDA(cudaMemcpyAsync(&t->sc->reserved, t->overflow, sizeof(double), cudaMemcpyDeviceToDevice, stream));
    WVN_PROPAGATE(trainer_comm_stats(&t->comm, &t->sc->sum_lr, t->conf.cs.method == CONF_MOVING_AVERAGE, stream));
  }
  if (phase_mask & 2) {
    double_conf_kernel<<<1, 32, 0, stream>>>(D, t->loss, t->conf.cs, cg_mean, cg_std, t->sc);
    WVN_CHECK_LAUNCH("double_conf_kernel");
    double_dout_kernel<<<row_blocks, kRowThreads, 0, stream>>>(t->out, t->xg, y, y_valid, t->loss_reco, t->raw, t->sc,
                                                               t->loss, t->conf.cs.method, t->d_out, conf_out, t->wraw,
                                                               t->n_live, D);
    WVN_CHECK_LAUNCH("double_dout_kernel");
    const Csr outc{t->out_start, t->out_cnt, t->out_dst, t->out_w, t->dinv};
    // layer l: y_l = Â^T dz_l, then dz_{l-1} = (y_l W_l) * (a_{l-1} > 0)
    float* dz[3] = {t->dz1, t->dz2, t->d_out};
    float* yb[3] = {t->y1, t->y2, t->y3};
    const float* act[3] = {t->xg, t->a1, t->a2};
    const int nin[3] = {D, h1, h2}, nout[3] = {h1, h2, n3};
    for (int l = 2; l >= 0; --l) {
      gcn_aggregate_kernel<<<rows, kAggThreads, 0, stream>>>(dz[l], nout[l], outc, nullptr, AGG_LINEAR, yb[l], t->n_live);
      WVN_CHECK_LAUNCH("gcn_aggregate_kernel");
      if (l == 0) break;
      GemmProblem p = gemm_problem(yb[l], nout[l], 1, params + o.w[l], nin[l], 1, dz[l - 1], nin[l], rows, nin[l],
                                   nout[l], 1);
      p.ref = act[l]; p.ld_ref = nin[l];
      WVN_PROPAGATE(launch_gemms(&p, 1, t->n_live, stream));
    }
    // dW_l = y_l^T X_l, the row reduction (K) bounded by *n_live
    GemmProblem wg[3];
    for (int l = 0; l < 3; ++l)
      wg[l] = gemm_problem(yb[l], 1, nout[l], act[l], nin[l], 1, t->grads + o.w[l], nin[l], nout[l], nin[l], rows, 2);
    WVN_PROPAGATE(launch_gemms(wg, 3, t->n_live, stream));
    ColSum cs[3];
    for (int l = 0; l < 3; ++l) cs[l] = ColSum{dz[l], nout[l], nout[l], t->grads + o.b[l]};
    gcn_colsum_kernel<<<dim3((std::max(std::max(h1, h2), n3) + 31) / 32, 3), 256, 0, stream>>>(cs[0], cs[1], cs[2],
                                                                                               t->n_live);
    WVN_CHECK_LAUNCH("gcn_colsum_kernel");
    double_trav_w_kernel<<<1, kStatThreads, 0, stream>>>(t->wraw, t->n_live, t->sc);
    WVN_CHECK_LAUNCH("double_trav_w_kernel");
    WVN_PROPAGATE(trainer_comm_sum(&t->comm, t->grads, o.total, false, stream));
    WVN_PROPAGATE(trainer_comm_sum(&t->comm, &t->sc->trav_w, 1, true, stream));
  }
  if (phase_mask & 4) {
    if (metrics) {
      double_finish_kernel<<<1, 32, 0, stream>>>(t->loss, t->sc, metrics);
      WVN_CHECK_LAUNCH("double_finish_kernel");
      gcn_overflow_metric_kernel<<<1, 32, 0, stream>>>(t->sc, metrics);
      WVN_CHECK_LAUNCH("gcn_overflow_metric_kernel");
    }
    WVN_PROPAGATE(mlp_adam_step(params, t->grads, exp_avg, exp_avg_sq, static_cast<long long>(o.total), t->adam,
                                step_counter, stream));
  }
  return WVN_OK;
}

int gcn_infer_rows(Trainer* base, const float* params, const float* x, int groups, int rows_per_group,
                   const int* n_rows, const long long* edges, int edges_per_group, const int* n_edges,
                   const float* cg_mean, const float* cg_std, float std_factor, float* out, float* trav, float* conf,
                   cudaStream_t stream) {
  WVN_PROPAGATE(trainer_check(base, TRAINER_GCN, "gcn infer rows"));
  GcnTrainer* t = static_cast<GcnTrainer*>(base);
  WVN_REQUIRE(params && x && (!conf || (cg_mean && cg_std)), "gcn infer rows: null argument");
  WVN_PROPAGATE(check_geometry(t, groups, rows_per_group, edges, edges_per_group, n_edges, "gcn infer rows"));
  const int D = t->s.dim, rows = groups * rows_per_group;
  WVN_PROPAGATE(forward(t, params, x, groups, rows_per_group, n_rows, edges, edges_per_group, n_edges, stream));
  if (trav || conf) {
    gcn_infer_rows_kernel<<<(rows * 32 + kRowThreads - 1) / kRowThreads, kRowThreads, 0, stream>>>(
        t->out, t->xg, t->comp, t->n_live, D, cg_mean, cg_std, std_factor, trav, conf);
    WVN_CHECK_LAUNCH("gcn_infer_rows_kernel");
  }
  if (out) {
    WVN_CHECK_CUDA(cudaMemcpyAsync(out, t->out, sizeof(float) * rows * (D + 1), cudaMemcpyDeviceToDevice, stream));
  }
  return WVN_OK;
}

}  // namespace wvn
