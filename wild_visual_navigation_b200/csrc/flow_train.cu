// wvn-b200: the LinearRnvp normalising flow (model/linear_rnvp.py) in fp32 — the row forward and the online train step
// of the anomaly-detection learner (TraversabilityEstimator(anomaly_detection=True).train(), traversability_estimator.py
// :464-477 with AnomalyLoss, utils/loss.py:16-54).
//
// Coupling forward (every coupling, mask m, nets S and T):   mu = u * m,  s = tanh(S(mu)),  t = T(mu)
//   x = mu + (1 - m) * (u * exp(s) + t),   log_det += sum((1 - m) * s),   then the permutation x = x[:, p].
// Loss: NLL_r = -(sum_j log N(z_rj; 0, 1) + log_det_r), loss = mean_r NLL_r; the ConfidenceGenerator is updated with
// x = x_positive = NLL over the (labelled) rows of the batch.
//
// The step is one fixed sequence of ~25 launches with every scalar on the device (no host synchronisation):
//   compact (the live rows of padded groups whose y_valid is set, train_core) -> gather -> per coupling 3 batched GEMMs
//   (s | t) + the coupling kernel -> NLL sums [data-parallel: all-reduced] -> confidence update (train_core.cuh) +
//   per-row confidence -> per coupling (last first): dx / ds / dt, 2-3 batched
//   data-gradient GEMMs, du -> one batched launch of all 12 weight-gradient products (+ bias gradients) [data-parallel:
//   the gradient all-reduced] -> Adam
//   (mlp_adam_step).  The GEMMs, Adam and the generator's state are the training core shared with the MLP trainers
//   (train_core.h / train_core.cuh).
// Training batches are small (~8 nodes x ~16 labelled segments), so the step is latency-bound: the GEMMs are plain
// fp32 CUDA-core tiles, every output element is summed by one thread in a fixed order (no atomics: bit-reproducible).
// The weight-gradient columns that see masked-out inputs (mu = 0) and the last-layer rows that feed masked-out outputs
// ((1 - m) = 0) come out as exact zeros, as in the reference, so Adam leaves those parameters bit-identical.
#include <cuda_bf16.h>
#include <stddef.h>
#include <string.h>

#include <algorithm>
#include <memory>

#include "common.cuh"
#include "flow_train.h"
#include "gemm.h"
#include "host_common.h"
#include "train_core.cuh"

namespace wvn {

namespace {

constexpr float kLogSqrt2Pi = 0.91893853320467274178f;   // math.log(math.sqrt(2 * math.pi)), torch.distributions.Normal
constexpr int kRowThreads = 128;
constexpr int kStatThreads = 256;

// u0 = x[comp], mu0 = u0 * mask
__global__ void __launch_bounds__(kRowThreads)
flow_gather_kernel(const float* __restrict__ x, const int* __restrict__ comp, const int* __restrict__ n_live, int dim,
                   const float* __restrict__ mask, float* __restrict__ u0, float* __restrict__ mu0) {
  const int r = blockIdx.x;
  if (r >= *n_live) return;
  const float* xr = x + static_cast<long long>(comp[r]) * dim;
  for (int j = threadIdx.x; j < dim; j += kRowThreads) {
    const float u = xr[j];
    u0[static_cast<long long>(r) * dim + j] = u;
    mu0[static_cast<long long>(r) * dim + j] = u * mask[j];
  }
}

// ------------------------------------------------------------------------------------------------ coupling forward
// One block per live row.  In: u, mu, the nets' outputs so (overwritten by s = tanh(so)) and to.  Out: the permuted
// x as the next coupling's u (+ its mu = u * next_mask), or for the last coupling z, log N(z; 0, 1), the NLL and, with
// trav set, the confidence of the NLL under the generator (inference_without_update).  ld_in / ld_out: log_det so far.
struct CouplingFwd {
  const float* u; const float* mu; const float* mask; float* so; const float* to; const long long* perm;
  const float* next_mask; float* u_next; float* mu_next;
  const float* ld_in; float* ld_out;
  float* z; float* logprob; float* nll;
  const float* cg_mean; const float* cg_std; float std_factor; float* trav;
};

__global__ void __launch_bounds__(kRowThreads)
flow_coupling_fwd_kernel(CouplingFwd c, int dim, const int* __restrict__ n_live) {
  const int r = blockIdx.x;
  if (r >= *n_live) return;
  extern __shared__ float xs[];   // [dim] the un-permuted coupling output of this row
  __shared__ float red[kRowThreads / 32];
  const long long base = static_cast<long long>(r) * dim;
  float ld = 0.f;
  for (int j = threadIdx.x; j < dim; j += kRowThreads) {
    const float m = c.mask[j], om = 1.f - m;
    const float s = tanhf(c.so[base + j]);
    c.so[base + j] = s;
    xs[j] = c.mu[base + j] + om * (c.u[base + j] * expf(s) + c.to[base + j]);
    ld += om * s;
  }
  ld = warp_sum(ld);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ld;
  __syncthreads();
  float ldr = 0.f;
#pragma unroll
  for (int w = 0; w < kRowThreads / 32; ++w) ldr += red[w];
  const float ld_total = c.ld_in ? c.ld_in[r] + ldr : ldr;
  if (c.z == nullptr) {
    for (int j = threadIdx.x; j < dim; j += kRowThreads) {
      const float v = xs[c.perm[j]];
      c.u_next[base + j] = v;
      c.mu_next[base + j] = v * c.next_mask[j];
    }
    if (threadIdx.x == 0) c.ld_out[r] = ld_total;
    return;
  }
  float lps = 0.f;
  for (int j = threadIdx.x; j < dim; j += kRowThreads) {
    const float v = xs[c.perm[j]];
    c.z[base + j] = v;
    const float lp = -(v * v) * 0.5f - kLogSqrt2Pi;   // Normal(0, 1).log_prob: -((z - 0)^2) / (2 * 1^2) - log(1) - log(sqrt(2 pi))
    if (c.logprob) c.logprob[base + j] = lp;
    lps += lp;
  }
  __syncthreads();   // red reused
  lps = warp_sum(lps);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = lps;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < kRowThreads / 32; ++w) s += red[w];
    const float nll = -(s + ld_total);
    if (c.ld_out) c.ld_out[r] = ld_total;
    if (c.nll) c.nll[r] = nll;
    if (c.trav) {   // ConfidenceGenerator.inference_without_update (confidence_generator.py:146-154)
      const float m = *c.cg_mean, sd = *c.cg_std, shifted = m + sd * c.std_factor;
      c.trav[r] = row_confidence(CONF_LATEST, nll, fmaxf(shifted - sd, 0.f), shifted + sd, 0.f, 0.f);
    }
  }
}

// ------------------------------------------------------------------------------------------------ statistics + confidence
// The first kStatDoubles are the statistics block every trainer exchanges (train_core.h): the sum of the NLL over the
// labelled rows, the sum of its squares, their number, then the NLL's extrema.
struct FlowScalars {
  double s1, s2, n, reserved[3], x_min, x_max;
  float inv_n;
  float lo, hi, cmin, cmax;   // the updated generator, for the per-row confidence (train_core.cuh)
};
static_assert(offsetof(FlowScalars, x_min) == kStatSums * sizeof(double) &&
              offsetof(FlowScalars, inv_n) == kStatDoubles * sizeof(double), "statistics block layout");

// One block of kStatThreads: this rank's sums / extrema of the NLL over its labelled rows.
__global__ void __launch_bounds__(kStatThreads, 1)
flow_sums_kernel(const float* __restrict__ nll, const int* __restrict__ n_live, FlowScalars* __restrict__ sc) {
  __shared__ double r1[kStatThreads / 32], r2[kStatThreads / 32];
  __shared__ float rmin[kStatThreads / 32], rmax[kStatThreads / 32];
  const int n = *n_live, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  double s1 = 0.0, s2 = 0.0;
  float mn = INFINITY, mx = -INFINITY;
  for (int i = t; i < n; i += kStatThreads) {
    const float v = nll[i];
    s1 += v;
    s2 += static_cast<double>(v) * v;
    mn = fminf(mn, v);
    mx = fmaxf(mx, v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if (lane == 0) { r1[warp] = s1; r2[warp] = s2; rmin[warp] = mn; rmax[warp] = mx; }
  __syncthreads();
  if (t != 0) return;
  double S1 = 0.0, S2 = 0.0;
  float MN = INFINITY, MX = -INFINITY;
  for (int w = 0; w < kStatThreads / 32; ++w) { S1 += r1[w]; S2 += r2[w]; MN = fminf(MN, rmin[w]); MX = fmaxf(MX, rmax[w]); }
  sc->s1 = S1; sc->s2 = S2; sc->n = static_cast<double>(n);
  sc->reserved[0] = sc->reserved[1] = sc->reserved[2] = 0.0;
  sc->x_min = MN; sc->x_max = MX;
}

// One thread: the generator update from the (all-reduced) sums, the metrics and the loss gradient scale 1 / n for the
// backward kernels.
__global__ void flow_conf_kernel(ConfState cs, float std_factor, float* __restrict__ cg_mean, float* __restrict__ cg_std,
                                 float* __restrict__ metrics, FlowScalars* __restrict__ sc) {
  if (threadIdx.x != 0) return;
  const double S1 = sc->s1, dn = sc->n;
  const ConfUpdate u = conf_generator_update(cs, std_factor, dn, S1, sc->s2, sc->x_min, sc->x_max, cg_mean);
  if (cg_mean) *cg_mean = u.mean;
  if (cg_std) *cg_std = u.std;
  sc->lo = u.lo; sc->hi = u.hi; sc->cmin = u.cmin; sc->cmax = u.cmax;
  sc->inv_n = 1.f / static_cast<float>(dn);   // d mean / d NLL_r (n == 0: no row reads it)
  if (metrics) {
    metrics[0] = static_cast<float>(S1 / dn);   // loss = -mean(logprob.sum(1) + log_det); NaN for an empty batch
    metrics[1] = 0.f;                            // AnomalyLoss reports loss_trav = loss_reco = 0
    metrics[2] = 0.f;
    metrics[3] = static_cast<float>(dn);
    metrics[4] = u.mean;
    metrics[5] = u.std;
  }
}

// what ConfidenceGenerator.update returns: the confidence of every live row's NLL
__global__ void __launch_bounds__(256)
flow_conf_rows_kernel(const float* __restrict__ nll, const int* __restrict__ n_live, int method,
                      const FlowScalars* __restrict__ sc, float* __restrict__ conf_out) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < *n_live) conf_out[i] = row_confidence(method, nll[i], sc->lo, sc->hi, sc->cmin, sc->cmax);
}

// ------------------------------------------------------------------------------------------------ coupling backward
// dx = dL/d(coupling output, before its permutation): for the last coupling z[invp] / n, otherwise the next coupling's
// du[invp].  With g = (1 - m) dx:  dt = g,  ds = g u exp(s) + (1 - m) dlog_det,  dso = ds (1 - s^2);  dlog_det = -1/n.
__global__ void __launch_bounds__(kRowThreads)
flow_coupling_bwd_pre_kernel(int dim, const int* __restrict__ n_live, const FlowScalars* __restrict__ sc,
                             const float* __restrict__ z, const float* __restrict__ du_next,
                             const long long* __restrict__ invp, const float* __restrict__ u,
                             const float* __restrict__ s, const float* __restrict__ mask, float* __restrict__ dx_out,
                             float* __restrict__ dso, float* __restrict__ dto) {
  const int r = blockIdx.x;
  if (r >= *n_live) return;
  const float g = sc->inv_n, dld = -g;
  const long long base = static_cast<long long>(r) * dim;
  for (int i = threadIdx.x; i < dim; i += kRowThreads) {
    const long long src = base + invp[i];
    const float dx = z ? z[src] * g : du_next[src];
    const float om = 1.f - mask[i];
    const float sv = s[base + i];
    const float gx = om * dx;
    const float ds = gx * u[base + i] * expf(sv) + om * dld;
    dx_out[base + i] = dx;
    dto[base + i] = gx;
    dso[base + i] = ds * (1.f - sv * sv);
  }
}

// du = (1 - m) dx exp(s) + m (dx + dmu_s + dmu_t)  (mu = u * m feeds the coupling output directly and both nets)
__global__ void __launch_bounds__(kRowThreads)
flow_coupling_bwd_post_kernel(int dim, const int* __restrict__ n_live, const float* __restrict__ dx,
                              const float* __restrict__ s, const float* __restrict__ mask,
                              const float* __restrict__ dmu_s, const float* __restrict__ dmu_t, float* __restrict__ du) {
  const int r = blockIdx.x;
  if (r >= *n_live) return;
  const long long base = static_cast<long long>(r) * dim;
  for (int i = threadIdx.x; i < dim; i += kRowThreads) {
    const float m = mask[i], d = dx[base + i];
    du[base + i] = (1.f - m) * d * expf(s[base + i]) + m * (d + dmu_s[base + i] + dmu_t[base + i]);
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------------ host side
size_t flow_net_params(const FlowShape& s) {
  const size_t D = s.dim, h = s.hidden;
  return h * D + h + h * h + h + D * h + D;
}
size_t flow_param_count(const FlowShape& s) { return 4 * flow_net_params(s); }

namespace {
struct NetOffsets {
  size_t w0, b0, w2, b2, w4, b4;
};
NetOffsets net_offsets(const FlowShape& s, int coupling, int net) {
  const size_t D = s.dim, h = s.hidden;
  NetOffsets o;
  o.w0 = (2 * coupling + net) * flow_net_params(s);
  o.b0 = o.w0 + h * D;
  o.w2 = o.b0 + h;
  o.b2 = o.w2 + h * h;
  o.w4 = o.b2 + h;
  o.b4 = o.w4 + D * h;
  return o;
}
}  // namespace

struct FlowTrainer : Trainer {
  FlowTrainer() : Trainer(TRAINER_FLOW) {}
  FlowShape s;
  int* comp = nullptr;
  int* n_live = nullptr;
  FlowScalars* sc = nullptr;
  // activations (rows x width)
  float *u[2], *mu[2], *s1[2][2], *s2[2][2], *so[2][2];   // [coupling][net]; so[c][0] holds s = tanh after the forward
  float *z, *ld, *nll;
  // gradients
  float *dx = nullptr, *dso[2] = {nullptr, nullptr}, *d2[2] = {nullptr, nullptr}, *d1[2] = {nullptr, nullptr},
        *dmu[2] = {nullptr, nullptr}, *du = nullptr;
  bool forward_only = false;   // inference: no backward workspaces, no gradient buffer
};

int flow_trainer_create(const FlowShape& s, int max_rows, float std_factor, const AdamCfg& adam, float* grads_ext,
                        bool forward_only, Trainer** out) {
  WVN_REQUIRE(out && max_rows > 0, "flow trainer: bad arguments");
  WVN_REQUIRE(s.dim >= 2 && s.dim <= 4096 && s.hidden >= 8 && s.hidden <= 512 && s.hidden % 8 == 0,
              "flow trainer: LinearRnvp(%d, [%d]) outside the kernels' range (2 <= dim <= 4096, hidden <= 512 and a "
              "multiple of 8)", s.dim, s.hidden);
  FlowTrainer* t = new FlowTrainer();
  t->s = s; t->adam = adam; t->loss.std_factor = std_factor; t->forward_only = forward_only;
  t->max_rows = (max_rows + 63) / 64 * 64;   // whole 64-row GEMM tiles
  const size_t R = t->max_rows, D = s.dim, h = s.hidden, np = flow_param_count(s);
  const int rc = trainer_alloc(t, [&](Carver& a) {
    t->sc = a.take<FlowScalars>(1);
    t->n_live = a.take<int>(1);
    t->comp = a.take<int>(R + 1);
    for (int c = 0; c < 2; ++c) {
      t->u[c] = a.take<float>(R * D);
      t->mu[c] = a.take<float>(R * D);
      for (int k = 0; k < 2; ++k) {
        t->s1[c][k] = a.take<float>(R * h);
        t->s2[c][k] = a.take<float>(R * h);
        t->so[c][k] = a.take<float>(R * D);
      }
    }
    t->z = a.take<float>(R * D);
    t->ld = a.take<float>(R);
    t->nll = a.take<float>(R);
    if (forward_only) return;
    t->dx = a.take<float>(R * D);
    t->du = a.take<float>(R * D);
    for (int k = 0; k < 2; ++k) {
      t->dso[k] = a.take<float>(R * D);
      t->d2[k] = a.take<float>(R * h);
      t->d1[k] = a.take<float>(R * h);
      t->dmu[k] = a.take<float>(R * D);
    }
    t->grads = grads_ext ? grads_ext : a.take<float>(np);
  }, "flow trainer");
  if (rc != WVN_OK) {
    delete t;
    return rc;
  }
  t->stats = &t->sc->s1;
  *out = t;
  return WVN_OK;
}

namespace {

// compaction of the padded rows (train_core) + both couplings' forward on the kept rows, `rows` = groups * rpg of
// them at most; the last coupling writes z / logprob / log_det / nll / trav as given
int flow_forward(FlowTrainer* t, const float* params, const FlowBuffers& b, const float* x, int groups, int rpg,
                 const int* n_rows, const unsigned char* y_valid, float* z, float* logprob, float* ld_out, float* trav,
                 const float* cg_mean, const float* cg_std, float std_factor, cudaStream_t stream) {
  const int D = t->s.dim, h = t->s.hidden, rows = groups * rpg;
  WVN_PROPAGATE(compact_rows(groups, rpg, n_rows, y_valid, t->comp, t->n_live, stream));
  if (rows == 0) return WVN_OK;
  flow_gather_kernel<<<rows, kRowThreads, 0, stream>>>(x, t->comp, t->n_live, D, b.mask0, t->u[0], t->mu[0]);
  WVN_CHECK_LAUNCH("flow_gather_kernel");
  for (int c = 0; c < 2; ++c) {
    GemmProblem ps[2];
    for (int k = 0; k < 2; ++k) {
      const NetOffsets o = net_offsets(t->s, c, k);
      ps[k] = gemm_problem(t->mu[c], D, 1, params + o.w0, 1, D, t->s1[c][k], h, rows, h, D, 1);
      ps[k].bias = params + o.b0;
      ps[k].act = F32_RELU;
    }
    WVN_PROPAGATE(launch_gemms(ps, 2, t->n_live, stream));
    for (int k = 0; k < 2; ++k) {
      const NetOffsets o = net_offsets(t->s, c, k);
      ps[k] = gemm_problem(t->s1[c][k], h, 1, params + o.w2, 1, h, t->s2[c][k], h, rows, h, h, 1);
      ps[k].bias = params + o.b2;
      ps[k].act = F32_RELU;
    }
    WVN_PROPAGATE(launch_gemms(ps, 2, t->n_live, stream));
    for (int k = 0; k < 2; ++k) {
      const NetOffsets o = net_offsets(t->s, c, k);
      ps[k] = gemm_problem(t->s2[c][k], h, 1, params + o.w4, 1, h, t->so[c][k], D, rows, D, h, 1);
      ps[k].bias = params + o.b4;
    }
    WVN_PROPAGATE(launch_gemms(ps, 2, t->n_live, stream));
    CouplingFwd cf;
    memset(&cf, 0, sizeof(cf));
    cf.u = t->u[c]; cf.mu = t->mu[c]; cf.mask = c == 0 ? b.mask0 : b.mask1;
    cf.so = t->so[c][0]; cf.to = t->so[c][1];
    cf.perm = c == 0 ? b.p1 : b.p3;
    if (c == 0) {
      cf.next_mask = b.mask1; cf.u_next = t->u[1]; cf.mu_next = t->mu[1];
      cf.ld_out = t->ld;
    } else {
      cf.ld_in = t->ld;
      cf.ld_out = ld_out ? ld_out : t->ld;
      cf.z = z ? z : t->z;
      cf.logprob = logprob;
      cf.nll = t->nll;
      cf.cg_mean = cg_mean; cf.cg_std = cg_std; cf.std_factor = std_factor; cf.trav = trav;
    }
    flow_coupling_fwd_kernel<<<rows, kRowThreads, D * sizeof(float), stream>>>(cf, D, t->n_live);
    WVN_CHECK_LAUNCH("flow_coupling_fwd_kernel");
  }
  return WVN_OK;
}

int check_args(FlowTrainer* t, const float* params, const FlowBuffers& b, const float* x, int rows) {
  WVN_REQUIRE(params && b.mask0 && b.mask1 && b.p1 && b.invp1 && b.p3 && b.invp3, "flow: null argument");
  WVN_REQUIRE(rows >= 0 && rows <= t->max_rows, "flow: %d rows exceed the handle's capacity %d", rows, t->max_rows);
  WVN_REQUIRE(rows == 0 || x, "flow: null rows");
  WVN_REQUIRE(static_cast<size_t>(t->s.dim) * sizeof(float) <= 48 * 1024, "flow: dim too large");
  return WVN_OK;
}

}  // namespace

int flow_forward_rows(Trainer* base, const float* params, const FlowBuffers& b, const float* x, int rows, float* z,
                      float* log_det, float* logprob, const float* cg_mean, const float* cg_std, float std_factor,
                      float* trav, cudaStream_t stream) {
  WVN_PROPAGATE(trainer_check(base, TRAINER_FLOW, "flow rows"));
  FlowTrainer* t = static_cast<FlowTrainer*>(base);
  WVN_PROPAGATE(check_args(t, params, b, x, rows));
  WVN_REQUIRE(!trav || (cg_mean && cg_std), "flow rows: trav needs the generator's mean and std");
  return flow_forward(t, params, b, x, 1, rows, nullptr, nullptr, z, logprob, log_det, trav, cg_mean, cg_std, std_factor,
                      stream);
}

namespace {

__global__ void fill_nan_kernel(float* __restrict__ out, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    out[i] = __int_as_float(0x7fc00000);
}

// out[comp[r]] = in[r] for the n_live compacted rows
__global__ void scatter_live_rows_kernel(const float* __restrict__ in, const int* __restrict__ comp,
                                         const int* __restrict__ n_live, float* __restrict__ out) {
  const int n = *n_live;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) out[comp[r]] = in[r];
}

}  // namespace

int flow_forward_rows_padded(Trainer* base, const float* params, const FlowBuffers& b, const float* x, int groups,
                             int rows_per_group, const int* n_rows, const float* cg_mean, const float* cg_std,
                             float std_factor, float* trav, cudaStream_t stream) {
  WVN_PROPAGATE(trainer_check(base, TRAINER_FLOW, "flow rows padded"));
  FlowTrainer* t = static_cast<FlowTrainer*>(base);
  WVN_REQUIRE(groups >= 0 && rows_per_group >= 0 && static_cast<long long>(groups) * rows_per_group <= t->max_rows,
              "flow rows padded: %d x %d rows exceed the handle's capacity %d", groups, rows_per_group, t->max_rows);
  const int rows = groups * rows_per_group;
  WVN_PROPAGATE(check_args(t, params, b, x, rows));
  WVN_REQUIRE(n_rows && trav && cg_mean && cg_std, "flow rows padded: null argument");
  if (rows == 0) return WVN_OK;
  // The live rows are compacted and run as flow_forward_rows runs them.  Their trav lands in compacted order in u[0],
  // which nothing reads after the first coupling, and is scattered back to the padded positions.
  float* trav_c = t->u[0];
  WVN_PROPAGATE(flow_forward(t, params, b, x, groups, rows_per_group, n_rows, nullptr, nullptr, nullptr, nullptr, trav_c,
                             cg_mean, cg_std, std_factor, stream));
  const int blocks = std::min((rows + 255) / 256, 4096);
  fill_nan_kernel<<<blocks, 256, 0, stream>>>(trav, rows);
  WVN_CHECK_LAUNCH("fill_nan_kernel");
  scatter_live_rows_kernel<<<blocks, 256, 0, stream>>>(trav_c, t->comp, t->n_live, trav);
  WVN_CHECK_LAUNCH("scatter_live_rows_kernel");
  return WVN_OK;
}

namespace {

// The stages of a step.  The compacted entry's phase 1 runs kFwd | kGen, the padded entry's phase 2 kGen | kBwd: the
// statistics exchange sits between kFwd and kGen.
enum : int { kFwd = 1, kBwd = 2, kAdam = 4, kGen = 8 };

int flow_step(Trainer* base, float* params, float* exp_avg, float* exp_avg_sq, long long* step_counter,
              const FlowBuffers& b, const float* x, int groups, int rpg, const int* n_rows, const unsigned char* y_valid,
              float* cg_mean, float* cg_std, float* conf_out, float* metrics, int stages, cudaStream_t stream) {
  WVN_PROPAGATE(trainer_check(base, TRAINER_FLOW, "flow train step"));
  FlowTrainer* t = static_cast<FlowTrainer*>(base);
  WVN_REQUIRE(groups >= 0 && rpg >= 0, "flow train step: %d x %d rows", groups, rpg);
  const long long cap = static_cast<long long>(groups) * rpg;
  WVN_REQUIRE(cap <= t->max_rows, "flow: %lld rows exceed the handle's capacity %d", cap, t->max_rows);
  const int rows = static_cast<int>(cap);
  WVN_PROPAGATE(check_args(t, params, b, x, rows));
  WVN_REQUIRE(exp_avg && exp_avg_sq && step_counter && conf_out, "flow train step: null argument");
  WVN_REQUIRE(!t->forward_only, "flow train step: the handle was created for inference only");
  const int D = t->s.dim, h = t->s.hidden;
  const int R = std::max(rows, 1);
  if (stages & kFwd) {   // kept rows -> forward -> this rank's NLL sums (-> all-reduce)
    WVN_PROPAGATE(flow_forward(t, params, b, x, groups, rpg, n_rows, y_valid, nullptr, nullptr, nullptr, nullptr, nullptr,
                               nullptr, 0.f, stream));
    flow_sums_kernel<<<1, kStatThreads, 0, stream>>>(t->nll, t->n_live, t->sc);
    WVN_CHECK_LAUNCH("flow_sums_kernel");
    WVN_PROPAGATE(trainer_comm_stats(&t->comm, &t->sc->s1, t->conf.cs.method == CONF_MOVING_AVERAGE, stream));
  }
  if (stages & kGen) {   // generator update from the global sums, metrics, per-row confidence
    flow_conf_kernel<<<1, 32, 0, stream>>>(t->conf.cs, t->loss.std_factor, cg_mean, cg_std, metrics, t->sc);
    WVN_CHECK_LAUNCH("flow_conf_kernel");
    flow_conf_rows_kernel<<<(R + 255) / 256, 256, 0, stream>>>(t->nll, t->n_live, t->conf.cs.method, t->sc, conf_out);
    WVN_CHECK_LAUNCH("flow_conf_rows_kernel");
  }
  if (stages & kBwd) {   // the flat gradient, scaled by 1 / the global labelled count (-> all-reduce)
    // couplings in reverse; coupling 0 needs no input gradient
    for (int c = 1; c >= 0; --c) {
      const float* mask = c == 0 ? b.mask0 : b.mask1;
      flow_coupling_bwd_pre_kernel<<<R, kRowThreads, 0, stream>>>(D, t->n_live, t->sc, c == 1 ? t->z : nullptr,
                                                                  c == 1 ? nullptr : t->du, c == 1 ? b.invp3 : b.invp1,
                                                                  t->u[c], t->so[c][0], mask, t->dx, t->dso[0],
                                                                  t->dso[1]);
      WVN_CHECK_LAUNCH("flow_coupling_bwd_pre_kernel");
      GemmProblem ps[2];
      for (int k = 0; k < 2; ++k) {   // d2 = (dso W4) * (s2 > 0)
        const NetOffsets o = net_offsets(t->s, c, k);
        ps[k] = gemm_problem(t->dso[k], D, 1, params + o.w4, h, 1, t->d2[k], h, R, h, D, 1);
        ps[k].ref = t->s2[c][k]; ps[k].ld_ref = h;
      }
      WVN_PROPAGATE(launch_gemms(ps, 2, t->n_live, stream));
      for (int k = 0; k < 2; ++k) {   // d1 = (d2 W2) * (s1 > 0)
        const NetOffsets o = net_offsets(t->s, c, k);
        ps[k] = gemm_problem(t->d2[k], h, 1, params + o.w2, h, 1, t->d1[k], h, R, h, h, 1);
        ps[k].ref = t->s1[c][k]; ps[k].ld_ref = h;
      }
      WVN_PROPAGATE(launch_gemms(ps, 2, t->n_live, stream));
      if (c == 1) {
        for (int k = 0; k < 2; ++k) {   // dmu = d1 W0
          const NetOffsets o = net_offsets(t->s, c, k);
          ps[k] = gemm_problem(t->d1[k], h, 1, params + o.w0, D, 1, t->dmu[k], D, R, D, h, 1);
        }
        WVN_PROPAGATE(launch_gemms(ps, 2, t->n_live, stream));
        flow_coupling_bwd_post_kernel<<<R, kRowThreads, 0, stream>>>(D, t->n_live, t->dx, t->so[1][0], mask, t->dmu[0],
                                                                     t->dmu[1], t->du);
        WVN_CHECK_LAUNCH("flow_coupling_bwd_post_kernel");
      }
      // this coupling's weight gradients (the data gradients it read are overwritten by coupling 0's backward)
      GemmProblem wg[6];
      for (int k = 0; k < 2; ++k) {
        const NetOffsets o = net_offsets(t->s, c, k);
        wg[3 * k + 0] = gemm_problem(t->dso[k], 1, D, t->s2[c][k], h, 1, t->grads + o.w4, h, D, h, R, 2);
        wg[3 * k + 0].db = t->grads + o.b4;
        wg[3 * k + 1] = gemm_problem(t->d2[k], 1, h, t->s1[c][k], h, 1, t->grads + o.w2, h, h, h, R, 2);
        wg[3 * k + 1].db = t->grads + o.b2;
        wg[3 * k + 2] = gemm_problem(t->d1[k], 1, h, t->mu[c], D, 1, t->grads + o.w0, D, h, D, R, 2);
        wg[3 * k + 2].db = t->grads + o.b0;
      }
      WVN_PROPAGATE(launch_gemms(wg, 6, t->n_live, stream));
    }
    WVN_PROPAGATE(trainer_comm_sum(&t->comm, t->grads, flow_param_count(t->s), false, stream));
  }
  if (stages & kAdam) {
    WVN_PROPAGATE(mlp_adam_step(params, t->grads, exp_avg, exp_avg_sq, static_cast<long long>(flow_param_count(t->s)),
                                t->adam, step_counter, stream));
  }
  return WVN_OK;
}

}  // namespace

int flow_train_step(Trainer* t, float* params, float* exp_avg, float* exp_avg_sq, long long* step_counter,
                    const FlowBuffers& b, const float* x, int rows, const unsigned char* y_valid, float* cg_mean,
                    float* cg_std, float* conf_out, float* metrics, int phase_mask, cudaStream_t stream) {
  const int stages = ((phase_mask & 1) ? kFwd | kGen : 0) | (phase_mask & (kBwd | kAdam));
  return flow_step(t, params, exp_avg, exp_avg_sq, step_counter, b, x, 1, rows, nullptr, y_valid, cg_mean, cg_std,
                   conf_out, metrics, stages, stream);
}

int flow_train_step_padded(Trainer* t, float* params, float* exp_avg, float* exp_avg_sq, long long* step_counter,
                           const FlowBuffers& b, const float* x, int groups, int rows_per_group, const int* n_rows,
                           const unsigned char* y_valid, float* cg_mean, float* cg_std, float* conf_out, float* metrics,
                           int phase_mask, cudaStream_t stream) {
  const int stages = (phase_mask & 1) | ((phase_mask & 2) ? kGen | kBwd : 0) | (phase_mask & kAdam);
  return flow_step(t, params, exp_avg, exp_avg_sq, step_counter, b, x, groups, rows_per_group, n_rows, y_valid, cg_mean,
                   cg_std, conf_out, metrics, stages, stream);
}

// ================================================================================================ per-pixel inference
// The node's per-pixel anomaly map (wvn_feature_extractor_node.py:332-338): bilinearly upsampled features (align_corners
// = True, dino_interface.py:87-88) -> LinearRnvp -> NLL -> inference_without_update.  Per chunk of pixels (sized so
// the chunk's activations stay near L2): a sampling kernel writes u (fp32) and mu = u * mask (bf16), every net layer is
// one wgmma GEMM with bf16 operands and fp32 accumulation (layer 1 of s and t as one GEMM of 2 h columns, bias + ReLU
// in the epilogue), and a coupling kernel applies tanh / exp / the affine update / log-det / the permutation in fp32,
// and for the last coupling the NLL and its confidence.  Neither the dense (B, D, H, W) map nor a frame of activations
// reaches HBM.
namespace {

__global__ void pack_bf16_kernel(const float* __restrict__ src, int rows, int cols, __nv_bfloat16* __restrict__ dst,
                                 int rows_p, int cols_p) {
  const long long n = static_cast<long long>(rows_p) * cols_p;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / cols_p), c = static_cast<int>(i % cols_p);
    dst[i] = __float2bfloat16_rn((r < rows && c < cols) ? src[static_cast<long long>(r) * cols + c] : 0.f);
  }
}

__global__ void pack_f32_kernel(const float* __restrict__ src, int n, float* __restrict__ dst, int n_p) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_p; i += gridDim.x * blockDim.x) dst[i] = i < n ? src[i] : 0.f;
}

struct PixelGeom {
  int dim, dim_p, gh, gw, H, W;
  float sy, sx;
};

// one block per pixel: u = bilinear(tokens) (fp32), mu = bf16(u * mask), padding columns of mu zeroed
__global__ void __launch_bounds__(kRowThreads)
flow_sample_kernel(const float* __restrict__ tokens, PixelGeom g, long long pix0, const float* __restrict__ mask,
                   float* __restrict__ u, __nv_bfloat16* __restrict__ mu) {
  const long long pix = pix0 + blockIdx.x;
  const long long hw = static_cast<long long>(g.H) * g.W;
  const int b = static_cast<int>(pix / hw);
  const int rem = static_cast<int>(pix - b * hw), y = rem / g.W, x = rem - (rem / g.W) * g.W;
  const float fy = y * g.sy, fx = x * g.sx;
  const int y0 = min(static_cast<int>(floorf(fy)), g.gh - 1), x0 = min(static_cast<int>(floorf(fx)), g.gw - 1);
  const int y1 = min(y0 + 1, g.gh - 1), x1 = min(x0 + 1, g.gw - 1);
  const float wy = fy - y0, wx = fx - x0;
  const float* t = tokens + static_cast<long long>(b) * g.gh * g.gw * g.dim;
  const float* t00 = t + (static_cast<long long>(y0) * g.gw + x0) * g.dim;
  const float* t01 = t + (static_cast<long long>(y0) * g.gw + x1) * g.dim;
  const float* t10 = t + (static_cast<long long>(y1) * g.gw + x0) * g.dim;
  const float* t11 = t + (static_cast<long long>(y1) * g.gw + x1) * g.dim;
  float* ur = u + static_cast<long long>(blockIdx.x) * g.dim;
  __nv_bfloat16* mr = mu + static_cast<long long>(blockIdx.x) * g.dim_p;
  for (int j = threadIdx.x; j < g.dim_p; j += kRowThreads) {
    if (j < g.dim) {
      const float v = (1.f - wy) * ((1.f - wx) * t00[j] + wx * t01[j]) + wy * ((1.f - wx) * t10[j] + wx * t11[j]);
      ur[j] = v;
      mr[j] = __float2bfloat16_rn(v * mask[j]);
    } else {
      mr[j] = __float2bfloat16_rn(0.f);
    }
  }
}

// One block per pixel of the chunk.  so / to: the nets' fp32 outputs (row pitch dim_p).  Not last: u <- x[perm] (in
// place), mu <- bf16(u * next_mask), ld <- log_det so far.  Last: nll / trav of the pixel.
struct PixelCoupling {
  const float* mask; const long long* perm; const float* next_mask; int last;
  const float* so; const float* to; float* u; __nv_bfloat16* mu; float* ld;
  long long pix0; float* nll; float* trav; const float* cg_mean; const float* cg_std; float std_factor;
};

__global__ void __launch_bounds__(kRowThreads)
flow_pixel_coupling_kernel(PixelCoupling c, int dim, int dim_p) {
  extern __shared__ float xs[];
  __shared__ float red[kRowThreads / 32];
  const long long r = blockIdx.x;
  float* ur = c.u + r * dim;
  float ld = 0.f;
  for (int j = threadIdx.x; j < dim; j += kRowThreads) {
    const float m = c.mask[j], om = 1.f - m, uv = ur[j];
    const float s = tanhf(c.so[r * dim_p + j]);
    xs[j] = uv * m + om * (uv * expf(s) + c.to[r * dim_p + j]);
    ld += om * s;
  }
  ld = warp_sum(ld);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ld;
  __syncthreads();
  float ldr = 0.f;
#pragma unroll
  for (int w = 0; w < kRowThreads / 32; ++w) ldr += red[w];
  const float ld_total = c.last ? c.ld[r] + ldr : ldr;
  if (!c.last) {
    for (int j = threadIdx.x; j < dim_p; j += kRowThreads) {
      if (j < dim) {
        const float v = xs[c.perm[j]];
        ur[j] = v;
        c.mu[r * dim_p + j] = __float2bfloat16_rn(v * c.next_mask[j]);
      }
    }
    if (threadIdx.x == 0) c.ld[r] = ld_total;
    return;
  }
  float lps = 0.f;
  for (int j = threadIdx.x; j < dim; j += kRowThreads) {
    const float v = xs[c.perm[j]];
    lps += -(v * v) * 0.5f - kLogSqrt2Pi;
  }
  __syncthreads();
  lps = warp_sum(lps);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = lps;
  __syncthreads();
  if (threadIdx.x == 0) {
    float sum = 0.f;
#pragma unroll
    for (int w = 0; w < kRowThreads / 32; ++w) sum += red[w];
    const float nll = -(sum + ld_total);
    if (c.nll) c.nll[c.pix0 + r] = nll;
    const float m = *c.cg_mean, sd = *c.cg_std, shifted = m + sd * c.std_factor;
    c.trav[c.pix0 + r] = row_confidence(CONF_LATEST, nll, fmaxf(shifted - sd, 0.f), shifted + sd, 0.f, 0.f);
  }
}

inline int rup(int v, int m) { return (v + m - 1) / m * m; }

}  // namespace

// The per-pixel path's bf16 operands and chunk workspaces
struct FlowPixels {
  FlowShape s;
  int dim_p = 0, hid_p = 0, chunk = 0;
  DevBuf arena;
  __nv_bfloat16 *w0[2], *w2[2][2], *w4[2][2];   // [coupling][net]; w0 holds s and t stacked (2 hid_p rows)
  float *b0[2], *b2[2][2], *b4[2][2];
  float *u, *so, *to, *ld;
  __nv_bfloat16 *mu, *h1, *h2;
  bool loaded = false;
};

}  // namespace wvn

// inference only: the fp32 row forward (a forward-only trainer) and the per-pixel wgmma path
struct wvn_flow_infer {
  std::unique_ptr<wvn::Trainer> rows;
  wvn::FlowPixels pix;
};

namespace wvn {

int flow_infer_create(const FlowShape& s, int max_rows, int chunk, wvn_flow_infer** out) {
  std::unique_ptr<wvn_flow_infer> h(new wvn_flow_infer());
  Trainer* rows = nullptr;
  WVN_PROPAGATE(flow_trainer_create(s, max_rows, 0.5f, AdamCfg(), nullptr, true, &rows));
  h->rows.reset(rows);
  FlowPixels* f = &h->pix;
  f->s = s;
  f->dim_p = rup(s.dim, 64);
  f->hid_p = rup(s.hidden, 64);
  f->chunk = chunk > 0 ? rup(chunk, 128) : 8192;
  const size_t Dp = f->dim_p, hp = f->hid_p, C = f->chunk, D = s.dim;
  WVN_PROPAGATE(carve(&f->arena, [&](Carver& a) {
    for (int c = 0; c < 2; ++c) {
      f->w0[c] = a.take<__nv_bfloat16>(2 * hp * Dp);   // s and t stacked: 2 hp rows of Dp
      f->b0[c] = a.take<float>(2 * hp);
      for (int k = 0; k < 2; ++k) {
        f->w2[c][k] = a.take<__nv_bfloat16>(hp * hp);
        f->b2[c][k] = a.take<float>(hp);
        f->w4[c][k] = a.take<__nv_bfloat16>(Dp * hp);
        f->b4[c][k] = a.take<float>(Dp);
      }
    }
    f->u = a.take<float>(C * D);
    f->so = a.take<float>(C * Dp);
    f->to = a.take<float>(C * Dp);
    f->ld = a.take<float>(C);
    f->mu = a.take<__nv_bfloat16>(C * Dp);
    f->h1 = a.take<__nv_bfloat16>(C * 2 * hp);
    f->h2 = a.take<__nv_bfloat16>(C * 2 * hp);
  }, "flow pixels"));
  *out = h.release();
  return WVN_OK;
}

void flow_infer_destroy(wvn_flow_infer* h) { delete h; }

Trainer* flow_infer_trainer(wvn_flow_infer* h) { return h->rows.get(); }

int flow_infer_set_params(wvn_flow_infer* fi, const float* params, cudaStream_t stream) {
  WVN_REQUIRE(params, "flow pixels: null argument");
  FlowPixels* f = &fi->pix;
  const int D = f->s.dim, h = f->s.hidden, Dp = f->dim_p, hp = f->hid_p;
  for (int c = 0; c < 2; ++c) {
    for (int k = 0; k < 2; ++k) {
      const NetOffsets o = net_offsets(f->s, c, k);
      pack_bf16_kernel<<<128, 256, 0, stream>>>(params + o.w0, h, D, f->w0[c] + static_cast<long long>(k) * hp * Dp, hp, Dp);
      WVN_CHECK_LAUNCH("pack_bf16_kernel");
      pack_f32_kernel<<<4, 256, 0, stream>>>(params + o.b0, h, f->b0[c] + k * hp, hp);
      WVN_CHECK_LAUNCH("pack_f32_kernel");
      pack_bf16_kernel<<<128, 256, 0, stream>>>(params + o.w2, h, h, f->w2[c][k], hp, hp);
      WVN_CHECK_LAUNCH("pack_bf16_kernel");
      pack_f32_kernel<<<4, 256, 0, stream>>>(params + o.b2, h, f->b2[c][k], hp);
      WVN_CHECK_LAUNCH("pack_f32_kernel");
      pack_bf16_kernel<<<128, 256, 0, stream>>>(params + o.w4, D, h, f->w4[c][k], Dp, hp);
      WVN_CHECK_LAUNCH("pack_bf16_kernel");
      pack_f32_kernel<<<16, 256, 0, stream>>>(params + o.b4, D, f->b4[c][k], Dp);
      WVN_CHECK_LAUNCH("pack_f32_kernel");
    }
  }
  f->loaded = true;
  return WVN_OK;
}

int flow_infer_pixels(wvn_flow_infer* fi, const FlowBuffers& b, const float* tokens, int batch, int gh, int gw,
                      int out_h, int out_w, const float* cg_mean, const float* cg_std, float std_factor, float* trav,
                      float* nll, cudaStream_t stream) {
  WVN_REQUIRE(tokens && trav && cg_mean && cg_std && b.mask0 && b.mask1 && b.p1 && b.p3, "flow pixels: null argument");
  FlowPixels* f = &fi->pix;
  if (!f->loaded) return set_error(WVN_ERR_STATE, "flow pixels: parameters were never set");
  WVN_REQUIRE(batch > 0 && gh > 0 && gw > 0 && out_h > 1 && out_w > 1, "flow pixels: bad geometry");
  const int D = f->s.dim, Dp = f->dim_p, hp = f->hid_p;
  PixelGeom g;
  g.dim = D; g.dim_p = Dp; g.gh = gh; g.gw = gw; g.H = out_h; g.W = out_w;
  g.sy = static_cast<float>(gh - 1) / static_cast<float>(out_h - 1);   // align_corners=True (dino_interface.py:87-88)
  g.sx = static_cast<float>(gw - 1) / static_cast<float>(out_w - 1);
  const long long total = static_cast<long long>(batch) * out_h * out_w;
  for (long long p0 = 0; p0 < total; p0 += f->chunk) {
    const int n = static_cast<int>(std::min<long long>(f->chunk, total - p0));
    flow_sample_kernel<<<n, kRowThreads, 0, stream>>>(tokens, g, p0, b.mask0, f->u, f->mu);
    WVN_CHECK_LAUNCH("flow_sample_kernel");
    for (int c = 0; c < 2; ++c) {
      GemmArgs g1;
      g1.M = n; g1.N = 2 * hp; g1.K = Dp; g1.epi = EPI_BF16; g1.act = ACT_RELU;
      g1.bias = f->b0[c]; g1.out = f->h1; g1.ldo = 2 * hp;
      WVN_PROPAGATE(gemm_bf16(g1, f->mu, Dp, f->w0[c], 0, stream));
      for (int k = 0; k < 2; ++k) {
        GemmArgs g2;
        g2.M = n; g2.N = hp; g2.K = hp; g2.epi = EPI_BF16; g2.act = ACT_RELU;
        g2.bias = f->b2[c][k]; g2.out = f->h2 + k * hp; g2.ldo = 2 * hp;
        WVN_PROPAGATE(gemm_bf16(g2, f->h1 + k * hp, 2 * hp, f->w2[c][k], 0, stream));
        GemmArgs g3;
        g3.M = n; g3.N = Dp; g3.K = hp; g3.epi = EPI_F32;
        g3.bias = f->b4[c][k]; g3.out = k == 0 ? f->so : f->to; g3.ldo = Dp;
        WVN_PROPAGATE(gemm_bf16(g3, f->h2 + k * hp, 2 * hp, f->w4[c][k], 0, stream));
      }
      PixelCoupling pc;
      memset(&pc, 0, sizeof(pc));
      pc.mask = c == 0 ? b.mask0 : b.mask1; pc.perm = c == 0 ? b.p1 : b.p3; pc.next_mask = b.mask1; pc.last = c;
      pc.so = f->so; pc.to = f->to; pc.u = f->u; pc.mu = f->mu; pc.ld = f->ld;
      pc.pix0 = p0; pc.nll = nll; pc.trav = trav; pc.cg_mean = cg_mean; pc.cg_std = cg_std; pc.std_factor = std_factor;
      flow_pixel_coupling_kernel<<<n, kRowThreads, D * sizeof(float), stream>>>(pc, D, Dp);
      WVN_CHECK_LAUNCH("flow_pixel_coupling_kernel");
    }
  }
  return WVN_OK;
}

}  // namespace wvn
