// wvn-b200: the fp32 training core shared by the MLP and LinearRnvp trainers (train_core.h): the private
// ConfidenceGenerator block, Adam, and the batched fp32 CUDA-core GEMM.
#include <string.h>

#include <algorithm>

#include "common.cuh"
#include "host_common.h"
#include "train_core.cuh"

namespace wvn {

// ------------------------------------------------------------------------------------------------ confidence state
// Private block (doubles): running_n, running_sum, running_sumsq | var as a float | ring [kConfWindow][3] + count.
constexpr int kConfBlockDoubles = 32;

int trainer_conf_create(TrainerConf* c) {
  if (cudaMalloc(&c->priv, sizeof(double) * kConfBlockDoubles) != cudaSuccess) {
    c->priv = nullptr;
    return set_error(WVN_ERR_CUDA, "trainer: cudaMalloc of the confidence state failed");
  }
  cudaMemset(c->priv, 0, sizeof(double) * kConfBlockDoubles);
  const float one = 1.f;   // private var = 1 (the reference's initial value) unless the caller binds its own
  cudaMemcpy(reinterpret_cast<float*>(c->priv + 3), &one, sizeof(float), cudaMemcpyHostToDevice);
  return trainer_conf_bind(c, CONF_LATEST, nullptr, nullptr, nullptr, nullptr, 0.2f, 1.0f);
}

void trainer_conf_destroy(TrainerConf* c) {
  if (c->priv) cudaFree(c->priv);
  c->priv = nullptr;
}

int trainer_conf_bind(TrainerConf* c, int method, float* var, double* running_n, double* running_sum,
                      double* running_sumsq, float kf_proc_cov, float kf_meas_cov) {
  WVN_REQUIRE(method >= CONF_LATEST && method <= CONF_MOVING_AVERAGE, "trainer: confidence method %d (0 "
              "latest_measurement, 1 running_mean, 2 kalman_filter, 3 moving_average)", method);
  ConfState& s = c->cs;
  s.method = method;
  s.running_n = running_n ? running_n : c->priv;
  s.running_sum = running_sum ? running_sum : c->priv + 1;
  s.running_sumsq = running_sumsq ? running_sumsq : c->priv + 2;
  s.var = var ? var : reinterpret_cast<float*>(c->priv + 3);
  s.kf_proc_cov = kf_proc_cov;
  s.kf_meas_cov = kf_meas_cov;
  s.ring = c->priv + 4;
  return WVN_OK;
}

int trainer_conf_copy(TrainerConf* dst, const TrainerConf* src, cudaStream_t stream) {
  WVN_CHECK_CUDA(cudaMemcpyAsync(dst->priv, src->priv, sizeof(double) * kConfBlockDoubles, cudaMemcpyDeviceToDevice,
                                 stream));
  return WVN_OK;
}

// ------------------------------------------------------------------------------------------------ Adam
namespace {

__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
            long long n, AdamCfg cfg, const long long* __restrict__ step_ptr) {
  adam_update(p, g, m, v, n, cfg, step_ptr);
}

__global__ void bump_step_kernel(long long* step) { *step += 1; }

}  // namespace

int mlp_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n,
                  const AdamCfg& cfg, long long* step_counter, cudaStream_t stream) {
  bump_step_kernel<<<1, 1, 0, stream>>>(step_counter);
  WVN_CHECK_LAUNCH("bump_step_kernel");
  int blocks = static_cast<int>((n + 255) / 256);
  if (blocks > sm_count() * 4) blocks = sm_count() * 4;
  adam_kernel<<<blocks, 256, 0, stream>>>(params, grads, exp_avg, exp_avg_sq, n, cfg, step_counter);
  WVN_CHECK_LAUNCH("adam_kernel");
  return WVN_OK;
}

// ------------------------------------------------------------------------------------------------ batched fp32 GEMM
namespace {

constexpr int GT = 64, GK = 16;

struct GemmBatch {
  GemmProblem p[kMaxGemmProblems];
  const int* n_live;
  int splits, k_per_split;   // blockIdx.z = problem * splits + split
};

// kBiasGrad: some problem of the launch has db; without it the column sums are compiled out of the inner loop.
// kSingle: one problem without a live bound (the MLP forward, the three-phase backward), read at a constant index.
// Four CTAs per SM cap the kernel at 64 registers, which it fits without spilling (a problem read by a dynamic index
// would otherwise keep its fields in registers, at 100+ and two CTAs per SM).
template <bool kBiasGrad, bool kSingle>
__global__ void __launch_bounds__(256, 4)
gemm_f32_kernel(GemmBatch g) {
  const int pi = kSingle ? 0 : blockIdx.z / g.splits, split = blockIdx.z - pi * g.splits;
  const GemmProblem& p = g.p[pi];
  int M = p.M, K = p.K;
  if (!kSingle && p.live == 1) M = min(M, *g.n_live);
  if (!kSingle && p.live == 2) K = min(K, *g.n_live);
  const int m0 = blockIdx.y * GT, n0 = blockIdx.x * GT;
  if (m0 >= M || n0 >= p.N) return;
  const bool atomic = g.splits > 1;
  const int kbeg = split * g.k_per_split, kend = atomic ? min(K, kbeg + g.k_per_split) : K;
  __shared__ float As[GK][GT + 1];
  __shared__ float Bs[GK][GT + 1];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const bool a_kfast = p.a_cs == 1, b_nfast = p.b_cs == 1;
  float acc[4][4], bsum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = kbeg; k0 < kend; k0 += GK) {
#pragma unroll
    for (int rr = 0; rr < 4; ++rr) {
      const int idx = tid + 256 * rr;
      int mm, kk;
      if (a_kfast) { mm = idx >> 4; kk = idx & 15; } else { kk = idx >> 6; mm = idx & 63; }
      const int gm = m0 + mm, gk = k0 + kk;
      As[kk][mm] = (gm < M && gk < kend) ? p.a[gm * p.a_rs + gk * p.a_cs] : 0.f;
      int nn;
      if (b_nfast) { kk = idx >> 6; nn = idx & 63; } else { nn = idx >> 4; kk = idx & 15; }
      const int gn = n0 + nn, gk2 = k0 + kk;
      Bs[kk][nn] = (gn < p.N && gk2 < kend) ? p.b[gk2 * p.b_rs + gn * p.b_cs] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < GK; ++k) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) av[i] = As[k][ty + 16 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) bv[j] = Bs[k][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (kBiasGrad) bsum[i] += av[i];
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gm = m0 + ty + 16 * i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx + 16 * j;
      if (gn >= p.N) continue;
      float v = acc[i][j];
      if (atomic) {
        atomicAdd(&p.c[gm * p.ldc + gn], v);
        continue;
      }
      if (p.bias) v += p.bias[gn];
      if (p.act == F32_RELU) v = v < 0.f ? 0.f : v;
      if (p.act == F32_RELU_FMAX) v = fmaxf(v, 0.f);
      if (p.act == F32_SIGMOID_COL0 && gn == 0) v = 1.f / (1.f + expf(-v));
      if (p.ref) v = p.ref[gm * p.ld_ref + gn] > 0.f ? v : 0.f;
      p.c[gm * p.ldc + gn] = v;
    }
    if (kBiasGrad && p.db && blockIdx.x == 0 && tx == 0) p.db[gm] = bsum[i];
  }
}

}  // namespace

GemmProblem gemm_problem(const float* a, long long a_rs, long long a_cs, const float* b, long long b_rs, long long b_cs,
                         float* c, long long ldc, int M, int N, int K, int live) {
  GemmProblem p;
  memset(&p, 0, sizeof(p));
  p.a = a; p.a_rs = a_rs; p.a_cs = a_cs;
  p.b = b; p.b_rs = b_rs; p.b_cs = b_cs;
  p.c = c; p.ldc = ldc;
  p.M = M; p.N = N; p.K = K; p.live = live;
  return p;
}

int launch_gemms(const GemmProblem* ps, int count, const int* n_live, cudaStream_t stream, int splits) {
  WVN_REQUIRE(count >= 1 && count <= kMaxGemmProblems, "gemm: %d problems in one launch", count);
  GemmBatch g;
  memset(&g, 0, sizeof(g));
  int gx = 1, gy = 1, kmax = 0;
  bool db = false;
  for (int i = 0; i < count; ++i) {
    // split-K adds raw partial sums with atomics: an epilogue would be dropped and a db column sum overwritten
    WVN_REQUIRE(splits <= 1 || (!ps[i].bias && ps[i].act == F32_LINEAR && !ps[i].ref && !ps[i].db),
                "gemm: split-K (%d splits) with a bias, activation, ReLU mask or bias gradient (problem %d)", splits, i);
    g.p[i] = ps[i];
    gx = std::max(gx, (ps[i].N + GT - 1) / GT);
    gy = std::max(gy, (ps[i].M + GT - 1) / GT);
    kmax = std::max(kmax, ps[i].K);
    db = db || ps[i].db;
  }
  g.n_live = n_live;
  g.splits = 1;
  if (splits > 1 && kmax > 0) {   // K ranges of a multiple of GK; fewer than `splits` when K is short
    const int kps = ((kmax + splits - 1) / splits + GK - 1) / GK * GK;
    const int z = (kmax + kps - 1) / kps;
    if (z > 1) { g.splits = z; g.k_per_split = kps; }
  }
  const dim3 grid(gx, gy, count * g.splits);
  if (db) gemm_f32_kernel<true, false><<<grid, 256, 0, stream>>>(g);
  else if (count == 1 && ps[0].live == 0) gemm_f32_kernel<false, true><<<grid, 256, 0, stream>>>(g);
  else gemm_f32_kernel<false, false><<<grid, 256, 0, stream>>>(g);
  WVN_CHECK_LAUNCH("gemm_f32_kernel");
  return WVN_OK;
}

}  // namespace wvn
