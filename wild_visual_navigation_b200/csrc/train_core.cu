// wvn-b200: the fp32 training core shared by the learners' trainers (train_core.h): the private ConfidenceGenerator
// block, Adam, the batched fp32 CUDA-core GEMM, the compaction of padded rows, the NCCL communicator of data-parallel
// steps and the trainer base's arena.
#include <dlfcn.h>
#include <string.h>

#include <algorithm>

#include "common.cuh"
#include "host_common.h"
#include "train_core.cuh"

namespace wvn {

// ------------------------------------------------------------------------------------------------ confidence state
// Private block (doubles): running_n, running_sum, running_sumsq | var as a float | ring [kConfWindow][3] + count.
constexpr int kConfBlockDoubles = 32;

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

// ------------------------------------------------------------------------------------------------ padded rows
namespace {

// Exclusive prefix sum of v over the block of 1024 threads; *total = the sum over the block.
__device__ __forceinline__ int block_exclusive_scan(int v, int* wsum, int* total) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  __syncthreads();   // wsum is free (a previous scan has been read)
  if (lane == 31) wsum[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    int w = wsum[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += u;
    }
    wsum[lane] = w;
  }
  __syncthreads();
  *total = wsum[31];
  return inc - v + (warp > 0 ? wsum[warp - 1] : 0);
}

// One block of 1024: every thread walks a contiguous range of padded rows three times (live count, kept count, write).
__global__ void __launch_bounds__(1024)
compact_rows_kernel(int groups, int rpg, const int* __restrict__ n_rows, const unsigned char* __restrict__ y_valid,
                    int* __restrict__ comp, int* __restrict__ n_live) {
  __shared__ int wsum[32];
  const long long rows = static_cast<long long>(groups) * rpg;
  const long long per = (rows + 1023) / 1024, b = threadIdx.x * per, e = min(rows, b + per);
  auto live = [&](long long r) {
    if (n_rows == nullptr) return true;
    const long long g = r / rpg;
    return r - g * rpg < n_rows[g];
  };
  int c = 0;
  for (long long r = b; r < e; ++r) c += live(r) ? 1 : 0;
  int total;
  const int ci0 = block_exclusive_scan(c, wsum, &total);   // compacted number of this range's first live row
  int k = 0, ci = ci0;
  for (long long r = b; r < e; ++r)
    if (live(r)) k += (y_valid == nullptr || y_valid[ci++] != 0) ? 1 : 0;
  int pos = block_exclusive_scan(k, wsum, &total);
  ci = ci0;
  for (long long r = b; r < e; ++r)
    if (live(r) && (y_valid == nullptr || y_valid[ci++] != 0)) comp[pos++] = static_cast<int>(r);
  if (threadIdx.x == 0) *n_live = total;
}

}  // namespace

int compact_rows(int groups, int rows_per_group, const int* n_rows, const unsigned char* y_valid, int* comp, int* n_live,
                 cudaStream_t stream) {
  WVN_REQUIRE(groups >= 0 && rows_per_group >= 0 && comp && n_live, "compact rows: bad arguments");
  compact_rows_kernel<<<1, 1024, 0, stream>>>(groups, rows_per_group, n_rows, y_valid, comp, n_live);
  WVN_CHECK_LAUNCH("compact_rows_kernel");
  return WVN_OK;
}

// ------------------------------------------------------------------------------------------------ NCCL (dlopen)
namespace {

typedef struct { char internal[128]; } NcclUniqueId;
typedef void* NcclComm;
struct NcclApi {
  int (*GetUniqueId)(NcclUniqueId*) = nullptr;
  int (*CommInitRank)(NcclComm*, int, NcclUniqueId, int) = nullptr;
  int (*CommDestroy)(NcclComm) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, NcclComm, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  bool ok = false;
};
constexpr int kNcclFloat32 = 7, kNcclFloat64 = 8, kNcclSum = 0, kNcclMax = 2, kNcclMin = 3;  // ncclDataType_t / ncclRedOp_t values (nccl.h)

NcclApi& nccl() {
  static NcclApi api;
  static bool tried = false;
  if (tried) return api;
  tried = true;
  // the process (torch.distributed) has normally loaded libnccl.so.2 already; RTLD_NOLOAD-first keeps a single copy
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) return api;
  api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(dlsym(h, "ncclGetUniqueId"));
  api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(dlsym(h, "ncclCommInitRank"));
  api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(dlsym(h, "ncclCommDestroy"));
  api.AllReduce = reinterpret_cast<decltype(api.AllReduce)>(dlsym(h, "ncclAllReduce"));
  api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(dlsym(h, "ncclGetErrorString"));
  api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllReduce && api.GetErrorString;
  return api;
}

int all_reduce(TrainerComm* c, void* buf, size_t n, int type, int op, const char* what, cudaStream_t stream) {
  NcclApi& api = nccl();
  const int rc = api.AllReduce(buf, buf, n, type, op, static_cast<NcclComm>(c->comm), stream);
  if (rc != 0) return set_error(WVN_ERR_CUDA, "ncclAllReduce(%s): %s", what, api.GetErrorString(rc));
  return WVN_OK;
}

}  // namespace

int comm_unique_id(void* id128) {
  WVN_REQUIRE(id128, "comm: null id buffer");
  NcclApi& api = nccl();
  if (!api.ok) return set_error(WVN_ERR_STATE, "comm: libnccl.so.2 is not loadable in this process");
  NcclUniqueId id;
  const int rc = api.GetUniqueId(&id);
  if (rc != 0) return set_error(WVN_ERR_CUDA, "ncclGetUniqueId: %s", api.GetErrorString(rc));
  memcpy(id128, &id, sizeof(id));
  return WVN_OK;
}

int trainer_comm_init(TrainerComm* c, const void* id128, int rank, int world) {
  WVN_REQUIRE(c && id128 && world >= 1 && rank >= 0 && rank < world, "comm: bad arguments");
  NcclApi& api = nccl();
  if (!api.ok) return set_error(WVN_ERR_STATE, "comm: libnccl.so.2 is not loadable in this process");
  NcclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  NcclComm comm = nullptr;
  const int rc = api.CommInitRank(&comm, world, id, rank);
  if (rc != 0) return set_error(WVN_ERR_CUDA, "ncclCommInitRank: %s", api.GetErrorString(rc));
  trainer_comm_destroy(c);
  c->comm = comm;
  c->world = world;
  return WVN_OK;
}

void trainer_comm_destroy(TrainerComm* c) {
  if (c->comm && nccl().ok) nccl().CommDestroy(static_cast<NcclComm>(c->comm));
  c->comm = nullptr;
  c->world = 1;
}

int trainer_comm_stats(TrainerComm* c, double* stats, bool extrema, cudaStream_t stream) {
  if (!c->comm) return WVN_OK;
  WVN_PROPAGATE(all_reduce(c, stats, kStatSums, kNcclFloat64, kNcclSum, "stats", stream));
  if (!extrema) return WVN_OK;
  WVN_PROPAGATE(all_reduce(c, stats + kStatSums, 1, kNcclFloat64, kNcclMin, "extrema", stream));
  return all_reduce(c, stats + kStatSums + 1, 1, kNcclFloat64, kNcclMax, "extrema", stream);
}

int trainer_comm_sum(TrainerComm* c, void* buf, size_t n, bool f64, cudaStream_t stream) {
  if (!c->comm) return WVN_OK;
  return all_reduce(c, buf, n, f64 ? kNcclFloat64 : kNcclFloat32, kNcclSum, "grads", stream);
}

// ------------------------------------------------------------------------------------------------ trainer
Trainer::~Trainer() { trainer_comm_destroy(&comm); }

int trainer_alloc(Trainer* t, const std::function<void(Carver&)>& layout, const char* who) {
  WVN_PROPAGATE(carve(&t->arena, [&](Carver& c) {
    t->conf.priv = c.take<double>(kConfBlockDoubles);
    layout(c);
  }, who));
  const float one = 1.f;   // private var = 1 (the reference's initial value) unless the caller binds its own
  WVN_CHECK_CUDA(cudaMemcpy(reinterpret_cast<float*>(t->conf.priv + 3), &one, sizeof(float), cudaMemcpyHostToDevice));
  return trainer_conf_bind(&t->conf, CONF_LATEST, nullptr, nullptr, nullptr, nullptr, 0.2f, 1.0f);
}

int trainer_check(const Trainer* t, TrainerKind kind, const char* who) {
  static const char* const names[] = {"SimpleMLP", "DoubleMLP", "SimpleGCN", "LinearRnvp"};
  WVN_REQUIRE(t, "%s: null trainer", who);
  WVN_REQUIRE(t->kind == kind, "%s: expected a %s trainer, got a %s trainer's handle", who, names[kind],
              names[t->kind]);
  return WVN_OK;
}

}  // namespace wvn
