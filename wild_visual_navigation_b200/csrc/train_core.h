// wvn-b200: the fp32 training core shared by the learners (mlp_train.cu, mlp_train_fused.cu, double_mlp_train.cu,
// gcn_train.cu, flow_train.cu): the ConfidenceGenerator state a trainer keeps, Adam, the batched fp32 tile GEMM, the
// compaction of padded rows, the data-parallel exchange and the trainer base every learner derives from.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>

#include "host_common.h"
#include "mlp_train.h"

namespace wvn {

struct AdamCfg {
  float lr = 1e-3f, beta1 = 0.9f, beta2 = 0.999f, eps = 1e-8f;
};

// torch.optim.Adam's update (no amsgrad, no weight decay): bumps *step_counter, then one update of n parameters.
int mlp_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n,
                  const AdamCfg& cfg, long long* step_counter, cudaStream_t stream);

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

// A trainer's generator: where its state lives (cs, passed to the kernels) and the device block holding what no caller
// buffer holds: moving_average's window, and var / the running sums when the caller binds none (var starts at 1, the
// reference's initial value).  The block is the first piece of the trainer's arena (trainer_alloc).
struct TrainerConf {
  ConfState cs;
  double* priv = nullptr;
};
// method: ConfMethod; pointers may be null for methods that do not use them (the private block then holds that state).
int trainer_conf_bind(TrainerConf* c, int method, float* var, double* running_n, double* running_sum,
                      double* running_sumsq, float kf_proc_cov, float kf_meas_cov);
// Copies src's private block into dst's, on `stream`: a caller that replaces a trainer by a larger one keeps the
// generator where it was.  Ordered after src's last step; destroying src afterwards frees its arena, which waits for
// the copy.
int trainer_conf_copy(TrainerConf* dst, const TrainerConf* src, cudaStream_t stream);

// ---- batched fp32 GEMM: 64 x 64 tiles, K step 16, 4 x 4 outputs per thread, CUDA cores
// C(m, n) = epilogue(sum_k A(m, k) B(k, n)) with A(m, k) = a[m a_rs + k a_cs], B(k, n) = b[k b_rs + n b_cs]: the same
// kernel does X W^T (forward), dY W (data gradients) and dY^T X (weight gradients).  live = 1: M is capped by *n_live,
// live = 2: K is.  Epilogue: + bias[n], then act, then * (ref(m, n) > 0) (ReLU's backward).  db (weight-gradient
// problems): db[m] = sum_k A(m, k), the bias gradient.
enum GemmF32Act : int {
  F32_LINEAR = 0,
  F32_RELU = 1,          // v < 0 ? 0 : v: NaN passes, like torch.relu
  F32_RELU_FMAX = 2,     // fmaxf(v, 0): NaN becomes 0
  F32_SIGMOID_COL0 = 3,  // column 0 through the sigmoid (SimpleMLP's traversability output)
};
struct GemmProblem {
  const float* a; long long a_rs, a_cs;
  const float* b; long long b_rs, b_cs;
  float* c; long long ldc;
  const float* bias;
  const float* ref; long long ld_ref;
  float* db;
  int M, N, K, act, live;
};
constexpr int kMaxGemmProblems = 12;

GemmProblem gemm_problem(const float* a, long long a_rs, long long a_cs, const float* b, long long b_rs, long long b_cs,
                         float* c, long long ldc, int M, int N, int K, int live = 0);
// One launch for `count` problems.  splits > 1 (one problem, no live bound, no epilogue, no db): K is cut into up to
// `splits` ranges of a multiple of 16 whose partial products are added into C with fp32 atomics (C zeroed by the caller).
int launch_gemms(const GemmProblem* ps, int count, const int* n_live, cudaStream_t stream, int splits = 1);

// ---- padded rows
// Rows arrive padded per group, as the segment pooling leaves them: padded row r = g * rows_per_group + s is live when
// s < n_rows[g] (n_rows NULL: every row).  Live rows are numbered group by group (the compacted numbering of
// `feat[mask]`); y_valid (NULL: keep every live row) is indexed by that number and drops the rows it does not set.
// comp[i] = padded index of the i-th kept row, *n_live = their number.  One launch; padding rows are never read.
int compact_rows(int groups, int rows_per_group, const int* n_rows, const unsigned char* y_valid, int* comp, int* n_live,
                 cudaStream_t stream);

// ---- data-parallel exchange
// Every trainer's statistics block begins with the same 8 doubles: six plain sums (all-reduced with SUM, one of them a
// row count), then the extrema of the confidence input (MIN / MAX; moving_average's min-max normalisation).
constexpr int kStatSums = 6;
constexpr int kStatDoubles = 8;
// The library's own NCCL communicator (libnccl.so.2 resolved from the running process): when a trainer has one, its step
// issues the collectives itself, between its kernels on the caller's stream.  Without one, every exchange is a no-op and
// a caller with another transport all-reduces the same buffers between the step's phases.
struct TrainerComm {
  void* comm = nullptr;
  int world = 1;
};
int comm_unique_id(void* id128);
int trainer_comm_init(TrainerComm* c, const void* id128, int rank, int world);
void trainer_comm_destroy(TrainerComm* c);
// stats[0, kStatSums) SUM; with `extrema` also stats[6] MIN and stats[7] MAX.
int trainer_comm_stats(TrainerComm* c, double* stats, bool extrema, cudaStream_t stream);
// SUM of n fp32 (f64 = false) or fp64 values in place.
int trainer_comm_sum(TrainerComm* c, void* buf, size_t n, bool f64, cudaStream_t stream);

// ---- the trainer every learner derives from
enum TrainerKind : int { TRAINER_MLP = 0, TRAINER_DOUBLE_MLP = 1, TRAINER_GCN = 2, TRAINER_FLOW = 3 };

// The state every learner's trainer (FusedTrainer, DoubleTrainer, GcnTrainer, FlowTrainer) keeps; the C ABI's
// wvn_trainer_t is a pointer to it.  Deleting a trainer destroys its communicator and frees its arena.
struct Trainer {
  explicit Trainer(TrainerKind k) : kind(k) {}
  virtual ~Trainer();
  const TrainerKind kind;
  LossCfg loss;
  AdamCfg adam;
  int max_rows = 0;
  DevBuf arena;            // the generator block and every device workspace of the learner, one allocation
  TrainerConf conf;        // ConfidenceGenerator method + where its state lives
  TrainerComm comm;        // the library's communicator of a data-parallel step
  double* stats = nullptr; // the statistics block: kStatDoubles, then the learner's own exchanged doubles
  int n_stats = kStatDoubles;
  float* grads = nullptr;
};
// Allocates t's arena, zeroed: the generator block (bound to latest_measurement, var = 1), then the pieces `layout`
// takes.  Each piece starts on a 256-byte boundary, so consecutive pieces need not be adjacent: no kernel, memset or
// copy may span two of them.  On failure the caller deletes t.
int trainer_alloc(Trainer* t, const std::function<void(Carver&)>& layout, const char* who);
// WVN_ERR_INVALID unless t is a trainer of `kind`: every entry point of a learner checks its handle on the host,
// before it enqueues anything.
int trainer_check(const Trainer* t, TrainerKind kind, const char* who);

}  // namespace wvn
