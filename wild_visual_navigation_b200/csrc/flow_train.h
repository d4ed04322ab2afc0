// wvn-b200: internal interface of the LinearRnvp flow kernels (flow_train.cu): the fp32 row forward and the fp32
// online train step of the anomaly-detection learner, and its inference handle.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>

#include "../../include/wvn_b200.h"
#include "train_core.h"

namespace wvn {

// LinearRnvp(input_size = dim, coupling_topology = [hidden]) with flow_n = 2 and use_permutation = True:
// flows = [coupling 0, permutation 1, coupling 2, permutation 3]; every coupling has two nets s and t, each
// Linear(dim, hidden) ReLU Linear(hidden, hidden) ReLU Linear(hidden, dim).
struct FlowShape {
  int dim = 384;
  int hidden = 200;
};

// The flat fp32 parameter buffer is in parameters() order: flows.0.s, flows.0.t, flows.2.s, flows.2.t, each net as
// 0.weight [hidden, dim], 0.bias, 2.weight [hidden, hidden], 2.bias, 4.weight [dim, hidden], 4.bias.
size_t flow_net_params(const FlowShape& s);
size_t flow_param_count(const FlowShape& s);

// The model's buffers, read by the kernels on every call (so a loaded mask or permutation takes effect at once):
// the two coupling masks [dim] fp32 and the two permutations p / invp [dim] int64.
struct FlowBuffers {
  const float* mask0 = nullptr;
  const float* mask1 = nullptr;
  const long long* p1 = nullptr;
  const long long* invp1 = nullptr;
  const long long* p3 = nullptr;
  const long long* invp3 = nullptr;
};

// grads_ext: caller-owned device buffer of flow_param_count floats, or NULL (the trainer allocates it).
// forward_only: allocate only what flow_forward_rows needs (no backward workspaces, no gradient buffer).
// The statistics block is the kStatDoubles of train_core.h: sum and sum of squares of the NLL over the labelled rows,
// their number, 0, 0, 0, the NLL's min and max.
int flow_trainer_create(const FlowShape& s, int max_rows, float std_factor, const AdamCfg& adam, float* grads_ext,
                        bool forward_only, Trainer** out);

// LinearRnvp.forward on rows x [rows, dim]: z / logprob [rows, dim], log_det [rows] (each may be NULL); with trav
// non-NULL also ConfidenceGenerator.inference_without_update of the per-row NLL -(sum(logprob) + log_det) from the
// generator state at cg_mean / cg_std.
int flow_forward_rows(Trainer* t, const float* params, const FlowBuffers& b, const float* x, int rows, float* z,
                      float* log_det, float* logprob, const float* cg_mean, const float* cg_std, float std_factor,
                      float* trav, cudaStream_t stream);
// trav of rows padded per group, x [groups, rows_per_group, dim] with n_rows[g] (device int32) live rows in group g:
// the live rows are compacted and run as above; trav [groups, rows_per_group] is NaN on padding rows, which are
// neither read nor computed.
int flow_forward_rows_padded(Trainer* t, const float* params, const FlowBuffers& b, const float* x, int groups,
                             int rows_per_group, const int* n_rows, const float* cg_mean, const float* cg_std,
                             float std_factor, float* trav, cudaStream_t stream);

// One step of TraversabilityEstimator.train in anomaly-detection mode on the rows of x [rows, dim] whose y_valid is set
// (y_valid NULL: every row).  phase_mask: 1 = forward, NLL statistics, confidence update; 2 = backward (the flat
// gradient); 4 = Adam (bumps step_counter); 7 = the whole step.  conf_out [rows] is in compacted order (the labelled
// rows in their order); metrics [6]: loss_total, loss_trav (0), loss_reco (0), number of rows, cg_mean, cg_std.
int flow_train_step(Trainer* t, float* params, float* exp_avg, float* exp_avg_sq, long long* step_counter,
                    const FlowBuffers& b, const float* x, int rows, const unsigned char* y_valid, float* cg_mean,
                    float* cg_std, float* conf_out, float* metrics, int phase_mask, cudaStream_t stream);
// The same step on rows padded per group, x [groups, rows_per_group, dim] with n_rows[g] (device int32; NULL: all) live
// rows in group g, of which those whose y_valid (compacted numbering; NULL: all) is set are trained on.  Padding rows
// are never read.  phase_mask splits the step around the data-parallel exchanges: 1 = forward + this rank's NLL sums
// (+ their all-reduce); 2 = generator update from the global sums, metrics, per-row confidence, backward scaled by the
// global labelled count (+ the gradient all-reduce); 4 = Adam; 7 = the whole step.
int flow_train_step_padded(Trainer* t, float* params, float* exp_avg, float* exp_avg_sq, long long* step_counter,
                           const FlowBuffers& b, const float* x, int groups, int rows_per_group, const int* n_rows,
                           const unsigned char* y_valid, float* cg_mean, float* cg_std, float* conf_out, float* metrics,
                           int phase_mask, cudaStream_t stream);

// The inference handle (wvn_flow_infer_*): a forward-only trainer of max_rows rows for the two row forwards above, and
// the per-pixel anomaly map on wgmma in chunks of chunk_pixels (0: 8192).
int flow_infer_create(const FlowShape& s, int max_rows, int chunk_pixels, wvn_flow_infer** out);
void flow_infer_destroy(wvn_flow_infer* h);
Trainer* flow_infer_trainer(wvn_flow_infer* h);
// Per-pixel anomaly map: bf16 operands packed by set_params (re-pack after the parameters change), fp32 accumulation;
// the masks and permutations are read from b on every call.  tokens: [batch, gh * gw, dim] fp32; trav
// [batch, out_h, out_w] = inference_without_update(NLL); nll (may be NULL): the per-pixel NLL.
int flow_infer_set_params(wvn_flow_infer* h, const float* params, cudaStream_t stream);
int flow_infer_pixels(wvn_flow_infer* h, const FlowBuffers& b, const float* tokens, int batch, int gh, int gw,
                      int out_h, int out_w, const float* cg_mean, const float* cg_std, float std_factor, float* trav,
                      float* nll, cudaStream_t stream);

}  // namespace wvn
