// wvn-b200: internal interface of the SimpleGCN learner's fp32 kernels (gcn_train.cu): the graph build over padded
// per-frame segment adjacency, the forward on rows, and the online train step.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>

#include "mlp_train.h"
#include "train_core.h"

namespace wvn {

// SimpleGCN(input_size = dim, reconstruction = True, hidden_sizes = [h1, h2, 1]): three graph convolutions
//   GCNConv(dim, h1) ReLU GCNConv(h1, h2) ReLU GCNConv(h2, 1 + dim), sigmoid on column 0,
// each  Z = D^-1/2 (A + I) D^-1/2 X W^T + b  with A[i, j] = the number of edges j -> i (self-loops of the input dropped)
// and D = 1 + the in-degree.  The output has SimpleMLP's (rows, 1 + dim) layout.  The flat fp32 parameter buffer is in
// parameters() order: layers.{0,1,2}.bias, then that layer's lin.weight [out, in].
struct GcnOffsets {
  size_t b[3], w[3], total;
};
GcnOffsets gcn_offsets(const MlpShape& s);
size_t gcn_param_count(const MlpShape& s);
// The shapes the kernels take: 1 <= dim <= 1024, 1 <= h1, h2 <= 512 (WVN_ERR_INVALID else).
int gcn_check_shape(const MlpShape& s, const char* who);

// Workspaces for max_rows padded rows and max_edges padded edges (groups * edges_per_group).  grads_ext: caller-owned
// device buffer of gcn_param_count floats, or NULL (the trainer allocates it).  The statistics block has 9 doubles,
// laid out as the DoubleMLP trainer's (double_mlp_train.h).
int gcn_trainer_create(const MlpShape& s, int max_rows, int max_edges, const LossCfg& loss, const AdamCfg& adam,
                       float* grads_ext, Trainer** out);

// One TraversabilityEstimator.train() body on a batch of frames: x [groups, rows_per_group, dim] with n_rows[g] (device
// int32; NULL: all) live rows in frame g; edges [groups, edges_per_group, 2] int64 (source, target) local row ids of
// which the first n_edges[g] (device int32) are read.  Edges with an endpoint outside the frame's live rows are dropped;
// a negative n_edges[g] (the segment reducer's overflow flag) reads no edge of that frame and sets metrics[6] to 1 (the
// flag rides in the statistics block's sixth sum, so under a data-parallel exchange every rank sees any rank's).
// y / y_valid (uint8) / conf_out are indexed by the compacted row number.  phase_mask: 1 = graph build, forward, per-row
// losses, the statistic sums (+ their all-reduce); 2 = generator update, dLoss/dOut, backward, gradients (+ the gradient
// all-reduce); 4 = loss metrics + Adam; 7 = the whole step.  metrics [7] (may be NULL): loss_total, loss_trav,
// loss_reco, loss_trav_conf, cg_mean, cg_std, the overflow flag.
int gcn_train_step_padded(Trainer* t, float* params, float* exp_avg, float* exp_avg_sq, long long* step_counter,
                          const float* x, int groups, int rows_per_group, const int* n_rows, const long long* edges,
                          int edges_per_group, const int* n_edges, const float* y, const unsigned char* y_valid,
                          float* cg_mean, float* cg_std, float* conf_out, float* metrics, int phase_mask,
                          cudaStream_t stream);

// SimpleGCN.forward on the same padded input (negative n_edges: no edges of that frame), then per live row
// traversability = out[:, 0] and the confidence of loss_reco under the generator (inference_without_update).
// out (may be NULL): [groups * rows_per_group, 1 + dim], the first live-count rows in compacted order.  trav / conf
// (may be NULL): [groups * rows_per_group] in PADDED order; padding rows are not written.
int gcn_infer_rows(Trainer* t, const float* params, const float* x, int groups, int rows_per_group,
                   const int* n_rows, const long long* edges, int edges_per_group, const int* n_edges,
                   const float* cg_mean, const float* cg_std, float std_factor, float* out, float* trav, float* conf,
                   cudaStream_t stream);

}  // namespace wvn
