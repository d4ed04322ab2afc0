// wvn-b200: internal interface of stego_kmeans.cu (per-image k-means of the STEGO code).
#pragma once

#include <cuda_runtime.h>

namespace wvn {

struct KmeansArgs {
  int batch = 0;
  int npad = 0;        // rows per frame of the head-output matrix (row 0 = CLS)
  int patches = 0;     // live patch rows per frame
  long long ld = 0;    // row pitch (floats)
  int code_col = 0, code_dim = 0;   // code columns [code_col, code_col + code_dim)
  int logit_col = 0;   // per-patch nearest-centroid scores are written to [logit_col, logit_col + k)
  int k = 0, iters = 0;
  float* centroids_out = nullptr;   // optional [batch, k, code_dim]
  int n_priv = 0;                   // set by stego_kmeans(): warp-private sum copies per CTA
  int rows_in_smem = 0;             // set by stego_kmeans(): the CTA's code rows are staged in shared memory
  unsigned int* frame_bar = nullptr;  // set by stego_kmeans(): [batch] arrival counters of the per-frame barrier
  int team = 0;                       // set by stego_kmeans(): CTAs per frame
};

// workspace: stego_kmeans_workspace_bytes(batch, k, code_dim) bytes of device memory (per-CTA partial sums).
size_t stego_kmeans_workspace_bytes(int batch, int k, int code_dim);
int stego_kmeans(float* rows, const KmeansArgs& a, float* workspace, cudaStream_t stream);

}  // namespace wvn
