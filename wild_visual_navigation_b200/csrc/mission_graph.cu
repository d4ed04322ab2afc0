// wvn-b200: label propagation of one supervision event into the mission graph's in-range nodes
// (TraversabilityEstimator.add_supervision_node, traversability_estimator.py:257-289, and
// MissionNode.update_supervision_signal, nodes.py:400-440).
//
// The reference renders the footprint into every in-range node's camera, takes fmin into the node's (3, H, W) mask and
// then re-pools each mask per segment through an (H, W, S) one-hot.  Composed from this library's kernels that is
// footprint_render (fused fmin) followed by supervision_pool: two launches and two full passes over every mask.  Here
// one launch does all of it in one pass: a block owns a band of rows of one slot, projects the footprint itself
// (shared device code with footprint_kernels.cu, so the rasterised pixels are the same), streams its rows once
// (read mask + segment id, write mask) and privatises (sum, count) per segment in shared memory.  The last block of a
// slot to finish (a ticket in the workspace) turns the sums into y / y_valid and returns its workspace rows to zero, so
// the call needs neither a memset nor a second launch.
//
// The mask is stored with one channel: the reference's three channels are rendered with colour (1, 1, 1) and stay
// identical, and its nanmean over them is reproduced by summing the value three times and dividing by 3, so the
// per-pixel signal rounds as the reference's (and as supervision_pool's) does.
#include "mission_graph.h"

#include "footprint_common.cuh"
#include "host_common.h"

namespace wvn {
namespace {

using namespace footprint;

constexpr int kRowsPerBlock = 16;
constexpr int kThreads = 256;
constexpr int kMaxPoints = 1024;
constexpr int kMaxSegments = 4096;

// smem: sum[smax] | cnt[smax] | px[n + 1] | py[n + 1] | Tcw[16]
__global__ void __launch_bounds__(kThreads)
mission_propagate_kernel(MissionPropagateArgs a, const int* __restrict__ slots, const unsigned char* __restrict__ restart,
                         const float* __restrict__ Kmat, const float* __restrict__ pose, const float* __restrict__ points,
                         const float* __restrict__ traversability, const int* __restrict__ seg, float* __restrict__ mask,
                         float* __restrict__ y_out, unsigned char* __restrict__ y_valid, int* __restrict__ slot_valid,
                         float* __restrict__ g_sum, float* __restrict__ g_cnt, unsigned int* __restrict__ tickets) {
  extern __shared__ float sm[];
  const int n = a.n_points, smax = a.smax;
  float* s_sum = sm;
  float* s_cnt = s_sum + smax;
  float* px = s_cnt + smax;
  float* py = px + n + 1;
  float* Tcw = py + n + 1;
  __shared__ int s_last;
  const int i = blockIdx.y;
  const long long slot = slots[i];
  const int t = threadIdx.x;
  if (t == 0) invert4x4(pose + 16 * slot, Tcw);
  for (int j = t; j < 2 * smax; j += kThreads) sm[j] = 0.f;
  __syncthreads();
  const float* Kb = Kmat + 16 * slot;
  for (int p = t; p < n; p += kThreads) {
    float u, v;
    bool ok;
    project_point(Tcw, Kb, points + 3 * static_cast<size_t>(p), a.w, a.h, u, v, ok);
    px[p] = u; py[p] = v;
  }
  __syncthreads();
  if (t == 0) { px[n] = px[0]; py[n] = py[0]; }
  __syncthreads();

  const float trav = *traversability;
  const bool zero = restart != nullptr && restart[i] != 0;   // the node's mask was dropped: restart from zeros
  const int warp = t >> 5, lane = t & 31;
  const float wf = static_cast<float>(a.w);
  const size_t plane = static_cast<size_t>(a.h) * a.w;
  float* mk = mask + slot * plane;
  const int* sg = seg + slot * plane;
  for (int ry = warp; ry < kRowsPerBlock; ry += kThreads / 32) {
    const int yy = blockIdx.x * kRowsPerBlock + ry;
    if (yy >= a.h) break;
    float xl, xr;
    row_span(px, py, n, static_cast<float>(yy), wf, lane, xl, xr);
    const size_t row = static_cast<size_t>(yy) * a.w;
    for (int x = lane; x < a.w; x += 32) {
      const float xf = static_cast<float>(x);
      const float v = (xf >= xl && xf <= xr) ? 1.f : nanf("");   // colour 1, masks[masks == 0] = nan
      const float m = fminf(zero ? 0.f : mk[row + x], v * trav);  // torch.fmin: NaN-ignoring
      mk[row + x] = m;
      if (m == m) {
        const int id = sg[row + x];
        if (id >= 0 && id < smax) {
          float s = 0.f;   // nanmean over the reference's three identical channels
          s += m; s += m; s += m;
          atomicAdd(&s_sum[id], s / 3.f);
          atomicAdd(&s_cnt[id], 1.f);
        }
      }
    }
  }
  __syncthreads();
  float* gs = g_sum + static_cast<size_t>(i) * smax;
  float* gc = g_cnt + static_cast<size_t>(i) * smax;
  for (int j = t; j < smax; j += kThreads) {
    if (s_cnt[j] > 0.f) {
      atomicAdd(&gs[j], s_sum[j]);
      atomicAdd(&gc[j], s_cnt[j]);
    }
  }
  __threadfence();
  __syncthreads();
  if (t == 0) s_last = atomicAdd(&tickets[i], 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  int any = 0;
  for (int j = t; j < smax; j += kThreads) {
    const float c = __ldcg(gc + j), s = __ldcg(gs + j);
    const float v = c > 0.f ? s / c : 0.f;   // 0 / 0 -> nan -> nan_to_num(0) in the reference
    y_out[slot * smax + j] = v;
    y_valid[slot * smax + j] = v > 0.f ? 1 : 0;
    any |= v > 0.f;
    gs[j] = 0.f;
    gc[j] = 0.f;
  }
  any = __syncthreads_or(any);
  if (t == 0) {
    tickets[i] = 0;
    if (slot_valid) slot_valid[slot] = any;
  }
}

}  // namespace

size_t mission_propagate_workspace_bytes(int max_slots, int smax) {
  if (max_slots <= 0 || smax <= 0) return 0;
  return static_cast<size_t>(max_slots) * (2 * static_cast<size_t>(smax) * sizeof(float) + sizeof(unsigned int));
}

int mission_propagate(const MissionPropagateArgs& a, const int* slots, const unsigned char* restart, const float* K,
                      const float* pose, const float* points, const float* traversability, const int* seg, float* mask,
                      float* y, unsigned char* y_valid, int* slot_valid, void* workspace, cudaStream_t stream) {
  WVN_REQUIRE(a.n_slots > 0 && a.n_slots <= 65535 && a.h > 0 && a.w > 0,
              "mission_propagate: bad sizes (slots %d, %dx%d)", a.n_slots, a.h, a.w);
  WVN_REQUIRE(a.n_points > 0 && a.n_points <= kMaxPoints, "mission_propagate: 1 to %d footprint points (got %d)",
              kMaxPoints, a.n_points);
  WVN_REQUIRE(a.smax > 0 && a.smax <= kMaxSegments, "mission_propagate: smax %d outside [1, %d]", a.smax, kMaxSegments);
  const size_t smem = sizeof(float) * (2 * static_cast<size_t>(a.smax) + 2 * (a.n_points + 1) + 16);   // <= 41 KB
  float* g_sum = reinterpret_cast<float*>(workspace);
  float* g_cnt = g_sum + static_cast<size_t>(a.n_slots) * a.smax;
  unsigned int* tickets = reinterpret_cast<unsigned int*>(g_cnt + static_cast<size_t>(a.n_slots) * a.smax);
  dim3 grid((a.h + kRowsPerBlock - 1) / kRowsPerBlock, a.n_slots);
  mission_propagate_kernel<<<grid, kThreads, smem, stream>>>(a, slots, restart, K, pose, points, traversability, seg, mask,
                                                             y, y_valid, slot_valid, g_sum, g_cnt, tickets);
  WVN_CHECK_LAUNCH("mission_propagate_kernel");
  return WVN_OK;
}

}  // namespace wvn
