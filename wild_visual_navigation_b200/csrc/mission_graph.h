// wvn-b200: internal interface of mission_graph.cu.
#pragma once

#include <cuda_runtime.h>

#include <cstddef>

namespace wvn {

struct MissionPropagateArgs {
  int n_slots = 0;   // entries of the slot list
  int n_points = 0;  // footprint polygon points (convex, in order)
  int h = 0, w = 0;  // mask / segmentation size
  int smax = 0;      // per-segment label rows per slot
};

// Bytes of the propagation workspace for up to max_slots list entries: per entry smax sums, smax counts and one
// block ticket.  It must be zero before the first call; every call leaves it zero again.
size_t mission_propagate_workspace_bytes(int max_slots, int smax);

// For every list entry i, slot s = slots[i]: project and rasterise the footprint into slot s's camera (K[s], pose[s]),
// mask[s] = fmin(restart[i] ? 0 : mask[s], render * *traversability) in place, then y[s] / y_valid[s] = the per-segment
// mean of the new mask over seg[s] (ids outside [0, smax) ignored) and slot_valid[s] = any(y_valid[s]).
int mission_propagate(const MissionPropagateArgs& a, const int* slots, const unsigned char* restart, const float* K,
                      const float* pose, const float* points, const float* traversability, const int* seg, float* mask,
                      float* y, unsigned char* y_valid, int* slot_valid, void* workspace, cudaStream_t stream);

}  // namespace wvn
