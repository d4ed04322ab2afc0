// wvn-b200: footprint projection + convex-polygon rasterisation into supervision masks.
//
// Replaces ImageProjector.project_and_render (image_projector/image_projector.py:152-197: pose inverse,
// kornia transform_points / PinholeCamera.project, NaN for points behind the camera, kornia draw_convex_polygon,
// 0 -> NaN) and, optionally fused, the mask update of TraversabilityEstimator.add_supervision_node
// (traversability_estimator.py:281-284: mask * traversability, fmin into the mission nodes' supervision masks).
// The reference expands an (H, N) edge table per image and three (B, 3, H, W) temporaries; here one block handles a band of
// rows of one image: it projects the N footprint points itself (N is ~40), each warp finds the [left, right] span of a
// row over the N edges with two shuffles trees and streams the row out.  HBM-bound: 12 B written per pixel (+ 24 B
// read-modify-write when fused).
#include "footprint_kernels.h"

#include "footprint_common.cuh"
#include "host_common.h"

namespace wvn {
namespace {

using namespace footprint;

constexpr int kRowsPerBlock = 16;
constexpr int kThreads = 256;

// smem: px[n + 1] | py[n + 1] (polygon closed by repeating point 0; kornia appends it unless last == first, and a
// repeated vertex only adds a zero-length edge that cannot change any span) | Tcw[16]
__global__ void __launch_bounds__(kThreads)
footprint_render_kernel(FootprintArgs a, const float* __restrict__ Kmat, const float* __restrict__ pose,
                        const float* __restrict__ points, const float* __restrict__ colors,
                        const float* __restrict__ traversability, float* __restrict__ masks,
                        float* __restrict__ projected, unsigned char* __restrict__ valid, float* __restrict__ sup) {
  extern __shared__ float sm[];
  const int n = a.n_points;
  float* px = sm;
  float* py = px + n + 1;
  float* Tcw = py + n + 1;
  const int b = blockIdx.y;
  const int t = threadIdx.x;
  if (t == 0) invert4x4(pose + 16 * static_cast<size_t>(b), Tcw);
  __syncthreads();
  const float* Kb = Kmat + 16 * static_cast<size_t>(b);
  for (int i = t; i < n; i += kThreads) {
    float u, v;
    bool ok;
    project_point(Tcw, Kb, points + (static_cast<size_t>(b) * n + i) * 3, a.w, a.h, u, v, ok);
    px[i] = u; py[i] = v;
    if (blockIdx.x == 0) {
      if (projected) { projected[(static_cast<size_t>(b) * n + i) * 2] = u; projected[(static_cast<size_t>(b) * n + i) * 2 + 1] = v; }
      if (valid) valid[static_cast<size_t>(b) * n + i] = ok ? 1 : 0;
    }
  }
  __syncthreads();
  if (t == 0) { px[n] = px[0]; py[n] = py[0]; }
  __syncthreads();
  if (!masks && !sup) return;

  float col[3];
  for (int c = 0; c < 3; ++c) col[c] = colors[(a.color_batched ? 3 * b : 0) + c];
  const float trav = traversability ? *traversability : 1.f;
  const int warp = t >> 5, lane = t & 31;
  const float wf = static_cast<float>(a.w);
  const size_t plane = static_cast<size_t>(a.h) * a.w;
  for (int ry = warp; ry < kRowsPerBlock; ry += kThreads / 32) {
    const int y = blockIdx.x * kRowsPerBlock + ry;
    if (y >= a.h) break;
    const float yf = static_cast<float>(y);
    float xl, xr;
    row_span(px, py, n, yf, wf, lane, xl, xr);
    const size_t row = static_cast<size_t>(b) * 3 * plane + static_cast<size_t>(y) * a.w;
    for (int x = lane; x < a.w; x += 32) {
      const float xf = static_cast<float>(x);
      const bool in = xf >= xl && xf <= xr;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float v0 = in ? col[c] : 0.f;
        const float v = v0 == 0.f ? nanf("") : v0;                  // masks[masks == 0] = nan
        const size_t idx = row + c * plane + x;
        if (masks) masks[idx] = v;
        if (sup) sup[idx] = fminf(sup[idx], v * trav);               // torch.fmin: NaN-ignoring, like fminf
      }
    }
  }
}

}  // namespace

int footprint_render(const FootprintArgs& a, const float* K, const float* pose, const float* points, const float* colors,
                     const float* traversability, float* masks, float* projected, unsigned char* valid, float* sup,
                     cudaStream_t stream) {
  WVN_REQUIRE(a.batch > 0 && a.n_points > 0 && a.h > 0 && a.w > 0, "footprint_render: bad sizes (batch %d, points %d, %dx%d)",
              a.batch, a.n_points, a.h, a.w);
  WVN_REQUIRE(a.n_points <= 8192, "footprint_render: at most 8192 polygon points (got %d)", a.n_points);
  const size_t smem = sizeof(float) * (2 * (a.n_points + 1) + 16);
  if (smem > 48 * 1024)
    WVN_CHECK_CUDA(cudaFuncSetAttribute(footprint_render_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  dim3 grid((a.h + kRowsPerBlock - 1) / kRowsPerBlock, a.batch);
  footprint_render_kernel<<<grid, kThreads, smem, stream>>>(a, K, pose, points, colors, traversability, masks, projected,
                                                            valid, sup);
  WVN_CHECK_LAUNCH("footprint_render_kernel");
  return WVN_OK;
}

}  // namespace wvn
