// wvn-b200: device code shared by the footprint kernels (footprint_kernels.cu) and the mission-graph label propagation
// (mission_graph.cu): pose inverse, kornia's homogeneous division, the pinhole projection of one footprint point and the
// [left, right] span of one image row of the convex polygon.  Both kernels inline the same code, so a footprint
// rasterised by either is the same set of pixels.
#pragma once

#include <cuda_runtime.h>

namespace wvn {
namespace footprint {

// General 4x4 inverse (the reference calls Tensor.inverse(), not an SE(3) shortcut) by cofactors in double.
__device__ inline void invert4x4(const float* __restrict__ m, float* __restrict__ out) {
  double a[16], inv[16];
  for (int i = 0; i < 16; ++i) a[i] = m[i];
  inv[0] = a[5] * a[10] * a[15] - a[5] * a[11] * a[14] - a[9] * a[6] * a[15] + a[9] * a[7] * a[14] + a[13] * a[6] * a[11] - a[13] * a[7] * a[10];
  inv[4] = -a[4] * a[10] * a[15] + a[4] * a[11] * a[14] + a[8] * a[6] * a[15] - a[8] * a[7] * a[14] - a[12] * a[6] * a[11] + a[12] * a[7] * a[10];
  inv[8] = a[4] * a[9] * a[15] - a[4] * a[11] * a[13] - a[8] * a[5] * a[15] + a[8] * a[7] * a[13] + a[12] * a[5] * a[11] - a[12] * a[7] * a[9];
  inv[12] = -a[4] * a[9] * a[14] + a[4] * a[10] * a[13] + a[8] * a[5] * a[14] - a[8] * a[6] * a[13] - a[12] * a[5] * a[10] + a[12] * a[6] * a[9];
  inv[1] = -a[1] * a[10] * a[15] + a[1] * a[11] * a[14] + a[9] * a[2] * a[15] - a[9] * a[3] * a[14] - a[13] * a[2] * a[11] + a[13] * a[3] * a[10];
  inv[5] = a[0] * a[10] * a[15] - a[0] * a[11] * a[14] - a[8] * a[2] * a[15] + a[8] * a[3] * a[14] + a[12] * a[2] * a[11] - a[12] * a[3] * a[10];
  inv[9] = -a[0] * a[9] * a[15] + a[0] * a[11] * a[13] + a[8] * a[1] * a[15] - a[8] * a[3] * a[13] - a[12] * a[1] * a[11] + a[12] * a[3] * a[9];
  inv[13] = a[0] * a[9] * a[14] - a[0] * a[10] * a[13] - a[8] * a[1] * a[14] + a[8] * a[2] * a[13] + a[12] * a[1] * a[10] - a[12] * a[2] * a[9];
  inv[2] = a[1] * a[6] * a[15] - a[1] * a[7] * a[14] - a[5] * a[2] * a[15] + a[5] * a[3] * a[14] + a[13] * a[2] * a[7] - a[13] * a[3] * a[6];
  inv[6] = -a[0] * a[6] * a[15] + a[0] * a[7] * a[14] + a[4] * a[2] * a[15] - a[4] * a[3] * a[14] - a[12] * a[2] * a[7] + a[12] * a[3] * a[6];
  inv[10] = a[0] * a[5] * a[15] - a[0] * a[7] * a[13] - a[4] * a[1] * a[15] + a[4] * a[3] * a[13] + a[12] * a[1] * a[7] - a[12] * a[3] * a[5];
  inv[14] = -a[0] * a[5] * a[14] + a[0] * a[6] * a[13] + a[4] * a[1] * a[14] - a[4] * a[2] * a[13] - a[12] * a[1] * a[6] + a[12] * a[2] * a[5];
  inv[3] = -a[1] * a[6] * a[11] + a[1] * a[7] * a[10] + a[5] * a[2] * a[11] - a[5] * a[3] * a[10] - a[9] * a[2] * a[7] + a[9] * a[3] * a[6];
  inv[7] = a[0] * a[6] * a[11] - a[0] * a[7] * a[10] - a[4] * a[2] * a[11] + a[4] * a[3] * a[10] + a[8] * a[2] * a[7] - a[8] * a[3] * a[6];
  inv[11] = -a[0] * a[5] * a[11] + a[0] * a[7] * a[9] + a[4] * a[1] * a[11] - a[4] * a[3] * a[9] - a[8] * a[1] * a[7] + a[8] * a[3] * a[5];
  inv[15] = a[0] * a[5] * a[10] - a[0] * a[6] * a[9] - a[4] * a[1] * a[10] + a[4] * a[2] * a[9] + a[8] * a[1] * a[6] - a[8] * a[2] * a[5];
  const double det = a[0] * inv[0] + a[1] * inv[4] + a[2] * inv[8] + a[3] * inv[12];
  const double r = 1.0 / det;  // singular pose -> inf / NaN, like Tensor.inverse() failing loudly is not possible here
  for (int i = 0; i < 16; ++i) out[i] = static_cast<float>(inv[i] * r);
}

// kornia convert_points_from_homogeneous: scale = 1 / (z + 1e-8) where |z| > 1e-8, else 1.
__device__ __forceinline__ float hom_scale(float z) { return fabsf(z) > 1e-8f ? 1.0f / (z + 1e-8f) : 1.0f; }

__device__ __forceinline__ void transform4(const float* __restrict__ T, float x, float y, float z, float& ox, float& oy,
                                           float& oz) {
  const float hx = T[0] * x + T[1] * y + T[2] * z + T[3];
  const float hy = T[4] * x + T[5] * y + T[6] * z + T[7];
  const float hz = T[8] * x + T[9] * y + T[10] * z + T[11];
  const float hw = T[12] * x + T[13] * y + T[14] * z + T[15];
  const float s = hom_scale(hw);
  ox = s * hx; oy = s * hy; oz = s * hz;
}

// One world point p[3] -> pixel (u, v) through Tcw (world -> camera) and K; NaN for points behind the camera.
// ok: check_validity (in front of the camera and inside [0, w] x [0, h]).
__device__ __forceinline__ void project_point(const float* __restrict__ Tcw, const float* __restrict__ K,
                                              const float* __restrict__ p, int w, int h, float& u, float& v, bool& ok) {
  float cx, cy, cz, ix, iy, iz;
  transform4(Tcw, p[0], p[1], p[2], cx, cy, cz);       // world -> camera
  transform4(K, cx, cy, cz, ix, iy, iz);               // PinholeCamera.project with identity extrinsics ...
  const float s = hom_scale(iz);                       // ... and its own homogeneous division
  u = s * ix; v = s * iy;
  const bool vz = cz >= 0.f;
  ok = vz && u >= 0.f && u <= static_cast<float>(w) && v >= 0.f && v <= static_cast<float>(h);
  if (!vz) u = v = nanf("");
}

// kornia _get_convex_edges for image row yf: the [xl, xr] span over the n edges of the closed polygon px / py[n + 1],
// reduced over the warp (every lane returns the span).  xl > xr when the row misses the polygon.
__device__ __forceinline__ void row_span(const float* __restrict__ px, const float* __restrict__ py, int n, float yf,
                                         float wf, int lane, float& xl_out, float& xr_out) {
  float xl = wf, xr = -1.f;
  for (int e = lane; e < n; e += 32) {
    const float xs = px[e], ys = py[e], xe = px[e + 1], ye = py[e + 1];
    const bool act = (ys <= yf && yf <= ye) || (ys >= yf && yf >= ye);   // false for NaN vertices
    if (act) {
      // same operation order as the reference's tensor expression (no fused multiply-add)
      float dx = __fdiv_rn(__fsub_rn(xe, xs), __fadd_rn(__fsub_rn(ye, ys), 1e-12f));
      dx = fminf(fmaxf(dx, -wf), wf);
      const float x = __fadd_rn(__fmul_rn(__fsub_rn(yf, ys), dx), xs);
      // torch.min / max propagate NaN; x can only be NaN for inf vertices, which the clamp removes except inf * 0
      xl = (x != x || xl != xl) ? nanf("") : fminf(xl, x);
      xr = (x != x || xr != xr) ? nanf("") : fmaxf(xr, x);
    }
  }
  for (int o = 16; o; o >>= 1) {
    const float ol = __shfl_xor_sync(0xffffffffu, xl, o), orr = __shfl_xor_sync(0xffffffffu, xr, o);
    xl = (ol != ol || xl != xl) ? nanf("") : fminf(xl, ol);
    xr = (orr != orr || xr != xr) ? nanf("") : fmaxf(xr, orr);
  }
  xl_out = xl; xr_out = xr;
}

}  // namespace footprint
}  // namespace wvn
