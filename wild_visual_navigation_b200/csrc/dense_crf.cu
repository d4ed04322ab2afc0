// wvn-b200: STEGO's dense CRF on sm_90a (definition: oracle/dense_crf.py) — replaces pydensecrf's DenseCRF2D with
// addPairwiseGaussian(sxy=1, compat=3), addPairwiseBilateral(sxy=67, srgb=3, compat=4) and inference(10), which
// upstream runs on the CPU one image at a time.
//
// Per chunk of frames, for each of the two kernels (spatial d = 2, bilateral d = 5):
//   lattice build : one thread per pixel elevates its features, finds its enclosing simplex and writes the d+1
//                   (packed vertex key, pixel * (d+1) + r) pairs with their barycentric weights; CUB's stable radix
//                   sort orders the pairs by key, a scan numbers the unique keys (the vertices, in ascending key order)
//                   and every pair learns its vertex; each vertex's 2 (d+1) blur neighbours are found once by binary
//                   search in the sorted keys.  The frame sits in the key's top bits, so a chunk is one lattice.
//   filter        : splat = one warp per vertex summing its sorted run in a fixed order (no atomics), d+1 blur
//                   passes, slice = one warp per pixel.  The spatial slice leaves w * norm * K(norm Q) per pixel; the
//                   bilateral slice adds its own term, the unary and does the exp-normalise into the next Q.
// Everything is sized at create for the worst case ((d+1) S^2 vertices per frame), so a run allocates nothing and never
// waits on the host; the vertex counts stay on the device and every kernel loops over them.
#include "dense_crf.h"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <math.h>

#include <algorithm>
#include <memory>

#include "host_common.h"

namespace wvn {

__host__ __device__ constexpr int key_bits(int d) { return d == 2 ? 16 : 11; }

struct LatticeBufs {
  int d = 0;
  long long entries = 0;           // chunk * S^2 * (d+1): also the worst-case vertex count
  float* bary = nullptr;           // [entries] weight of entry p*(d+1)+r
  int* offs = nullptr;             // [entries] vertex of entry
  int* sorted = nullptr;           // [entries] entry ids in vertex order
  int* start = nullptr;            // [entries + 1] first sorted position of each vertex
  unsigned long long* ukeys = nullptr;  // [entries] packed key of each vertex
  int2* nbr = nullptr;             // [(d+1) * entries] blur neighbours of each vertex per axis, -1 = none
  float* norm = nullptr;           // [chunk * S^2]
  float weight = 0.f;
  float feat_div[2] = {1.f, 1.f};  // spatial and colour standard deviations
  float scale[5] = {};
};

}  // namespace wvn

struct wvn_crf {
  int S = 0, N = 0, K = 0, chunk = 0, iters = 0;
  wvn::DevBuf arena;
  wvn::LatticeBufs lat[2];
  unsigned long long *keys_in = nullptr, *keys_out = nullptr;
  int *vals_in = nullptr, *scan = nullptr, *m = nullptr;  // m[2]: vertex counts
  float *va = nullptr, *vb = nullptr;                    // [entries_max * K] vertex values, double-buffered
  float *U = nullptr, *Q = nullptr, *acc = nullptr;      // [chunk * N * K]
  uchar4* bgr = nullptr;                                 // [chunk * N]
  void* cub_tmp = nullptr;
  size_t cub_bytes = 0;
  int frames = 0;                                        // frames of the chunk whose lattices are built
};

namespace wvn {

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

struct ImgGeom {
  const void* img;
  int u8, in_h, in_w, S, frame0;
  int crop_top, crop_left;
  float scale_y, scale_x;
};

// np.array(to_pil_image(unnorm(normalize(v))))[:, :, ::-1]: float32, no contraction, truncation
__global__ void __launch_bounds__(kThreads) crf_image_kernel(ImgGeom g, int frames, uchar4* __restrict__ bgr) {
  const long long n = static_cast<long long>(g.S) * g.S;
  for (long long i = blockIdx.x * static_cast<long long>(kThreads) + threadIdx.x; i < frames * n;
       i += static_cast<long long>(gridDim.x) * kThreads) {
    const int f = static_cast<int>(i / n), p = static_cast<int>(i % n);
    const int y = p / g.S, x = p % g.S;
    const int sy = min(static_cast<int>(floorf((y + g.crop_top) * g.scale_y)), g.in_h - 1);
    const int sx = min(static_cast<int>(floorf((x + g.crop_left) * g.scale_x)), g.in_w - 1);
    const long long b = g.frame0 + f;
    const float mean[3] = {0.485f, 0.456f, 0.406f}, sd[3] = {0.229f, 0.224f, 0.225f};
    unsigned char out[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v;
      if (g.u8) {
        const unsigned char* im = reinterpret_cast<const unsigned char*>(g.img);
        v = __fdiv_rn(static_cast<float>(im[((b * g.in_h + sy) * g.in_w + sx) * 3 + c]), 255.f);
      } else {
        const float* im = reinterpret_cast<const float*>(g.img);
        v = im[((b * 3 + c) * g.in_h + sy) * g.in_w + sx];
      }
      const float xn = __fdiv_rn(__fsub_rn(v, mean[c]), sd[c]);
      const float u = __fadd_rn(__fmul_rn(xn, sd[c]), mean[c]);
      const int q = static_cast<int>(__fmul_rn(u, 255.f));
      out[c] = static_cast<unsigned char>(min(255, max(0, q)));
    }
    bgr[i] = make_uchar4(out[2], out[1], out[0], 0);  // b, g, r
  }
}

// One thread per pixel of the chunk: elevation, simplex, barycentric weights, the d+1 (key, entry) pairs.
template <int D>
__global__ void __launch_bounds__(kThreads)
crf_elevate_kernel(LatticeBufs L, int S, int frames, const uchar4* __restrict__ bgr,
                   unsigned long long* __restrict__ keys, int* __restrict__ vals) {
  const long long n = static_cast<long long>(S) * S;
  constexpr int bits = key_bits(D);
  for (long long i = blockIdx.x * static_cast<long long>(kThreads) + threadIdx.x; i < frames * n;
       i += static_cast<long long>(gridDim.x) * kThreads) {
    const int f = static_cast<int>(i / n), p = static_cast<int>(i % n);
    float feat[D];
    feat[0] = __fdiv_rn(static_cast<float>(p % S), L.feat_div[0]);
    feat[1] = __fdiv_rn(static_cast<float>(p / S), L.feat_div[0]);
    if (D == 5) {
      const uchar4 c = bgr[i];
      feat[2 % D] = __fdiv_rn(static_cast<float>(c.x), L.feat_div[1]);
      feat[3 % D] = __fdiv_rn(static_cast<float>(c.y), L.feat_div[1]);
      feat[4 % D] = __fdiv_rn(static_cast<float>(c.z), L.feat_div[1]);
    }
    float E[D + 1];
    float sm = 0.f;
#pragma unroll
    for (int j = D; j > 0; --j) {
      const float cf = __fmul_rn(feat[j - 1], L.scale[j - 1]);
      E[j] = __fsub_rn(sm, __fmul_rn(static_cast<float>(j), cf));
      sm = __fadd_rn(sm, cf);
    }
    E[0] = sm;
    const float down = 1.0f / (D + 1), up = static_cast<float>(D + 1);
    int rem0[D + 1], rank[D + 1];
    int total = 0;
#pragma unroll
    for (int j = 0; j <= D; ++j) {
      const float v = __fmul_rn(down, E[j]);
      const float hi = __fmul_rn(ceilf(v), up), lo = __fmul_rn(floorf(v), up);
      rem0[j] = static_cast<int>(__fsub_rn(hi, E[j]) < __fsub_rn(E[j], lo) ? hi : lo);
      total += rem0[j] / (D + 1);
      rank[j] = 0;
    }
#pragma unroll
    for (int a = 0; a < D; ++a) {
      const float da = __fsub_rn(E[a], static_cast<float>(rem0[a]));
#pragma unroll
      for (int b = a + 1; b <= D; ++b) {
        if (da < __fsub_rn(E[b], static_cast<float>(rem0[b]))) ++rank[a];
        else ++rank[b];
      }
    }
#pragma unroll
    for (int j = 0; j <= D; ++j) {
      rank[j] += total;
      if (rank[j] < 0) { rank[j] += D + 1; rem0[j] += D + 1; }
      else if (rank[j] > D) { rank[j] -= D + 1; rem0[j] -= D + 1; }
    }
    float bary[D + 2];
#pragma unroll
    for (int s = 0; s < D + 2; ++s) bary[s] = 0.f;
#pragma unroll
    for (int j = 0; j <= D; ++j) {
      const float v = __fmul_rn(__fsub_rn(E[j], static_cast<float>(rem0[j])), down);
      const int s0 = D - rank[j];
#pragma unroll
      for (int s = 0; s <= D; ++s) {
        if (s == s0) {
          bary[s] = __fadd_rn(bary[s], v);
          bary[s + 1] = __fsub_rn(bary[s + 1], v);
        }
      }
    }
    bary[0] = __double2float_rn(static_cast<double>(bary[0]) + (1.0 + static_cast<double>(bary[D + 1])));
    const unsigned long long frame_bits = static_cast<unsigned long long>(f) << (bits * D);
#pragma unroll
    for (int r = 0; r <= D; ++r) {
      unsigned long long key = frame_bits;
#pragma unroll
      for (int j = 0; j < D; ++j) {
        const int k = rem0[j] + (rank[j] <= D - r ? r : r - (D + 1));
        key |= static_cast<unsigned long long>(k + (1 << (bits - 1))) << (bits * j);
      }
      const long long e = i * (D + 1) + r;
      keys[e] = key;
      vals[e] = static_cast<int>(e);
      L.bary[e] = bary[r];
    }
  }
}

__global__ void __launch_bounds__(kThreads)
crf_flag_kernel(const unsigned long long* __restrict__ keys, long long n, int* __restrict__ flags) {
  for (long long i = blockIdx.x * static_cast<long long>(kThreads) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * kThreads)
    flags[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1 : 0;
}

// vid: inclusive scan of the flags (1-based vertex number of every sorted pair)
__global__ void __launch_bounds__(kThreads)
crf_vertex_kernel(LatticeBufs L, const unsigned long long* __restrict__ keys, const int* __restrict__ sorted_ids,
                  const int* __restrict__ vid, long long n, int* __restrict__ m) {
  for (long long i = blockIdx.x * static_cast<long long>(kThreads) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * kThreads) {
    const int v = vid[i] - 1;
    const int e = sorted_ids[i];
    L.sorted[i] = e;
    L.offs[e] = v;
    if (i == 0 || v != vid[i - 1] - 1) {
      L.start[v] = static_cast<int>(i);
      L.ukeys[v] = keys[i];
    }
    if (i == n - 1) {
      L.start[v + 1] = static_cast<int>(n);
      *m = v + 1;
    }
  }
}

__device__ __forceinline__ int find_key(const unsigned long long* __restrict__ keys, int m, unsigned long long k) {
  int lo = 0, hi = m;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (keys[mid] < k) lo = mid + 1;
    else hi = mid;
  }
  return (lo < m && keys[lo] == k) ? lo : -1;
}

template <int D>
__global__ void __launch_bounds__(kThreads) crf_neighbour_kernel(LatticeBufs L, const int* __restrict__ m_ptr) {
  constexpr int bits = key_bits(D);
  constexpr unsigned long long mask = (1ull << bits) - 1;
  const int m = *m_ptr;
  for (int v = blockIdx.x * kThreads + threadIdx.x; v < m; v += gridDim.x * kThreads) {
    const unsigned long long key = L.ukeys[v];
    const unsigned long long frame = key >> (bits * D) << (bits * D);
    int k[D];
#pragma unroll
    for (int j = 0; j < D; ++j) k[j] = static_cast<int>((key >> (bits * j)) & mask);  // biased
#pragma unroll 1
    for (int ax = 0; ax <= D; ++ax) {
      unsigned long long k1 = frame, k2 = frame;
#pragma unroll
      for (int j = 0; j < D; ++j) {
        const int a = j == ax ? k[j] + D : k[j] - 1;
        const int b = j == ax ? k[j] - D : k[j] + 1;
        k1 |= static_cast<unsigned long long>(a) << (bits * j);
        k2 |= static_cast<unsigned long long>(b) << (bits * j);
      }
      L.nbr[static_cast<long long>(ax) * L.entries + v] = make_int2(find_key(L.ukeys, m, k1), find_key(L.ukeys, m, k2));
    }
  }
}

// One warp per vertex: sum of w * scale[p] * in[p][k] over the vertex's sorted run (in == nullptr: in = 1).
template <int D>
__global__ void __launch_bounds__(kThreads)
crf_splat_kernel(LatticeBufs L, const int* __restrict__ m_ptr, const float* __restrict__ in, const float* __restrict__ scale,
                 int V, float* __restrict__ out) {
  const int m = *m_ptr;
  const int lane = threadIdx.x & 31;
  for (int v = blockIdx.x * kWarps + (threadIdx.x >> 5); v < m; v += gridDim.x * kWarps) {
    float acc[2] = {0.f, 0.f};
    const int e1 = L.start[v + 1];
    for (int e = L.start[v]; e < e1; ++e) {
      const int id = L.sorted[e];
      const long long p = id / (D + 1);
      const float w = L.bary[id];
      const float s = scale ? scale[p] : 1.f;
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        const int k = lane + 32 * t;
        if (k < V) acc[t] = __fadd_rn(acc[t], __fmul_rn(w, in ? __fmul_rn(s, in[p * V + k]) : s));
      }
    }
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const int k = lane + 32 * t;
      if (k < V) out[static_cast<long long>(v) * V + k] = acc[t];
    }
  }
}

__global__ void __launch_bounds__(kThreads)
crf_blur_kernel(const int2* __restrict__ nbr, const int* __restrict__ m_ptr, int V, const float* __restrict__ src,
                float* __restrict__ dst) {
  const long long n = static_cast<long long>(*m_ptr) * V;
  for (long long i = blockIdx.x * static_cast<long long>(kThreads) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * kThreads) {
    const long long v = i / V;
    const int k = static_cast<int>(i % V);
    const int2 nb = nbr[v];
    const float a = nb.x >= 0 ? src[static_cast<long long>(nb.x) * V + k] : 0.f;
    const float b = nb.y >= 0 ? src[static_cast<long long>(nb.y) * V + k] : 0.f;
    dst[i] = __fadd_rn(src[i], __fmul_rn(0.5f, __fadd_rn(a, b)));
  }
}

enum SliceMode : int { SLICE_WRITE = 0, SLICE_NORM = 1, SLICE_ACC = 2, SLICE_UPDATE = 3 };

// One warp per pixel: sum_r w_r * vertex_r * alpha, then
//   SLICE_WRITE : out = that;   SLICE_NORM : norm = 1 / sqrt(that + 1e-20)  (V = 1)
//   SLICE_ACC   : acc = weight * norm * that
//   SLICE_UPDATE: Q = softmax(-U + acc + weight * norm * that)
template <int D>
__global__ void __launch_bounds__(kThreads)
crf_slice_kernel(LatticeBufs L, long long npix, const float* __restrict__ vals, int V, int mode, float* __restrict__ out,
                 const float* __restrict__ U, const float* __restrict__ acc, float* __restrict__ Q) {
  const float alpha = 1.0f / (1.0f + exp2f(-static_cast<float>(D)));
  const int lane = threadIdx.x & 31;
  for (long long p = blockIdx.x * static_cast<long long>(kWarps) + (threadIdx.x >> 5); p < npix;
       p += static_cast<long long>(gridDim.x) * kWarps) {
    float s[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r <= D; ++r) {
      const long long e = p * (D + 1) + r;
      const long long o = L.offs[e];
      const float w = L.bary[e];
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        const int k = lane + 32 * t;
        if (k < V) s[t] = __fadd_rn(s[t], __fmul_rn(__fmul_rn(w, vals[o * V + k]), alpha));
      }
    }
    if (mode == SLICE_NORM) {
      if (lane == 0) L.norm[p] = 1.f / sqrtf(s[0] + 1e-20f);
      continue;
    }
    if (mode == SLICE_WRITE) {
#pragma unroll
      for (int t = 0; t < 2; ++t)
        if (lane + 32 * t < V) out[p * V + lane + 32 * t] = s[t];
      continue;
    }
    const float c = L.weight * L.norm[p];
    if (mode == SLICE_ACC) {
#pragma unroll
      for (int t = 0; t < 2; ++t)
        if (lane + 32 * t < V) out[p * V + lane + 32 * t] = c * s[t];
      continue;
    }
    float x[2];
    float mx = -INFINITY;
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const int k = lane + 32 * t;
      x[t] = k < V ? -U[p * V + k] + acc[p * V + k] + c * s[t] : -INFINITY;
      mx = fmaxf(mx, x[t]);
    }
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      x[t] = lane + 32 * t < V ? __expf(x[t] - mx) : 0.f;
      sum += x[t];
    }
    const float inv = 1.f / warp_sum(sum);
#pragma unroll
    for (int t = 0; t < 2; ++t)
      if (lane + 32 * t < V) Q[p * V + lane + 32 * t] = x[t] * inv;
  }
}

__device__ __forceinline__ void ac_false(int dst, float scale, int in_size, int& i0, int& i1, float& w1) {
  float s = (dst + 0.5f) * scale - 0.5f;
  s = fmaxf(s, 0.f);
  i0 = min(static_cast<int>(s), in_size - 1);
  i1 = min(i0 + 1, in_size - 1);
  w1 = s - static_cast<float>(i0);
}

// One warp per pixel: bilinear (align_corners=False) logits from the 4 neighbouring patch rows, the unary
// U = -log(clip(softmax, 1e-5, 1)) and Q0 = softmax(-U).
__global__ void __launch_bounds__(kThreads)
crf_unary_kernel(CrfInput in, int frame0, int frames, int S, float* __restrict__ U, float* __restrict__ Q) {
  const int lane = threadIdx.x & 31;
  const long long n = static_cast<long long>(S) * S;
  const int K = in.classes;
  const float sc = static_cast<float>(in.grid) / static_cast<float>(S);
  for (long long i = blockIdx.x * static_cast<long long>(kWarps) + (threadIdx.x >> 5); i < frames * n;
       i += static_cast<long long>(gridDim.x) * kWarps) {
    const long long b = frame0 + i / n;
    const int p = static_cast<int>(i % n);
    int x0, x1, y0, y1;
    float wx, wy;
    ac_false(p % S, sc, in.grid, x0, x1, wx);
    ac_false(p / S, sc, in.grid, y0, y1, wy);
    const float* base = in.head + (b * in.npad + 1) * in.ld;
    const float* r00 = base + (static_cast<long long>(y0) * in.grid + x0) * in.ld;
    const float* r01 = base + (static_cast<long long>(y0) * in.grid + x1) * in.ld;
    const float* r10 = base + (static_cast<long long>(y1) * in.grid + x0) * in.ld;
    const float* r11 = base + (static_cast<long long>(y1) * in.grid + x1) * in.ld;
    auto blend = [&](int c) {
      return (1.f - wy) * ((1.f - wx) * __ldg(r00 + c) + wx * __ldg(r01 + c)) +
             wy * ((1.f - wx) * __ldg(r10 + c) + wx * __ldg(r11 + c));
    };
    float scale = in.logit_scale;
    if (in.code_dim > 0) {
      float ss = 0.f;
      for (int c = lane; c < in.code_dim; c += 32) {
        const float v = blend(in.code_col + c);
        ss += v * v;
      }
      scale = in.logit_scale / fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
    }
    float z[2];
    float mx = -INFINITY;
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const int k = lane + 32 * t;
      z[t] = k < K ? scale * blend(in.col0 + k) : -INFINITY;
      mx = fmaxf(mx, z[t]);
    }
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      z[t] = lane + 32 * t < K ? expf(z[t] - mx) : 0.f;
      sum += z[t];
    }
    sum = warp_sum(sum);
    float u[2];
    float umin = INFINITY;
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      u[t] = -logf(fminf(fmaxf(z[t] / sum, 1e-5f), 1.f));
      if (lane + 32 * t < K) umin = fminf(umin, u[t]);
    }
    umin = -warp_max(-umin);
    float qs = 0.f, q[2];
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      q[t] = lane + 32 * t < K ? expf(umin - u[t]) : 0.f;
      qs += q[t];
    }
    const float inv = 1.f / warp_sum(qs);
    const long long row = (i)*K;
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const int k = lane + 32 * t;
      if (k < K) {
        U[row + k] = u[t];
        Q[row + k] = q[t] * inv;
      }
    }
  }
}

// One warp per pixel: first maximum of Q -> int64 label; optional copy of Q.
__global__ void __launch_bounds__(kThreads)
crf_argmax_kernel(const float* __restrict__ Q, long long npix, int K, long long* __restrict__ labels, float* __restrict__ q_out) {
  const int lane = threadIdx.x & 31;
  for (long long p = blockIdx.x * static_cast<long long>(kWarps) + (threadIdx.x >> 5); p < npix;
       p += static_cast<long long>(gridDim.x) * kWarps) {
    float best = -INFINITY;
    int arg = 1 << 30;
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const int k = lane + 32 * t;
      if (k < K) {
        const float q = Q[p * K + k];
        if (q_out) q_out[p * K + k] = q;
        if (q > best) { best = q; arg = k; }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
      if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
    }
    if (lane == 0) labels[p] = arg;
  }
}

unsigned grid_for(long long work, int per_block) {
  const long long cap = static_cast<long long>(sm_count()) * 16;
  long long b = (work + per_block - 1) / per_block;
  return static_cast<unsigned>(std::max(1ll, std::min(b, cap)));
}

// Largest |key coordinate| a lattice can produce from features in [0, fmax_j]: |E[j]| <= sum_{i>=j} cf_i + j cf_{j-1},
// plus the remainder-0 rounding and the rank correction.
double key_bound(int d, const float* scale, const double* fmax) {
  double worst = 0.0;
  for (int j = 0; j <= d; ++j) {
    double hi = 0.0;
    for (int i = j; i < d; ++i) hi += fmax[i] * scale[i];
    const double lo = j > 0 ? j * fmax[j - 1] * scale[j - 1] : 0.0;
    worst = std::max(worst, std::max(hi, lo));
  }
  return worst + 2.0 * (d + 1) + 1.0;
}

}  // namespace

int crf_create(int size, int max_classes, int chunk, int iterations, wvn_crf** out) {
  WVN_REQUIRE(out, "wvn_crf_create: null argument");
  WVN_REQUIRE(size >= 2 && size <= 4096, "wvn_crf_create: size %d outside [2, 4096]", size);
  WVN_REQUIRE(max_classes >= 1 && max_classes <= 64, "wvn_crf_create: classes %d outside [1, 64]", max_classes);
  WVN_REQUIRE(chunk >= 1 && chunk <= 256, "wvn_crf_create: chunk %d outside [1, 256]", chunk);
  WVN_REQUIRE(iterations >= 0, "wvn_crf_create: negative iteration count");
  std::unique_ptr<wvn_crf> h(new wvn_crf());
  h->S = size; h->N = size * size; h->K = max_classes; h->chunk = chunk; h->iters = iterations;
  const long long npix = static_cast<long long>(chunk) * h->N;
  const int dims[2] = {2, 5};
  for (int l = 0; l < 2; ++l) {
    LatticeBufs& L = h->lat[l];
    L.d = dims[l];
    L.entries = npix * (L.d + 1);
    const double inv_std = static_cast<float>(sqrt(2.0 / 3.0) * (L.d + 1));
    for (int i = 0; i < L.d; ++i) L.scale[i] = static_cast<float>(1.0 / sqrt(static_cast<double>((i + 2) * (i + 1))) * inv_std);
    L.feat_div[0] = l == 0 ? 1.f : 67.f;
    L.feat_div[1] = 3.f;
    L.weight = l == 0 ? 3.f : 4.f;
    double fmax[5] = {(size - 1) / L.feat_div[0], (size - 1) / L.feat_div[0], 85.0, 85.0, 85.0};
    const int bits = key_bits(L.d);
    if (key_bound(L.d, L.scale, fmax) >= (1 << (bits - 1)) || (chunk - 1) >= (1ll << (64 - bits * L.d)))
      return set_error(WVN_ERR_INVALID, "wvn_crf_create: size %d / chunk %d overflow the %d-bit lattice keys", size,
                       chunk, bits);
  }
  const long long emax = h->lat[1].entries;
  if (emax >= (1ll << 31))
    return set_error(WVN_ERR_INVALID, "wvn_crf_create: chunk %d of %dx%d frames exceeds 2^31 lattice entries", chunk,
                     size, size);
  size_t sort_bytes = 0, scan_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, static_cast<unsigned long long*>(nullptr),
                                  static_cast<unsigned long long*>(nullptr), static_cast<int*>(nullptr),
                                  static_cast<int*>(nullptr), static_cast<int>(emax), 0, 64);
  cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, static_cast<int*>(nullptr), static_cast<int*>(nullptr),
                                static_cast<int>(emax));
  h->cub_bytes = std::max(sort_bytes, scan_bytes);
  WVN_PROPAGATE(carve(&h->arena, [&](Carver& a) {
    h->keys_in = a.take<unsigned long long>(emax);
    h->keys_out = a.take<unsigned long long>(emax);
    h->vals_in = a.take<int>(emax);
    h->scan = a.take<int>(emax);
    h->m = a.take<int>(2);
    h->va = a.take<float>(emax * h->K);
    h->vb = a.take<float>(emax * h->K);
    h->U = a.take<float>(npix * h->K);
    h->Q = a.take<float>(npix * h->K);
    h->acc = a.take<float>(npix * h->K);
    h->bgr = a.take<uchar4>(npix);
    for (int l = 0; l < 2; ++l) {
      LatticeBufs& L = h->lat[l];
      L.bary = a.take<float>(L.entries);
      L.offs = a.take<int>(L.entries);
      L.sorted = a.take<int>(L.entries);
      L.start = a.take<int>(L.entries + 1);
      L.ukeys = a.take<unsigned long long>(L.entries);
      L.nbr = a.take<int2>(L.entries * (L.d + 1));
      L.norm = a.take<float>(npix);
    }
    h->cub_tmp = a.take<char>(h->cub_bytes);
  }, "wvn_crf_create"));
  *out = h.release();
  return WVN_OK;
}

void crf_destroy(wvn_crf* h) { delete h; }

size_t crf_workspace_bytes(const wvn_crf* h) { return h ? h->arena.bytes : 0; }

namespace {

template <int D>
int filter_lattice(wvn_crf* h, int l, const float* in, const float* scale, int V, int mode, float* out, cudaStream_t s) {
  LatticeBufs& L = h->lat[l];
  const long long npix = static_cast<long long>(h->frames) * h->N;
  crf_splat_kernel<D><<<grid_for(L.entries, kWarps), kThreads, 0, s>>>(L, h->m + l, in, scale, V, h->va);
  WVN_CHECK_LAUNCH("crf_splat_kernel");
  float* src = h->va;
  float* dst = h->vb;
  for (int j = 0; j <= D; ++j) {
    crf_blur_kernel<<<grid_for(L.entries * V, kThreads), kThreads, 0, s>>>(L.nbr + j * L.entries, h->m + l, V, src, dst);
    WVN_CHECK_LAUNCH("crf_blur_kernel");
    std::swap(src, dst);
  }
  crf_slice_kernel<D><<<grid_for(npix, kWarps), kThreads, 0, s>>>(L, npix, src, V, mode, out, h->U, h->acc, h->Q);
  WVN_CHECK_LAUNCH("crf_slice_kernel");
  return WVN_OK;
}

int run_filter(wvn_crf* h, int l, const float* in, const float* scale, int V, int mode, float* out, cudaStream_t s) {
  return l == 0 ? filter_lattice<2>(h, 0, in, scale, V, mode, out, s) : filter_lattice<5>(h, 1, in, scale, V, mode, out, s);
}

template <int D>
int build_lattice(wvn_crf* h, int l, cudaStream_t s) {
  LatticeBufs& L = h->lat[l];
  const long long npix = static_cast<long long>(h->frames) * h->N;
  const long long n = npix * (D + 1);
  crf_elevate_kernel<D><<<grid_for(npix, kThreads), kThreads, 0, s>>>(L, h->S, h->frames, h->bgr, h->keys_in, h->vals_in);
  WVN_CHECK_LAUNCH("crf_elevate_kernel");
  int fbits = 0;
  while ((1 << fbits) < h->frames) ++fbits;
  size_t tmp = h->cub_bytes;
  WVN_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(h->cub_tmp, tmp, h->keys_in, h->keys_out, h->vals_in, h->scan,
                                                 static_cast<int>(n), 0, key_bits(D) * D + fbits, s));
  count_launch();
  // flags go to vals_in (free after the sort), the scan to L.sorted's slot is not free yet: use keys_in's storage
  int* flags = h->vals_in;
  int* vid = reinterpret_cast<int*>(h->keys_in);
  crf_flag_kernel<<<grid_for(n, kThreads), kThreads, 0, s>>>(h->keys_out, n, flags);
  WVN_CHECK_LAUNCH("crf_flag_kernel");
  tmp = h->cub_bytes;
  WVN_CHECK_CUDA(cub::DeviceScan::InclusiveSum(h->cub_tmp, tmp, flags, vid, static_cast<int>(n), s));
  count_launch();
  crf_vertex_kernel<<<grid_for(n, kThreads), kThreads, 0, s>>>(L, h->keys_out, h->scan, vid, n, h->m + l);
  WVN_CHECK_LAUNCH("crf_vertex_kernel");
  crf_neighbour_kernel<D><<<grid_for(L.entries, kThreads), kThreads, 0, s>>>(L, h->m + l);
  WVN_CHECK_LAUNCH("crf_neighbour_kernel");
  return filter_lattice<D>(h, l, nullptr, nullptr, 1, SLICE_NORM, nullptr, s);
}

int build_chunk(wvn_crf* h, const CrfInput& in, int frame0, int frames, cudaStream_t s) {
  WVN_REQUIRE(in.img, "wvn_crf: null image");
  WVN_REQUIRE(in.resized_h >= h->S && in.resized_w >= h->S, "wvn_crf: resized image %dx%d smaller than the crop %d",
              in.resized_h, in.resized_w, h->S);
  ImgGeom g;
  g.img = in.img; g.u8 = in.u8_hwc; g.in_h = in.in_h; g.in_w = in.in_w; g.S = h->S; g.frame0 = frame0;
  g.crop_top = static_cast<int>(lrintf((in.resized_h - h->S) / 2.0f));
  g.crop_left = static_cast<int>(lrintf((in.resized_w - h->S) / 2.0f));
  g.scale_y = static_cast<float>(in.in_h) / static_cast<float>(in.resized_h);
  g.scale_x = static_cast<float>(in.in_w) / static_cast<float>(in.resized_w);
  h->frames = frames;
  crf_image_kernel<<<grid_for(static_cast<long long>(frames) * h->N, kThreads), kThreads, 0, s>>>(g, frames, h->bgr);
  WVN_CHECK_LAUNCH("crf_image_kernel");
  WVN_PROPAGATE(build_lattice<2>(h, 0, s));
  return build_lattice<5>(h, 1, s);
}

}  // namespace

int crf_build(wvn_crf* h, const CrfInput& in, cudaStream_t s) {
  WVN_REQUIRE(h, "wvn_crf_build: null handle");
  WVN_REQUIRE(in.batch >= 1 && in.batch <= h->chunk, "wvn_crf_build: batch %d outside [1, chunk %d]", in.batch, h->chunk);
  return build_chunk(h, in, 0, in.batch, s);
}

int crf_filter(wvn_crf* h, int which, const float* values, int v, float* out, cudaStream_t s) {
  WVN_REQUIRE(h && values && out, "wvn_crf_filter: null argument");
  WVN_REQUIRE(which == 0 || which == 1, "wvn_crf_filter: lattice %d is not 0 (spatial) or 1 (bilateral)", which);
  WVN_REQUIRE(v >= 1 && v <= h->K, "wvn_crf_filter: %d values outside [1, %d]", v, h->K);
  WVN_REQUIRE(h->frames > 0, "wvn_crf_filter: no lattice was built");
  return run_filter(h, which, values, nullptr, v, SLICE_WRITE, out, s);
}

namespace {
__global__ void crf_counts_kernel(const int* __restrict__ start, const int* __restrict__ m_ptr, int* __restrict__ counts) {
  const int m = *m_ptr;
  for (int v = blockIdx.x * kThreads + threadIdx.x; v < m; v += gridDim.x * kThreads) counts[v] = start[v + 1] - start[v];
}
}  // namespace

int crf_export(wvn_crf* h, int which, unsigned long long* keys, int* counts, int* offsets, float* bary, int* m,
               cudaStream_t s) {
  WVN_REQUIRE(h && keys && counts && offsets && bary && m, "wvn_crf_export: null argument");
  WVN_REQUIRE(which == 0 || which == 1, "wvn_crf_export: lattice %d is not 0 or 1", which);
  const LatticeBufs& L = h->lat[which];
  const long long e = static_cast<long long>(h->frames) * h->N * (L.d + 1);
  WVN_CHECK_CUDA(cudaMemcpyAsync(keys, L.ukeys, 8 * e, cudaMemcpyDeviceToDevice, s));
  WVN_CHECK_CUDA(cudaMemcpyAsync(offsets, L.offs, 4 * e, cudaMemcpyDeviceToDevice, s));
  WVN_CHECK_CUDA(cudaMemcpyAsync(bary, L.bary, 4 * e, cudaMemcpyDeviceToDevice, s));
  WVN_CHECK_CUDA(cudaMemcpyAsync(m, h->m + which, 4, cudaMemcpyDeviceToDevice, s));
  crf_counts_kernel<<<grid_for(e, kThreads), kThreads, 0, s>>>(L.start, h->m + which, counts);
  WVN_CHECK_LAUNCH("crf_counts_kernel");
  return WVN_OK;
}

int crf_run(wvn_crf* h, const CrfInput& in, long long* labels, float* q_out, cudaStream_t s) {
  WVN_REQUIRE(h && in.head && labels, "wvn_crf_run: null argument");
  WVN_REQUIRE(in.batch >= 1, "wvn_crf_run: empty batch");
  WVN_REQUIRE(in.classes >= 1 && in.classes <= h->K, "wvn_crf_run: classes %d outside [1, %d]", in.classes, h->K);
  WVN_REQUIRE(in.grid >= 1 && in.npad >= 1 + in.grid * in.grid, "wvn_crf_run: bad token grid");
  WVN_REQUIRE(in.code_dim >= 0 && in.ld >= in.col0 + in.classes && in.ld >= in.code_col + in.code_dim,
              "wvn_crf_run: columns outside the row");
  const int K = in.classes;
  for (int b0 = 0; b0 < in.batch; b0 += h->chunk) {
    const int nf = std::min(h->chunk, in.batch - b0);
    WVN_PROPAGATE(build_chunk(h, in, b0, nf, s));
    const long long npix = static_cast<long long>(nf) * h->N;
    crf_unary_kernel<<<grid_for(npix, kWarps), kThreads, 0, s>>>(in, b0, nf, h->S, h->U, h->Q);
    WVN_CHECK_LAUNCH("crf_unary_kernel");
    for (int it = 0; it < h->iters; ++it) {
      WVN_PROPAGATE(run_filter(h, 0, h->Q, h->lat[0].norm, K, SLICE_ACC, h->acc, s));
      WVN_PROPAGATE(run_filter(h, 1, h->Q, h->lat[1].norm, K, SLICE_UPDATE, nullptr, s));
    }
    crf_argmax_kernel<<<grid_for(npix, kWarps), kThreads, 0, s>>>(
        h->Q, npix, K, labels + static_cast<long long>(b0) * h->N, q_out ? q_out + static_cast<long long>(b0) * h->N * K : nullptr);
    WVN_CHECK_LAUNCH("crf_argmax_kernel");
  }
  return WVN_OK;
}

}  // namespace wvn
