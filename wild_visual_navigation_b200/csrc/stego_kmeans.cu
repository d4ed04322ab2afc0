// wvn-b200: per-image k-means of the STEGO code (run_clustering=True, the reference's default for stego
// segmentation: feature_extractor.py:47-53 -> StegoInterface -> Stego.postprocess(image_clustering=True)).
//
// [EXTERNAL-RECALLED] The clustering itself lives in the un-vendored `stego` package; what the reference fixes is the
// call (n_image_clusters clusters per image over the 90-d code, stego_interface.py:43,91-100).  Restated here — and in
// oracle/stego_head.py:image_kmeans, which the tests hold this kernel to — as plain Lloyd iterations (Euclidean, fixed
// iteration count, deterministic evenly-spaced initial centroids, empty clusters keep their centroid) over the code at
// PATCH resolution, followed by `postprocess`'s order of operations for the prediction: the code is upsampled
// (bilinear, align_corners=False) and every pixel takes its nearest centroid.  The nearest-centroid score
// <x, c_k> - |c_k|^2 / 2 is affine in x, so it commutes with the interpolation: this kernel leaves the per-patch scores
// in the head buffer's cluster-logit columns and the existing upsample+argmax kernel (dense_kernels.cu) produces the
// pixel labels — the (H, W, 90) tensor is never formed.
//
// ONE launch runs all iterations for the whole batch: a TEAM of 8 CTAs owns a frame (8 x 392 of the 3136 patches at
// 448 px), so a batch of 32 frames fills the GPU instead of 32 SMs (16 teams = 128 of the H100's 132 SMs: two full
// rounds).  The team synchronises once per iteration through a per-frame arrival counter in global memory (release /
// acquire); the partial sums travel through global memory anyway.  Free CTAs rather than hardware thread-block
// clusters: a cluster has to sit inside one GPC, which leaves SMs unused.  CTAs are dispatched in block order, so a team
// split by the residency boundary only waits for earlier teams to retire (no circular wait); the spin is bounded and traps.
// The CTA's code rows are staged in
// shared memory ONCE (coalesced; the first version re-read them from L2 every pass with one row per lane — with the
// shared-memory carve-out at its maximum there is no L1 left, and every such request touches 32 sectors).
// Per iteration and CTA:
//   1. one thread = one patch: the 90-d code row sits in registers, the K centroids are read as float4 broadcasts from
//      shared memory; nearest centroid -> assign[] (shared)
//   2. one warp = one patch at a time (lane = channel): the row is added to a WARP-PRIVATE copy of the K x C sums — no
//      atomics (large clusters are hot spots for shared-memory atomics), deterministic
//   3. the warp copies are summed, the CTA's partial sums go to global memory; after one team barrier
//      (release / acquire) every CTA adds the team's partials in the same order and updates its own copy of the centroids.
#include "common.cuh"
#include "host_common.h"
#include "stego_kmeans.h"

namespace wvn {

namespace {

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr int kTeam = 8;       // CTAs per frame at large batches: 16 teams = 128 SMs, 32 frames = 2 full rounds
constexpr int kMaxTeam = 32;   // small batches (the one-camera deployment case) spread a frame over more CTAs

// CTAs per frame: as many as keep every team resident in ONE round (132 SMs, one CTA each), between kTeam and kMaxTeam.
inline int team_size(int batch) {
  const int fit = sm_count() / (batch > 0 ? batch : 1);
  return fit < kTeam ? kTeam : (fit > kMaxTeam ? kMaxTeam : fit);
}

// Arrive at the frame's counter and wait until `target` arrivals: release before, acquire after; bounded (traps after
// ~2 s instead of hanging the GPU if a team member never shows up).
__device__ __forceinline__ void team_barrier(unsigned int* counter, unsigned int target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1u);
    const long long t0 = clock64();
    unsigned int v;
    for (;;) {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
      if (v >= target) break;
      __nanosleep(64);
      if (clock64() - t0 > 4000000000ll) {
        printf("[wvn] stego_kmeans: team barrier timed out (block %d, %u of %u)\n", blockIdx.x, v, target);
        __trap();
      }
    }
  }
  __syncthreads();
}
constexpr int kMaxK = 64;
constexpr int kMaxC = 128;   // code_dim <= 128 (row registers: 128)

// CREG: code_dim rounded up (centroid rows and the per-thread code row are padded to it with zeros, so the score loop
// has no bounds checks); ROWS_SMEM: the CTA's code rows are staged in shared memory.  Shared-memory operands of the hot
// loops are addressed through explicit 32-bit shared addresses (lds128 / plain typed pointers that never mix with
// global ones): with a pointer that could be either space the compiler falls back to generic loads.
template <int CREG, bool ROWS_SMEM>
__global__ void __launch_bounds__(kThreads, 1)
stego_kmeans_kernel(float* __restrict__ rows, KmeansArgs a, float* __restrict__ partial) {
  extern __shared__ __align__(16) float ksm[];
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int K = a.k, C = a.code_dim, P = a.patches;
  constexpr int CP = CREG;                     // centroid row stride
  const int n_priv = a.n_priv;                 // warp-private sum copies that fit in shared memory
  float* cent = ksm;                           // [K][CP], padding columns zero
  float* half_norm = cent + K * CP;            // [K]
  float* cnt_priv = half_norm + kMaxK;         // [n_priv][K]
  float* sum_priv = cnt_priv + kWarps * kMaxK; // [n_priv][K][CP]
  float* rows_s = sum_priv + n_priv * K * CP;  // [per][C + 1] (odd row stride: one row per lane is conflict-free)
  __shared__ unsigned char assign[1024];       // per CTA: <= 1024 patches (8 CTAs per frame)

  const int T = a.team;                       // CTAs of this frame
  const uint32_t rank = blockIdx.x % T;
  const int frame = blockIdx.x / T;
  const int per = (P + T - 1) / T;
  const int p0 = rank * per, p1 = min(P, p0 + per);
  float* base = rows + (static_cast<long long>(frame) * a.npad + 1) * a.ld;  // row 0 of a frame is the CLS token
  auto code = [&](int p) { return base + static_cast<long long>(p) * a.ld + a.code_col; };
  float* part_frame = partial + static_cast<long long>(frame) * 2 * T * (K * CP + K);  // [2 buffers][T ranks][K*CP + K]
  const int RS = C + 1;
  const uint32_t cent_addr = smem_u32(cent);

  if (ROWS_SMEM) {
    for (int p = warp; p < p1 - p0; p += kWarps) {  // one warp per row: coalesced, no integer division
      const float* src = code(p0 + p);
      for (int c = lane; c < C; c += 32) rows_s[p * RS + c] = src[c];
    }
  }
  // deterministic init: K patches evenly spaced over the frame's token sequence (every CTA builds the same copy)
  for (int k = warp; k < K; k += kWarps) {
    const int p = static_cast<int>((static_cast<long long>(2 * k + 1) * P) / (2 * K));
    const float* src = code(p);
    for (int c = lane; c < CP; c += 32) cent[k * CP + c] = c < C ? src[c] : 0.f;
  }
  __syncthreads();

  for (int it = 0; it <= a.iters; ++it) {
    const bool last = it == a.iters;  // the last pass only writes the scores of the final centroids
    for (int k = warp; k < K; k += kWarps) {  // |c_k|^2 / 2: one warp per centroid
      float n2 = 0.f;
      for (int c = lane; c < C; c += 32) n2 = fmaf(cent[k * CP + c], cent[k * CP + c], n2);
      n2 = warp_sum(n2);
      if (lane == 0) half_norm[k] = 0.5f * n2;
    }
    {
      float4* z = reinterpret_cast<float4*>(sum_priv);
      for (int i = t; i < n_priv * K * CP / 4; i += kThreads) z[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int i = t; i < n_priv * K; i += kThreads) cnt_priv[i] = 0.f;
    }
    __syncthreads();
    // ---- 1. nearest centroid per patch (one thread = one patch, row in registers)
    for (int p = p0 + t; p < p1; p += kThreads) {
      float x[CREG];
      if (ROWS_SMEM) {
        const float* src = rows_s + (p - p0) * RS;
#pragma unroll
        for (int c = 0; c < CREG; ++c) x[c] = c < C ? src[c] : 0.f;
      } else {
        const float* src = code(p);
#pragma unroll
        for (int c = 0; c < CREG; ++c) x[c] = c < C ? src[c] : 0.f;
      }
      float best = -INFINITY;
      int arg = 0;
      for (int k = 0; k < K; k += 2) {  // two centroids per pass: 8 independent FMA chains hide the LDS / FMA latencies
        const bool two = k + 1 < K;
        const uint32_t ca = cent_addr + static_cast<uint32_t>(k) * (CP * 4);
        const uint32_t cb = two ? ca + CP * 4 : ca;
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f, u0 = 0.f, u1 = 0.f, u2 = 0.f, u3 = 0.f;
#pragma unroll
        for (int c4 = 0; c4 < CREG / 4; ++c4) {
          const uint4 cv = lds128(ca + 16 * c4);   // same address in every lane: a broadcast
          const uint4 dv = lds128(cb + 16 * c4);
          s0 = fmaf(x[4 * c4 + 0], __uint_as_float(cv.x), s0);
          s1 = fmaf(x[4 * c4 + 1], __uint_as_float(cv.y), s1);
          s2 = fmaf(x[4 * c4 + 2], __uint_as_float(cv.z), s2);
          s3 = fmaf(x[4 * c4 + 3], __uint_as_float(cv.w), s3);
          u0 = fmaf(x[4 * c4 + 0], __uint_as_float(dv.x), u0);
          u1 = fmaf(x[4 * c4 + 1], __uint_as_float(dv.y), u1);
          u2 = fmaf(x[4 * c4 + 2], __uint_as_float(dv.z), u2);
          u3 = fmaf(x[4 * c4 + 3], __uint_as_float(dv.w), u3);
        }
        const float sa = ((s0 + s1) + (s2 + s3)) - half_norm[k];
        if (last) code(p)[a.logit_col - a.code_col + k] = sa;
        if (sa > best) { best = sa; arg = k; }  // first maximum wins, like torch.argmax
        if (two) {
          const float sb = ((u0 + u1) + (u2 + u3)) - half_norm[k + 1];
          if (last) code(p)[a.logit_col - a.code_col + k + 1] = sb;
          if (sb > best) { best = sb; arg = k + 1; }
        }
      }
      assign[p - p0] = static_cast<unsigned char>(arg);
    }
    if (last) break;
    __syncthreads();
    // ---- 2. warp-private sums: warp w < n_priv adds the rows of patches p0 + w, p0 + w + n_priv, ...
    if (warp < n_priv) {
      float* sp = sum_priv + warp * K * CP;
      float* cp = cnt_priv + warp * K;
      // software-pipelined over patches: the next patch's row values are in registers before this patch's
      // read-modify-write of the sums starts (the RMW chain itself must stay in order: patches may share a cluster)
      int p = warp;
      float r0 = 0.f, r1 = 0.f, r2 = 0.f, r3 = 0.f;
      int kcur = 0;
      auto load_row = [&](int pp, float& a0, float& a1, float& a2, float& a3, int& kk) {
        kk = assign[pp];
        const float* row = ROWS_SMEM ? rows_s + pp * RS : code(p0 + pp);
        a0 = lane < C ? row[lane] : 0.f;
        a1 = lane + 32 < C ? row[lane + 32] : 0.f;
        a2 = lane + 64 < C ? row[lane + 64] : 0.f;
        a3 = lane + 96 < C ? row[lane + 96] : 0.f;
      };
      if (p < p1 - p0) load_row(p, r0, r1, r2, r3, kcur);
      while (p < p1 - p0) {
        const int pn = p + n_priv;
        float n0 = 0.f, n1 = 0.f, n2 = 0.f, n3 = 0.f;
        int knext = 0;
        if (pn < p1 - p0) load_row(pn, n0, n1, n2, n3, knext);
        float* dst = sp + kcur * CP;
        if (lane < C) dst[lane] += r0;
        if (lane + 32 < C) dst[lane + 32] += r1;
        if (lane + 64 < C) dst[lane + 64] += r2;
        if (lane + 96 < C) dst[lane + 96] += r3;
        if (lane == 0) cp[kcur] += 1.f;
        __syncwarp();
        r0 = n0; r1 = n1; r2 = n2; r3 = n3; kcur = knext; p = pn;
      }
    }
    __syncthreads();
    // ---- 3. CTA partial -> global; team barrier; every CTA sums the team's partials in rank order
    float* mine = part_frame + ((it & 1) * T + rank) * (K * CP + K);
    for (int i = t; i < K * CP + K; i += kThreads) {
      float sacc = 0.f;
      if (i < K * CP) {
        for (int w = 0; w < n_priv; ++w) sacc += sum_priv[w * K * CP + i];
      } else {
        for (int w = 0; w < n_priv; ++w) sacc += cnt_priv[w * K + (i - K * CP)];
      }
      mine[i] = sacc;
    }
    team_barrier(a.frame_bar + frame, static_cast<unsigned int>(T) * (it + 1));
    const float* all = part_frame + (it & 1) * T * (K * CP + K);
    for (int k = warp; k < K; k += kWarps) {  // one warp per centroid
      float n = 0.f;
      for (int r = 0; r < T; ++r) n += __ldcg(all + r * (K * CP + K) + K * CP + k);
      if (n > 0.f) {  // empty cluster: keep its centroid
        for (int c = lane; c < C; c += 32) {
          float sacc = 0.f;
          for (int r = 0; r < T; ++r) sacc += __ldcg(all + r * (K * CP + K) + k * CP + c);
          cent[k * CP + c] = sacc / n;
        }
      }
    }
    __syncthreads();
  }
  if (a.centroids_out && rank == 0) {
    __syncthreads();
    for (int i = t; i < K * C; i += kThreads) {
      const int k = i / C, c = i - k * C;
      a.centroids_out[(static_cast<long long>(frame) * K + k) * C + c] = cent[k * CP + c];
    }
  }
}

}  // namespace

size_t stego_kmeans_workspace_bytes(int batch, int k, int code_dim) {
  const int CP = code_dim <= 96 ? 96 : 128;
  return sizeof(float) * static_cast<size_t>(batch) * 2 * team_size(batch) * (static_cast<size_t>(k) * CP + k) +
         sizeof(unsigned int) * static_cast<size_t>(batch) + 16;
}

int stego_kmeans(float* rows, const KmeansArgs& a_in, float* workspace, cudaStream_t stream) {
  KmeansArgs a = a_in;
  WVN_REQUIRE(rows && workspace && a.batch > 0 && a.patches > 0, "kmeans: empty problem");
  WVN_REQUIRE(a.k > 0 && a.k <= kMaxK && a.code_dim > 0 && a.code_dim <= kMaxC, "kmeans: k=%d (<= %d), code_dim=%d (<= %d)",
              a.k, kMaxK, a.code_dim, kMaxC);
  a.team = team_size(a.batch);
  WVN_REQUIRE(a.patches >= a.k && a.patches <= a.team * 1024 && a.iters >= 0 && a.logit_col % 4 == 0 &&
                  a.logit_col + a.k <= a.ld && (a.logit_col >= a.code_col + a.code_dim || a.logit_col + a.k <= a.code_col),
              "kmeans: bad geometry (patches=%d) / column layout / iteration count", a.patches);
  const int CP = a.code_dim <= 96 ? 96 : 128;
  const int per = (a.patches + a.team - 1) / a.team;
  const size_t fixed = sizeof(float) * (static_cast<size_t>(a.k) * CP + kMaxK + kWarps * kMaxK);
  const size_t per_copy = sizeof(float) * static_cast<size_t>(a.k) * CP;
  const size_t rows_bytes = sizeof(float) * static_cast<size_t>(per) * (a.code_dim + 1);
  const size_t budget = 220 * 1024;
  // the CTA's rows live in shared memory when at least 4 private sum copies still fit next to them
  a.rows_in_smem = fixed + rows_bytes + 4 * per_copy <= budget ? 1 : 0;
  const size_t avail = budget - fixed - (a.rows_in_smem ? rows_bytes : 0);
  int n_priv = static_cast<int>(avail / per_copy);
  if (n_priv > kWarps) n_priv = kWarps;
  WVN_REQUIRE(n_priv >= 1, "kmeans: k * code_dim too large for shared memory");
  a.n_priv = n_priv;
  const size_t smem = fixed + per_copy * n_priv + (a.rows_in_smem ? rows_bytes : 0);
  auto kern = a.code_dim <= 96 ? (a.rows_in_smem ? stego_kmeans_kernel<96, true> : stego_kmeans_kernel<96, false>)
                               : (a.rows_in_smem ? stego_kmeans_kernel<128, true> : stego_kmeans_kernel<128, false>);
  WVN_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  // the per-frame arrival counters live behind the partial sums and start from zero
  const size_t part_floats = static_cast<size_t>(a.batch) * 2 * a.team * (static_cast<size_t>(a.k) * CP + a.k);
  a.frame_bar = reinterpret_cast<unsigned int*>(workspace + ((part_floats + 3) & ~static_cast<size_t>(3)));
  WVN_CHECK_CUDA(cudaMemsetAsync(a.frame_bar, 0, sizeof(unsigned int) * a.batch, stream));
  kern<<<a.batch * a.team, kThreads, smem, stream>>>(rows, a, workspace);
  WVN_CHECK_LAUNCH("stego_kmeans_kernel");
  return WVN_OK;
}

}  // namespace wvn
