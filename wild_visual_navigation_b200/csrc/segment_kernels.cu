// wvn-b200: per-segment reductions over a segmentation map (sm_90a, HBM/L2-bound integer work).
//
// Replaces three Python per-segment loops of the reference, each of which costs one host
// sync per segment:
//   FeatureExtractor.sparsify_features  (feature_extractor.py:389-396)  per-segment feature mean
//   SegmentExtractor.centers            (segment_extractor.py:70-92)    per-segment centroid (x=col, y=row)
//   SegmentExtractor.adjacency_list     (segment_extractor.py:40-67)    4-neighbour segment graph
//   FeatureExtractor.segment_stego      (feature_extractor.py:245-246)  relabel to 0..S-1
// and, the other way round, paints per-segment values back into per-pixel maps (segment_maps: the node's segment-wise
// mode, wvn_feature_extractor_node.py:323-338).
//
// The dense (B, D, H, H) feature tensor is never formed: the mean of bilinearly upsampled
// (align_corners=True) features over a segment is a linear function of the patch tokens,
//   feat[s] = (sum_p W[s,p] * tok[p]) / count[s],   W[s,p] = sum_{pixels in s} bilinear weight of patch p,
// so one pass over the pixels accumulates W (plus counts, coordinate sums and adjacency bits)
// and a small second kernel contracts W with the token grid.
#include <stdint.h>

#include <algorithm>

#include "common.cuh"
#include "host_common.h"
#include "segment_kernels.h"

namespace wvn {

namespace {

__device__ __forceinline__ void ac_true_coord(int dst, float scale, int in_size, int& i0, int& i1, float& w1) {
  const float s = dst * scale;
  i0 = min(static_cast<int>(s), in_size - 1);
  i1 = min(i0 + 1, in_size - 1);
  w1 = s - static_cast<float>(i0);
}

__global__ void __launch_bounds__(256)
segment_accumulate_kernel(const long long* __restrict__ seg, SegmentArgs a, unsigned long long* __restrict__ stats,
                          float* __restrict__ wseg, unsigned int* __restrict__ adj) {
  const long long total = static_cast<long long>(a.batch) * a.h * a.w;
  const int adj_words = (a.smax + 31) >> 5;
  const int P = a.grid_h * a.grid_w;
  for (long long p = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; p < total;
       p += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(p % a.w);
    const int y = static_cast<int>((p / a.w) % a.h);
    const long long b = p / (static_cast<long long>(a.w) * a.h);
    const long long s = seg[p];
    if (s < 0 || s >= a.smax) continue;
    unsigned long long* st = stats + (b * a.smax + s) * 3;
    atomicAdd(st + 0, 1ull);
    atomicAdd(st + 1, static_cast<unsigned long long>(x));
    atomicAdd(st + 2, static_cast<unsigned long long>(y));
    if (wseg != nullptr) {
      // dense features are (H, H): pixel (row=y, col=x) reads dense[:, y, x]; guard x < out size
      int x0, x1, y0, y1;
      float wx, wy;
      ac_true_coord(x, a.scale_x, a.grid_w, x0, x1, wx);
      ac_true_coord(y, a.scale_y, a.grid_h, y0, y1, wy);
      float* wrow = wseg + (b * a.smax + s) * P;
      atomicAdd(wrow + y0 * a.grid_w + x0, (1.f - wy) * (1.f - wx));
      atomicAdd(wrow + y0 * a.grid_w + x1, (1.f - wy) * wx);
      atomicAdd(wrow + y1 * a.grid_w + x0, wy * (1.f - wx));
      atomicAdd(wrow + y1 * a.grid_w + x1, wy * wx);
    }
    if (adj != nullptr) {
      // directed pair (left/top id -> right/bottom id), as the reference's shifted filters pair them
      if (x + 1 < a.w) {
        const long long r = seg[p + 1];
        if (r != s && r >= 0 && r < a.smax)
          atomicOr(adj + (b * a.smax + r) * adj_words + (s >> 5), 1u << (s & 31));
      }
      if (y + 1 < a.h) {
        const long long r = seg[p + a.w];
        if (r != s && r >= 0 && r < a.smax)
          atomicOr(adj + (b * a.smax + r) * adj_words + (s >> 5), 1u << (s & 31));
      }
    }
  }
}

// ---- privatised accumulation -----------------------------------------------------------------
// One block = one TILE_H x TILE_W pixel tile of one frame.  The tile touches only a small window
// of the token grid, so the bilinear weights W[s, token], the per-segment statistics and the
// adjacency bits are first accumulated in shared memory (cheap, contention-free across SMs) and
// only the non-zero entries are flushed with global atomics.  Used when smax <= kPrivMaxSeg.
constexpr int kTileH = 32, kTileW = 64, kPrivMaxSeg = 128;
constexpr int kRun = 8;  // consecutive pixels of one row per thread: 256 threads = 32 rows x 8 runs

// Each thread walks kRun consecutive pixels of one row and keeps the contribution of the current
// (segment, token cell) run in registers; shared-memory atomics are issued once per run instead of seven per
// pixel (neighbouring pixels almost always share segment and cell, so the per-pixel version serialised on
// same-address atomics).
__global__ void __launch_bounds__(256)
segment_accumulate_tiled_kernel(const long long* __restrict__ seg, SegmentArgs a, int win_h, int win_w,
                                unsigned long long* __restrict__ stats, float* __restrict__ wseg,
                                unsigned int* __restrict__ adj) {
  extern __shared__ float sm_w[];                               // [smax][win_h][win_w]
  int* sm_stats = reinterpret_cast<int*>(sm_w + a.smax * win_h * win_w);  // [smax][3]
  unsigned int* sm_adj = reinterpret_cast<unsigned int*>(sm_stats + a.smax * 3);  // [smax][words]
  const int adj_words = (a.smax + 31) >> 5;
  const int P = a.grid_h * a.grid_w;
  const long long b = blockIdx.z;
  const int px0 = blockIdx.x * kTileW, py0 = blockIdx.y * kTileH;
  const int n_w = a.smax * win_h * win_w;
  for (int i = threadIdx.x; i < n_w; i += blockDim.x) sm_w[i] = 0.f;
  for (int i = threadIdx.x; i < a.smax * 3; i += blockDim.x) sm_stats[i] = 0;
  for (int i = threadIdx.x; i < a.smax * adj_words; i += blockDim.x) sm_adj[i] = 0u;
  // token window origin of this tile
  int wy0, wx0, t1;
  float tw;
  ac_true_coord(py0, a.scale_y, a.grid_h, wy0, t1, tw);
  ac_true_coord(px0, a.scale_x, a.grid_w, wx0, t1, tw);
  __syncthreads();
  const long long* segb = seg + b * a.h * a.w;
  const int y = py0 + static_cast<int>(threadIdx.x) / (kTileW / kRun);
  const int xs = px0 + (static_cast<int>(threadIdx.x) % (kTileW / kRun)) * kRun;
  if (y < a.h && xs < a.w) {
    const int n = min(kRun, a.w - xs);
    long long ids[kRun + 1], below[kRun];
    const long long* row = segb + static_cast<long long>(y) * a.w + xs;
#pragma unroll
    for (int i = 0; i <= kRun; ++i) ids[i] = (i < n || (i == n && xs + i < a.w)) ? row[i] : -1;  // ids[n] = right neighbour
#pragma unroll
    for (int i = 0; i < kRun; ++i) below[i] = (adj != nullptr && i < n && y + 1 < a.h) ? row[a.w + i] : -1;
    int y0, y1;
    float wy;
    ac_true_coord(y, a.scale_y, a.grid_h, y0, y1, wy);
    long long cur_s = -1;
    int cur_x0 = -1, cur_x1 = -1, cnt = 0, sumx = 0;
    float s_l = 0.f, s_r = 0.f;  // sums of (1 - wx) and wx over the run
    auto flush = [&]() {
      if (cur_s < 0) return;
      atomicAdd(&sm_stats[cur_s * 3 + 0], cnt);
      atomicAdd(&sm_stats[cur_s * 3 + 1], sumx);
      atomicAdd(&sm_stats[cur_s * 3 + 2], cnt * y);
      if (wseg != nullptr) {
        float* w = sm_w + cur_s * win_h * win_w;
        atomicAdd(w + (y0 - wy0) * win_w + (cur_x0 - wx0), (1.f - wy) * s_l);
        atomicAdd(w + (y0 - wy0) * win_w + (cur_x1 - wx0), (1.f - wy) * s_r);
        atomicAdd(w + (y1 - wy0) * win_w + (cur_x0 - wx0), wy * s_l);
        atomicAdd(w + (y1 - wy0) * win_w + (cur_x1 - wx0), wy * s_r);
      }
    };
#pragma unroll
    for (int i = 0; i < kRun; ++i) {
      if (i >= n) break;
      const long long sid = ids[i];
      if (sid < 0 || sid >= a.smax) { flush(); cur_s = -1; continue; }
      const int x = xs + i;
      int x0, x1;
      float wx;
      ac_true_coord(x, a.scale_x, a.grid_w, x0, x1, wx);
      if (sid != cur_s || x0 != cur_x0) {
        flush();
        cur_s = sid; cur_x0 = x0; cur_x1 = x1; cnt = 0; sumx = 0; s_l = 0.f; s_r = 0.f;
      }
      ++cnt; sumx += x; s_l += 1.f - wx; s_r += wx;
      if (adj != nullptr) {
        const long long r = ids[i + 1];
        if (r != sid && r >= 0 && r < a.smax) atomicOr(&sm_adj[r * adj_words + (sid >> 5)], 1u << (sid & 31));
        const long long d = below[i];
        if (d != sid && d >= 0 && d < a.smax) atomicOr(&sm_adj[d * adj_words + (sid >> 5)], 1u << (sid & 31));
      }
    }
    flush();
  }
  __syncthreads();
  for (int i = threadIdx.x; i < a.smax; i += blockDim.x) {
    if (sm_stats[i * 3] != 0) {
      unsigned long long* st = stats + (b * a.smax + i) * 3;
      atomicAdd(st + 0, static_cast<unsigned long long>(sm_stats[i * 3 + 0]));
      atomicAdd(st + 1, static_cast<unsigned long long>(sm_stats[i * 3 + 1]));
      atomicAdd(st + 2, static_cast<unsigned long long>(sm_stats[i * 3 + 2]));
    }
  }
  if (wseg != nullptr) {
    for (int i = threadIdx.x; i < n_w; i += blockDim.x) {
      const float v = sm_w[i];
      if (v != 0.f) {
        const int s = i / (win_h * win_w), r = (i / win_w) % win_h, c = i % win_w;
        const int ty = wy0 + r, tx = wx0 + c;
        if (ty < a.grid_h && tx < a.grid_w) atomicAdd(wseg + (b * a.smax + s) * P + ty * a.grid_w + tx, v);
      }
    }
  }
  if (adj != nullptr) {
    for (int i = threadIdx.x; i < a.smax * adj_words; i += blockDim.x)
      if (sm_adj[i] != 0u) atomicOr(adj + b * a.smax * adj_words + i, sm_adj[i]);
  }
}

// feat_sum[b][s][d] += sum_p W[b][s][p] * tok[b][p][d]   (small dense GEMM; W is segments x tokens).
// The token matrix (154 MB for 32 frames) is read exactly once, with 16-byte loads: CTA = (frame, 32-segment block,
// token range); per 32-token step the W tile [32 seg][32 tok] and the token tile [32 tok][dim] are staged in shared
// memory; warp w owns segments 4w..4w+3, lane l owns float4 columns l, l+32, l+64 (dim <= 384) — 48 accumulators,
// 3 + 4 shared loads per 48 FMAs; wider features (ViT-B: 768) take one CTA column block of 384 each (blockIdx.x).
// Partial sums are flushed with vector atomics (ksplit CTAs per output block).
constexpr int kPoolTok = 32;      // tokens per step
constexpr int kPoolMaxV4 = 3;     // float4 column groups per lane: dim <= 384

__global__ void __launch_bounds__(256)
segment_pool_gemm_kernel(const float* __restrict__ wseg, const float* __restrict__ tok, float* __restrict__ feat,
                         SegmentArgs a, int ksplit) {
  extern __shared__ float4 pool_sm[];                       // [kPoolTok][dim/4] token tile, then [32][kPoolTok+1] W tile
  const int row_v4 = a.dim / 4;                              // float4 per token row
  const int c_base = blockIdx.x * 32 * kPoolMaxV4;           // first float4 column of this CTA's block
  const int dv4 = min(32 * kPoolMaxV4, row_v4 - c_base);     // float4 columns handled here
  float4* Ts = pool_sm;
  float* Ws = reinterpret_cast<float*>(pool_sm + kPoolTok * 32 * kPoolMaxV4);
  const int P = a.grid_h * a.grid_w;
  const long long b = blockIdx.z / ksplit;
  const int split = blockIdx.z % ksplit;
  const int kper = ((P + ksplit - 1) / ksplit + kPoolTok - 1) / kPoolTok * kPoolTok;
  const int k_beg = split * kper, k_end = min(P, k_beg + kper);
  const int s0 = blockIdx.y * 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float4 acc[4][kPoolMaxV4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < kPoolMaxV4; ++j) acc[i][j] = make_float4(0.f, 0.f, 0.f, 0.f);
  const float* wb = wseg + (b * a.smax) * P;
  const float4* tb = reinterpret_cast<const float4*>(tok + b * P * a.dim);
  for (int k0 = k_beg; k0 < k_end; k0 += kPoolTok) {
    for (int i = threadIdx.x; i < 32 * kPoolTok; i += 256) {
      const int r = i / kPoolTok, k = i % kPoolTok;
      Ws[r * (kPoolTok + 1) + k] =
          (s0 + r < a.smax && k0 + k < k_end) ? __ldg(wb + static_cast<long long>(s0 + r) * P + k0 + k) : 0.f;
    }
    for (int i = threadIdx.x; i < kPoolTok * dv4; i += 256) {
      const int k = i / dv4, c = i - k * dv4;
      Ts[i] = (k0 + k < k_end) ? __ldg(tb + static_cast<long long>(k0 + k) * row_v4 + c_base + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();
#pragma unroll 4
    for (int k = 0; k < kPoolTok; ++k) {
      float w[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) w[i] = Ws[(warp * 4 + i) * (kPoolTok + 1) + k];
      if (w[0] == 0.f && w[1] == 0.f && w[2] == 0.f && w[3] == 0.f) continue;  // W is sparse: most tokens touch few segments
#pragma unroll
      for (int j = 0; j < kPoolMaxV4; ++j) {
        const int c = lane + 32 * j;
        if (c < dv4) {
          const float4 t = Ts[k * dv4 + c];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            acc[i][j].x = fmaf(w[i], t.x, acc[i][j].x);
            acc[i][j].y = fmaf(w[i], t.y, acc[i][j].y);
            acc[i][j].z = fmaf(w[i], t.z, acc[i][j].z);
            acc[i][j].w = fmaf(w[i], t.w, acc[i][j].w);
          }
        }
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int sidx = s0 + warp * 4 + i;
    if (sidx >= a.smax) continue;
    float* dst = feat + (b * a.smax + sidx) * a.dim;
#pragma unroll
    for (int j = 0; j < kPoolMaxV4; ++j) {
      const int c = lane + 32 * j;
      if (c < dv4 && (acc[i][j].x != 0.f || acc[i][j].y != 0.f || acc[i][j].z != 0.f || acc[i][j].w != 0.f))
        asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + 4 * (c_base + c)), "f"(acc[i][j].x), "f"(acc[i][j].y),
                     "f"(acc[i][j].z), "f"(acc[i][j].w)
                     : "memory");
    }
  }
}

// Generic fallback of the pooling GEMM for feature widths that are not a multiple of 4 (the 90-d STEGO code):
// scalar loads, 32 x 64 output block per CTA.
// grid (ceil(dim/64), ceil(smax/32), B * ksplit); 256 threads: thread -> column tx, 8 rows.
__global__ void __launch_bounds__(256)
segment_pool_gemm_scalar_kernel(const float* __restrict__ wseg, const float* __restrict__ tok, float* __restrict__ feat,
                         SegmentArgs a, int ksplit) {
  __shared__ float Ws[32][33];
  __shared__ float Ts[32][64];
  const int P = a.grid_h * a.grid_w;
  const long long b = blockIdx.z / ksplit;
  const int split = blockIdx.z % ksplit;
  const int kper = ((P + ksplit - 1) / ksplit + 31) / 32 * 32;
  const int k_beg = split * kper, k_end = min(P, k_beg + kper);
  const int c0 = blockIdx.x * 64, s0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 63, ry = threadIdx.x >> 6;  // rows ry*8 .. ry*8+7
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  const float* wb = wseg + (b * a.smax) * P;
  const float* tb = tok + b * P * a.dim;
  for (int k0 = k_beg; k0 < k_end; k0 += 32) {
    for (int i = threadIdx.x; i < 32 * 32; i += 256) {
      const int r = i >> 5, k = i & 31;
      Ws[r][k] = (s0 + r < a.smax && k0 + k < k_end) ? wb[static_cast<long long>(s0 + r) * P + k0 + k] : 0.f;
    }
    for (int i = threadIdx.x; i < 32 * 64; i += 256) {
      const int k = i >> 6, c = i & 63;
      Ts[k][c] = (k0 + k < k_end && c0 + c < a.dim) ? tb[static_cast<long long>(k0 + k) * a.dim + c0 + c] : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int k = 0; k < 32; ++k) {
      const float t = Ts[k][tx];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(Ws[ry * 8 + i][k], t, acc[i]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int s = s0 + ry * 8 + i;
    if (s < a.smax && c0 + tx < a.dim && acc[i] != 0.f) atomicAdd(&feat[(b * a.smax + s) * a.dim + c0 + tx], acc[i]);
  }
}

// feat = feat_sum / count; centers = (mean col, mean row).  Empty segment -> NaN, like torch's mean of empty.
__global__ void __launch_bounds__(256)
segment_finalize_kernel(const unsigned long long* __restrict__ stats, float* __restrict__ feat,
                        float* __restrict__ centers, SegmentArgs a) {
  const long long n_seg = static_cast<long long>(a.batch) * a.smax;
  const long long total = feat ? n_seg * a.dim : n_seg;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long sidx = feat ? i / a.dim : i;
    const unsigned long long* st = stats + sidx * 3;
    if (feat) feat[i] = feat[i] / static_cast<float>(st[0]);
    if (centers && (!feat || i % a.dim == 0)) {
      centers[sidx * 2 + 0] = static_cast<float>(static_cast<double>(st[1]) / static_cast<double>(st[0]));
      centers[sidx * 2 + 1] = static_cast<float>(static_cast<double>(st[2]) / static_cast<double>(st[0]));
    }
  }
}

// One block per frame: walk the adjacency bitset in (right, left) order — the order
// torch.unique gives the reference's float64 keys left + right*div — and emit int64 pairs.
__global__ void __launch_bounds__(1024)
adjacency_emit_kernel(const unsigned int* __restrict__ adj, long long* __restrict__ edges, int* __restrict__ n_edges,
                      int smax, int max_edges) {
  __shared__ int row_off[1025];
  const long long b = blockIdx.x;
  const int adj_words = (smax + 31) >> 5;
  const unsigned int* ab = adj + b * smax * adj_words;
  const int r = threadIdx.x;
  int cnt = 0;
  if (r < smax)
    for (int wd = 0; wd < adj_words; ++wd) cnt += __popc(ab[r * adj_words + wd]);
  row_off[r + 1] = (r < smax) ? cnt : 0;
  if (r == 0) row_off[0] = 0;
  __syncthreads();
  if (r == 0)
    for (int i = 1; i <= 1024; ++i) row_off[i] += row_off[i - 1];
  __syncthreads();
  // the count is clamped to the caller's capacity; a negative value (-(true count)) flags the overflow
  if (r == 0) n_edges[b] = row_off[1024] <= max_edges ? row_off[1024] : -row_off[1024];
  if (r < smax) {
    int o = row_off[r];
    long long* eb = edges + b * max_edges * 2;
    for (int wd = 0; wd < adj_words; ++wd) {
      unsigned int bits = ab[r * adj_words + wd];
      while (bits) {
        const int l = __ffs(bits) - 1;
        bits &= bits - 1;
        if (o < max_edges) {
          eb[2 * o + 0] = wd * 32 + l;  // le_idx (left / top segment)
          eb[2 * o + 1] = r;            // ri_idx (right / bottom segment)
        }
        ++o;
      }
    }
  }
}

// ---- relabel: compact the set of labels present in a frame to 0..S-1 (sorted order)
// grid = (slices per frame, batch): the labels a block meets are collected in a shared-memory flag array first — letting
// every pixel store its flag to global memory would make millions of stores hit a few hundred addresses
__global__ void __launch_bounds__(256)
label_presence_kernel(const long long* __restrict__ seg, int* __restrict__ present, long long pix_per_frame, int num_labels) {
  extern __shared__ int flags[];
  for (int i = threadIdx.x; i < num_labels; i += blockDim.x) flags[i] = 0;
  __syncthreads();
  const long long per = (pix_per_frame + gridDim.x - 1) / gridDim.x;
  const long long p0 = blockIdx.x * per, p1 = min(pix_per_frame, p0 + per);
  const long long* fr = seg + blockIdx.y * pix_per_frame;
  for (long long p = p0 + threadIdx.x; p < p1; p += blockDim.x) {
    const long long v = fr[p];
    if (v >= 0 && v < num_labels && flags[v] == 0) flags[v] = 1;   // benign race: every writer stores 1
  }
  __syncthreads();
  for (int i = threadIdx.x; i < num_labels; i += blockDim.x)
    if (flags[i]) present[static_cast<long long>(blockIdx.y) * num_labels + i] = 1;
}

__global__ void label_scan_kernel(int* __restrict__ present, int* __restrict__ counts, int num_labels) {
  // one thread per frame; num_labels is tiny (<= 1024).  present[] becomes the remap table.
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= gridDim.x * blockDim.x) return;
  int* pr = present + static_cast<long long>(b) * num_labels;
  int run = 0;
  for (int i = 0; i < num_labels; ++i) {
    const int has = pr[i];
    pr[i] = has ? run : -1;
    run += has;
  }
  counts[b] = run;
}

__global__ void __launch_bounds__(256)
label_apply_kernel(long long* __restrict__ seg, const int* __restrict__ remap, int batch, long long pix_per_frame,
                   int num_labels) {
  const long long total = batch * pix_per_frame;
  for (long long p = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; p < total;
       p += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long v = seg[p];
    if (v >= 0 && v < num_labels) seg[p] = remap[(p / pix_per_frame) * num_labels + v];
  }
}

// ---------------------------------------------------------------------------------------------
// Supervision label pooling (MissionNode.update_supervision_signal, nodes.py:400-440): the reference expands
// the (H, W) signal against an (H, W, S) one-hot of the segment map (20-200 MB) to average it per segment;
// here each block privatises (sum, count) per segment in shared memory and flushes with two atomics per
// touched segment.  signal = nanmean over the mask's channels; NaN (no channel labelled) pixels are skipped.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
supervision_pool_kernel(const long long* __restrict__ seg, const float* __restrict__ mask, int channels,
                        long long pix, int smax, float* __restrict__ sum, float* __restrict__ cnt) {
  extern __shared__ float sh[];  // [smax] sums | [smax] counts
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < 2 * smax; i += blockDim.x) sh[i] = 0.f;
  __syncthreads();
  const long long* sg = seg + b * pix;
  const float* mk = mask + static_cast<long long>(b) * channels * pix;
  for (long long p = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; p < pix;
       p += static_cast<long long>(gridDim.x) * blockDim.x) {
    float s = 0.f;
    int n = 0;
    for (int c = 0; c < channels; ++c) {
      const float v = __ldg(mk + c * pix + p);
      if (v == v) { s += v; ++n; }
    }
    const long long id = sg[p];
    if (n > 0 && id >= 0 && id < smax) {
      atomicAdd(&sh[id], s / static_cast<float>(n));
      atomicAdd(&sh[smax + id], 1.f);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < smax; i += blockDim.x) {
    if (sh[smax + i] > 0.f) {
      atomicAdd(&sum[b * smax + i], sh[i]);
      atomicAdd(&cnt[b * smax + i], sh[smax + i]);
    }
  }
}

__global__ void supervision_finalize_kernel(float* __restrict__ y, const float* __restrict__ cnt,
                                            unsigned char* __restrict__ valid, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = cnt[i] > 0.f ? y[i] / cnt[i] : 0.f;  // 0 / 0 -> nan -> nan_to_num(0) in the reference
  y[i] = v;
  valid[i] = v > 0.f ? 1 : 0;
}

}  // namespace

int segment_accumulate(const long long* seg, const SegmentArgs& a, unsigned long long* stats, float* wseg,
                       unsigned int* adj, cudaStream_t stream) {
  WVN_REQUIRE(a.batch > 0 && a.h > 0 && a.w > 0 && a.smax > 0 && a.smax <= 1024, "segment: bad geometry (smax=%d)",
              a.smax);
  const long long P = static_cast<long long>(a.grid_h) * a.grid_w;
  WVN_CHECK_CUDA(cudaMemsetAsync(stats, 0, sizeof(unsigned long long) * 3 * a.batch * a.smax, stream));
  if (wseg) WVN_CHECK_CUDA(cudaMemsetAsync(wseg, 0, sizeof(float) * a.batch * a.smax * P, stream));
  if (adj) WVN_CHECK_CUDA(cudaMemsetAsync(adj, 0, sizeof(unsigned int) * a.batch * a.smax * ((a.smax + 31) >> 5), stream));
  if (a.smax <= kPrivMaxSeg) {
    const int win_h = static_cast<int>((kTileH - 1) * a.scale_y) + 3;
    const int win_w = static_cast<int>((kTileW - 1) * a.scale_x) + 3;
    const size_t smem = sizeof(float) * a.smax * win_h * win_w + sizeof(int) * a.smax * 3 +
                        sizeof(unsigned int) * a.smax * ((a.smax + 31) >> 5);
    if (smem <= 160 * 1024) {
      static size_t attr_bytes = 0;
      if (smem > 48 * 1024 && smem > attr_bytes) {
        WVN_CHECK_CUDA(cudaFuncSetAttribute(segment_accumulate_tiled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            static_cast<int>(smem)));
        attr_bytes = smem;
      }
      dim3 grid((a.w + kTileW - 1) / kTileW, (a.h + kTileH - 1) / kTileH, a.batch);
      segment_accumulate_tiled_kernel<<<grid, 256, smem, stream>>>(seg, a, win_h, win_w, stats, wseg, adj);
      WVN_CHECK_LAUNCH("segment_accumulate_tiled_kernel");
      return WVN_OK;
    }
  }
  const long long total = static_cast<long long>(a.batch) * a.h * a.w;
  long long blocks = (total + 255) / 256;
  const long long max_blocks = static_cast<long long>(sm_count()) * 16;
  if (blocks > max_blocks) blocks = max_blocks;
  segment_accumulate_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(seg, a, stats, wseg, adj);
  WVN_CHECK_LAUNCH("segment_accumulate_kernel");
  return WVN_OK;
}

int segment_pool(const float* wseg, const float* tokens, const unsigned long long* stats, float* feat, float* centers,
                 const SegmentArgs& a, cudaStream_t stream) {
  if (feat) {
    const int P = a.grid_h * a.grid_w;
    WVN_CHECK_CUDA(cudaMemsetAsync(feat, 0, sizeof(float) * a.batch * a.smax * a.dim, stream));
    int ksplit = (P + 447) / 448;
    if (ksplit < 1) ksplit = 1;
    if (a.dim % 4 == 0) {
      // 128 tokens per CTA: ~800 CTAs at 32 frames, 4 resident per SM, so one CTA's (unpipelined) tile load overlaps
      // the others' FMAs; the extra partial sums are cheap vector atomics
      ksplit = (P + 127) / 128;
      const int col_blocks = (a.dim / 4 + 32 * kPoolMaxV4 - 1) / (32 * kPoolMaxV4);
      dim3 grid(col_blocks, (a.smax + 31) / 32, a.batch * ksplit);
      const size_t smem = (static_cast<size_t>(kPoolTok) * 32 * kPoolMaxV4 * 4 + 32 * (kPoolTok + 1)) * sizeof(float);
      static bool attr_set = false;
      if (!attr_set) {
        WVN_CHECK_CUDA(cudaFuncSetAttribute(segment_pool_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        attr_set = true;
      }
      segment_pool_gemm_kernel<<<grid, 256, smem, stream>>>(wseg, tokens, feat, a, ksplit);
    } else {
      dim3 grid((a.dim + 63) / 64, (a.smax + 31) / 32, a.batch * ksplit);
      segment_pool_gemm_scalar_kernel<<<grid, 256, 0, stream>>>(wseg, tokens, feat, a, ksplit);
    }
    WVN_CHECK_LAUNCH("segment_pool_gemm_kernel");
  }
  if (feat || centers) {
    const long long total = static_cast<long long>(a.batch) * a.smax * (feat ? a.dim : 1);
    int blocks = static_cast<int>(std::min<long long>((total + 255) / 256, static_cast<long long>(sm_count()) * 8));
    segment_finalize_kernel<<<blocks, 256, 0, stream>>>(stats, feat, centers, a);
    WVN_CHECK_LAUNCH("segment_finalize_kernel");
  }
  return WVN_OK;
}

int adjacency_emit(const unsigned int* adj, long long* edges, int* n_edges, int batch, int smax, int max_edges,
                   cudaStream_t stream) {
  WVN_REQUIRE(smax <= 1024, "adjacency_emit: smax %d > 1024", smax);
  adjacency_emit_kernel<<<batch, 1024, 0, stream>>>(adj, edges, n_edges, smax, max_edges);
  WVN_CHECK_LAUNCH("adjacency_emit_kernel");
  return WVN_OK;
}

int relabel_compact(long long* seg, int* scratch, int* counts, int batch, long long pix_per_frame, int num_labels,
                    cudaStream_t stream) {
  WVN_REQUIRE(num_labels > 0 && num_labels <= 1024, "relabel: num_labels %d unsupported", num_labels);
  WVN_CHECK_CUDA(cudaMemsetAsync(scratch, 0, sizeof(int) * batch * num_labels, stream));
  const long long total = batch * pix_per_frame;
  long long blocks = (total + 255) / 256;
  const long long max_blocks = static_cast<long long>(sm_count()) * 16;
  if (blocks > max_blocks) blocks = max_blocks;
  const int slices = static_cast<int>(std::min<long long>((pix_per_frame + 4095) / 4096, 32));
  label_presence_kernel<<<dim3(slices, batch), 256, sizeof(int) * num_labels, stream>>>(seg, scratch, pix_per_frame, num_labels);
  WVN_CHECK_LAUNCH("label_presence_kernel");
  label_scan_kernel<<<batch, 1, 0, stream>>>(scratch, counts, num_labels);
  WVN_CHECK_LAUNCH("label_scan_kernel");
  label_apply_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(seg, scratch, batch, pix_per_frame, num_labels);
  WVN_CHECK_LAUNCH("label_apply_kernel");
  return WVN_OK;
}

int supervision_pool(const long long* seg, const float* mask, int batch, int channels, int h, int w, int smax, float* y,
                     unsigned char* y_valid, float* cnt_ws, cudaStream_t stream) {
  WVN_REQUIRE(batch > 0 && channels > 0 && h > 0 && w > 0 && smax > 0 && smax <= 4096,
              "supervision_pool: bad geometry (batch=%d channels=%d %dx%d smax=%d)", batch, channels, h, w, smax);
  const long long pix = static_cast<long long>(h) * w;
  WVN_CHECK_CUDA(cudaMemsetAsync(y, 0, sizeof(float) * batch * smax, stream));
  WVN_CHECK_CUDA(cudaMemsetAsync(cnt_ws, 0, sizeof(float) * batch * smax, stream));
  const int per_frame = static_cast<int>(std::min<long long>((pix + 256 * 16 - 1) / (256 * 16), 64));
  supervision_pool_kernel<<<dim3(per_frame, batch), 256, 2 * smax * sizeof(float), stream>>>(seg, mask, channels, pix, smax,
                                                                                            y, cnt_ws);
  WVN_CHECK_LAUNCH("supervision_pool_kernel");
  const int n = batch * smax;
  supervision_finalize_kernel<<<(n + 255) / 256, 256, 0, stream>>>(y, cnt_ws, y_valid, n);
  WVN_CHECK_LAUNCH("supervision_finalize_kernel");
  return WVN_OK;
}

// ------------------------------------------------------------------------------------------------ segment-wise maps
namespace {

constexpr int kMapThreads = 256;

// v[id] for a live id, NaN otherwise.  The unsigned compare sends negative ids to NaN as well.
template <typename Id>
__device__ __forceinline__ float row_value(const float* __restrict__ v, Id id, unsigned live) {
  return static_cast<unsigned long long>(static_cast<long long>(id)) < live ? v[id] : __int_as_float(0x7fc00000);
}

// One (frame, pixel block) per CTA.  VEC: 4 pixels per thread, one 16-byte load of int32 ids or two of int64 ids, and
// one float4 store per map; needs hw % 4 == 0 and 16-byte aligned pointers.  The per-segment values stay in L1 / L2:
// a frame reads at most smax of them.
template <typename Id, bool VEC>
__global__ void __launch_bounds__(kMapThreads)
segment_maps_kernel(const Id* __restrict__ seg, long long hw, const float* __restrict__ trav,
                    const float* __restrict__ conf, int smax, const int* __restrict__ n_rows, float* __restrict__ tmap,
                    float* __restrict__ cmap) {
  const int b = blockIdx.y;
  const unsigned live = static_cast<unsigned>(min(max(n_rows[b], 0), smax));
  const Id* s = seg + b * hw;
  const float* tv = trav + static_cast<long long>(b) * smax;
  const float* cv = conf ? conf + static_cast<long long>(b) * smax : nullptr;
  float* to = tmap + b * hw;
  float* co = cmap ? cmap + b * hw : nullptr;
  const long long stride = static_cast<long long>(gridDim.x) * kMapThreads;
  if constexpr (VEC) {
    const long long groups = hw / 4;
    for (long long g = blockIdx.x * static_cast<long long>(kMapThreads) + threadIdx.x; g < groups; g += stride) {
      Id id[4];
      if constexpr (sizeof(Id) == 8) {
        const longlong2 a = reinterpret_cast<const longlong2*>(s)[2 * g];
        const longlong2 c = reinterpret_cast<const longlong2*>(s)[2 * g + 1];
        id[0] = a.x; id[1] = a.y; id[2] = c.x; id[3] = c.y;
      } else {
        const int4 a = reinterpret_cast<const int4*>(s)[g];
        id[0] = a.x; id[1] = a.y; id[2] = a.z; id[3] = a.w;
      }
      reinterpret_cast<float4*>(to)[g] = make_float4(row_value(tv, id[0], live), row_value(tv, id[1], live),
                                                     row_value(tv, id[2], live), row_value(tv, id[3], live));
      if (co)
        reinterpret_cast<float4*>(co)[g] = make_float4(row_value(cv, id[0], live), row_value(cv, id[1], live),
                                                       row_value(cv, id[2], live), row_value(cv, id[3], live));
    }
  } else {
    for (long long p = blockIdx.x * static_cast<long long>(kMapThreads) + threadIdx.x; p < hw; p += stride) {
      const Id id = s[p];
      to[p] = row_value(tv, id, live);
      if (co) co[p] = row_value(cv, id, live);
    }
  }
}

template <typename Id>
int launch_segment_maps(const Id* seg, int batch, long long hw, const float* trav, const float* conf, int smax,
                        const int* n_rows, float* tmap, float* cmap, cudaStream_t stream) {
  auto aligned = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  const bool vec = hw % 4 == 0 && aligned(seg) && aligned(tmap) && (cmap == nullptr || aligned(cmap));
  const long long per_thread = vec ? 4 : 1;
  const long long blocks = std::min<long long>((hw + per_thread * kMapThreads - 1) / (per_thread * kMapThreads), 65535);
  const dim3 grid(static_cast<unsigned>(blocks), static_cast<unsigned>(batch));
  if (vec)
    segment_maps_kernel<Id, true><<<grid, kMapThreads, 0, stream>>>(seg, hw, trav, conf, smax, n_rows, tmap, cmap);
  else
    segment_maps_kernel<Id, false><<<grid, kMapThreads, 0, stream>>>(seg, hw, trav, conf, smax, n_rows, tmap, cmap);
  WVN_CHECK_LAUNCH("segment_maps_kernel");
  return WVN_OK;
}

}  // namespace

int segment_maps(const void* seg, bool seg_int64, int batch, long long hw, const float* trav, const float* conf, int smax,
                 const int* n_rows, float* trav_map, float* conf_map, cudaStream_t stream) {
  WVN_REQUIRE(seg && trav && n_rows && trav_map, "segment_maps: null argument");
  WVN_REQUIRE((conf == nullptr) == (conf_map == nullptr), "segment_maps: conf and conf_map go together");
  WVN_REQUIRE(batch >= 0 && batch <= 65535 && hw >= 0 && smax > 0,
              "segment_maps: bad geometry (batch=%d hw=%lld smax=%d)", batch, hw, smax);
  if (batch == 0 || hw == 0) return WVN_OK;
  if (seg_int64)
    return launch_segment_maps(static_cast<const long long*>(seg), batch, hw, trav, conf, smax, n_rows, trav_map,
                               conf_map, stream);
  return launch_segment_maps(static_cast<const int*>(seg), batch, hw, trav, conf, smax, n_rows, trav_map, conf_map,
                             stream);
}

}  // namespace wvn
