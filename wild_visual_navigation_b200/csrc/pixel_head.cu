// wvn-b200: fused per-pixel traversability head (sm_90a).
//
// Replaces, per frame (wvn_feature_extractor_node.py:319-370, simple_mlp.py:33-39,
// confidence_generator.py:182-193):
//     x = dense_feat[0].permute(1,2,0).reshape(-1, D)          # 200704 x 384, bilinear(align_corners=True)
//     pred = SimpleMLP(x);  trav = pred[:, 0]
//     loss_reco = mse(pred[:, 1:], x).mean(1);  conf = inference_without_update(loss_reco)
//
// The per-pixel work is restructured algebraically so that neither x (384-d) nor pred (385-d) is
// ever formed per pixel — only the 256-d hidden layer is:
//   * layer 1 is affine and bilinear weights sum to 1:  W1 x + b1 = sum_k w_k (W1 t_k + b1)
//     -> G = tokens @ W1^T + b1 is computed ONCE PER TOKEN (3136 rows/frame, wgmma GEMM) and the
//        kernel below interpolates G (256 ch) instead of x (384 ch) followed by a 384->256 GEMM;
//   * with r = R h2 + c the reconstruction (R = W3[1:], c = b3[1:]):
//       D*loss = |r|^2 - 2 r.x + |x|^2
//       |r|^2  = h2^T (R^T R) h2 + 2 (R^T c).h2 + c.c          (32x32 quadratic form, fp32)
//       r.x    = sum_k w_k ( h2 . (R^T t_k) + c.t_k )            (U = tokens @ R, cT = tokens @ c: per token)
//       |x|^2  = bilinear form of the 2x2 neighbourhood's Gram    (5 dot products per token)
// Per pixel that leaves: interpolate 256+33 channels, one 256->32 layer on the tensor core
// (wgmma, M=128 pixels, N=32), and ~650 fp32 FMAs — ~12x fewer FLOPs than the direct form, and
// no HBM traffic beyond the two output maps.  bf16 rounding points are the same as the unfused
// path (tokens, weights, h1); everything downstream of the layer-2 accumulator is fp32.
//
// The same kernel serves the DoubleMLP (two networks of widths h1 / 32 on the same features, net 0 -> traversability,
// net 1 -> reconstruction): G = tokens @ [W1_0; W1_1]^T + [b1_0; b1_1] (2 h1 channels), U / cT from net 1's last layer,
// and layer 2 as TWO m64n32 wgmma chains over the two K halves of the h1 tile, one per network.  The block-diagonal
// alternative (one N = 64 chain over all 2 h1 channels) would spend half of its MMAs on the zero blocks and keep 64
// accumulators live per thread; two chains keep the SimpleMLP head's instruction, W2 tile and shared-memory layout, and
// net 0's chain (which only feeds the logit) is reduced to one partial sum per fragment row before net 1's (which only
// feeds the reconstruction terms) is issued, so at most 32 accumulators are live, as in the SimpleMLP head.
#include <algorithm>

#include "common.cuh"
#include "double_mlp_train.h"
#include "host_common.h"
#include "pixel_head.h"

namespace wvn {

namespace {

constexpr int kH1 = 256, kH2 = 32;
constexpr int kTileW = 64, kTileH = 2;            // 128 pixels per tile: row i = r*64 + px
constexpr int kWinMax = 10;                        // token-window columns per tile (ratio 8: 7 + 3)
constexpr int kGvStride = 292;                     // 256 G + 32 U + cT_hi + cT_lo, padded to float4 (the largest row)
constexpr int kThreads = 256;
constexpr uint32_t kOffA = 0;                      // [4 K-blocks][128 rows][128 B]  h1 tile (bf16, swizzled); once layer 2
                                                   // has consumed it: [128 pixels][kH2Stride] fp32 layer-2 accumulator
constexpr int kH2Stride = 36;                      // floats per pixel row of that tile (16-byte aligned, conflict-free)
constexpr uint32_t kOffW2 = 65536;                 // [4 K-blocks][32 rows][128 B]
constexpr uint32_t kOffGv = kOffW2 + 16384;        // [2][kWinMax][kGvStride] fp32
constexpr uint32_t kOffN2 = kOffGv + 2 * kWinMax * kGvStride * 4;  // [2][kWinMax][2] fp32: |xv|^2, xv_c.xv_{c+1}
constexpr uint32_t kOffPix = kOffN2 + 2 * kWinMax * 2 * 4;        // per-tile pixel tables (see PixTables)
struct PixTables {
  float wx[kTileW];         // horizontal blend weight of pixel px
  int c0[kTileW];           // its left window column (token column - cx0)
  int start[kWinMax + 2];   // first pixel of each window cell (kTileW for cells with no pixel)
  int row0[kTileH * kWinMax], row1[kTileH * kWinMax];  // element offsets of the upper / lower source token row of window cell (r, c)
};
constexpr uint32_t kOffBar = kOffPix + ((sizeof(PixTables) + 15) / 16) * 16;
constexpr uint32_t kSmemBytes = kOffBar + 64;

// Weight-only constants of the head (2 * R^T c, R^T R, b2, ...): read as constant-bank operands of the
// epilogue's FMAs.  Copied device-to-device on the launch stream before every launch (pixel_head()).
__constant__ PixelHeadConsts c_ph;

__device__ __forceinline__ void ac_true(int dst, float scale, int in_size, int& i0, float& w1) {
  const float s = dst * scale;
  i0 = min(static_cast<int>(s), in_size - 1);
  w1 = s - static_cast<float>(i0);
}

// max(x, 0) fused into the bf16x2 conversion
__device__ __forceinline__ uint32_t pack_bf16x2_relu(float lo, float hi) {
  uint32_t d;
  asm("cvt.rn.relu.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}

// kK: channels of the h1 tile (= layer 2's K; 256 for the SimpleMLP head, 2 h1 for the DoubleMLP), kNets: 1 (SimpleMLP)
// or 2 (DoubleMLP: net 0's h1 in channels [0, kK/2), net 1's in [kK/2, kK); W2's K blocks of net 1 are read from rows
// 32..63 of the W2 operand, i.e. the block-diagonal layer 2 of the packed unfused operands).
template <int kK, int kNets>
__global__ void __launch_bounds__(kThreads, kNets == 1 ? 2 : 1)
pixel_head_kernel(const __grid_constant__ CUtensorMap tmap_w2, const PixelHeadArgs a) {
  static_assert(kK % 64 == 0 && kK <= kH1 && (kNets == 1 || kK % 128 == 0), "pixel_head_kernel: h1 tile shape");
  constexpr int kGvS = (kK + kH2 + 2 + 3) / 4 * 4;   // G | U | cT_hi | cT_lo, padded to float4 (292 for kK = 256)
  constexpr int kKB = kK / 64;                       // 64-channel K blocks of the h1 tile
  extern __shared__ __align__(1024) uint8_t smem[];
  float* gv = reinterpret_cast<float*>(smem + kOffGv);
  float* n2 = reinterpret_cast<float*>(smem + kOffN2);
  PixTables* pt = reinterpret_cast<PixTables*>(smem + kOffPix);
  uint64_t* w2_full = reinterpret_cast<uint64_t*>(smem + kOffBar);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_x = a.W / kTileW, tiles_y = a.H / kTileH;
  const long long tiles_per_frame = static_cast<long long>(tiles_x) * tiles_y;
  const long long num_tiles = tiles_per_frame * a.batch;
  const int P = a.gh * a.gw;
  const int ww = a.ww;

  if (threadIdx.x == 0) {
    if ((smem_u32(smem) & 1023u) != 0) { printf("[wvn] pixel_head: smem base not 1024B aligned\n"); __trap(); }
    mbar_init(w2_full, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(w2_full, kKB * 32 * 128);
    for (int kb = 0; kb < kKB; ++kb)
      tma_load_2d(&tmap_w2, w2_full, smem + kOffW2 + kb * 4096, kb * 64, (kNets == 2 && kb >= kKB / 2) ? 32 : 0);
  }

  // Tile geometry: pixel rows [py0, py0+2), pixel columns [px0, px0+64) of frame b; cx0 = first token column of the window.
  struct TileGeo { int b, py0, px0, cx0; };
  auto tile_geo = [&](long long tile) {
    TileGeo g;
    g.b = static_cast<int>(tile / tiles_per_frame);
    const int trem = static_cast<int>(tile - g.b * tiles_per_frame);
    g.py0 = (trem / tiles_x) * kTileH;
    g.px0 = (trem % tiles_x) * kTileW;
    float tmpw;
    ac_true(g.px0, a.sx, a.gw, g.cx0, tmpw);
    return g;
  };

  // ---------------- phase A (warps 4-7, one tile AHEAD of the consumers): vertical blend of the token window
  // (G | U | cT) into gv, the |x|^2 ingredients into n2, and the per-pixel horizontal tables.
  auto phase_a = [&](const TileGeo& g) {
    const int t = threadIdx.x - 128;  // 0..127
    const float* gub = a.gu + (static_cast<long long>(g.b) * (a.frame_rows ? a.frame_rows : P) + a.row0) * a.ldg;
    int y0r[kTileH], y1r[kTileH];
    float wyr[kTileH];
#pragma unroll
    for (int r = 0; r < kTileH; ++r) {
      ac_true(g.py0 + r, a.sy, a.gh, y0r[r], wyr[r]);
      y1r[r] = min(y0r[r] + 1, a.gh - 1);
    }
    // element offsets of the window's source rows: one table entry per (r, c), built by 2 * ww threads, so
    // that the copy loop below carries no per-item address arithmetic beyond a table lookup
    if (t < kTileH * ww) {
      const int r = t >= ww ? 1 : 0, c = t - r * ww;
      const int tc = min(g.cx0 + c, a.gw - 1);
      pt->row0[t] = (y0r[r] * a.gw + tc) * static_cast<int>(a.ldg);
      pt->row1[t] = (y1r[r] * a.gw + tc) * static_cast<int>(a.ldg);
    }
    named_bar_sync(2, 128);
    constexpr int kV4 = kGvS / 4;
    constexpr int kBatch = 6;  // float4 pairs in flight per thread and pass (48 registers)
    constexpr int kStepRc = 128 / kV4, kStepV4 = 128 % kV4;
    const int n_rc = kTileH * ww;
    // item i = t + 128 * k  <->  (rc, v4) = (i / kV4, i % kV4), advanced incrementally (128 = kStepRc kV4 + kStepV4)
    int rc, v4;
    if constexpr (2 * kV4 > 128) {
      rc = t >= kV4 ? 1 : 0;
      v4 = t - rc * kV4;
    } else {
      rc = t / kV4;
      v4 = t - rc * kV4;
    }
    while (rc < n_rc) {
      float4 g0[kBatch], g1[kBatch];
      int rcs[kBatch], v4s[kBatch];
#pragma unroll
      for (int it = 0; it < kBatch; ++it) {
        rcs[it] = rc; v4s[it] = v4;
        if (rc < n_rc) {
          g0[it] = __ldg(reinterpret_cast<const float4*>(gub + pt->row0[rc]) + v4);
          g1[it] = __ldg(reinterpret_cast<const float4*>(gub + pt->row1[rc]) + v4);
        }
        v4 += kStepV4; rc += kStepRc;
        if (v4 >= kV4) { v4 -= kV4; rc += 1; }
      }
#pragma unroll
      for (int it = 0; it < kBatch; ++it) {
        if (rcs[it] < n_rc) {
          const float wy = wyr[rcs[it] >= ww ? 1 : 0];
          float4 o;
          o.x = fmaf(wy, g1[it].x - g0[it].x, g0[it].x);
          o.y = fmaf(wy, g1[it].y - g0[it].y, g0[it].y);
          o.z = fmaf(wy, g1[it].z - g0[it].z, g0[it].z);
          o.w = fmaf(wy, g1[it].w - g0[it].w, g0[it].w);
          reinterpret_cast<float4*>(gv)[rcs[it] * kV4 + v4s[it]] = o;
        }
      }
    }
    if (t < kTileW) {  // per-pixel horizontal source column / weight, first pixel of every window cell
      int x0, xp, xl;
      float wx, wp;
      ac_true(g.px0 + t, a.sx, a.gw, x0, wx);
      pt->wx[t] = wx;
      pt->c0[t] = x0 - g.cx0;
      ac_true(g.px0 + t - 1, a.sx, a.gw, xp, wp);
      if (t == 0 || xp != x0) pt->start[x0 - g.cx0] = t;
      ac_true(g.px0 + kTileW - 1, a.sx, a.gw, xl, wp);
      if (t > xl - g.cx0 && t < kWinMax + 2) pt->start[t] = kTileW;  // cells right of the last pixel
    } else if (t - kTileW < kTileH * ww) {
      // xv_c = (1-wy) t[y0,c] + wy t[y1,c]:  |xv_c|^2 and xv_c . xv_{c+1} from the per-token Gram entries
      // (0 self, 1 right neighbour, 2 lower neighbour, 3 lower-right, 4 right . lower); all loads unconditional
      const int q = t - kTileW;
      const int r = q >= ww ? 1 : 0, c = q - r * ww;
      const float wy = wyr[r], u = 1.f - wy;
      const bool same_y = (y0r[r] + 1 > a.gh - 1);
      const int tc = min(g.cx0 + c, a.gw - 1);
      const bool same_x = (tc + 1 > a.gw - 1);
      const float* gr = a.gram + (static_cast<long long>(g.b) * (a.frame_rows ? a.frame_rows : P) + a.row0) * 5;
      const float* e0 = gr + (static_cast<long long>(y0r[r]) * a.gw + tc) * 5;
      const float* e1 = gr + (static_cast<long long>(y1r[r]) * a.gw + tc) * 5;
      const float s00 = __ldg(e0), h0 = __ldg(e0 + 1), v0r = __ldg(e0 + 2), dr = __ldg(e0 + 3), anr = __ldg(e0 + 4);
      const float s10 = __ldg(e1), h1 = __ldg(e1 + 1);
      const float v0 = same_y ? s00 : v0r;
      const float nn = u * u * s00 + 2.f * u * wy * v0 + wy * wy * s10;
      const float d = same_y ? h0 : dr, an = same_y ? h0 : anr;
      const float xx = same_x ? nn : u * u * h0 + u * wy * (d + an) + wy * wy * h1;
      n2[(r * ww + c) * 2 + 0] = nn;
      n2[(r * ww + c) * 2 + 1] = xx;
    }
  };

  if (warp >= 4 && blockIdx.x < num_tiles) phase_a(tile_geo(blockIdx.x));
  for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const TileGeo g = tile_geo(tile);
    const int b = g.b, py0 = g.py0, px0 = g.px0, cx0 = g.cx0;
    __syncthreads();  // phase A of this tile is visible; the previous tile's A operand / accumulator are drained

    // ---------------- phase B (all warps): horizontal blend -> ReLU -> bf16 -> swizzled A tile (h1)
    {
      const int units = kTileH * (ww - 1);  // (row, cell) pairs; cell c spans window columns [c, c+1]
      for (int u = warp; u < units; u += kThreads / 32) {
        if (kK < kH1 && 8 * lane >= kK) continue;   // lanes past the tile's channels
        const int r = u >= (ww - 1) ? 1 : 0, cell = u - r * (ww - 1);
        const int p_begin = pt->start[cell], p_end = pt->start[cell + 1];  // contiguous run of this cell's pixels
        if (p_begin >= p_end) continue;
        const float* g0p = gv + (r * ww + cell) * kGvS + 8 * lane;
        const float4 a0 = reinterpret_cast<const float4*>(g0p)[0], a1 = reinterpret_cast<const float4*>(g0p)[1];
        const float4 b0 = reinterpret_cast<const float4*>(g0p + kGvS)[0];
        const float4 b1 = reinterpret_cast<const float4*>(g0p + kGvS)[1];
        const float gg[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float dg[8] = {b0.x - a0.x, b0.y - a0.y, b0.z - a0.z, b0.w - a0.w,
                             b1.x - a1.x, b1.y - a1.y, b1.z - a1.z, b1.w - a1.w};
        // channel block 8*lane..8*lane+7: K-block lane/8, 16-byte chunk lane%8 (128B swizzle)
        const uint32_t kb_base = smem_u32(smem + kOffA) + (lane >> 3) * 16384;
        for (int pxb = p_begin; pxb < p_end; pxb += 3) {
#pragma unroll
          for (int k = 0; k < 3; ++k) {  // three independent pixels in flight
            const int px = pxb + k;
            if (px < p_end) {
              const float wx = pt->wx[px];
              float h[8];
#pragma unroll
              for (int i = 0; i < 8; ++i) h[i] = fmaf(wx, dg[i], gg[i]);
              const int row = r * kTileW + px;
              sts128(kb_base + row * 128 + (((lane & 7) ^ (row & 7)) << 4), pack_bf16x2_relu(h[0], h[1]),
                     pack_bf16x2_relu(h[2], h[3]), pack_bf16x2_relu(h[4], h[5]), pack_bf16x2_relu(h[6], h[7]));
            }
          }
        }
      }
    }
    fence_proxy_async_smem();
    __syncthreads();

    if (warp >= 4) {
      // ---------------- producers: once the consumers have taken what they need from gv / n2 / the pixel
      // tables, build the NEXT tile's while the tensor core and the epilogue warpgroup work on this one
      named_bar_sync(1, kThreads);
      if (tile + gridDim.x < num_tiles) phase_a(tile_geo(tile + gridDim.x));
    } else {
      if constexpr (kNets == 1) {
      // ---------------- layer 2 on the tensor core: D[128, 32] = h1[128, 256] @ W2^T, issued by this warpgroup
        // (two 64-row halves) and left in flight while each thread prepares its pixel's blend terms
        float d2[2][16];
        mbar_wait(w2_full, 0);  // completes once; later tiles pass at once
        wgmma_fence();
  #pragma unroll
        for (int ks = 0; ks < kK / 16; ++ks) {
          const uint64_t db = make_sw128_kmajor_desc(smem_u32(smem + kOffW2 + (ks >> 2) * 4096)) + 2 * (ks & 3);
  #pragma unroll
          for (int half = 0; half < 2; ++half)
            wgmma_m64n32k16_ss(d2[half], make_sw128_kmajor_desc(smem_u32(smem + kOffA + (ks >> 2) * 16384 + half * 8192)) + 2 * (ks & 3),
                               db, ks != 0);
        }
        wgmma_commit();
        // ---------------- epilogue: one thread per pixel
        const int i = threadIdx.x;  // pixel
        const int r = i >> 6, px = i & 63;
        const float wx = pt->wx[px];
        const int c0 = pt->c0[px];
        const bool same_x = (cx0 + c0 + 1 > a.gw - 1);
        // U columns of the two neighbouring window columns (c0+1 is a clamped duplicate at the right border)
        const float4* u0 = reinterpret_cast<const float4*>(gv + (r * ww + c0) * kGvS + kK);
        const float4* u1 = u0 + kGvS / 4;
        float ub[kH2 + 4];  // blended U (32) | cT_hi, cT_lo
  #pragma unroll
        for (int j4 = 0; j4 < kH2 / 4 + 1; ++j4) {
          const float4 p0 = u0[j4], p1 = u1[j4];
          ub[4 * j4 + 0] = fmaf(wx, p1.x - p0.x, p0.x);
          ub[4 * j4 + 1] = fmaf(wx, p1.y - p0.y, p0.y);
          ub[4 * j4 + 2] = fmaf(wx, p1.z - p0.z, p0.z);
          ub[4 * j4 + 3] = fmaf(wx, p1.w - p0.w, p0.w);
        }
        const float* nn = n2 + (r * ww + c0) * 2;
        const float ux = 1.f - wx;
        const float n_c1 = same_x ? nn[0] : nn[2];
        const float xx = same_x ? nn[0] : nn[1];
        const float gram = ux * ux * nn[0] + 2.f * ux * wx * xx + wx * wx * n_c1;
        asm volatile("bar.arrive 1, %0;" ::"n"(kThreads) : "memory");  // gv / n2 / tables consumed: producers may refill
  
        wgmma_wait<0>();
        wgmma_fence_regs(d2[0]);
        wgmma_fence_regs(d2[1]);
        // fragments -> one pixel per thread, through the h1 tile once every warp's MMAs have consumed it
        named_bar_sync(3, 128);
        float* h2s = reinterpret_cast<float*>(smem + kOffA);
  #pragma unroll
        for (int half = 0; half < 2; ++half)
  #pragma unroll
          for (int j = 0; j < 4; ++j)
  #pragma unroll
            for (int hh = 0; hh < 2; ++hh)
              *reinterpret_cast<float2*>(h2s + (half * 64 + warp * 16 + (lane >> 2) + 8 * hh) * kH2Stride + 8 * j + 2 * (lane & 3)) =
                  make_float2(d2[half][4 * j + 2 * hh], d2[half][4 * j + 2 * hh + 1]);
        named_bar_sync(3, 128);
        float h2[kH2];
  #pragma unroll
        for (int j4 = 0; j4 < kH2 / 4; ++j4) {
          const float4 raw = reinterpret_cast<const float4*>(h2s + i * kH2Stride)[j4];
          h2[4 * j4 + 0] = fmaxf(raw.x + c_ph.b2[4 * j4 + 0], 0.f);
          h2[4 * j4 + 1] = fmaxf(raw.y + c_ph.b2[4 * j4 + 1], 0.f);
          h2[4 * j4 + 2] = fmaxf(raw.z + c_ph.b2[4 * j4 + 2], 0.f);
          h2[4 * j4 + 3] = fmaxf(raw.w + c_ph.b2[4 * j4 + 3], 0.f);
        }
        // traversability logit, |r|^2 quadratic form (upper-triangular M with doubled off-diagonals), r.x
        float t = c_ph.b0, q = c_ph.cc, cross = ub[kH2] + ub[kH2 + 1];
  #pragma unroll
        for (int j = 0; j < kH2; ++j) {
          t = fmaf(c_ph.w0[j], h2[j], t);
          float acc = c_ph.tv[j];
  #pragma unroll
          for (int k = j; k < kH2; ++k) acc = fmaf(c_ph.m[j * kH2 + k], h2[k], acc);
          q = fmaf(h2[j], acc, q);
          cross = fmaf(h2[j], ub[j], cross);
        }
        const float loss = fmaxf(q - 2.f * cross + gram, 0.f) / static_cast<float>(a.feat);
        const float mean = __ldg(a.cg_mean), sd = __ldg(a.cg_std);
        const float shifted = mean + sd * a.std_factor;
        const float lo = fmaxf(shifted - sd, 0.f), hi = shifted + sd;
        const float xc = fminf(fmaxf(loss, lo), hi);
        const long long o = (static_cast<long long>(b) * a.H + py0 + r) * a.W + px0 + px;
        a.trav[o] = 1.f / (1.f + __expf(-t));
        a.conf[o] = 1.f - (xc - lo) / (hi - lo);
        if (a.loss_reco != nullptr) a.loss_reco[o] = loss;
      } else {
        // ---------------- layer 2 on the tensor core, one m64n32 chain per network over its half of the h1 tile:
        // D_n[128, 32] = h1_n[128, kK/2] @ W2_n^T, net 0 first
        float d0[2][16], d1[2][16];
        mbar_wait(w2_full, 0);  // completes once; later tiles pass at once
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < kK / 32; ++ks) {
          const uint64_t db = make_sw128_kmajor_desc(smem_u32(smem + kOffW2 + (ks >> 2) * 4096)) + 2 * (ks & 3);
#pragma unroll
          for (int half = 0; half < 2; ++half)
            wgmma_m64n32k16_ss(d0[half], make_sw128_kmajor_desc(smem_u32(smem + kOffA + (ks >> 2) * 16384 + half * 8192)) + 2 * (ks & 3),
                               db, ks != 0);
        }
        wgmma_commit();
        // net 0 only feeds the logit: once its chain completes, reduce its fragments to one partial sum per fragment
        // row, w0 . ReLU(z + b2) over this thread's 8 columns, then over the 4 lanes that share the row
        wgmma_wait<0>();
        wgmma_fence_regs(d0[0]);
        wgmma_fence_regs(d0[1]);
        float tp[2][2];
#pragma unroll
        for (int half = 0; half < 2; ++half)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            float acc = 0.f;
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int col = 8 * j + 2 * (lane & 3) + e;
                acc = fmaf(c_ph.w0[col], fmaxf(d0[half][4 * j + 2 * hh + e] + c_ph.b2[col], 0.f), acc);
              }
            acc += __shfl_xor_sync(0xffffffffu, acc, 1);
            acc += __shfl_xor_sync(0xffffffffu, acc, 2);
            tp[half][hh] = acc;
          }
        // net 1's chain, left in flight while each thread prepares its pixel's blend terms
        wgmma_fence();
#pragma unroll
        for (int ks = kK / 32; ks < kK / 16; ++ks) {
          const uint64_t db = make_sw128_kmajor_desc(smem_u32(smem + kOffW2 + (ks >> 2) * 4096)) + 2 * (ks & 3);
#pragma unroll
          for (int half = 0; half < 2; ++half)
            wgmma_m64n32k16_ss(d1[half], make_sw128_kmajor_desc(smem_u32(smem + kOffA + (ks >> 2) * 16384 + half * 8192)) + 2 * (ks & 3),
                               db, ks != kK / 32);
        }
        wgmma_commit();
        // ---------------- epilogue: one thread per pixel
        const int i = threadIdx.x;  // pixel
        const int r = i >> 6, px = i & 63;
        const float wx = pt->wx[px];
        const int c0 = pt->c0[px];
        const bool same_x = (cx0 + c0 + 1 > a.gw - 1);
        const float4* u0 = reinterpret_cast<const float4*>(gv + (r * ww + c0) * kGvS + kK);
        const float4* u1 = u0 + kGvS / 4;
        float ub[kH2 + 4];  // blended U (32) | cT_hi, cT_lo
#pragma unroll
        for (int j4 = 0; j4 < kH2 / 4 + 1; ++j4) {
          const float4 p0 = u0[j4], p1 = u1[j4];
          ub[4 * j4 + 0] = fmaf(wx, p1.x - p0.x, p0.x);
          ub[4 * j4 + 1] = fmaf(wx, p1.y - p0.y, p0.y);
          ub[4 * j4 + 2] = fmaf(wx, p1.z - p0.z, p0.z);
          ub[4 * j4 + 3] = fmaf(wx, p1.w - p0.w, p0.w);
        }
        const float* nn = n2 + (r * ww + c0) * 2;
        const float ux = 1.f - wx;
        const float n_c1 = same_x ? nn[0] : nn[2];
        const float xx = same_x ? nn[0] : nn[1];
        const float gram = ux * ux * nn[0] + 2.f * ux * wx * xx + wx * wx * n_c1;
        asm volatile("bar.arrive 1, %0;" ::"n"(kThreads) : "memory");  // gv / n2 / tables consumed: producers may refill

        wgmma_wait<0>();
        wgmma_fence_regs(d1[0]);
        wgmma_fence_regs(d1[1]);
        // net 1's fragments and net 0's logit partials -> one pixel per thread, through the h1 tile
        named_bar_sync(3, 128);
        float* h2s = reinterpret_cast<float*>(smem + kOffA);
        float* ts = h2s + 128 * kH2Stride;
#pragma unroll
        for (int half = 0; half < 2; ++half)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int row = half * 64 + warp * 16 + (lane >> 2) + 8 * hh;
#pragma unroll
            for (int j = 0; j < 4; ++j)
              *reinterpret_cast<float2*>(h2s + row * kH2Stride + 8 * j + 2 * (lane & 3)) =
                  make_float2(d1[half][4 * j + 2 * hh], d1[half][4 * j + 2 * hh + 1]);
            if ((lane & 3) == 0) ts[row] = tp[half][hh];
          }
        named_bar_sync(3, 128);
        const float t = c_ph.b0 + ts[i];
        float h2[kH2];
#pragma unroll
        for (int j4 = 0; j4 < kH2 / 4; ++j4) {
          const float4 raw = reinterpret_cast<const float4*>(h2s + i * kH2Stride)[j4];
          h2[4 * j4 + 0] = fmaxf(raw.x + c_ph.b2r[4 * j4 + 0], 0.f);
          h2[4 * j4 + 1] = fmaxf(raw.y + c_ph.b2r[4 * j4 + 1], 0.f);
          h2[4 * j4 + 2] = fmaxf(raw.z + c_ph.b2r[4 * j4 + 2], 0.f);
          h2[4 * j4 + 3] = fmaxf(raw.w + c_ph.b2r[4 * j4 + 3], 0.f);
        }
        float q = c_ph.cc, cross = ub[kH2] + ub[kH2 + 1];
  #pragma unroll
        for (int j = 0; j < kH2; ++j) {
          float acc = c_ph.tv[j];
  #pragma unroll
          for (int k = j; k < kH2; ++k) acc = fmaf(c_ph.m[j * kH2 + k], h2[k], acc);
          q = fmaf(h2[j], acc, q);
          cross = fmaf(h2[j], ub[j], cross);
        }
        const float loss = fmaxf(q - 2.f * cross + gram, 0.f) / static_cast<float>(a.feat);
        const float mean = __ldg(a.cg_mean), sd = __ldg(a.cg_std);
        const float shifted = mean + sd * a.std_factor;
        const float lo = fmaxf(shifted - sd, 0.f), hi = shifted + sd;
        const float xc = fminf(fmaxf(loss, lo), hi);
        const long long o = (static_cast<long long>(b) * a.H + py0 + r) * a.W + px0 + px;
        a.trav[o] = 1.f / (1.f + __expf(-t));
        a.conf[o] = 1.f - (xc - lo) / (hi - lo);
        if (a.loss_reco != nullptr) a.loss_reco[o] = loss;
      }
    }
  }
}

// One warp per token: self / right / lower / lower-right / (right . lower) dot products (bf16 tokens).
__global__ void __launch_bounds__(256)
token_gram_kernel(const __nv_bfloat16* __restrict__ tok, float* __restrict__ gram, int batch, int gh, int gw, int dim,
                  long long frame_rows, int row0) {
  const int lane = threadIdx.x & 31;
  const long long warp_global = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const long long warps_total = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const long long P = static_cast<long long>(gh) * gw;
  for (long long t = warp_global; t < batch * P; t += warps_total) {
    const int x = static_cast<int>(t % gw), y = static_cast<int>((t / gw) % gh);
    const bool has_r = x + 1 < gw, has_d = y + 1 < gh;
    const long long row = (t / P) * frame_rows + row0 + (t % P);   // token t of the batch in the (possibly padded) buffer
    const __nv_bfloat16* p00 = tok + row * dim;
    const __nv_bfloat16* p01 = has_r ? p00 + dim : p00;
    const __nv_bfloat16* p10 = has_d ? p00 + static_cast<long long>(gw) * dim : p00;
    const __nv_bfloat16* p11 = p10 + (has_r ? dim : 0);
    float s = 0.f, h = 0.f, v = 0.f, d = 0.f, an = 0.f;
    for (int c = lane * 2; c < dim; c += 64) {
      const float2 a00 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p00 + c));
      const float2 a01 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p01 + c));
      const float2 a10 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p10 + c));
      const float2 a11 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p11 + c));
      s = fmaf(a00.x, a00.x, fmaf(a00.y, a00.y, s));
      h = fmaf(a00.x, a01.x, fmaf(a00.y, a01.y, h));
      v = fmaf(a00.x, a10.x, fmaf(a00.y, a10.y, v));
      d = fmaf(a00.x, a11.x, fmaf(a00.y, a11.y, d));
      an = fmaf(a01.x, a10.x, fmaf(a01.y, a10.y, an));
    }
    s = warp_sum(s); h = warp_sum(h); v = warp_sum(v); d = warp_sum(d); an = warp_sum(an);
    if (lane == 0) {
      float* g = gram + row * 5;
      g[0] = s; g[1] = h; g[2] = v; g[3] = d; g[4] = an;
    }
  }
}

// Weight-only constants of the fused head, from the flat fp32 state-dict parameters (bf16-rounded R,
// to match the U = tokens @ R columns the tensor core produces from bf16 operands).
// One block of 32 x 32 threads: thread (j, k) owns M[j][k]; row 0 also produces tv / b2 / w0.  R (bf16-rounded) and c
// are staged in shared memory in chunks of 384 channels and every thread runs four independent accumulators over the
// chunk (instead of walking the 384 channels with two dependent global loads each).
// The operands, as pointers into the flat parameters: R [dim][32] and c [dim] (the reconstruction rows of the last
// layer and their bias), w0 [32] / b0 (the traversability row and its bias), b2 / b2r [32] (layer 2's bias of the
// traversability / reconstruction path: the same for a SimpleMLP).
struct HeadSources {
  const float *R, *c, *w0, *b0, *b2, *b2r;
};

__global__ void __launch_bounds__(1024)
pixel_head_consts_kernel(HeadSources hs, int dim, PixelHeadConsts* out) {
  constexpr int kChunk = 384;
  __shared__ __nv_bfloat16 rs[kChunk * kH2];
  __shared__ float cs[kChunk];
  const int k = threadIdx.x & 31, j = threadIdx.x >> 5;
  const float* w3 = hs.R;
  float m4[4] = {0.f, 0.f, 0.f, 0.f}, tv4[4] = {0.f, 0.f, 0.f, 0.f}, cc4[4] = {0.f, 0.f, 0.f, 0.f};
  for (int d0 = 0; d0 < dim; d0 += kChunk) {
    const int nd = min(kChunk, dim - d0);
    for (int i = threadIdx.x; i < nd * kH2; i += 1024) rs[i] = __float2bfloat16_rn(w3[static_cast<long long>(d0) * kH2 + i]);
    for (int i = threadIdx.x; i < nd; i += 1024) cs[i] = hs.c[d0 + i];
    __syncthreads();
    auto step = [&](int d, int q) {
      const float rj = __bfloat162float(rs[d * kH2 + j]);
      const float rk = __bfloat162float(rs[d * kH2 + k]);
      const float c = cs[d];
      m4[q] = fmaf(rj, rk, m4[q]);
      tv4[q] = fmaf(rj, c, tv4[q]);
      cc4[q] = fmaf(c, c, cc4[q]);
    };
    int d = 0;
    for (; d + 4 <= nd; d += 4) { step(d, 0); step(d + 1, 1); step(d + 2, 2); step(d + 3, 3); }
    for (; d < nd; ++d) step(d, 0);
    __syncthreads();
  }
  const float m = (m4[0] + m4[1]) + (m4[2] + m4[3]);
  const float tv = (tv4[0] + tv4[1]) + (tv4[2] + tv4[3]);
  const float cc = (cc4[0] + cc4[1]) + (cc4[2] + cc4[3]);
  out->m[j * kH2 + k] = (k == j) ? m : (k > j ? 2.f * m : 0.f);
  if (k == 0) {
    out->tv[j] = 2.f * tv;
    out->b2[j] = hs.b2[j];
    out->b2r[j] = hs.b2r[j];
    out->w0[j] = __bfloat162float(__float2bfloat16_rn(hs.w0[j]));  // the logit row (bf16 like the GEMM path)
  }
  if (threadIdx.x == 0) {
    out->b0 = *hs.b0;
    out->cc = cc;
  }
}

// Wcat [n, dim_p] bf16 = [W1 ; R^T ; c_hi ; c_lo ; 0], bias [n] = [b1 ; 0], n = pixel_head_columns(ng).  The ng G rows
// come from w1a / b1a (rows [0, ha)) and w1b / b1b (rows [ha, ng): the DoubleMLP's second network).
__global__ void pixel_head_pack_kernel(const float* __restrict__ w1a, const float* __restrict__ b1a, int ha,
                                       const float* __restrict__ w1b, const float* __restrict__ b1b, int ng, HeadSources hs,
                                       int n, int dim, int dim_p, __nv_bfloat16* __restrict__ wcat, float* __restrict__ bias) {
  const long long total = static_cast<long long>(n) * dim_p;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / dim_p), d = static_cast<int>(i % dim_p);
    float v = 0.f;
    if (d < dim) {
      if (r < ha) v = w1a[static_cast<long long>(r) * dim + d];
      else if (r < ng) v = w1b[static_cast<long long>(r - ha) * dim + d];
      else if (r < ng + kH2) v = hs.R[static_cast<long long>(d) * kH2 + (r - ng)];
      else if (r == ng + kH2) v = hs.c[d];
      else if (r == ng + kH2 + 1) {
        const float c = hs.c[d];
        v = c - __bfloat162float(__float2bfloat16_rn(c));
      }
    }
    wcat[i] = __float2bfloat16_rn(v);
    if (d == 0) bias[r] = r < ha ? b1a[r] : (r < ng ? b1b[r - ha] : 0.f);
  }
}

int window_width(int gh, int gw, int H, int W) {
  if (H % kTileH != 0 || W % kTileW != 0 || H < 2 || W < 2) return 0;
  const float sx = static_cast<float>(gw - 1) / static_cast<float>(W - 1);
  const int ww = static_cast<int>((kTileW - 1) * sx) + 3;
  return (ww >= 2 && ww <= kWinMax) ? ww : 0;
}

template <int kK, int kNets>
int launch_pixel_head(const PixelHeadArgs& a, const void* w2_bf16, int w2_ld, cudaStream_t stream) {
  constexpr int kGvS = (kK + kH2 + 2 + 3) / 4 * 4;
  WVN_REQUIRE(a.ww >= 2 && a.ww <= kWinMax && a.W % kTileW == 0 && a.H % kTileH == 0, "pixel_head: unsupported geometry");
  WVN_REQUIRE(a.ldg >= kGvS && a.ldg % 4 == 0, "pixel_head: ldg %lld too small", a.ldg);
  WVN_REQUIRE(static_cast<long long>(a.gh) * a.gw * a.ldg < (1ll << 31), "pixel_head: token grid too large for 32-bit row offsets");
  CUtensorMap tw;
  WVN_PROPAGATE(make_tmap_bf16_2d(&tw, w2_bf16, kK, kNets * kH2, static_cast<uint64_t>(w2_ld) * 2, 64, kH2));
  static bool attr_set = false;
  if (!attr_set) {
    WVN_CHECK_CUDA(cudaFuncSetAttribute(pixel_head_kernel<kK, kNets>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        kSmemBytes));
    attr_set = true;
  }
  const long long tiles = static_cast<long long>(a.batch) * (a.H / kTileH) * (a.W / kTileW);
  // one resident CTA per SM for the DoubleMLP instantiation (189 registers: it spills at the SimpleMLP head's 128)
  int grid = static_cast<int>(std::min<long long>(tiles, static_cast<long long>(sm_count()) * (kNets == 1 ? 2 : 1)));
  WVN_CHECK_CUDA(cudaMemcpyToSymbolAsync(c_ph, a.consts, sizeof(PixelHeadConsts), 0, cudaMemcpyDeviceToDevice, stream));
  pixel_head_kernel<kK, kNets><<<grid, kThreads, kSmemBytes, stream>>>(tw, a);
  WVN_CHECK_LAUNCH("pixel_head_kernel");
  return WVN_OK;
}

}  // namespace

int pixel_head_supported(int h1, int h2, int gh, int gw, int H, int W) {
  if (h1 != kH1 || h2 != kH2) return 0;
  return window_width(gh, gw, H, W);
}

bool pixel_head_double_shape(int h1, int h2) { return (h1 == 64 || h1 == 128) && h2 == kH2; }

int pixel_head_supported_double(int h1, int h2, int gh, int gw, int H, int W) {
  return pixel_head_double_shape(h1, h2) ? window_width(gh, gw, H, W) : 0;
}

int pixel_head_columns(int g_channels) { return (g_channels + kH2 + 2 + 63) / 64 * 64; }

int pixel_head_pack(const float* params, const MlpShape& s, int dim_p, void* wcat_bf16, float* bias,
                    PixelHeadConsts* consts, cudaStream_t stream) {
  const MlpOffsets o = mlp_offsets(s);
  const HeadSources hs{params + o.w3 + kH2, params + o.b3 + 1, params + o.w3, params + o.b3, params + o.b2, params + o.b2};
  pixel_head_pack_kernel<<<128, 256, 0, stream>>>(params + o.w1, params + o.b1, kH1, nullptr, nullptr, kH1, hs,
                                                  kPixelHeadN, s.dim, dim_p, reinterpret_cast<__nv_bfloat16*>(wcat_bf16),
                                                  bias);
  WVN_CHECK_LAUNCH("pixel_head_pack_kernel");
  pixel_head_consts_kernel<<<1, 1024, 0, stream>>>(hs, s.dim, consts);
  WVN_CHECK_LAUNCH("pixel_head_consts_kernel");
  return WVN_OK;
}

int pixel_head_pack_double(const float* params, const MlpShape& net, int dim_p, void* wcat_bf16, float* bias,
                           PixelHeadConsts* consts, cudaStream_t stream) {
  WVN_REQUIRE(pixel_head_double_shape(net.h1, net.h2), "pixel_head_pack_double: h1 = %d, h2 = %d outside the "
              "fused head", net.h1, net.h2);
  const DoubleOffsets o = double_mlp_offsets(net);
  const HeadSources hs{params + o.w3[1], params + o.b3[1], params + o.w3[0], params + o.b3[0], params + o.b2[0],
                       params + o.b2[1]};
  pixel_head_pack_kernel<<<128, 256, 0, stream>>>(params + o.w1[0], params + o.b1[0], net.h1, params + o.w1[1],
                                                  params + o.b1[1], 2 * net.h1, hs, pixel_head_columns(2 * net.h1),
                                                  net.dim, dim_p, reinterpret_cast<__nv_bfloat16*>(wcat_bf16), bias);
  WVN_CHECK_LAUNCH("pixel_head_pack_kernel");
  pixel_head_consts_kernel<<<1, 1024, 0, stream>>>(hs, net.dim, consts);
  WVN_CHECK_LAUNCH("pixel_head_consts_kernel");
  return WVN_OK;
}

int token_gram(const void* tok_bf16, float* gram, int batch, int gh, int gw, int dim, long long frame_rows, int row0,
               cudaStream_t stream) {
  if (frame_rows <= 0) frame_rows = static_cast<long long>(gh) * gw;
  WVN_REQUIRE(dim % 64 == 0, "token_gram: dim %d must be a multiple of 64", dim);
  const long long warps = static_cast<long long>(batch) * gh * gw;
  int blocks = static_cast<int>(std::min<long long>((warps * 32 + 255) / 256, static_cast<long long>(sm_count()) * 16));
  token_gram_kernel<<<blocks, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(tok_bf16), gram, batch, gh, gw, dim,
                                                frame_rows, row0);
  WVN_CHECK_LAUNCH("token_gram_kernel");
  return WVN_OK;
}

int pixel_head(const PixelHeadArgs& a, const void* w2_bf16, int w2_ld, cudaStream_t stream) {
  return launch_pixel_head<kH1, 1>(a, w2_bf16, w2_ld, stream);
}

int pixel_head_double(const PixelHeadArgs& a, int h1, const void* w2_bf16, int w2_ld, cudaStream_t stream) {
  if (h1 == 64) return launch_pixel_head<128, 2>(a, w2_bf16, w2_ld, stream);
  if (h1 == 128) return launch_pixel_head<256, 2>(a, w2_bf16, w2_ld, stream);
  return set_error(WVN_ERR_INVALID, "pixel_head_double: h1 = %d outside the fused head (64 or 128)", h1);
}

}  // namespace wvn
