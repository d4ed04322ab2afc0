// wvn-b200: persistent warp-specialised bf16 GEMM on wgmma (sm_90a).
//
//   C[M,N] = A[M,K] (bf16, row-major / K-major) x W[N,K]^T (bf16, row-major / K-major)
//
// with fp32 accumulation in registers and a fused epilogue.  This one kernel family
// carries every dense contraction of the WVN hot path (SURVEY.md §2.1 K1/K3/K5/K6/K8 and
// the per-pixel traversability MLP K11): patch-embed, QKV, attention out-proj, MLP fc1/fc2,
// the STEGO head and the 384->256->32 layers of the traversability MLP.
//
// Structure (one CTA per SM, persistent over 64 x BN output tiles, three warpgroups):
//   warpgroup 0    : TMA producer (one warp: cp.async.bulk.tensor, 128B swizzle, mbarrier complete_tx); the warpgroup
//                    gives its registers up (setmaxnreg) to the consumers
//   warpgroups 1-2 : consumers in ping-pong: the CTA's tiles alternate between them, and each owns a whole tile —
//                    wgmma.mma_async on the shared-memory ring (both operands through descriptors, one wgmma group in
//                    flight while the next is issued), then the epilogue.  Named barriers 1 and 2 hand the turn to
//                    issue MMAs from one warpgroup to the other at the end of its k-loop, so one warpgroup's epilogue
//                    runs while the other's MMAs keep the tensor core busy.
// The epilogue (bias / activation) goes through a double-buffered shared-memory staging area, 32 columns at a time,
// and leaves as TMA bulk tensor stores (a bulk reduce-add into the fp32 residual stream; Q / K and the transposed V^T
// for attention); the warpgroup does not wait for a store except before it reuses its buffer.  The patch-embed and
// MLP-head epilogues store (or reduce) straight from the accumulator fragments.
// A tile's BN columns are covered by the widest wgmma shapes that fit (n128, then n64, then n32), so one kernel serves
// BN = 64 ... 256.
#include <stdlib.h>

#include <algorithm>

#include "common.cuh"
#include "gemm.h"
#include "host_common.h"

namespace wvn {

namespace {

constexpr int BM = 64;                        // rows of a tile: one consumer warpgroup's m64 wgmma
constexpr int BK = 64;
constexpr int kConsumerWarps = 8;             // two warpgroups of four warps
constexpr int kNumThreads = 128 + kConsumerWarps * 32;
constexpr int kMaxSmemBytes = 227 * 1024;
constexpr int kMaxStages = 8;
constexpr int kFixedSmemBytes = 1024 /*barriers*/ + 1024 /*align slack*/;
constexpr int kSliceCols = 32;                // columns per staged store
constexpr int kResidMaxBlockN = 192;          // widest tile of EPI_BF16_RESID

// Tile enumeration.  Default: tile ids run n-fastest over the whole (m, n)
// grid and are dealt round-robin to CTAs (neighbouring CTAs share the A tile through L2).  ROW_OWNER
// (used by EPI_MLP_HEAD): a CTA owns whole 64-row blocks and visits their n-chunks in order, so
// per-row reductions across n-chunks stay inside one thread quad.
template <bool ROW_OWNER>
struct TileIter {
  int num_m, num_n, m_blk, n_blk, lin;
  __device__ TileIter(int nm, int nn) : num_m(nm), num_n(nn), m_blk(0), n_blk(0), lin(0) {
    if (ROW_OWNER) { m_blk = blockIdx.x; n_blk = 0; }
    else { lin = blockIdx.x; m_blk = lin / num_n; n_blk = lin % num_n; }
  }
  __device__ bool valid() const { return m_blk < num_m; }
  __device__ void next() {
    if (ROW_OWNER) { if (++n_blk == num_n) { n_blk = 0; m_blk += gridDim.x; } }
    else { lin += gridDim.x; m_blk = lin / num_n; n_blk = lin % num_n; }
  }
};

template <int EPI>
constexpr bool kStaged = EPI == EPI_BF16 || EPI == EPI_F32 || EPI == EPI_RESID_F32 || EPI == EPI_QKV ||
                         EPI == EPI_BF16_RESID || EPI == EPI_SWIGLU;

template <int BN, int EPI>
struct GemmCfg {
  static constexpr uint32_t kABytes = BM * BK * 2;
  static constexpr uint32_t kBBytes = BN * BK * 2;
  static constexpr uint32_t kStageBytes = kABytes + kBBytes;
  // staging: one 64-row x 32-column slice of the output element type, two buffers per consumer warpgroup
  static constexpr uint32_t kSliceBytes = BM * kSliceCols * ((EPI == EPI_F32 || EPI == EPI_RESID_F32) ? 4 : 2);
  static constexpr uint32_t kStagingBytes = kStaged<EPI> ? 2 * 2 * kSliceBytes : 0;
  static constexpr int kStagesRaw = (kMaxSmemBytes - kFixedSmemBytes - kStagingBytes) / kStageBytes;
  static constexpr int kStages = kStagesRaw > kMaxStages ? kMaxStages : kStagesRaw;
  static constexpr uint32_t kSmemBytes = kStages * kStageBytes + kStagingBytes + kFixedSmemBytes;
  // wgmma shapes covering the BN columns: columns [0, 128 * kN128) by n128, the next 64 * kN64 by n64, the rest by n32
  static constexpr int kN128 = BN / 128;
  static constexpr int kN64 = (BN % 128) / 64;
  static constexpr int kN32 = (BN % 64) / 32;
};

// GELU(x) = x * Phi(x) with the erf form's Phi.  Phi(-|x|) = 2^p(|x|) (degree-5 minimax fit of log2 Phi(-t) on
// [0, 5.5], clamped beyond) and GELU(x) = max(x, 0) - t * Phi(-t), t = min(|x|, 5.5): max |error| 1.5e-6 —
// three orders below the bf16 rounding of the output.  1 MUFU + ~8 FMA/ALU issue slots per element instead of
// erff's ~30.
__device__ __forceinline__ float gelu_erf_fast(float x) {
  const float t = fminf(fabsf(x), 5.5f);
  float p = fmaf(-0.0003865310864f, t, 0.006509808358f);
  p = fmaf(p, t, -0.05048002675f);
  p = fmaf(p, t, -0.4613505006f);
  p = fmaf(p, t, -1.150225043f);
  p = fmaf(p, t, -1.00010848f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(p));
  return fmaf(-t, e, fmaxf(x, 0.f));
}

template <int ACT>
__device__ __forceinline__ float activate(float v) {
  if (ACT == ACT_RELU) return fmaxf(v, 0.f);
  if (ACT == ACT_GELU) return gelu_erf_fast(v);
  // SiLU; the fast division keeps the 256-column tiles free of spills, and gives -0 once 1 + e^-v exceeds 2^126
  if (ACT == ACT_SILU) return __fdividef(v, 1.f + __expf(-v));
  return v;
}

// Unstaged epilogue of one accumulator fragment (EPI_PATCH, EPI_MLP_HEAD): NREG / 4 groups of 8 columns starting at
// global column col_base; the thread holds columns col + {0, 1} (col = col_base + 8 j + 2 q) of rows row0 and
// row0 + 8.  The four lanes of a quad cover 8 consecutive columns of a row, so fp32 outputs leave as full 32-byte
// sectors.
template <int EPI, int ACT, int NREG>
__device__ __forceinline__ void epilogue_frag(const GemmArgs& args, const float (&d)[NREG], const int row0,
                                              const int col_base, const int lane, float (&head_partial)[2]) {
  const int q = lane & 3;
  bool ok[2];
  long long orow[2];
  int tok[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + 8 * h;
    ok[h] = row < args.M;
    orow[h] = row;
    tok[h] = 0;
    if (EPI == EPI_PATCH) {
      // patch row -> token row (frame * npad + 1 + registers + token) of the residual stream
      const int frame = row / args.tokens_in;
      tok[h] = row - frame * args.tokens_in;
      orow[h] = static_cast<long long>(frame) * args.npad + (1 + args.registers) + tok[h];
    }
  }
#pragma unroll
  for (int j = 0; j < NREG / 4; ++j) {
    const int col = col_base + 8 * j + 2 * q;
    float2 b = make_float2(0.f, 0.f);
    if (args.bias != nullptr) b = __ldg(reinterpret_cast<const float2*>(args.bias + col));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float v0 = activate<ACT>(d[4 * j + 2 * h] + b.x), v1 = activate<ACT>(d[4 * j + 2 * h + 1] + b.y);
      if (!ok[h]) continue;
      if (EPI == EPI_PATCH) {
        const float2 pe = __ldg(reinterpret_cast<const float2*>(args.pos + static_cast<long long>(1 + tok[h]) * args.ldo + col));
        *reinterpret_cast<float2*>(reinterpret_cast<float*>(args.out) + orow[h] * args.ldo + col) = make_float2(v0 + pe.x, v1 + pe.y);
      } else if (EPI == EPI_MLP_HEAD) {
        // columns [0, feat) = reconstruction of x, column trav_col = traversability logit
        if (col < args.feat) {
          const uint32_t xv = __ldg(reinterpret_cast<const uint32_t*>(
              reinterpret_cast<const __nv_bfloat16*>(args.x) + orow[h] * args.ldx + col));
          const float d0 = v0 - bf16_lo(xv), d1 = v1 - bf16_hi(xv);
          head_partial[h] = fmaf(d0, d0, head_partial[h]);
          if (col + 1 < args.feat) head_partial[h] = fmaf(d1, d1, head_partial[h]);
        } else if (col == args.trav_col) {
          args.trav[orow[h]] = 1.f / (1.f + __expf(-v0));
        }
      }
    }
  }
}

// Staged epilogue of one accumulator fragment: its columns [col_base, col_base + NREG * 2) leave in 32-column slices.
// For each slice the warpgroup waits until the store that last read the buffer has finished reading (one elected
// thread tracks the bulk groups), writes the slice into shared memory in the swizzled layout the store's tensor map
// expects, makes it visible to the async proxy, and the elected thread issues the store without waiting for it.
// Layouts (r = row of the tile, 0..63; 16-byte chunks XORed as TMA's swizzle modes do, so the quad-per-row fragment
// writes are free of bank conflicts):
//   fp32        : [64 rows][32 cols], 128-byte rows, 128B swizzle (chunk ^= r & 7)
//   bf16, Q / K : [64 rows][32 cols], 64-byte rows, 64B swizzle (chunk ^= (r >> 1) & 3)
//   V^T         : [32 head dims][64 tokens], 128-byte rows, 128B swizzle (chunk ^= dim & 7)
// EPI_SWIGLU: d is the gate fragment (tile columns [0, 128)) and dv the value fragment (columns [128, 256)).  They are
// two m64n128 accumulators of the same thread, register i of one and register i of the other holding the same row and
// the same column within its half, so gate column j meets value column j without a shuffle.  Each slice stores
// silu(g + b_g) * (v + b_v), computed in fp32 and rounded to bf16 once, at output column col_base / 2 + 32 s (col_base
// is the tile's first column of W and bias).  Every other epilogue ignores dv.
template <int EPI, int ACT, int NREG>
__device__ __forceinline__ void store_frag(const GemmArgs& args, const CUtensorMap* tm0, const CUtensorMap* tm1,
                                           const CUtensorMap* tm2, const float (&d)[NREG], const float (&dv)[NREG],
                                           const int row_tile,
                                           const int col_base, const int row_local, const int lane, const bool leader,
                                           const int bar_id, const uint32_t staging, const uint32_t slice_bytes,
                                           const int slice0) {
  const int q = lane & 3;
#pragma unroll
  for (int s = 0; s < NREG / 16; ++s) {
    const int col = col_base + kSliceCols * s;
    const int si = slice0 + s;  // slice of the tile: buffer si % 2
    const uint32_t buf = staging + (si & 1) * slice_bytes;
    int which = 0, within = 0;
    if (EPI == EPI_QKV) {
      which = col / args.dim;
      within = col - which * args.dim;
    }
    // the store that last read this buffer: the previous tile's (all of them are done reading by the time this tile's
    // k-loop has run) or the one of slice si - 2 (at most slice si - 1's is still reading)
    if (leader) {
      if (si == 0) tma_store_wait_read<0>();
      else tma_store_wait_read<1>();
    }
    named_bar_sync(bar_id, 128);
#pragma unroll
    for (int js = 0; js < 4; ++js) {
      const int j = 4 * s + js;
      const int c = col + 8 * js + 2 * q;
      float2 b = make_float2(0.f, 0.f), bv = make_float2(0.f, 0.f);
      if (args.bias != nullptr) b = __ldg(reinterpret_cast<const float2*>(args.bias + c));
      if (EPI == EPI_SWIGLU && args.bias != nullptr) bv = __ldg(reinterpret_cast<const float2*>(args.bias + c + 128));
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = row_local + 8 * h;
        float a0 = d[4 * j + 2 * h] + b.x, a1 = d[4 * j + 2 * h + 1] + b.y;
        if (EPI == EPI_SWIGLU) {
          a0 = activate<ACT_SILU>(a0) * (dv[4 * j + 2 * h] + bv.x);
          a1 = activate<ACT_SILU>(a1) * (dv[4 * j + 2 * h + 1] + bv.y);
        }
        if (EPI == EPI_BF16_RESID && row_tile + r < args.M) {
          // the residual is added before the activation: out = act(conv + bias + shortcut)
          const uint32_t rv = __ldg(reinterpret_cast<const uint32_t*>(
              reinterpret_cast<const __nv_bfloat16*>(args.residual) + static_cast<long long>(row_tile + r) * args.ldr + c));
          a0 += bf16_lo(rv);
          a1 += bf16_hi(rv);
        }
        const float v0 = activate<ACT>(a0), v1 = activate<ACT>(a1);
        if (EPI == EPI_F32 || EPI == EPI_RESID_F32) {
          sts64(buf + r * 128 + ((((2 * js + (q >> 1)) ^ (r & 7))) << 4) + (q & 1) * 8, v0, v1);
        } else if (EPI == EPI_QKV && which == 2) {
          const int dd = 8 * js + 2 * q;
          const uint32_t t = 2 * r;
          sts16(buf + dd * 128 + (((t >> 4) ^ (dd & 7)) << 4) + (t & 15), __float2bfloat16_rn(v0));
          sts16(buf + (dd + 1) * 128 + (((t >> 4) ^ ((dd + 1) & 7)) << 4) + (t & 15), __float2bfloat16_rn(v1));
        } else {
          sts32(buf + r * 64 + ((js ^ ((r >> 1) & 3)) << 4) + q * 4, pack_bf16x2(v0, v1));
        }
      }
    }
    fence_proxy_async_smem();
    named_bar_sync(bar_id, 128);
    if (leader) {
      if (EPI == EPI_BF16 || EPI == EPI_F32 || EPI == EPI_BF16_RESID) {
        tma_store_2d(tm0, buf, col, row_tile);
      } else if (EPI == EPI_SWIGLU) {
        tma_store_2d(tm0, buf, col_base / 2 + kSliceCols * s, row_tile);
      } else if (EPI == EPI_RESID_F32) {
        // x += acc + bias: one fp32 add per element, performed at L2
        tma_reduce_add_2d(tm0, buf, col, row_tile);
      } else if (EPI == EPI_QKV) {
        // a tile lies inside one frame (npad % BM == 0); Q / K are [b*h*npad, 64], V^T is [b*h*64, npad]
        const int frame = row_tile / args.npad;
        const int tok0 = row_tile - frame * args.npad;
        const int bh = frame * args.heads + (within >> 6);
        if (which < 2) tma_store_2d(which == 0 ? tm0 : tm1, buf, within & 63, bh * args.npad + tok0);
        else tma_store_2d(tm2, buf, tok0, bh * 64 + (within & 63));
      }
      tma_store_commit();
    }
  }
}

// ------------------------------------------------------------------------------------------------
// 64 x BN tiles, operands streamed through a kStages-deep TMA ring; consumer warpgroups take alternate tiles.
// ------------------------------------------------------------------------------------------------
template <int BN, int EPI, int ACT>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const __grid_constant__ CUtensorMap tmap_c0, const __grid_constant__ CUtensorMap tmap_c1,
                 const __grid_constant__ CUtensorMap tmap_c2, const GemmArgs args) {
  using Cfg = GemmCfg<BN, EPI>;
  constexpr int STAGES = Cfg::kStages;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_b = smem;
  uint8_t* smem_a = smem + STAGES * Cfg::kBBytes;
  uint8_t* smem_c = smem_a + STAGES * Cfg::kABytes;  // staging, 1024-aligned: [warpgroup][buffer][slice]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_c + Cfg::kStagingBytes);
  uint64_t* full_bar = bars;                // [kMaxStages]  TMA -> consumers
  uint64_t* empty_bar = bars + kMaxStages;  // [kMaxStages]  consumers -> TMA (one arrival per warp of the consuming warpgroup)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int num_m = (args.M + BM - 1) / BM;
  const int num_n = args.N / BN;
  // the last k-block may run past K: the tensor maps' inner extent is K, so TMA fills those columns with zeros
  const int num_k = (args.K + BK - 1) / BK;
  constexpr bool ROW_OWNER = (EPI == EPI_MLP_HEAD);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int i = 0; i < kMaxStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kConsumerWarps / 2);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------------------------------------------ TMA producer (whole warp in the loop, one
    // elected lane issues — see elect_one_sync in common.cuh)
    setmaxnreg_dec<40>();
    if (warp == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (TileIter<ROW_OWNER> it(num_m, num_n); it.valid(); it.next()) {
        const int m_eff = args.reverse_m ? num_m - 1 - it.m_blk : it.m_blk;
        for (int kb = 0; kb < num_k; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          if (elect_one_sync()) {
            mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
            tma_load_2d(&tmap_a, &full_bar[stage], smem_a + stage * Cfg::kABytes, kb * BK, m_eff * BM);
            tma_load_2d(&tmap_b, &full_bar[stage], smem_b + stage * Cfg::kBBytes, kb * BK, it.n_blk * BN);
          }
          __syncwarp();
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers: MMA + epilogue, ping-pong
    setmaxnreg_inc<232>();
    const int cwarp = warp - 4;               // 0..7
    const int wg = cwarp >> 2;                // which consumer warpgroup
    const int row_local = (cwarp & 3) * 16 + (lane >> 2);
    const bool leader = (threadIdx.x & 127) == 0;
    const uint32_t staging = smem_u32(smem_c) + wg * 2 * Cfg::kSliceBytes;
    if (kStaged<EPI> && leader) {
      tma_prefetch_desc(&tmap_c0);
      if (EPI == EPI_QKV) {
        tma_prefetch_desc(&tmap_c1);
        tma_prefetch_desc(&tmap_c2);
      }
    }
    // The CTA's work comes in units — a tile, or for ROW_OWNER a 64-row block with all its n-chunks — and unit u
    // belongs to warpgroup u % 2.  Turns to issue MMAs follow the units: warpgroup wg takes its turn on named barrier
    // 1 + wg and passes it on barrier 2 - wg once its k-loop is issued.  Warpgroup 1 opens with a pass to warpgroup 0
    // and the owner of the last unit does not pass, which keeps both barriers balanced for any unit count.
    if (wg == 1) named_bar_arrive(1, 256);
    float acc128[Cfg::kN128 > 0 ? Cfg::kN128 : 1][64];
    float acc64[32];
    float acc32[16];
    float head_partial[2] = {0.f, 0.f};
    int stage = 0;
    uint32_t phase = 0;
    int unit = 0;
    for (TileIter<ROW_OWNER> it(num_m, num_n); it.valid(); it.next()) {
      const bool unit_end = !ROW_OWNER || it.n_blk == num_n - 1;
      if ((unit & 1) != wg) {
        // the other warpgroup's tile: step the ring past its k-blocks
        for (int kb = 0; kb < num_k; ++kb)
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        if (unit_end) ++unit;
        continue;
      }
      if (!ROW_OWNER || it.n_blk == 0) named_bar_sync(1 + wg, 256);
      int prev_stage = 0;
      for (int kb = 0; kb < num_k; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t desc_a = make_sw128_kmajor_desc(smem_u32(smem_a + stage * Cfg::kABytes));
        const uint32_t b_addr = smem_u32(smem_b + stage * Cfg::kBBytes);
#pragma unroll
        for (int c = 0; c < Cfg::kN128; ++c) wgmma_fence_regs(acc128[c]);
        if (Cfg::kN64) wgmma_fence_regs(acc64);
        if (Cfg::kN32) wgmma_fence_regs(acc32);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          // advance 16 elements (32 B) along K inside the 128B swizzle atom: +2 in (addr>>4) units
          const uint32_t accumulate = (kb | k) != 0 ? 1u : 0u;
#pragma unroll
          for (int c = 0; c < Cfg::kN128; ++c)
            wgmma_m64n128k16_ss(acc128[c], desc_a + 2 * k, make_sw128_kmajor_desc(b_addr + c * 128 * 128) + 2 * k, accumulate);
          if (Cfg::kN64)
            wgmma_m64n64k16_ss(acc64, desc_a + 2 * k, make_sw128_kmajor_desc(b_addr + Cfg::kN128 * 128 * 128) + 2 * k, accumulate);
          if (Cfg::kN32)
            wgmma_m64n32k16_ss(acc32, desc_a + 2 * k,
                               make_sw128_kmajor_desc(b_addr + (Cfg::kN128 * 128 + Cfg::kN64 * 64) * 128) + 2 * k, accumulate);
        }
        wgmma_commit();
        if (kb > 0) {
          wgmma_wait<1>();  // the previous k-block's MMAs have retired: its ring slot is free
          if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
        }
        prev_stage = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      // pass the turn unless this was the CTA's last unit
      if (unit_end && (ROW_OWNER ? it.m_blk + static_cast<int>(gridDim.x) < num_m : it.lin + static_cast<int>(gridDim.x) < num_m * num_n))
        named_bar_arrive(2 - wg, 256);
      wgmma_wait<0>();
#pragma unroll
      for (int c = 0; c < Cfg::kN128; ++c) wgmma_fence_regs(acc128[c]);
      if (Cfg::kN64) wgmma_fence_regs(acc64);
      if (Cfg::kN32) wgmma_fence_regs(acc32);
      if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);

      const int m_eff = args.reverse_m ? num_m - 1 - it.m_blk : it.m_blk;
      const int row_tile = m_eff * BM;
      const int col0 = it.n_blk * BN;
      if constexpr (EPI == EPI_SWIGLU) {
        static_assert(BN == 256, "EPI_SWIGLU pairs the two n128 halves of a 256-column tile");
        store_frag<EPI, ACT_NONE>(args, &tmap_c0, &tmap_c1, &tmap_c2, acc128[0], acc128[1], row_tile, col0, row_local,
                                  lane, leader, 3 + wg, staging, Cfg::kSliceBytes, 0);
      } else if (kStaged<EPI>) {
        const int bar_id = 3 + wg;
#pragma unroll
        for (int c = 0; c < Cfg::kN128; ++c)
          store_frag<EPI, ACT>(args, &tmap_c0, &tmap_c1, &tmap_c2, acc128[c], acc128[c], row_tile, col0 + c * 128,
                               row_local, lane, leader, bar_id, staging, Cfg::kSliceBytes, 4 * c);
        if (Cfg::kN64)
          store_frag<EPI, ACT>(args, &tmap_c0, &tmap_c1, &tmap_c2, acc64, acc64, row_tile, col0 + Cfg::kN128 * 128,
                               row_local, lane, leader, bar_id, staging, Cfg::kSliceBytes, 4 * Cfg::kN128);
        if (Cfg::kN32)
          store_frag<EPI, ACT>(args, &tmap_c0, &tmap_c1, &tmap_c2, acc32, acc32, row_tile,
                               col0 + Cfg::kN128 * 128 + Cfg::kN64 * 64, row_local, lane, leader, bar_id, staging, Cfg::kSliceBytes, 4 * Cfg::kN128 + 2 * Cfg::kN64);
      } else {
        const int row0 = row_tile + row_local;
#pragma unroll
        for (int c = 0; c < Cfg::kN128; ++c)
          epilogue_frag<EPI, ACT>(args, acc128[c], row0, col0 + c * 128, lane, head_partial);
        if (Cfg::kN64) epilogue_frag<EPI, ACT>(args, acc64, row0, col0 + Cfg::kN128 * 128, lane, head_partial);
        if (Cfg::kN32) epilogue_frag<EPI, ACT>(args, acc32, row0, col0 + Cfg::kN128 * 128 + Cfg::kN64 * 64, lane, head_partial);
      }

      if (EPI == EPI_MLP_HEAD && it.n_blk == num_n - 1) {
        // a row's columns live in the four lanes of a quad: combine them, then loss_reco -> confidence
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float s = head_partial[h];
          s += __shfl_xor_sync(0xffffffffu, s, 1);
          s += __shfl_xor_sync(0xffffffffu, s, 2);
          head_partial[h] = 0.f;
          const int row = row_tile + row_local + 8 * h;
          if ((lane & 3) == 0 && row < args.M) {
            const float loss = s / static_cast<float>(args.feat);
            // ConfidenceGenerator.inference_without_update (utils/confidence_generator.py:182-193)
            const float mean = __ldg(args.cg_mean), sd = __ldg(args.cg_std);
            const float shifted = mean + sd * args.cg_std_factor;
            const float lo = fmaxf(shifted - sd, 0.f);
            const float hi = shifted + sd;
            const float xc = fminf(fmaxf(loss, lo), hi);
            args.conf[row] = 1.f - (xc - lo) / (hi - lo);
            if (args.loss_reco != nullptr) args.loss_reco[row] = loss;
          }
        }
      }
      if (unit_end) ++unit;
    }
    // the staging buffers must outlive the stores that read them
    if (kStaged<EPI> && leader) tma_store_wait_all<0>();
  }
}

template <int BN, int EPI, int ACT>
int launch_gemm(const GemmArgs& a, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap (&tc)[3],
                cudaStream_t stream) {
  using Cfg = GemmCfg<BN, EPI>;
  static_assert(Cfg::kStages >= 2, "tile too wide for the shared-memory budget");
  auto kern = gemm_bf16_kernel<BN, EPI, ACT>;
  static bool attr_set = false;
  if (!attr_set) {
    WVN_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmemBytes));
    attr_set = true;
  }
  const int num_m = (a.M + BM - 1) / BM, num_n = a.N / BN;
  const int num_tiles = (EPI == EPI_MLP_HEAD) ? num_m : num_m * num_n;
  int grid = sm_count();
  if (a.max_ctas > 0 && a.max_ctas < grid) grid = a.max_ctas;
  if (grid > num_tiles) grid = num_tiles;
  prof_begin(PROF_GEMM, stream);
  kern<<<grid, kNumThreads, Cfg::kSmemBytes, stream>>>(ta, tb, tc[0], tc[1], tc[2], a);
  prof_end(PROF_GEMM, stream);
  WVN_CHECK_LAUNCH("gemm_bf16_kernel");
  return WVN_OK;
}

template <int BN>
int dispatch_epi(const GemmArgs& a, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap (&tc)[3],
                 cudaStream_t s) {
  switch (a.epi) {
    case EPI_BF16:
      if (a.act == ACT_NONE) return launch_gemm<BN, EPI_BF16, ACT_NONE>(a, ta, tb, tc, s);
      if (a.act == ACT_RELU) return launch_gemm<BN, EPI_BF16, ACT_RELU>(a, ta, tb, tc, s);
      if (a.act == ACT_GELU) return launch_gemm<BN, EPI_BF16, ACT_GELU>(a, ta, tb, tc, s);
      if (a.act == ACT_SILU) return launch_gemm<BN, EPI_BF16, ACT_SILU>(a, ta, tb, tc, s);
      break;
    case EPI_F32:
      if (a.act == ACT_NONE) return launch_gemm<BN, EPI_F32, ACT_NONE>(a, ta, tb, tc, s);
      break;
    case EPI_RESID_F32:
      if (a.act == ACT_NONE) return launch_gemm<BN, EPI_RESID_F32, ACT_NONE>(a, ta, tb, tc, s);
      break;
    case EPI_PATCH:
      if (a.act == ACT_NONE) return launch_gemm<BN, EPI_PATCH, ACT_NONE>(a, ta, tb, tc, s);
      break;
    case EPI_QKV:
      if (a.act == ACT_NONE) return launch_gemm<BN, EPI_QKV, ACT_NONE>(a, ta, tb, tc, s);
      break;
    case EPI_MLP_HEAD:
      if (a.act == ACT_NONE) return launch_gemm<BN, EPI_MLP_HEAD, ACT_NONE>(a, ta, tb, tc, s);
      break;
    case EPI_BF16_RESID:
      // the residual's loads do not fit beside 224- and 256-column accumulators without spilling (gemm_bf16 keeps
      // block_n <= kResidMaxBlockN for this epilogue)
      if constexpr (BN <= kResidMaxBlockN) {
        if (a.act == ACT_NONE) return launch_gemm<BN, EPI_BF16_RESID, ACT_NONE>(a, ta, tb, tc, s);
        if (a.act == ACT_RELU) return launch_gemm<BN, EPI_BF16_RESID, ACT_RELU>(a, ta, tb, tc, s);
      }
      break;
    case EPI_SWIGLU:
      if constexpr (BN == 256) {
        if (a.act == ACT_NONE) return launch_gemm<BN, EPI_SWIGLU, ACT_NONE>(a, ta, tb, tc, s);
      }
      break;
  }
  return set_error(WVN_ERR_INVALID, "gemm: unsupported epilogue/activation combination (%d, %d)", a.epi, a.act);
}

}  // namespace

int pick_block_n(int N) {
  if (N % 256 == 0) return 256;
  if (N % 224 == 0) return 224;
  if (N % 192 == 0) return 192;
  if (N % 128 == 0) return 128;
  if (N % 64 == 0) return 64;
  return 0;
}

int gemm_bf16(const GemmArgs& a, const void* A, long long lda, const void* W, int block_n, cudaStream_t stream) {
  WVN_REQUIRE(a.M > 0 && a.N > 0 && a.K > 0, "gemm: empty problem (M=%d N=%d K=%d)", a.M, a.N, a.K);
  WVN_REQUIRE(lda >= a.K, "gemm: lda=%lld is smaller than K=%d", lda, a.K);
  if (block_n == 0) {
    block_n = a.epi == EPI_SWIGLU ? 256 : pick_block_n(a.N);
    if (a.epi == EPI_BF16_RESID && block_n > kResidMaxBlockN) block_n = a.N % 192 == 0 ? 192 : (a.N % 128 == 0 ? 128 : 64);
  }
  WVN_REQUIRE(a.epi != EPI_BF16_RESID || block_n <= kResidMaxBlockN, "gemm: the residual epilogue takes block_n <= %d",
              kResidMaxBlockN);
  WVN_REQUIRE(block_n == 64 || block_n == 128 || block_n == 192 || block_n == 224 || block_n == 256,
              "gemm: bad block_n %d", block_n);
  WVN_REQUIRE(a.N % block_n == 0, "gemm: N=%d must be a multiple of block_n=%d (pad the weights)", a.N, block_n);
  if (a.epi == EPI_MLP_HEAD)
    WVN_REQUIRE(a.feat > 0 && a.trav_col % 32 == 0 && a.trav_col >= a.feat && a.trav_col < a.N && a.x != nullptr &&
                    a.trav != nullptr && a.conf != nullptr && a.cg_mean != nullptr && a.cg_std != nullptr &&
                    a.ldx % 8 == 0 && a.ldx >= a.trav_col,
                "gemm: bad MLP-head epilogue arguments (feat=%d trav_col=%d N=%d)", a.feat, a.trav_col, a.N);
  // QKV: a 64-row tile must lie inside one frame, so that each of its 32-column slices is one box of Q, K or V^T
  if (a.epi == EPI_QKV)
    WVN_REQUIRE(a.dim % 64 == 0 && a.N == 3 * a.dim && a.heads * 64 == a.dim && a.npad % 8 == 0 && a.npad % BM == 0 &&
                    a.M % a.npad == 0,
                "gemm: bad QKV epilogue geometry (dim=%d heads=%d npad=%d N=%d M=%d)", a.dim, a.heads, a.npad, a.N, a.M);
  // patch embed: the CLS row, the register rows and the patch rows of a frame fit in its npad rows
  if (a.epi == EPI_PATCH)
    WVN_REQUIRE(a.tokens_in > 0 && a.registers >= 0 && 1 + a.registers + a.tokens_in <= a.npad,
                "gemm: bad patch-embed epilogue geometry (tokens_in=%d registers=%d npad=%d)", a.tokens_in, a.registers,
                a.npad);
  if (a.epi == EPI_SWIGLU)
    WVN_REQUIRE(block_n == 256 && a.act == ACT_NONE && a.ldo % 8 == 0 && a.ldo >= a.N / 2,
                "gemm: the SwiGLU epilogue takes block_n 256, no activation and a bf16 output pitch ldo >= N / 2, a "
                "multiple of 8 (block_n=%d act=%d ldo=%lld N=%d)", block_n, a.act, a.ldo, a.N);
  if (a.epi == EPI_F32 || a.epi == EPI_RESID_F32) WVN_REQUIRE(a.ldo % 4 == 0, "gemm: fp32 output pitch must be a multiple of 4");
  if (a.epi == EPI_BF16 || a.epi == EPI_BF16_RESID) WVN_REQUIRE(a.ldo % 8 == 0, "gemm: bf16 output pitch must be a multiple of 8");
  if (a.epi == EPI_BF16_RESID)
    WVN_REQUIRE(a.residual != nullptr && a.ldr >= a.N && a.ldr % 2 == 0,
                "gemm: the residual epilogue needs a bf16 residual with an even pitch ldr >= N (ldr=%lld N=%d)", a.ldr, a.N);
  CUtensorMap ta, tb, tc[3] = {};
  // Both maps take the true K as their inner extent, so the pad columns of a K that is not a multiple of 64 are never
  // read (TMA zero-fills the last k-block past K, whatever the pad columns hold).  W's rows sit at a 16-byte pitch.
  WVN_PROPAGATE(make_tmap_bf16_2d(&ta, A, a.K, a.M, static_cast<uint64_t>(lda) * 2, BK, BM));
  WVN_PROPAGATE(make_tmap_bf16_2d(&tb, W, a.K, a.N, static_cast<uint64_t>(gemm_w_pitch(a.K)) * 2, BK, block_n));
  // output maps for the staged epilogues: 32-column x 64-row boxes (store_frag's layouts); rows past M are clipped
  if (a.epi == EPI_BF16 || a.epi == EPI_BF16_RESID)
    WVN_PROPAGATE(make_tmap_2d(&tc[0], a.out, 2, a.N, a.M, static_cast<uint64_t>(a.ldo) * 2, kSliceCols, BM, 64));
  if (a.epi == EPI_SWIGLU)
    WVN_PROPAGATE(make_tmap_2d(&tc[0], a.out, 2, a.N / 2, a.M, static_cast<uint64_t>(a.ldo) * 2, kSliceCols, BM, 64));
  if (a.epi == EPI_F32 || a.epi == EPI_RESID_F32)
    WVN_PROPAGATE(make_tmap_2d(&tc[0], a.out, 4, a.N, a.M, static_cast<uint64_t>(a.ldo) * 4, kSliceCols, BM, 128));
  if (a.epi == EPI_QKV) {
    const uint64_t bh = static_cast<uint64_t>(a.M / a.npad) * a.heads;
    WVN_PROPAGATE(make_tmap_2d(&tc[0], a.q, 2, 64, bh * a.npad, 128, kSliceCols, BM, 64));
    WVN_PROPAGATE(make_tmap_2d(&tc[1], a.k, 2, 64, bh * a.npad, 128, kSliceCols, BM, 64));
    WVN_PROPAGATE(make_tmap_2d(&tc[2], a.vt, 2, a.npad, bh * 64, static_cast<uint64_t>(a.npad) * 2, BM, kSliceCols, 128));
  }
  switch (block_n) {
    case 64: return dispatch_epi<64>(a, ta, tb, tc, stream);
    case 128: return dispatch_epi<128>(a, ta, tb, tc, stream);
    case 192: return dispatch_epi<192>(a, ta, tb, tc, stream);
    case 224: return dispatch_epi<224>(a, ta, tb, tc, stream);
    case 256: return dispatch_epi<256>(a, ta, tb, tc, stream);
  }
  return set_error(WVN_ERR_INVALID, "gemm: unreachable");
}

}  // namespace wvn
