// wvn-b200: persistent warp-specialised bf16 GEMM on wgmma (sm_90a).
//
//   C[M,N] = A[M,K] (bf16, row-major / K-major) x W[N,K]^T (bf16, row-major / K-major)
//
// with fp32 accumulation in registers and a fused epilogue.  This one kernel family
// carries every dense contraction of the WVN hot path (SURVEY.md §2.1 K1/K3/K5/K6/K8 and
// the per-pixel traversability MLP K11): patch-embed, QKV, attention out-proj, MLP fc1/fc2,
// the STEGO head and the 384->256->32 layers of the traversability MLP.
//
// Structure (one CTA per SM, persistent over 128 x BN output tiles, three warpgroups):
//   warpgroup 0    : TMA producer (one warp: cp.async.bulk.tensor, 128B swizzle, mbarrier complete_tx); the warpgroup
//                    gives its registers up (setmaxnreg) to the consumers
//   warpgroups 1-2 : consumers, 64 rows of the tile each: wgmma.mma_async on the shared-memory ring (both operands
//                    through descriptors, one wgmma group in flight while the next is issued), then the epilogue
//                    straight from the accumulator fragments (bias / activation / residual -> global memory).  The
//                    producer keeps filling the ring with the next tile's operands during the epilogue.
// A tile's BN columns are covered by the widest wgmma shapes that fit (n128, then n64, then n32), so one kernel serves
// BN = 64 ... 256.
#include <stdlib.h>

#include <algorithm>

#include "common.cuh"
#include "gemm.h"
#include "host_common.h"

namespace wvn {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int kConsumerWarps = 8;             // two warpgroups of four warps
constexpr int kNumThreads = 128 + kConsumerWarps * 32;
constexpr int kMaxSmemBytes = 227 * 1024;
constexpr int kMaxStages = 8;
constexpr int kFixedSmemBytes = 1024 /*barriers*/ + 1024 /*align slack*/;

// Tile enumeration.  Default: tile ids run n-fastest over the whole (m, n)
// grid and are dealt round-robin to CTAs (neighbouring CTAs share the A tile through L2).  ROW_OWNER
// (used by EPI_MLP_HEAD): a CTA owns whole 128-row blocks and visits their n-chunks in order, so
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

template <int BN>
struct GemmCfg {
  static constexpr uint32_t kABytes = BM * BK * 2;
  static constexpr uint32_t kBBytes = BN * BK * 2;
  static constexpr uint32_t kStageBytes = kABytes + kBBytes;
  static constexpr int kStagesRaw = (kMaxSmemBytes - kFixedSmemBytes) / kStageBytes;
  static constexpr int kStages = kStagesRaw > kMaxStages ? kMaxStages : kStagesRaw;
  static constexpr uint32_t kSmemBytes = kStages * kStageBytes + kFixedSmemBytes;
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

// Epilogue of one accumulator fragment: NREG / 4 groups of 8 columns starting at global column col_base; the thread
// holds columns col + {0, 1} (col = col_base + 8 j + 2 q) of rows row0 and row0 + 8.  The four lanes of a quad cover
// 8 consecutive columns of a row, so fp32 outputs leave as full 32-byte sectors.
template <int EPI, int ACT, int NREG>
__device__ __forceinline__ void epilogue_frag(const GemmArgs& args, const float (&d)[NREG], const int row0,
                                              const int col_base, const int lane, float (&head_partial)[2]) {
  const int q = lane & 3;
  bool ok[2];
  long long orow[2];
  int frame[2], tok[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + 8 * h;
    ok[h] = row < args.M;
    orow[h] = row;
    frame[h] = tok[h] = 0;
    if (EPI == EPI_PATCH) {
      // patch row -> token row (frame * npad + 1 + token) of the residual stream
      frame[h] = row / args.tokens_in;
      tok[h] = row - frame[h] * args.tokens_in;
      orow[h] = static_cast<long long>(frame[h]) * args.npad + 1 + tok[h];
    } else if (EPI == EPI_QKV) {
      frame[h] = row / args.npad;
      tok[h] = row - frame[h] * args.npad;
    }
  }
#pragma unroll
  for (int j = 0; j < NREG / 4; ++j) {
    const int col = col_base + 8 * j + 2 * q;
    float2 b = make_float2(0.f, 0.f);
    if (args.bias != nullptr) b = __ldg(reinterpret_cast<const float2*>(args.bias + col));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float v0 = d[4 * j + 2 * h] + b.x, v1 = d[4 * j + 2 * h + 1] + b.y;
      if (ACT == ACT_RELU) {
        v0 = fmaxf(v0, 0.f);
        v1 = fmaxf(v1, 0.f);
      } else if (ACT == ACT_GELU) {
        v0 = gelu_erf_fast(v0);
        v1 = gelu_erf_fast(v1);
      }
      if (!ok[h]) continue;
      if (EPI == EPI_BF16) {
        *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(args.out) + orow[h] * args.ldo + col) = pack_bf16x2(v0, v1);
      } else if (EPI == EPI_F32) {
        *reinterpret_cast<float2*>(reinterpret_cast<float*>(args.out) + orow[h] * args.ldo + col) = make_float2(v0, v1);
      } else if (EPI == EPI_RESID_F32) {
        // the residual stream is updated with vector reductions: x += acc + bias happens at L2, no load
        asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(reinterpret_cast<float*>(args.out) + orow[h] * args.ldo + col),
                     "f"(v0), "f"(v1)
                     : "memory");
      } else if (EPI == EPI_PATCH) {
        const float2 pe = __ldg(reinterpret_cast<const float2*>(args.pos + static_cast<long long>(1 + tok[h]) * args.ldo + col));
        *reinterpret_cast<float2*>(reinterpret_cast<float*>(args.out) + orow[h] * args.ldo + col) = make_float2(v0 + pe.x, v1 + pe.y);
      } else if (EPI == EPI_QKV) {
        const int which = col / args.dim;
        const int within = col - which * args.dim;
        const long long bh = static_cast<long long>(frame[h]) * args.heads + (within >> 6);
        if (which < 2) {  // Q / K: [b*h, npad, 64]
          __nv_bfloat16* base = reinterpret_cast<__nv_bfloat16*>(which == 0 ? args.q : args.k);
          *reinterpret_cast<uint32_t*>(base + (bh * args.npad + tok[h]) * 64 + (within & 63)) = pack_bf16x2(v0, v1);
        } else {
          // V is stored transposed ([b, h, d, token]) so that P·V consumes it K-major: the 8 lanes that share q hold
          // 8 consecutive tokens of one column
          __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(args.vt) + (bh * 64 + (within & 63)) * args.npad + tok[h];
          dst[0] = __float2bfloat16_rn(v0);
          dst[args.npad] = __float2bfloat16_rn(v1);
        }
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

// ------------------------------------------------------------------------------------------------
// 128 x BN tiles, operands streamed through a kStages-deep TMA ring.
// ------------------------------------------------------------------------------------------------
template <int BN, int EPI, int ACT>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const GemmArgs args) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::kStages;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_b = smem;
  uint8_t* smem_a = smem + STAGES * Cfg::kBBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_a + STAGES * Cfg::kABytes);
  uint64_t* full_bar = bars;                // [kMaxStages]  TMA -> consumers
  uint64_t* empty_bar = bars + kMaxStages;  // [kMaxStages]  consumers -> TMA (one arrival per consumer warp)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int num_m = (args.M + BM - 1) / BM;
  const int num_n = args.N / BN;
  const int num_k = args.K / BK;
  constexpr bool ROW_OWNER = (EPI == EPI_MLP_HEAD);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int i = 0; i < kMaxStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kConsumerWarps);
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
    // ------------------------------------------------------------------ consumers: MMA + epilogue
    setmaxnreg_inc<232>();
    const int cwarp = warp - 4;               // 0..7
    const int wg = cwarp >> 2;                // which 64-row half of the tile
    const int row_in_tile = wg * 64 + (cwarp & 3) * 16 + (lane >> 2);
    float acc128[Cfg::kN128 > 0 ? Cfg::kN128 : 1][64];
    float acc64[32];
    float acc32[16];
    float head_partial[2] = {0.f, 0.f};
    int stage = 0;
    uint32_t phase = 0;
    for (TileIter<ROW_OWNER> it(num_m, num_n); it.valid(); it.next()) {
      int prev_stage = 0;
      for (int kb = 0; kb < num_k; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t desc_a = make_sw128_kmajor_desc(smem_u32(smem_a + stage * Cfg::kABytes + wg * 64 * 128));
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
      wgmma_wait<0>();
#pragma unroll
      for (int c = 0; c < Cfg::kN128; ++c) wgmma_fence_regs(acc128[c]);
      if (Cfg::kN64) wgmma_fence_regs(acc64);
      if (Cfg::kN32) wgmma_fence_regs(acc32);
      if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);

      const int m_eff = args.reverse_m ? num_m - 1 - it.m_blk : it.m_blk;
      const int row0 = m_eff * BM + row_in_tile;
      const int col0 = it.n_blk * BN;
#pragma unroll
      for (int c = 0; c < Cfg::kN128; ++c)
        epilogue_frag<EPI, ACT>(args, acc128[c], row0, col0 + c * 128, lane, head_partial);
      if (Cfg::kN64) epilogue_frag<EPI, ACT>(args, acc64, row0, col0 + Cfg::kN128 * 128, lane, head_partial);
      if (Cfg::kN32) epilogue_frag<EPI, ACT>(args, acc32, row0, col0 + Cfg::kN128 * 128 + Cfg::kN64 * 64, lane, head_partial);

      if (EPI == EPI_MLP_HEAD && it.n_blk == num_n - 1) {
        // a row's columns live in the four lanes of a quad: combine them, then loss_reco -> confidence
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float s = head_partial[h];
          s += __shfl_xor_sync(0xffffffffu, s, 1);
          s += __shfl_xor_sync(0xffffffffu, s, 2);
          head_partial[h] = 0.f;
          const int row = row0 + 8 * h;
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
    }
  }
}

template <int BN, int EPI, int ACT>
int launch_gemm(const GemmArgs& a, const CUtensorMap& ta, const CUtensorMap& tb, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
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
  kern<<<grid, kNumThreads, Cfg::kSmemBytes, stream>>>(ta, tb, a);
  prof_end(PROF_GEMM, stream);
  WVN_CHECK_LAUNCH("gemm_bf16_kernel");
  return WVN_OK;
}

template <int BN>
int dispatch_epi(const GemmArgs& a, const CUtensorMap& ta, const CUtensorMap& tb, cudaStream_t s) {
  switch (a.epi) {
    case EPI_BF16:
      if (a.act == ACT_NONE) return launch_gemm<BN, EPI_BF16, ACT_NONE>(a, ta, tb, s);
      if (a.act == ACT_RELU) return launch_gemm<BN, EPI_BF16, ACT_RELU>(a, ta, tb, s);
      if (a.act == ACT_GELU) return launch_gemm<BN, EPI_BF16, ACT_GELU>(a, ta, tb, s);
      break;
    case EPI_F32:
      if (a.act == ACT_NONE) return launch_gemm<BN, EPI_F32, ACT_NONE>(a, ta, tb, s);
      break;
    case EPI_RESID_F32:
      if (a.act == ACT_NONE) return launch_gemm<BN, EPI_RESID_F32, ACT_NONE>(a, ta, tb, s);
      break;
    case EPI_PATCH:
      if (a.act == ACT_NONE) return launch_gemm<BN, EPI_PATCH, ACT_NONE>(a, ta, tb, s);
      break;
    case EPI_QKV:
      if (a.act == ACT_NONE) return launch_gemm<BN, EPI_QKV, ACT_NONE>(a, ta, tb, s);
      break;
    case EPI_MLP_HEAD:
      if (a.act == ACT_NONE) return launch_gemm<BN, EPI_MLP_HEAD, ACT_NONE>(a, ta, tb, s);
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
  WVN_REQUIRE(a.K % BK == 0, "gemm: K=%d must be a multiple of %d (pad the operands)", a.K, BK);
  if (block_n == 0) block_n = pick_block_n(a.N);
  WVN_REQUIRE(block_n == 64 || block_n == 128 || block_n == 192 || block_n == 224 || block_n == 256,
              "gemm: bad block_n %d", block_n);
  WVN_REQUIRE(a.N % block_n == 0, "gemm: N=%d must be a multiple of block_n=%d (pad the weights)", a.N, block_n);
  if (a.epi == EPI_MLP_HEAD)
    WVN_REQUIRE(a.feat > 0 && a.trav_col % 32 == 0 && a.trav_col >= a.feat && a.trav_col < a.N && a.x != nullptr &&
                    a.trav != nullptr && a.conf != nullptr && a.cg_mean != nullptr && a.cg_std != nullptr &&
                    a.ldx % 8 == 0 && a.ldx >= a.trav_col,
                "gemm: bad MLP-head epilogue arguments (feat=%d trav_col=%d N=%d)", a.feat, a.trav_col, a.N);
  if (a.epi == EPI_QKV)
    WVN_REQUIRE(a.dim % 64 == 0 && a.N == 3 * a.dim && a.heads * 64 == a.dim && a.npad % 8 == 0,
                "gemm: bad QKV epilogue geometry (dim=%d heads=%d npad=%d N=%d)", a.dim, a.heads, a.npad, a.N);
  if (a.epi == EPI_F32 || a.epi == EPI_RESID_F32) WVN_REQUIRE(a.ldo % 4 == 0, "gemm: fp32 output pitch must be a multiple of 4");
  if (a.epi == EPI_BF16) WVN_REQUIRE(a.ldo % 8 == 0, "gemm: bf16 output pitch must be a multiple of 8");
  CUtensorMap ta, tb;
  WVN_PROPAGATE(make_tmap_bf16_2d(&ta, A, a.K, a.M, static_cast<uint64_t>(lda) * 2, BK, BM));
  WVN_PROPAGATE(make_tmap_bf16_2d(&tb, W, a.K, a.N, static_cast<uint64_t>(a.K) * 2, BK, block_n));
  switch (block_n) {
    case 64: return dispatch_epi<64>(a, ta, tb, stream);
    case 128: return dispatch_epi<128>(a, ta, tb, stream);
    case 192: return dispatch_epi<192>(a, ta, tb, stream);
    case 224: return dispatch_epi<224>(a, ta, tb, stream);
    case 256: return dispatch_epi<256>(a, ta, tb, stream);
  }
  return set_error(WVN_ERR_INVALID, "gemm: unreachable");
}

}  // namespace wvn
