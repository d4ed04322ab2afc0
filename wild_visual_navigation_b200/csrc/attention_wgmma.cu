// wvn-b200: fused non-causal multi-head attention (flash-style) on wgmma, head dim 64 (sm_90a).
//
// Replaces the materialised `softmax(q @ k^T * scale) @ v` of the DINO ViT blocks
// (SURVEY.md §8 a3 / K4): per (frame, head) the 3137x3137 (ViT-S/8 @448) score matrix is
// never written to HBM; S, P and O all live in registers: the bf16 P fragments are the A operand of
// P·V directly (the accumulator layout of S is the register-operand layout of wgmma) — no shared-memory round trip.
//
// Inputs (written by the QKV GEMM epilogue, bf16):
//   Q, K : [B*H, npad, 64]   row-major (K-major for the MMA)
//   V^T  : [B*H, 64, npad]   row-major (so P·V also sees a K-major B operand)
// Output: O [B, npad, H*64] bf16 (the layout the out-projection GEMM reads).
//
// One CTA = one 128-row query tile of one (frame, head), three warpgroups:
//   warpgroup 0    : one warp is the TMA producer (Q once; K / V^T tiles of 128 keys through a kStages ring); the
//                    warpgroup gives its registers up (setmaxnreg) to the consumers
//   warpgroups 1-2 : 64 query rows each.  Per KV tile: S = Q K^T (4 x wgmma m64n128k16, operands in shared memory),
//                    online softmax on the fragments (a row lives in the 4 lanes of a quad: 2 shuffles per reduction),
//                    O += P V (8 x wgmma m64n64k16 with P in registers).  P·V of tile j stays in flight while
//                    Q·K^T of tile j+1 is issued, and the two warpgroups run out of phase, so the tensor core works
//                    on one while the other is in its softmax.
// The padded last KV tile runs a separate, masked instantiation of the softmax, which keeps the other tiles free of
// mask arithmetic.
#include <stdlib.h>

#include "attention.h"
#include "common.cuh"
#include "host_common.h"

namespace wvn {

namespace {

constexpr int kThreads = 384;
constexpr int kConsumerWarps = 8;
constexpr int kTileQ = 128;
constexpr int kTileKV = 128;
constexpr int kDh = 64;
constexpr uint32_t kQBytes = kTileQ * kDh * 2;       // 16 KB
constexpr uint32_t kKBytes = kTileKV * kDh * 2;      // 16 KB
constexpr uint32_t kVBytes = kDh * kTileKV * 2;      // 16 KB (two 8 KB blocks of 64 keys)
constexpr int kStages = 4;                           // K / V^T ring depth
constexpr uint32_t kOffQ = 0;
constexpr uint32_t kOffK = kOffQ + kQBytes;
constexpr uint32_t kOffV = kOffK + kStages * kKBytes;
constexpr uint32_t kOffBar = kOffV + kStages * kVBytes;
constexpr uint32_t kSmemBytes = kOffBar + 256 + 1024 /*align slack*/;

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}

// One KV tile of the online softmax on a 64 x 128 score fragment: s[4 j + 2 h + e] is the score of query row h
// (of this thread's two) and key 8 j + 2 q + e.  Rescales o and l, leaves P (bf16 pairs, register-operand layout of
// the 8 k-steps of P·V) in p.  MASKED handles the padded last tile (keys >= valid are excluded).
template <bool MASKED>
__device__ __forceinline__ void softmax_tile(float (&s)[64], float (&o)[32], uint32_t (&p)[32], float (&m)[2], float (&l)[2],
                                             const float sl2, const int valid, const int q) {
  if (MASKED) {
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e)
        if (8 * j + 2 * q + e >= valid) s[4 * j + e] = s[4 * j + 2 + e] = -INFINITY;
  }
  float neg_m[2], alpha[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float mx = s[2 * h];
#pragma unroll
    for (int j = 0; j < 16; ++j) mx = fmaxf(mx, fmaxf(s[4 * j + 2 * h], s[4 * j + 2 * h + 1]));
    mx = fmaxf(quad_max(mx), m[h]);
    alpha[h] = fast_exp2((m[h] - mx) * sl2);
    m[h] = mx;
    neg_m[h] = -mx * sl2;
  }
  float sum[2] = {0.f, 0.f};
#pragma unroll
  for (int j = 0; j < 16; ++j) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float e0 = fast_exp2(fmaf(s[4 * j + 2 * h], sl2, neg_m[h]));
      const float e1 = fast_exp2(fmaf(s[4 * j + 2 * h + 1], sl2, neg_m[h]));
      sum[h] += e0 + e1;
      // k-step j / 2 of P·V: registers {row g | row g + 8} x {keys 2q.. | keys 2q + 8..}
      p[4 * (j >> 1) + 2 * (j & 1) + h] = pack_bf16x2(e0, e1);
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) l[h] = fmaf(l[h], alpha[h], sum[h]);   // per-thread partial; the quad is summed at the end
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    o[4 * j + 0] *= alpha[0];
    o[4 * j + 1] *= alpha[0];
    o[4 * j + 2] *= alpha[1];
    o[4 * j + 3] *= alpha[1];
  }
}

__global__ void __launch_bounds__(kThreads, 1)
attention_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                 const __grid_constant__ CUtensorMap tmap_v, const AttnArgs args) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBar);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;             // [kStages]  TMA -> consumers
  uint64_t* kv_empty = bars + 1 + kStages;  // [kStages]  consumers -> TMA (one arrival per consumer warp)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ntiles = args.npad / kTileQ;
  const int q_tile = args.reverse ? ntiles - 1 - static_cast<int>(blockIdx.x) : static_cast<int>(blockIdx.x);
  const int bh = args.reverse ? static_cast<int>(gridDim.y) - 1 - static_cast<int>(blockIdx.y) : static_cast<int>(blockIdx.y);
  const int num_kv = args.npad / kTileKV;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
    mbar_init(q_full, 1);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], kConsumerWarps);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (warp == 0) {
      if (elect_one_sync()) {
        mbar_arrive_expect_tx(q_full, kQBytes);
        tma_load_2d(&tmap_q, q_full, smem + kOffQ, 0, bh * args.npad + q_tile * kTileQ);
      }
      __syncwarp();
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < num_kv; ++j) {
        mbar_wait(&kv_empty[stage], phase ^ 1);
        if (elect_one_sync()) {
          mbar_arrive_expect_tx(&kv_full[stage], kKBytes + kVBytes);
          tma_load_2d(&tmap_k, &kv_full[stage], smem + kOffK + stage * kKBytes, 0, bh * args.npad + j * kTileKV);
          tma_load_2d(&tmap_v, &kv_full[stage], smem + kOffV + stage * kVBytes, j * kTileKV, bh * kDh);
          tma_load_2d(&tmap_v, &kv_full[stage], smem + kOffV + stage * kVBytes + kVBytes / 2, j * kTileKV + 64, bh * kDh);
        }
        __syncwarp();
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers: 64 query rows per warpgroup
    setmaxnreg_inc<232>();
    const int cwarp = warp - 4;
    const int wg = cwarp >> 2;
    const int q = lane & 3;
    const float sl2 = args.scale_log2;
    float s[64], o[32];
    uint32_t p[32];
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;

    mbar_wait(q_full, 0);
    const uint64_t desc_q = make_sw128_kmajor_desc(smem_u32(smem + kOffQ + wg * 64 * 128));
    int stage = 0, prev_stage = 0;
    uint32_t phase = 0;
    for (int j = 0; j < num_kv; ++j) {
      mbar_wait(&kv_full[stage], phase);
      const uint64_t desc_k = make_sw128_kmajor_desc(smem_u32(smem + kOffK + stage * kKBytes));
      wgmma_fence_regs(s);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kDh / 16; ++k) wgmma_m64n128k16_ss(s, desc_q + 2 * k, desc_k + 2 * k, k != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();  // S(j) is complete, and with it P·V(j-1): that tile's ring slot is free
      wgmma_fence_regs(s);
      wgmma_fence_regs(o);
      if (j > 0 && lane == 0) mbar_arrive(&kv_empty[prev_stage]);

      if (j == num_kv - 1) softmax_tile<true>(s, o, p, m, l, sl2, args.n_valid - j * kTileKV, q);
      else softmax_tile<false>(s, o, p, m, l, sl2, kTileKV, q);

      const uint32_t v_addr = smem_u32(smem + kOffV + stage * kVBytes);
      wgmma_fence_regs(o);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kTileKV / 16; ++k)
        wgmma_m64n64k16_rs(o, p[4 * k], p[4 * k + 1], p[4 * k + 2], p[4 * k + 3],
                           make_sw128_kmajor_desc(v_addr + (k >> 2) * (kVBytes / 2)) + 2 * (k & 3), 1u);
      wgmma_commit();
      prev_stage = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(o);

    // ---------------- O / l -> bf16 -> out[frame, row, head * 64 + col]
    const int frame = bh / args.heads, head = bh - frame * args.heads;
    const int row0 = q_tile * kTileQ + wg * 64 + (cwarp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float lt = l[h];
      lt += __shfl_xor_sync(0xffffffffu, lt, 1);
      lt += __shfl_xor_sync(0xffffffffu, lt, 2);
      const float inv = 1.f / lt;
      __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(args.out) +
                           (static_cast<long long>(frame) * args.npad + row0 + 8 * h) * args.ldo + head * kDh + 2 * q;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(dst + 8 * jj) = pack_bf16x2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
    }
  }
}

}  // namespace

int attention_bf16(const AttnArgs& a, const void* q, const void* k, const void* vt, cudaStream_t stream) {
  WVN_REQUIRE(a.batch > 0 && a.heads > 0, "attention: empty problem");
  WVN_REQUIRE(a.npad % kTileKV == 0 && a.n_valid > 0 && a.n_valid <= a.npad && a.n_valid > a.npad - kTileKV,
              "attention: npad=%d must be a multiple of 128 and n_valid=%d must lie in the last tile", a.npad,
              a.n_valid);
  const long long bh = static_cast<long long>(a.batch) * a.heads;
  WVN_REQUIRE(bh <= 65535, "attention: batch * heads = %lld exceeds the grid's y extent", bh);
  CUtensorMap tq, tk, tv;
  WVN_PROPAGATE(make_tmap_bf16_2d(&tq, q, kDh, bh * a.npad, kDh * 2, 64, kTileQ));
  WVN_PROPAGATE(make_tmap_bf16_2d(&tk, k, kDh, bh * a.npad, kDh * 2, 64, kTileKV));
  WVN_PROPAGATE(make_tmap_bf16_2d(&tv, vt, a.npad, bh * kDh, static_cast<uint64_t>(a.npad) * 2, 64, kDh));
  static bool attr_set = false;
  if (!attr_set) {
    WVN_CHECK_CUDA(cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    attr_set = true;
  }
  dim3 grid(a.npad / kTileQ, static_cast<unsigned>(bh));
  prof_begin(PROF_ATTENTION, stream);
  attention_kernel<<<grid, kThreads, kSmemBytes, stream>>>(tq, tk, tv, a);
  prof_end(PROF_ATTENTION, stream);
  WVN_CHECK_LAUNCH("attention_kernel");
  return WVN_OK;
}

}  // namespace wvn
