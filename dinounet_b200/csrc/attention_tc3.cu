// Flash attention on the sm_90a warpgroup MMA for the DINOv3 ViT (head_dim 64 / 128, non-causal, ntok = 1029 at 512^2).
// Replaces F.scaled_dot_product_attention at dinounet/dinov3/layers/attention.py:116 (math: :106-118).
//
// One CTA per (batch*head, 128-row query tile), 288 threads:
//   warp 8     : TMA producer - the Q tile once, then a 2-stage ring of {K chunk [128 keys x HD], V^T chunk [HD x 128 keys]}
//   warps 0-7  : two consumer warpgroups, 64 query rows each.  Per key chunk j:
//                  S = Q K_j^T        wgmma m64n128k16, both operands from shared memory, S in registers
//                  online softmax     row max over the 4 lanes that share a row, P = exp2(S * scale*log2(e) - m), O *= corr
//                  O += P V_j         wgmma m64nHDk16 with P as the REGISTER A operand: the accumulator fragment of S for
//                                     16 key columns is exactly the A fragment of one K = 16 step, so P never touches smem
//                and release the stage.  Scores of keys >= ntok are -inf (P = 0 exactly), so every chunk runs the same 8 PV
//                steps: the V^T padding is zero (callers zero it, TMA zero-fills past npad), and no wgmma sits in a branch.
// Occupancy: one CTA per SM.  The S, O and P fragments take 168 registers x 288 threads; two CTAs would need <= 113
// registers per thread, and at that cap (ptxas: 96) the fragments spill to local memory (0.8 KB at head_dim 64, 4 KB at
// 128).  The two consumer warpgroups run their chunks independently, so one's softmax can overlap the other's MMAs.
// Every shared-memory operand is K-major SW128; V is consumed as V^T [B,H,HD,npad] (written transposed by the QKV epilogue).
#include "common.cuh"
#include "../../include/dinounet_b200.h"
#include "host_util.h"
#include "gemm_common.h"
#include "attention_common.h"
#include "wgmma.cuh"

namespace b2u {

template <int HD> struct AttCfg {
  static constexpr int kStages = 2;
  static constexpr int kKB = HD / 64;                       // 64-wide K blocks of the head dim
  static constexpr int kQBytes = 128 * HD * 2;              // kKB blocks of [128 rows x 64 dims]
  static constexpr int kKBytes = 128 * HD * 2;              // kKB blocks of [128 keys x 64 dims]
  static constexpr int kVBytes = 2 * HD * 128;              // two key blocks of [HD rows x 64 keys]
  static constexpr int kConsumerWarps = 8;
  static constexpr int kThreads = 32 * kConsumerWarps + 32;
  static constexpr int kSmem = kQBytes + kStages * (kKBytes + kVBytes) + 1024 + 256;
};

template <typename T, int HD>
__global__ void __launch_bounds__(AttCfg<HD>::kThreads, 1) attn_tc3_kernel(const __grid_constant__ AttnMaps maps, const AttnArgs args) {
  using TT = T16<T>;
  using CF = AttCfg<HD>;
  constexpr int KB = CF::kKB, NST = CF::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + CF::kQBytes;                   // [stages][kKBytes]
  uint8_t* sV = sK + NST * CF::kKBytes;             // [stages][kVBytes]
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sV + NST * CF::kVBytes);
  uint64_t* kv_full = q_full + 1;                   // [NST]
  uint64_t* kv_empty = kv_full + NST;               // [NST]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&maps.q);
    tma_prefetch_desc(&maps.k);
    tma_prefetch_desc(&maps.vt);
    mbar_init(q_full, 1);
    for (int s = 0; s < NST; ++s) { mbar_init(&kv_full[s], 1); mbar_init(&kv_empty[s], CF::kConsumerWarps); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();                              // prologue done: wait for the QKV kernel's q / k / v^T
  const int bh = static_cast<int>(blockIdx.x / args.qtiles);
  const int q0 = args.q_begin + static_cast<int>(blockIdx.x - static_cast<long long>(bh) * args.qtiles) * 128;
  const int J = args.nchunks;
  const int tail_valid = args.ntok - (J - 1) * 128;          // valid keys of the last chunk, 1..128

  if (warp == CF::kConsumerWarps) {
    // ===================== TMA producer =====================
    if (elect_one()) {
      mbar_expect_tx(q_full, CF::kQBytes);
      for (int kb = 0; kb < KB; ++kb) tma_load_3d(sQ + kb * (128 * 128), &maps.q, q_full, kb * 64, q0, bh);
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < J; ++j) {
        mbar_wait(&kv_empty[stage], phase ^ 1);
        mbar_expect_tx(&kv_full[stage], CF::kKBytes + CF::kVBytes);
        for (int kb = 0; kb < KB; ++kb)
          tma_load_3d(sK + stage * CF::kKBytes + kb * (128 * 128), &maps.k, &kv_full[stage], kb * 64, j * 128, bh);
        tma_load_3d(sV + stage * CF::kVBytes, &maps.vt, &kv_full[stage], j * 128, 0, bh);
        tma_load_3d(sV + stage * CF::kVBytes + HD * 128, &maps.vt, &kv_full[stage], j * 128 + 64, 0, bh);
        if (++stage == NST) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ===================== consumer warpgroups =====================
    const int wg = warp >> 2;
    const float sl2 = args.scale_log2e;
    float o[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows lane/4 and lane/4 + 8 of this warp's 16
    mbar_wait(q_full, 0);
    int stage = 0;
    uint32_t phase = 0;
    for (int j = 0; j < J; ++j) {
      const int lim = j + 1 == J ? tail_valid : 128;       // valid keys of this chunk
      mbar_wait(&kv_full[stage], phase);
      float s[64];
      wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < KB; ++kb) {
        const uint64_t da = make_gdesc_k128(smem_u32(sQ + kb * (128 * 128) + wg * 64 * 128));
        const uint64_t db = make_gdesc_k128(smem_u32(sK + stage * CF::kKBytes + kb * (128 * 128)));
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_ss<TT::kFmt, 128>(s, da + static_cast<uint64_t>(k * 2), db + static_cast<uint64_t>(k * 2), (kb | k) != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      // ---- online softmax.  s[4c + {0,1}]: row 0, keys 8c + 2(lane%4) + {0,1}; s[4c + {2,3}]: row 1, same keys
#pragma unroll
      for (int c = 0; c < 16; ++c) {                        // selects, not branches
        const int key = 8 * c + 2 * (lane & 3);
        s[4 * c] = key < lim ? s[4 * c] : -INFINITY;
        s[4 * c + 2] = key < lim ? s[4 * c + 2] : -INFINITY;
        s[4 * c + 1] = key + 1 < lim ? s[4 * c + 1] : -INFINITY;
        s[4 * c + 3] = key + 1 < lim ? s[4 * c + 3] : -INFINITY;
      }
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int c = 0; c < 16; ++c) {
        mx0 = fmaxf(mx0, fmaxf(s[4 * c], s[4 * c + 1]));
        mx1 = fmaxf(mx1, fmaxf(s[4 * c + 2], s[4 * c + 3]));
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      const float mn0 = fmaxf(m0, mx0 * sl2), mn1 = fmaxf(m1, mx1 * sl2);   // chunk 0 always has valid keys -> finite
      const float corr0 = ex2(m0 - mn0), corr1 = ex2(m1 - mn1);             // 0 on the first chunk
      m0 = mn0;
      m1 = mn1;
      float rs0 = 0.f, rs1 = 0.f;
      uint32_t pa[8][4];                                    // P as the A fragments of the 8 K = 16 steps
#pragma unroll
      for (int c = 0; c < 16; ++c) {
        const float p0 = ex2(fmaf(s[4 * c], sl2, -mn0)), p1 = ex2(fmaf(s[4 * c + 1], sl2, -mn0));
        const float p2 = ex2(fmaf(s[4 * c + 2], sl2, -mn1)), p3 = ex2(fmaf(s[4 * c + 3], sl2, -mn1));
        rs0 += p0 + p1;
        rs1 += p2 + p3;
        pa[c >> 1][(c & 1) * 2] = TT::pack2(p0, p1);
        pa[c >> 1][(c & 1) * 2 + 1] = TT::pack2(p2, p3);
      }
      l0 = l0 * corr0 + rs0;                                // per-lane partial sums of the un-rounded probabilities
      l1 = l1 * corr1 + rs1;
#pragma unroll
      for (int c = 0; c < HD / 8; ++c) {
        o[4 * c] *= corr0; o[4 * c + 1] *= corr0;
        o[4 * c + 2] *= corr1; o[4 * c + 3] *= corr1;
      }
      // ---- O += P V_j
      wgmma_fence();
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const uint64_t db = make_gdesc_k128(smem_u32(sV + stage * CF::kVBytes + (t >> 2) * (HD * 128)));
        wgmma_rs<TT::kFmt, HD>(o, pa[t], db + static_cast<uint64_t>((t & 3) * 2), 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(&kv_empty[stage]);
      if (++stage == NST) { stage = 0; phase ^= 1; }
    }
    // ---- normalise and store: rows q0 + 64 wg + 16 (warp % 4) + lane / 4 (+ 8), head dims 8c + 2 (lane % 4) + {0, 1}
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float inv0 = 1.f / l0, inv1 = 1.f / l1;
    const int b = bh / args.heads, hd = bh - b * args.heads;
    const int D = args.heads * HD;
    const int t0 = q0 + wg * 64 + (warp & 3) * 16 + (lane >> 2), t1 = t0 + 8;
    T* outp = reinterpret_cast<T*>(args.out) + static_cast<long long>(b) * args.ntok * D + hd * HD + 2 * (lane & 3);
#pragma unroll
    for (int c = 0; c < HD / 8; ++c) {
      if (t0 < args.ntok)
        *reinterpret_cast<uint32_t*>(outp + static_cast<long long>(t0) * D + 8 * c) = TT::pack2(o[4 * c] * inv0, o[4 * c + 1] * inv0);
      if (t1 < args.ntok)
        *reinterpret_cast<uint32_t*>(outp + static_cast<long long>(t1) * D + 8 * c) = TT::pack2(o[4 * c + 2] * inv1, o[4 * c + 3] * inv1);
    }
  }
  pdl_launch_dependents();   // this CTA's rows are done
}

template <typename T, int HD>
static int launch_attn_tc3(const AttnMaps& maps, const AttnArgs& a, cudaStream_t stream) {
  auto kern = attn_tc3_kernel<T, HD>;
  using CF = AttCfg<HD>;
  static_assert(CF::kSmem <= 227 * 1024, "attention smem budget");
  static bool configured_dev[64] = {};
  bool& configured = configured_dev[current_device_index()];
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, CF::kSmem);
    if (e != cudaSuccess) return set_error(-2, "cudaFuncSetAttribute(attn_tc3): %s", cudaGetErrorString(e));
    configured = true;
  }
  if (a.items > 0x7fffffffLL) return set_error(-1, "b2u_attention_tc: too many query tiles");
  launch_pdl(kern, static_cast<int>(a.items), CF::kThreads, CF::kSmem, stream, maps, a);
  return check_launch("attention_tc3");
}

int attention_tc3_dispatch(const AttnMaps& maps, const AttnArgs& a, int head_dim, int dtype, cudaStream_t stream) {
  const bool bf = dtype == B2U_BF16;
  if (head_dim == 64) return bf ? launch_attn_tc3<__nv_bfloat16, 64>(maps, a, stream) : launch_attn_tc3<__half, 64>(maps, a, stream);
  return bf ? launch_attn_tc3<__nv_bfloat16, 128>(maps, a, stream) : launch_attn_tc3<__half, 128>(maps, a, stream);
}

}  // namespace b2u
