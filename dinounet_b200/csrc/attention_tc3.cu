// Flash attention on the sm_90a warpgroup MMA for the DINOv3 ViT (head_dim 64 / 128, non-causal, ntok = 1029 at 512^2).
// Replaces F.scaled_dot_product_attention at dinounet/dinov3/layers/attention.py:116 (math: :106-118).
//
// Persistent CTAs, one per SM.  Tiles of 64 x kConsumers query rows of one (batch, head) are handed out statically,
// query tile fastest, so that the CTAs resident at one time read the same heads' K / V^T out of L2.
//   warpgroup 0  : TMA producer (setmaxnreg down to 24; one elected thread): the tile's Q into a 2-deep ring (the next
//                  tile's Q lands while the current one finishes), then {K chunk [128 keys x HD], V^T chunk [HD x 128 keys]}
//                  into a ring of kStages stages shared by the consumers.
//   warpgroups 1..: kConsumers consumers of 64 query rows each (setmaxnreg up to kConsumerRegs).  Per key chunk j:
//                    S(j) = Q K_j^T       wgmma m64nWk16, both operands in shared memory, S in registers
//                    O += P(j-1) V_{j-1}  wgmma m64nHDk16 with P as the REGISTER A operand (the accumulator fragment of S
//                                         for 16 key columns is the A fragment of one K = 16 step)
//                    softmax of S(j)      overlaps the PV MMA: wgmma_wait<1> retires S(j) only; P(j) is packed after
//                                         wgmma_wait<0> has retired PV(j-1), which also releases that K/V stage.
//   The consumers issue their MMAs in turn (a ring of named barriers), so that softmax runs while another warpgroup's MMAs
//   occupy the tensor pipe.  At head_dim 64 one warpgroup's softmax takes longer than another's MMAs, so three consumers
//   (192-row tiles, 160 registers each) keep two softmaxes under every warpgroup's MMAs: measured 339 against 394 us with
//   two consumers (32 x 16 x 1029, bf16, H100 80GB at 700 W).  head_dim 128 doubles the MMA work per chunk and needs 240
//   registers for S, O and P, so it keeps two consumers on 128-row tiles.
// Exponentials: the running maximum is updated lazily - kept while a chunk raises it by at most 8 (log2 domain), so P <= 2^8
// stays finite in both 16-bit types and the O rescale is skipped on most chunks.  Every exp2 runs on MUFU: moving every 3rd
// (or 4th) one to the FMA pipe as a degree-3 polynomial was measured slower at head_dim 64 on H100 80GB at 700 W (421 / 414 against
// 407 us at 32 x 16 x 1029, bf16) - the softmax is bound by instruction issue, not by the MUFU rate.
// Key tail: only the last chunk is masked.  It runs QK^T at the next instantiated width >= its valid keys (16/32/64/128;
// ntok = 1029: 5 keys -> n16) and PV with K = 16 steps over that width; K rows past ntok are zero-filled by TMA and the V^T
// padding columns are zero (callers zero [ntok, npad), TMA zero-fills past npad), so masked P = 0 meets finite V.
// Query tail: a consumer whose 64 rows all lie at or past ntok skips its MMAs and softmax and only keeps the barrier protocol.
// Every shared-memory operand is K-major SW128; V is consumed as V^T [B,H,HD,npad] (written transposed by the QKV epilogue).
#include "common.cuh"
#include "../../include/dinounet_b200.h"
#include "host_util.h"
#include "gemm_common.h"
#include "attention_common.h"
#include "wgmma.cuh"

namespace b2u {

template <int HD> struct AttCfg {
  static constexpr int kStages = HD == 64 ? 3 : 2;          // K/V ring depth: what 227 KB of shared memory holds
  static constexpr int kKB = HD / 64;                       // 64-wide K blocks of the head dim
  static constexpr int kConsumers = HD == 64 ? 3 : 2;       // consumer warpgroups of 64 query rows each
  static constexpr int kRows = 64 * kConsumers;             // query rows per tile
  static constexpr int kQBytes = kRows * HD * 2;            // kKB blocks of [kRows rows x 64 dims]
  static constexpr int kKBytes = 128 * HD * 2;              // kKB blocks of [128 keys x 64 dims]
  static constexpr int kVBytes = 2 * HD * 128;              // two key blocks of [HD rows x 64 keys]
  static constexpr int kConsumerWarps = 4 * kConsumers;
  static constexpr int kThreads = 128 * (kConsumers + 1);   // producer warpgroup + the consumer warpgroups
  // setmaxnreg budgets: 128 x 24 + 128 x kConsumers x kConsumerRegs stays within the 64 K registers of the SM
  static constexpr int kConsumerRegs = kConsumers == 3 ? 160 : 240;
  static constexpr int kSmem = 2 * kQBytes + kStages * (kKBytes + kVBytes) + 1024 + 256;
};

__device__ __forceinline__ void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

template <int N> struct IntC { static constexpr int value = N; };

template <typename T, int HD>
__global__ void __launch_bounds__(AttCfg<HD>::kThreads, 1) attn_tc3_kernel(const __grid_constant__ AttnMaps maps, const AttnArgs args) {
  using TT = T16<T>;
  using CF = AttCfg<HD>;
  constexpr int KB = CF::kKB, NST = CF::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                               // [2][kQBytes]
  uint8_t* sK = sQ + 2 * CF::kQBytes;               // [stages][kKBytes]
  uint8_t* sV = sK + NST * CF::kKBytes;             // [stages][kVBytes]
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sV + NST * CF::kVBytes);   // [2]
  uint64_t* q_empty = q_full + 2;                   // [2]
  uint64_t* kv_full = q_empty + 2;                  // [NST]
  uint64_t* kv_empty = kv_full + NST;               // [NST]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&maps.q);
    tma_prefetch_desc(&maps.k);
    tma_prefetch_desc(&maps.vt);
    for (int b = 0; b < 2; ++b) { mbar_init(&q_full[b], 1); mbar_init(&q_empty[b], CF::kConsumerWarps); }
    for (int s = 0; s < NST; ++s) { mbar_init(&kv_full[s], 1); mbar_init(&kv_empty[s], CF::kConsumerWarps); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();                              // prologue done: wait for the QKV kernel's q / k / v^T
  const int J = args.nchunks;
  const int tail_valid = args.ntok - (J - 1) * 128;          // valid keys of the last chunk, 1..128
  const int items = static_cast<int>(args.items);            // the launcher checks that it fits

  if (warp < 4) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<24>();
    if (warp == 0 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      int it = 0;
      for (int t = blockIdx.x; t < items; t += gridDim.x, ++it) {
        const int bh = t / args.qtiles;
        const int q0 = args.q_begin + (t - bh * args.qtiles) * CF::kRows;
        const int qb = it & 1;
        mbar_wait(&q_empty[qb], ((it >> 1) & 1) ^ 1);
        mbar_expect_tx(&q_full[qb], CF::kQBytes);
        for (int kb = 0; kb < KB; ++kb) tma_load_3d(sQ + qb * CF::kQBytes + kb * (CF::kRows * 128), &maps.q, &q_full[qb], kb * 64, q0, bh);
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
    }
  } else {
    // ===================== consumer warpgroups =====================
    setmaxnreg_inc<CF::kConsumerRegs>();
    constexpr int NC = CF::kConsumers;
    const int cw = (warp >> 2) - 1;                          // consumer cw: query rows [64 cw, 64 cw + 64) of the tile
    const int bar_own = 1 + cw, bar_other = 1 + (cw + 1) % NC;   // turns in a ring: wait on our barrier, release the next
    const float sl2 = args.scale_log2e;
    if (cw == NC - 1) named_bar_arrive(1, 256);              // consumer 0 issues first
    int stage = 0, pstage = 0;                               // K/V stage of chunk j / of chunk j - 1 (read by PV(j-1))
    uint32_t phase = 0;
    int it = 0;
    for (int t = blockIdx.x; t < items; t += gridDim.x, ++it) {
      const int bh = t / args.qtiles;
      const int q0 = args.q_begin + (t - bh * args.qtiles) * CF::kRows;
      const int qb = it & 1;
      mbar_wait(&q_full[qb], (it >> 1) & 1);
      if (q0 + cw * 64 >= args.ntok) {
        // all 64 rows past ntok: keep the ping-pong turns and the K/V releases (after the stage has been filled, so the
        // arrivals count toward this round of the ring) and nothing else
        for (int j = 0; j < J; ++j) {
          mbar_wait(&kv_full[stage], phase);
          named_bar_sync(bar_own, 256);
          named_bar_arrive(bar_other, 256);
          if (lane == 0) mbar_arrive(&kv_empty[stage]);
          if (++stage == NST) { stage = 0; phase ^= 1; }
        }
        if (lane == 0) mbar_arrive(&q_empty[qb]);
        continue;
      }
      float o[HD / 2];
#pragma unroll
      for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
      float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows lane/4 and lane/4 + 8 of this warp's 16
      float corr0 = 1.f, corr1 = 1.f;                       // O rescale owed before the next PV
      bool rescale = false;                                  // warp-uniform: some row of this warp owes one
      uint32_t pa[8][4];                                     // P(j-1) as the A fragments of the 8 K = 16 steps
      const uint32_t qaddr = smem_u32(sQ + qb * CF::kQBytes + cw * 64 * 128);

      // O *= corr for the rows whose maximum moved on the last chunk (PV(j-2) has retired: O is ours)
      auto rescale_o = [&]() {
        if (rescale) {
#pragma unroll
          for (int c = 0; c < HD / 8; ++c) {
            o[4 * c] *= corr0; o[4 * c + 1] *= corr0;
            o[4 * c + 2] *= corr1; o[4 * c + 3] *= corr1;
          }
        }
      };
      // O += P(j-1) V_{j-1}: K = 16 steps over the first NW keys of the chunk
      auto issue_pv = [&](auto nw_tag) {
        constexpr int NW = decltype(nw_tag)::value;
#pragma unroll
        for (int t8 = 0; t8 < NW / 16; ++t8) {
          const uint64_t db = make_gdesc_k128(smem_u32(sV + pstage * CF::kVBytes + (t8 >> 2) * (HD * 128)));
          wgmma_rs<TT::kFmt, HD>(o, pa[t8], db + static_cast<uint64_t>((t8 & 3) * 2), 1u);
        }
        wgmma_commit();
      };
      // One key chunk j: S(j) and PV(j-1) issued in our turn, softmax(j) under PV(j-1).  NW: MMA width of S(j);
      // MASK: the last chunk (keys >= lim are masked, P = 0 exactly); FIRST: j = 0, no PV(j-1).  Every wgmma of a
      // variant is unconditional: a wgmma behind a runtime branch makes ptxas serialise the whole pipeline.
      auto chunk = [&](auto nw_tag, auto mask_tag, auto first_tag, int lim) {
        constexpr int NW = decltype(nw_tag)::value;
        constexpr bool MASK = decltype(mask_tag)::value != 0, FIRST = decltype(first_tag)::value != 0;
        if constexpr (!FIRST) rescale_o();
        float s[NW / 2];
        mbar_wait(&kv_full[stage], phase);
        named_bar_sync(bar_own, 256);
        wgmma_fence_operand(o);
        wgmma_fence();
#pragma unroll
        for (int kb = 0; kb < KB; ++kb) {
          const uint64_t da = make_gdesc_k128(qaddr + kb * (CF::kRows * 128));
          const uint64_t db = make_gdesc_k128(smem_u32(sK + stage * CF::kKBytes + kb * (128 * 128)));
#pragma unroll
          for (int k = 0; k < 4; ++k)
            wgmma_ss<TT::kFmt, NW>(s, da + static_cast<uint64_t>(k * 2), db + static_cast<uint64_t>(k * 2), (kb | k) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        if constexpr (!FIRST) issue_pv(IntC<128>{});
        named_bar_arrive(bar_other, 256);
        if constexpr (FIRST) wgmma_wait<0>();
        else wgmma_wait<1>();
        wgmma_fence_operand(s);
        // ---- online softmax.  s[4c + {0,1}]: row 0, keys 8c + 2(lane%4) + {0,1}; s[4c + {2,3}]: row 1, same keys
        if constexpr (MASK) {
#pragma unroll
          for (int c = 0; c < NW / 8; ++c) {
            const int key = 8 * c + 2 * (lane & 3);
            s[4 * c] = key < lim ? s[4 * c] : -INFINITY;
            s[4 * c + 2] = key < lim ? s[4 * c + 2] : -INFINITY;
            s[4 * c + 1] = key + 1 < lim ? s[4 * c + 1] : -INFINITY;
            s[4 * c + 3] = key + 1 < lim ? s[4 * c + 3] : -INFINITY;
          }
        }
        float mx0 = s[0], mx1 = s[2], mx0b = s[1], mx1b = s[3];   // two chains per row
#pragma unroll
        for (int c = 1; c < NW / 8; ++c) {
          mx0 = fmaxf(mx0, s[4 * c]); mx0b = fmaxf(mx0b, s[4 * c + 1]);
          mx1 = fmaxf(mx1, s[4 * c + 2]); mx1b = fmaxf(mx1b, s[4 * c + 3]);
        }
        mx0 = fmaxf(mx0, mx0b);
        mx1 = fmaxf(mx1, mx1b);
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        // lazy maximum: keep the reference while exp2 stays <= 2^8 (chunk 0 always has valid keys: m becomes finite)
        const float mc0 = fmaxf(m0, mx0 * sl2), mc1 = fmaxf(m1, mx1 * sl2);
        const bool need0 = mc0 - m0 > 8.0f, need1 = mc1 - m1 > 8.0f;
        corr0 = need0 ? ex2(m0 - mc0) : 1.f;                // 0 on the first chunk
        corr1 = need1 ? ex2(m1 - mc1) : 1.f;
        if (need0) m0 = mc0;
        if (need1) m1 = mc1;
        rescale = !FIRST && __any_sync(0xffffffffu, need0 || need1);
        float rs0 = 0.f, rs1 = 0.f, rs0b = 0.f, rs1b = 0.f;
#pragma unroll
        for (int c = 0; c < NW / 8; ++c) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int i = 4 * c + e;
            const float x = fmaf(s[i], sl2, e < 2 ? -m0 : -m1);
            s[i] = ex2(x);                                   // masked keys: ex2(-inf) = 0
          }
          rs0 += s[4 * c]; rs0b += s[4 * c + 1];
          rs1 += s[4 * c + 2]; rs1b += s[4 * c + 3];
        }
        l0 = l0 * corr0 + (rs0 + rs0b);                      // per-lane partial sums of the un-rounded probabilities
        l1 = l1 * corr1 + (rs1 + rs1b);
        if constexpr (!FIRST) {
          wgmma_wait<0>();                                   // PV(j-1) retired: its K/V stage and P registers are free
          wgmma_fence_operand(o);
          if (lane == 0) mbar_arrive(&kv_empty[pstage]);
        }
#pragma unroll
        for (int c = 0; c < NW / 8; ++c) {
          pa[c >> 1][(c & 1) * 2] = TT::pack2(s[4 * c], s[4 * c + 1]);
          pa[c >> 1][(c & 1) * 2 + 1] = TT::pack2(s[4 * c + 2], s[4 * c + 3]);
        }
        pstage = stage;
        if (++stage == NST) { stage = 0; phase ^= 1; }
      };
      // the last chunk's PV, over the K = 16 steps of its MMA width
      auto last_pv = [&](auto nw_tag) {
        rescale_o();
        wgmma_fence_operand(o);
        wgmma_fence();
        issue_pv(nw_tag);
        wgmma_wait<0>();
        wgmma_fence_operand(o);
        if (lane == 0) mbar_arrive(&kv_empty[pstage]);
      };

      if (J == 1) {                                          // ntok <= 128: one masked chunk, nothing to prefetch
        chunk(IntC<128>{}, IntC<1>{}, IntC<1>{}, tail_valid);
        last_pv(IntC<128>{});
      } else {
        chunk(IntC<128>{}, IntC<0>{}, IntC<1>{}, 128);
        for (int j = 1; j + 1 < J; ++j) chunk(IntC<128>{}, IntC<0>{}, IntC<0>{}, 128);
        if (tail_valid <= 16) { chunk(IntC<16>{}, IntC<1>{}, IntC<0>{}, tail_valid); last_pv(IntC<16>{}); }
        else if (tail_valid <= 32) { chunk(IntC<32>{}, IntC<1>{}, IntC<0>{}, tail_valid); last_pv(IntC<32>{}); }
        else if (tail_valid <= 64) { chunk(IntC<64>{}, IntC<1>{}, IntC<0>{}, tail_valid); last_pv(IntC<64>{}); }
        else { chunk(IntC<128>{}, IntC<1>{}, IntC<0>{}, tail_valid); last_pv(IntC<128>{}); }
      }
      if (lane == 0) mbar_arrive(&q_empty[qb]);
      // ---- normalise and store: rows q0 + 64 cw + 16 (warp % 4) + lane / 4 (+ 8), head dims 8c + 2 (lane % 4) + {0, 1}
      l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
      l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
      const float inv0 = 1.f / l0, inv1 = 1.f / l1;
      const int b = bh / args.heads, hd = bh - b * args.heads;
      const int D = args.heads * HD;
      const int t0 = q0 + cw * 64 + (warp & 3) * 16 + (lane >> 2), t1 = t0 + 8;
      T* outp = reinterpret_cast<T*>(args.out) + static_cast<long long>(b) * args.ntok * D + hd * HD + 2 * (lane & 3);
#pragma unroll
      for (int c = 0; c < HD / 8; ++c) {
        if (t0 < args.ntok)
          *reinterpret_cast<uint32_t*>(outp + static_cast<long long>(t0) * D + 8 * c) = TT::pack2(o[4 * c] * inv0, o[4 * c + 1] * inv0);
        if (t1 < args.ntok)
          *reinterpret_cast<uint32_t*>(outp + static_cast<long long>(t1) * D + 8 * c) = TT::pack2(o[4 * c + 2] * inv1, o[4 * c + 3] * inv1);
      }
    }
    if (cw == 0) named_bar_sync(1, 256);                     // consume the last consumer's final hand-over
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
  const int grid = static_cast<int>(std::min<long long>(a.items, num_sms()));
  launch_pdl(kern, grid, CF::kThreads, CF::kSmem, stream, maps, a);
  return check_launch("attention_tc3");
}

int attention_tc3_tile_rows(int head_dim) { return head_dim == 64 ? AttCfg<64>::kRows : AttCfg<128>::kRows; }

int attention_tc3_dispatch(const AttnMaps& maps, const AttnArgs& a, int head_dim, int dtype, cudaStream_t stream) {
  const bool bf = dtype == B2U_BF16;
  if (head_dim == 64) return bf ? launch_attn_tc3<__nv_bfloat16, 64>(maps, a, stream) : launch_attn_tc3<__half, 64>(maps, a, stream);
  return bf ? launch_attn_tc3<__nv_bfloat16, 128>(maps, a, stream) : launch_attn_tc3<__half, 128>(maps, a, stream);
}

}  // namespace b2u
