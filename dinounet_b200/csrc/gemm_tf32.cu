// TF32 tensor-core GEMM (sm_90a wgmma kind tf32) for the TRAINING path: same parameter block, addressing modes and epilogue
// as b2u_f32_gemm (csrc/fp32_tier.cu) - plain / transposed rows, the 3x3 window of an NHWC image on the A side (conv
// forward, conv data gradient) or on the W side (conv weight gradient, K = output pixels), row remap, 2x2 pixel shuffle,
// split-K atomics - but the products run on the tensor cores: fp32 operands rounded to TF32 (cvt.rna: 10 mantissa bits,
// the mantissa width of the fp16 autocast the reference trains under, nnUNetTrainer.py:899-929, with fp32's exponent
// range), fp32 accumulation.  The fp32 SIMT kernel stays the parity tier (1e-5); this one is the fast tier of the train
// step, whose time the SIMT GEMM dominates.
//
// Why register-path loaders instead of TMA: five of the eight operand modes are gathers that no tensor map expresses
// without a transposed copy in HBM (A[k][m], W[k][n], flipped 3x3 weights, the per-pixel window with K = pixel index).
// Every mode is therefore loaded with ordinary global loads - 16-byte ones where the mode is K-contiguous; for the
// convolution gradients' row-contiguous operands 4 x 4 blocks (four LDG.128 along the rows, transposed in registers:
// tf32::Roles in gemm_tf32_addr.h) - rounded to TF32 in registers and written to shared memory in exactly the layout a SWIZZLE_128B K-major tensor map would produce
// (row r of a k-block = 128 B = 32 floats; 16-byte chunk c of row r lives at r*128 + ((c ^ (r & 7)) << 4)), so the
// wgmma descriptors are the 16-bit GEMM's (make_gdesc_k128; +32 B per K = 8 step).
//
// CTA = one 128 x BN output tile of one K slice (grid = tiles (n fastest) x ksplit), 256 threads = two warpgroups of 64
// tile rows each, 3-stage smem ring:
//   all threads: st.shared the k-block fetched kPF iterations earlier -> fence.proxy.async -> issue the global loads of
//   k-block kb + kPF into the freed register set (in flight across kPF barriers) -> __syncthreads -> each warpgroup issues
//   4 x wgmma m64nBNk8 on its rows and waits until at most this k-block's group is in flight, so a stage is rewritten
//   only after the MMAs of two iterations earlier have completed.
// Epilogue: the accumulator fragments go through the (then idle) ring as a row-major fp32 tile, thread = accumulator row.
// Two CTAs fit an SM's shared memory (60-96 KB each).
#include <math.h>

#include "common.cuh"
#include "../../include/dinounet_b200.h"
#include "gemm_tf32_addr.h"
#include "wgmma.cuh"
#include "host_util.h"

namespace b2u {
namespace {

using namespace tf32;

// A/B knobs (python csrc/build.py with B2U_EXTRA_FLAGS): register prefetch depth in k-blocks, resident CTAs per SM
#ifndef B2U_TF32_PF
#define B2U_TF32_PF 1
#endif
#ifndef B2U_TF32_MINB
#define B2U_TF32_MINB 2
#endif
constexpr int kPF = B2U_TF32_PF;
static_assert(kPF >= 1 && kPF <= kTStages, "a k-block is stored into the ring before its register set is refilled");

template <int BN> struct TfCfg {
  static constexpr int kABytes = kTM * 128;
  static constexpr int kBBytes = BN * 128;
  static constexpr int kStage = kABytes + kBBytes;
  static constexpr int kAccRow = BN + 4;               // fp32 accumulator tile row stride (+16 B: conflict-free row reads)
  static_assert(kTM * kAccRow * 4 <= kTStages * kStage, "the accumulator tile reuses the ring");
  static constexpr int kSmem = kTStages * kStage + 1024;   // + alignment slack
};

__device__ __forceinline__ uint32_t to_tf32(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return r;
}
struct SmemPut {            // tf32::stage's sink: round to TF32, one 16-byte shared-memory store
  uint32_t base;
  __device__ __forceinline__ void operator()(uint32_t off, float4 v) const {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(base + off), "r"(to_tf32(v.x)), "r"(to_tf32(v.y)), "r"(to_tf32(v.z)),
                 "r"(to_tf32(v.w))
                 : "memory");
  }
};

// ABLK / WBLK: staging shape of the two operands (tf32::pick_modes), compile-time so that each instantiation carries only
// its own loader (a runtime switch cost the row-mode shapes 6-15 %)
template <int BN, bool ABLK, bool WBLK>
__global__ void __launch_bounds__(kTThreads, B2U_TF32_MINB) gemm_tf32_kernel(const b2u_f32_gemm_params p) {
  using C = TfCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  int k_lo, k_hi;
  k_slice(p, static_cast<int>(blockIdx.z), k_lo, k_hi);
  if (k_lo >= k_hi) return;                            // empty K slice (uniform per CTA): nothing to add
  const int nkb = (k_hi - k_lo + kTK - 1) / kTK;

  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t smem_base = smem_u32(smem);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;                            // MMA: tile rows [64 wg, 64 wg + 64)
  long long m0;
  int n0;
  tile_origin(p, BN, static_cast<long long>(blockIdx.x), m0, n0);

  const Roles R = make_roles(p, tid, m0, n0, BN, ABLK, WBLK);   // this thread's rows / chunks of the two operand tiles
  constexpr int kWN = BN / 32;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;

  // kPF register sets: k-block kb lives in set kb % kPF from the moment its loads are issued (kPF iterations ahead) until it
  // is stored to the ring.  Default 1: the kernel is bound by L2->SM operand bytes (32 FLOP per operand byte of a 128 x 128
  // fp32 tile), not by load latency, and deeper prefetch costs registers at two CTAs per SM.
  float4 ra[kPF][4], rw[kPF][4];
#pragma unroll
  for (int u = 0; u < kPF; ++u) {
    const int kh = u < nkb ? k_hi : 0;                 // beyond the slice: fetch_* return zeros without touching memory
    fetch_a<ABLK>(p, R, k_lo + u * kTK, kh, ra[u]);
    fetch_w<WBLK, kWN>(p, R, k_lo + u * kTK, kh, rw[u]);
  }

  for (int kb0 = 0; kb0 < nkb; kb0 += kPF) {
#pragma unroll
    for (int u = 0; u < kPF; ++u) {
      const int kb = kb0 + u;
      if (kb >= nkb) break;                            // uniform over the CTA
      const int s = kb % kTStages;                     // free: every warpgroup has waited for the MMAs of k-block kb - 2
      const uint32_t sbase = smem_base + static_cast<uint32_t>(s) * C::kStage;
      stage<ABLK, 4>(R.a_r, R.a_c0, true, ra[u], SmemPut{sbase});
      stage<WBLK, kWN>(R.w_r, R.w_c0, R.w_n != 0, rw[u], SmemPut{sbase + C::kABytes});
      fence_proxy_async();                             // generic-proxy writes -> visible to the wgmma async proxy
      if (kb + kPF < nkb) {                            // refill this register set: in flight across kPF barriers / MMA issues
        fetch_a<ABLK>(p, R, k_lo + (kb + kPF) * kTK, k_hi, ra[u]);
        fetch_w<WBLK, kWN>(p, R, k_lo + (kb + kPF) * kTK, k_hi, rw[u]);
      }
      __syncthreads();
      {
        const uint64_t da = make_gdesc_k128(sbase + static_cast<uint32_t>(wg * 64 * 128));
        const uint64_t db = make_gdesc_k128(sbase + C::kABytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kTK / 8; ++k)
          wgmma_ss<2, BN>(acc, da + static_cast<uint64_t>(k * 2), db + static_cast<uint64_t>(k * 2), (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
      }
    }
  }

  // ---------------------------------------------------------------- epilogue: thread = accumulator row
  wgmma_wait<0>();
  __syncthreads();                                     // every MMA has read its stage: the ring holds the accumulator tile
  float* s_acc = reinterpret_cast<float*>(smem);       // [kTM][kAccRow]
  {
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int c = 8 * j + 2 * (lane & 3);
      *reinterpret_cast<float2*>(s_acc + r0 * C::kAccRow + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(s_acc + (r0 + 8) * C::kAccRow + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
  __syncthreads();
  {
    const int q = warp & 3, half = warp >> 2;          // rows [32 q, 32 q + 32), column half
    constexpr int kCols = BN / 2;
    const int row = q * 32 + lane;
    const EpiRow e = make_epi_row(p, m0 + row);
    const float* src = s_acc + row * C::kAccRow + half * kCols;
#pragma unroll 1
    for (int c0 = 0; c0 < kCols; c0 += 4) {
      const float4 v = *reinterpret_cast<const float4*>(src + c0);
      const float a4[4] = {v.x, v.y, v.z, v.w};
      emit4(p, e, n0 + half * kCols + c0, a4);
    }
  }
}

template <int BN, bool ABLK, bool WBLK>
int launch_tf32(const b2u_f32_gemm_params& p, cudaStream_t stream) {
  auto kern = gemm_tf32_kernel<BN, ABLK, WBLK>;
  static bool configured_dev[64] = {};
  bool& configured = configured_dev[current_device_index()];
  constexpr int kSmem = TfCfg<BN>::kSmem;
  static_assert(kSmem <= 113 * 1024, "two CTAs per SM must fit in shared memory");
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
    if (e != cudaSuccess) return set_error(-2, "cudaFuncSetAttribute(gemm_tf32): %s", cudaGetErrorString(e));
    configured = true;
  }
  const long long tiles = ((p.M + kTM - 1) / kTM) * ((p.N + BN - 1) / BN);
  if (tiles > 0x7fffffffLL) return set_error(-1, "b2u_tf32_gemm: too many output tiles");
  dim3 grid(static_cast<unsigned>(tiles), 1, p.ksplit > 1 ? p.ksplit : 1);
  kern<<<grid, kTThreads, kSmem, stream>>>(p);
  return check_launch("tf32_gemm");
}

}  // namespace

extern "C" int b2u_tf32_gemm(const b2u_f32_gemm_params* p, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (const char* why = tf32::validate(p)) return set_error(-1, "b2u_tf32_gemm: %s", why);
  bool a_blk, w_blk;
  tf32::pick_modes(*p, a_blk, w_blk);
  const int mode = a_blk ? 2 : (w_blk ? 1 : 0);        // a_blk implies w_blk
  switch (tf32::pick_bn(p->N) + mode) {
    case 32: return launch_tf32<32, false, false>(*p, stream);
    case 33: return launch_tf32<32, false, true>(*p, stream);
    case 34: return launch_tf32<32, true, true>(*p, stream);
    case 64: return launch_tf32<64, false, false>(*p, stream);
    case 65: return launch_tf32<64, false, true>(*p, stream);
    case 66: return launch_tf32<64, true, true>(*p, stream);
    case 128: return launch_tf32<128, false, false>(*p, stream);
    case 129: return launch_tf32<128, false, true>(*p, stream);
    default: return launch_tf32<128, true, true>(*p, stream);
  }
}

}  // namespace b2u
