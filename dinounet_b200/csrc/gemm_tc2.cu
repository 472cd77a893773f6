// Warp-specialised persistent GEMM / implicit-GEMM 3x3 convolution on the sm_90a warpgroup MMA (wgmma), fp16 / bf16
// operands, fp32 accumulation.
//
//   grid = min(#tiles, #SMs) CTAs of 640 threads, one per SM, each looping over 128 x BN output tiles (n fastest, so the
//   CTAs running concurrently share A rows through L2):
//     warps 16-19: TMA producer warpgroup (one elected thread issues) - a ring of {A 128x64, W BNx64} 128B-swizzled
//                  k-blocks (as many stages as shared memory holds next to the accumulator tile: 3-8)
//     warps 8-15 : two MMA warpgroups, 64 tile rows each: wgmma m64nBNk16 straight from the ring (one k-block stays in
//                  flight while the previous stage is released), then the accumulator fragments go to a row-major fp32
//                  tile in shared memory (s_acc)
//     warps 0-7  : two epilogue warpgroups run the fused epilogue on s_acc with one thread per tile row: per-column
//                  parameters are per-lane constants, and a swizzled 4 KB patch per warp transposes the result for fully
//                  coalesced 16 B loads / stores (residual / skip tensors / output).
//   s_acc is handed over with two mbarriers: acc_full (fragments stored) and acc_empty (every epilogue thread has loaded
//   its last columns).  The MMA warps wait for acc_empty only when the next tile's main loop is done, so the epilogue of
//   tile t runs while the tensor cores work on tile t+1.  setmaxnreg moves registers from the producer (32) to the
//   epilogue (128); the MMA warps keep the 96 of the launch.
//   Convolution mode: A tiles are 4-D TMA boxes of the NHWC image (9 taps x channel blocks, OOB = zero padding).
#include "common.cuh"
#include "../../include/dinounet_b200.h"
#include "host_util.h"
#include "gemm_common.h"
#include "wgmma.cuh"

namespace b2u {

constexpr int kRopeBytes = 128 * 32 * 2 * 4;   // (rope_h + rope_w) rows x (<=32 angles x {sin, cos} fp32 + 16 B pad): host-checked
constexpr int kSmemMax = 227 * 1024;           // dynamic shared memory of one CTA on sm_90

template <int BN, int EPI = 0> struct Cfg2 {
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kAccBytes = BM * BN * 4;           // the fp32 accumulator tile handed to the epilogue
  static constexpr int kStagingBytes = 8 * 4096;          // 8 epilogue warps x (32 rows x 128 B)
  static constexpr int kBiasBytes = BN * 4;
  static constexpr int kRope = EPI == 2 ? kRopeBytes : 0;
  static constexpr int kFixed = kAccBytes + kStagingBytes + kBiasBytes + kRope + 1024 /*align*/ + 256 /*barriers*/;
  static constexpr int kStages = (kSmemMax - kFixed) / kStageBytes > 8 ? 8 : (kSmemMax - kFixed) / kStageBytes;
  static constexpr int kSmem = kStages * kStageBytes + kFixed;
  static constexpr int kEpiWarps = 8;                          // warps 0-7: two epilogue warpgroups
  static constexpr int kMmaWarps = 8;                          // warps 8-15: two MMA warpgroups
  static constexpr int kThreads = 32 * (kEpiWarps + kMmaWarps) + 128;   // + the producer warpgroup (warps 16-19)
  // Registers per thread of each role (setmaxnreg).  The launch gives every thread 65536 / 640 -> 96, and the warpgroups
  // only trade registers among themselves: 32 + 2 x 96 + 2 x 128 = 5 x 96.
  static constexpr int kRegLaunch = 96;
  static constexpr int kRegProducer = 32;
  static constexpr int kRegMma = 96;
  static constexpr int kRegEpi = 128;
  static_assert(kRegProducer + 2 * kRegMma + 2 * kRegEpi <= 5 * kRegLaunch, "register budget");
  static_assert(kStages >= 3, "shared-memory budget");
};

// byte offset of accumulator (row, col) in the fp32 tile: 16-byte chunk c of a row sits at chunk c ^ (row & 7) of its
// 128-byte group, so that both the fragment stores and the row-per-thread loads of 8 consecutive rows spread over all banks
template <int BN>
__device__ __forceinline__ uint32_t acc_off(int row, int col) {
  return static_cast<uint32_t>(row * (BN * 4) + ((((col >> 2) ^ (row & 7))) << 4) + ((col & 3) << 2));
}
// 32 consecutive accumulator columns of one tile row
template <int BN>
__device__ __forceinline__ void acc_ld32_t(uint32_t base, int row, int col, uint32_t (&v)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint32_t a = base + acc_off<BN>(row, col + 4 * i);
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v[4 * i]), "=r"(v[4 * i + 1]), "=r"(v[4 * i + 2]), "=r"(v[4 * i + 3]) : "r"(a) : "memory");
  }
}
#define acc_ld32(base, row, col, v) acc_ld32_t<BN>(base, row, col, v)

template <int kEpiThreads = 256>
__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kEpiThreads) : "memory"); }

__device__ __forceinline__ void sts128(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 r;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr) : "memory");
  return r;
}
__device__ __forceinline__ float4 lds128f(uint32_t addr) {
  const uint4 r = lds128(addr);
  return make_float4(__uint_as_float(r.x), __uint_as_float(r.y), __uint_as_float(r.z), __uint_as_float(r.w));
}
__device__ __forceinline__ float rcp_approx(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

__device__ __forceinline__ float ex2_approx(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// erf via Abramowitz-Stegun 7.1.26 (|abs err| <= 1.5e-7): branch-free, 2 MUFU + 11 FMA-pipe instructions.  Constants
// are folded (z = |x|/sqrt2 never materialises) and exp goes straight to ex2.approx.ftz: __expf() wraps it in a
// compare / pre-scale / square sequence for arguments below -126 that costs 3 more instructions per element, and an
// underflow to zero is exactly what erf -> 1 wants here.
__device__ __forceinline__ float gelu_fast(float x) {
  const float t = rcp_approx(fmaf(0.3275911f * 0.70710678118654752440f, fabsf(x), 1.0f));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float e = ex2_approx((x * x) * (-0.5f * 1.4426950408889634f));   // exp(-x^2/2)
  const float er = fmaf(-(p * t), e, 1.0f);                                // erf(|x|/sqrt2)
  const float h = 0.5f * x;
  return fmaf(h, copysignf(er, x), h);
}

// the same for the two values of a float2
__device__ __forceinline__ float2 gelu_fast2(float2 x) {
  const float2 ax = make_float2(fabsf(x.x), fabsf(x.y));
  const float2 u = fma2(make_float2(0.3275911f * 0.70710678118654752440f, 0.3275911f * 0.70710678118654752440f), ax, make_float2(1.0f, 1.0f));
  const float2 t = make_float2(rcp_approx(u.x), rcp_approx(u.y));
  float2 p = fma2(make_float2(1.061405429f, 1.061405429f), t, make_float2(-1.453152027f, -1.453152027f));
  p = fma2(p, t, make_float2(1.421413741f, 1.421413741f));
  p = fma2(p, t, make_float2(-0.284496736f, -0.284496736f));
  p = fma2(p, t, make_float2(0.254829592f, 0.254829592f));
  const float2 q = mul2(mul2(x, x), make_float2(-0.5f * 1.4426950408889634f, -0.5f * 1.4426950408889634f));
  const float2 e = make_float2(ex2_approx(q.x), ex2_approx(q.y));
  const float2 pt = mul2(p, t);
  const float2 er = fma2(make_float2(-pt.x, -pt.y), e, make_float2(1.0f, 1.0f));       // erf(|x|/sqrt2)
  const float2 h = mul2(x, make_float2(0.5f, 0.5f));
  return fma2(h, make_float2(copysignf(er.x, x.x), copysignf(er.y, x.y)), h);
}

// a pair of fp32 values rounded to the 16-bit type and back (what the reference's autocast Linear hands the next op)
template <typename TT>
__device__ __forceinline__ float2 round16v(float2 a) { return TT::unpack2(TT::pack2(a.x, a.y)); }

template <int ACT, int NV>
__device__ __forceinline__ void act_vec(float (&f)[NV]) {
  constexpr int act = ACT;
  if (act == B2U_ACT_GELU) {
#pragma unroll
    for (int j = 0; j < NV; j += 2) {
      const float2 r = gelu_fast2(make_float2(f[j], f[j + 1]));
      f[j] = r.x;
      f[j + 1] = r.y;
    }
  } else if (act == B2U_ACT_RELU) {
#pragma unroll
    for (int j = 0; j < NV; ++j) f[j] = fmaxf(f[j], 0.f);
  } else if (act == B2U_ACT_LRELU) {
#pragma unroll
    for (int j = 0; j < NV; ++j) f[j] = f[j] > 0.f ? f[j] : 0.01f * f[j];
  }
}

// EPI: 0 = generic 16-bit out, 1 = generic fp32 out, 2 = QKV(+RoPE, head split), 3 = SwiGLU (silu(x1)*x2).  ACT1 / ACT2:
// compile-time activations after the bias / after the affine (B2U_ACT_*), so the fully unrolled epilogue stays small enough
// for the I-cache.
template <int BN, int EPI, int ACT1, int ACT2, typename T>
__global__ void __launch_bounds__((Cfg2<BN, EPI>::kThreads), 1) gemm_tc2_kernel(const __grid_constant__ GemmMaps maps, const GemmArgs args) {
  using C = Cfg2<BN, EPI>;
  using TT = T16<T>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_acc = smem + C::kStages * C::kStageBytes;
  uint8_t* staging = s_acc + C::kAccBytes;
  float* s_bias = reinterpret_cast<float*>(staging + C::kStagingBytes);
  float* s_rope = reinterpret_cast<float*>(staging + C::kStagingBytes + C::kBiasBytes);   // [h+w][2*hq + 4] = (sin | cos | pad)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + C::kStagingBytes + C::kBiasBytes + C::kRope);
  uint64_t* empty_bar = full_bar + 8;
  uint64_t* acc_full = empty_bar + 8;    // s_acc holds a finished tile: every MMA thread has stored its fragments
  uint64_t* acc_empty = acc_full + 1;    // s_acc may be overwritten: every epilogue thread has loaded what it needs

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const long long total_tiles = static_cast<long long>(args.m_tiles) * args.n_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&maps.a[0]);
    tma_prefetch_desc(&maps.b);
    // a stage is free again once every MMA warp has seen the MMAs that read it complete
    for (int s = 0; s < 8; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], C::kMmaWarps); }
    mbar_init(acc_full, 32 * C::kMmaWarps);
    mbar_init(acc_empty, 32 * C::kEpiWarps);
    fence_mbar_init();
  }
  if constexpr (EPI == 2) {
    if (args.rope_w > 0) {
      // rows 0..h-1: the hq angles that depend on the patch row (table columns 0..hq-1 of patch (py, 0));
      // rows h..h+w-1: the hq angles that depend on the patch column (table columns hq..2hq-1 of patch (0, px))
      const int HDm = args.head_dim, hq = HDm >> 2;
      const int n = (args.rope_h + args.rope_w) * 2 * hq;
      for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int r = i / (2 * hq), c = i - r * 2 * hq;
        const bool is_cos = c >= hq;
        const int a = c - (is_cos ? hq : 0);
        const long long src = r < args.rope_h ? static_cast<long long>(r) * args.rope_w * HDm + a
                                              : static_cast<long long>(r - args.rope_h) * HDm + hq + a;
        s_rope[r * (2 * hq + 4) + c] = is_cos ? __ldg(args.rope_cos + src) : __ldg(args.rope_sin + src);   // rows padded by 16 B (below)
      }
    }
  }
  __syncthreads();
  pdl_wait();                              // barriers and tensor maps are set up: now wait for the producer kernel's data

  if (warp >= C::kEpiWarps + C::kMmaWarps) {
    // ===================== TMA producer: one elected thread of warp 16 =====================
    setmaxnreg_dec<C::kRegProducer>();
    if (warp == C::kEpiWarps + C::kMmaWarps && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int nt = static_cast<int>(tile % args.n_tiles);
        const int mt = static_cast<int>(tile / args.n_tiles);
        int img = 0, y0 = 0, x0 = 0;
        if (args.conv) {
          const int per_img = args.tiles_x * args.tiles_y;
          img = mt / per_img;
          const int r = mt - img * per_img;
          y0 = (r / args.tiles_x) * args.TH;
          x0 = (r % args.tiles_x) * args.TW;
        }
        for (int kb = 0; kb < args.num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sA = smem + stage * C::kStageBytes;
          uint8_t* sB = sA + C::kABytes;
          mbar_expect_tx(&full_bar[stage], C::kStageBytes);
          if (args.conv == 0) {
            tma_load_2d(sA, &maps.a[0], &full_bar[stage], kb * BK, mt * BM);
          } else {
            const int tap = kb / args.cb;
            const int c0 = (kb - tap * args.cb) * BK;
            const int dy = tap / 3, dx = tap - dy * 3;
            if (args.conv == 1) {
              tma_load_4d(sA, &maps.a[0], &full_bar[stage], c0, x0 + dx - 1, y0 + dy - 1, img);
            } else {
              const int py = (dy + 1) & 1, px = (dx + 1) & 1;
              tma_load_4d(sA, &maps.a[py * 2 + px], &full_bar[stage], c0, x0 + (dx == 0 ? -1 : 0),
                          y0 + (dy == 0 ? -1 : 0), img);
            }
          }
          tma_load_2d(sB, &maps.b, &full_bar[stage], kb * BK, nt * BN);
          if (++stage == C::kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp >= C::kEpiWarps) {
    // ===================== MMA warpgroups: main loop, then the fragments go to s_acc =====================
    if constexpr (C::kRegMma > C::kRegLaunch) setmaxnreg_inc<C::kRegMma>();
    else if constexpr (C::kRegMma < C::kRegLaunch) setmaxnreg_dec<C::kRegMma>();
    const int wg = (warp - C::kEpiWarps) >> 2;       // tile rows [64 wg, 64 wg + 64) of the MMA
    const int q4 = warp & 3;
    const uint32_t acc_u32 = smem_u32(s_acc);
    int stage = 0;
    uint32_t phase = 0, acc_phase = 0;
    for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < args.num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sA = smem_u32(smem + stage * C::kStageBytes);
        const uint64_t da = make_gdesc_k128(sA + wg * 64 * 128);
        const uint64_t db = make_gdesc_k128(sA + C::kABytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          wgmma_ss<TT::kFmt, BN>(acc, da + static_cast<uint64_t>(k * 2), db + static_cast<uint64_t>(k * 2), (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();                             // the previous k-block's MMAs are done: its stage may be refilled
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == C::kStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      // accumulator fragments -> s_acc (row-major fp32), once the previous tile's epilogue has loaded its part of it
      mbar_wait(acc_empty, acc_phase ^ 1);
      {
        const int r0 = wg * 64 + q4 * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int c = 8 * j + 2 * (lane & 3);
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(acc_u32 + acc_off<BN>(r0, c)), "f"(acc[4 * j]), "f"(acc[4 * j + 1]) : "memory");
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(acc_u32 + acc_off<BN>(r0 + 8, c)), "f"(acc[4 * j + 2]), "f"(acc[4 * j + 3]) : "memory");
        }
      }
      mbar_arrive(acc_full);
      acc_phase ^= 1;
    }
  } else {
    // ===================== epilogue warpgroups: the fused epilogue of the tile in s_acc =====================
    if constexpr (C::kRegEpi > C::kRegLaunch) setmaxnreg_inc<C::kRegEpi>();
    else if constexpr (C::kRegEpi < C::kRegLaunch) setmaxnreg_dec<C::kRegEpi>();
    const int q4 = warp & 3;                         // tile rows [32 q4, 32 q4 + 32), one per lane
    const int ew = warp;                             // staging patch index
    const int half = warp >> 2;                      // which half of the tile's columns this warp drains
    const int arow = q4 * 32 + lane;
    uint8_t* patch = staging + ew * 4096;
    const uint32_t patch_u32 = smem_u32(patch);
    const uint32_t acc_u32 = smem_u32(s_acc);
    const b2u_epilogue& e = args.epi;
    const int etid = threadIdx.x;                    // 0..255 among epilogue threads
    uint32_t acc_phase = 0;
    // s_acc back to the MMA warps: right after this thread's last load from it, so that the next tile's fragments can be
    // stored while the last columns are still being processed
    auto release_acc = [&]() { mbar_arrive(acc_empty); };
    for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int nt = static_cast<int>(tile % args.n_tiles);
      const int mt = static_cast<int>(tile / args.n_tiles);
      mbar_wait(acc_full, acc_phase);
      acc_phase ^= 1;
      const int n0 = nt * BN;
      int img = 0, y0 = 0, x0 = 0;
      if (args.conv) {
        const int per_img = args.tiles_x * args.tiles_y;
        img = mt / per_img;
        const int r = mt - img * per_img;
        y0 = (r / args.tiles_x) * args.TH;
        x0 = (r % args.tiles_x) * args.TW;
      }
      // logical row (token / pixel) of tile row `tr`, validity
      auto row_of = [&](int tr, long long& m) -> bool {
        if (args.conv == 0) {
          m = static_cast<long long>(mt) * BM + tr;
          return m < args.M;
        }
        const int ty = tr / args.TW, tx = tr - ty * args.TW;
        const int y = y0 + ty, x = x0 + tx;
        m = (static_cast<long long>(img) * args.Ho + y) * args.Wo + x;
        return (y < args.Ho) && (x < args.Wo);
      };


      if constexpr (EPI == 2) {
        // stage the (masked) bias of this tile's columns once
        epi_bar_sync();
        for (int i = etid; i < BN; i += 256) s_bias[i] = (e.bias && n0 + i < args.N) ? __ldg(e.bias + n0 + i) : 0.f;
        epi_bar_sync();
        const int HDm = args.head_dim;                 // 64 or 128
        const int hq = HDm >> 2;                       // angles per axis (rope_position_encoding.py: D_head / 4)
        // phase-1 owner row
        long long m1;
        const bool v1 = row_of(q4 * 32 + lane, m1);
        const unsigned ntok_u = static_cast<unsigned>(args.ntok);   // token rows fit 32 bits (host-checked): 32-bit divides
        const int b1 = static_cast<int>(static_cast<unsigned>(m1) / ntok_u);
        const int t1 = static_cast<int>(static_cast<unsigned>(m1) - static_cast<unsigned>(b1) * ntok_u);
        const bool rot = v1 && t1 >= args.prefix;
        const float* sinr = args.rope_sin + static_cast<long long>(rot ? t1 - args.prefix : 0) * HDm;
        const float* cosr = args.rope_cos + static_cast<long long>(rot ? t1 - args.prefix : 0) * HDm;
        // phase-2 rows of this lane: rr = i*4 + lane/8  (8 lanes x 16 B = the unit's two 64 B segments of a row)
        long long dst_off[8];
        bool dst_ok[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          long long m2;
          dst_ok[i] = row_of(q4 * 32 + i * 4 + (lane >> 3), m2);
          const int b2 = static_cast<int>(static_cast<unsigned>(m2) / ntok_u);
          const int t2 = static_cast<int>(static_cast<unsigned>(m2) - static_cast<unsigned>(b2) * ntok_u);
          dst_off[i] = (static_cast<long long>(b2) * args.heads * args.ntok + t2) * HDm;
        }
        // A "unit" = 64 accumulator columns = the 32 low + 32 matching high rope columns of one head:
        //   head_dim 64 : unit u = head u of the tile, lo = [0,32), hi = [32,64)
        //   head_dim 128: unit u = (head u/2, pass p = u&1), lo = [32p, 32p+32), hi = [64+32p, 64+32p+32)
#pragma unroll 1
        for (int u = half * (BN / 128); u < (half + 1) * (BN / 128); ++u) {
          const int hcol = HDm == 64 ? u * 64 : (u >> 1) * 128;          // first accumulator column of the head
          const int pss = HDm == 64 ? 0 : (u & 1);
          const int lo_off = pss * 32, hi_off = (HDm >> 1) + pss * 32;    // element offsets inside the head
          uint32_t v0[32], v1r[32];
          acc_ld32(acc_u32, arow, hcol + lo_off, v0);
          acc_ld32(acc_u32, arow, hcol + hi_off, v1r);
          if (u + 1 == (half + 1) * (BN / 128)) release_acc();
          const int n = n0 + hcol;
          if (n >= args.N) continue;   // warp-uniform
          const int which = n / args.D;
          const int head = (n - which * args.D) / HDm;
          float x[64];
#pragma unroll
          for (int j = 0; j < 32; j += 2) {   // Linear output rounded to 16 bits
            const float2 blo = *reinterpret_cast<const float2*>(&s_bias[hcol + lo_off + j]);
            const float2 bhi = *reinterpret_cast<const float2*>(&s_bias[hcol + hi_off + j]);
            const float2 alo = add2(make_float2(__uint_as_float(v0[j]), __uint_as_float(v0[j + 1])), blo);
            const float2 ahi = add2(make_float2(__uint_as_float(v1r[j]), __uint_as_float(v1r[j + 1])), bhi);
            const float2 lo = TT::unpack2(TT::pack2(alo.x, alo.y));
            const float2 hi = TT::unpack2(TT::pack2(ahi.x, ahi.y));
            x[j] = lo.x; x[j + 1] = lo.y;
            x[32 + j] = hi.x; x[33 + j] = hi.y;
          }
          if (which == 2 && args.npad > 0) {
            // V^T [B, heads, head_dim, npad]: lane = token, loop over d -> each store instruction writes 32 consecutive keys
            if (v1) {
              T* dst = reinterpret_cast<T*>(args.v) + (static_cast<long long>(b1) * args.heads + head) * HDm * args.npad + t1;
#pragma unroll
              for (int j = 0; j < 32; ++j) {
                dst[static_cast<long long>(lo_off + j) * args.npad] = TT::from_f(x[j]);
                dst[static_cast<long long>(hi_off + j) * args.npad] = TT::from_f(x[32 + j]);
              }
            }
            continue;   // warp-uniform
          }
          uint32_t packed[32];
          if (which < 2 && rot && args.rope_w > 0) {
            // separable tables from smem ([h + w] rows of (sin[hq] | cos[hq])): angle A < hq comes from the patch row's
            // table, A >= hq from the patch column's; cos/sin[A + head_dim/2] == cos/sin[A]
            const int pidx = t1 - args.prefix;
            const int py = pidx / args.rope_w, px = pidx - py * args.rope_w;
            // bytes per table row: + 16 B so that the 32 lanes (32 consecutive patch columns = 32 table rows) spread over all
            // banks; with the dense 128 B rows every LDS.128 of the column table was an 8-way bank conflict (ncu: short_sb 28 %)
            const uint32_t rstride = hq * 8 + 16;
            const uint32_t ry = smem_u32(s_rope) + py * rstride, rx = smem_u32(s_rope) + (args.rope_h + px) * rstride;
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              const int A = lo_off + j;                // angle index in [0, head_dim/2)
              const uint32_t rbase_ = (A < hq ? ry : rx) + (A & (hq - 1)) * 4;
              const float4 sn = lds128f(rbase_), cs = lds128f(rbase_ + hq * 4);
              // rotation: lo' = lo*cos - hi*sin, hi' = hi*cos + lo*sin (two angles per instruction)
              const float2 c01 = make_float2(cs.x, cs.y), c23 = make_float2(cs.z, cs.w);
              const float2 s01 = make_float2(sn.x, sn.y), s23 = make_float2(sn.z, sn.w);
              const float2 l01 = make_float2(x[j], x[j + 1]), l23 = make_float2(x[j + 2], x[j + 3]);
              const float2 h01 = make_float2(x[j + 32], x[j + 33]), h23 = make_float2(x[j + 34], x[j + 35]);
              const float2 a01 = fma2(l01, c01, mul2(h01, make_float2(-s01.x, -s01.y)));
              const float2 a23 = fma2(l23, c23, mul2(h23, make_float2(-s23.x, -s23.y)));
              const float2 b01 = fma2(h01, c01, mul2(l01, s01));
              const float2 b23 = fma2(h23, c23, mul2(l23, s23));
              packed[j / 2] = TT::pack2(a01.x, a01.y);
              packed[j / 2 + 1] = TT::pack2(a23.x, a23.y);
              packed[16 + j / 2] = TT::pack2(b01.x, b01.y);
              packed[16 + j / 2 + 1] = TT::pack2(b23.x, b23.y);
            }
          } else if (which < 2 && rot) {
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              const float4 c_lo = *reinterpret_cast<const float4*>(cosr + lo_off + j), s_lo = *reinterpret_cast<const float4*>(sinr + lo_off + j);
              const float4 c_hi = *reinterpret_cast<const float4*>(cosr + hi_off + j), s_hi = *reinterpret_cast<const float4*>(sinr + hi_off + j);
              packed[j / 2] = TT::pack2(x[j] * c_lo.x - x[j + 32] * s_lo.x, x[j + 1] * c_lo.y - x[j + 33] * s_lo.y);
              packed[j / 2 + 1] = TT::pack2(x[j + 2] * c_lo.z - x[j + 34] * s_lo.z, x[j + 3] * c_lo.w - x[j + 35] * s_lo.w);
              packed[16 + j / 2] = TT::pack2(x[j + 32] * c_hi.x + x[j] * s_hi.x, x[j + 33] * c_hi.y + x[j + 1] * s_hi.y);
              packed[16 + j / 2 + 1] = TT::pack2(x[j + 34] * c_hi.z + x[j + 2] * s_hi.z, x[j + 35] * c_hi.w + x[j + 3] * s_hi.w);
            }
          } else {
#pragma unroll
            for (int j = 0; j < 64; j += 2) packed[j / 2] = TT::pack2(x[j], x[j + 1]);
          }
          // stage: row = lane, 8 x 16 B chunks (4 of the lo segment, 4 of the hi segment), chunk position c ^ (row & 7)
          __syncwarp();
#pragma unroll
          for (int c = 0; c < 8; ++c)
            sts128(patch_u32 + lane * 128 + ((c ^ (lane & 7)) << 4), packed[4 * c], packed[4 * c + 1], packed[4 * c + 2], packed[4 * c + 3]);
          __syncwarp();
          T* base = reinterpret_cast<T*>(which == 0 ? args.q : (which == 1 ? args.k : args.v)) +
                    static_cast<long long>(head) * args.ntok * HDm + ((lane & 4) ? hi_off : lo_off) + (lane & 3) * 8;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int rr = i * 4 + (lane >> 3);
            const uint4 val = lds128(patch_u32 + rr * 128 + (((lane & 7) ^ (rr & 7)) << 4));
            if (dst_ok[i]) *reinterpret_cast<uint4*>(base + dst_off[i]) = val;
          }
        }
      } else if constexpr (EPI == 3) {
        // ---- SwiGLU (ffn_layers.py:73-77): the weight rows are packed in 32-row blocks [w1 block j | w2 block j], so the
        // accumulator columns come in 64-column groups (x1[32] | x2[32]); out[:, 32j..32j+31] = silu(x1 + b1) * (x2 + b2)
        // with the reference's 16-bit roundings (each Linear output, silu, the product).  Output is 16-bit [M, N/2].
        epi_bar_sync();
        for (int i = etid; i < BN; i += 256) s_bias[i] = (e.bias && n0 + i < args.N) ? __ldg(e.bias + n0 + i) : 0.f;
        epi_bar_sync();
        long long dst_row[4];
        bool dst_ok[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {             // phase-2 rows: rr = i*8 + lane/4 (4 lanes x 16 B = one 64 B row segment)
          long long m2;
          dst_ok[i] = row_of(q4 * 32 + i * 8 + (lane >> 2), m2);
          dst_row[i] = dst_ok[i] ? m2 : 0;
        }
#pragma unroll 1
        for (int g = half * (BN / 128); g < (half + 1) * (BN / 128); ++g) {
          uint32_t v0[32], v1r[32];
          acc_ld32(acc_u32, arow, g * 64, v0);
          acc_ld32(acc_u32, arow, g * 64 + 32, v1r);
          if (g + 1 == (half + 1) * (BN / 128)) release_acc();
          const int n = n0 + g * 64;
          if (n >= args.N) continue;   // warp-uniform
          uint32_t packed[16];
#pragma unroll
          for (int j = 0; j < 32; j += 2) {
            float h[2];
#pragma unroll
            for (int q = 0; q < 2; ++q) {
              const float a = TT::to_f(TT::from_f(__uint_as_float(v0[j + q]) + s_bias[g * 64 + j + q]));
              const float b = TT::to_f(TT::from_f(__uint_as_float(v1r[j + q]) + s_bias[g * 64 + 32 + j + q]));
              const float sg = TT::to_f(TT::from_f(a * rcp_approx(1.0f + ex2_approx(a * -1.4426950408889634f))));   // silu(a), 16-bit like F.silu
              h[q] = sg * b;
            }
            packed[j >> 1] = TT::pack2(h[0], h[1]);
          }
          // stage: row = lane, 64 B of output (4 x 16 B chunks) at chunk position c ^ ((row >> 1) & 3) within a 64 B slot
          __syncwarp();
#pragma unroll
          for (int c = 0; c < 4; ++c)
            sts128(patch_u32 + lane * 64 + ((c ^ ((lane >> 1) & 3)) << 4), packed[4 * c], packed[4 * c + 1], packed[4 * c + 2], packed[4 * c + 3]);
          __syncwarp();
          const int ocol = (n >> 1) + (lane & 3) * 8 + e.col_off;      // hidden column = accumulator column / 2
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int rr = i * 8 + (lane >> 2);
            const uint4 val = lds128(patch_u32 + rr * 64 + (((lane & 3) ^ ((rr >> 1) & 3)) << 4));
            if (dst_ok[i]) *reinterpret_cast<uint4*>(reinterpret_cast<T*>(e.out) + dst_row[i] * e.ldc + ocol) = val;
          }
        }
      } else {
        // ---- phase-2 row assignment: fp32 output -> 8 lanes per row (4 cols each), 4 rows per pass, 8 passes;
        //                              16-bit output -> 4 lanes per row (8 cols each), 8 rows per pass, 4 passes.
        constexpr bool o32 = (EPI == 1);
        if constexpr (BN >= 64) {
          // Short-K GEMMs with an fp32 residual stream (extractor out-proj / ffn2) are bound by the latency of these residual
          // loads.  Pull the NEXT tile's residual rows into L2 now, one tile ahead of their use.
          if (args.res_prefetch && e.residual != nullptr && args.conv == 0 && e.ps_cout == 0) {
            const long long nx = tile + gridDim.x;
            if (nx < total_tiles) {
              const int ntn = static_cast<int>(nx % args.n_tiles);
              const long long mtn = nx / args.n_tiles;
              const long long mn = mtn * BM + (etid >> 1);
              if (mn < args.M && (ntn + 1) * BN <= args.N) {
                long long row = mn;
                if (e.rows_in > 0) {
                  const long long qb = mn / e.rows_in;
                  row = qb * e.rows_out + e.row_off + (mn - qb * e.rows_in);
                }
                const char* pf = reinterpret_cast<const char*>(e.residual + row * e.ldres + ntn * BN + e.col_off) + (etid & 1) * (BN * 2);
#pragma unroll
                for (int l = 0; l < BN / 64; ++l) asm volatile("prefetch.global.L2 [%0];" ::"l"(pf + l * 128));
              }
            }
          }
        }
        const int lpr = o32 ? 8 : 4;                 // lanes per row
        const int rpp = 32 / lpr;                    // rows per pass
        const int npass = 32 / rpp;
        const int lcol = (lane % lpr) * (32 / lpr);  // first column (within the 32-col chunk) of this lane
        long long rbase[8];                          // output row index (or pixel-shuffle base) per pass
        bool rok[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          rok[i] = false;
          rbase[i] = 0;
          if (i < npass) {
            long long m;
            rok[i] = row_of(q4 * 32 + i * rpp + lane / lpr, m);
            if (!rok[i]) m = 0;   // keep addresses in bounds for the unconditional operand prefetch (stores stay predicated)
            const unsigned mu = static_cast<unsigned>(m);   // logical row counts fit 32 bits (checked on the host)
            if (e.ps_cout > 0) {
              const unsigned hw = static_cast<unsigned>(e.ps_h) * e.ps_w;
              const unsigned pb = mu / hw;
              const unsigned rem = mu - pb * hw;
              const unsigned pi = rem / e.ps_w, pj = rem - pi * e.ps_w;
              rbase[i] = (static_cast<long long>(pb) * (2 * e.ps_h) + 2 * pi) * (2 * e.ps_w) + 2 * pj;
            } else if (e.rows_in > 0) {
              const unsigned qb = mu / static_cast<unsigned>(e.rows_in);
              rbase[i] = static_cast<long long>(qb) * e.rows_out + e.row_off + (mu - qb * e.rows_in);
            } else {
              rbase[i] = m;
            }
          }
        }
        constexpr int kChunks = BN / 32;
        constexpr int kPerHalf = kChunks >= 2 ? kChunks / 2 : 1;
        const int ch_begin = kChunks >= 2 ? half * kPerHalf : 0;
        const int ch_end = kChunks >= 2 ? ch_begin + kPerHalf : (half == 0 ? 1 : 0);   // BN 32: the first warp set takes the only chunk
        if (ch_begin == ch_end) release_acc();
#pragma unroll 1
        for (int ch = ch_begin; ch < ch_end; ++ch) {
          uint32_t v[32];
          acc_ld32(acc_u32, arow, ch * 32, v);
          if (ch + 1 == ch_end) release_acc();
          const int n = n0 + ch * 32;
          if (n >= args.N) continue;   // warp-uniform
          // stage raw fp32 accumulators: row = lane, 8 x 16 B groups at position j ^ (row & 7).  Done before the operand
          // loads below so that v[] is dead by then, which keeps the epilogue inside its 128 registers.
          __syncwarp();
#pragma unroll
          for (int j = 0; j < 8; ++j)
            sts128(patch_u32 + lane * 128 + ((j ^ (lane & 7)) << 4), v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
          __syncwarp();
          int ocol = n + lcol;
          long long radd = 0;
          if (e.ps_cout > 0) {
            const int qd = n / e.ps_cout;
            ocol -= qd * e.ps_cout;
            radd = static_cast<long long>(qd >> 1) * (2 * e.ps_w) + (qd & 1);
          }
          ocol += e.col_off;
          // ---- prefetch residual / skip operands for every pass of this chunk
          float4 res[8];
          uint4 add[4];
          if (e.residual) {
            if (o32) {
#pragma unroll
              for (int i = 0; i < 8; ++i) res[i] = *reinterpret_cast<const float4*>(e.residual + (rbase[i] + radd) * e.ldres + ocol);
            } else {
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                res[2 * i] = *reinterpret_cast<const float4*>(e.residual + (rbase[i] + radd) * e.ldres + ocol);
                res[2 * i + 1] = *reinterpret_cast<const float4*>(e.residual + (rbase[i] + radd) * e.ldres + ocol + 4);
              }
            }
          }
          if (e.add16) {
            if (o32) {
#pragma unroll
              for (int i = 0; i < 4; ++i) {   // two passes per register (uint2 each)
                const uint2 a0 = *reinterpret_cast<const uint2*>(reinterpret_cast<const T*>(e.add16) + (rbase[2 * i] + radd) * e.ldadd + ocol);
                const uint2 a1 = *reinterpret_cast<const uint2*>(reinterpret_cast<const T*>(e.add16) + (rbase[2 * i + 1] + radd) * e.ldadd + ocol);
                add[i] = make_uint4(a0.x, a0.y, a1.x, a1.y);
              }
            } else {
#pragma unroll
              for (int i = 0; i < 4; ++i) add[i] = *reinterpret_cast<const uint4*>(reinterpret_cast<const T*>(e.add16) + (rbase[i] + radd) * e.ldadd + ocol);
            }
          }
          // per-column parameters of this lane (constant over the rows)
          constexpr int NV = o32 ? 4 : 8;
          const bool affine = e.scale != nullptr || e.shift != nullptr;   // warp-uniform
          float bi[NV], sc[NV], sh[NV];
#pragma unroll
          for (int j = 0; j < NV; ++j) { bi[j] = 0.f; sc[j] = 1.f; sh[j] = 0.f; }
#pragma unroll
          for (int h = 0; h < NV / 4; ++h) {
            if (e.bias) { const float4 t = __ldg(reinterpret_cast<const float4*>(e.bias + n + lcol + 4 * h)); bi[4 * h] = t.x; bi[4 * h + 1] = t.y; bi[4 * h + 2] = t.z; bi[4 * h + 3] = t.w; }
            if (e.scale) { const float4 t = __ldg(reinterpret_cast<const float4*>(e.scale + n + lcol + 4 * h)); sc[4 * h] = t.x; sc[4 * h + 1] = t.y; sc[4 * h + 2] = t.z; sc[4 * h + 3] = t.w; }
            if (e.shift) { const float4 t = __ldg(reinterpret_cast<const float4*>(e.shift + n + lcol + 4 * h)); sh[4 * h] = t.x; sh[4 * h + 1] = t.y; sh[4 * h + 2] = t.z; sh[4 * h + 3] = t.w; }
          }
          if constexpr (o32) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int rr = i * 4 + (lane >> 3);
              const float4 a4 = lds128f(patch_u32 + rr * 128 + (((lane & 7) ^ (rr & 7)) << 4));
              const float2 p01 = add2(make_float2(a4.x, a4.y), make_float2(bi[0], bi[1]));
              const float2 p23 = add2(make_float2(a4.z, a4.w), make_float2(bi[2], bi[3]));
              float f[4] = {p01.x, p01.y, p23.x, p23.y};
              if (e.round16) {
#pragma unroll
                for (int j = 0; j < 4; j += 2) {
                  const float2 t = TT::unpack2(TT::pack2(f[j], f[j + 1]));
                  f[j] = t.x;
                  f[j + 1] = t.y;
                }
              }
              act_vec<ACT1, 4>(f);
              if (affine) {
#pragma unroll
                for (int j = 0; j < 4; j += 2) {
                  const float2 t = fma2(make_float2(f[j], f[j + 1]), make_float2(sc[j], sc[j + 1]), make_float2(sh[j], sh[j + 1]));
                  f[j] = t.x; f[j + 1] = t.y;
                }
              }
              act_vec<ACT2, 4>(f);
              if (e.residual) {
                const float2 r01 = add2(make_float2(f[0], f[1]), make_float2(res[i].x, res[i].y));
                const float2 r23 = add2(make_float2(f[2], f[3]), make_float2(res[i].z, res[i].w));
                f[0] = r01.x; f[1] = r01.y; f[2] = r23.x; f[3] = r23.y;
              }
              if (e.add16) {
                const uint4 pr = add[i >> 1];
                const float2 t0 = TT::unpack2((i & 1) ? pr.z : pr.x), t1 = TT::unpack2((i & 1) ? pr.w : pr.y);
                f[0] += t0.x; f[1] += t0.y; f[2] += t1.x; f[3] += t1.y;
              }
              if (rok[i])
                *reinterpret_cast<float4*>(reinterpret_cast<float*>(e.out) + (rbase[i] + radd) * e.ldc + ocol) = make_float4(f[0], f[1], f[2], f[3]);
            }
          } else {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int rr = i * 8 + (lane >> 2);
              const int g0 = (lane & 3) * 2;
              const float4 a4 = lds128f(patch_u32 + rr * 128 + ((g0 ^ (rr & 7)) << 4));
              const float4 b4 = lds128f(patch_u32 + rr * 128 + (((g0 + 1) ^ (rr & 7)) << 4));
              float f[8] = {a4.x + bi[0], a4.y + bi[1], a4.z + bi[2], a4.w + bi[3], b4.x + bi[4], b4.y + bi[5], b4.z + bi[6], b4.w + bi[7]};
              if (e.round16) {   // packed convert: one F2FP per two values
#pragma unroll
                for (int j = 0; j < 8; j += 2) {
                  const float2 t = TT::unpack2(TT::pack2(f[j], f[j + 1]));
                  f[j] = t.x;
                  f[j + 1] = t.y;
                }
              }
              act_vec<ACT1, 8>(f);
              if (affine) {
#pragma unroll
                for (int j = 0; j < 8; ++j) f[j] = fmaf(f[j], sc[j], sh[j]);
              }
              act_vec<ACT2, 8>(f);
              if (e.residual) {
                f[0] += res[2 * i].x; f[1] += res[2 * i].y; f[2] += res[2 * i].z; f[3] += res[2 * i].w;
                f[4] += res[2 * i + 1].x; f[5] += res[2 * i + 1].y; f[6] += res[2 * i + 1].z; f[7] += res[2 * i + 1].w;
              }
              if (e.add16) {
                const float2 t0 = TT::unpack2(add[i].x), t1 = TT::unpack2(add[i].y), t2 = TT::unpack2(add[i].z), t3 = TT::unpack2(add[i].w);
                f[0] += t0.x; f[1] += t0.y; f[2] += t1.x; f[3] += t1.y; f[4] += t2.x; f[5] += t2.y; f[6] += t3.x; f[7] += t3.y;
              }
              if (rok[i])
                *reinterpret_cast<uint4*>(reinterpret_cast<T*>(e.out) + (rbase[i] + radd) * e.ldc + ocol) =
                    make_uint4(TT::pack2(f[0], f[1]), TT::pack2(f[2], f[3]), TT::pack2(f[4], f[5]), TT::pack2(f[6], f[7]));
            }
          }
        }
      }
    }
  }
  pdl_launch_dependents();   // this CTA's tiles are done: once every CTA is here the next kernel may start its prologue
}
#undef acc_ld32

// ------------------------------------------------------------------------------------------------ host side
template <int BN, int EPI, int ACT1, int ACT2, typename T>
static int launch_variant2(const GemmMaps& maps, const GemmArgs& args, cudaStream_t stream) {
  auto kern = gemm_tc2_kernel<BN, EPI, ACT1, ACT2, T>;
  using C = Cfg2<BN, EPI>;
  static bool configured_dev[64] = {};
  bool& configured = configured_dev[current_device_index()];
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmem);
    if (e != cudaSuccess) return set_error(-2, "cudaFuncSetAttribute(gemm_tc2): %s", cudaGetErrorString(e));
    configured = true;
  }
  const long long tiles = static_cast<long long>(args.m_tiles) * args.n_tiles;
  const int sms = num_sms();
  const int grid = static_cast<int>(tiles < sms ? tiles : sms);
  launch_pdl(kern, grid, C::kThreads, C::kSmem, stream, maps, args);
  return check_launch("gemm_tc2");
}

template <int BN, typename T>
static int dispatch_epi(bool qkv, const GemmMaps& maps, const GemmArgs& args, cudaStream_t stream) {
  if (qkv) {
    if constexpr (BN >= 128) return launch_variant2<BN, 2, 0, 0, T>(maps, args, stream);
    else return set_error(-3, "gemm_tc2: QKV epilogue needs BLOCK_N >= 128");
  }
  const int a1 = args.epi.act1, a2 = args.epi.act2;
  if (a1 == B2U_ACT_SWIGLU) {
    if constexpr (BN >= 128) {
      if (!args.epi.out_fp32 && a2 == 0) return launch_variant2<BN, 3, 0, 0, T>(maps, args, stream);
    }
    return set_error(-3, "gemm_tc2: SwiGLU epilogue needs BLOCK_N >= 128, a 16-bit output and no second activation");
  }
  if (args.epi.out_fp32) {
    if (a1 == 0 && a2 == 0) return launch_variant2<BN, 1, 0, 0, T>(maps, args, stream);
  } else {
    if (a1 == 0 && a2 == 0) return launch_variant2<BN, 0, 0, 0, T>(maps, args, stream);
    if (a1 == B2U_ACT_GELU && a2 == 0) {
      return launch_variant2<BN, 0, B2U_ACT_GELU, 0, T>(maps, args, stream);
    }
    if (a1 == 0 && a2 == B2U_ACT_RELU) return launch_variant2<BN, 0, 0, B2U_ACT_RELU, T>(maps, args, stream);
    if (a1 == 0 && a2 == B2U_ACT_LRELU) return launch_variant2<BN, 0, 0, B2U_ACT_LRELU, T>(maps, args, stream);
  }
  return set_error(-3, "gemm_tc2: epilogue combination (out_fp32=%d, act1=%d, act2=%d) is not instantiated",
                   args.epi.out_fp32, a1, a2);
}

template <typename T>
int gemm_v2_dispatch_t(bool qkv, int bn, const GemmMaps& maps, const GemmArgs& args, cudaStream_t stream) {
  if (args.M < 0) return set_error(-1, "gemm_tc2: M too large");
  switch (bn) {
    case 32: return dispatch_epi<32, T>(qkv, maps, args, stream);
    case 64: return dispatch_epi<64, T>(qkv, maps, args, stream);
    case 128: return dispatch_epi<128, T>(qkv, maps, args, stream);
    default: break;
  }
  return set_error(-3, "gemm_tc2: unsupported BLOCK_N %d", bn);
}

#ifndef B2U_GEMM2_TYPE
#error "compile gemm_tc2.cu once per 16-bit type with -DB2U_GEMM2_TYPE=0 (fp16) / 1 (bf16)"
#endif
#if B2U_GEMM2_TYPE == 1
int gemm_v2_dispatch_bf16(bool qkv, int bn, const GemmMaps& maps, const GemmArgs& args, cudaStream_t stream) {
  return gemm_v2_dispatch_t<__nv_bfloat16>(qkv, bn, maps, args, stream);
}
#else
int gemm_v2_dispatch_f16(bool qkv, int bn, const GemmMaps& maps, const GemmArgs& args, cudaStream_t stream) {
  return gemm_v2_dispatch_t<__half>(qkv, bn, maps, args, stream);
}
#endif

}  // namespace b2u
