// Common device helpers for the sm_90a kernels: mbarrier / TMA PTX wrappers, 16-bit type traits.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2u {

// ---------------------------------------------------------------- 16-bit element traits
template <typename T> struct T16;
template <> struct T16<__nv_bfloat16> {
  static constexpr int kFmt = 1;  // = B2U_BF16 (wgmma_ss / wgmma_rs kind)
  __device__ static __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
  __device__ static __forceinline__ __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
  __device__ static __forceinline__ uint32_t pack2(float a, float b) {
    __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&t);
  }
  __device__ static __forceinline__ float2 unpack2(uint32_t u) {
    __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&u);
    return __bfloat1622float2(t);
  }
};
template <> struct T16<__half> {
  static constexpr int kFmt = 0;  // = B2U_F16
  __device__ static __forceinline__ float to_f(__half v) { return __half2float(v); }
  __device__ static __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
  __device__ static __forceinline__ uint32_t pack2(float a, float b) {
    __half2 t = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&t);
  }
  __device__ static __forceinline__ float2 unpack2(uint32_t u) {
    __half2 t = *reinterpret_cast<__half2*>(&u);
    return __half22float2(t);
  }
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- programmatic dependent launch (see host_util.h)
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// Elementwise kernels: wait only.  (Triggering the dependents at kernel START was measured: -3.6 % - hundreds of early
// blocks of the next kernel sit on the SMs next to the running one; the implicit trigger at block exit is kept instead.)
__device__ __forceinline__ void pdl_begin() { pdl_wait(); }

// ---------------------------------------------------------------- per-warpgroup register budget (sm_90a setmaxnreg)
// Every warp of the warpgroup must execute it.  `dec` returns registers to the CTA's pool, `inc` waits until the pool holds
// enough: the budgets of all warpgroups may not sum past what the kernel was launched with.
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// (B2U_MBAR_HINT_NS: try_wait with a suspend-time hint.  Measured with 20 us: GEMMs unchanged, attention 240.7 -> 265.5 us
// per layer - the wake-up is slower than the default poll - so the default build does not define it.)
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t addr = smem_u32(bar);
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
#ifdef B2U_MBAR_HINT_NS
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n"
#else
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
#endif
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(addr),
      "r"(parity)
#ifdef B2U_MBAR_HINT_NS
      , "r"(static_cast<uint32_t>(B2U_MBAR_HINT_NS))
#endif
      : "memory");
}

// non-blocking probe: true once the phase with this parity has completed
__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}

// One elected lane of a fully converged warp (PTX elect.sync).  Unlike `lane == 0`, the compiler KNOWS that exactly one
// thread executes the guarded region, so uniform-datapath instructions (UTMALDG) are emitted straight instead of inside a
// waterfall loop each.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "elect.sync _|p, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- TMA (cp.async.bulk.tensor)
__device__ __forceinline__ void tma_prefetch_desc(const void* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::
          "r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const void* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// fp32 pair arithmetic (two lanes of a float2; sm_90 has no packed f32x2 instructions, so each is two scalar ones)
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

}  // namespace b2u
