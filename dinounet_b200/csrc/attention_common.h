// Shared by the attention translation units (attention_tc.cu: host entry points + few-row companion, attention_tc3.cu: kernel).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace b2u {

struct alignas(64) AttnMaps {
  CUtensorMap q, k, vt;
};
struct AttnArgs {
  int BH, heads, ntok, nchunks;
  int q_begin;      // first query row handled by this launch (rows [q_begin, ntok)); keys always span [0, ntok)
  int qtiles;       // 128-row query tiles per (batch, head)
  long long items;  // BH * qtiles: one CTA each
  float scale_log2e;
  void* out;
};

__device__ __forceinline__ void tma_load_3d(void* smem_dst, const void* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::
          "r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void sts128a(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ uint4 lds128a(uint32_t addr) {
  uint4 r;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr) : "memory");
  return r;
}
__device__ __forceinline__ float ex2(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

int attention_tc3_dispatch(const AttnMaps& maps, const AttnArgs& a, int head_dim, int dtype, cudaStream_t stream);

}  // namespace b2u
