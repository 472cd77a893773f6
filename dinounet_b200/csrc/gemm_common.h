// Shared between the GEMM host API (gemm_api.cu) and the persistent wgmma kernel family (gemm_tc2.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include "../../include/dinounet_b200.h"

namespace b2u {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 x 16-bit = 128 B = one swizzle row

struct alignas(64) GemmMaps {
  CUtensorMap a[4];
  CUtensorMap b;
};

struct GemmArgs {
  int M, N;
  int num_kb;
  int n_tiles;
  int m_tiles;
  int conv;  // 0 plain, 1 3x3 s1, 2 3x3 s2
  int cb;    // channel blocks per tap
  int Ho, Wo;
  int TW, TH, tiles_x, tiles_y;
  b2u_epilogue epi;
  // QKV epilogue
  int ntok, D, heads, prefix, head_dim;
  const float* rope_sin;
  const float* rope_cos;
  void* q;
  void* k;
  void* v;
  int npad;  // > 0: V is written transposed as V^T [B, heads, 64, npad]
  int rope_h, rope_w;  // > 0: separable rope tables staged in smem
  int res_prefetch; // 1: the epilogue pulls the NEXT tile's residual rows into L2 while it drains the current tile
};

int num_sms();
int gemm_v2_dispatch_bf16(bool qkv, int bn, const GemmMaps& maps, const GemmArgs& args, cudaStream_t stream);
int gemm_v2_dispatch_f16(bool qkv, int bn, const GemmMaps& maps, const GemmArgs& args, cudaStream_t stream);
inline int gemm_v2_dispatch(bool qkv, int bn, int dtype, const GemmMaps& maps, const GemmArgs& args, cudaStream_t stream) {
  return dtype == B2U_BF16 ? gemm_v2_dispatch_bf16(qkv, bn, maps, args, stream)
                           : gemm_v2_dispatch_f16(qkv, bn, maps, args, stream);
}
int get_option(int key);

}  // namespace b2u
