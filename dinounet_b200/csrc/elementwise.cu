// HBM-bound kernels of the Dino U-Net forward: LayerNorm, casts, patchify, stem conv, pooling, depthwise conv,
// InstanceNorm, adapter tail, FiLM, squeeze-excitation, segmentation head.  All tensors are channels-last; every thread
// moves 16-byte vectors (8 x 16-bit or 4 x fp32) along the channel dim so warps issue fully coalesced 128 B lines.
#include "common.cuh"
#include "../../include/dinounet_b200.h"
#include "host_util.h"
#include "gemm_common.h"

namespace b2u {

template <typename T> struct Vec8 {
  uint4 u;
  __device__ __forceinline__ void load(const T* p) { u = *reinterpret_cast<const uint4*>(p); }
  __device__ __forceinline__ void store(T* p) const { *reinterpret_cast<uint4*>(p) = u; }
  __device__ __forceinline__ void zero() { u = make_uint4(0u, 0u, 0u, 0u); }
  __device__ __forceinline__ void to_float(float (&f)[8]) const {
    float2 a = T16<T>::unpack2(u.x), b = T16<T>::unpack2(u.y), c = T16<T>::unpack2(u.z), d = T16<T>::unpack2(u.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
  }
  __device__ __forceinline__ void from_float(const float (&f)[8]) {
    u.x = T16<T>::pack2(f[0], f[1]); u.y = T16<T>::pack2(f[2], f[3]);
    u.z = T16<T>::pack2(f[4], f[5]); u.w = T16<T>::pack2(f[6], f[7]);
  }
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

#define B2U_DISPATCH_T(dtype, ...)                          \
  if ((dtype) == B2U_BF16) { using T = __nv_bfloat16; __VA_ARGS__; } \
  else { using T = __half; __VA_ARGS__; }

static inline int blocks_for(long long n, int per_block) { return static_cast<int>((n + per_block - 1) / per_block); }

// ------------------------------------------------------------------------------------------------ LayerNorm
// one warp per row; three passes over the (L1-resident) row: mean, centred variance, normalise.
// IN16: the input stream is 16-bit (the adapter's query stream in "c16" mode) instead of fp32.
template <typename T, bool IN16> struct LnIn;
template <typename T> struct LnIn<T, false> {
  static constexpr int kV = 4;   // elements per vector load
  __device__ static __forceinline__ void load(const void* base, long long row, int D, int i, float (&f)[4]) {
    const float4 v = reinterpret_cast<const float4*>(static_cast<const float*>(base) + row * D)[i];
    f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
  }
};
template <typename T> struct LnIn<T, true> {
  static constexpr int kV = 4;
  __device__ static __forceinline__ void load(const void* base, long long row, int D, int i, float (&f)[4]) {
    const uint2 u = reinterpret_cast<const uint2*>(static_cast<const T*>(base) + row * D)[i];
    const float2 a = T16<T>::unpack2(u.x), b = T16<T>::unpack2(u.y);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y;
  }
};

template <typename T, bool OUT32, bool IN16>
__global__ void __launch_bounds__(256) layernorm_kernel(const void* __restrict__ in, void* __restrict__ out,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                                        int rows, int D, float eps, int rows_in, int rows_out,
                                                        int row_off) {
  pdl_begin();
  using In = LnIn<T, IN16>;
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  long long ir = r;
  if (rows_out > 0) ir = static_cast<long long>(r / rows_out) * rows_in + row_off + (r % rows_out);
  const int nv = D >> 2;
  float s = 0.f;
  for (int i = lane; i < nv; i += 32) { float v[4]; In::load(in, ir, D, i, v); s += (v[0] + v[1]) + (v[2] + v[3]); }
  const float mean = warp_sum(s) / D;
  float q = 0.f;
  for (int i = lane; i < nv; i += 32) {
    float v[4];
    In::load(in, ir, D, i, v);
    const float a = v[0] - mean, b = v[1] - mean, c = v[2] - mean, d = v[3] - mean;
    q += (a * a + b * b) + (c * c + d * d);
  }
  const float rstd = rsqrtf(warp_sum(q) / D + eps);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
  for (int i = lane; i < nv; i += 32) {
    float v[4];
    In::load(in, ir, D, i, v);
    const float4 g = g4[i], b = b4[i];
    const float y0 = (v[0] - mean) * rstd * g.x + b.x, y1 = (v[1] - mean) * rstd * g.y + b.y;
    const float y2 = (v[2] - mean) * rstd * g.z + b.z, y3 = (v[3] - mean) * rstd * g.w + b.w;
    if (OUT32) {
      reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + static_cast<long long>(r) * D)[i] = make_float4(y0, y1, y2, y3);
    } else {
      uint2 pk = make_uint2(T16<T>::pack2(y0, y1), T16<T>::pack2(y2, y3));
      reinterpret_cast<uint2*>(reinterpret_cast<T*>(out) + static_cast<long long>(r) * D)[i] = pk;
    }
  }
}

// Row held in registers (NV vectors of 4 per lane, D = 128 * NV): one global read per element instead of three L1 passes.
template <typename T, bool OUT32, bool IN16, int NV>
__global__ void __launch_bounds__(256) layernorm_reg_kernel(const void* __restrict__ in, void* __restrict__ out,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta,
                                                            int rows, float eps, int rows_in, int rows_out, int row_off) {
  pdl_begin();
  using In = LnIn<T, IN16>;
  constexpr int D = 128 * NV;
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  long long ir = r;
  if (rows_out > 0) ir = static_cast<long long>(r / rows_out) * rows_in + row_off + (r % rows_out);
  float v[NV][4];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    In::load(in, ir, D, lane + 32 * k, v[k]);
    s += (v[k][0] + v[k][1]) + (v[k][2] + v[k][3]);
  }
  const float mean = warp_sum(s) * (1.f / D);
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const float a = v[k][0] - mean, b = v[k][1] - mean, c = v[k][2] - mean, d = v[k][3] - mean;
    q += (a * a + b * b) + (c * c + d * d);
  }
  const float rstd = rsqrtf(warp_sum(q) * (1.f / D) + eps);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int i = lane + 32 * k;
    const float4 g = __ldg(g4 + i), b = __ldg(b4 + i);
    const float y0 = (v[k][0] - mean) * rstd * g.x + b.x, y1 = (v[k][1] - mean) * rstd * g.y + b.y;
    const float y2 = (v[k][2] - mean) * rstd * g.z + b.z, y3 = (v[k][3] - mean) * rstd * g.w + b.w;
    if (OUT32) {
      reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + static_cast<long long>(r) * D)[i] = make_float4(y0, y1, y2, y3);
    } else {
      uint2 pk = make_uint2(T16<T>::pack2(y0, y1), T16<T>::pack2(y2, y3));
      reinterpret_cast<uint2*>(reinterpret_cast<T*>(out) + static_cast<long long>(r) * D)[i] = pk;
    }
  }
}

template <typename T, bool OUT32, bool IN16>
static void layernorm_launch(const void* in, void* out, const float* gamma, const float* beta, int rows, int D, float eps,
                             int rows_in, int rows_out, int row_off, cudaStream_t stream) {
  const int grid = blocks_for(rows, 8);
#define B2U_LN_REG(NV_)                                                                                                 \
  case 128 * NV_:                                                                                                       \
    launch_pdl(layernorm_reg_kernel<T, OUT32, IN16, NV_>, grid, 256, 0, stream, in, out, gamma, beta, rows, eps, rows_in, rows_out, row_off); \
    return;
  switch (D) {
    B2U_LN_REG(3) B2U_LN_REG(6) B2U_LN_REG(8)      // 384 / 768 / 1024 (ViT-S/B/L and their adapters)
    default: break;
  }
#undef B2U_LN_REG
  launch_pdl(layernorm_kernel<T, OUT32, IN16>, grid, 256, 0, stream, in, out, gamma, beta, rows, D, eps, rows_in, rows_out, row_off);
}

static int layernorm_impl(const void* in, bool in16, void* out, const float* gamma, const float* beta, int32_t rows,
                          int32_t D, float eps, int32_t rows_in, int32_t rows_out, int32_t row_off, int32_t out_fp32,
                          int32_t dtype, cudaStream_t stream) {
  if (D % 4) return set_error(-1, "b2u_layernorm: D %% 4 != 0");
  B2U_DISPATCH_T(dtype, {
    if (in16) {
      if (out_fp32) layernorm_launch<T, true, true>(in, out, gamma, beta, rows, D, eps, rows_in, rows_out, row_off, stream);
      else layernorm_launch<T, false, true>(in, out, gamma, beta, rows, D, eps, rows_in, rows_out, row_off, stream);
    } else {
      if (out_fp32) layernorm_launch<T, true, false>(in, out, gamma, beta, rows, D, eps, rows_in, rows_out, row_off, stream);
      else layernorm_launch<T, false, false>(in, out, gamma, beta, rows, D, eps, rows_in, rows_out, row_off, stream);
    }
  });
  return check_launch("layernorm");
}

extern "C" int b2u_layernorm(const float* in, void* out, const float* gamma, const float* beta, int32_t rows, int32_t D,
                             float eps, int32_t rows_in, int32_t rows_out, int32_t row_off, int32_t out_fp32,
                             int32_t dtype, b2u_stream_t stream_) {
  return layernorm_impl(in, false, out, gamma, beta, rows, D, eps, rows_in, rows_out, row_off, out_fp32, dtype,
                        static_cast<cudaStream_t>(stream_));
}

extern "C" int b2u_layernorm16(const void* in, void* out, const float* gamma, const float* beta, int32_t rows, int32_t D,
                               float eps, int32_t rows_in, int32_t rows_out, int32_t row_off, int32_t out_fp32,
                               int32_t dtype, b2u_stream_t stream_) {
  return layernorm_impl(in, true, out, gamma, beta, rows, D, eps, rows_in, rows_out, row_off, out_fp32, dtype,
                        static_cast<cudaStream_t>(stream_));
}

// ------------------------------------------------------------------------------------------------ cast rows
template <typename T>
__global__ void cast_rows_kernel(const float* __restrict__ in, T* __restrict__ out, long long total8, int D8,
                                 int rows_in, int rows_out, int row_off) {
  pdl_begin();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total8) return;
  const long long r = i / D8;
  const int c8 = static_cast<int>(i - r * D8);
  long long ir = r;
  if (rows_out > 0) ir = (r / rows_out) * rows_in + row_off + (r % rows_out);
  const float4* p = reinterpret_cast<const float4*>(in + (ir * D8 + c8) * 8);
  const float4 a = p[0], b = p[1];
  const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  Vec8<T> v;
  v.from_float(f);
  v.store(out + i * 8);
}

extern "C" int b2u_cast_rows(const float* in, void* out, int32_t rows, int32_t D, int32_t rows_in, int32_t rows_out,
                             int32_t row_off, int32_t dtype, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (D % 8) return set_error(-1, "b2u_cast_rows: D %% 8 != 0");
  const long long total8 = static_cast<long long>(rows) * (D / 8);
  B2U_DISPATCH_T(dtype, (launch_pdl(cast_rows_kernel<T>, blocks_for(total8, 256), 256, 0, stream, 
                             in, static_cast<T*>(out), total8, D / 8, rows_in, rows_out, row_off)));
  return check_launch("cast_rows");
}

// 16-bit row gather (same row selection as b2u_cast_rows): 16 bytes per thread
__global__ void copy_rows16_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, long long total8, int D8,
                                   int rows_in, int rows_out, int row_off) {
  pdl_begin();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total8) return;
  const long long r = i / D8;
  const int c8 = static_cast<int>(i - r * D8);
  long long ir = r;
  if (rows_out > 0) ir = (r / rows_out) * rows_in + row_off + (r % rows_out);
  out[i] = in[ir * D8 + c8];
}

extern "C" int b2u_copy_rows16(const void* in, void* out, int32_t rows, int32_t D, int32_t rows_in, int32_t rows_out,
                               int32_t row_off, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (D % 8) return set_error(-1, "b2u_copy_rows16: D %% 8 != 0");
  const long long total8 = static_cast<long long>(rows) * (D / 8);
  launch_pdl(copy_rows16_kernel, blocks_for(total8, 256), 256, 0, stream, static_cast<const uint4*>(in), static_cast<uint4*>(out),
                                                                 total8, D / 8, rows_in, rows_out, row_off);
  return check_launch("copy_rows16");
}

// ------------------------------------------------------------------------------------------------ patchify
template <typename T>
__global__ void patchify_kernel(const float* __restrict__ x, T* __restrict__ out, int B, int S) {
  pdl_begin();
  // one thread per (patch, c, ky, half) -> 8 consecutive kx
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int w = S / 16;
  const long long total = static_cast<long long>(B) * w * w * 96;  // 768 / 8
  if (i >= total) return;
  const long long patch = i / 96;
  const int k8 = static_cast<int>(i - patch * 96);
  const int c = k8 >> 5, ky = (k8 >> 1) & 15, half = k8 & 1;
  const int b = static_cast<int>(patch / (w * w));
  const int pr = static_cast<int>(patch - static_cast<long long>(b) * w * w);
  const int py = pr / w, px = pr - py * w;
  const float* src = x + ((static_cast<long long>(b) * 3 + c) * S + (py * 16 + ky)) * S + px * 16 + half * 8;
  const float4 a = reinterpret_cast<const float4*>(src)[0], d = reinterpret_cast<const float4*>(src)[1];
  const float f[8] = {a.x, a.y, a.z, a.w, d.x, d.y, d.z, d.w};
  Vec8<T> v;
  v.from_float(f);
  v.store(out + patch * 768 + k8 * 8);
}

extern "C" int b2u_patchify(const float* x, void* out, int32_t B, int32_t S, int32_t dtype, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (S % 16) return set_error(-1, "b2u_patchify: S %% 16 != 0");
  const long long total = static_cast<long long>(B) * (S / 16) * (S / 16) * 96;
  B2U_DISPATCH_T(dtype, (launch_pdl(patchify_kernel<T>, blocks_for(total, 256), 256, 0, stream, x, static_cast<T*>(out), B, S)));
  return check_launch("patchify");
}

__global__ void write_prefix_kernel(float* __restrict__ X, const float* __restrict__ prefix, int B, int ntok,
                                    int n_prefix, int D) {
  pdl_begin();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int total = B * n_prefix * D;
  if (i >= total) return;
  const int d = i % D, t = (i / D) % n_prefix, b = i / (D * n_prefix);
  X[(static_cast<long long>(b) * ntok + t) * D + d] = prefix[t * D + d];
}

extern "C" int b2u_write_prefix(float* X, const float* prefix, int32_t B, int32_t ntok, int32_t n_prefix, int32_t D,
                                b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  launch_pdl(write_prefix_kernel, blocks_for(static_cast<long long>(B) * n_prefix * D, 256), 256, 0, stream, X, prefix, B, ntok, n_prefix, D);
  return check_launch("write_prefix");
}

// ------------------------------------------------------------------------------------------------ SPM stem conv0
// Conv2d(3,64,k3,s2,p1) + folded BN + ReLU.  thread = (4 consecutive output pixels of a row, 8 channels): the 9 input
// columns each (ci, ky) needs are loaded once and every weight vector fetched from smem ([27][64]) is reused 4 times.
template <typename T>
__global__ void __launch_bounds__(256) stem_conv0_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                         const float* __restrict__ scale, const float* __restrict__ shift,
                                                         T* __restrict__ out, int B, int S) {
  pdl_begin();
  __shared__ float sw[27 * 64];
  __shared__ float ssc[64], ssh[64];
  for (int i = threadIdx.x; i < 27 * 64; i += 256) {
    const int co = i & 63, k = i >> 6;  // w is [64][3][3][3] -> k = ci*9 + ky*3 + kx
    sw[i] = w[co * 27 + k];
  }
  if (threadIdx.x < 64) { ssc[threadIdx.x] = scale[threadIdx.x]; ssh[threadIdx.x] = shift[threadIdx.x]; }
  __syncthreads();
  const int So = S / 2, Q = So / 4;   // 4-pixel groups per output row
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  const long long total = static_cast<long long>(B) * So * Q * 8;
  if (i >= total) return;
  const int cg = static_cast<int>(i & 7);
  const long long grp = i >> 3;
  const int qx = static_cast<int>(grp % Q), oy = static_cast<int>((grp / Q) % So), b = static_cast<int>(grp / (static_cast<long long>(Q) * So));
  const int ox0 = qx * 4;
  float acc[4][8];
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[p][j] = 0.f;
#pragma unroll
  for (int ci = 0; ci < 3; ++ci)
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = 2 * oy + ky - 1;
      if (iy < 0 || iy >= S) continue;
      const float* row = x + ((static_cast<long long>(b) * 3 + ci) * S + iy) * S;
      float in[9];                                   // input columns 2*ox0-1 .. 2*ox0+7
#pragma unroll
      for (int c = 0; c < 9; ++c) {
        const int ix = 2 * ox0 - 1 + c;
        in[c] = (ix >= 0 && ix < S) ? __ldg(row + ix) : 0.f;
      }
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const float4 w0 = *reinterpret_cast<const float4*>(sw + (ci * 9 + ky * 3 + kx) * 64 + cg * 8);
        const float4 w1 = *reinterpret_cast<const float4*>(sw + (ci * 9 + ky * 3 + kx) * 64 + cg * 8 + 4);
        const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const float xv = in[2 * p + kx];
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[p][j] = fmaf(xv, wv[j], acc[p][j]);
        }
      }
    }
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    float f[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float r16 = T16<T>::to_f(T16<T>::from_f(acc[p][j]));  // conv output is 16-bit under autocast
      f[j] = fmaxf(r16 * ssc[cg * 8 + j] + ssh[cg * 8 + j], 0.f);
    }
    Vec8<T> v;
    v.from_float(f);
    v.store(out + ((static_cast<long long>(b) * So + oy) * So + ox0 + p) * 64 + cg * 8);
  }
}

extern "C" int b2u_stem_conv0(const float* x, const float* w, const float* scale, const float* shift, void* out,
                              int32_t B, int32_t S, int32_t dtype, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (S % 8) return set_error(-1, "b2u_stem_conv0: S %% 8 != 0");
  const long long total = static_cast<long long>(B) * (S / 2) * (S / 8) * 8;
  B2U_DISPATCH_T(dtype, (launch_pdl(stem_conv0_kernel<T>, blocks_for(total, 256), 256, 0, stream, x, w, scale, shift, static_cast<T*>(out), B, S)));
  return check_launch("stem_conv0");
}

// ------------------------------------------------------------------------------------------------ maxpool 3x3 s2 p1
template <typename T>
__global__ void maxpool_kernel(const T* __restrict__ in, T* __restrict__ out, int B, int H, int W, int C8) {
  pdl_begin();
  const int Ho = H / 2, Wo = W / 2;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * Ho * Wo * C8;
  if (i >= total) return;
  const int c8 = static_cast<int>(i % C8);
  const long long pix = i / C8;
  const int ox = static_cast<int>(pix % Wo), oy = static_cast<int>((pix / Wo) % Ho), b = static_cast<int>(pix / (static_cast<long long>(Wo) * Ho));
  float m[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) m[j] = -INFINITY;
  for (int ky = 0; ky < 3; ++ky) {
    const int iy = 2 * oy + ky - 1;
    if (iy < 0 || iy >= H) continue;
    for (int kx = 0; kx < 3; ++kx) {
      const int ix = 2 * ox + kx - 1;
      if (ix < 0 || ix >= W) continue;
      Vec8<T> v;
      v.load(in + ((static_cast<long long>(b) * H + iy) * W + ix) * C8 * 8 + c8 * 8);
      float f[8];
      v.to_float(f);
#pragma unroll
      for (int j = 0; j < 8; ++j) m[j] = fmaxf(m[j], f[j]);
    }
  }
  Vec8<T> o;
  o.from_float(m);
  o.store(out + pix * C8 * 8 + c8 * 8);
}

extern "C" int b2u_maxpool3x3s2(const void* in, void* out, int32_t B, int32_t H, int32_t W, int32_t C, int32_t dtype,
                                b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (C % 8) return set_error(-1, "b2u_maxpool3x3s2: C %% 8 != 0");
  const long long total = static_cast<long long>(B) * (H / 2) * (W / 2) * (C / 8);
  B2U_DISPATCH_T(dtype, (launch_pdl(maxpool_kernel<T>, blocks_for(total, 256), 256, 0, stream, static_cast<const T*>(in), static_cast<T*>(out), B, H, W, C / 8)));
  return check_launch("maxpool3x3s2");
}

// ------------------------------------------------------------------------------------------------ depthwise 3x3
// w9 is [9][C] fp32 (tap-major).  thread = (4 consecutive pixels of a plane row, 8 channels): the 9 x 8 weights live in
// registers and the 3 x 6 input vectors are loaded once for the 4 outputs (3x fewer loads than one pixel per thread).
template <typename T>
__global__ void __launch_bounds__(256) dwconv_kernel(const T* __restrict__ in, T* __restrict__ out,
                                                     const float* __restrict__ w9, const float* __restrict__ bias, int B,
                                                     int H, int W, int C8, int planes, int act) {
  pdl_begin();
  // 4-pixel groups per image: planes==3 -> (2H x 2W) + (H x W) + (H/2 x W/2) planes, every plane width is a multiple of 4
  const long long rows_per_img = planes == 3 ? (static_cast<long long>(H) * W * 21) / 4 : static_cast<long long>(H) * W;
  const long long groups_per_img = rows_per_img / 4;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * groups_per_img * C8;
  if (i >= total) return;
  const int c8 = static_cast<int>(i % C8);
  const long long grp = i / C8;
  const int b = static_cast<int>(grp / groups_per_img);
  long long t = (grp - static_cast<long long>(b) * groups_per_img) * 4;   // first token of the group within the image
  int ph = H, pw = W;
  long long poff = 0;
  if (planes == 3) {
    const long long n0 = static_cast<long long>(H) * W * 4, n1 = static_cast<long long>(H) * W;
    if (t < n0) { ph = 2 * H; pw = 2 * W; }
    else if (t < n0 + n1) { poff = n0; t -= n0; }
    else { poff = n0 + n1; t -= n0 + n1; ph = H / 2; pw = W / 2; }
  }
  const int y = static_cast<int>(t / pw), x0 = static_cast<int>(t - static_cast<long long>(y) * pw);
  const int C = C8 * 8;
  const T* base = in + (static_cast<long long>(b) * rows_per_img + poff) * C + c8 * 8;
  float acc[4][8];
  {
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + c8 * 8)), b1 = __ldg(reinterpret_cast<const float4*>(bias + c8 * 8) + 1);
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      acc[p][0] = b0.x; acc[p][1] = b0.y; acc[p][2] = b0.z; acc[p][3] = b0.w; acc[p][4] = b1.x; acc[p][5] = b1.y; acc[p][6] = b1.z; acc[p][7] = b1.w;
    }
  }
  // per tap row: the 6 input vectors are requested together (6 independent 16-byte loads in flight), the 3 x 8 weights
  // of the row come from L1 (keeping all 72 in registers cost 128 registers/thread = 512 threads/SM, latency-bound)
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int iy = y + ky - 1;
    if (iy < 0 || iy >= ph) continue;                 // warp-uniform for whole-row groups except at plane borders
    Vec8<T> v[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      const int ix = x0 - 1 + c;
      if (ix >= 0 && ix < pw) v[c].load(base + (static_cast<long long>(iy) * pw + ix) * C);
      else v[c].zero();
    }
    float wr[3][8];
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const float4 w0 = __ldg(reinterpret_cast<const float4*>(w9 + (ky * 3 + kx) * C + c8 * 8)), w1 = __ldg(reinterpret_cast<const float4*>(w9 + (ky * 3 + kx) * C + c8 * 8) + 1);
      wr[kx][0] = w0.x; wr[kx][1] = w0.y; wr[kx][2] = w0.z; wr[kx][3] = w0.w; wr[kx][4] = w1.x; wr[kx][5] = w1.y; wr[kx][6] = w1.z; wr[kx][7] = w1.w;
    }
#pragma unroll
    for (int c = 0; c < 6; ++c) {                      // input columns x0-1 .. x0+4
      float f[8];
      v[c].to_float(f);
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const int kx = c - p;                          // output pixel x0+p sees this column as tap kx
        if (kx < 0 || kx > 2) continue;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[p][j] = fmaf(f[j], wr[kx][j], acc[p][j]);
      }
    }
  }
  T* obase = out + ((static_cast<long long>(b) * rows_per_img + poff) + static_cast<long long>(y) * pw + x0) * C + c8 * 8;
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    if (act == B2U_ACT_GELU) {
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[p][j] = gelu_erf(T16<T>::to_f(T16<T>::from_f(acc[p][j])));
    }
    Vec8<T> o;
    o.from_float(acc[p]);
    o.store(obase + static_cast<long long>(p) * C);
  }
}

extern "C" int b2u_dwconv3x3(const void* in, void* out, const float* w, const float* bias, int32_t B, int32_t H,
                             int32_t W, int32_t C, int32_t planes, int32_t act, int32_t dtype, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (C % 8) return set_error(-1, "b2u_dwconv3x3: C %% 8 != 0");
  if (planes != 1 && planes != 3) return set_error(-1, "b2u_dwconv3x3: planes must be 1 or 3");
  if ((planes == 3 && (W % 8 || H % 2)) || (planes == 1 && W % 4)) return set_error(-1, "b2u_dwconv3x3: plane widths must be multiples of 4");
  const long long rows = planes == 3 ? (static_cast<long long>(H) * W * 21) / 4 : static_cast<long long>(H) * W;
  const long long total = static_cast<long long>(B) * (rows / 4) * (C / 8);
  B2U_DISPATCH_T(dtype, (launch_pdl(dwconv_kernel<T>, blocks_for(total, 256), 256, 0, stream, static_cast<const T*>(in), static_cast<T*>(out), w, bias, B, H, W, C / 8, planes, act)));
  return check_launch("dwconv3x3");
}

// ------------------------------------------------------------------------------------------------ adapter tail
template <typename T>
__global__ void tail_fuse_kernel(const void* __restrict__ base, int base_fp32, long long base_bstride,
                                 const float* __restrict__ tap, T* __restrict__ out, const float* __restrict__ scale,
                                 const float* __restrict__ shift, int B, int H, int W, int Ht, int Wt, int D8) {
  pdl_begin();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * H * W * D8;
  if (i >= total) return;
  const int c8 = static_cast<int>(i % D8);
  const long long pix = i / D8;
  const int x = static_cast<int>(pix % W), y = static_cast<int>((pix / W) % H), b = static_cast<int>(pix / (static_cast<long long>(W) * H));
  const int D = D8 * 8;
  // bilinear source (align_corners=False), PyTorch upsample_bilinear2d index rule
  const float sy = fmaxf((y + 0.5f) * (static_cast<float>(Ht) / H) - 0.5f, 0.f);
  const float sx = fmaxf((x + 0.5f) * (static_cast<float>(Wt) / W) - 0.5f, 0.f);
  const int y0 = static_cast<int>(sy), x0 = static_cast<int>(sx);
  const int y1 = y0 + (y0 < Ht - 1 ? 1 : 0), x1 = x0 + (x0 < Wt - 1 ? 1 : 0);
  const float ly = sy - y0, lx = sx - x0;
  const float w00 = (1.f - ly) * (1.f - lx), w01 = (1.f - ly) * lx, w10 = ly * (1.f - lx), w11 = ly * lx;
  const float* tb = tap + static_cast<long long>(b) * Ht * Wt * D + c8 * 8;
  float f[8];
  if (base_fp32) {
    const float* bp = reinterpret_cast<const float*>(base) + static_cast<long long>(b) * base_bstride + (static_cast<long long>(y) * W + x) * D + c8 * 8;
    const float4 a = reinterpret_cast<const float4*>(bp)[0], c = reinterpret_cast<const float4*>(bp)[1];
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = c.x; f[5] = c.y; f[6] = c.z; f[7] = c.w;
  } else {
    Vec8<T> v;
    v.load(reinterpret_cast<const T*>(base) + static_cast<long long>(b) * base_bstride + (static_cast<long long>(y) * W + x) * D + c8 * 8);
    v.to_float(f);
  }
  const float* p00 = tb + (static_cast<long long>(y0) * Wt + x0) * D;
  const float* p01 = tb + (static_cast<long long>(y0) * Wt + x1) * D;
  const float* p10 = tb + (static_cast<long long>(y1) * Wt + x0) * D;
  const float* p11 = tb + (static_cast<long long>(y1) * Wt + x1) * D;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float4 a = reinterpret_cast<const float4*>(p00)[h], c = reinterpret_cast<const float4*>(p01)[h];
    const float4 d = reinterpret_cast<const float4*>(p10)[h], e = reinterpret_cast<const float4*>(p11)[h];
    f[4 * h + 0] += w00 * a.x + w01 * c.x + w10 * d.x + w11 * e.x;
    f[4 * h + 1] += w00 * a.y + w01 * c.y + w10 * d.y + w11 * e.y;
    f[4 * h + 2] += w00 * a.z + w01 * c.z + w10 * d.z + w11 * e.z;
    f[4 * h + 3] += w00 * a.w + w01 * c.w + w10 * d.w + w11 * e.w;
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) f[j] = f[j] * __ldg(scale + c8 * 8 + j) + __ldg(shift + c8 * 8 + j);
  Vec8<T> o;
  o.from_float(f);
  o.store(out + pix * D + c8 * 8);
}

// Integer up-scaling (S = 2, 4): one thread per SOURCE cell (between tap rows cy, cy+1 and columns cx, cx+1) and 8
// channels.  The 4 corner vectors are loaded once and reused for the S x S output pixels whose bilinear footprint is that
// cell (output rows S*cy + S/2 + t, t < S, weight (t + 0.5) / S; border cells clamp, which reproduces PyTorch's
// src = max((dst + 0.5) / S - 0.5, 0) rule), so the fp32 tap traffic drops by S^2 compared to the per-output gather.
template <typename T, int S>
__global__ void tail_fuse_up_kernel(const void* __restrict__ base, int base_fp32, long long base_bstride,
                                    const float* __restrict__ tap, T* __restrict__ out, const float* __restrict__ scale,
                                    const float* __restrict__ shift, int B, int Ht, int Wt, int D8) {
  pdl_begin();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int CW = Wt + 1, CH = Ht + 1;
  const long long total = static_cast<long long>(B) * CH * CW * D8;
  if (i >= total) return;
  const int c8 = static_cast<int>(i % D8);
  const long long cell = i / D8;
  const int cx = static_cast<int>(cell % CW) - 1, cy = static_cast<int>((cell / CW) % CH) - 1;
  const int b = static_cast<int>(cell / (static_cast<long long>(CW) * CH));
  const int D = D8 * 8, H = S * Ht, W = S * Wt;
  const int y0 = max(cy, 0), y1 = min(cy + 1, Ht - 1), x0 = max(cx, 0), x1 = min(cx + 1, Wt - 1);
  const float* tb = tap + static_cast<long long>(b) * Ht * Wt * D + c8 * 8;
  float c00[8], c01[8], c10[8], c11[8], sc[8], sh[8];
  auto ld8 = [](const float* p, float (&f)[8]) {
    const float4 a = reinterpret_cast<const float4*>(p)[0], c = reinterpret_cast<const float4*>(p)[1];
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = c.x; f[5] = c.y; f[6] = c.z; f[7] = c.w;
  };
  ld8(tb + (static_cast<long long>(y0) * Wt + x0) * D, c00);
  ld8(tb + (static_cast<long long>(y0) * Wt + x1) * D, c01);
  ld8(tb + (static_cast<long long>(y1) * Wt + x0) * D, c10);
  ld8(tb + (static_cast<long long>(y1) * Wt + x1) * D, c11);
  ld8(scale + c8 * 8, sc);
  ld8(shift + c8 * 8, sh);
#pragma unroll
  for (int ty = 0; ty < S; ++ty) {
    const int y = S * cy + S / 2 + ty;
    if (y < 0 || y >= H) continue;
    const float ly = (ty + 0.5f) / S;
    // the S base vectors of this output row are requested together (S independent loads in flight per thread)
    float f[S][8];
    bool ok[S];
#pragma unroll
    for (int tx = 0; tx < S; ++tx) {
      const int x = S * cx + S / 2 + tx;
      ok[tx] = x >= 0 && x < W;
      const long long pix = static_cast<long long>(y) * W + (ok[tx] ? x : 0);
      if (base_fp32) {
        ld8(reinterpret_cast<const float*>(base) + static_cast<long long>(b) * base_bstride + pix * D + c8 * 8, f[tx]);
      } else {
        Vec8<T> v;
        v.load(reinterpret_cast<const T*>(base) + static_cast<long long>(b) * base_bstride + pix * D + c8 * 8);
        v.to_float(f[tx]);
      }
    }
#pragma unroll
    for (int tx = 0; tx < S; ++tx) {
      if (!ok[tx]) continue;
      const int x = S * cx + S / 2 + tx;
      const float lx = (tx + 0.5f) / S;
      const float w00 = (1.f - ly) * (1.f - lx), w01 = (1.f - ly) * lx, w10 = ly * (1.f - lx), w11 = ly * lx;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        f[tx][j] = (f[tx][j] + (w00 * c00[j] + w01 * c01[j] + w10 * c10[j] + w11 * c11[j])) * sc[j] + sh[j];
      Vec8<T> o;
      o.from_float(f[tx]);
      o.store(out + (static_cast<long long>(b) * H * W + static_cast<long long>(y) * W + x) * D + c8 * 8);
    }
  }
}

extern "C" int b2u_tail_fuse(const void* base, int32_t base_fp32, int64_t base_batch_stride, const float* tap, void* out,
                             const float* scale, const float* shift, int32_t B, int32_t H, int32_t W, int32_t Ht,
                             int32_t Wt, int32_t D, int32_t dtype, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (D % 8) return set_error(-1, "b2u_tail_fuse: D %% 8 != 0");
  if ((H == 4 * Ht && W == 4 * Wt) || (H == 2 * Ht && W == 2 * Wt)) {
    const long long cells = static_cast<long long>(B) * (Ht + 1) * (Wt + 1) * (D / 8);
    if (H == 4 * Ht) {
      B2U_DISPATCH_T(dtype, (launch_pdl(tail_fuse_up_kernel<T, 4>, blocks_for(cells, 256), 256, 0, stream, base, base_fp32, base_batch_stride, tap, static_cast<T*>(out), scale, shift, B, Ht, Wt, D / 8)));
    } else {
      B2U_DISPATCH_T(dtype, (launch_pdl(tail_fuse_up_kernel<T, 2>, blocks_for(cells, 256), 256, 0, stream, base, base_fp32, base_batch_stride, tap, static_cast<T*>(out), scale, shift, B, Ht, Wt, D / 8)));
    }
    return check_launch("tail_fuse(up)");
  }
  const long long total = static_cast<long long>(B) * H * W * (D / 8);
  B2U_DISPATCH_T(dtype, (launch_pdl(tail_fuse_kernel<T>, blocks_for(total, 256), 256, 0, stream, base, base_fp32, base_batch_stride, tap, static_cast<T*>(out), scale, shift, B, H, W, Ht, Wt, D / 8)));
  return check_launch("tail_fuse");
}

// ------------------------------------------------------------------------------------------------ InstanceNorm
// stats: block = (row chunk, image b); thread = (row lane, 8-channel group); smem tree over row lanes.  Each block makes two
// passes over its chunk (the second from L2): the chunk sum, then the sum of squares about the chunk's own mean.  The block's
// partial (sum, centred sumsq) per channel goes to a workspace slot, and the LAST block of each image (ticket counter)
// merges the slots in fixed chunk order (Chan et al.'s pairwise update) -> bitwise deterministic, no float atomics, no
// zero-fill of `sums` needed.  Output per (image, channel): (sum x, sum (x - mean)^2).
// Workspace: kInTickets ticket counters, then the partials.  The partials start at the same offset for every (B, rows, C),
// so one workspace can serve calls of different shapes: partials of one call never land on another call's counters.
constexpr int kInTickets = 1024;
static inline int in_stats_chunk(int rows) { return rows >= 8192 ? 2048 : (rows >= 1024 ? 256 : 64); }

template <typename T>
__global__ void __launch_bounds__(256) in_stats_kernel(const T* __restrict__ x, long long ldx, float* __restrict__ sums,
                                                       float* __restrict__ work, int rows, int C8, int chunk) {
  pdl_begin();
  extern __shared__ float red[];  // [rows_par][C8*16], then the chunk sums [C8*8]
  __shared__ int s_last;
  const int b = blockIdx.y, nchunks = gridDim.x, B = gridDim.y;
  const int cg = threadIdx.x % C8, rl = threadIdx.x / C8;
  const int rows_par = 256 / C8;
  const int r0 = blockIdx.x * chunk;
  const int r1 = min(rows, r0 + chunk);
  const int nout = C8 * 16;  // per image: C channels x (sum, sumsq), laid out [cg][k][j]
  float* csum = red + rows_par * nout;
  // Sums are taken of x - x0 (x0 = the image's first pixel of the channel) so that they stay small when |mean| >> std.
  // The squares are taken about the chunk mean, not about x0: a first pixel far from the mean (a padded border, a hot
  // pixel) would otherwise leave the variance as the difference of two large, nearly equal sums.
  float sh[8];
  {
    Vec8<T> v0;
    v0.load(x + static_cast<long long>(b) * rows * ldx + cg * 8);
    v0.to_float(sh);
  }
  float s[8] = {0, 0, 0, 0, 0, 0, 0, 0}, q[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int r = r0 + rl; r < r1; r += rows_par) {
    Vec8<T> v;
    v.load(x + (static_cast<long long>(b) * rows + r) * ldx + cg * 8);
    float f[8];
    v.to_float(f);
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] += f[j] - sh[j];
  }
  float* my = red + (rl * C8 + cg) * 16;
#pragma unroll
  for (int j = 0; j < 8; ++j) my[j] = s[j];
  __syncthreads();
  for (int o = threadIdx.x; o < C8 * 8; o += 256) {
    const int g = o >> 3, j = o & 7;
    float t = 0.f;
    for (int p = 0; p < rows_par; ++p) t += red[p * nout + g * 16 + j];
    csum[o] = t;
  }
  __syncthreads();
  float mc[8];
  const float inv_n = 1.f / static_cast<float>(r1 - r0);
#pragma unroll
  for (int j = 0; j < 8; ++j) mc[j] = csum[cg * 8 + j] * inv_n;
  for (int r = r0 + rl; r < r1; r += rows_par) {
    Vec8<T> v;
    v.load(x + (static_cast<long long>(b) * rows + r) * ldx + cg * 8);
    float f[8];
    v.to_float(f);
#pragma unroll
    for (int j = 0; j < 8; ++j) { const float d = (f[j] - sh[j]) - mc[j]; q[j] = fmaf(d, d, q[j]); }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) my[8 + j] = q[j];
  __syncthreads();
  int* counters = reinterpret_cast<int*>(work);
  float* part = work + kInTickets + (static_cast<long long>(b) * nchunks + blockIdx.x) * nout;
  for (int o = threadIdx.x; o < nout; o += 256) {
    float t = 0.f;
    for (int p = 0; p < rows_par; ++p) t += red[p * nout + o];
    part[o] = t;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(counters + b, 1) == nchunks - 1);
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const float* pb = work + kInTickets + static_cast<long long>(b) * nchunks * nout;
  for (int o = threadIdx.x; o < C8 * 8; o += 256) {       // one thread per channel: fixed chunk order -> deterministic
    const int g = o >> 3, j = o & 7;
    float ts = 0.f, tq = 0.f;
    for (int c = 0; c < nchunks; ++c) ts += __ldcg(pb + static_cast<long long>(c) * nout + g * 16 + j);
    const float md = ts / static_cast<float>(rows);
    for (int c = 0; c < nchunks; ++c) {   // M2 = sum_c [M2_c + n_c (mean_c - mean)^2]
      const float n_c = static_cast<float>(min(chunk, rows - c * chunk));
      const float dm = __ldcg(pb + static_cast<long long>(c) * nout + g * 16 + j) / n_c - md;
      tq += fmaf(n_c * dm, dm, __ldcg(pb + static_cast<long long>(c) * nout + g * 16 + 8 + j));
    }
    const float x0 = T16<T>::to_f(x[static_cast<long long>(b) * rows * ldx + o]);
    float* dst = sums + (static_cast<long long>(b) * C8 * 8 + o) * 2;
    dst[0] = fmaf(static_cast<float>(rows), x0, ts);                  // sum x
    dst[1] = tq;                                                      // sum (x - mean)^2
  }
  if (threadIdx.x == 0) counters[b] = 0;  // self-resetting ticket
}

extern "C" int64_t b2u_in_stats_work_floats(int32_t B, int32_t rows, int32_t C) {
  const int chunk = in_stats_chunk(rows);
  return static_cast<int64_t>(kInTickets) + static_cast<int64_t>(B) * ((rows + chunk - 1) / chunk) * C * 2;
}

extern "C" int b2u_in_stats(const void* x, int64_t ldx, float* sums, float* work, int32_t B, int32_t rows, int32_t C,
                            int32_t dtype, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (C % 8 || C > 2048 || (256 % (C / 8))) return set_error(-1, "b2u_in_stats: C must be 8*2^k <= 2048");
  if (!work) return set_error(-1, "b2u_in_stats: workspace required");
  if (B > kInTickets) return set_error(-1, "b2u_in_stats: B > %d", kInTickets);
  const int C8 = C / 8;
  const int chunk = in_stats_chunk(rows);
  dim3 grid((rows + chunk - 1) / chunk, B);
  const size_t smem = (static_cast<size_t>(256 / C8) * C8 * 16 + C8 * 8) * sizeof(float);
  B2U_DISPATCH_T(dtype, (launch_pdl(in_stats_kernel<T>, grid, 256, smem, stream, static_cast<const T*>(x), ldx, sums, work, rows, C8, chunk)));
  return check_launch("in_stats");
}

// block = (row chunk, image); thread = (row lane, 8-channel group).  The per-channel affine y = x * a + b (a = rstd * gamma,
// b = beta - mean * a) is formed ONCE per thread and applied to up to 64 rows: the first version recomputed mean / var /
// rsqrt (24 small loads + 8 rsqrt) for every 16 bytes of data and ran at 55 % of the HBM rate.
template <typename T>
__global__ void __launch_bounds__(256) in_apply_kernel(const T* __restrict__ x, long long ldx, T* __restrict__ y,
                                                       long long ldy, const float* __restrict__ sums,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                                       int rows, int C8, float eps, int chunk) {
  pdl_begin();
  const int b = blockIdx.y;
  const int cg = threadIdx.x % C8, rl = threadIdx.x / C8;
  const int rows_par = 256 / C8;
  if (rl >= rows_par) return;
  float sa[8], sb[8];
  const float inv = 1.f / rows;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = cg * 8 + j;
    const float2 sq = *reinterpret_cast<const float2*>(sums + (static_cast<long long>(b) * C8 * 8 + c) * 2);
    const float mean = sq.x * inv;
    const float var = sq.y * inv;                     // centred second moment (b2u_in_stats)
    // same operation order as before: (x - mean) * rstd * gamma + beta
    sa[j] = rsqrtf(var + eps);
    sb[j] = mean;
  }
  float g[8], be[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { g[j] = __ldg(gamma + cg * 8 + j); be[j] = __ldg(beta + cg * 8 + j); }
  const int r0 = blockIdx.x * chunk;
  const int r1 = min(rows, r0 + chunk);
  const T* xb = x + static_cast<long long>(b) * rows * ldx + cg * 8;
  T* yb = y + static_cast<long long>(b) * rows * ldy + cg * 8;
#pragma unroll 4
  for (int r = r0 + rl; r < r1; r += rows_par) {
    Vec8<T> v;
    v.load(xb + static_cast<long long>(r) * ldx);
    float f[8];
    v.to_float(f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float t = (f[j] - sb[j]) * sa[j] * g[j] + be[j];
      f[j] = t > 0.f ? t : 0.01f * t;
    }
    Vec8<T> o;
    o.from_float(f);
    o.store(yb + static_cast<long long>(r) * ldy);
  }
}

extern "C" int b2u_in_apply(const void* x, int64_t ldx, void* y, int64_t ldy, const float* sums, const float* gamma,
                            const float* beta, int32_t B, int32_t rows, int32_t C, float eps, int32_t dtype,
                            b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (C % 8 || C > 2048) return set_error(-1, "b2u_in_apply: C %% 8 != 0 or C > 2048");
  const int C8 = C / 8;
  const int rows_par = 256 / C8;
  // up to 64 rows per thread, but keep >= ~4 blocks per SM in flight for small images
  int per_thread = 64;
  while (per_thread > 4 && static_cast<long long>(B) * ((rows + rows_par * per_thread - 1) / (rows_par * per_thread)) < 4LL * num_sms())
    per_thread >>= 1;
  const int chunk = rows_par * per_thread;
  dim3 grid((rows + chunk - 1) / chunk, B);
  B2U_DISPATCH_T(dtype, (launch_pdl(in_apply_kernel<T>, grid, 256, 0, stream, static_cast<const T*>(x), ldx, static_cast<T*>(y), ldy, sums, gamma, beta, rows, C8, eps, chunk)));
  return check_launch("in_apply");
}

// ------------------------------------------------------------------------------------------------ FiLM
template <typename T>
__global__ void film_kernel(const T* __restrict__ gb, const T* __restrict__ zz, long long ldzz, int zoff,
                            T* __restrict__ z, long long rows, int R8) {
  pdl_begin();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= rows * R8) return;
  const int c8 = static_cast<int>(i % R8);
  const long long r = i / R8;
  const int R = R8 * 8;
  Vec8<T> g, bt, zs;
  g.load(gb + r * 2 * R + c8 * 8);
  bt.load(gb + r * 2 * R + R + c8 * 8);
  zs.load(zz + r * ldzz + zoff + c8 * 8);
  float fg[8], fb[8], fz[8];
  g.to_float(fg); bt.to_float(fb); zs.to_float(fz);
#pragma unroll
  for (int j = 0; j < 8; ++j) fz[j] = fg[j] * fz[j] + fb[j];
  Vec8<T> o;
  o.from_float(fz);
  o.store(z + r * R + c8 * 8);
}

extern "C" int b2u_film(const void* gb, const void* zz, int64_t ldzz, int32_t zoff, void* z, int32_t rows, int32_t R,
                        int32_t dtype, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (R % 8) return set_error(-1, "b2u_film: R %% 8 != 0");
  const long long total = static_cast<long long>(rows) * (R / 8);
  B2U_DISPATCH_T(dtype, (launch_pdl(film_kernel<T>, blocks_for(total, 256), 256, 0, stream, static_cast<const T*>(gb), static_cast<const T*>(zz), ldzz, zoff, static_cast<T*>(z), rows, R / 8)));
  return check_launch("film");
}

// ------------------------------------------------------------------------------------------------ squeeze-excitation
__global__ void se_gate_kernel(const float* __restrict__ sums, const float* __restrict__ w1, const float* __restrict__ b1,
                               const float* __restrict__ w2, const float* __restrict__ b2, float* __restrict__ gate,
                               int C, int Cr, int rows) {
  pdl_begin();
  extern __shared__ float sm[];  // pooled[C] + hidden[Cr]
  float* pooled = sm;
  float* hidden = sm + C;
  const int b = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) pooled[c] = sums[(static_cast<long long>(b) * C + c) * 2] / rows;
  __syncthreads();
  for (int h = threadIdx.x; h < Cr; h += blockDim.x) {
    float a = b1[h];
    for (int c = 0; c < C; ++c) a = fmaf(w1[h * C + c], pooled[c], a);
    hidden[h] = fmaxf(a, 0.f);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float a = b2[c];
    for (int h = 0; h < Cr; ++h) a = fmaf(w2[c * Cr + h], hidden[h], a);
    gate[static_cast<long long>(b) * C + c] = 1.f / (1.f + __expf(-a));
  }
}

extern "C" int b2u_se_gate(const float* sums, const float* w1, const float* b1, const float* w2, const float* b2,
                           float* gate, int32_t B, int32_t C, int32_t Cr, int32_t rows, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  launch_pdl(se_gate_kernel, B, 256, (C + Cr) * sizeof(float), stream, sums, w1, b1, w2, b2, gate, C, Cr, rows);
  return check_launch("se_gate");
}

template <typename T>
__global__ void se_apply_kernel(const T* __restrict__ t, const T* __restrict__ sc, long long ldsc,
                                const float* __restrict__ gate, T* __restrict__ out, int B, int rows, int C8) {
  pdl_begin();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * rows * C8;
  if (i >= total) return;
  const int cg = static_cast<int>(i % C8);
  const long long row = i / C8;
  const int b = static_cast<int>(row / rows);
  Vec8<T> a, s;
  a.load(t + row * C8 * 8 + cg * 8);
  s.load(sc + row * ldsc + cg * 8);
  float fa[8], fs[8];
  a.to_float(fa); s.to_float(fs);
  const float* g = gate + static_cast<long long>(b) * C8 * 8 + cg * 8;
#pragma unroll
  for (int j = 0; j < 8; ++j) fa[j] = fa[j] * __ldg(g + j) + fs[j];
  Vec8<T> o;
  o.from_float(fa);
  o.store(out + row * C8 * 8 + cg * 8);
}

extern "C" int b2u_se_apply(const void* t, const void* sc, int64_t ldsc, const float* gate, void* out, int32_t B,
                            int32_t rows, int32_t C, int32_t dtype, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (C % 8) return set_error(-1, "b2u_se_apply: C %% 8 != 0");
  const long long total = static_cast<long long>(B) * rows * (C / 8);
  B2U_DISPATCH_T(dtype, (launch_pdl(se_apply_kernel<T>, blocks_for(total, 256), 256, 0, stream, static_cast<const T*>(t), static_cast<const T*>(sc), ldsc, gate, static_cast<T*>(out), B, rows, C / 8)));
  return check_launch("se_apply");
}

// ------------------------------------------------------------------------------------------------ seg head
// thread per pixel: InstanceNorm + LeakyReLU on C channels (kept in registers), 1x1 conv to ncls (<= 128) classes in
// groups of 8 accumulators, NCHW fp32 logits, argmax (first maximum, like torch.argmax).
constexpr int kSegMaxClasses = 128;
template <typename T, int C>
__global__ void __launch_bounds__(256) seg_head_kernel(const T* __restrict__ x, const float* __restrict__ sums,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                                       float eps, const float* __restrict__ w, const float* __restrict__ bias,
                                                       float* __restrict__ logits, uint8_t* __restrict__ labels,
                                                       int rows, int ncls) {
  pdl_begin();
  __shared__ float s_a[C], s_b[C];       // per-image affine: y = x*a + b
  __shared__ float s_w[kSegMaxClasses * 32], s_bias[kSegMaxClasses];   // ncls * C <= kSegMaxClasses * 32
  const int b = blockIdx.y;
  for (int c = threadIdx.x; c < C; c += 256) {
    const float mean = sums[(static_cast<long long>(b) * C + c) * 2] / rows;
    const float var = sums[(static_cast<long long>(b) * C + c) * 2 + 1] / rows;   // centred second moment (b2u_in_stats)
    const float a = rsqrtf(var + eps) * gamma[c];
    s_a[c] = a;
    s_b[c] = beta[c] - mean * a;
  }
  for (int i = threadIdx.x; i < ncls * C; i += 256) s_w[i] = w[i];
  for (int i = threadIdx.x; i < ncls; i += 256) s_bias[i] = bias[i];
  __syncthreads();
  const int p = blockIdx.x * 256 + threadIdx.x;
  if (p >= rows) return;
  const T* xp = x + (static_cast<long long>(b) * rows + p) * C;
  float t[C];
#pragma unroll
  for (int g = 0; g < C / 8; ++g) {
    Vec8<T> v;
    v.load(xp + g * 8);
    float f[8];
    v.to_float(f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float u = f[j] * s_a[g * 8 + j] + s_b[g * 8 + j];
      u = u > 0.f ? u : 0.01f * u;
      t[g * 8 + j] = T16<T>::to_f(T16<T>::from_f(u));  // the normalised activation is a 16-bit tensor in the reference regime
    }
  }
  int best = 0;
  float bv = -INFINITY;
  for (int k0 = 0; k0 < ncls; k0 += 8) {   // warp-uniform trip count
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = k0 + k < ncls ? s_bias[k0 + k] : -INFINITY;
#pragma unroll
    for (int c = 0; c < C; ++c) {
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (k0 + k < ncls) acc[k] = fmaf(t[c], s_w[(k0 + k) * C + c], acc[k]);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (k0 + k < ncls) {
        logits[(static_cast<long long>(b) * ncls + k0 + k) * rows + p] = acc[k];
        if (acc[k] > bv) { bv = acc[k]; best = k0 + k; }
      }
    }
  }
  if (labels) labels[static_cast<long long>(b) * rows + p] = static_cast<uint8_t>(best);
}

// <= 8 classes (the common case): everything unrolled, the activations are consumed as they are loaded.
template <typename T, int C>
__global__ void __launch_bounds__(256) seg_head_kernel8(const T* __restrict__ x, const float* __restrict__ sums,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                                       float eps, const float* __restrict__ w, const float* __restrict__ bias,
                                                       float* __restrict__ logits, uint8_t* __restrict__ labels,
                                                       int rows, int ncls) {
  pdl_begin();
  __shared__ float s_a[C], s_b[C];       // per-image affine: y = x*a + b
  __shared__ float s_w[8 * C], s_bias[8];
  const int b = blockIdx.y;
  for (int c = threadIdx.x; c < C; c += 256) {
    const float mean = sums[(static_cast<long long>(b) * C + c) * 2] / rows;
    const float var = sums[(static_cast<long long>(b) * C + c) * 2 + 1] / rows;   // centred second moment (b2u_in_stats)
    const float a = rsqrtf(var + eps) * gamma[c];
    s_a[c] = a;
    s_b[c] = beta[c] - mean * a;
  }
  for (int i = threadIdx.x; i < ncls * C; i += 256) s_w[i] = w[i];
  if (threadIdx.x < ncls) s_bias[threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  const int p = blockIdx.x * 256 + threadIdx.x;
  if (p >= rows) return;
  const T* xp = x + (static_cast<long long>(b) * rows + p) * C;
  float acc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) acc[k] = k < ncls ? s_bias[k] : -INFINITY;
#pragma unroll
  for (int g = 0; g < C / 8; ++g) {
    Vec8<T> v;
    v.load(xp + g * 8);
    float f[8];
    v.to_float(f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float t = f[j] * s_a[g * 8 + j] + s_b[g * 8 + j];
      t = t > 0.f ? t : 0.01f * t;
      t = T16<T>::to_f(T16<T>::from_f(t));  // the normalised activation is a 16-bit tensor in the reference regime
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (k < ncls) acc[k] = fmaf(t, s_w[k * C + g * 8 + j], acc[k]);
    }
  }
  int best = 0;
  float bv = acc[0];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (k < ncls) {
      logits[(static_cast<long long>(b) * ncls + k) * rows + p] = acc[k];
      if (acc[k] > bv) { bv = acc[k]; best = k; }
    }
  }
  if (labels) labels[static_cast<long long>(b) * rows + p] = static_cast<uint8_t>(best);
}

extern "C" int b2u_seg_head(const void* x, const float* sums, const float* gamma, const float* beta, float eps,
                            const float* w, const float* b, float* logits, uint8_t* labels, int32_t B, int32_t rows,
                            int32_t C, int32_t ncls, int32_t dtype, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  // C = 32: the last decoder stage (seg_layers[-1]); 64 / 128: the deep-supervision heads on the earlier stages
  if (C != 32 && C != 64 && C != 128) return set_error(-1, "b2u_seg_head: C must be 32, 64 or 128 (features_per_stage[:3])");
  if (ncls < 1 || ncls * C > kSegMaxClasses * 32)
    return set_error(-1, "b2u_seg_head: 1 <= ncls <= %d at C=%d", kSegMaxClasses * 32 / C, C);
  dim3 grid((rows + 255) / 256, B);
#define B2U_SEG_HEAD(CC)                                                                                                         \
  if (ncls <= 8) {                                                                                                              \
    B2U_DISPATCH_T(dtype, (launch_pdl(seg_head_kernel8<T, CC>, grid, 256, 0, stream, static_cast<const T*>(x), sums, gamma, beta, eps, w, b, logits, labels, rows, ncls))); \
  } else {                                                                                                                      \
    B2U_DISPATCH_T(dtype, (launch_pdl(seg_head_kernel<T, CC>, grid, 256, 0, stream, static_cast<const T*>(x), sums, gamma, beta, eps, w, b, logits, labels, rows, ncls))); \
  }
  if (C == 32) {
    B2U_SEG_HEAD(32)
  } else if (C == 64) {
    B2U_SEG_HEAD(64)
  } else {
    B2U_SEG_HEAD(128)
  }
#undef B2U_SEG_HEAD
  return check_launch("seg_head");
}

}  // namespace b2u
