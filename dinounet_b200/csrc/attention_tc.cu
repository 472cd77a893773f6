// Host entry points of the wgmma flash attention (kernel: attention_tc3.cu) and its few-row companion kernel.
// Replaces F.scaled_dot_product_attention at dinounet/dinov3/layers/attention.py:116.
#include <type_traits>

#include "common.cuh"
#include "../../include/dinounet_b200.h"
#include "host_util.h"
#include "gemm_common.h"
#include "attention_common.h"

namespace b2u {

static int make_map_3d(CUtensorMap* map, const void* base, int dtype, uint64_t d0, uint64_t d1, uint64_t d2,
                       uint64_t stride1_elems, uint64_t stride2_elems, uint32_t b0, uint32_t b1) {
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {stride1_elems * 2, stride2_elems * 2};
  cuuint32_t box[3] = {b0, b1, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  return encode_tensor_map(map, dtype, 3, base, dims, strides, box, estr);
}

// ---- few-row companion (the cls/storage prefix rows): one CTA per (batch, head), up to 8 query rows -----------------
// phase 1: thread <-> key: each K row is read once (8 x 16 B) and dotted with all query rows (smem broadcast);
// phase 2: exact fp32 softmax per row (block reductions); phase 3: thread <-> (d, key quarter) streams V^T rows
// (keys contiguous) against the probabilities in smem; the 4 key quarters are reduced through smem.
constexpr int AR_MAXROWS = 8;
template <typename T>
__global__ void __launch_bounds__(256) attn_rows_kernel(const T* __restrict__ q, const T* __restrict__ k,
                                                        const T* __restrict__ vt, T* __restrict__ out, int heads, int ntok,
                                                        int npad, int row_begin, int nrows, float scale_log2e) {
  extern __shared__ float smf[];
  float* sq = smf;                                   // [8][64]
  float* sp = sq + AR_MAXROWS * 64;                  // [8][npad]
  float* red = sp + AR_MAXROWS * npad;               // [8][8]  per-warp partials, then [8] results in red[0..7]
  float* res = red + AR_MAXROWS * 8;                 // [8] row max, later row sum
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int bh = blockIdx.x;
  const T* kb = k + static_cast<size_t>(bh) * ntok * 64;
  const T* vb = vt + static_cast<size_t>(bh) * 64 * npad;
  for (int i = tid; i < nrows * 64; i += 256)
    sq[i] = T16<T>::to_f(q[(static_cast<size_t>(bh) * ntok + row_begin + (i >> 6)) * 64 + (i & 63)]);
  __syncthreads();
  // ---- phase 1: scores.  lane = (key-in-group-of-4, 16-byte chunk): every warp load is 512 contiguous bytes of K;
  // the 8 lanes of a key reduce their partial dot products with shuffles.
  float mx[AR_MAXROWS];
#pragma unroll
  for (int r = 0; r < AR_MAXROWS; ++r) mx[r] = -INFINITY;
  {
    const int kq = lane >> 3, ch = lane & 7;
    float qv[AR_MAXROWS][8];
#pragma unroll
    for (int r = 0; r < AR_MAXROWS; ++r)
#pragma unroll
      for (int e = 0; e < 8; ++e) qv[r][e] = r < nrows ? sq[r * 64 + ch * 8 + e] : 0.f;
    for (int k0 = warp * 4; k0 < ntok; k0 += 32) {
      const int key = k0 + kq;
      uint4 u = make_uint4(0, 0, 0, 0);
      if (key < ntok) u = __ldg(reinterpret_cast<const uint4*>(kb + static_cast<size_t>(key) * 64) + ch);
      const float2 a = T16<T>::unpack2(u.x), b = T16<T>::unpack2(u.y), c = T16<T>::unpack2(u.z), d = T16<T>::unpack2(u.w);
      const float kv[8] = {a.x, a.y, b.x, b.y, c.x, c.y, d.x, d.y};
#pragma unroll
      for (int r = 0; r < AR_MAXROWS; ++r) {
        if (r < nrows) {
          float sc = 0.f;
#pragma unroll
          for (int e = 0; e < 8; ++e) sc = fmaf(qv[r][e], kv[e], sc);
          sc += __shfl_xor_sync(0xffffffffu, sc, 1);
          sc += __shfl_xor_sync(0xffffffffu, sc, 2);
          sc += __shfl_xor_sync(0xffffffffu, sc, 4);
          if (ch == 0 && key < ntok) {
            const float v = sc * scale_log2e;
            sp[r * npad + key] = v;
            mx[r] = fmaxf(mx[r], v);
          }
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < AR_MAXROWS; ++r) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], o));
    if (lane == 0) red[r * 8 + warp] = mx[r];
  }
  __syncthreads();
  if (tid < AR_MAXROWS) {
    float m = red[tid * 8];
    for (int w = 1; w < 8; ++w) m = fmaxf(m, red[tid * 8 + w]);
    res[tid] = m;
  }
  __syncthreads();
  // ---- phase 2: probabilities (16-bit rounded for the PV product, like the MMA path) and fp32 row sums
  float sm[AR_MAXROWS];
#pragma unroll
  for (int r = 0; r < AR_MAXROWS; ++r) sm[r] = 0.f;
  for (int key = tid; key < npad; key += 256) {
#pragma unroll
    for (int r = 0; r < AR_MAXROWS; ++r) {
      if (r < nrows) {
        float e = 0.f;
        if (key < ntok) { e = ex2(sp[r * npad + key] - res[r]); sm[r] += e; }
        sp[r * npad + key] = T16<T>::to_f(T16<T>::from_f(e));
      }
    }
  }
  __syncthreads();   // everyone has read res[] (row max) before it is reused for the sums
#pragma unroll
  for (int r = 0; r < AR_MAXROWS; ++r) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sm[r] += __shfl_xor_sync(0xffffffffu, sm[r], o);
    if (lane == 0) red[r * 8 + warp] = sm[r];
  }
  __syncthreads();
  if (tid < AR_MAXROWS) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += red[tid * 8 + w];
    res[tid] = t;
  }
  __syncthreads();
  // ---- phase 3: O[r][d] = sum_key p[r][key] * V^T[d][key].  One warp per d row at a time, lane = 8-key chunk: every
  // warp load is 512 contiguous bytes of the V^T row; per-row partials are reduced with shuffles.
  const int b = bh / heads, hd = bh - b * heads;
  for (int d = warp; d < 64; d += 8) {
    const T* vr = vb + static_cast<size_t>(d) * npad;
    float acc[AR_MAXROWS];
#pragma unroll
    for (int r = 0; r < AR_MAXROWS; ++r) acc[r] = 0.f;
    for (int key = lane * 8; key < npad; key += 256) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(vr + key));
      const float2 a = T16<T>::unpack2(u.x), bb = T16<T>::unpack2(u.y), c = T16<T>::unpack2(u.z), dd = T16<T>::unpack2(u.w);
      const float vv[8] = {a.x, a.y, bb.x, bb.y, c.x, c.y, dd.x, dd.y};
#pragma unroll
      for (int r = 0; r < AR_MAXROWS; ++r) {
        if (r < nrows) {
          const float4 p0 = *reinterpret_cast<const float4*>(sp + r * npad + key);
          const float4 p1 = *reinterpret_cast<const float4*>(sp + r * npad + key + 4);
          acc[r] = fmaf(p0.x, vv[0], acc[r]); acc[r] = fmaf(p0.y, vv[1], acc[r]); acc[r] = fmaf(p0.z, vv[2], acc[r]);
          acc[r] = fmaf(p0.w, vv[3], acc[r]); acc[r] = fmaf(p1.x, vv[4], acc[r]); acc[r] = fmaf(p1.y, vv[5], acc[r]);
          acc[r] = fmaf(p1.z, vv[6], acc[r]); acc[r] = fmaf(p1.w, vv[7], acc[r]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < AR_MAXROWS; ++r) {
      if (r < nrows) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
        if (lane == 0)
          out[(static_cast<size_t>(b) * ntok + row_begin + r) * (heads * 64) + hd * 64 + d] = T16<T>::from_f(acc[r] / res[r]);
      }
    }
  }
}

extern "C" int b2u_attention_rows(const void* q, const void* k, const void* vt, void* out, int32_t B, int32_t heads,
                                  int32_t ntok, int32_t npad, int32_t row_begin, int32_t nrows, float scale, int32_t dtype,
                                  b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!q || !k || !vt || !out) return set_error(-1, "b2u_attention_rows: null pointer");
  if (nrows <= 0) return 0;
  if (npad % 8 || npad < ntok || row_begin < 0 || row_begin + nrows > ntok) return set_error(-1, "b2u_attention_rows: bad range");
  if (nrows > AR_MAXROWS) return set_error(-1, "b2u_attention_rows: at most 8 rows");
  const size_t smem = (static_cast<size_t>(AR_MAXROWS) * (64 + npad + 8 + 1) + 4 * AR_MAXROWS * 64) * sizeof(float);
  if (smem > 200 * 1024) return set_error(-1, "b2u_attention_rows: ntok too large for the few-row kernel");
  static bool configured[128] = {};
  const int di = current_device_index() * 2 + (dtype == B2U_BF16 ? 1 : 0);
  if (!configured[di]) {
    cudaError_t e = dtype == B2U_BF16
                        ? cudaFuncSetAttribute(attn_rows_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)
                        : cudaFuncSetAttribute(attn_rows_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) return set_error(-2, "cudaFuncSetAttribute(attn_rows): %s", cudaGetErrorString(e));
    configured[di] = true;
  }
  const float sl2 = scale * 1.4426950408889634f;
  if (dtype == B2U_BF16)
    attn_rows_kernel<__nv_bfloat16><<<B * heads, 256, smem, stream>>>(
        static_cast<const __nv_bfloat16*>(q), static_cast<const __nv_bfloat16*>(k), static_cast<const __nv_bfloat16*>(vt),
        static_cast<__nv_bfloat16*>(out), heads, ntok, npad, row_begin, nrows, sl2);
  else
    attn_rows_kernel<__half><<<B * heads, 256, smem, stream>>>(
        static_cast<const __half*>(q), static_cast<const __half*>(k), static_cast<const __half*>(vt),
        static_cast<__half*>(out), heads, ntok, npad, row_begin, nrows, sl2);
  return check_launch("attention_rows");
}

static int attention_tc_impl(const void* q, const void* k, const void* vt, void* out, int B, int heads, int ntok, int npad,
                             int q_begin, int head_dim, float scale, int dtype, cudaStream_t stream) {
  if (!q || !k || !vt || !out) return set_error(-1, "b2u_attention_tc: null pointer");
  if (npad % 8 || npad < ntok) return set_error(-1, "b2u_attention_tc: npad must be a multiple of 8 and >= ntok");
  if (head_dim != 64 && head_dim != 128) return set_error(-1, "b2u_attention_tc: head_dim must be 64 or 128");
  if (q_begin < 0 || q_begin >= ntok) return set_error(-1, "b2u_attention_tc: bad q_begin");
  AttnMaps maps;
  AttnArgs a{};
  a.BH = B * heads;
  a.heads = heads;
  a.ntok = ntok;
  a.q_begin = q_begin;
  a.nchunks = (ntok + 127) / 128;
  const int rows = attention_tc3_tile_rows(head_dim);
  a.qtiles = (ntok - q_begin + rows - 1) / rows;
  a.items = static_cast<long long>(a.BH) * a.qtiles;
  a.scale_log2e = scale * 1.4426950408889634f;
  a.out = out;
  int rc;
  const uint64_t BH = static_cast<uint64_t>(a.BH), hd = static_cast<uint64_t>(head_dim);
  const uint32_t kc = 128u;
  if ((rc = make_map_3d(&maps.q, q, dtype, hd, ntok, BH, hd, static_cast<uint64_t>(ntok) * hd, 64, static_cast<uint32_t>(rows)))) return rc;
  if ((rc = make_map_3d(&maps.k, k, dtype, hd, ntok, BH, hd, static_cast<uint64_t>(ntok) * hd, 64, kc))) return rc;
  if ((rc = make_map_3d(&maps.vt, vt, dtype, npad, hd, BH, npad, static_cast<uint64_t>(npad) * hd, 64, static_cast<uint32_t>(head_dim)))) return rc;
  return attention_tc3_dispatch(maps, a, head_dim, dtype, stream);
}

extern "C" int b2u_attention_tc(const void* q, const void* k, const void* vt, void* out, int32_t B, int32_t heads,
                                int32_t ntok, int32_t npad, int32_t q_begin, float scale, int32_t dtype,
                                b2u_stream_t stream_) {
  return attention_tc_impl(q, k, vt, out, B, heads, ntok, npad, q_begin, 64, scale, dtype, static_cast<cudaStream_t>(stream_));
}

extern "C" int b2u_attention_tc_hd(const void* q, const void* k, const void* vt, void* out, int32_t B, int32_t heads,
                                   int32_t ntok, int32_t npad, int32_t head_dim, float scale, int32_t dtype,
                                   b2u_stream_t stream_) {
  return attention_tc_impl(q, k, vt, out, B, heads, ntok, npad, 0, head_dim, scale, dtype, static_cast<cudaStream_t>(stream_));
}

}  // namespace b2u
