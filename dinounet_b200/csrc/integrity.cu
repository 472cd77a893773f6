// Dataset integrity check on the device (reference: experiment_planning/verify_dataset_integrity.py:32-116, the array
// checks of `verify_labels` and `check_cases`).
//
//   b2u_vi_scan  one read of a case: its images (fp32, every channel) for NaN and +-inf, and its seg (the stored dtype)
//                for the voxels that are not an integral value in [lo, hi] and, for a float32 seg, NaN.  The reference
//                asserts that the expected labels are consecutive, so `i not in expected_labels` is exactly this range
//                test (-0.0 compares equal to 0, NaN is in no range).
//
// Integer segs are compared in an unsigned "biased" domain (v - min(T)), where membership of [lo, hi] is one modular
// subtraction and one unsigned compare; 8- and 16-bit segs do that on 4 / 2 voxels at once with the SIMD-in-a-word
// intrinsics, so a uint8 seg costs about one instruction per 4 voxels and the scan stays bound by memory.  Loads are
// 16 bytes where the base pointer allows (a scalar head and tail otherwise), grid-stride; warp reductions and at most
// one atomic per block and result word (none for a clean case).
#include <algorithm>
#include <climits>
#include <cmath>

#include "../../include/dinounet_b200.h"
#include "host_util.h"

namespace b2u {

constexpr int kViThreads = 256;
constexpr int kViBlocksPerSm = 8;

// Integer seg of T: the biased value u = v - min(T) (v ^ sign bit for signed T); a voxel offends iff
// ((u - lo) mod 2^bits) > span, with lo / span the clamped expected range in the same domain (or always, with all).
template <typename T>
struct ViInt {
  static constexpr int kBits = 8 * sizeof(T);
  static constexpr unsigned kMask = kBits == 32 ? 0xffffffffu : ((1u << kBits) - 1u);
  static constexpr unsigned kBias = (T(-1) < T(0)) ? (1u << (kBits - 1)) : 0u;
};

struct ViRange {
  unsigned lo;    // biased lower bound, replicated into every lane of a word for 8 / 16-bit T
  unsigned span;  // hi - lo, replicated likewise
  int all;        // the expected range misses T's range: every voxel offends
  double flo, fhi;  // float32 seg: [lo, hi]
};

template <typename T>
__device__ __forceinline__ unsigned vi_one(T v, const ViRange& r, unsigned&) {
  using I = ViInt<T>;
  const unsigned u = (static_cast<unsigned>(v) ^ I::kBias) & I::kMask;
  return r.all ? 1u : static_cast<unsigned>(((u - (r.lo & I::kMask)) & I::kMask) > (r.span & I::kMask));
}

template <>
__device__ __forceinline__ unsigned vi_one<float>(float v, const ViRange& r, unsigned& flags) {
  if (isnan(v)) flags |= B2U_VI_SEG_NAN;
  const double d = v;
  return static_cast<unsigned>(!(d >= r.flo && d <= r.fhi && d == floor(d)));
}

// The offenders among the 16 / sizeof(T) voxels of one 16-byte word.
template <typename T>
__device__ __forceinline__ unsigned vi_word(const uint4& w, const ViRange& r, unsigned& flags) {
  const unsigned x[4] = {w.x, w.y, w.z, w.w};
  unsigned bad = 0;
  if constexpr (sizeof(T) == 1) {
    const unsigned bias = ViInt<T>::kBias * 0x01010101u;
#pragma unroll
    for (int k = 0; k < 4; ++k) bad += __popc(__vcmpgtu4(__vsub4(x[k] ^ bias, r.lo), r.span)) >> 3;
    return r.all ? 16u : bad;
  } else if constexpr (sizeof(T) == 2) {
    const unsigned bias = ViInt<T>::kBias * 0x00010001u;
#pragma unroll
    for (int k = 0; k < 4; ++k) bad += __popc(__vcmpgtu2(__vsub2(x[k] ^ bias, r.lo), r.span)) >> 4;
    return r.all ? 8u : bad;
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      T v;
      memcpy(&v, &x[k], sizeof(T));
      bad += vi_one<T>(v, r, flags);
    }
    return bad;
  }
}

__device__ __forceinline__ unsigned vi_image_flags(float v) {
  return (isnan(v) ? B2U_VI_IMAGE_NAN : 0u) | (isinf(v) ? B2U_VI_IMAGE_INF : 0u);
}

// The scalar head (up to the first 16-byte boundary) and tail of x[n], and the number of whole words between.
template <typename T>
__device__ __forceinline__ void vi_split(const T* x, long long n, long long& head, long long& words) {
  constexpr int V = 16 / sizeof(T);
  head = static_cast<long long>(((16u - (reinterpret_cast<uintptr_t>(x) & 15u)) & 15u) / sizeof(T));
  if (head > n) head = n;
  words = (n - head) / V;
}

template <typename T>
__global__ void __launch_bounds__(kViThreads) b2u_vi_scan(const float* __restrict__ img, long long n_img,
                                                          const T* __restrict__ seg, long long n_seg, ViRange r,
                                                          b2u_vi_result* __restrict__ out) {
  const long long tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
  unsigned flags = 0, bad = 0;

  long long head, words;
  if (n_img > 0) {
    vi_split(img, n_img, head, words);
    const float4* v = reinterpret_cast<const float4*>(img + head);
    for (long long i = tid; i < words; i += nthreads) {
      const float4 q = __ldcs(v + i);
      flags |= vi_image_flags(q.x) | vi_image_flags(q.y) | vi_image_flags(q.z) | vi_image_flags(q.w);
    }
    for (long long i = tid; i < head; i += nthreads) flags |= vi_image_flags(img[i]);
    for (long long i = head + words * 4 + tid; i < n_img; i += nthreads) flags |= vi_image_flags(img[i]);
  }

  constexpr int V = 16 / sizeof(T);
  vi_split(seg, n_seg, head, words);
  const uint4* s = reinterpret_cast<const uint4*>(seg + head);
  for (long long i = tid; i < words; i += nthreads) bad += vi_word<T>(__ldcs(s + i), r, flags);
  for (long long i = tid; i < head; i += nthreads) bad += vi_one<T>(seg[i], r, flags);
  for (long long i = head + words * V + tid; i < n_seg; i += nthreads) bad += vi_one<T>(seg[i], r, flags);

  bad = __reduce_add_sync(0xffffffffu, bad);
  flags = __reduce_or_sync(0xffffffffu, flags);
  __shared__ unsigned s_bad[kViThreads / 32], s_flags[kViThreads / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    s_bad[warp] = bad;
    s_flags[warp] = flags;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long total = 0;
    unsigned f = 0;
#pragma unroll
    for (int k = 0; k < kViThreads / 32; ++k) {
      total += s_bad[k];
      f |= s_flags[k];
    }
    if (total) atomicAdd(reinterpret_cast<unsigned long long*>(&out->offenders), total);
    if (f) atomicOr(&out->flags, f);
  }
}

// [lo, hi] clamped to T's range in the biased domain, replicated into the lanes of a 32-bit word for 8 / 16-bit T.
template <typename T>
ViRange int_range(int64_t lo, int64_t hi) {
  using I = ViInt<T>;
  const long long tmin = I::kBias ? -static_cast<long long>(I::kBias) : 0;
  const long long tmax = tmin + static_cast<long long>(I::kMask);
  ViRange r{};
  const long long a = lo < tmin ? tmin : lo, b = hi > tmax ? tmax : hi;
  if (a > b) {
    r.all = 1;
    return r;
  }
  unsigned l = static_cast<unsigned>(a - tmin), span = static_cast<unsigned>(b - a);
  if (sizeof(T) == 1) {
    l *= 0x01010101u;
    span *= 0x01010101u;
  } else if (sizeof(T) == 2) {
    l *= 0x00010001u;
    span *= 0x00010001u;
  }
  r.lo = l;
  r.span = span;
  return r;
}

template <typename T>
int launch_scan(const float* img, int64_t n_img, const void* seg, int64_t n_seg, const ViRange& r,
                b2u_vi_result* out, cudaStream_t stream) {
  static int sms[64] = {};
  const int dev = current_device_index();
  if (!sms[dev]) {
    int cur = 0, count = 0;
    cudaGetDevice(&cur);
    if (cudaDeviceGetAttribute(&count, cudaDevAttrMultiProcessorCount, cur) != cudaSuccess || count <= 0)
      return set_error(-1, "b2u_vi_scan: cannot read the SM count");
    sms[dev] = count;
  }
  const long long work = std::max<long long>((n_img + 3) / 4, (n_seg + 16 / sizeof(T) - 1) / (16 / sizeof(T)));
  const long long want = (work + kViThreads - 1) / kViThreads;
  const int blocks = static_cast<int>(std::max<long long>(1, std::min<long long>(want, 1LL * sms[dev] * kViBlocksPerSm)));
  b2u_vi_scan<T><<<blocks, kViThreads, 0, stream>>>(img, n_img, static_cast<const T*>(seg), n_seg, r, out);
  return check_launch("vi_scan");
}

}  // namespace b2u

using namespace b2u;

extern "C" int b2u_vi_scan(const float* img, int64_t n_img, const void* seg, int32_t dtype, int64_t n_seg, int64_t lo,
                           int64_t hi, b2u_vi_result* result, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!seg || !result || (n_img > 0 && !img)) return set_error(-1, "b2u_vi_scan: null pointer");
  if (n_img < 0 || n_seg <= 0 || n_seg >= (1LL << 31) || lo > hi)
    return set_error(-1, "b2u_vi_scan: n_img=%lld n_seg=%lld lo=%lld hi=%lld", static_cast<long long>(n_img),
                     static_cast<long long>(n_seg), static_cast<long long>(lo), static_cast<long long>(hi));
  static const int kSize[6] = {1, 1, 2, 2, 4, 4};
  if (dtype < B2U_EVAL_U8 || dtype > B2U_EVAL_F32) return set_error(-1, "b2u_vi_scan: seg dtype code %d", dtype);
  if ((reinterpret_cast<uintptr_t>(img) & 3u) || (reinterpret_cast<uintptr_t>(seg) & (kSize[dtype] - 1)))
    return set_error(-1, "b2u_vi_scan: a base pointer is not aligned to its element size");
  if (cudaMemsetAsync(result, 0, sizeof(b2u_vi_result), stream) != cudaSuccess)
    return set_error(-1, "b2u_vi_scan: cudaMemsetAsync failed: %s", cudaGetErrorString(cudaGetLastError()));
  switch (dtype) {
    case B2U_EVAL_U8: return launch_scan<uint8_t>(img, n_img, seg, n_seg, int_range<uint8_t>(lo, hi), result, stream);
    case B2U_EVAL_I8: return launch_scan<int8_t>(img, n_img, seg, n_seg, int_range<int8_t>(lo, hi), result, stream);
    case B2U_EVAL_I16: return launch_scan<int16_t>(img, n_img, seg, n_seg, int_range<int16_t>(lo, hi), result, stream);
    case B2U_EVAL_U16:
      return launch_scan<uint16_t>(img, n_img, seg, n_seg, int_range<uint16_t>(lo, hi), result, stream);
    case B2U_EVAL_I32: return launch_scan<int32_t>(img, n_img, seg, n_seg, int_range<int32_t>(lo, hi), result, stream);
    default: {
      ViRange r{};
      r.flo = static_cast<double>(lo);
      r.fhi = static_cast<double>(hi);
      return launch_scan<float>(img, n_img, seg, n_seg, r, result, stream);
    }
  }
}
