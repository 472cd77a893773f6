// Ensembling of saved probabilities (reference: ensembling/ensemble.py:17-46, `merge_files`).
//
// b2u_ensemble_accumulate is `average_probabilities`' sum, operation for operation: the first member is converted to
// fp32 (`avg.astype(np.float32)`), every later one added with one fp32 add of its exact fp32 value (numpy's float32
// `+=` of an fp16 array upcasts first), so the sums are bit-identical to numpy's.
// b2u_ensemble_segment is the `avg /= n` that ends it (one correctly rounded fp32 division, in place) followed by
// `LabelManager.convert_logits_to_segmentation` of the average: the export's segment kernel (export_segment.cuh) on fp32
// input.
#include <cuda_fp16.h>

#include <algorithm>

#include "../../include/dinounet_b200.h"
#include "common.cuh"
#include "export_segment.cuh"
#include "gemm_common.h"
#include "host_util.h"

namespace b2u {

__device__ __forceinline__ void load8(const float* p, float (&v)[8]) {
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

__device__ __forceinline__ void load8(const __half* p, float (&v)[8]) {
  const uint4 raw = *reinterpret_cast<const uint4*>(p);
  const __half2* h = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __half22float2(h[i]);  // exact
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}

// Groups of 8 elements (16-byte loads of fp16, two of fp32, two 16-byte stores) when both pointers are 16-byte aligned;
// the tail, or everything when they are not, element by element.
template <typename T>
__global__ void __launch_bounds__(256) ensemble_accumulate_kernel(const T* __restrict__ src, float* __restrict__ acc,
                                                                  long long n, int first, int vec) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long groups = vec ? n / 8 : 0;
  for (long long g = tid; g < groups; g += stride) {
    float s[8];
    load8(src + g * 8, s);
    float4* out = reinterpret_cast<float4*>(acc + g * 8);
    if (!first) {
      const float4 a = out[0], b = out[1];
      s[0] = __fadd_rn(a.x, s[0]); s[1] = __fadd_rn(a.y, s[1]); s[2] = __fadd_rn(a.z, s[2]); s[3] = __fadd_rn(a.w, s[3]);
      s[4] = __fadd_rn(b.x, s[4]); s[5] = __fadd_rn(b.y, s[5]); s[6] = __fadd_rn(b.z, s[6]); s[7] = __fadd_rn(b.w, s[7]);
    }
    out[0] = make_float4(s[0], s[1], s[2], s[3]);
    out[1] = make_float4(s[4], s[5], s[6], s[7]);
  }
  for (long long i = groups * 8 + tid; i < n; i += stride) {
    const float x = load_as_float(src + i);
    acc[i] = first ? x : __fadd_rn(acc[i], x);
  }
}

}  // namespace b2u

using namespace b2u;

extern "C" int b2u_ensemble_accumulate(const void* src, int32_t src_bytes, float* acc, int64_t n, int32_t first,
                                       b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!src || !acc) return set_error(-1, "b2u_ensemble_accumulate: null pointer");
  if (src_bytes != 2 && src_bytes != 4)
    return set_error(-1, "b2u_ensemble_accumulate: src_bytes %d is neither 2 (fp16) nor 4 (fp32)", src_bytes);
  if (n <= 0) return set_error(-1, "b2u_ensemble_accumulate: n=%lld", static_cast<long long>(n));
  const int vec = (reinterpret_cast<uintptr_t>(src) % 16 == 0 && reinterpret_cast<uintptr_t>(acc) % 16 == 0) ? 1 : 0;
  const long long work = vec ? (n + 7) / 8 : n;
  const int blocks = static_cast<int>(std::min<long long>((work + 255) / 256, static_cast<long long>(num_sms()) * 8));
  if (src_bytes == 2)
    ensemble_accumulate_kernel<__half><<<blocks, 256, 0, stream>>>(static_cast<const __half*>(src), acc, n, first, vec);
  else
    ensemble_accumulate_kernel<float><<<blocks, 256, 0, stream>>>(static_cast<const float*>(src), acc, n, first, vec);
  return check_launch("ensemble_accumulate");
}

extern "C" int b2u_ensemble_segment(float* acc, int32_t C, int64_t voxels, int32_t n_members, int32_t mode,
                                    const int32_t* region_labels, void* labels, int32_t label_bytes,
                                    b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!acc || !labels) return set_error(-1, "b2u_ensemble_segment: null pointer");
  if (C < 1 || C > kMaxExportChannels)
    return set_error(-1, "b2u_ensemble_segment: C=%d outside 1..%d", C, kMaxExportChannels);
  if (voxels <= 0) return set_error(-1, "b2u_ensemble_segment: voxels=%lld", static_cast<long long>(voxels));
  if (n_members < 1 || n_members > (1 << 24))
    return set_error(-1, "b2u_ensemble_segment: n_members=%d outside 1..2^24", n_members);
  if (mode != 0 && mode != 1) return set_error(-1, "b2u_ensemble_segment: mode %d is neither 0 (labels) nor 1 (regions)", mode);
  if (mode == 1 && !region_labels) return set_error(-1, "b2u_ensemble_segment: region mode needs region_labels");
  if (label_bytes != 1 && label_bytes != 2)
    return set_error(-1, "b2u_ensemble_segment: label_bytes %d is neither 1 nor 2", label_bytes);
  return launch_segment<float, false>(static_cast<const float*>(acc), C, voxels, mode, region_labels, labels,
                                      label_bytes, nullptr, 0, acc, static_cast<float>(n_members), stream, "ensemble_segment");
}
