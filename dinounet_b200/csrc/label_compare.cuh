// numpy's `seg == label` for a label volume read in its stored dtype, shared by the evaluation (evaluation.cu) and the
// postprocessing (postprocessing.cu): integer dtypes compare exactly as int64 (a label outside the dtype's range
// matches nothing), float32 volumes compare with the label rounded to float32, as numpy casts a Python int to the
// array's dtype.  dtype codes: B2U_EVAL_U8, _I8, _I16, _U16, _I32, _F32.
#pragma once
#include <stdint.h>

#include "../../include/dinounet_b200.h"

namespace b2u {

__host__ __device__ __forceinline__ float label_as_f32(long long v) { return static_cast<float>(v); }

__device__ __forceinline__ long long load_int_label(const void* p, int dtype, long long i) {
  switch (dtype) {
    case B2U_EVAL_U8: return static_cast<const uint8_t*>(p)[i];
    case B2U_EVAL_I8: return static_cast<const int8_t*>(p)[i];
    case B2U_EVAL_I16: return static_cast<const int16_t*>(p)[i];
    case B2U_EVAL_U16: return static_cast<const uint16_t*>(p)[i];
    default: return static_cast<const int32_t*>(p)[i];
  }
}

// f is label_as_f32(v).
__device__ __forceinline__ bool equals(const void* p, int dtype, long long i, long long v, float f) {
  switch (dtype) {
    case B2U_EVAL_U8: return static_cast<const uint8_t*>(p)[i] == v;
    case B2U_EVAL_I8: return static_cast<const int8_t*>(p)[i] == v;
    case B2U_EVAL_I16: return static_cast<const int16_t*>(p)[i] == v;
    case B2U_EVAL_U16: return static_cast<const uint16_t*>(p)[i] == v;
    case B2U_EVAL_I32: return static_cast<const int32_t*>(p)[i] == v;
    default: return static_cast<const float*>(p)[i] == f;
  }
}

// Whether element i equals any of labels[0..n) (ascending, distinct int64) under the rule above: a binary search for
// the first label not below the value.  Rounding to float32 is monotone, so the rounded labels stay sorted (equal
// neighbours are harmless); a NaN voxel compares false everywhere and matches nothing.
__device__ __forceinline__ bool in_sorted_labels(const void* p, int dtype, long long i, const long long* labels, int n) {
  int lo = 0, hi = n;
  if (dtype == B2U_EVAL_F32) {
    const float x = static_cast<const float*>(p)[i];
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (label_as_f32(__ldg(labels + mid)) < x) lo = mid + 1; else hi = mid;
    }
    return lo < n && label_as_f32(__ldg(labels + lo)) == x;
  }
  const long long x = load_int_label(p, dtype, i);
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(labels + mid) < x) lo = mid + 1; else hi = mid;
  }
  return lo < n && __ldg(labels + lo) == x;
}

}  // namespace b2u
