// LabelManager.apply_inference_nonlin + convert_probabilities_to_segmentation (utilities/label_handling/
// label_handling.py:128-175) per voxel, shared by the prediction export (fp16 logits, export.cu) and the ensemble
// (fp32 averaged probabilities, ensemble.cu): fp32 softmax over channels and the first maximum, or fp32 sigmoid and
// `p > 0.5` painted in channel order.
#pragma once

#include <cuda_fp16.h>

#include <algorithm>
#include <cstdint>
#include <type_traits>
#include <utility>

#include "gemm_common.h"
#include "host_util.h"

namespace b2u {

// fp32 sigmoid(x) > 0.5 holds exactly for x > 1.5 * 2^-24 (torch's CPU sigmoid, every fp32 value checked): below it
// exp(-x) rounds to 1 - 2^-24 or above, 1 + that rounds to 2 and 1 / 2 = 0.5; from the next float up 1 + exp(-x) rounds
// below 2.  No fp16 value lies between 1.5 * 2^-24 and 2^-23, so fp16 logits get the same decision as `x >= 2^-23`.
// Deciding on x keeps the threshold independent of the last bit of expf.
#define B2U_SIGMOID_HALF_THRESHOLD 0x1.8p-24f

constexpr int kMaxExportChannels = 32;

__device__ __forceinline__ float load_as_float(const __half* p) { return __half2float(*p); }
__device__ __forceinline__ float load_as_float(const float* p) { return *p; }

// in: [C, voxels] fp16 logits (the export), or an fp32 sum of ensemble members' probabilities (the ensemble).
// ACCUMULATE false: labels = the segmentation, uint8 (label_bytes 1) or uint16 (2); probs (when non-NULL) = the
//   nonlinearity's output.  For fp32 input each voxel is first divided by `divisor` (one correctly rounded fp32
//   division) and the quotient, the ensemble's average, written back to avg, which may be `in`: each thread reads a
//   voxel before it writes it.
// ACCUMULATE true: probs += the nonlinearity's output (one fp32 add; first != 0 stores), no labels: one member of a
//   one-pass model ensemble.
template <typename T, int C, bool ACCUMULATE>
__global__ void __launch_bounds__(256, 1) export_segment_kernel(const T* in, long long voxels, int mode,
                                                             const int32_t* __restrict__ region_labels,
                                                             void* __restrict__ labels, int label_bytes,
                                                             float* __restrict__ probs, int first, float* avg,
                                                             float divisor) {
  int rl[C];
  if (!ACCUMULATE && mode == 1) {
#pragma unroll
    for (int c = 0; c < C; ++c) rl[c] = region_labels[c];
  }
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long v = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; v < voxels; v += stride) {
    float x[C];
#pragma unroll
    for (int c = 0; c < C; ++c) x[c] = load_as_float(in + c * voxels + v);
    if constexpr (std::is_same<T, float>::value) {
#pragma unroll
      for (int c = 0; c < C; ++c) {
        x[c] = __fdiv_rn(x[c], divisor);
        avg[c * voxels + v] = x[c];
      }
    }
    int lab = 0;
    if (mode == 0) {
      float m = x[0];
#pragma unroll
      for (int c = 1; c < C; ++c) m = fmaxf(m, x[c]);
      float s = 0.f;
#pragma unroll
      for (int c = 0; c < C; ++c) {
        x[c] = expf(__fsub_rn(x[c], m));
        s = __fadd_rn(s, x[c]);
      }
      float best = -1.f;
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const float p = __fdiv_rn(x[c], s);
        if (ACCUMULATE) {
          float* q = probs + c * voxels + v;
          *q = first ? p : __fadd_rn(*q, p);
        } else {
          if (probs) probs[c * voxels + v] = p;
          if (p > best) {  // strict: the first maximum wins, as torch.argmax
            best = p;
            lab = c;
          }
        }
      }
    } else {
#pragma unroll
      for (int c = 0; c < C; ++c) {
        if (ACCUMULATE) {
          const float p = __frcp_rn(__fadd_rn(1.f, expf(-x[c])));
          float* q = probs + c * voxels + v;
          *q = first ? p : __fadd_rn(*q, p);
        } else {
          if (probs) probs[c * voxels + v] = __frcp_rn(__fadd_rn(1.f, expf(-x[c])));
          if (x[c] > B2U_SIGMOID_HALF_THRESHOLD) lab = rl[c];
        }
      }
    }
    if (ACCUMULATE) continue;
    if (label_bytes == 1)
      static_cast<uint8_t*>(labels)[v] = static_cast<uint8_t>(lab);
    else
      static_cast<uint16_t*>(labels)[v] = static_cast<uint16_t>(lab);
  }
}

template <typename T>
using SegmentKernel = void (*)(const T*, long long, int, const int32_t*, void*, int, float*, int, float*, float);

template <typename T, bool ACCUMULATE, std::size_t... I>
static SegmentKernel<T> segment_kernel_for(int C, std::index_sequence<I...>) {
  static const SegmentKernel<T> table[] = {export_segment_kernel<T, static_cast<int>(I) + 1, ACCUMULATE>...};
  return table[C - 1];
}

// Launches the kernel for 1 <= C <= kMaxExportChannels (the caller checks), a grid-stride of at most 16 blocks per SM.
template <typename T, bool ACCUMULATE>
static int launch_segment(const T* in, int C, long long voxels, int mode, const int32_t* region_labels, void* labels,
                          int label_bytes, float* probs, int first, float* avg, float divisor, cudaStream_t stream,
                          const char* what) {
  const int blocks = static_cast<int>(std::min<long long>((voxels + 255) / 256, static_cast<long long>(num_sms()) * 16));
  segment_kernel_for<T, ACCUMULATE>(C, std::make_index_sequence<kMaxExportChannels>{})<<<blocks, 256, 0, stream>>>(
      in, voxels, mode, region_labels, labels, label_bytes, probs, first, avg, divisor);
  return check_launch(what);
}

}  // namespace b2u
