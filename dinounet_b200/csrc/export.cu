// Prediction export on the device (reference: inference/export_prediction.py:15-68).
//
// b2u_export_resample_f16 is `resampling_fn_probabilities` of a 2D configuration: resample_data_or_seg_to_shape with
// order 1 (default_resampling.py), i.e. `data.astype(float)`, skimage `resize(order=1, mode='edge',
// anti_aliasing=False)` = scipy `ndimage.zoom(order=1, mode='nearest', grid_mode=True)` in float64, then
// `.astype(float16)`.  The arithmetic is scipy's NI_ZoomShift, operation for operation, so results are bit-identical:
//   cc = (k + 0.5) * (n_in / n_out) - 0.5          (no clamping of cc for mode 'nearest')
//   w0 = 1 - (cc - floor(cc)),  w1 = 1 - w0         (order-1 spline weights)
//   taps floor(cc), floor(cc) + 1, each index clamped to [0, n_in - 1]
//   t = 0.0;  t += v[y0][x0] * wy0 * wx0;  t += v[y0][x1] * wy0 * wx1;  t += v[y1][x0] * wy1 * wx0;  t += v[y1][x1] * wy1 * wx1
// Every product and sum is an explicit round-to-nearest fp64 intrinsic, so nvcc contracts nothing into an FMA.  With Z
// unchanged the reference's 3D zoom multiplies each tap by a z weight of exactly 1 and adds taps of weight 0, so for
// finite logits it equals this per-slice form (a non-finite neighbour slice would turn those zero taps into NaN there).
//
// b2u_export_segment is LabelManager.apply_inference_nonlin + convert_probabilities_to_segmentation
// (utilities/label_handling/label_handling.py:128-175) on fp16 logits: fp32 softmax over channels and the first maximum,
// or fp32 sigmoid and `p > 0.5` painted in channel order.
#include <cuda_fp16.h>

#include <algorithm>
#include <utility>

#include "../../include/dinounet_b200.h"
#include "common.cuh"
#include "gemm_common.h"
#include "host_util.h"

namespace b2u {

struct AxisTaps {
  int i0, i1;
  double w0, w1;
};

__device__ __forceinline__ AxisTaps zoom_taps(int k, int n_in, double zoom) {
  const double cc = __dsub_rn(__dmul_rn(__dadd_rn(static_cast<double>(k), 0.5), zoom), 0.5);
  const double fl = floor(cc);
  AxisTaps t;
  t.w0 = __dsub_rn(1.0, __dsub_rn(cc, fl));
  t.w1 = __dsub_rn(1.0, t.w0);
  const int s = static_cast<int>(fl);
  t.i0 = min(max(s, 0), n_in - 1);
  t.i1 = min(max(s + 1, 0), n_in - 1);
  return t;
}

__device__ __forceinline__ double tap(const __half* p, double wy, double wx) {
  return __dmul_rn(__dmul_rn(static_cast<double>(__half2float(*p)), wy), wx);
}

// One output row Y per blockIdx.y, columns over blockIdx.x * blockDim.x; the [C * Z] planes are strided over blockIdx.z,
// so the axis taps of a (Y, X) pair are computed once and reused for every plane it visits.
__global__ void export_resample_kernel(const __half* __restrict__ in, __half* __restrict__ out, int planes, int h, int w,
                                       int H, int W, double zoom_y, double zoom_x) {
  const int X = blockIdx.x * blockDim.x + threadIdx.x;
  const int Y = blockIdx.y;
  if (X >= W) return;
  const AxisTaps ty = zoom_taps(Y, h, zoom_y), tx = zoom_taps(X, w, zoom_x);
  const long long in_plane = static_cast<long long>(h) * w, out_plane = static_cast<long long>(H) * W;
  const int r0 = ty.i0 * w, r1 = ty.i1 * w;
  for (int p = blockIdx.z; p < planes; p += gridDim.z) {
    const __half* src = in + p * in_plane;
    double t = 0.0;
    t = __dadd_rn(t, tap(src + r0 + tx.i0, ty.w0, tx.w0));
    t = __dadd_rn(t, tap(src + r0 + tx.i1, ty.w0, tx.w1));
    t = __dadd_rn(t, tap(src + r1 + tx.i0, ty.w1, tx.w0));
    t = __dadd_rn(t, tap(src + r1 + tx.i1, ty.w1, tx.w1));
    out[p * out_plane + static_cast<long long>(Y) * W + X] = __double2half(t);  // cvt.rn.f16.f64: one rounding
  }
}

// fp32 sigmoid(x) > 0.5 holds exactly for x >= 2^-23: for 0 < x <= 2^-24, exp(-x) rounds to 1 - 2^-24 and 1 + that ties
// to 2, so 1 / 2 = 0.5; at x = 2^-23, 1 / (2 - 2^-23) rounds up to 0.5 + 2^-24.  Deciding on x keeps the threshold
// independent of the last bit of expf.
#define B2U_SIGMOID_HALF_THRESHOLD 0x1p-23f

template <int C>
__global__ void __launch_bounds__(256) export_segment_kernel(const __half* __restrict__ logits, long long voxels,
                                                             int mode, const int32_t* __restrict__ region_labels,
                                                             void* __restrict__ labels, int label_bytes,
                                                             float* __restrict__ probs) {
  int rl[C];
  if (mode == 1) {
#pragma unroll
    for (int c = 0; c < C; ++c) rl[c] = region_labels[c];
  }
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long v = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; v < voxels; v += stride) {
    float x[C];
#pragma unroll
    for (int c = 0; c < C; ++c) x[c] = __half2float(logits[c * voxels + v]);
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
        if (probs) probs[c * voxels + v] = p;
        if (p > best) {  // strict: the first maximum wins, as torch.argmax
          best = p;
          lab = c;
        }
      }
    } else {
#pragma unroll
      for (int c = 0; c < C; ++c) {
        if (probs) probs[c * voxels + v] = __frcp_rn(__fadd_rn(1.f, expf(-x[c])));
        if (x[c] >= B2U_SIGMOID_HALF_THRESHOLD) lab = rl[c];
      }
    }
    if (label_bytes == 1)
      static_cast<uint8_t*>(labels)[v] = static_cast<uint8_t>(lab);
    else
      static_cast<uint16_t*>(labels)[v] = static_cast<uint16_t>(lab);
  }
}

using SegmentKernel = void (*)(const __half*, long long, int, const int32_t*, void*, int, float*);
constexpr int kMaxExportChannels = 32;

template <std::size_t... I>
static SegmentKernel segment_kernel_for(int C, std::index_sequence<I...>) {
  static const SegmentKernel table[] = {export_segment_kernel<static_cast<int>(I) + 1>...};
  return table[C - 1];
}

}  // namespace b2u

using namespace b2u;

extern "C" int b2u_export_resample_f16(const void* in, void* out, int32_t C, int32_t Z, int32_t h, int32_t w,
                                       int32_t H, int32_t W, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!in || !out) return set_error(-1, "b2u_export_resample_f16: null pointer");
  if (C <= 0 || Z <= 0 || h <= 0 || w <= 0 || H <= 0 || W <= 0 || H > 65535)
    return set_error(-1, "b2u_export_resample_f16: bad shape C=%d Z=%d %dx%d -> %dx%d", C, Z, h, w, H, W);
  const long long planes = static_cast<long long>(C) * Z;
  if (planes > (1LL << 30)) return set_error(-1, "b2u_export_resample_f16: %lld planes", planes);
  if (h == H && w == W) {  // the reference returns the array unchanged: copy bits, including -0 and NaN payloads
    if (in == out) return 0;
    cudaError_t e = cudaMemcpyAsync(out, in, static_cast<size_t>(planes) * h * w * sizeof(__half),
                                    cudaMemcpyDeviceToDevice, stream);
    if (e != cudaSuccess) return set_error(-11, "b2u_export_resample_f16: cudaMemcpyAsync: %s", cudaGetErrorString(e));
    return 0;
  }
  // numpy's n_in / n_out (ndimage.zoom with grid_mode=True): a correctly rounded host division
  const double zoom_y = static_cast<double>(h) / H, zoom_x = static_cast<double>(w) / W;
  const int xblocks = (W + 255) / 256;
  const long long want = static_cast<long long>(num_sms()) * 32;  // enough resident blocks without a long tail
  const long long rows = static_cast<long long>(xblocks) * H;
  const int zblocks = static_cast<int>(std::min<long long>(std::max<long long>((want + rows - 1) / rows, 1), std::min<long long>(planes, 65535)));
  export_resample_kernel<<<dim3(xblocks, H, zblocks), 256, 0, stream>>>(
      static_cast<const __half*>(in), static_cast<__half*>(out), static_cast<int>(planes), h, w, H, W, zoom_y, zoom_x);
  return check_launch("export_resample_f16");
}

extern "C" int b2u_export_segment(const void* logits, int32_t C, int64_t voxels, int32_t mode,
                                  const int32_t* region_labels, void* labels, int32_t label_bytes, float* probs,
                                  b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!logits || !labels) return set_error(-1, "b2u_export_segment: null pointer");
  if (C < 1 || C > kMaxExportChannels)
    return set_error(-1, "b2u_export_segment: C=%d outside 1..%d", C, kMaxExportChannels);
  if (voxels <= 0) return set_error(-1, "b2u_export_segment: voxels=%lld", static_cast<long long>(voxels));
  if (mode != 0 && mode != 1) return set_error(-1, "b2u_export_segment: mode %d is neither 0 (labels) nor 1 (regions)", mode);
  if (mode == 1 && !region_labels) return set_error(-1, "b2u_export_segment: region mode needs region_labels");
  if (label_bytes != 1 && label_bytes != 2)
    return set_error(-1, "b2u_export_segment: label_bytes %d is neither 1 nor 2", label_bytes);
  const int blocks = static_cast<int>(std::min<long long>((voxels + 255) / 256, static_cast<long long>(num_sms()) * 16));
  segment_kernel_for(C, std::make_index_sequence<kMaxExportChannels>{})<<<blocks, 256, 0, stream>>>(
      static_cast<const __half*>(logits), voxels, mode, region_labels, labels, label_bytes, probs);
  return check_launch("export_segment");
}
