// nnUNetDataLoader2D's crop and padding on the device (reference: data_loader_2d.py:7-91 with the boxes of
// base_data_loader.py:64-134, and the validation transforms of nnUNetTrainer.py:778-805).  The host
// (dinounet_b200/dataloading.py) draws the keys, slices and boxes and stages, per sample, only the part of the box that
// lies inside the slice (`valid_bbox_lbs/ubs`): the data channels as float32 [C, h, w] and the seg as stored [h, w],
// int8 or int16 per sample (the preprocessor picks the type per case).  One launch places every sample at its offset (y0, x0) = (-min(0, bbox_lbs)) in the patch:
//   data     fp32 [B, C, H, W]: the staged values bit for bit inside the box, 0 outside (np.pad constant 0).
//   train    target int16 [B, 1, H, W]: the stored labels inside, -1 outside (np.pad constant -1).  Stored -1 values pass.
//   val      target fp32: RemoveLabelTransform(-1, 0), then the label map [B, 1, H, W] or, with a region table,
//            ConvertSegmentationToRegionsTransform [B, R, H, W] (region q is 1 where the label is one of its labels).
// One block row per plane (B*C data planes, then B target planes); each thread writes V consecutive pixels of a row
// with one vector store (V = 4, 2 or 1, the largest that divides W), consecutive threads consecutive vectors.
#include <algorithm>

#include "../../include/dinounet_b200.h"
#include "gemm_common.h"
#include "host_util.h"

namespace b2u {
namespace {

constexpr int kT = 256;

template <int V, typename T> struct Vec;
template <> struct Vec<4, float> { using type = float4; };
template <> struct Vec<2, float> { using type = float2; };
template <> struct Vec<1, float> { using type = float; };
template <> struct Vec<4, int16_t> { using type = short4; };
template <> struct Vec<2, int16_t> { using type = short2; };
template <> struct Vec<1, int16_t> { using type = short; };

template <int V, typename T>
__device__ __forceinline__ void store(T* dst, const T (&v)[V]) {
  typename Vec<V, T>::type u;
  T* w = reinterpret_cast<T*>(&u);
#pragma unroll
  for (int k = 0; k < V; ++k) w[k] = v[k];
  *reinterpret_cast<typename Vec<V, T>::type*>(dst) = u;
}

// desc: int64 [B, B2U_DL_DESC] {data byte offset, seg byte offset, y0, x0, h, w, seg bytes, 0} relative to `staged`.
template <typename S>
__device__ __forceinline__ int seg_at(const char* base, long long idx) {
  return static_cast<int>(reinterpret_cast<const S*>(base)[idx]);
}

template <int V>
__global__ void __launch_bounds__(kT) crop_kernel(const char* __restrict__ staged, const long long* __restrict__ desc,
                                                  int B, int C, int H, int W, int val,
                                                  const int32_t* __restrict__ regions, int R,
                                                  float* __restrict__ data, void* __restrict__ target) {
  const int p = blockIdx.x;
  const bool is_data = p < B * C;
  const int b = is_data ? p / C : p - B * C;
  const long long* d = desc + static_cast<long long>(b) * B2U_DL_DESC;
  const int y0 = static_cast<int>(d[2]), x0 = static_cast<int>(d[3]);
  const int h = static_cast<int>(d[4]), w = static_cast<int>(d[5]);
  const int Wv = W / V;
  const long long hw = static_cast<long long>(H) * W, nv = static_cast<long long>(H) * Wv;
  const long long stride = static_cast<long long>(gridDim.y) * kT;
  for (long long e = static_cast<long long>(blockIdx.y) * kT + threadIdx.x; e < nv; e += stride) {
    const int i = static_cast<int>(e / Wv), j0 = static_cast<int>(e - static_cast<long long>(i) * Wv) * V;
    const int yi = i - y0;
    const bool row_in = static_cast<unsigned>(yi) < static_cast<unsigned>(h);
    const long long dst = static_cast<long long>(i) * W + j0;
    if (is_data) {
      const float* src = reinterpret_cast<const float*>(staged + d[0]) + (static_cast<long long>(p % C) * h + yi) * w;
      float v[V];
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const int x = j0 + k - x0;
        v[k] = row_in && static_cast<unsigned>(x) < static_cast<unsigned>(w) ? src[x] : 0.f;
      }
      store<V, float>(data + static_cast<long long>(p) * hw + dst, v);
      continue;
    }
    const char* src = staged + d[1];
    const bool i8 = d[6] == 1;
    int s[V];
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const int x = j0 + k - x0;
      const long long at = static_cast<long long>(yi) * w + x;
      s[k] = !(row_in && static_cast<unsigned>(x) < static_cast<unsigned>(w)) ? -1
             : i8 ? seg_at<int8_t>(src, at) : seg_at<int16_t>(src, at);
    }
    if (!val) {
      int16_t t[V];
#pragma unroll
      for (int k = 0; k < V; ++k) t[k] = static_cast<int16_t>(s[k]);
      store<V, int16_t>(static_cast<int16_t*>(target) + static_cast<long long>(b) * hw + dst, t);
      continue;
    }
#pragma unroll
    for (int k = 0; k < V; ++k) s[k] = s[k] == -1 ? 0 : s[k];
    if (R == 0) {
      float t[V];
#pragma unroll
      for (int k = 0; k < V; ++k) t[k] = static_cast<float>(s[k]);
      store<V, float>(static_cast<float*>(target) + static_cast<long long>(b) * hw + dst, t);
      continue;
    }
    for (int q = 0; q < R; ++q) {
      float t[V];
#pragma unroll
      for (int k = 0; k < V; ++k) t[k] = 0.f;
      for (int m = regions[q]; m < regions[q + 1]; ++m) {
        const int lab = regions[R + 1 + m];
#pragma unroll
        for (int k = 0; k < V; ++k) t[k] = s[k] == lab ? 1.f : t[k];
      }
      store<V, float>(static_cast<float*>(target) + (static_cast<long long>(b) * R + q) * hw + dst, t);
    }
  }
}

template <int V>
int launch(const void* staged, const int64_t* desc, int B, int C, int H, int W, int val, const int32_t* regions, int R,
           float* data, void* target, cudaStream_t stream) {
  const long long nv = static_cast<long long>(H) * (W / V);
  const dim3 grid(static_cast<unsigned>(B * C + B),
                  static_cast<unsigned>(std::min<long long>((nv + kT - 1) / kT, 65535)));
  crop_kernel<V><<<grid, kT, 0, stream>>>(static_cast<const char*>(staged), reinterpret_cast<const long long*>(desc),
                                             B, C, H, W, val, regions, R, data, target);
  return check_launch("dl_crop");
}

}  // namespace
}  // namespace b2u

using namespace b2u;

extern "C" int b2u_dl_crop(const void* staged, const int64_t* desc, int32_t B, int32_t C, int32_t H, int32_t W,
                           int32_t mode, const int32_t* regions, int32_t R, float* data, void* target,
                           b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!staged || !desc || !data || !target || (R > 0 && !regions))
    return set_error(-1, "b2u_dl_crop: null pointer");
  if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || static_cast<long long>(B) * C > 65535 || R < 0)
    return set_error(-1, "b2u_dl_crop: bad shape B=%d C=%d %dx%d R=%d", B, C, H, W, R);
  if ((mode != 0 && mode != 1) || (mode == 0 && R > 0)) return set_error(-1, "b2u_dl_crop: mode=%d R=%d", mode, R);
  if (W % 4 == 0) return launch<4>(staged, desc, B, C, H, W, mode, regions, R, data, target, stream);
  if (W % 2 == 0) return launch<2>(staged, desc, B, C, H, W, mode, regions, R, data, target, stream);
  return launch<1>(staged, desc, B, C, H, W, mode, regions, R, data, target, stream);
}
