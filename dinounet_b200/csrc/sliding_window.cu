// Sliding-window prediction kernels (reference caller: inference/predict_from_raw_data.py:537-621).
// The reference keeps fp16 accumulators and does, per tile:  prediction (fp16 under autocast) = mean over mirror
// variants;  predicted_logits[tile] += prediction * gaussian;  n_predictions[tile] += gaussian;  and at the end
// predicted_logits /= n_predictions.  Every fp16 rounding of that sequence is reproduced here (each half op of torch is
// "compute in fp32, round to half"), so the result is bit-identical to running the reference loop around the same network.
#include "common.cuh"
#include "host_util.h"
#include "gemm_common.h"
#include <algorithm>
#include "../../include/dinounet_b200.h"

namespace b2u {

// tile descriptor (device int32[4] per batch entry): slice d, y0, x0, flip bits (1 = flip rows / dim 2, 2 = flip cols / dim 3)
__global__ void sw_gather_kernel(const float* __restrict__ vol, float* __restrict__ batch,
                                 const int32_t* __restrict__ desc, int Cin, int D, int H, int W, int th, int tw) {
  const int n = blockIdx.z, k = blockIdx.y;  // batch entry, output channel 0..2
  const int d = desc[4 * n], y0 = desc[4 * n + 1], x0 = desc[4 * n + 2], flip = desc[4 * n + 3];
  const int src_c = Cin < 3 ? k % Cin : k;  // 1/2-channel repeat, >3 truncation (dinounet_training.py:491-497)
  const float* src = vol + (static_cast<long long>(src_c) * D + d) * H * W;
  float* dst = batch + (static_cast<long long>(n) * 3 + k) * th * tw;
  const int total = th * tw;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int y = i / tw, x = i - y * tw;
    const int sy = (flip & 1) ? th - 1 - y : y, sx = (flip & 2) ? tw - 1 - x : x;
    dst[i] = src[static_cast<long long>(y0 + sy) * W + x0 + sx];
  }
}

__device__ __forceinline__ float h_round(float v) { return __half2float(__float2half_rn(v)); }

// One tile: entries first..first+nvar-1 of `logits` are its mirror variants (variant 0 unflipped).  npred == nullptr:
// accumulate the logits only (the other folds of an ensemble share one weight count).
__global__ void sw_accumulate_kernel(const float* __restrict__ logits, const int32_t* __restrict__ desc, int first,
                                     int nvar, const __half* __restrict__ gauss, __half* __restrict__ acc,
                                     __half* __restrict__ npred, int C, int D, int H, int W, int th, int tw) {
  const int total = th * tw;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int y = i / tw, x = i - y * tw;
  const int d = desc[4 * first], y0 = desc[4 * first + 1], x0 = desc[4 * first + 2];
  const float g = gauss ? __half2float(gauss[i]) : 1.f;
  const long long pix = (static_cast<long long>(d) * H + y0 + y) * W + x0 + x;
  const long long cstride = static_cast<long long>(D) * H * W;
  const float inv = 1.f / static_cast<float>(nvar);  // nvar is a power of two: exact
  for (int c = 0; c < C; ++c) {
    float p = 0.f;
    for (int v = 0; v < nvar; ++v) {
      const int flip = desc[4 * (first + v) + 3];
      const int sy = (flip & 1) ? th - 1 - y : y, sx = (flip & 2) ? tw - 1 - x : x;
      const float l = h_round(logits[((static_cast<long long>(first + v) * C + c) * th + sy) * tw + sx]);
      p = v == 0 ? l : h_round(p + l);
    }
    if (nvar > 1) p = h_round(p * inv);
    const float pg = gauss ? h_round(p * g) : p;
    const long long o = c * cstride + pix;
    acc[o] = __float2half_rn(__half2float(acc[o]) + pg);
  }
  if (npred) npred[pix] = __float2half_rn(__half2float(npred[pix]) + g);
}

__global__ void sw_finalize_kernel(__half* __restrict__ acc, const __half* __restrict__ npred, int C, long long plane,
                                   int* __restrict__ inf_flag) {
  const long long total = plane * C;
  bool bad = false;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float q = __fdiv_rn(__half2float(acc[i]), __half2float(npred[i % plane]));
    const __half h = __float2half_rn(q);
    acc[i] = h;
    bad |= __hisinf(h);
  }
  if (bad) atomicOr(inf_flag, 1);
}

extern "C" int b2u_sw_gather_tiles(const float* volume, float* batch, const int32_t* tile_desc, int32_t n_entries,
                                   int32_t Cin, int32_t D, int32_t H, int32_t W, int32_t th, int32_t tw,
                                   b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!volume || !batch || !tile_desc) return set_error(-1, "b2u_sw_gather_tiles: null pointer");
  if (n_entries <= 0 || Cin <= 0 || th > H || tw > W || th <= 0 || tw <= 0)
    return set_error(-1, "b2u_sw_gather_tiles: bad dimensions (tile %dx%d in %dx%d, %d entries)", th, tw, H, W, n_entries);
  dim3 grid((th * tw + 1023) / 1024, 3, n_entries);
  sw_gather_kernel<<<grid, 256, 0, stream>>>(volume, batch, tile_desc, Cin, D, H, W, th, tw);
  return check_launch("sw_gather_tiles");
}

extern "C" int b2u_sw_accumulate(const float* logits, const int32_t* tile_desc, int32_t first, int32_t nvar,
                                 const void* gaussian, void* acc, void* npred, int32_t C, int32_t D, int32_t H,
                                 int32_t W, int32_t th, int32_t tw, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!logits || !tile_desc || !acc) return set_error(-1, "b2u_sw_accumulate: null pointer");
  if (nvar != 1 && nvar != 2 && nvar != 4) return set_error(-1, "b2u_sw_accumulate: nvar %d not in {1,2,4}", nvar);
  sw_accumulate_kernel<<<(th * tw + 255) / 256, 256, 0, stream>>>(
      logits, tile_desc, first, nvar, static_cast<const __half*>(gaussian), static_cast<__half*>(acc),
      static_cast<__half*>(npred), C, D, H, W, th, tw);
  return check_launch("sw_accumulate");
}

extern "C" int b2u_sw_finalize(void* acc, const void* npred, int32_t C, int64_t plane, int32_t* inf_flag,
                               b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!acc || !npred || !inf_flag) return set_error(-1, "b2u_sw_finalize: null pointer");
  const long long total = static_cast<long long>(plane) * C;
  const int blocks = static_cast<int>(std::min<long long>((total + 255) / 256, static_cast<long long>(num_sms()) * 16));
  sw_finalize_kernel<<<blocks, 256, 0, stream>>>(static_cast<__half*>(acc), static_cast<const __half*>(npred), C, plane,
                                                inf_flag);
  return check_launch("sw_finalize");
}

}  // namespace b2u
