// Training-case segmentation preprocessing on the device (reference: default_preprocessor.py:40-118 `run_case_npy` with
// a seg, and `_sample_foreground_locations` at lines 156-181).  Labels are read in their stored dtype (the codes and
// comparison rule of label_compare.cuh).
//
//   b2u_pre_seg_check     min, max and a non-integer / non-finite flag of a label volume, for the host's one read.
//   b2u_pre_resample_seg  resample_data_or_seg_to_shape(is_seg=True, order=1) of a 2D configuration (Z unchanged):
//                         batchgenerators' resize_segmentation paints, in ascending label order, every voxel whose
//                         skimage order-1 resize of the label's float64 indicator is >= 0.5.  That resize is scipy's
//                         NI_ZoomShift (export.cu's taps: cc = (k + 0.5) * (n_in / n_out) - 0.5, weights 1 - (cc -
//                         floor(cc)) and its complement, indices clamped) summed as t += v * wy * wx in tap order, then a
//                         clip to the indicator's [min, max] that cannot move a value across 0.5.  For a 0/1 indicator
//                         each term is +0.0 or wy * wx, so one pass per output voxel sums, for each distinct label among
//                         its 2x2 taps, that label's products in tap order (every product and sum a _rn intrinsic: ties
//                         at exactly 0.5 are common); the largest label with a sum >= 0.5 wins, else 0.  With Z unchanged
//                         the reference's 3-D resize gives each tap a z weight of exactly 1 or adds zero taps, so the
//                         per-slice and 3-D paths are this same kernel.
//   b2u_pre_seg_count     per-class voxel counts, a class being a sorted label set (in_sorted_labels).
//   b2u_pre_seg_compact   np.argwhere order of one class: the ascending linear indices of its voxels (block counts, one
//                         scan, an in-order scatter).
//   b2u_pre_seg_gather    rows[i] = (0, z, y, x) of the voxel of rank ranks[i] in that list (the host draws the ranks).
//   b2u_fp_fg_compact     the same compaction for the fingerprint's foreground `seg > 0` (fingerprint_extractor.py:60),
//                         and its voxel count.
#include <algorithm>
#include <climits>

#include "../../include/dinounet_b200.h"
#include "gemm_common.h"
#include "host_util.h"
#include "label_compare.cuh"

namespace b2u {

constexpr int kSegThreads = 256;
constexpr int kCompactTile = kSegThreads;                  // elements per step of a compaction block
constexpr int kCompactChunk = kCompactTile * 16;           // elements per compaction block
constexpr int kMaxClasses = 4096;

// ---- label check ----------------------------------------------------------------------------------------------------

// A stored label as an int32 (clamped: anything outside int32 is out of range anyway); bad for a float32 value that is
// not a finite integer.
__device__ __forceinline__ int label_value(const void* p, int dtype, long long i, bool& bad) {
  if (dtype == B2U_EVAL_F32) {
    const float v = static_cast<const float*>(p)[i];
    if (!isfinite(v) || v != truncf(v)) {
      bad = true;
      return 0;
    }
    return v >= 2147483647.f ? INT_MAX : v <= -2147483648.f ? INT_MIN : static_cast<int>(v);
  }
  return static_cast<int>(load_int_label(p, dtype, i));
}

__global__ void seg_check_init_kernel(int32_t* out) {
  out[0] = INT_MAX;
  out[1] = INT_MIN;
  out[2] = 0;
}

__global__ void __launch_bounds__(kSegThreads) seg_check_kernel(const void* __restrict__ seg, int dtype, long long n,
                                                                int32_t* __restrict__ out) {
  int lo = INT_MAX, hi = INT_MIN;
  bool bad = false;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    bool b = false;
    const int v = label_value(seg, dtype, i, b);
    if (b) {
      bad = true;
    } else {
      lo = min(lo, v);
      hi = max(hi, v);
    }
  }
  lo = __reduce_min_sync(0xffffffffu, lo);
  hi = __reduce_max_sync(0xffffffffu, hi);
  bad = __any_sync(0xffffffffu, bad);
  if ((threadIdx.x & 31) == 0) {
    atomicMin(out, lo);
    atomicMax(out + 1, hi);
    if (bad) out[2] = 1;  // every writer stores the same value
  }
}

// ---- order-1 label resampling -------------------------------------------------------------------------------------

struct SegTaps {
  int i0, i1;
  double w0, w1;
};

// scipy's order-1 NI_ZoomShift along one axis (mode 'nearest', grid_mode=True), as export.cu's zoom_taps.
__device__ __forceinline__ SegTaps seg_taps(int k, int n_in, double zoom) {
  const double cc = __dsub_rn(__dmul_rn(__dadd_rn(static_cast<double>(k), 0.5), zoom), 0.5);
  const double fl = floor(cc);
  SegTaps t;
  t.w0 = __dsub_rn(1.0, __dsub_rn(cc, fl));
  t.w1 = __dsub_rn(1.0, t.w0);
  const int s = static_cast<int>(fl);
  t.i0 = min(max(s, 0), n_in - 1);
  t.i1 = min(max(s + 1, 0), n_in - 1);
  return t;
}

template <typename T>
__device__ __forceinline__ int as_label(T v) { return static_cast<int>(v); }

// One output row Y per blockIdx.y and slice per blockIdx.z, columns over blockIdx.x * blockDim.x.  The inputs hold
// integers in [0, 32767] (b2u_pre_seg_check), so every stored label converts exactly.  *out_max (zeroed by the caller)
// becomes the largest label written.
template <typename T>
__global__ void __launch_bounds__(128) resample_seg_kernel(const T* __restrict__ seg, int h, int w, int H, int W,
                                                           double zoom_y, double zoom_x, T* __restrict__ out,
                                                           int64_t* __restrict__ out_max) {
  const int X = blockIdx.x * blockDim.x + threadIdx.x;
  const int Y = blockIdx.y, z = blockIdx.z;
  int result = 0;
  if (X < W) {
    const SegTaps ty = seg_taps(Y, h, zoom_y), tx = seg_taps(X, w, zoom_x);
    const T* s = seg + static_cast<long long>(z) * h * w;
    const int lab[4] = {as_label(s[ty.i0 * w + tx.i0]), as_label(s[ty.i0 * w + tx.i1]),
                        as_label(s[ty.i1 * w + tx.i0]), as_label(s[ty.i1 * w + tx.i1])};
    const double wt[4] = {__dmul_rn(ty.w0, tx.w0), __dmul_rn(ty.w0, tx.w1), __dmul_rn(ty.w1, tx.w0),
                          __dmul_rn(ty.w1, tx.w1)};
#pragma unroll
    for (int t = 0; t < 4; ++t) {  // each distinct label: its products summed in tap order, as its own indicator would
      double sum = 0.0;
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (lab[u] == lab[t]) sum = __dadd_rn(sum, wt[u]);
      if (sum >= 0.5 && lab[t] > result) result = lab[t];
    }
    out[(static_cast<long long>(z) * H + Y) * W + X] = static_cast<T>(result);
  }
  __shared__ int wmax[4];
  const int m = __reduce_max_sync(0xffffffffu, result);
  if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    const int b = max(max(wmax[0], wmax[1]), max(wmax[2], wmax[3]));
    if (b > 0) atomicMax(reinterpret_cast<long long*>(out_max), static_cast<long long>(b));
  }
}

// ---- class counts and locations -----------------------------------------------------------------------------------

// counts[k] += the voxels whose label is in labels[offsets[k] .. offsets[k+1]).  The warps of a block walk the volume in
// lockstep (every lane runs the same number of steps), so one ballot per class and step feeds a shared counter.
__global__ void __launch_bounds__(kSegThreads) seg_count_kernel(const void* __restrict__ seg, int dtype, long long n,
                                                                const long long* __restrict__ labels,
                                                                const int32_t* __restrict__ offsets, int K,
                                                                unsigned long long* __restrict__ counts) {
  extern __shared__ unsigned int block_counts[];
  for (int k = threadIdx.x; k < K; k += blockDim.x) block_counts[k] = 0;
  __syncthreads();
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long steps = (n + stride - 1) / stride;
  const long long first = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (long long s = 0; s < steps; ++s) {
    const long long i = first + s * stride;
    const bool in = i < n;
    for (int k = 0; k < K; ++k) {
      const int b = __ldg(offsets + k), e = __ldg(offsets + k + 1);
      const unsigned hit = __ballot_sync(0xffffffffu, in && in_sorted_labels(seg, dtype, i, labels + b, e - b));
      if ((threadIdx.x & 31) == 0 && hit) atomicAdd(block_counts + k, static_cast<unsigned>(__popc(hit)));
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < K; k += blockDim.x)
    if (block_counts[k]) atomicAdd(counts + k, static_cast<unsigned long long>(block_counts[k]));
}

// The compaction's predicates: membership in a sorted label set, or numpy's `seg > 0` (a NaN voxel is not foreground).
struct InLabels {
  const long long* labels;
  int n;
  __device__ __forceinline__ bool operator()(const void* seg, int dtype, long long i) const {
    return in_sorted_labels(seg, dtype, i, labels, n);
  }
};

struct Positive {
  __device__ __forceinline__ bool operator()(const void* seg, int dtype, long long i) const {
    if (dtype == B2U_EVAL_F32) return static_cast<const float*>(seg)[i] > 0.f;
    return load_int_label(seg, dtype, i) > 0;
  }
};

// block_counts[b] = the voxels in [b * kCompactChunk, (b + 1) * kCompactChunk) that satisfy `pred`.
template <typename Pred>
__global__ void __launch_bounds__(kSegThreads) compact_count_kernel(const void* __restrict__ seg, int dtype, long long n,
                                                                    Pred pred, int32_t* __restrict__ block_counts) {
  const long long b = static_cast<long long>(blockIdx.x) * kCompactChunk, e = min(n, b + kCompactChunk);
  int c = 0;
  for (long long t = b; t < e; t += kCompactTile) {
    const long long i = t + threadIdx.x;
    c += __syncthreads_count(i < e && pred(seg, dtype, i));
  }
  if (threadIdx.x == 0) block_counts[blockIdx.x] = c;
}

// Exclusive scan of v[m] in place, one block of 1024 threads.
__global__ void __launch_bounds__(1024) exclusive_scan_kernel(int32_t* __restrict__ v, int m) {
  __shared__ int warp_sums[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < m; base += 1024) {
    const int i = base + threadIdx.x;
    const int x = i < m ? v[i] : 0;
    int incl = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int ws = warp_sums[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, ws, o);
        if (lane >= o) ws += y;
      }
      warp_sums[lane] = ws;  // inclusive over warps
    }
    __syncthreads();
    const int before = carry + (warp ? warp_sums[warp - 1] : 0);
    if (i < m) v[i] = before + incl - x;
    __syncthreads();
    if (threadIdx.x == 0) carry += warp_sums[31];
    __syncthreads();
  }
}

// Block b writes the linear indices of its chunk's voxels that satisfy `pred`, ascending, at idx[offsets[b] ...]; the
// last block stores the total in *total when it is not null.
template <typename Pred>
__global__ void __launch_bounds__(kSegThreads) compact_scatter_kernel(const void* __restrict__ seg, int dtype,
                                                                      long long n, Pred pred,
                                                                      const int32_t* __restrict__ offsets,
                                                                      int32_t* __restrict__ idx,
                                                                      int64_t* __restrict__ total) {
  __shared__ int warp_sums[kSegThreads / 32];
  const long long b = static_cast<long long>(blockIdx.x) * kCompactChunk, e = min(n, b + kCompactChunk);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int base = offsets[blockIdx.x];
  for (long long t = b; t < e; t += kCompactTile) {
    const long long i = t + threadIdx.x;
    const bool hit = i < e && pred(seg, dtype, i);
    const unsigned ballot = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) warp_sums[warp] = __popc(ballot);
    __syncthreads();
    int before = 0, sum = 0;
#pragma unroll
    for (int q = 0; q < kSegThreads / 32; ++q) {
      before += q < warp ? warp_sums[q] : 0;
      sum += warp_sums[q];
    }
    if (hit) idx[base + before + __popc(ballot & ((1u << lane) - 1u))] = static_cast<int32_t>(i);
    base += sum;
    __syncthreads();
  }
  if (total && threadIdx.x == 0 && blockIdx.x == gridDim.x - 1) *total = base;
}

__global__ void __launch_bounds__(kSegThreads) gather_rows_kernel(const int32_t* __restrict__ idx,
                                                                  const int64_t* __restrict__ ranks, long long t,
                                                                  int H, int W, int64_t* __restrict__ rows) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= t) return;
  const long long lin = idx[ranks[i]];
  const long long plane = static_cast<long long>(H) * W;
  const long long rem = lin % plane;
  rows[4 * i + 0] = 0;
  rows[4 * i + 1] = lin / plane;
  rows[4 * i + 2] = rem / W;
  rows[4 * i + 3] = rem % W;
}

static bool valid_dtype(int dtype) { return dtype >= B2U_EVAL_U8 && dtype <= B2U_EVAL_F32; }

static int resident_grid(long long n, int threads) {
  return static_cast<int>(std::max<long long>(1, std::min<long long>((n + threads - 1) / threads,
                                                                    static_cast<long long>(num_sms()) * 8)));
}

template <typename T>
static void launch_resample(const void* seg, int Z, int h, int w, int H, int W, void* out, int64_t* out_max,
                            cudaStream_t stream) {
  const dim3 grid((W + 127) / 128, H, Z);
  resample_seg_kernel<T><<<grid, 128, 0, stream>>>(static_cast<const T*>(seg), h, w, H, W,
                                                   static_cast<double>(h) / H, static_cast<double>(w) / W,
                                                   static_cast<T*>(out), out_max);
}

// count -> exclusive scan -> in-order scatter of the voxels that satisfy `pred`.
template <typename Pred>
static int compact(const void* seg, int dtype, long long n, Pred pred, int32_t* work, int32_t* idx, int64_t* total,
                   cudaStream_t stream, const char* what) {
  const long long blocks = (n + kCompactChunk - 1) / kCompactChunk;
  compact_count_kernel<Pred><<<static_cast<unsigned>(blocks), kSegThreads, 0, stream>>>(seg, dtype, n, pred, work);
  int rc = check_launch(what);
  if (rc) return rc;
  exclusive_scan_kernel<<<1, 1024, 0, stream>>>(work, static_cast<int>(blocks));
  if ((rc = check_launch(what))) return rc;
  compact_scatter_kernel<Pred><<<static_cast<unsigned>(blocks), kSegThreads, 0, stream>>>(seg, dtype, n, pred, work,
                                                                                           idx, total);
  return check_launch(what);
}

}  // namespace b2u

using namespace b2u;

extern "C" int b2u_pre_seg_check(const void* seg, int32_t dtype, int64_t n, int32_t* out, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!seg || !out) return set_error(-1, "b2u_pre_seg_check: null pointer");
  if (n <= 0 || !valid_dtype(dtype))
    return set_error(-1, "b2u_pre_seg_check: n=%lld dtype=%d", static_cast<long long>(n), dtype);
  seg_check_init_kernel<<<1, 1, 0, stream>>>(out);
  int rc = check_launch("pre_seg_check_init");
  if (rc) return rc;
  seg_check_kernel<<<resident_grid(n, kSegThreads), kSegThreads, 0, stream>>>(seg, dtype, n, out);
  return check_launch("pre_seg_check");
}

extern "C" int b2u_pre_resample_seg(const void* seg, int32_t dtype, int32_t Z, int32_t h, int32_t w, int32_t H,
                                    int32_t W, void* out, int64_t* out_max, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!seg || !out || !out_max) return set_error(-1, "b2u_pre_resample_seg: null pointer");
  if (!valid_dtype(dtype) || Z <= 0 || h <= 0 || w <= 0 || H <= 0 || W <= 0 || H > 65535 || Z > 65535)
    return set_error(-1, "b2u_pre_resample_seg: bad shape Z=%d %dx%d -> %dx%d (dtype %d)", Z, h, w, H, W, dtype);
  switch (dtype) {
    case B2U_EVAL_U8: launch_resample<uint8_t>(seg, Z, h, w, H, W, out, out_max, stream); break;
    case B2U_EVAL_I8: launch_resample<int8_t>(seg, Z, h, w, H, W, out, out_max, stream); break;
    case B2U_EVAL_I16: launch_resample<int16_t>(seg, Z, h, w, H, W, out, out_max, stream); break;
    case B2U_EVAL_U16: launch_resample<uint16_t>(seg, Z, h, w, H, W, out, out_max, stream); break;
    case B2U_EVAL_I32: launch_resample<int32_t>(seg, Z, h, w, H, W, out, out_max, stream); break;
    default: launch_resample<float>(seg, Z, h, w, H, W, out, out_max, stream); break;
  }
  return check_launch("pre_resample_seg");
}

extern "C" int b2u_pre_seg_count(const void* seg, int32_t dtype, int64_t n, const int64_t* labels,
                                 const int32_t* offsets, int32_t K, int64_t* counts, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!seg || !labels || !offsets || !counts) return set_error(-1, "b2u_pre_seg_count: null pointer");
  if (n <= 0 || !valid_dtype(dtype) || K < 1 || K > kMaxClasses)
    return set_error(-1, "b2u_pre_seg_count: n=%lld dtype=%d K=%d", static_cast<long long>(n), dtype, K);
  seg_count_kernel<<<resident_grid(n, kSegThreads), kSegThreads, K * sizeof(unsigned), stream>>>(
      seg, dtype, n, reinterpret_cast<const long long*>(labels), offsets, K,
      reinterpret_cast<unsigned long long*>(counts));
  return check_launch("pre_seg_count");
}

extern "C" int64_t b2u_pre_seg_compact_work_ints(int64_t n) { return (n + kCompactChunk - 1) / kCompactChunk; }

extern "C" int b2u_pre_seg_compact(const void* seg, int32_t dtype, int64_t n, const int64_t* labels, int32_t n_labels,
                                   int32_t* work, int32_t* idx, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!seg || !labels || !work || !idx) return set_error(-1, "b2u_pre_seg_compact: null pointer");
  if (n <= 0 || n > INT_MAX || !valid_dtype(dtype) || n_labels < 1)
    return set_error(-1, "b2u_pre_seg_compact: n=%lld dtype=%d n_labels=%d", static_cast<long long>(n), dtype,
                     n_labels);
  return compact(seg, dtype, n, InLabels{reinterpret_cast<const long long*>(labels), n_labels}, work, idx, nullptr,
                 stream, "pre_seg_compact");
}

extern "C" int b2u_fp_fg_compact(const void* seg, int32_t dtype, int64_t n, int32_t* work, int32_t* idx, int64_t* count,
                                 b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!seg || !work || !idx || !count) return set_error(-1, "b2u_fp_fg_compact: null pointer");
  if (n <= 0 || n > INT_MAX || !valid_dtype(dtype))
    return set_error(-1, "b2u_fp_fg_compact: n=%lld dtype=%d", static_cast<long long>(n), dtype);
  return compact(seg, dtype, n, Positive{}, work, idx, count, stream, "fp_fg_compact");
}

extern "C" int b2u_pre_seg_gather(const int32_t* idx, const int64_t* ranks, int64_t t, int32_t H, int32_t W,
                                  int64_t* rows, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!idx || !ranks || !rows) return set_error(-1, "b2u_pre_seg_gather: null pointer");
  if (t <= 0 || H <= 0 || W <= 0)
    return set_error(-1, "b2u_pre_seg_gather: t=%lld %dx%d", static_cast<long long>(t), H, W);
  gather_rows_kernel<<<static_cast<unsigned>((t + kSegThreads - 1) / kSegThreads), kSegThreads, 0, stream>>>(
      idx, ranks, t, H, W, rows);
  return check_launch("pre_seg_gather");
}
