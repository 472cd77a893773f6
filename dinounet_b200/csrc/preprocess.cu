// Case preprocessing on the device (reference: preprocessing/preprocessors/default_preprocessor.py:40-118 `run_case_npy`,
// preprocessing/normalization/default_normalization_schemes.py, preprocessing/resampling/default_resampling.py:77-216),
// and the fp16 fold ensemble of predict_logits_from_preprocessed_data (inference/predict_from_raw_data.py:466-501).
//
// Normalization runs in fp32 exactly as numpy does it:
//   b2u_pre_zscore    numpy's float32 `mean()` / `std()` of one channel are ONE pairwise sum over the channel in a given
//                     order (numpy's pairwise_sum: runs of <= 128 elements are leaves summed in 8 lanes and combined
//                     ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the rest added in order; a longer run splits at n/2
//                     rounded down to a multiple of 8).  The tree is evaluated level by level, deepest first, one thread
//                     per node, each node's value stored at the slot of its first 8-element group: no atomics.
//                     mean = f32(f64(sum) / n), std = sqrt(f32(f64(sum((x - mean)^2)) / n)), divisor max(std, 1e-8f).
//   b2u_pre_normalize CT (clip, - mean, / max(std, 1e-8)), RescaleTo01 (- min, / max(max - min, 1e-8)), RGBTo01 (/ 255).
//   b2u_pre_minmax_f32 exact min / max of a channel and a non-finite flag.
//
// b2u_pre_resample3 is `resample_data_or_seg_to_shape(order=3)` of a 2D configuration (Z unchanged): skimage
// `resize(order=3, mode='edge', anti_aliasing=False)` = scipy `ndimage.zoom(order=3, mode='nearest', grid_mode=True)`
// on float64 followed by a clip to the [min, max] of that call's input, then `.astype(float32)`.  scipy's arithmetic,
// operation for operation (every product and sum an explicit _rn intrinsic, so nvcc forms no FMA):
//   np.pad(x, 12, mode='edge') on every axis of the call's input (a [h, w] slice, or the whole [Z, h, w] channel);
//   spline_filter(order 3, mode 'nearest'), axis 0 first, per line of length n:
//     c *= gain;  c0 = c[0];  s = c0 + z^n c[n-1];  s += z^i (c[i] + z^n c[n-1-i]) for i = 1..n-1 (z^i by repeated
//     multiplication);  c[0] = s * (z / (1 - z^2n)) + c0;  c[i] += z c[i-1];  c[n-1] *= z / (z - 1);
//     c[i] = z (c[i+1] - c[i]);   z = the correctly rounded pole sqrt(3) - 2; z^n, the gain and the two factors come
//     from the host (glibc pow, not CUDA's);
//   NI_ZoomShift: cc = ((k + 0.5) * (n_in / n_out) - 0.5) + 12, y = cc - floor(cc), taps floor(cc) - 1 .. + 2 of the
//     padded array, weights w0 = (1-y)^3 / 6, w1 = (y*y*(y-2)*3 + 4) / 6, w2 = ((1-y)*(1-y)*((1-y)-2)*3 + 4) / 6,
//     w3 = 1 - w0 - w1 - w2;  t = 0.0; t += coef * w_axis0 * w_axis1 (* w_axis2), taps with the last axis fastest.
// Per slice (separate z along axis 0): 16 taps, clip to the slice's min / max.  3-D (no separate z): Z is padded and
// filtered too and interpolated with 4 taps at a zoom of exactly 1; 64 taps, clip to the channel's min / max.
#include <cuda_fp16.h>

#include <algorithm>
#include <set>
#include <vector>

#include "../../include/dinounet_b200.h"
#include "common.cuh"
#include "gemm_common.h"
#include "host_util.h"
#include "spline.cuh"

namespace b2u {

constexpr int kLeaf = 128;         // numpy's PW_BLOCKSIZE
constexpr long long kMinMaxChunk = 1 << 16;

// ---- exact min / max (and a non-finite flag) --------------------------------------------------------------------

template <typename T>
__device__ __forceinline__ bool finite_val(T v) { return isfinite(v); }

// Block g reduces lo_src / hi_src over [g*chunk, min(n, (g+1)*chunk)): lo_out[g] = min, hi_out[g] = max.
template <typename T>
__global__ void __launch_bounds__(256) minmax_kernel(const T* __restrict__ lo_src, const T* __restrict__ hi_src,
                                                     long long n, long long chunk, T* __restrict__ lo_out,
                                                     T* __restrict__ hi_out, int* __restrict__ nonfinite) {
  __shared__ T slo[256], shi[256];
  const long long b = static_cast<long long>(blockIdx.x) * chunk, e = min(n, b + chunk);
  T lo = lo_src[b], hi = hi_src[b];
  bool bad = false;
  for (long long i = b + threadIdx.x; i < e; i += blockDim.x) {
    const T a = lo_src[i], c = hi_src[i];
    bad |= !finite_val(a) || !finite_val(c);
    lo = a < lo ? a : lo;
    hi = c > hi ? c : hi;
  }
  if (bad && nonfinite) *nonfinite = 1;  // every writer stores the same value
  slo[threadIdx.x] = lo;
  shi[threadIdx.x] = hi;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      slo[threadIdx.x] = slo[threadIdx.x + s] < slo[threadIdx.x] ? slo[threadIdx.x + s] : slo[threadIdx.x];
      shi[threadIdx.x] = shi[threadIdx.x + s] > shi[threadIdx.x] ? shi[threadIdx.x + s] : shi[threadIdx.x];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    lo_out[blockIdx.x] = slo[0];
    hi_out[blockIdx.x] = shi[0];
  }
}

// ---- numpy's pairwise sum (float32 here, float64 for the evaluation's mean surface distance) ----------------------

struct Order3 {  // element i of the summation order lives at i0*s0 + i1*s1 + i2*s2, i = (i0*n1 + i1)*n2 + i2
  long long n1, n2, s0, s1, s2;
  bool flat;     // s2 == 1 and the order is memory order
};

template <typename T>
__device__ __forceinline__ T elem(const T* x, const Order3& o, long long i) {
  if (o.flat) return x[i];
  const long long i2 = i % o.n2, r = i / o.n2;
  return x[(r / o.n1) * o.s0 + (r % o.n1) * o.s1 + i2 * o.s2];
}

__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }

template <typename T>
__device__ __forceinline__ T term(const T* x, const Order3& o, long long i, bool sq, T mean) {
  const T v = elem(x, o, i);
  if (!sq) return v;
  const T d = sub_rn(v, mean);
  return mul_rn(d, d);
}

__device__ __forceinline__ long long split_of(long long m) {
  long long m2 = m / 2;
  return m2 - m2 % 8;
}

// One thread per node of depth k (path bits, root decision first).  A leaf (m <= 128) writes its sum to val[o / 8]; an
// inner node adds its children, both already evaluated at depth k + 1, into the slot it shares with its left child.
// blockIdx.y is the plane of a batch of equal runs: x, stats and val advance by xs, ss and vs per plane.
template <typename T>
__global__ void __launch_bounds__(256) tree_level_kernel(const T* __restrict__ x, long long n, int k, Order3 ord,
                                                         int sq, const T* __restrict__ stats, T* __restrict__ val,
                                                         long long xs, long long ss, long long vs) {
  x += blockIdx.y * xs;
  stats += blockIdx.y * ss;
  val += blockIdx.y * vs;
  const long long b = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (b >= (1LL << k)) return;
  long long o = 0, m = n;
  for (int j = k - 1; j >= 0; --j) {
    if (m <= kLeaf) return;  // a leaf above depth k: evaluated at its own depth
    const long long m2 = split_of(m);
    if ((b >> j) & 1) {
      o += m2;
      m -= m2;
    } else {
      m = m2;
    }
  }
  if (m > kLeaf) {
    const long long m2 = split_of(m);
    val[o / 8] = add_rn(val[o / 8], val[(o + m2) / 8]);
    return;
  }
  const bool squares = sq != 0;
  const T mean = squares ? stats[0] : T(0);
  T res;
  if (m < 8) {
    res = T(0);
    for (long long i = 0; i < m; ++i) res = add_rn(res, term(x, ord, o + i, squares, mean));
  } else {
    T r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = term(x, ord, o + j, squares, mean);
    long long i = 8;
    for (; i < m - m % 8; i += 8) {
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = add_rn(r[j], term(x, ord, o + i + j, squares, mean));
    }
    res = add_rn(add_rn(add_rn(r[0], r[1]), add_rn(r[2], r[3])), add_rn(add_rn(r[4], r[5]), add_rn(r[6], r[7])));
    for (; i < m; ++i) res = add_rn(res, term(x, ord, o + i, squares, mean));
  }
  val[o / 8] = res;
}

// numpy's _mean / _var on a float32 array: the float32 sum divided by the intp count in float64, rounded to float32;
// std = float32 sqrt; ZScore's divisor max(std, 1e-8) with 1e-8 as a float32 scalar.
__global__ void zscore_finalize_kernel(const float* __restrict__ val, long long n, int stage, float* __restrict__ stats) {
  const double q = __ddiv_rn(static_cast<double>(val[0]), static_cast<double>(n));
  if (stage == 0) {
    stats[0] = __double2float_rn(q);
  } else {
    const float sd = __fsqrt_rn(__double2float_rn(q));
    stats[1] = 1e-8f > sd ? 1e-8f : sd;
  }
}

// scheme 0 ZScore: (x - stats[0]) / stats[1];  1 CT: clip(x, a, b) - c, / d;  2 RescaleTo01: x - stats[0], / max(stats[1]
// - stats[0], 1e-8f) (the max of x - min is max - min: rounding is monotone);  3 RGBTo01: x / 255.
__global__ void __launch_bounds__(256) normalize_kernel(float* __restrict__ x, long long n, int scheme,
                                                        const float* __restrict__ stats, float a, float b, float c,
                                                        float d) {
  float sub = 0.f, div = 1.f;
  if (scheme == 0) {
    sub = stats[0];
    div = stats[1];
  } else if (scheme == 1) {
    sub = c;
    div = d;
  } else if (scheme == 2) {
    sub = stats[0];
    const float r = __fsub_rn(stats[1], stats[0]);
    div = r < 1e-8f ? 1e-8f : r;
  } else {
    div = 255.f;
  }
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    float v = x[i];
    if (scheme == 1) v = fminf(fmaxf(v, a), b);
    if (scheme != 3) v = __fsub_rn(v, sub);
    x[i] = __fdiv_rn(v, div);
  }
}

// ---- order-3 resampling -------------------------------------------------------------------------------------------

// Edge-padded fp64 copy of a [Z, h, w] view (element strides sz, sy, sx) into [Z + 2*pz, h + 24, w + 24].
__global__ void __launch_bounds__(256) pad_kernel(const float* __restrict__ x, int Z, int h, int w, long long sz,
                                                  long long sy, long long sx, int pz, double* __restrict__ out) {
  const int Wp = w + 2 * kPad, Hp = h + 2 * kPad, Zp = Z + 2 * pz;
  const long long total = static_cast<long long>(Zp) * Hp * Wp;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int xp = static_cast<int>(i % Wp);
    const long long r = i / Wp;
    const int yp = static_cast<int>(r % Hp), zp = static_cast<int>(r / Hp);
    const int zi = min(max(zp - pz, 0), Z - 1), yi = min(max(yp - kPad, 0), h - 1), xi = min(max(xp - kPad, 0), w - 1);
    out[i] = static_cast<double>(x[zi * sz + yi * sy + xi * sx]);
  }
}

// One thread per line of the contiguous [d0, d1, d2] array along `axis` (scipy's NI_SplineFilter1D, mode 'nearest').
__global__ void __launch_bounds__(128) spline_filter_kernel(double* __restrict__ c, int d0, int d1, int d2, int axis,
                                                            FilterConsts k) {
  const long long lines = axis == 0 ? static_cast<long long>(d1) * d2 : axis == 1 ? static_cast<long long>(d0) * d2
                                                                                  : static_cast<long long>(d0) * d1;
  const long long l = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (l >= lines) return;
  long long base, st;
  int n;
  if (axis == 0) {
    base = l; st = static_cast<long long>(d1) * d2; n = d0;
  } else if (axis == 1) {
    base = (l / d2) * d1 * d2 + l % d2; st = d2; n = d1;
  } else {
    base = l * d2; st = 1; n = d2;
  }
  spline_filter_line<false>(c + base, st, n, k);
}

// One output row (z, Y) per blockIdx.y / blockIdx.z, columns over blockIdx.x * blockDim.x.  three_d = 0: coef is
// [Z, h + 24, w + 24] and lo / hi are per slice;  three_d = 1: coef is [Z + 24, h + 24, w + 24], lo / hi are [1].
template <bool kThreeD>
__global__ void __launch_bounds__(128) zoom3_kernel(const double* __restrict__ coef, int Z, int h, int w, int H, int W,
                                                    double zoom_y, double zoom_x, const double* __restrict__ lo,
                                                    const double* __restrict__ hi, float* __restrict__ out) {
  const int X = blockIdx.x * blockDim.x + threadIdx.x;
  const int Y = blockIdx.y, zo = blockIdx.z;
  if (X >= W) return;
  const long long Wp = w + 2 * kPad, plane = static_cast<long long>(h + 2 * kPad) * Wp;
  const Taps3 ty = cubic_taps(Y, zoom_y), tx = cubic_taps(X, zoom_x);
  double t = 0.0;
  if (kThreeD) {
    const Taps3 tz = cubic_taps(zo, 1.0);
    for (int a = 0; a < 4; ++a) {
      const double* pz = coef + (tz.start + a) * plane;
      for (int b = 0; b < 4; ++b) {
        const double* row = pz + (ty.start + b) * Wp + tx.start;
#pragma unroll
        for (int c = 0; c < 4; ++c) t = __dadd_rn(t, __dmul_rn(__dmul_rn(__dmul_rn(row[c], tz.w[a]), ty.w[b]), tx.w[c]));
      }
    }
  } else {
    t = cubic16(coef + zo * plane, Wp, ty, tx);
  }
  const int g = kThreeD ? 0 : zo;
  t = fmin(fmax(t, lo[g]), hi[g]);  // np.clip(out, min, max): minimum(maximum(x, min), max)
  out[(static_cast<long long>(zo) * H + Y) * W + X] = __double2float_rn(t);
}

// ---- fold ensemble ------------------------------------------------------------------------------------------------

// acc += x (x != NULL), then acc /= divisor (divisor > 0), each as torch's CPU fp16 ops: in fp32, rounded to fp16.
__global__ void __launch_bounds__(256) ensemble_kernel(__half* __restrict__ acc, const __half* __restrict__ x,
                                                       long long n, float divisor) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    __half v = acc[i];
    if (x) v = __float2half_rn(__fadd_rn(__half2float(v), __half2float(x[i])));
    if (divisor > 0.f) v = __float2half_rn(__fdiv_rn(__half2float(v), divisor));
    acc[i] = v;
  }
}

static int grid_for(long long n, int threads, int per_sm = 8) {
  return static_cast<int>(std::max<long long>(1, std::min<long long>((n + threads - 1) / threads,
                                                                    static_cast<long long>(num_sms()) * per_sm)));
}

// Depth of the deepest node of numpy's pairwise tree over n elements (0 when the root is a leaf).
static int tree_depth(long long n) {
  std::set<long long> sizes{n};
  int depth = 0;
  for (;;) {
    std::set<long long> next;
    for (long long s : sizes)
      if (s > kLeaf) {
        const long long m2 = (s / 2) - (s / 2) % 8;
        next.insert(m2);
        next.insert(s - m2);
      }
    if (next.empty()) return depth;
    sizes.swap(next);
    ++depth;
  }
}

// Evaluates the whole tree over x[n] (in the order `ord`; sq: sum of (x - stats[0])^2), deepest level first: the sum
// lands in work[0].  work: ceil(n / 8) elements.  A batch of `planes` equal runs: plane p reads x + p * xs, its mean at
// stats + p * ss, and sums into work + p * ws.
template <typename T>
static int pairwise_sum_tree(const T* x, long long n, const Order3& ord, int sq, const T* stats, T* work,
                             cudaStream_t stream, const char* what, int planes = 1, long long xs = 0,
                             long long ss = 0, long long ws = 0) {
  const int depth = tree_depth(n);
  if (depth > 40) return set_error(-1, "%s: tree depth %d", what, depth);
  if (planes < 1 || planes > 65535) return set_error(-1, "%s: %d planes", what, planes);
  for (int k = depth; k >= 0; --k) {
    const long long nodes = 1LL << k;
    const dim3 grid(static_cast<unsigned>((nodes + 255) / 256), planes);
    tree_level_kernel<T><<<grid, 256, 0, stream>>>(x, n, k, ord, sq, stats, work, xs, ss, ws);
    int rc = check_launch(what);
    if (rc) return rc;
  }
  return 0;
}

int pairwise_sum_f64(const double* x, long long n, double* work, cudaStream_t stream) {
  return pairwise_sum_tree<double>(x, n, Order3{1, n, 0, 0, 1, true}, 0, nullptr, work, stream, "pairwise_sum_f64");
}

int pairwise_sum_sq_f64(const double* x, long long n, const double* mean, double* work, cudaStream_t stream) {
  return pairwise_sum_tree<double>(x, n, Order3{1, n, 0, 0, 1, true}, 1, mean, work, stream, "pairwise_sum_sq_f64");
}

int pairwise_sum_planes_f32(const float* x, long long n, int planes, int sq, const float* mean, float* work,
                            long long ws, cudaStream_t stream) {
  return pairwise_sum_tree<float>(x, n, Order3{1, n, 0, 0, 1, true}, sq, mean, work, stream, "pairwise_sum_planes_f32",
                                  planes, n, 1, ws);
}

int minmax_planes_f32(const float* x, long long n, int planes, float* lo, float* hi, cudaStream_t stream) {
  minmax_kernel<float><<<planes, 256, 0, stream>>>(x, x, n * planes, n, lo, hi, nullptr);
  return check_launch("minmax_planes_f32");
}

}  // namespace b2u

using namespace b2u;

extern "C" int b2u_pre_minmax_f32(const float* x, int64_t n, float* work, float* lo_hi, int32_t* nonfinite,
                                  b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!x || !work || !lo_hi) return set_error(-1, "b2u_pre_minmax_f32: null pointer");
  if (n <= 0) return set_error(-1, "b2u_pre_minmax_f32: n=%lld", static_cast<long long>(n));
  const long long groups = (n + kMinMaxChunk - 1) / kMinMaxChunk;
  if (groups > (1LL << 30)) return set_error(-1, "b2u_pre_minmax_f32: n=%lld too large", static_cast<long long>(n));
  minmax_kernel<float><<<static_cast<unsigned>(groups), 256, 0, stream>>>(x, x, n, kMinMaxChunk, work, work + groups,
                                                                           nonfinite);
  int rc = check_launch("pre_minmax_f32");
  if (rc) return rc;
  minmax_kernel<float><<<1, 256, 0, stream>>>(work, work + groups, groups, groups, lo_hi, lo_hi + 1, nullptr);
  return check_launch("pre_minmax_f32");
}

extern "C" int b2u_pre_zscore(float* x, int64_t n, int32_t n0, int32_t n1, int32_t n2, int64_t s0, int64_t s1,
                              int64_t s2, float* work, float* stats, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!x || !work || !stats) return set_error(-1, "b2u_pre_zscore: null pointer");
  if (n <= 0 || n0 <= 0 || n1 <= 0 || n2 <= 0 || static_cast<long long>(n0) * n1 * n2 != n)
    return set_error(-1, "b2u_pre_zscore: order %dx%dx%d does not cover n=%lld", n0, n1, n2, static_cast<long long>(n));
  Order3 ord{n1, n2, s0, s1, s2, (n0 == 1 && n1 == 1 && s2 == 1)};
  for (int stage = 0; stage < 2; ++stage) {
    int rc = pairwise_sum_tree<float>(x, n, ord, stage, stats, work, stream, "pre_zscore_tree");
    if (rc) return rc;
    zscore_finalize_kernel<<<1, 1, 0, stream>>>(work, n, stage, stats);
    rc = check_launch("pre_zscore_finalize");
    if (rc) return rc;
  }
  normalize_kernel<<<grid_for(n, 256), 256, 0, stream>>>(x, n, 0, stats, 0.f, 0.f, 0.f, 0.f);
  return check_launch("pre_zscore_apply");
}

extern "C" int b2u_pre_normalize(float* x, int64_t n, int32_t scheme, const float* stats, float a, float b, float c,
                                 float d, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!x) return set_error(-1, "b2u_pre_normalize: null pointer");
  if (n <= 0) return set_error(-1, "b2u_pre_normalize: n=%lld", static_cast<long long>(n));
  if (scheme < 1 || scheme > 3) return set_error(-1, "b2u_pre_normalize: scheme %d is not 1 (CT), 2 (RescaleTo01) or 3 "
                                                     "(RGBTo01)", scheme);
  if (scheme == 2 && !stats) return set_error(-1, "b2u_pre_normalize: RescaleTo01 needs the channel's [min, max]");
  normalize_kernel<<<grid_for(n, 256), 256, 0, stream>>>(x, n, scheme, stats, a, b, c, d);
  return check_launch("pre_normalize");
}

extern "C" int64_t b2u_pre_resample3_work_doubles(int32_t Z, int32_t h, int32_t w, int32_t three_d) {
  const long long Zp = Z + (three_d ? 2 * kPad : 0);
  return Zp * (h + 2 * kPad) * (w + 2 * kPad) + 2 * Zp + 2;
}

extern "C" int b2u_pre_resample3(const float* x, int32_t Z, int32_t h, int32_t w, int64_t sz, int64_t sy, int64_t sx,
                                 int32_t H, int32_t W, int32_t three_d, const double* consts, double* work, float* out,
                                 b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!x || !consts || !work || !out) return set_error(-1, "b2u_pre_resample3: null pointer");
  if (Z <= 0 || h <= 0 || w <= 0 || H <= 0 || W <= 0 || H > 65535 || Z > 65535 || (three_d != 0 && three_d != 1))
    return set_error(-1, "b2u_pre_resample3: bad shape Z=%d %dx%d -> %dx%d (three_d %d)", Z, h, w, H, W, three_d);
  const int pz = three_d ? kPad : 0;
  const int Zp = Z + 2 * pz, Hp = h + 2 * kPad, Wp = w + 2 * kPad;
  const long long plane = static_cast<long long>(Hp) * Wp, vol = plane * Zp;
  double* coef = work;
  double* lo = work + vol;
  double* hi = lo + Zp;
  pad_kernel<<<grid_for(vol, 256, 16), 256, 0, stream>>>(x, Z, h, w, sz, sy, sx, pz, coef);
  int rc = check_launch("pre_resample3_pad");
  if (rc) return rc;
  // edge padding adds no new values: the padded slices' min / max are the input slices' (skimage's clip range)
  minmax_kernel<double><<<Zp, 256, 0, stream>>>(coef, coef, vol, plane, lo, hi, nullptr);
  if ((rc = check_launch("pre_resample3_minmax"))) return rc;
  if (three_d) {
    minmax_kernel<double><<<1, 256, 0, stream>>>(lo, hi, Zp, Zp, hi + Zp, hi + Zp + 1, nullptr);
    if ((rc = check_launch("pre_resample3_minmax"))) return rc;
  }
  // consts: per axis (z, y, x) the 5 filter constants {z, z^n, gain, z/(1-z^2n), z/(z-1)} with n the padded length
  const int dims[3] = {Zp, Hp, Wp};
  for (int axis = three_d ? 0 : 1; axis < 3; ++axis) {
    FilterConsts k{consts[axis * 5 + 0], consts[axis * 5 + 1], consts[axis * 5 + 2], consts[axis * 5 + 3],
                   consts[axis * 5 + 4]};
    const long long lines = vol / dims[axis];
    spline_filter_kernel<<<static_cast<unsigned>((lines + 127) / 128), 128, 0, stream>>>(coef, Zp, Hp, Wp, axis, k);
    if ((rc = check_launch("pre_resample3_filter"))) return rc;
  }
  const double zoom_y = static_cast<double>(h) / H, zoom_x = static_cast<double>(w) / W;
  const dim3 grid((W + 127) / 128, H, Z);
  if (three_d)
    zoom3_kernel<true><<<grid, 128, 0, stream>>>(coef, Z, h, w, H, W, zoom_y, zoom_x, hi + Zp, hi + Zp + 1, out);
  else
    zoom3_kernel<false><<<grid, 128, 0, stream>>>(coef, Z, h, w, H, W, zoom_y, zoom_x, lo, hi, out);
  return check_launch("pre_resample3_zoom");
}

extern "C" int b2u_pre_ensemble_f16(void* acc, const void* x, int64_t n, int32_t divisor, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!acc) return set_error(-1, "b2u_pre_ensemble_f16: null pointer");
  if (n <= 0 || divisor < 0) return set_error(-1, "b2u_pre_ensemble_f16: n=%lld divisor=%d", static_cast<long long>(n),
                                              divisor);
  ensemble_kernel<<<grid_for(n, 256), 256, 0, stream>>>(static_cast<__half*>(acc), static_cast<const __half*>(x), n,
                                                        static_cast<float>(divisor));
  return check_launch("pre_ensemble_f16");
}
