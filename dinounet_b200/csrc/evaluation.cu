// Scoring predictions against the ground truth on the device (reference: evaluation/evaluate_predictions.py:152-230
// `compute_metrics`, with medpy's hd95 / asd: `__surface_distances`).
//
//   b2u_eval_masks  one pass over the two label volumes per label or region: the masks `seg == r` (numpy's `==`,
//                   label_compare.cuh: exact for integer dtypes, the label rounded to float32 for float32 volumes), their face-connectivity
//                   borders x ^ binary_erosion(x) with out-of-range neighbours 0 (scipy's border_value), and the exact
//                   int64 TP / FP / FN / TN over the voxels whose reference is not the ignore label, plus the two masks'
//                   populations.  Block reduction, then one integer atomic per block and counter.
//   b2u_eval_edt    scipy's distance_transform_edt(~border, sampling) in float64: the squared distance is three separable
//                   lower envelopes of parabolas per line (Felzenszwalb-Huttenlocher), axis 0, then 1, then 2, each
//                   adding (s_a * d_a)^2 to the previous axes' minimum.  The sum is therefore ((s0 d0)^2 + (s1 d1)^2) +
//                   (s2 d2)^2, scipy's association ((ft - indices) * sampling, squared, add.reduce over the axes);
//                   every product and sum is an explicit _rn intrinsic so nothing is contracted into an FMA, and the
//                   square root is IEEE.  At integer spacings every term is an exact integer and the result equals scipy
//                   bit for bit.  Axes 0 and 1: one thread per line, neighbouring threads on neighbouring x (coalesced),
//                   the envelope's vertex list in a global int32 scratch volume with the data's addressing.  Axis 2: the
//                   rows of a block are staged through shared memory with coalesced loads and stores.
//   b2u_eval_sum_f64 numpy's float64 pairwise sum (preprocess.cu's tree): the mean surface distance is that sum over
//                   the gathered distances in C order, divided by their number on the host (numpy's `mean`).
#include <math_constants.h>

#include <algorithm>

#include "../../include/dinounet_b200.h"
#include "gemm_common.h"
#include "host_util.h"
#include "label_compare.cuh"

namespace b2u {

constexpr int kMaxRegionLabels = B2U_EVAL_MAX_REGION_LABELS;
constexpr int kMaskThreads = 256;
constexpr int kEdtLineThreads = 128;
constexpr int kRowBytesPerVoxel = 20;     // axis-2 pass: f (double), vertex (int32), out (double) per voxel of a row
constexpr int kRowSmemBudget = 96 * 1024;

struct RegionLabels {
  long long v[kMaxRegionLabels];
  float f[kMaxRegionLabels];  // the same labels rounded to float32 (numpy compares a float32 volume in float32)
  int n;
  int has_ignore;
  long long ignore_v;
  float ignore_f;
};

__device__ __forceinline__ bool in_region(const void* p, int dtype, long long i, const RegionLabels& L) {
  bool m = false;
#pragma unroll
  for (int j = 0; j < kMaxRegionLabels; ++j) m |= j < L.n && equals(p, dtype, i, L.v[j], L.f[j]);
  return m;
}

// A voxel is on the border when it is in the mask and a face neighbour is not (or lies outside the volume) along one of
// the axes >= first_axis; axes below first_axis are padding of a lower-rank mask and are not eroded.
__device__ __forceinline__ bool on_border(const void* p, int dtype, long long i, int z, int y, int x, int Z, int Y, int X,
                                          int first_axis, const RegionLabels& L) {
  const long long plane = static_cast<long long>(Y) * X;
  bool interior = true;
  if (first_axis <= 0)
    interior = z > 0 && z < Z - 1 && in_region(p, dtype, i - plane, L) && in_region(p, dtype, i + plane, L);
  if (interior && first_axis <= 1)
    interior = y > 0 && y < Y - 1 && in_region(p, dtype, i - X, L) && in_region(p, dtype, i + X, L);
  if (interior) interior = x > 0 && x < X - 1 && in_region(p, dtype, i - 1, L) && in_region(p, dtype, i + 1, L);
  return !interior;
}

__device__ __forceinline__ unsigned long long block_sum(unsigned long long v, unsigned long long* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  v = 0;
  if (threadIdx.x < blockDim.x / 32) v = red[threadIdx.x];
  if (warp == 0) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  }
  return v;  // valid in thread 0
}

// counts: [TP, FP, FN, TN, n_ref, n_pred] (the last two over all voxels, ignored or not).
__global__ void __launch_bounds__(kMaskThreads) masks_kernel(const void* __restrict__ ref, int ref_dtype,
                                                             const void* __restrict__ pred, int pred_dtype, int Z, int Y,
                                                             int X, int first_axis, RegionLabels L,
                                                             uint8_t* __restrict__ border_ref,
                                                             uint8_t* __restrict__ border_pred,
                                                             unsigned long long* __restrict__ counts) {
  __shared__ unsigned long long red[kMaskThreads / 32];
  const long long n = static_cast<long long>(Z) * Y * X;
  unsigned c[6] = {0, 0, 0, 0, 0, 0};  // per thread: at most ceil(n / (grid * block)) voxels
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int x = static_cast<int>(i % X);
    const long long r = i / X;
    const int y = static_cast<int>(r % Y), z = static_cast<int>(r / Y);
    const bool mr = in_region(ref, ref_dtype, i, L), mp = in_region(pred, pred_dtype, i, L);
    const bool ignored = L.has_ignore && equals(ref, ref_dtype, i, L.ignore_v, L.ignore_f);
    if (!ignored) {
      c[0] += mr && mp;
      c[1] += !mr && mp;
      c[2] += mr && !mp;
      c[3] += !mr && !mp;
    }
    c[4] += mr;
    c[5] += mp;
    border_ref[i] = mr && on_border(ref, ref_dtype, i, z, y, x, Z, Y, X, first_axis, L);
    border_pred[i] = mp && on_border(pred, pred_dtype, i, z, y, x, Z, Y, X, first_axis, L);
  }
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    const unsigned long long s = block_sum(c[j], red);
    if (threadIdx.x == 0 && s) atomicAdd(counts + j, s);
  }
}

// ---- exact squared Euclidean distance transform --------------------------------------------------------------------

// Line accessors: f(q) is the value entering this axis' pass (0 / +inf from the border mask on axis 0, the previous
// pass' squared distance otherwise).
struct MaskLine {
  const uint8_t* p;
  long long st;
  __device__ __forceinline__ double f(int q) const { return p[q * st] ? 0.0 : CUDART_INF; }
};
struct VolLine {
  const double* p;
  long long st;
  __device__ __forceinline__ double f(int q) const { return p[q * st]; }
};

// Abscissa where parabola q (vertex f(q) at q) starts to lie below parabola r < q: both are f + (s (p - .))^2.
__device__ __forceinline__ double meet(double fr, int r, double fq, int q, double s2) {
  const double num = __dadd_rn(__dsub_rn(fq, fr), __dmul_rn(s2, static_cast<double>(static_cast<long long>(q) * q -
                                                                                     static_cast<long long>(r) * r)));
  return __ddiv_rn(num, __dmul_rn(2.0 * s2, static_cast<double>(q - r)));
}

// Felzenszwalb-Huttenlocher along one line of n voxels: out(p) = min_q f(q) + (s (p - q))^2, evaluated for the minimising
// q as f(q) + (s * (p - q))^2 with round-to-nearest products and sums; sqrt_out takes the IEEE square root.  The
// envelope's vertices live in v (stride vst); the boundaries between them are recomputed from f, not stored.
template <typename In, typename V, typename Out>
__device__ __forceinline__ void envelope_line(const In& in, V v, long long vst, int n, double s, bool sqrt_out,
                                              Out out) {
  const double s2 = __dmul_rn(s, s);
  int k = -1;
  for (int q = 0; q < n; ++q) {
    const double fq = in.f(q);
    if (fq == CUDART_INF) continue;
    // the top vertex r is hidden when q overtakes it no later than r overtook its predecessor r0
    while (k >= 1) {
      const int r = v[k * vst], r0 = v[(k - 1) * vst];
      const double fr = in.f(r);
      if (meet(fr, r, fq, q, s2) > meet(in.f(r0), r0, fr, r, s2)) break;
      --k;
    }
    v[++k * vst] = q;
  }
  if (k < 0) {
    for (int p = 0; p < n; ++p) out(p, CUDART_INF);
    return;
  }
  int j = 0, vj = v[0];
  double fj = in.f(vj);
  double next = CUDART_INF;
  if (j < k) {
    const int vn = v[vst];
    next = meet(fj, vj, in.f(vn), vn, s2);
  }
  for (int p = 0; p < n; ++p) {
    while (next < static_cast<double>(p)) {
      ++j;
      vj = v[j * vst];
      fj = in.f(vj);
      next = CUDART_INF;
      if (j < k) {
        const int vn = v[(j + 1) * vst];
        next = meet(fj, vj, in.f(vn), vn, s2);
      }
    }
    const double t = __dmul_rn(s, static_cast<double>(p - vj));
    const double d = __dadd_rn(fj, __dmul_rn(t, t));
    out(p, sqrt_out ? __dsqrt_rn(d) : d);
  }
}

struct GlobalOut {
  double* p;
  long long st;
  __device__ __forceinline__ void operator()(int q, double d) const { p[q * st] = d; }
};

// One thread per line along axis 0 or 1 of a [D0, D1, D2] volume.
template <typename In, typename Src>
__global__ void __launch_bounds__(kEdtLineThreads) edt_lines_kernel(const Src* __restrict__ src, int D0, int D1, int D2,
                                                                    int axis, double s, int* __restrict__ scratch,
                                                                    double* __restrict__ dst) {
  const long long lines = axis == 0 ? static_cast<long long>(D1) * D2 : static_cast<long long>(D0) * D2;
  const long long l = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (l >= lines) return;
  long long base, st;
  int n;
  if (axis == 0) {
    base = l; st = static_cast<long long>(D1) * D2; n = D0;
  } else {
    base = (l / D2) * D1 * D2 + l % D2; st = D2; n = D1;
  }
  envelope_line(In{src + base, st}, scratch + base, st, n, s, false, GlobalOut{dst + base, st});
}

struct SharedOut {
  double* p;
  __device__ __forceinline__ void operator()(int q, double d) const { p[q] = d; }
};

// Axis 2: `rows` rows of length X per block of 32 threads, staged in dynamic shared memory as [rows][X] f, then
// [rows][X] out, then [rows][X] int32 vertices; thread t < rows runs the envelope of row t.
__global__ void __launch_bounds__(32) edt_rows_kernel(const double* __restrict__ src, long long nrows, int X, int rows,
                                                      double s, double* __restrict__ dst) {
  extern __shared__ double smem[];
  double* f = smem;
  double* o = f + static_cast<long long>(rows) * X;
  int* v = reinterpret_cast<int*>(o + static_cast<long long>(rows) * X);
  const long long row0 = static_cast<long long>(blockIdx.x) * rows;
  const int nr = static_cast<int>(min(static_cast<long long>(rows), nrows - row0));
  const long long count = static_cast<long long>(nr) * X;
  const double* in = src + row0 * X;
  for (long long i = threadIdx.x; i < count; i += blockDim.x) f[i] = in[i];
  __syncthreads();
  if (threadIdx.x < nr) {
    const long long off = static_cast<long long>(threadIdx.x) * X;
    envelope_line(VolLine{f + off, 1}, v + off, 1, X, s, true, SharedOut{o + off});
  }
  __syncthreads();
  double* out = dst + row0 * X;
  for (long long i = threadIdx.x; i < count; i += blockDim.x) out[i] = o[i];
}

}  // namespace b2u

using namespace b2u;

extern "C" int b2u_eval_masks(const void* ref, int32_t ref_dtype, const void* pred, int32_t pred_dtype, int32_t ndim,
                              int32_t Z, int32_t Y, int32_t X, const int64_t* labels, int32_t n_labels,
                              int32_t has_ignore, int64_t ignore_label, uint8_t* border_ref, uint8_t* border_pred,
                              int64_t* counts, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!ref || !pred || !labels || !border_ref || !border_pred || !counts)
    return set_error(-1, "b2u_eval_masks: null pointer");
  if (Z <= 0 || Y <= 0 || X <= 0 || ndim < 1 || ndim > 3 || (ndim < 3 && Z != 1) || (ndim < 2 && Y != 1))
    return set_error(-1, "b2u_eval_masks: bad shape %dx%dx%d (rank %d)", Z, Y, X, ndim);
  if (ref_dtype < B2U_EVAL_U8 || ref_dtype > B2U_EVAL_F32 || pred_dtype < B2U_EVAL_U8 || pred_dtype > B2U_EVAL_F32)
    return set_error(-1, "b2u_eval_masks: dtype codes %d / %d", ref_dtype, pred_dtype);
  if (n_labels < 1 || n_labels > kMaxRegionLabels)
    return set_error(-1, "b2u_eval_masks: %d label values (1..%d)", n_labels, kMaxRegionLabels);
  RegionLabels L{};
  for (int j = 0; j < n_labels; ++j) {
    L.v[j] = labels[j];
    L.f[j] = label_as_f32(labels[j]);
  }
  L.n = n_labels;
  L.has_ignore = has_ignore != 0;
  L.ignore_v = ignore_label;
  L.ignore_f = label_as_f32(ignore_label);
  if (cudaMemsetAsync(counts, 0, 6 * sizeof(int64_t), stream) != cudaSuccess)
    return set_error(-1, "b2u_eval_masks: cudaMemsetAsync failed");
  const long long n = static_cast<long long>(Z) * Y * X;
  const long long blocks = std::min<long long>((n + kMaskThreads - 1) / kMaskThreads, static_cast<long long>(num_sms()) * 8);
  masks_kernel<<<static_cast<unsigned>(blocks), kMaskThreads, 0, stream>>>(
      ref, ref_dtype, pred, pred_dtype, Z, Y, X, 3 - ndim, L, border_ref, border_pred,
      reinterpret_cast<unsigned long long*>(counts));
  return check_launch("eval_masks");
}

// Longest row the axis-2 pass can stage (one row per block, the device's opt-in shared memory).
static long long edt_max_row() {
  int dev = 0, optin = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  return optin / kRowBytesPerVoxel;
}

extern "C" int b2u_eval_edt(const uint8_t* border, int32_t Z, int32_t Y, int32_t X, double s0, double s1, double s2,
                            double* tmp, int32_t* scratch, double* dt, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!border || !tmp || !scratch || !dt) return set_error(-1, "b2u_eval_edt: null pointer");
  if (Z <= 0 || Y <= 0 || X <= 0) return set_error(-1, "b2u_eval_edt: bad shape %dx%dx%d", Z, Y, X);
  if (!(s0 > 0.0 && s1 > 0.0 && s2 > 0.0) || isinf(s0) || isinf(s1) || isinf(s2))
    return set_error(-1, "b2u_eval_edt: spacing (%g, %g, %g) must be positive and finite", s0, s1, s2);
  const long long max_row = edt_max_row();
  if (X > max_row) return set_error(-1, "b2u_eval_edt: rows of %d voxels exceed the %lld a block can stage", X, max_row);
  // axis 0: border -> dt, axis 1: dt -> tmp, axis 2 (+ sqrt): tmp -> dt
  const long long l0 = static_cast<long long>(Y) * X, l1 = static_cast<long long>(Z) * X;
  edt_lines_kernel<MaskLine, uint8_t><<<static_cast<unsigned>((l0 + kEdtLineThreads - 1) / kEdtLineThreads),
                                        kEdtLineThreads, 0, stream>>>(border, Z, Y, X, 0, s0, scratch, dt);
  int rc = check_launch("eval_edt_axis0");
  if (rc) return rc;
  edt_lines_kernel<VolLine, double><<<static_cast<unsigned>((l1 + kEdtLineThreads - 1) / kEdtLineThreads),
                                      kEdtLineThreads, 0, stream>>>(dt, Z, Y, X, 1, s1, scratch, tmp);
  if ((rc = check_launch("eval_edt_axis1"))) return rc;
  const int rows = static_cast<int>(std::max<long long>(1, std::min<long long>(32, kRowSmemBudget / (kRowBytesPerVoxel * static_cast<long long>(X)))));
  const size_t smem = static_cast<size_t>(rows) * X * kRowBytesPerVoxel;
  if (cudaFuncSetAttribute(edt_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)) !=
      cudaSuccess)
    return set_error(-1, "b2u_eval_edt: cannot reserve %zu bytes of shared memory", smem);
  const long long nrows = static_cast<long long>(Z) * Y;
  edt_rows_kernel<<<static_cast<unsigned>((nrows + rows - 1) / rows), 32, smem, stream>>>(tmp, nrows, X, rows, s2, dt);
  return check_launch("eval_edt_axis2");
}

extern "C" int b2u_eval_sum_f64(const double* x, int64_t n, double* work, b2u_stream_t stream) {
  if (!x || !work) return set_error(-1, "b2u_eval_sum_f64: null pointer");
  if (n <= 0) return set_error(-1, "b2u_eval_sum_f64: n=%lld", static_cast<long long>(n));
  return pairwise_sum_f64(x, n, work, static_cast<cudaStream_t>(stream));
}
