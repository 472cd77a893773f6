// Dataset fingerprint on the device (reference: experiment_planning/dataset_fingerprint/fingerprint_extractor.py:41-80
// `collect_foreground_intensities` and the dataset statistics of `run`, lines 156-184).  The foreground voxel list
// itself comes from preprocess_seg.cu's `b2u_fp_fg_compact` (`seg[0] > 0` in C order).
//
//   b2u_fp_gather   samples[c][j] = img[c][idx[ranks[c][j]]] for every channel in one launch (ranks drawn on the host
//                   by the reference's RandomState, one stream across the channels), or the whole foreground
//                   img[c][idx[j]] when ranks is null.  The output rows are strided, so a case's samples land in
//                   place in the dataset's preallocated vector.
//   b2u_fp_select   the values at R <= 8 given 0-based ranks of a float32 vector, exact (what np.partition puts there):
//                   an MSD radix select over order-preserving uint32 keys (-0.0 keyed as +0.0, so zeros tie as in
//                   numpy's comparisons), four passes of 8 bits.  Each pass builds one 256-bin histogram per distinct
//                   prefix in shared memory (warp-aggregated with match_any, so ties cost one atomic per warp), merges
//                   it into global memory with atomics, and one block picks the next digit of every rank on the
//                   device: no host synchronisation between passes.
//   b2u_fp_moments  numpy's `_mean` and `_var` (std without ZScore's clamp) in float32, or in float64 on a converted
//                   copy (a vector the reference's concatenation promoted): preprocess.cu's pairwise-sum tree, then
//                   mean = T(f64(sum) / n), std = sqrt(T(f64(sum((x - mean)^2)) / n)).
#include <algorithm>
#include <climits>

#include "../../include/dinounet_b200.h"
#include "gemm_common.h"
#include "host_util.h"

namespace b2u {

constexpr int kFpThreads = 256;
constexpr int kMaxRanks = B2U_FP_MAX_RANKS;
constexpr int kBins = 256;

struct SelectState {
  unsigned long long k[kMaxRanks];  // the rank still to find inside the current prefix
  uint32_t prefix[kMaxRanks];       // the key bits decided so far
  int slot[kMaxRanks];              // the first rank with the same prefix: its histogram serves this rank
};

struct SelectRanks {
  long long k[kMaxRanks];
};

__device__ __forceinline__ uint32_t to_key(float v) {
  uint32_t b = __float_as_uint(v);
  if (b == 0x80000000u) b = 0u;
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ float from_key(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// ---- gathers --------------------------------------------------------------------------------------------------------

// blockIdx.y = channel.
__global__ void __launch_bounds__(kFpThreads) fp_gather_kernel(const float* __restrict__ img, long long n_vox,
                                                               const int32_t* __restrict__ idx,
                                                               const int64_t* __restrict__ ranks, long long m,
                                                               float* __restrict__ out, long long out_stride) {
  const long long j = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (j >= m) return;
  const long long v = idx[ranks ? ranks[blockIdx.y * m + j] : j];
  out[blockIdx.y * out_stride + j] = img[blockIdx.y * n_vox + v];
}

// ---- radix select ---------------------------------------------------------------------------------------------------

__global__ void select_init_kernel(SelectRanks r, int R, SelectState* __restrict__ st,
                                   unsigned long long* __restrict__ hist) {
  for (int i = threadIdx.x; i < kMaxRanks * kBins; i += blockDim.x) hist[i] = 0ull;
  if (threadIdx.x < kMaxRanks) {
    st->k[threadIdx.x] = threadIdx.x < R ? static_cast<unsigned long long>(r.k[threadIdx.x]) : 0ull;
    st->prefix[threadIdx.x] = 0u;
    st->slot[threadIdx.x] = 0;
  }
}

// Pass p (digit bits [shift, shift + 8), shift = 24 - 8p): every distinct prefix counts the digits of the keys that
// carry it.  The warps walk the vector in lockstep so the ballots and match_any see whole warps.
__global__ void __launch_bounds__(kFpThreads) select_hist_kernel(const float* __restrict__ x, long long n, int R,
                                                                 int shift, const SelectState* __restrict__ st,
                                                                 unsigned long long* __restrict__ hist) {
  __shared__ uint32_t sh[kMaxRanks][kBins];
  __shared__ uint32_t s_prefix[kMaxRanks];
  __shared__ int s_own[kMaxRanks];
  for (int i = threadIdx.x; i < kMaxRanks * kBins; i += blockDim.x) (&sh[0][0])[i] = 0u;
  if (threadIdx.x < R) {
    s_prefix[threadIdx.x] = st->prefix[threadIdx.x];
    s_own[threadIdx.x] = st->slot[threadIdx.x] == static_cast<int>(threadIdx.x);
  }
  __syncthreads();
  const uint32_t decided = shift == 24 ? 0u : ~((1u << (shift + 8)) - 1u);
  const int lane = threadIdx.x & 31;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long steps = (n + stride - 1) / stride;
  const long long first = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (long long s = 0; s < steps; ++s) {
    const long long i = first + s * stride;
    const bool valid = i < n;
    const uint32_t key = valid ? to_key(x[i]) : 0u;
    const uint32_t digit = (key >> shift) & 0xffu;
    for (int r = 0; r < R; ++r) {
      if (!s_own[r]) continue;  // block-uniform
      const bool hit = valid && ((key ^ s_prefix[r]) & decided) == 0u;
      const unsigned act = __ballot_sync(0xffffffffu, hit);
      if (hit) {
        const unsigned peers = __match_any_sync(act, digit);
        if (lane == __ffs(peers) - 1) atomicAdd(&sh[r][digit], static_cast<uint32_t>(__popc(peers)));
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < R * kBins; i += blockDim.x) {
    const uint32_t c = (&sh[0][0])[i];
    if (c) atomicAdd(hist + i, static_cast<unsigned long long>(c));
  }
}

// One warp per rank: the bin of the merged histogram that holds the rank, then the prefixes' new owners, then the
// histograms are cleared for the next pass.  The last pass writes the values.
__global__ void __launch_bounds__(kMaxRanks * 32) select_pick_kernel(int R, int shift, SelectState* __restrict__ st,
                                                                     unsigned long long* __restrict__ hist,
                                                                     float* __restrict__ out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp < R) {
    const unsigned long long* h = hist + st->slot[warp] * kBins;
    const unsigned long long k = st->k[warp];
    unsigned long long c[8], local = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      c[j] = h[lane * 8 + j];
      local += c[j];
    }
    unsigned long long incl = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    unsigned long long before = incl - local;
    // exactly one lane holds the rank: before <= k < incl
    if (before <= k && k < incl) {
      int d = -1;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (d < 0) {
          if (k < before + c[j]) d = j;
          else before += c[j];
        }
      }
      st->k[warp] = k - before;
      st->prefix[warp] |= static_cast<uint32_t>(lane * 8 + d) << shift;
    }
  }
  __syncthreads();
  if (threadIdx.x < R) {
    const uint32_t p = st->prefix[threadIdx.x];
    int s = threadIdx.x;
    for (int q = 0; q < static_cast<int>(threadIdx.x); ++q)
      if (st->prefix[q] == p) {
        s = q;
        break;
      }
    st->slot[threadIdx.x] = s;
    if (shift == 0) out[threadIdx.x] = from_key(p);
  }
  for (int i = threadIdx.x; i < kMaxRanks * kBins; i += blockDim.x) hist[i] = 0ull;
}

// ---- moments --------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kFpThreads) widen_kernel(const float* __restrict__ x, long long n,
                                                           double* __restrict__ y) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) y[i] = static_cast<double>(x[i]);
}

// numpy's _mean (stage 0) and the std of _var (stage 1) from the pairwise sum in val[0]; no clamp.
__global__ void moments_finalize_f32_kernel(const float* __restrict__ val, long long n, int stage,
                                            float* __restrict__ stats) {
  const float q = __double2float_rn(__ddiv_rn(static_cast<double>(val[0]), static_cast<double>(n)));
  stats[stage] = stage == 0 ? q : __fsqrt_rn(q);
}

__global__ void moments_finalize_f64_kernel(const double* __restrict__ val, long long n, int stage,
                                            double* __restrict__ stats) {
  const double q = __ddiv_rn(val[0], static_cast<double>(n));
  stats[stage] = stage == 0 ? q : __dsqrt_rn(q);
}

static long long tree_slots(long long n) { return (n + 7) / 8; }

}  // namespace b2u

using namespace b2u;

extern "C" int b2u_fp_gather(const float* img, int32_t C, int64_t n_vox, const int32_t* idx, const int64_t* ranks,
                             int64_t m, float* out, int64_t out_stride, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!img || !idx || !out) return set_error(-1, "b2u_fp_gather: null pointer");
  if (C < 1 || C > 65535 || n_vox <= 0 || m <= 0 || out_stride < m)
    return set_error(-1, "b2u_fp_gather: C=%d n_vox=%lld m=%lld stride=%lld", C, static_cast<long long>(n_vox),
                     static_cast<long long>(m), static_cast<long long>(out_stride));
  const long long blocks = (m + kFpThreads - 1) / kFpThreads;
  if (blocks > INT_MAX) return set_error(-1, "b2u_fp_gather: m=%lld too large", static_cast<long long>(m));
  fp_gather_kernel<<<dim3(static_cast<unsigned>(blocks), C), kFpThreads, 0, stream>>>(img, n_vox, idx, ranks, m, out,
                                                                                     out_stride);
  return check_launch("fp_gather");
}

extern "C" int64_t b2u_fp_select_work_bytes(void) {
  return static_cast<int64_t>(sizeof(SelectState) + sizeof(unsigned long long) * kMaxRanks * kBins);
}

extern "C" int b2u_fp_select(const float* x, int64_t n, const int64_t* ranks, int32_t R, void* work, float* out,
                             b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!x || !ranks || !work || !out) return set_error(-1, "b2u_fp_select: null pointer");
  if (n <= 0 || R < 1 || R > kMaxRanks)
    return set_error(-1, "b2u_fp_select: n=%lld R=%d", static_cast<long long>(n), R);
  SelectRanks r{};
  for (int i = 0; i < R; ++i) {
    if (ranks[i] < 0 || ranks[i] >= n)
      return set_error(-1, "b2u_fp_select: rank %lld outside [0, %lld)", static_cast<long long>(ranks[i]),
                       static_cast<long long>(n));
    r.k[i] = ranks[i];
  }
  SelectState* st = static_cast<SelectState*>(work);
  unsigned long long* hist = reinterpret_cast<unsigned long long*>(static_cast<char*>(work) + sizeof(SelectState));
  select_init_kernel<<<1, kFpThreads, 0, stream>>>(r, R, st, hist);
  int rc = check_launch("fp_select_init");
  if (rc) return rc;
  const int grid = static_cast<int>(std::max<long long>(
      1, std::min<long long>((n + kFpThreads - 1) / kFpThreads, static_cast<long long>(num_sms()) * 8)));
  for (int shift = 24; shift >= 0; shift -= 8) {
    select_hist_kernel<<<grid, kFpThreads, 0, stream>>>(x, n, R, shift, st, hist);
    if ((rc = check_launch("fp_select_hist"))) return rc;
    select_pick_kernel<<<1, kMaxRanks * 32, 0, stream>>>(R, shift, st, hist, out);
    if ((rc = check_launch("fp_select_pick"))) return rc;
  }
  return 0;
}

extern "C" int64_t b2u_fp_moments_work_bytes(int64_t n, int32_t f64) {
  if (n <= 0) return 0;
  return f64 ? 8 * (n + tree_slots(n)) : 4 * tree_slots(n);
}

extern "C" int b2u_fp_moments(const float* x, int64_t n, int32_t f64, int32_t with_std, void* work, void* stats,
                              b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!x || !work || !stats) return set_error(-1, "b2u_fp_moments: null pointer");
  if (n <= 0) return set_error(-1, "b2u_fp_moments: n=%lld", static_cast<long long>(n));
  const int stages = with_std ? 2 : 1;
  int rc;
  if (f64) {
    double* y = static_cast<double*>(work);
    double* tree = y + n;
    double* s = static_cast<double*>(stats);
    widen_kernel<<<static_cast<unsigned>((n + kFpThreads - 1) / kFpThreads), kFpThreads, 0, stream>>>(x, n, y);
    if ((rc = check_launch("fp_moments_widen"))) return rc;
    for (int stage = 0; stage < stages; ++stage) {
      rc = stage == 0 ? pairwise_sum_f64(y, n, tree, stream) : pairwise_sum_sq_f64(y, n, s, tree, stream);
      if (rc) return rc;
      moments_finalize_f64_kernel<<<1, 1, 0, stream>>>(tree, n, stage, s);
      if ((rc = check_launch("fp_moments_finalize"))) return rc;
    }
    return 0;
  }
  float* tree = static_cast<float*>(work);
  float* s = static_cast<float*>(stats);
  for (int stage = 0; stage < stages; ++stage) {
    if ((rc = pairwise_sum_planes_f32(x, n, 1, stage, s, tree, tree_slots(n), stream))) return rc;
    moments_finalize_f32_kernel<<<1, 1, 0, stream>>>(tree, n, stage, s);
    if ((rc = check_launch("fp_moments_finalize"))) return rc;
  }
  return 0;
}
