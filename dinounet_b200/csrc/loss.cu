// Dice + cross-entropy loss and the online-validation statistics, fused (reference: training/loss/compound_losses.py:31-56,
// dice.py:72-119, robust_ce_loss.py:12-16, nnUNetTrainer.py:363-365 [build], :961-1005 [validation_step]).
//
// The reference runs, on the logits [B,C,H,W] the forward path produces: softmax, a one-hot scatter, three masked
// reductions, cross_entropy, argmax, another scatter and the tp/fp/fn products — about a dozen full passes over
// B*C*H*W.  Here ONE pass reads the logits and labels once and produces every sum (block partials in fp64, fixed
// reduction order -> deterministic), a one-block epilogue forms the loss, and a second pass writes dLoss/dlogits.
// HBM-bound: (4C + label) B/pixel forward, (8C + label) B/pixel backward.
//
// Region-based training (DC_and_BCE_loss, compound_losses.py:59-99, sigmoid Dice with do_bg, optional ignore channel)
// uses the same three-step shape on [B, R, plane] logits and [B, R(+1), plane] real-valued targets.
//
// Data-parallel batch Dice (dice.py:106-110): given a batch_sums buffer, the statistics pass also writes the per-class
// batch sums [C][3] (intersect, sum_pred, sum_gt; fp64, on the device), which the caller all-reduces across ranks before
// the finalisation; without one (label maps only), the finalisation and the gradient sum the per-sample records
// themselves, in the same order.  The backward may take the incoming gradient as device scalars: the CE/BCE part is
// scaled by the local one, the Dice part by the all-reduced one (the backward of AllGatherGrad, ddp_allgather.py:43-48).
// No host sync.
//
// An ignore label (DC_and_CE_loss(..., ignore_label), compound_losses.py:38-53) runs the kernels' IGN instantiations:
// masked sums, a valid-pixel count per sample, CE over the valid pixels only.
#include "common.cuh"
#include "host_util.h"
#include "gemm_common.h"
#include "../../include/dinounet_b200.h"

#include <algorithm>
#include <initializer_list>
#include <type_traits>
#include <utility>

namespace b2u {

constexpr int kStat = 6;  // per (sample, class): intersect, sum_pred, sum_gt, tp, fp, fn

// one sample's record of label-map sums: kStat per class, then the CE sum (and, with an ignore label, the valid-pixel
// count)
__host__ __device__ constexpr int record_len(int C, bool ign) { return C * kStat + 1 + (ign ? 1 : 0); }

template <typename L> __device__ __forceinline__ int load_label(const void* t, long long i) {
  return static_cast<int>(static_cast<const L*>(t)[i]);
}
__device__ __forceinline__ int label_at(const void* t, int kind, long long i) {
  switch (kind) {
    case 0: return load_label<uint8_t>(t, i);
    case 1: return load_label<int32_t>(t, i);
    case 2: return load_label<int64_t>(t, i);
    default: return load_label<float>(t, i);
  }
}

// softmax of one pixel (class stride = plane); returns log-sum-exp pieces
template <int C>
__device__ __forceinline__ void pixel_softmax(const float* __restrict__ z, long long plane, float (&p)[C], float& mx,
                                              float& lse, int& amax) {
  float v[C];
#pragma unroll
  for (int c = 0; c < C; ++c) v[c] = z[c * plane];
  mx = v[0];
  amax = 0;
#pragma unroll
  for (int c = 1; c < C; ++c)
    if (v[c] > mx) { mx = v[c]; amax = c; }  // first maximum wins, like torch.argmax
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < C; ++c) { p[c] = expf(v[c] - mx); s += p[c]; }
  const float inv = 1.f / s;
#pragma unroll
  for (int c = 0; c < C; ++c) p[c] *= inv;
  lse = logf(s);
}

// target value as a real number (region targets are used as they are, not as booleans)
__device__ __forceinline__ float value_at(const void* t, int kind, long long i) {
  switch (kind) {
    case 0: return static_cast<float>(static_cast<const uint8_t*>(t)[i]);
    case 1: return static_cast<float>(static_cast<const int32_t*>(t)[i]);
    case 2: return static_cast<float>(static_cast<const int64_t*>(t)[i]);
    default: return static_cast<const float*>(t)[i];
  }
}

// fp64 block reduction (256 threads) of N per-thread fp32 sums in a fixed order; thread k < N writes sum k to out[k]
template <int N>
__device__ __forceinline__ void block_sum_store(const float (&acc)[N], double* __restrict__ out) {
  static_assert(N <= 256, "one output per thread");
  __shared__ double red[8][N];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    double v = static_cast<double>(acc[k]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < N) {
    double v = 0;
    for (int w = 0; w < 8; ++w) v += red[w][threadIdx.x];
    out[threadIdx.x] = v;
  }
}

// IGN: pixels labelled `ignore_label` add nothing, and each sample's record gains the valid-pixel count after the CE sum
// (RobustCrossEntropyLoss ignore_index + MemoryEfficientSoftDiceLoss loss_mask).  Their logits are read as without IGN,
// but reach no sum.
template <int C, bool IGN = false>
__global__ void __launch_bounds__(256) loss_stats_kernel(const float* __restrict__ logits, const void* __restrict__ target,
                                                         int tkind, double* __restrict__ partial, int* __restrict__ bad,
                                                         long long plane, int ignore_label) {
  const int b = blockIdx.y;
  const float* zb = logits + static_cast<long long>(b) * C * plane;
  constexpr int K = record_len(C, IGN);
  float acc[K];
#pragma unroll
  for (int k = 0; k < K; ++k) acc[k] = 0.f;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < plane;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float p[C], mx, lse;
    int amax;
    pixel_softmax<C>(zb + i, plane, p, mx, lse, amax);
    int t = label_at(target, tkind, static_cast<long long>(b) * plane + i);
    if constexpr (IGN) {
      if (t == ignore_label) continue;
      acc[C * kStat + 1] += 1.f;
    }
    if (t < 0 || t >= C) { *bad = 1; t = 0; }
    acc[C * kStat] += lse - (zb[t * plane + i] - mx);
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const float y = t == c ? 1.f : 0.f, h = amax == c ? 1.f : 0.f;
      acc[c * kStat + 0] += p[c] * y;
      acc[c * kStat + 1] += p[c];
      acc[c * kStat + 2] += y;
      acc[c * kStat + 3] += h * y;
      acc[c * kStat + 4] += h * (1.f - y);
      acc[c * kStat + 5] += (1.f - h) * y;
    }
  }
  block_sum_store<K>(acc, partial + (static_cast<long long>(b) * gridDim.x + blockIdx.x) * K);
}

// stats[b][k] = sum over the blocks of sample b of partial sum k, in block order
__device__ __forceinline__ void reduce_sample_stats(const double* __restrict__ partial, double* __restrict__ stats, int B,
                                                    int K, int nblk) {
  for (int j = threadIdx.x; j < B * K; j += blockDim.x) {
    const int b = j / K, k = j - b * K;
    double v = 0;
    for (int n = 0; n < nblk; ++n) v += partial[(static_cast<long long>(b) * nblk + n) * K + k];
    stats[j] = v;
  }
}

// (intersect, sum_pred, sum_gt) of class c: gsum[c] when the batch sums [C][3] are given, else the records of samples
// b0 <= b < b1 summed in sample order from 0 -- the order dice_batch_sums_kernel sums in, so that skipping it changes no
// bit.  K = per-sample record length; class c's record at c*kStat.
__device__ __forceinline__ void dice_sums(const double* __restrict__ gsum, const double* __restrict__ stats, int K, int c,
                                          int b0, int b1, double& I, double& P, double& G) {
  if (gsum) {
    I = gsum[c * 3];
    P = gsum[c * 3 + 1];
    G = gsum[c * 3 + 2];
    return;
  }
  I = P = G = 0;
  for (int b = b0; b < b1; ++b) {
    I += stats[b * K + c * kStat];
    P += stats[b * K + c * kStat + 1];
    G += stats[b * K + c * kStat + 2];
  }
}

// bsum[c][3] = (intersect, sum_pred, sum_gt) of class c over the batch: per sample in block order, then in sample order.
// The per-sample sums go through `stats` (B*K doubles) so that every thread of the block takes part in the long first
// level, instead of one thread per output running over all B*nblk partials.
__global__ void dice_batch_sums_kernel(const double* __restrict__ partial, double* __restrict__ stats,
                                       double* __restrict__ bsum, int B, int C, int K, int nblk) {
  reduce_sample_stats(partial, stats, B, K, nblk);
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x)
    dice_sums(nullptr, stats, K, c, 0, B, bsum[c * 3], bsum[c * 3 + 1], bsum[c * 3 + 2]);
}

// stats: double [B][C*6 + 1 (+1 with IGN)] (the sample's CE sum, and its valid-pixel count).  out: float[3] = loss, ce,
// dice term.  gsum (optional): batch sums [C][3] to take the batch Dice from (all-reduced across data-parallel ranks).
template <bool IGN = false>
__global__ void loss_finalize_kernel(const double* __restrict__ partial, double* __restrict__ stats,
                                     const double* __restrict__ gsum, float* __restrict__ out,
                                     int64_t* __restrict__ tpfpfn, int B, int C, int nblk, long long plane, float w_ce,
                                     float w_dice, int batch_dice, int do_bg, float smooth) {
  const int K = record_len(C, IGN);
  reduce_sample_stats(partial, stats, B, K, nblk);
  __syncthreads();
  if (threadIdx.x != 0) return;
  double ce = 0;
  for (int b = 0; b < B; ++b) ce += stats[b * K + C * kStat];
  if constexpr (IGN) {
    double valid = 0;
    for (int b = 0; b < B; ++b) valid += stats[b * K + C * kStat + 1];
    ce = valid > 0 ? ce / valid : 0.0;  // no valid pixel: the reference skips the CE (compound_losses.py:52-53)
  } else {
    ce /= static_cast<double>(B) * static_cast<double>(plane);
  }
  const int c0 = do_bg ? 0 : 1, nd = batch_dice ? 1 : B;  // Dice terms: one of the batch, or one per sample
  double dc = 0;
  for (int d = 0; d < nd; ++d)
    for (int c = c0; c < C; ++c) {
      double I, P, G;
      dice_sums(batch_dice ? gsum : nullptr, stats, K, c, batch_dice ? 0 : d, batch_dice ? B : d + 1, I, P, G);
      dc += (2 * I + smooth) / fmax(G + P + smooth, 1e-8);
    }
  dc /= static_cast<double>(nd) * (C - c0);
  out[1] = static_cast<float>(ce);
  out[2] = static_cast<float>(-dc);
  out[0] = static_cast<float>(w_ce * ce - w_dice * dc);
  if (tpfpfn)
    for (int c = 0; c < C; ++c)
      for (int s = 0; s < 3; ++s) {
        double v = 0;
        for (int b = 0; b < B; ++b) v += stats[b * K + c * kStat + 3 + s];
        tpfpfn[s * C + c] = static_cast<int64_t>(v + 0.5);
      }
}

// IGN: the CE weight is w_ce / (valid pixels of the batch), 0 without any, and the gradient is 0 at ignored pixels.
template <int C, bool IGN = false>
__global__ void __launch_bounds__(256) loss_grad_kernel(const float* __restrict__ logits, const void* __restrict__ target,
                                                        int tkind, const double* __restrict__ stats,
                                                        const double* __restrict__ gsum, float* __restrict__ grad,
                                                        int B, long long plane, float w_ce, float w_dice, int batch_dice,
                                                        int do_bg, float smooth, float grad_scale,
                                                        const float* __restrict__ ce_scale,
                                                        const float* __restrict__ dice_scale, int ignore_label) {
  const int b = blockIdx.y;
  constexpr int K = record_len(C, IGN);
  // per-class dice coefficients a_c, b_c with d(dice term)/dp_c = a_c * y_c + b_c
  __shared__ float sa[C], sb[C], s_ce;
  if (IGN && threadIdx.x == 32) {
    double valid = 0;
    for (int n = 0; n < B; ++n) valid += stats[n * K + C * kStat + 1];
    s_ce = valid > 0 ? static_cast<float>(w_ce / valid) * (ce_scale ? *ce_scale : 1.f) : 0.f;
  }
  if (threadIdx.x < C) {
    const int c = threadIdx.x, c0 = do_bg ? 0 : 1;
    float a = 0.f, bb = 0.f;
    if (c >= c0) {
      double I = 0, P = 0, G = 0;
      if (batch_dice && gsum) {
        I = gsum[c * 3];
        P = gsum[c * 3 + 1];
        G = gsum[c * 3 + 2];
      } else {
        for (int n = batch_dice ? 0 : b; n < (batch_dice ? B : b + 1); ++n) {
          I += stats[n * K + c * kStat];
          P += stats[n * K + c * kStat + 1];
          G += stats[n * K + c * kStat + 2];
        }
      }
      const double num = 2 * I + smooth, raw = G + P + smooth, den = fmax(raw, 1e-8);
      const double cnt = batch_dice ? static_cast<double>(C - c0) : static_cast<double>(B) * (C - c0);
      a = static_cast<float>(-2.0 / (den * cnt));                              // through the intersection
      bb = raw > 1e-8 ? static_cast<float>(num / (den * den * cnt)) : 0.f;      // through sum_pred (clip passes no grad)
    }
    const float ds = dice_scale ? *dice_scale : 1.f;
    sa[c] = a * ds;
    sb[c] = bb * ds;
  }
  __syncthreads();
  const float* zb = logits + static_cast<long long>(b) * C * plane;
  float* gb = grad + static_cast<long long>(b) * C * plane;
  const float ce_w = IGN ? s_ce
                         : w_ce / (static_cast<float>(B) * static_cast<float>(plane)) * (ce_scale ? *ce_scale : 1.f);
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < plane;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float p[C], mx, lse;
    int amax;
    pixel_softmax<C>(zb + i, plane, p, mx, lse, amax);
    int t = label_at(target, tkind, static_cast<long long>(b) * plane + i);
    if constexpr (IGN) {
      if (t == ignore_label) {
#pragma unroll
        for (int c = 0; c < C; ++c) gb[c * plane + i] = 0.f;
        continue;
      }
    }
    if (t < 0 || t >= C) t = 0;
    float g[C], dot = 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      g[c] = w_dice * (sa[c] * (t == c ? 1.f : 0.f) + sb[c]);
      dot += g[c] * p[c];
    }
#pragma unroll
    for (int c = 0; c < C; ++c)
      gb[c * plane + i] = grad_scale * (ce_w * (p[c] - (t == c ? 1.f : 0.f)) + p[c] * (g[c] - dot));
  }
}

// ---- region-based (sigmoid) Dice + BCE.  Per (sample, region): intersect, sum_pred, sum_gt over valid pixels and the
// validation tp, fp, fn of sigmoid(z) > 0.5 weighted by 1 - t_ign; per sample: BCE sum over valid pixels, valid count.
__host__ __device__ constexpr int region_record_len(int R) { return R * kStat + 2; }

__device__ __forceinline__ float bce_with_logits(float z, float y) {
  return fmaxf(z, 0.f) - z * y + log1pf(expf(-fabsf(z)));
}

template <int R>
__global__ void __launch_bounds__(256) region_stats_kernel(const float* __restrict__ logits, const void* __restrict__ target,
                                                           int tkind, int has_ignore, double* __restrict__ partial,
                                                           long long plane) {
  const int b = blockIdx.y;
  const float* zb = logits + static_cast<long long>(b) * R * plane;
  const long long tb = static_cast<long long>(b) * (R + has_ignore) * plane;
  constexpr int K = region_record_len(R);
  float acc[K];
#pragma unroll
  for (int k = 0; k < K; ++k) acc[k] = 0.f;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < plane;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float w = 1.f, m = 1.f;  // validation weight 1 - t_ign, loss mask (1 - t_ign) != 0
    if (has_ignore) {
      w = 1.f - value_at(target, tkind, tb + R * plane + i);
      m = w != 0.f ? 1.f : 0.f;
    }
    float bce = 0.f;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const float z = zb[r * plane + i], y = value_at(target, tkind, tb + r * plane + i);
      const float x = 1.f / (1.f + expf(-z));
      const float h = x > 0.5f ? 1.f : 0.f;  // == torch.sigmoid(z) > 0.5 on fp32 (fast math is off)
      acc[r * kStat + 0] += x * y * m;
      acc[r * kStat + 1] += x * m;
      acc[r * kStat + 2] += y * m;
      acc[r * kStat + 3] += h * y * w;
      acc[r * kStat + 4] += h * (1.f - y) * w;
      acc[r * kStat + 5] += (1.f - h) * y * w;
      bce += bce_with_logits(z, y);
    }
    acc[R * kStat] += bce * m;
    acc[R * kStat + 1] += m;
  }
  block_sum_store<K>(acc, partial + (static_cast<long long>(b) * gridDim.x + blockIdx.x) * K);
}

// out: float[3] = loss, BCE, dice term.  tpfpfn: float [3][R] summed over the batch.
__global__ void region_finalize_kernel(const double* __restrict__ partial, double* __restrict__ stats,
                                       const double* __restrict__ bsum, float* __restrict__ out,
                                       float* __restrict__ tpfpfn, int B, int R, int nblk, long long plane, float w_ce,
                                       float w_dice, int batch_dice, int has_ignore, float smooth) {
  const int K = region_record_len(R);
  reduce_sample_stats(partial, stats, B, K, nblk);
  __syncthreads();
  if (threadIdx.x != 0) return;
  double bce = 0, valid = 0;
  for (int b = 0; b < B; ++b) {
    bce += stats[b * K + R * kStat];
    valid += stats[b * K + R * kStat + 1];
  }
  // masked: sum(bce * mask) / clip(#valid pixels, 1e-8) -- pixels, not pixel x region pairs (compound_losses.py:95)
  bce /= has_ignore ? fmax(valid, 1e-8) : static_cast<double>(B) * R * static_cast<double>(plane);
  double dc = 0;
  if (batch_dice) {
    for (int r = 0; r < R; ++r)
      dc += (2 * bsum[r * 3] + smooth) / fmax(bsum[r * 3 + 2] + bsum[r * 3 + 1] + smooth, 1e-8);
    dc /= R;
  } else {
    for (int b = 0; b < B; ++b)
      for (int r = 0; r < R; ++r) {
        const double I = stats[b * K + r * kStat], P = stats[b * K + r * kStat + 1], G = stats[b * K + r * kStat + 2];
        dc += (2 * I + smooth) / fmax(G + P + smooth, 1e-8);
      }
    dc /= static_cast<double>(B) * R;
  }
  out[1] = static_cast<float>(bce);
  out[2] = static_cast<float>(-dc);
  out[0] = static_cast<float>(w_ce * bce - w_dice * dc);
  if (tpfpfn)
    for (int r = 0; r < R; ++r)
      for (int s = 0; s < 3; ++s) {
        double v = 0;
        for (int b = 0; b < B; ++b) v += stats[b * K + r * kStat + 3 + s];
        tpfpfn[s * R + r] = static_cast<float>(v);
      }
}

template <int R>
__global__ void __launch_bounds__(256) region_grad_kernel(const float* __restrict__ logits, const void* __restrict__ target,
                                                          int tkind, int has_ignore, const double* __restrict__ stats,
                                                          const double* __restrict__ bsum, float* __restrict__ grad,
                                                          int B, long long plane, float w_ce, float w_dice,
                                                          int batch_dice, float smooth,
                                                          const float* __restrict__ ce_scale,
                                                          const float* __restrict__ dice_scale) {
  const int b = blockIdx.y;
  constexpr int K = region_record_len(R);
  // d(dice term)/dx_r = (a_r * y_r + b_r) * m;  d BCE / dz_r = bce_w * (x_r - y_r) * m
  __shared__ float sa[R], sb[R], s_bce;
  if (threadIdx.x < R) {
    const int r = threadIdx.x;
    double I = 0, P = 0, G = 0;
    if (batch_dice) {
      I = bsum[r * 3];
      P = bsum[r * 3 + 1];
      G = bsum[r * 3 + 2];
    } else {
      I = stats[b * K + r * kStat];
      P = stats[b * K + r * kStat + 1];
      G = stats[b * K + r * kStat + 2];
    }
    const double num = 2 * I + smooth, raw = G + P + smooth, den = fmax(raw, 1e-8);
    const double cnt = batch_dice ? static_cast<double>(R) : static_cast<double>(B) * R;
    const float ds = w_dice * (dice_scale ? *dice_scale : 1.f);
    sa[r] = ds * static_cast<float>(-2.0 / (den * cnt));
    sb[r] = raw > 1e-8 ? ds * static_cast<float>(num / (den * den * cnt)) : 0.f;  // the clip passes no gradient
  }
  if (threadIdx.x == 32) {
    double norm = static_cast<double>(B) * R * static_cast<double>(plane);
    if (has_ignore) {
      double valid = 0;
      for (int n = 0; n < B; ++n) valid += stats[n * K + R * kStat + 1];
      norm = fmax(valid, 1e-8);
    }
    s_bce = static_cast<float>(w_ce / norm) * (ce_scale ? *ce_scale : 1.f);
  }
  __syncthreads();
  const float* zb = logits + static_cast<long long>(b) * R * plane;
  float* gb = grad + static_cast<long long>(b) * R * plane;
  const long long tb = static_cast<long long>(b) * (R + has_ignore) * plane;
  const float bw = s_bce;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < plane;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float m = 1.f;
    if (has_ignore) m = 1.f - value_at(target, tkind, tb + R * plane + i) != 0.f ? 1.f : 0.f;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const float z = zb[r * plane + i], y = value_at(target, tkind, tb + r * plane + i);
      const float x = 1.f / (1.f + expf(-z));
      gb[r * plane + i] = m * (bw * (x - y) + x * (1.f - x) * (sa[r] * y + sb[r]));
    }
  }
}

static int stats_blocks(long long plane) {
  return static_cast<int>(std::max<long long>(1, std::min<long long>((plane + 256 * 16 - 1) / (256 * 16), 1024)));
}

static int grad_blocks(long long plane) {
  return static_cast<int>(std::max<long long>(1, std::min<long long>((plane + 1023) / 1024, 4096)));
}

// work: B*nblk block partials of K doubles each, then the B per-sample records (K = the record length)
static int64_t work_doubles(int32_t B, int64_t plane, int K) {
  return static_cast<int64_t>(B) * stats_blocks(plane) * K + static_cast<int64_t>(B) * K;
}

template <typename T> static T* sample_records(T* work, int32_t B, int64_t plane, int K) {
  return work + static_cast<int64_t>(B) * stats_blocks(plane) * K;
}

// f(std::integral_constant<int, n>{}) for the count n in [Lo, Hi] (the caller checked the range): one instantiation per
// count, so that every per-class sum lives in a named register (large counts spill, which is fine for a pass that is
// run once per step)
template <int Lo, typename F, int... I> static void with_count(int n, F&& f, std::integer_sequence<int, I...>) {
  (void)((n == Lo + I && (f(std::integral_constant<int, Lo + I>{}), true)) || ...);
}
template <int Lo, int Hi, typename F> static void with_count(int n, F&& f) {
  with_count<Lo>(n, f, std::make_integer_sequence<int, Hi - Lo + 1>{});
}

// label maps: f(classes, ignore label?) as compile-time constants, 2 <= C <= 32
template <typename F> static void with_classes(int C, int has_ignore, F&& f) {
  if (has_ignore)
    with_count<2, 32>(C, [&](auto c) { f(c, std::true_type{}); });
  else
    with_count<2, 32>(C, [&](auto c) { f(c, std::false_type{}); });
}

// argument checks of the label-map entry points: the buffers the call needs, then the sizes (the finalisation reads
// no target and passes target_kind 0)
static int dice_ce_args(const char* fn, std::initializer_list<const void*> bufs, int32_t target_kind, int32_t B,
                        int32_t C, int64_t plane) {
  for (const void* p : bufs)
    if (!p) return set_error(-1, "%s: null pointer", fn);
  if (B <= 0 || plane <= 0 || target_kind < 0 || target_kind > 3) return set_error(-1, "%s: bad argument", fn);
  if (C < 2 || C > 32) return set_error(-1, "dice_ce: %d classes not in [2, 32]", C);
  return 0;
}

extern "C" int64_t b2u_dice_ce_work_doubles(int32_t B, int32_t C, int64_t plane, int32_t has_ignore) {
  return work_doubles(B, plane, record_len(C, has_ignore));
}

extern "C" int b2u_dice_ce_stats(const float* logits, const void* target, int32_t target_kind, int32_t has_ignore,
                                 int32_t ignore_label, double* work, double* batch_sums, int32_t* bad_label, int32_t B,
                                 int32_t C, int64_t plane, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = dice_ce_args("b2u_dice_ce_stats", {logits, target, work, bad_label}, target_kind, B, C, plane)) return rc;
  const int nblk = stats_blocks(plane), K = record_len(C, has_ignore);
  with_classes(C, has_ignore, [&](auto c, auto ign) {
    loss_stats_kernel<decltype(c)::value, decltype(ign)::value><<<dim3(nblk, B), 256, 0, stream>>>(
        logits, target, target_kind, work, bad_label, plane, ignore_label);
  });
  if (int rc = check_launch("dice_ce_stats")) return rc;
  if (!batch_sums) return 0;
  dice_batch_sums_kernel<<<1, 256, 0, stream>>>(work, sample_records(work, B, plane, K), batch_sums, B, C, K, nblk);
  return check_launch("dice_ce_batch_sums");
}

extern "C" int b2u_dice_ce_finalize(double* work, const double* batch_sums, float* out3, int64_t* tp_fp_fn, int32_t B,
                                    int32_t C, int64_t plane, int32_t has_ignore, float weight_ce, float weight_dice,
                                    int32_t batch_dice, int32_t do_bg, float smooth, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = dice_ce_args("b2u_dice_ce_finalize", {work, out3}, 0, B, C, plane)) return rc;
  double* stats = sample_records(work, B, plane, record_len(C, has_ignore));
  auto* finalize = has_ignore ? loss_finalize_kernel<true> : loss_finalize_kernel<false>;
  finalize<<<1, 256, 0, stream>>>(work, stats, batch_sums, out3, tp_fp_fn, B, C, stats_blocks(plane), plane, weight_ce,
                                  weight_dice, batch_dice, do_bg, smooth);
  return check_launch("dice_ce_finalize");
}

extern "C" int b2u_dice_ce_backward(const float* logits, const void* target, int32_t target_kind, int32_t has_ignore,
                                    int32_t ignore_label, const double* work, const double* batch_sums,
                                    float* grad_logits, int32_t B, int32_t C, int64_t plane, float weight_ce,
                                    float weight_dice, int32_t batch_dice, int32_t do_bg, float smooth,
                                    const float* ce_scale, const float* dice_scale, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = dice_ce_args("b2u_dice_ce_backward", {logits, target, work, grad_logits}, target_kind, B, C, plane))
    return rc;
  const double* stats = sample_records(work, B, plane, record_len(C, has_ignore));
  with_classes(C, has_ignore, [&](auto c, auto ign) {
    loss_grad_kernel<decltype(c)::value, decltype(ign)::value><<<dim3(grad_blocks(plane), B), 256, 0, stream>>>(
        logits, target, target_kind, stats, batch_sums, grad_logits, B, plane, weight_ce, weight_dice, batch_dice,
        do_bg, smooth, 1.f, ce_scale, dice_scale, ignore_label);
  });
  return check_launch("dice_ce_backward");
}

// ---- regions (1 <= R <= 32: a single region is one sigmoid head).  The region kernels take the batch Dice from
// batch_sums only, so that buffer is required.
static int dice_bce_args(const char* fn, std::initializer_list<const void*> bufs, int32_t target_kind, int32_t B,
                         int32_t R, int64_t plane) {
  for (const void* p : bufs)
    if (!p) return set_error(-1, "%s: null pointer", fn);
  if (B <= 0 || plane <= 0 || target_kind < 0 || target_kind > 3) return set_error(-1, "%s: bad argument", fn);
  if (R < 1 || R > 32) return set_error(-1, "%s: %d regions not in [1, 32]", fn, R);
  return 0;
}

extern "C" int64_t b2u_dice_bce_work_doubles(int32_t B, int32_t R, int64_t plane) {
  return work_doubles(B, plane, region_record_len(R));
}

extern "C" int b2u_dice_bce_stats(const float* logits, const void* target, int32_t target_kind, int32_t has_ignore,
                                  double* work, double* batch_sums, int32_t B, int32_t R, int64_t plane,
                                  b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = dice_bce_args("b2u_dice_bce_stats", {logits, target, work, batch_sums}, target_kind, B, R, plane))
    return rc;
  const int nblk = stats_blocks(plane), K = region_record_len(R), ign = has_ignore ? 1 : 0;
  with_count<1, 32>(R, [&](auto r) {
    region_stats_kernel<decltype(r)::value><<<dim3(nblk, B), 256, 0, stream>>>(logits, target, target_kind, ign, work,
                                                                                plane);
  });
  if (int rc = check_launch("dice_bce_stats")) return rc;
  dice_batch_sums_kernel<<<1, 256, 0, stream>>>(work, sample_records(work, B, plane, K), batch_sums, B, R, K, nblk);
  return check_launch("dice_bce_batch_sums");
}

extern "C" int b2u_dice_bce_finalize(double* work, const double* batch_sums, float* out3, float* tp_fp_fn, int32_t B,
                                     int32_t R, int64_t plane, float weight_ce, float weight_dice, int32_t batch_dice,
                                     int32_t has_ignore, float smooth, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = dice_bce_args("b2u_dice_bce_finalize", {work, batch_sums, out3}, 0, B, R, plane)) return rc;
  double* stats = sample_records(work, B, plane, region_record_len(R));
  region_finalize_kernel<<<1, 256, 0, stream>>>(work, stats, batch_sums, out3, tp_fp_fn, B, R, stats_blocks(plane),
                                                plane, weight_ce, weight_dice, batch_dice, has_ignore ? 1 : 0, smooth);
  return check_launch("dice_bce_finalize");
}

extern "C" int b2u_dice_bce_backward(const float* logits, const void* target, int32_t target_kind, int32_t has_ignore,
                                     const double* work, const double* batch_sums, float* grad_logits, int32_t B,
                                     int32_t R, int64_t plane, float weight_ce, float weight_dice, int32_t batch_dice,
                                     float smooth, const float* ce_scale, const float* dice_scale,
                                     b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = dice_bce_args("b2u_dice_bce_backward",
                             {logits, target, work, batch_sums, grad_logits, ce_scale, dice_scale}, target_kind, B, R,
                             plane))
    return rc;
  const double* stats = sample_records(work, B, plane, region_record_len(R));
  const int ign = has_ignore ? 1 : 0;
  with_count<1, 32>(R, [&](auto r) {
    region_grad_kernel<decltype(r)::value><<<dim3(grad_blocks(plane), B), 256, 0, stream>>>(
        logits, target, target_kind, ign, stats, batch_sums, grad_logits, B, plane, weight_ce, weight_dice, batch_dice,
        smooth, ce_scale, dice_scale);
  });
  return check_launch("dice_bce_backward");
}

}  // namespace b2u
