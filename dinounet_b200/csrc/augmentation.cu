// nnU-Net's 2-D training augmentation on the device (reference: nnUNetTrainer.get_training_transforms,
// nnUNetTrainer.py:684-775, batchgenerators 0.25 transforms).  Every random decision comes from a per-plane record of
// B2U_AUG_REC doubles on the device (plane = sample * C + channel; sample-wide fields are repeated in every plane of
// the sample), written by dinounet_b200/augmentation.py.  Each step is one launch over the whole batch; a plane whose
// step did not fire returns at once, so the launch sequence does not depend on the record (capturable in a graph).
//
//   spatial   augment_spatial without elastic deformation: coordinates c = ((i - (H-1)/2, j - (W-1)/2) rotated by
//             (c0 cos + c1 sin, c1 cos - c0 sin), times the scale) + (h/2 - 0.5, w/2 - 0.5).  Data: scipy
//             map_coordinates(order 3, mode 'constant', cval 0) in fp64: the spline prefilter with mirror boundaries
//             along axis 0 then 1 (only planes that are transformed), then cval outside [0, n-1] and otherwise 16
//             mirrored taps.  Seg: interpolate_img(is_seg, order 1, cval -1) in one pass: the bilinear weights of the
//             four taps summed per label in tap order; the largest label with a sum >= 0.5 wins, 0 if none (or outside).
//             Untransformed samples: the centre crop at ((h-H)//2, (w-W)//2).
//   noise     x = f32(f64(x) + std * n), n standard normal from Philox4x32-10 keyed by (seed, sample, channel, pixel).
//   blur      scipy gaussian_filter (reflect, truncate 4): symmetric correlation in fp64 along axis 0 then 1, f32 between.
//   brightness, contrast, gamma (twice; the first on the negated sample): float32 as numpy computes them with weak
//             python scalars; mean / std are numpy's pairwise float32 reductions (preprocess.cu's tree, batched).
//   low-res   skimage resize order 0 down to (th, tw), then order 3 (mode 'edge') back up, clipped to the downsampled
//             plane's range: the gather, scipy's edge padding and reflect-boundary prefilter, and the zoom's 16 taps.
//   finalize  mirror, mask (channels with use_mask_for_norm: 0 where seg < 0), remove label -1 -> 0, and either the
//             label map or the region channels, written as float32.
#include <algorithm>

#include "../../include/dinounet_b200.h"
#include "common.cuh"
#include "gemm_common.h"
#include "host_util.h"
#include "spline.cuh"

namespace b2u {
namespace {

// record fields (doubles per plane); keep in sync with dinounet_b200/augmentation.py
enum : int {
  kSpatial = 0, kRot, kCos, kSin, kScaleOn, kScale, kNoise, kNoiseStd, kBlurR, kBlurW,  // kBlurW: 5 weights, centre first
  kBright = 14, kBrightM, kContrast, kContrastF, kLowH, kLowW, kLowY /* 5 consts */, kLowX = 25 /* 5 consts */,
  kGamInvOn = 30, kGamInv, kGamOn, kGam, kFlip0, kFlip1, kMask, kRec = B2U_AUG_REC
};
static_assert(kMask < kRec, "record too short");

constexpr int kT = 256;

__device__ __forceinline__ const double* rec_of(const double* rec, long long plane) { return rec + plane * kRec; }

__device__ __forceinline__ int mirror_idx(int i, int n) {
  if (n <= 1) return 0;
  const int s2 = 2 * n - 2;
  if (i < 0) {
    i = s2 * (-i / s2) + i;
    return i <= 1 - n ? i + s2 : -i;
  }
  if (i >= n) {
    i -= s2 * (i / s2);
    if (i >= n) i = s2 - i;
  }
  return i;
}

__device__ __forceinline__ int reflect_idx(int i, int n) {
  while (i < 0 || i >= n) i = i < 0 ? -i - 1 : 2 * n - i - 1;
  return i;
}

struct Coords {
  double c0, c1;
};

__device__ __forceinline__ Coords spatial_coords(const double* r, int i, int j, int h, int w, int H, int W) {
  double c0 = __dsub_rn(static_cast<double>(i), (H - 1) / 2.0), c1 = __dsub_rn(static_cast<double>(j), (W - 1) / 2.0);
  if (r[kRot] != 0.0) {
    const double cs = r[kCos], sn = r[kSin];
    const double n0 = __dadd_rn(__dmul_rn(c0, cs), __dmul_rn(c1, sn));
    const double n1 = __dsub_rn(__dmul_rn(c1, cs), __dmul_rn(c0, sn));
    c0 = n0;
    c1 = n1;
  }
  if (r[kScaleOn] != 0.0) {
    c0 = __dmul_rn(c0, r[kScale]);
    c1 = __dmul_rn(c1, r[kScale]);
  }
  return {__dadd_rn(c0, __dsub_rn(h / 2.0, 0.5)), __dadd_rn(c1, __dsub_rn(w / 2.0, 0.5))};
}

// ---- spatial ------------------------------------------------------------------------------------------------------

// axis 0: one thread per (plane, column), copying the plane to fp64 first; axis 1: one thread per (plane, row).
__global__ void __launch_bounds__(128) spatial_prefilter_kernel(const float* __restrict__ x, int P, int C, int h, int w,
                                                                const double* __restrict__ rec, int axis,
                                                                FilterConsts k, double* __restrict__ coef) {
  const int per = axis == 0 ? w : h;
  const long long l = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (l >= static_cast<long long>(P) * per) return;
  const long long p = l / per;
  const int q = static_cast<int>(l % per);
  if (rec_of(rec, p)[kSpatial] == 0.0) return;
  const long long plane = static_cast<long long>(h) * w;
  double* c = coef + p * plane;
  if (axis == 0) {
    const float* xs = x + p * plane;
    for (int i = 0; i < h; ++i) c[static_cast<long long>(i) * w + q] = static_cast<double>(xs[static_cast<long long>(i) * w + q]);
    spline_filter_line<true>(c + q, w, h, k);
  } else {
    spline_filter_line<true>(c + static_cast<long long>(q) * w, 1, w, k);
  }
}

__global__ void __launch_bounds__(kT) spatial_data_kernel(const float* __restrict__ x, const double* __restrict__ coef,
                                                          int P, int h, int w, int H, int W,
                                                          const double* __restrict__ rec, float* __restrict__ out) {
  const long long n = static_cast<long long>(P) * H * W;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < n; e += stride) {
    const int j = static_cast<int>(e % W);
    const int i = static_cast<int>((e / W) % H);
    const long long p = e / (static_cast<long long>(H) * W);
    const double* r = rec_of(rec, p);
    const long long plane = static_cast<long long>(h) * w;
    if (r[kSpatial] == 0.0) {
      out[e] = x[p * plane + static_cast<long long>(i + (h - H) / 2) * w + j + (w - W) / 2];
      continue;
    }
    const Coords cc = spatial_coords(r, i, j, h, w, H, W);
    double t = 0.0;  // cval
    if (cc.c0 >= 0.0 && cc.c0 <= h - 1.0 && cc.c1 >= 0.0 && cc.c1 <= w - 1.0) {
      const Taps3 ty = cubic_taps_at(cc.c0), tx = cubic_taps_at(cc.c1);
      const double* c = coef + p * plane;
      int xi[4];
#pragma unroll
      for (int b = 0; b < 4; ++b) xi[b] = mirror_idx(tx.start + b, w);
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        const double* row = c + static_cast<long long>(mirror_idx(ty.start + a, h)) * w;
#pragma unroll
        for (int b = 0; b < 4; ++b) t = __dadd_rn(t, __dmul_rn(__dmul_rn(row[xi[b]], ty.w[a]), tx.w[b]));
      }
    }
    out[e] = __double2float_rn(t);
  }
}

// seg [B, h, w] int16 -> labels [B, H, W] int32 (before the removal of -1).
__global__ void __launch_bounds__(kT) spatial_seg_kernel(const int16_t* __restrict__ seg, int B, int C, int h, int w,
                                                         int H, int W, const double* __restrict__ rec,
                                                         int32_t* __restrict__ out) {
  const long long n = static_cast<long long>(B) * H * W;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < n; e += stride) {
    const int j = static_cast<int>(e % W);
    const int i = static_cast<int>((e / W) % H);
    const long long b = e / (static_cast<long long>(H) * W);
    const double* r = rec_of(rec, b * C);
    const int16_t* s = seg + b * h * static_cast<long long>(w);
    if (r[kSpatial] == 0.0) {
      out[e] = s[static_cast<long long>(i + (h - H) / 2) * w + j + (w - W) / 2];
      continue;
    }
    const Coords cc = spatial_coords(r, i, j, h, w, H, W);
    int result = 0;
    if (cc.c0 >= 0.0 && cc.c0 <= h - 1.0 && cc.c1 >= 0.0 && cc.c1 <= w - 1.0) {
      const double f0 = floor(cc.c0), f1 = floor(cc.c1);
      const double wy0 = __dsub_rn(1.0, __dsub_rn(cc.c0, f0)), wx0 = __dsub_rn(1.0, __dsub_rn(cc.c1, f1));
      const double wy[2] = {wy0, __dsub_rn(1.0, wy0)}, wx[2] = {wx0, __dsub_rn(1.0, wx0)};
      int lab[4];
      double wt[4];
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        const int yi = mirror_idx(static_cast<int>(f0) + a, h);
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          lab[a * 2 + q] = s[static_cast<long long>(yi) * w + mirror_idx(static_cast<int>(f1) + q, w)];
          wt[a * 2 + q] = __dmul_rn(wy[a], wx[q]);
        }
      }
      bool found = false;
#pragma unroll
      for (int t = 0; t < 4; ++t) {  // each distinct label: its weights summed in tap order, as its own map would
        double sum = 0.0;
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (lab[u] == lab[t]) sum = __dadd_rn(sum, wt[u]);
        if (sum >= 0.5 && (!found || lab[t] > result)) {
          result = lab[t];
          found = true;
        }
      }
    }
    out[e] = result;
  }
}

// ---- noise --------------------------------------------------------------------------------------------------------

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const unsigned hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const unsigned hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}

// Standard normal of pixel e of plane (b, c): Box-Muller on two 53-bit uniforms in (0, 1) from one Philox block per
// pixel pair.
__device__ __forceinline__ double philox_normal(unsigned long long seed, int b, int c, long long e) {
  const uint4 r = philox4x32_10(make_uint4(static_cast<unsigned>(e >> 1), static_cast<unsigned>(e >> 33),
                                           static_cast<unsigned>(c), static_cast<unsigned>(b)),
                                make_uint2(static_cast<unsigned>(seed), static_cast<unsigned>(seed >> 32)));
  const double u1 = ((r.x >> 5) * 67108864.0 + (r.y >> 6) + 0.5) * 0x1p-53;
  const double u2 = ((r.z >> 5) * 67108864.0 + (r.w >> 6) + 0.5) * 0x1p-53;
  const double rad = sqrt(-2.0 * log(u1));
  double s, co;
  sincospi(2.0 * u2, &s, &co);
  return (e & 1) ? rad * s : rad * co;
}

__global__ void __launch_bounds__(kT) noise_field_kernel(unsigned long long seed, int B, int C, long long n,
                                                         double* __restrict__ out) {
  const long long total = static_cast<long long>(B) * C * n;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total; e += stride) {
    const long long p = e / n;
    out[e] = philox_normal(seed, static_cast<int>(p / C), static_cast<int>(p % C), e % n);
  }
}

__global__ void __launch_bounds__(kT) noise_kernel(float* __restrict__ x, int P, int C, long long n,
                                                   unsigned long long seed, const double* __restrict__ rec) {
  const long long total = static_cast<long long>(P) * n;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total; e += stride) {
    const long long p = e / n;
    const double* r = rec_of(rec, p);
    if (r[kNoise] == 0.0) continue;
    const double z = philox_normal(seed, static_cast<int>(p / C), static_cast<int>(p % C), e % n);
    x[e] = __double2float_rn(__dadd_rn(static_cast<double>(x[e]), __dmul_rn(r[kNoiseStd], z)));
  }
}

// ---- blur ---------------------------------------------------------------------------------------------------------

// NI_Correlate1D's symmetric branch: x[i] w0 + sum_{k = r .. 1} (x[i-k] + x[i+k]) w_k, reflect boundaries.
__global__ void __launch_bounds__(kT) blur_kernel(const float* __restrict__ in, float* __restrict__ out, int P, int H,
                                                  int W, int axis, const double* __restrict__ rec) {
  const long long n = static_cast<long long>(P) * H * W;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < n; e += stride) {
    const long long p = e / (static_cast<long long>(H) * W);
    const double* r = rec_of(rec, p);
    const int rad = static_cast<int>(r[kBlurR]);
    if (rad == 0) continue;
    const int j = static_cast<int>(e % W), i = static_cast<int>((e / W) % H);
    const float* pl = in + p * H * static_cast<long long>(W);
    const int pos = axis == 0 ? i : j, len = axis == 0 ? H : W;
    auto at = [&](int q) {
      q = reflect_idx(q, len);
      return static_cast<double>(axis == 0 ? pl[static_cast<long long>(q) * W + j] : pl[static_cast<long long>(i) * W + q]);
    };
    double t = __dmul_rn(at(pos), r[kBlurW]);
    for (int k = rad; k >= 1; --k) t = __dadd_rn(t, __dmul_rn(__dadd_rn(at(pos - k), at(pos + k)), r[kBlurW + k]));
    out[e] = __double2float_rn(t);
  }
}

// ---- intensity ----------------------------------------------------------------------------------------------------

enum : int { kOpBright = 0, kOpContrast, kOpNegate, kOpGamma, kOpRetain };

// stats: [4, P] floats: mean, std, min, max.  gamma_idx: kGamInvOn or kGamOn (which gamma the op belongs to).
__global__ void __launch_bounds__(kT) pointwise_kernel(float* __restrict__ x, int P, long long n, int op, int gamma_idx,
                                                       const double* __restrict__ rec, const float* __restrict__ st0,
                                                       const float* __restrict__ st1) {
  const long long total = static_cast<long long>(P) * n;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total; e += stride) {
    const long long p = e / n;
    const double* r = rec_of(rec, p);
    float v = x[e];
    if (op == kOpBright) {
      if (r[kBright] == 0.0) continue;
      v = __fmul_rn(v, static_cast<float>(r[kBrightM]));
    } else if (op == kOpContrast) {
      if (r[kContrast] == 0.0) continue;
      const float mn = st0[p], lo = st0[2 * P + p], hi = st0[3 * P + p];
      v = __fadd_rn(__fmul_rn(__fsub_rn(v, mn), static_cast<float>(r[kContrastF])), mn);
      v = v < lo ? lo : v;
      v = v > hi ? hi : v;
    } else if (op == kOpNegate) {
      if (r[kGamInvOn] == 0.0) continue;
      v = -v;
    } else if (op == kOpGamma) {
      if (r[gamma_idx] == 0.0) continue;
      const float minm = st0[2 * P + p], rng = __fadd_rn(__fsub_rn(st0[3 * P + p], minm), 1e-7f);
      v = __fadd_rn(__fmul_rn(powf(__fdiv_rn(__fsub_rn(v, minm), rng), static_cast<float>(r[gamma_idx + 1])), rng),
                    minm);
    } else {  // kOpRetain: st0 = stats before the power, st1 = after
      if (r[gamma_idx] == 0.0) continue;
      v = __fsub_rn(v, st1[p]);
      v = __fmul_rn(__fdiv_rn(v, __fadd_rn(st1[P + p], 1e-8f)), st0[P + p]);
      v = __fadd_rn(v, st0[p]);
    }
    x[e] = v;
  }
}

// numpy's mean / std from the pairwise sums in work[p * ws]: f32(f64(sum) / n); std = sqrtf of that for squares.
__global__ void stats_finalize_kernel(const float* __restrict__ work, long long ws, int P, long long n, int stage,
                                      float* __restrict__ st) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const float q = __double2float_rn(__ddiv_rn(static_cast<double>(work[p * ws]), static_cast<double>(n)));
  st[stage * P + p] = stage == 0 ? q : __fsqrt_rn(q);
}

// ---- low-resolution simulation ------------------------------------------------------------------------------------

// The order-0 downsample of plane p to (th, tw), edge-padded by 12 into a [th + 24, tw + 24] fp64 plane at pitch
// (tw + 24), plane stride ps.
__global__ void __launch_bounds__(kT) lowres_pad_kernel(const float* __restrict__ x, int P, int H, int W,
                                                        const double* __restrict__ rec, long long ps,
                                                        double* __restrict__ coef) {
  const long long per = static_cast<long long>(H + 2 * kPad) * (W + 2 * kPad);
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < P * per; e += stride) {
    const long long p = e / per;
    const double* r = rec_of(rec, p);
    const int th = static_cast<int>(r[kLowH]), tw = static_cast<int>(r[kLowW]);
    if (th == 0) continue;
    const int Wp = tw + 2 * kPad;
    const long long q = e % per;
    const int yp = static_cast<int>(q / Wp), xp = static_cast<int>(q % Wp);
    if (yp >= th + 2 * kPad) continue;
    const int yi = min(max(yp - kPad, 0), th - 1), xi = min(max(xp - kPad, 0), tw - 1);
    const double zy = static_cast<double>(H) / th, zx = static_cast<double>(W) / tw;
    const int sy = min(max(static_cast<int>(floor(__dadd_rn(__dsub_rn(__dmul_rn(yi + 0.5, zy), 0.5), 0.5))), 0), H - 1);
    const int sx = min(max(static_cast<int>(floor(__dadd_rn(__dsub_rn(__dmul_rn(xi + 0.5, zx), 0.5), 0.5))), 0), W - 1);
    coef[p * ps + q] = static_cast<double>(x[(p * H + sy) * W + sx]);
  }
}

// One block per plane: min / max of its padded plane (the downsampled values) into lohi[2p], lohi[2p + 1].
__global__ void __launch_bounds__(kT) lowres_minmax_kernel(const double* __restrict__ coef, long long ps,
                                                           const double* __restrict__ rec, double* __restrict__ lohi) {
  const long long p = blockIdx.x;
  const double* r = rec_of(rec, p);
  const int th = static_cast<int>(r[kLowH]), tw = static_cast<int>(r[kLowW]);
  if (th == 0) return;
  const long long m = static_cast<long long>(th + 2 * kPad) * (tw + 2 * kPad);
  const double* c = coef + p * ps;
  double lo = c[0], hi = c[0];
  for (long long i = threadIdx.x; i < m; i += blockDim.x) {
    lo = fmin(lo, c[i]);
    hi = fmax(hi, c[i]);
  }
  __shared__ double slo[kT], shi[kT];
  slo[threadIdx.x] = lo;
  shi[threadIdx.x] = hi;
  __syncthreads();
  for (int s = kT / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      slo[threadIdx.x] = fmin(slo[threadIdx.x], slo[threadIdx.x + s]);
      shi[threadIdx.x] = fmax(shi[threadIdx.x], shi[threadIdx.x + s]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    lohi[2 * p] = slo[0];
    lohi[2 * p + 1] = shi[0];
  }
}

// axis 0: one thread per (plane, padded column); axis 1: per (plane, padded row); reflect boundaries, the plane's consts.
__global__ void __launch_bounds__(128) lowres_filter_kernel(double* __restrict__ coef, int P, int H, int W, long long ps,
                                                            int axis, const double* __restrict__ rec) {
  const int per = axis == 0 ? W + 2 * kPad : H + 2 * kPad;
  const long long l = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (l >= static_cast<long long>(P) * per) return;
  const long long p = l / per;
  const int q = static_cast<int>(l % per);
  const double* r = rec_of(rec, p);
  const int th = static_cast<int>(r[kLowH]), tw = static_cast<int>(r[kLowW]);
  if (th == 0) return;
  const int Hp = th + 2 * kPad, Wp = tw + 2 * kPad;
  const double* kc = r + (axis == 0 ? kLowY : kLowX);
  const FilterConsts k{kc[0], kc[1], kc[2], kc[3], kc[4]};
  if (axis == 0) {
    if (q < Wp) spline_filter_line<false>(coef + p * ps + q, Wp, Hp, k);
  } else {
    if (q < Hp) spline_filter_line<false>(coef + p * ps + static_cast<long long>(q) * Wp, 1, Wp, k);
  }
}

__global__ void __launch_bounds__(kT) lowres_zoom_kernel(const double* __restrict__ coef, int P, int H, int W,
                                                         long long ps, const double* __restrict__ rec,
                                                         const double* __restrict__ lohi, float* __restrict__ x) {
  const long long n = static_cast<long long>(P) * H * W;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < n; e += stride) {
    const long long p = e / (static_cast<long long>(H) * W);
    const double* r = rec_of(rec, p);
    const int th = static_cast<int>(r[kLowH]), tw = static_cast<int>(r[kLowW]);
    if (th == 0) continue;
    const int j = static_cast<int>(e % W), i = static_cast<int>((e / W) % H);
    const Taps3 ty = cubic_taps(i, static_cast<double>(th) / H), tx = cubic_taps(j, static_cast<double>(tw) / W);
    double t = cubic16(coef + p * ps, tw + 2 * kPad, ty, tx);
    t = fmin(fmax(t, lohi[2 * p]), lohi[2 * p + 1]);
    x[e] = __double2float_rn(t);
  }
}

// ---- finalize -----------------------------------------------------------------------------------------------------

// One thread per output pixel of a sample: mirror, mask, remove label -1, target.  regions: HOST-built device int32
// [R + 1 offsets, labels...]; R == 0 writes the label map.
__global__ void __launch_bounds__(kT) finalize_kernel(const float* __restrict__ x, const int32_t* __restrict__ seg,
                                                      int B, int C, int H, int W, const double* __restrict__ rec,
                                                      const int32_t* __restrict__ regions, int R,
                                                      float* __restrict__ out, float* __restrict__ target) {
  const long long hw = static_cast<long long>(H) * W, n = B * hw;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < n; e += stride) {
    const long long b = e / hw;
    const int j = static_cast<int>(e % W), i = static_cast<int>((e / W) % H);
    const double* r = rec_of(rec, b * C);
    const int si = r[kFlip0] != 0.0 ? H - 1 - i : i, sj = r[kFlip1] != 0.0 ? W - 1 - j : j;
    const long long src = static_cast<long long>(si) * W + sj, dst = static_cast<long long>(i) * W + j;
    int s = seg[b * hw + src];
    for (int c = 0; c < C; ++c) {
      const float v = x[(b * C + c) * hw + src];
      out[(b * C + c) * hw + dst] = (s < 0 && rec_of(rec, b * C + c)[kMask] != 0.0) ? 0.f : v;
    }
    if (s == -1) s = 0;
    if (R == 0) {
      target[b * hw + dst] = static_cast<float>(s);
    } else {
      for (int q = 0; q < R; ++q) {
        float v = 0.f;
        for (int k = regions[q]; k < regions[q + 1]; ++k) v = regions[R + 1 + k] == s ? 1.f : v;
        target[(b * R + q) * hw + dst] = v;
      }
    }
  }
}

int grid_for(long long n, int threads) {
  return static_cast<int>(std::max<long long>(1, std::min<long long>((n + threads - 1) / threads,
                                                                    static_cast<long long>(num_sms()) * 16)));
}

struct Work {
  double* coef;   // spatial prefilter [P, h, w], then the low-res planes [P, (H + 24) (W + 24)]
  float* x;       // [P, H, W]
  float* tmp;     // [P, H, W] (blur's axis-0 result)
  int32_t* seg;   // [B, H, W]
  float* st0;     // [4, P]
  float* st1;     // [4, P]
  float* tree;    // [P, ceil(H W / 8)]
  double* lohi;   // [2 P]
  long long tree_ws;
};

// Byte offsets of the Work buffers (each 256-aligned); the last entry is the total.
void layout(int B, int C, int h, int w, int H, int W, long long off[9]) {
  const long long P = static_cast<long long>(B) * C, hw = static_cast<long long>(H) * W;
  const long long coef = std::max(static_cast<long long>(h) * w, static_cast<long long>(H + 2 * kPad) * (W + 2 * kPad));
  const long long bytes[8] = {P * coef * 8, 2 * P * 8, P * hw * 4, P * hw * 4, B * hw * 4, 4 * P * 4, 4 * P * 4,
                              P * ((hw + 7) / 8) * 4};
  off[0] = 0;
  for (int i = 0; i < 8; ++i) off[i + 1] = off[i] + (bytes[i] + 255) / 256 * 256;
}

Work carve(void* base, int B, int C, int h, int w, int H, int W) {
  long long off[9];
  layout(B, C, h, w, H, W, off);
  char* p = static_cast<char*>(base);
  Work k;
  k.coef = reinterpret_cast<double*>(p + off[0]);
  k.lohi = reinterpret_cast<double*>(p + off[1]);
  k.x = reinterpret_cast<float*>(p + off[2]);
  k.tmp = reinterpret_cast<float*>(p + off[3]);
  k.seg = reinterpret_cast<int32_t*>(p + off[4]);
  k.st0 = reinterpret_cast<float*>(p + off[5]);
  k.st1 = reinterpret_cast<float*>(p + off[6]);
  k.tree = reinterpret_cast<float*>(p + off[7]);
  k.tree_ws = (static_cast<long long>(H) * W + 7) / 8;
  return k;
}

// mean (stage 0) and std (stage 1) of every plane into st[0..P), st[P..2P); min / max into st[2P..4P).
int plane_stats(const float* x, int P, long long n, bool with_std, const Work& k, float* st, cudaStream_t stream) {
  int rc = pairwise_sum_planes_f32(x, n, P, 0, nullptr, k.tree, k.tree_ws, stream);
  if (rc) return rc;
  stats_finalize_kernel<<<(P + 127) / 128, 128, 0, stream>>>(k.tree, k.tree_ws, P, n, 0, st);
  if ((rc = check_launch("aug_stats"))) return rc;
  if (with_std) {
    if ((rc = pairwise_sum_planes_f32(x, n, P, 1, st, k.tree, k.tree_ws, stream))) return rc;
    stats_finalize_kernel<<<(P + 127) / 128, 128, 0, stream>>>(k.tree, k.tree_ws, P, n, 1, st);
    if ((rc = check_launch("aug_stats"))) return rc;
  }
  return minmax_planes_f32(x, n, P, st + 2 * P, st + 3 * P, stream);
}

}  // namespace
}  // namespace b2u

using namespace b2u;

extern "C" int64_t b2u_aug_work_bytes(int32_t B, int32_t C, int32_t h, int32_t w, int32_t H, int32_t W) {
  long long off[9];
  layout(B, C, h, w, H, W, off);
  return off[8];
}

extern "C" int b2u_aug_noise_field(uint64_t seed, int32_t B, int32_t C, int64_t n, double* out, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!out) return set_error(-1, "b2u_aug_noise_field: null pointer");
  if (B <= 0 || C <= 0 || n <= 0) return set_error(-1, "b2u_aug_noise_field: B=%d C=%d n=%lld", B, C,
                                                   static_cast<long long>(n));
  const long long total = static_cast<long long>(B) * C * n;
  noise_field_kernel<<<grid_for(total, kT), kT, 0, stream>>>(seed, B, C, n, out);
  return check_launch("aug_noise_field");
}

extern "C" int b2u_aug_apply(const float* data, const int16_t* seg, int32_t B, int32_t C, int32_t h, int32_t w,
                             int32_t H, int32_t W, const double* rec, const double* consts, uint64_t seed, const int32_t* regions, int32_t R,
                             void* work, float* out, float* target, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!data || !seg || !rec || !consts || !work || !out || !target || (R > 0 && !regions))
    return set_error(-1, "b2u_aug_apply: null pointer");
  if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || h < H || w < W || static_cast<long long>(B) * C > 65535 || R < 0)
    return set_error(-1, "b2u_aug_apply: bad shape B=%d C=%d %dx%d -> %dx%d R=%d", B, C, h, w, H, W, R);
  const int P = B * C;
  const long long hw = static_cast<long long>(H) * W;
  const Work k = carve(work, B, C, h, w, H, W);
  int rc;
  // spatial
  const FilterConsts ky{consts[0], consts[1], consts[3], 0.0, consts[4]}, kx{consts[0], consts[2], consts[3], 0.0, consts[4]};
  spatial_prefilter_kernel<<<static_cast<unsigned>((static_cast<long long>(P) * w + 127) / 128), 128, 0, stream>>>(
      data, P, C, h, w, rec, 0, ky, k.coef);
  if ((rc = check_launch("aug_spatial_prefilter"))) return rc;
  spatial_prefilter_kernel<<<static_cast<unsigned>((static_cast<long long>(P) * h + 127) / 128), 128, 0, stream>>>(
      data, P, C, h, w, rec, 1, kx, k.coef);
  if ((rc = check_launch("aug_spatial_prefilter"))) return rc;
  spatial_data_kernel<<<grid_for(P * hw, kT), kT, 0, stream>>>(data, k.coef, P, h, w, H, W, rec, k.x);
  if ((rc = check_launch("aug_spatial_data"))) return rc;
  spatial_seg_kernel<<<grid_for(B * hw, kT), kT, 0, stream>>>(seg, B, C, h, w, H, W, rec, k.seg);
  if ((rc = check_launch("aug_spatial_seg"))) return rc;
  // noise, blur, brightness
  noise_kernel<<<grid_for(P * hw, kT), kT, 0, stream>>>(k.x, P, C, hw, seed, rec);
  if ((rc = check_launch("aug_noise"))) return rc;
  blur_kernel<<<grid_for(P * hw, kT), kT, 0, stream>>>(k.x, k.tmp, P, H, W, 0, rec);
  if ((rc = check_launch("aug_blur"))) return rc;
  blur_kernel<<<grid_for(P * hw, kT), kT, 0, stream>>>(k.tmp, k.x, P, H, W, 1, rec);
  if ((rc = check_launch("aug_blur"))) return rc;
  pointwise_kernel<<<grid_for(P * hw, kT), kT, 0, stream>>>(k.x, P, hw, kOpBright, 0, rec, nullptr, nullptr);
  if ((rc = check_launch("aug_brightness"))) return rc;
  // contrast
  if ((rc = plane_stats(k.x, P, hw, false, k, k.st0, stream))) return rc;
  pointwise_kernel<<<grid_for(P * hw, kT), kT, 0, stream>>>(k.x, P, hw, kOpContrast, 0, rec, k.st0, nullptr);
  if ((rc = check_launch("aug_contrast"))) return rc;
  // low resolution
  const long long ps = static_cast<long long>(H + 2 * kPad) * (W + 2 * kPad);
  lowres_pad_kernel<<<grid_for(P * ps, kT), kT, 0, stream>>>(k.x, P, H, W, rec, ps, k.coef);
  if ((rc = check_launch("aug_lowres_pad"))) return rc;
  lowres_minmax_kernel<<<P, kT, 0, stream>>>(k.coef, ps, rec, k.lohi);
  if ((rc = check_launch("aug_lowres_minmax"))) return rc;
  for (int axis = 0; axis < 2; ++axis) {
    const long long lines = static_cast<long long>(P) * (axis == 0 ? W + 2 * kPad : H + 2 * kPad);
    lowres_filter_kernel<<<static_cast<unsigned>((lines + 127) / 128), 128, 0, stream>>>(k.coef, P, H, W, ps, axis, rec);
    if ((rc = check_launch("aug_lowres_filter"))) return rc;
  }
  lowres_zoom_kernel<<<grid_for(P * hw, kT), kT, 0, stream>>>(k.coef, P, H, W, ps, rec, k.lohi, k.x);
  if ((rc = check_launch("aug_lowres_zoom"))) return rc;
  // gamma on the negated samples, then gamma
  for (int g = 0; g < 2; ++g) {
    const int idx = g == 0 ? kGamInvOn : kGamOn;
    if (g == 0) {
      pointwise_kernel<<<grid_for(P * hw, kT), kT, 0, stream>>>(k.x, P, hw, kOpNegate, idx, rec, nullptr, nullptr);
      if ((rc = check_launch("aug_gamma_negate"))) return rc;
    }
    if ((rc = plane_stats(k.x, P, hw, true, k, k.st0, stream))) return rc;
    pointwise_kernel<<<grid_for(P * hw, kT), kT, 0, stream>>>(k.x, P, hw, kOpGamma, idx, rec, k.st0, nullptr);
    if ((rc = check_launch("aug_gamma"))) return rc;
    if ((rc = plane_stats(k.x, P, hw, true, k, k.st1, stream))) return rc;
    pointwise_kernel<<<grid_for(P * hw, kT), kT, 0, stream>>>(k.x, P, hw, kOpRetain, idx, rec, k.st0, k.st1);
    if ((rc = check_launch("aug_gamma_retain"))) return rc;
    if (g == 0) {
      pointwise_kernel<<<grid_for(P * hw, kT), kT, 0, stream>>>(k.x, P, hw, kOpNegate, idx, rec, nullptr, nullptr);
      if ((rc = check_launch("aug_gamma_negate"))) return rc;
    }
  }
  finalize_kernel<<<grid_for(B * hw, kT), kT, 0, stream>>>(k.x, k.seg, B, C, H, W, rec, regions, R, out, target);
  return check_launch("aug_finalize");
}
