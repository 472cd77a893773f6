// Backward kernels of the trainable part of Dino U-Net (everything outside the frozen DINOv3 backbone:
// dinov3_adapter.py:326,422-426) + the fused SGD step - SURVEY.md section 8f rank 2 / BASELINE.json config 3.
// fp32, token-major / NHWC like the fp32 tier whose forward kernels (fp32_tier.cu) they differentiate; the matrix
// products of the backward (data and weight gradients of every Linear / 1x1 / 3x3 / transposed conv) run through
// b2u_f32_gemm's transposed / conv-dgrad / split-K modes.  What the reference executes here is ATen autograd + the one
// native op ms_deform_attn_backward (already replaced by b2u_msda_backward_f32, msda.cu); nnUNetTrainer.py:899-929.
// Reductions into parameter gradients use fp32 atomics (sum order varies run to run at the 1e-7 level, like the
// reference's cuDNN / cuBLAS backward).  Gradient buffers must be zero-initialised by the caller.
#include <math.h>

#include "common.cuh"
#include "../../include/dinounet_b200.h"
#include "host_util.h"

namespace b2u {

__device__ __forceinline__ float act_grad(float x, int act) {   // d act(x) / dx from the PRE-activation value
  if (act == B2U_ACT_GELU) {
    const float c = 0.70710678118654752440f;
    return 0.5f * (1.0f + erff(x * c)) + x * 0.3989422804014327f * expf(-0.5f * x * x);
  }
  if (act == B2U_ACT_RELU) return x > 0.f ? 1.f : 0.f;
  if (act == B2U_ACT_LRELU) return x > 0.f ? 1.f : 0.01f;
  return 1.f;
}

static inline unsigned blocks_for(long long n, int t = 256) { return static_cast<unsigned>((n + t - 1) / t); }

// ---------------------------------------------------------------------------------------- elementwise
__global__ void f32_act_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx, long long n, int act) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) dx[i] = dy[i] * act_grad(x[i], act);
}
extern "C" int b2u_f32_act_bwd(const float* x, const float* dy, float* dx, int64_t n, int32_t act, b2u_stream_t s) {
  f32_act_bwd_kernel<<<blocks_for(n), 256, 0, static_cast<cudaStream_t>(s)>>>(x, dy, dx, n, act);
  return check_launch("f32_act_bwd");
}

__global__ void f32_act_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, int act) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = x[i];
  float r = v;
  if (act == B2U_ACT_GELU) r = 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f));
  else if (act == B2U_ACT_RELU) r = fmaxf(v, 0.f);
  else if (act == B2U_ACT_LRELU) r = v > 0.f ? v : 0.01f * v;
  y[i] = r;
}
extern "C" int b2u_f32_act(const float* x, float* y, int64_t n, int32_t act, b2u_stream_t s) {
  f32_act_kernel<<<blocks_for(n), 256, 0, static_cast<cudaStream_t>(s)>>>(x, y, n, act);
  return check_launch("f32_act");
}

__global__ void f32_add_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, long long n) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) out[i] = a[i] + b[i];
}
extern "C" int b2u_f32_add(const float* a, const float* b, float* out, int64_t n, b2u_stream_t s) {
  f32_add_kernel<<<blocks_for(n), 256, 0, static_cast<cudaStream_t>(s)>>>(a, b, out, n);
  return check_launch("f32_add");
}

// out[c] += sum_r in[r*ld + c]      (bias gradients; grid (C/32, splits), block 32 x 8)
__global__ void __launch_bounds__(256) f32_colsum_kernel(const float* __restrict__ in, long long ld, long long rows, int Cc, float* __restrict__ out) {
  __shared__ float red[8][33];
  const int cx = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  const long long per = (rows + gridDim.y - 1) / gridDim.y;
  const long long lo = blockIdx.y * per, hi = lo + per < rows ? lo + per : rows;
  float s = 0.f;
  if (c < Cc)
    for (long long r = lo + rg; r < hi; r += 8) s += in[r * ld + c];
  red[rg][cx] = s;
  __syncthreads();
  if (rg == 0 && c < Cc) {
    float t = 0.f;
    for (int k = 0; k < 8; ++k) t += red[k][cx];
    atomicAdd(&out[c], t);
  }
}
extern "C" int b2u_f32_colsum(const float* in, int64_t ld, int64_t rows, int32_t Cc, float* out, b2u_stream_t s) {
  const int splits = static_cast<int>(rows > 65536 ? 64 : (rows > 2048 ? 8 : 1));
  f32_colsum_kernel<<<dim3((Cc + 31) / 32, splits), 256, 0, static_cast<cudaStream_t>(s)>>>(in, ld, rows, Cc, out);
  return check_launch("f32_colsum");
}

// ---------------------------------------------------------------------------------------- LayerNorm backward
// one warp per row (grid-stride); dx = rstd * (g - mean(g) - xhat * mean(g * xhat)), g = dy * w;  dw += dy * xhat, db += dy.
// blockIdx.y picks a chunk of LN_BWD_COLS columns: the row statistics cover the whole row, dx and the dw / db partials
// this chunk only (one chunk up to D = 1024, four at dinounet_7b's 4096)
constexpr int LN_BWD_COLS = 1024;
__global__ void __launch_bounds__(256) f32_layernorm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                                const float* __restrict__ dy, float* __restrict__ dx,
                                                                float* __restrict__ dw, float* __restrict__ db, long long rows,
                                                                int D, float eps) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const int c0 = blockIdx.y * LN_BWD_COLS, c1 = min(D, c0 + LN_BWD_COLS);
  float pw[32], pb[32];                       // column partials of this lane: columns c0 + lane + 32 i
#pragma unroll
  for (int i = 0; i < 32; ++i) { pw[i] = 0.f; pb[i] = 0.f; }
  for (long long r = warp0; r < rows; r += nwarps) {
    const float* xr = x + r * D;
    const float* gr = dy + r * D;
    float s = 0.f;
    for (int c = lane; c < D; c += 32) s += xr[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / D;
    float q = 0.f;
    for (int c = lane; c < D; c += 32) { const float d = xr[c] - mean; q = fmaf(d, d, q); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = 1.0f / sqrtf(q / D + eps);
    float m1 = 0.f, m2 = 0.f;
    for (int c = lane; c < D; c += 32) {
      const float xh = (xr[c] - mean) * rstd, g = gr[c] * w[c];
      m1 += g;
      m2 = fmaf(g, xh, m2);
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int c = c0 + lane + 32 * i;
      if (c < c1) {
        const float xh = (xr[c] - mean) * rstd;
        pw[i] = fmaf(gr[c], xh, pw[i]);
        pb[i] += gr[c];
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { m1 += __shfl_xor_sync(0xffffffffu, m1, o); m2 += __shfl_xor_sync(0xffffffffu, m2, o); }
    m1 /= D; m2 /= D;
    for (int c = c0 + lane; c < c1; c += 32) {
      const float xh = (xr[c] - mean) * rstd;
      dx[r * D + c] = rstd * (gr[c] * w[c] - m1 - xh * m2);
    }
  }
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int c = c0 + lane + 32 * i;
    if (c < c1) { atomicAdd(&dw[c], pw[i]); atomicAdd(&db[c], pb[i]); }
  }
}
extern "C" int b2u_f32_layernorm_bwd(const float* x, const float* w, const float* dy, float* dx, float* dw, float* db,
                                     int64_t rows, int32_t D, float eps, b2u_stream_t s) {
  if (D < 1) return set_error(-1, "b2u_f32_layernorm_bwd: D %d", D);
  const long long want = (rows + 7) / 8;
  const unsigned grid = static_cast<unsigned>(want < 1184 ? (want < 1 ? 1 : want) : 1184);
  const dim3 g(grid, (D + LN_BWD_COLS - 1) / LN_BWD_COLS);
  f32_layernorm_bwd_kernel<<<g, 256, 0, static_cast<cudaStream_t>(s)>>>(x, w, dy, dx, dw, db, rows, D, eps);
  return check_launch("f32_layernorm_bwd");
}

// ---------------------------------------------------------------------------------------- InstanceNorm (+LeakyReLU) backward
// y = lrelu(xhat * w + b), xhat = (x - mean) * rstd over HW per (n, c); (mean, rstd) = stats[B][C][2] saved by the forward.
// pass 1 (rows split over gridDim.z, fp64 atomics): T1 = sum dy', T2 = sum dy' xhat per (n, c)  (dy' = dy * lrelu'(y));
//         db += T1, dw += T2;   pass 2 (elementwise): dx = rstd * w * (dy' - T1/HW - xhat * T2/HW).
__global__ void __launch_bounds__(256) f32_in_bwd_sum_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ dy,
                                                             long long lddy, const float* __restrict__ stats, const float* __restrict__ w,
                                                             const float* __restrict__ bb, double* __restrict__ work, long long HW, int Cc,
                                                             int B, int lrelu) {
  __shared__ double red[8][33], red2[8][33];
  const int cx = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  const long long b = blockIdx.y;
  const long long per = (HW + gridDim.z - 1) / gridDim.z;
  const long long lo = blockIdx.z * per, hi = lo + per < HW ? lo + per : HW;
  double t1 = 0.0, t2 = 0.0;
  if (c < Cc) {
    const float mean = stats[2 * (b * Cc + c)], rstd = stats[2 * (b * Cc + c) + 1], g = w[c], be = bb[c];
    const float* xb = x + b * HW * ldx;
    const float* gb = dy + b * HW * lddy;
    for (long long r = lo + rg; r < hi; r += 8) {
      const float xh = (xb[r * ldx + c] - mean) * rstd;
      float d = gb[r * lddy + c];
      if (lrelu && xh * g + be <= 0.f) d *= 0.01f;
      t1 += d;
      t2 += static_cast<double>(d) * xh;
    }
  }
  red[rg][cx] = t1; red2[rg][cx] = t2;
  __syncthreads();
  if (rg == 0 && c < Cc) {
    double a = 0.0, b2 = 0.0;
    for (int k = 0; k < 8; ++k) { a += red[k][cx]; b2 += red2[k][cx]; }
    atomicAdd(&work[b * Cc + c], a);
    atomicAdd(&work[(static_cast<long long>(B) + b) * Cc + c], b2);
  }
}
__global__ void f32_in_bwd_params_kernel(const double* __restrict__ work, float* __restrict__ dw, float* __restrict__ db, int B, int Cc) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= Cc) return;
  double a = 0.0, b2 = 0.0;
  for (int b = 0; b < B; ++b) { a += work[static_cast<long long>(b) * Cc + c]; b2 += work[(static_cast<long long>(B) + b) * Cc + c]; }
  db[c] += static_cast<float>(a);
  dw[c] += static_cast<float>(b2);
}
__global__ void f32_in_bwd_dx_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ dy, long long lddy,
                                     const float* __restrict__ stats, const float* __restrict__ w, const float* __restrict__ bb,
                                     const double* __restrict__ work, float* __restrict__ dx, long long lddx, int B, long long HW, int Cc,
                                     int lrelu) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= B * HW * Cc) return;
  const int c = static_cast<int>(i % Cc);
  const long long r = i / Cc, b = r / HW;
  const float mean = stats[2 * (b * Cc + c)], rstd = stats[2 * (b * Cc + c) + 1], g = w[c], be = bb[c];
  const float inv = 1.0f / static_cast<float>(HW);
  const float T1 = static_cast<float>(work[b * Cc + c]), T2 = static_cast<float>(work[(static_cast<long long>(B) + b) * Cc + c]);
  const float xh = (x[r * ldx + c] - mean) * rstd;
  float d = dy[r * lddy + c];
  if (lrelu && xh * g + be <= 0.f) d *= 0.01f;
  dx[r * lddx + c] = rstd * g * (d - inv * T1 - xh * inv * T2);
}
extern "C" int b2u_f32_instnorm_bwd(const float* x, int64_t ldx, const float* dy, int64_t lddy, const float* w, const float* b,
                                    const float* stats, double* work, float* dx, int64_t lddx, float* dw, float* db, int32_t B,
                                    int64_t HW, int32_t Cc, int32_t lrelu, b2u_stream_t s_) {
  cudaStream_t s = static_cast<cudaStream_t>(s_);
  cudaError_t e = cudaMemsetAsync(work, 0, sizeof(double) * 2 * B * Cc, s);
  if (e != cudaSuccess) return set_error(-2, "b2u_f32_instnorm_bwd: memset: %s", cudaGetErrorString(e));
  const int splits = static_cast<int>(HW >= 65536 ? 32 : (HW >= 4096 ? 8 : 1));
  f32_in_bwd_sum_kernel<<<dim3((Cc + 31) / 32, B, splits), 256, 0, s>>>(x, ldx, dy, lddy, stats, w, b, work, HW, Cc, B, lrelu);
  f32_in_bwd_params_kernel<<<(Cc + 255) / 256, 256, 0, s>>>(work, dw, db, B, Cc);
  const long long total = static_cast<long long>(B) * HW * Cc;
  f32_in_bwd_dx_kernel<<<blocks_for(total), 256, 0, s>>>(x, ldx, dy, lddy, stats, w, b, work, dx, lddx, B, HW, Cc, lrelu);
  return check_launch("f32_instnorm_bwd");
}

// ---------------------------------------------------------------------------------------- eval-mode BatchNorm (+ act)
// y = act(u), u = (x - rm) * rs * gamma + beta, rs = 1/sqrt(rv + eps)   (SyncBatchNorm in eval mode = the gradient oracle's
// semantics, oracle/grad_oracle.py).  forward and backward (dx = dy' * rs * gamma, dgamma += dy' (x - rm) rs, dbeta += dy').
__global__ void f32_bn_act_kernel(const float* __restrict__ x, float* __restrict__ y, const float* __restrict__ gamma,
                                  const float* __restrict__ beta, const float* __restrict__ rm, const float* __restrict__ rv,
                                  float eps, long long rows, int Cc, int act) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= rows * Cc) return;
  const int c = static_cast<int>(i % Cc);
  const float u = (x[i] - rm[c]) * (1.0f / sqrtf(rv[c] + eps)) * gamma[c] + beta[c];
  y[i] = act == B2U_ACT_RELU ? fmaxf(u, 0.f) : u;
}
extern "C" int b2u_f32_bn_act(const float* x, float* y, const float* gamma, const float* beta, const float* rm, const float* rv,
                              float eps, int64_t rows, int32_t Cc, int32_t act, b2u_stream_t s) {
  f32_bn_act_kernel<<<blocks_for(rows * Cc), 256, 0, static_cast<cudaStream_t>(s)>>>(x, y, gamma, beta, rm, rv, eps, rows, Cc, act);
  return check_launch("f32_bn_act");
}
__global__ void __launch_bounds__(256) f32_bn_act_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta,
                                                             const float* __restrict__ rm, const float* __restrict__ rv, float eps,
                                                             float* __restrict__ dx, float* __restrict__ dgamma,
                                                             float* __restrict__ dbeta, long long rows, int Cc, int act) {
  __shared__ float red[8][33], red2[8][33];
  const int cx = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  const long long per = (rows + gridDim.y - 1) / gridDim.y;
  const long long lo = blockIdx.y * per, hi = lo + per < rows ? lo + per : rows;
  float a = 0.f, b = 0.f;
  if (c < Cc) {
    const float rs = 1.0f / sqrtf(rv[c] + eps), g = gamma[c], be = beta[c], m = rm[c];
    for (long long r = lo + rg; r < hi; r += 8) {
      const float xn = (x[r * Cc + c] - m) * rs;
      float d = dy[r * Cc + c];
      if (act == B2U_ACT_RELU && xn * g + be <= 0.f) d = 0.f;
      dx[r * Cc + c] = d * rs * g;
      a = fmaf(d, xn, a);
      b += d;
    }
  }
  red[rg][cx] = a; red2[rg][cx] = b;
  __syncthreads();
  if (rg == 0 && c < Cc) {
    float t = 0.f, u = 0.f;
    for (int k = 0; k < 8; ++k) { t += red[k][cx]; u += red2[k][cx]; }
    atomicAdd(&dgamma[c], t);
    atomicAdd(&dbeta[c], u);
  }
}
extern "C" int b2u_f32_bn_act_bwd(const float* x, const float* dy, const float* gamma, const float* beta, const float* rm,
                                  const float* rv, float eps, float* dx, float* dgamma, float* dbeta, int64_t rows, int32_t Cc,
                                  int32_t act, b2u_stream_t s) {
  const int splits = static_cast<int>(rows > 65536 ? 64 : (rows > 2048 ? 8 : 1));
  f32_bn_act_bwd_kernel<<<dim3((Cc + 31) / 32, splits), 256, 0, static_cast<cudaStream_t>(s)>>>(x, dy, gamma, beta, rm, rv, eps, dx, dgamma, dbeta, rows, Cc, act);
  return check_launch("f32_bn_act_bwd");
}

// ---------------------------------------------------------------------------------------- depthwise 3x3 weight gradient
// dw9[tap][c] += sum_p dy[p, c] * x[p + tap, c];  db[c] += sum_p dy[p, c]   (same plane layout as b2u_f32_dwconv3x3)
__global__ void __launch_bounds__(256) f32_dwconv_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                               float* __restrict__ dw9, float* __restrict__ db, int B, int H, int W,
                                                               int Cc, int planes) {
  __shared__ float red[8][10][33];
  const int cx = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  const long long per_b = planes == 3 ? static_cast<long long>(H) * W * 21 / 4 : static_cast<long long>(H) * W;
  const long long total = B * per_b;
  const long long per = (total + gridDim.y - 1) / gridDim.y;
  const long long lo = blockIdx.y * per, hi = lo + per < total ? lo + per : total;
  float acc[10];
#pragma unroll
  for (int i = 0; i < 10; ++i) acc[i] = 0.f;
  if (c < Cc)
    for (long long i = lo + rg; i < hi; i += 8) {
      const long long b = i / per_b, t = i - b * per_b;
      long long base = 0, local = t;
      int ph = H, pw = W;
      if (planes == 3) {
        const long long n16 = static_cast<long long>(H) * W * 4, n4 = static_cast<long long>(H) * W;
        if (t < n16) { ph = 2 * H; pw = 2 * W; }
        else if (t < n16 + n4) { base = n16; local = t - n16; }
        else { base = n16 + n4; local = t - n16 - n4; ph = H / 2; pw = W / 2; }
      }
      const int y = static_cast<int>(local / pw), xx = static_cast<int>(local - static_cast<long long>(y) * pw);
      const float d = dy[i * Cc + c];
      acc[9] += d;
#pragma unroll
      for (int dyy = 0; dyy < 3; ++dyy)
#pragma unroll
        for (int dxx = 0; dxx < 3; ++dxx) {
          const int iy = y + dyy - 1, ix = xx + dxx - 1;
          if (iy >= 0 && iy < ph && ix >= 0 && ix < pw)
            acc[dyy * 3 + dxx] = fmaf(d, x[(b * per_b + base + static_cast<long long>(iy) * pw + ix) * Cc + c], acc[dyy * 3 + dxx]);
        }
    }
#pragma unroll
  for (int i = 0; i < 10; ++i) red[rg][i][cx] = acc[i];
  __syncthreads();
  if (rg == 0 && c < Cc) {
    for (int i = 0; i < 10; ++i) {
      float t = 0.f;
      for (int k = 0; k < 8; ++k) t += red[k][i][cx];
      if (i < 9) atomicAdd(&dw9[i * Cc + c], t);
      else atomicAdd(&db[c], t);
    }
  }
}
extern "C" int b2u_f32_dwconv_wgrad(const float* x, const float* dy, float* dw9, float* db, int32_t B, int32_t H, int32_t W,
                                    int32_t Cc, int32_t planes, b2u_stream_t s) {
  const long long per_b = planes == 3 ? static_cast<long long>(H) * W * 21 / 4 : static_cast<long long>(H) * W;
  const long long total = B * per_b;
  const int splits = static_cast<int>(total > 65536 ? 64 : (total > 2048 ? 8 : 1));
  f32_dwconv_wgrad_kernel<<<dim3((Cc + 31) / 32, splits), 256, 0, static_cast<cudaStream_t>(s)>>>(x, dy, dw9, db, B, H, W, Cc, planes);
  return check_launch("f32_dwconv_wgrad");
}

// ---------------------------------------------------------------------------------------- max-pool 3x3 s2 backward
// dx[argmax window] += dy  (first maximum in row-major window order, like ATen's saved indices); dx zero-initialised
__global__ void f32_maxpool_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx, int B, int H,
                                       int W, int Cc) {
  const int Ho = H / 2, Wo = W / 2;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * Ho * Wo * Cc;
  if (i >= total) return;
  const int c = static_cast<int>(i % Cc);
  const long long pr = i / Cc;
  const int xo = static_cast<int>(pr % Wo), yo = static_cast<int>((pr / Wo) % Ho), b = static_cast<int>(pr / (static_cast<long long>(Wo) * Ho));
  float m = -INFINITY;
  long long arg = -1;
  for (int dyy = -1; dyy <= 1; ++dyy)
    for (int dxx = -1; dxx <= 1; ++dxx) {
      const int iy = 2 * yo + dyy, ix = 2 * xo + dxx;
      if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
        const long long idx = ((static_cast<long long>(b) * H + iy) * W + ix) * Cc + c;
        const float v = x[idx];
        if (v > m) { m = v; arg = idx; }
      }
    }
  if (arg >= 0) atomicAdd(&dx[arg], dy[i]);
}
extern "C" int b2u_f32_maxpool3x3s2_bwd(const float* x, const float* dy, float* dx, int32_t B, int32_t H, int32_t W, int32_t Cc,
                                        b2u_stream_t s) {
  const long long total = static_cast<long long>(B) * (H / 2) * (W / 2) * Cc;
  f32_maxpool_bwd_kernel<<<blocks_for(total), 256, 0, static_cast<cudaStream_t>(s)>>>(x, dy, dx, B, H, W, Cc);
  return check_launch("f32_maxpool_bwd");
}

// ---------------------------------------------------------------------------------------- FiLM backward
// z = gamma * zp + beta: dgb = (dz * zp | dz);  dzz[:, R:] = dz * gamma   (dzz[:, :R] is written by the film_gen data gradient)
__global__ void f32_film_bwd_kernel(const float* __restrict__ gb, const float* __restrict__ zz, const float* __restrict__ dz,
                                    float* __restrict__ dgb, float* __restrict__ dzz, long long px, int R) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= px * R) return;
  const long long r = i / R;
  const int c = static_cast<int>(i - r * R);
  const float d = dz[i];
  dgb[r * 2 * R + c] = d * zz[r * 2 * R + R + c];
  dgb[r * 2 * R + R + c] = d;
  dzz[r * 2 * R + R + c] = d * gb[r * 2 * R + c];
}
extern "C" int b2u_f32_film_bwd(const float* gb, const float* zz, const float* dz, float* dgb, float* dzz, int64_t px, int32_t R,
                                b2u_stream_t s) {
  f32_film_bwd_kernel<<<blocks_for(px * R), 256, 0, static_cast<cudaStream_t>(s)>>>(gb, zz, dz, dgb, dzz, px, R);
  return check_launch("f32_film_bwd");
}

// ---------------------------------------------------------------------------------------- SqueezeExcitation backward
// out = t * gate[b, c] + sc.  (1) dgate[b, c] = sum_hw dy * t  (2) one block per batch item: gate MLP backward ->
// dpooled[b, c] and the weight gradients  (3) dt = dy * gate + dpooled / HW   (dsc = dy is the caller's view).
__global__ void __launch_bounds__(256) f32_se_dgate_kernel(const float* __restrict__ t, const float* __restrict__ dy, float* __restrict__ dgate,
                                                           long long HW, int Cc) {
  __shared__ float red[8][33];
  const int cx = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  const long long b = blockIdx.y;
  float s = 0.f;
  if (c < Cc)
    for (long long r = rg; r < HW; r += 8) s = fmaf(dy[(b * HW + r) * Cc + c], t[(b * HW + r) * Cc + c], s);
  red[rg][cx] = s;
  __syncthreads();
  if (rg == 0 && c < Cc) {
    float u = 0.f;
    for (int k = 0; k < 8; ++k) u += red[k][cx];
    dgate[b * Cc + c] = u;
  }
}
__global__ void __launch_bounds__(256) f32_se_mlp_bwd_kernel(const float* __restrict__ pooled, const float* __restrict__ dgate,
                                                             const float* __restrict__ w1, const float* __restrict__ b1,
                                                             const float* __restrict__ w2, const float* __restrict__ b2,
                                                             float* __restrict__ gate, float* __restrict__ dpooled, float* __restrict__ dw1,
                                                             float* __restrict__ db1, float* __restrict__ dw2, float* __restrict__ db2,
                                                             int Cc, int hid) {
  __shared__ float s_a1[64], s_h[64], s_da2[256], s_da1[64];
  const int b = blockIdx.x;
  const float* pl = pooled + static_cast<long long>(b) * Cc;
  for (int j = threadIdx.x; j < hid; j += 256) {
    float a = b1[j];
    for (int c = 0; c < Cc; ++c) a = fmaf(w1[j * Cc + c], pl[c], a);
    s_a1[j] = a;
    s_h[j] = fmaxf(a, 0.f);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < Cc; c += 256) {
    float a = b2[c];
    for (int j = 0; j < hid; ++j) a = fmaf(w2[c * hid + j], s_h[j], a);
    const float g = 1.0f / (1.0f + expf(-a));
    gate[static_cast<long long>(b) * Cc + c] = g;
    const float da2 = dgate[static_cast<long long>(b) * Cc + c] * g * (1.0f - g);
    s_da2[c] = da2;
    atomicAdd(&db2[c], da2);
    for (int j = 0; j < hid; ++j) atomicAdd(&dw2[c * hid + j], da2 * s_h[j]);
  }
  __syncthreads();
  for (int j = threadIdx.x; j < hid; j += 256) {
    float dh = 0.f;
    for (int c = 0; c < Cc; ++c) dh = fmaf(w2[c * hid + j], s_da2[c], dh);
    const float da1 = s_a1[j] > 0.f ? dh : 0.f;
    s_da1[j] = da1;
    atomicAdd(&db1[j], da1);
    for (int c = 0; c < Cc; ++c) atomicAdd(&dw1[j * Cc + c], da1 * pl[c]);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < Cc; c += 256) {
    float d = 0.f;
    for (int j = 0; j < hid; ++j) d = fmaf(w1[j * Cc + c], s_da1[j], d);
    dpooled[static_cast<long long>(b) * Cc + c] = d;
  }
}
__global__ void f32_se_dt_kernel(const float* __restrict__ dy, const float* __restrict__ gate, const float* __restrict__ dpooled,
                                 float* __restrict__ dt, int B, long long HW, int Cc) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= B * HW * Cc) return;
  const int c = static_cast<int>(i % Cc);
  const long long b = i / (HW * Cc);
  dt[i] = dy[i] * gate[b * Cc + c] + dpooled[b * Cc + c] / static_cast<float>(HW);
}
extern "C" int b2u_f32_se_bwd(const float* t, const float* dy, const float* pooled, const float* w1, const float* b1, const float* w2,
                              const float* b2, float* work /* 3*B*C: dgate | gate | dpooled */, float* dt, float* dw1, float* db1,
                              float* dw2, float* db2, int32_t B, int64_t HW, int32_t Cc, int32_t hid, b2u_stream_t s_) {
  if (Cc > 256 || hid > 64) return set_error(-1, "b2u_f32_se_bwd: at most 256 channels / 64 hidden");
  cudaStream_t s = static_cast<cudaStream_t>(s_);
  float* dgate = work;
  float* gate = work + static_cast<long long>(B) * Cc;
  float* dpooled = gate + static_cast<long long>(B) * Cc;
  f32_se_dgate_kernel<<<dim3((Cc + 31) / 32, B), 256, 0, s>>>(t, dy, dgate, HW, Cc);
  int rc = check_launch("f32_se_dgate");
  if (rc) return rc;
  f32_se_mlp_bwd_kernel<<<B, 256, 0, s>>>(pooled, dgate, w1, b1, w2, b2, gate, dpooled, dw1, db1, dw2, db2, Cc, hid);
  if ((rc = check_launch("f32_se_mlp_bwd"))) return rc;
  f32_se_dt_kernel<<<blocks_for(static_cast<long long>(B) * HW * Cc), 256, 0, s>>>(dy, gate, dpooled, dt, B, HW, Cc);
  return check_launch("f32_se_dt");
}

// ---------------------------------------------------------------------------------------- MSDA prologue (training path)
// offaw [B*Lq, heads*12] -> loc [B, Lq, heads, 1, 4, 2], attw [B, Lq, heads, 1, 4] for b2u_msda_forward_f32 / backward_f32,
// and back: doffaw from (dloc, dattw).  Same maths as f32_msda_kernel's prologue.
__global__ void f32_msda_prep_kernel(const float* __restrict__ offaw, float* __restrict__ loc, float* __restrict__ attw, int B, int Hv,
                                     int Wv, int heads) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int HW = Hv * Wv;
  const long long Lq = static_cast<long long>(HW) * 21 / 4;
  if (i >= B * Lq * heads) return;
  const int m = static_cast<int>(i % heads);
  const long long bq = i / heads;
  const long long q = bq % Lq;
  int gh, gw;
  long long local;
  if (q < 4LL * HW) { gh = 2 * Hv; gw = 2 * Wv; local = q; }
  else if (q < 5LL * HW) { gh = Hv; gw = Wv; local = q - 4LL * HW; }
  else { gh = Hv / 2; gw = Wv / 2; local = q - 5LL * HW; }
  const int ry = static_cast<int>(local / gw), rx = static_cast<int>(local - static_cast<long long>(ry) * gw);
  const float refx = (rx + 0.5f) / gw, refy = (ry + 0.5f) / gh;
  const float* o = offaw + bq * (heads * 12) + m * 8;
  const float* a = offaw + bq * (heads * 12) + heads * 8 + m * 4;
  const float mx = fmaxf(fmaxf(a[0], a[1]), fmaxf(a[2], a[3]));
  float e[4], s = 0.f;
  for (int p = 0; p < 4; ++p) { e[p] = expf(a[p] - mx); s += e[p]; }
  for (int p = 0; p < 4; ++p) {
    loc[(i * 4 + p) * 2] = refx + o[2 * p] / Wv;
    loc[(i * 4 + p) * 2 + 1] = refy + o[2 * p + 1] / Hv;
    attw[i * 4 + p] = e[p] / s;
  }
}
__global__ void f32_msda_prep_bwd_kernel(const float* __restrict__ attw, const float* __restrict__ dloc, const float* __restrict__ dattw,
                                         float* __restrict__ doffaw, long long n_bqm, int Hv, int Wv, int heads) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n_bqm) return;
  const int m = static_cast<int>(i % heads);
  const long long bq = i / heads;
  float* o = doffaw + bq * (heads * 12) + m * 8;
  float* a = doffaw + bq * (heads * 12) + heads * 8 + m * 4;
  float dot = 0.f;
  for (int p = 0; p < 4; ++p) dot = fmaf(attw[i * 4 + p], dattw[i * 4 + p], dot);
  for (int p = 0; p < 4; ++p) {
    o[2 * p] = dloc[(i * 4 + p) * 2] / Wv;
    o[2 * p + 1] = dloc[(i * 4 + p) * 2 + 1] / Hv;
    a[p] = attw[i * 4 + p] * (dattw[i * 4 + p] - dot);
  }
}
extern "C" int b2u_f32_msda_prep(const float* offaw, float* loc, float* attw, int32_t B, int32_t Hv, int32_t Wv, int32_t heads, b2u_stream_t s) {
  const long long n = static_cast<long long>(B) * (static_cast<long long>(Hv) * Wv * 21 / 4) * heads;
  f32_msda_prep_kernel<<<blocks_for(n), 256, 0, static_cast<cudaStream_t>(s)>>>(offaw, loc, attw, B, Hv, Wv, heads);
  return check_launch("f32_msda_prep");
}
extern "C" int b2u_f32_msda_prep_bwd(const float* attw, const float* dloc, const float* dattw, float* doffaw, int32_t B, int32_t Hv,
                                     int32_t Wv, int32_t heads, b2u_stream_t s) {
  const long long n = static_cast<long long>(B) * (static_cast<long long>(Hv) * Wv * 21 / 4) * heads;
  f32_msda_prep_bwd_kernel<<<blocks_for(n), 256, 0, static_cast<cudaStream_t>(s)>>>(attw, dloc, dattw, doffaw, n, Hv, Wv, heads);
  return check_launch("f32_msda_prep_bwd");
}

// ---------------------------------------------------------------------------------------- transposed-conv helpers
// dy image [B, 2h, 2w, ld] (columns col_off .. col_off+Cout) -> rows [B*h*w, 4*Cout] with n = (2a+b)*Cout + co: the
// inverse of the pixel-shuffle store of the forward GEMM, so that ConvTranspose2d(k2,s2) backward is two plain GEMMs.
__global__ void f32_unshuffle_kernel(const float* __restrict__ dy, long long ld, int col_off, float* __restrict__ out, int B, int h, int w, int Cout) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * h * w * 4 * Cout;
  if (i >= total) return;
  const int n = static_cast<int>(i % (4 * Cout));
  const long long m = i / (4 * Cout);
  const int q = n / Cout, co = n - q * Cout;
  const int j = static_cast<int>(m % w), ii = static_cast<int>((m / w) % h);
  const long long b = m / (static_cast<long long>(w) * h);
  const long long row = (b * (2 * h) + 2 * ii + (q >> 1)) * (2 * w) + 2 * j + (q & 1);
  out[i] = dy[row * ld + col_off + co];
}
extern "C" int b2u_f32_unshuffle(const float* dy, int64_t ld, int32_t col_off, float* out, int32_t B, int32_t h, int32_t w, int32_t Cout,
                                 b2u_stream_t s) {
  const long long total = static_cast<long long>(B) * h * w * 4 * Cout;
  f32_unshuffle_kernel<<<blocks_for(total), 256, 0, static_cast<cudaStream_t>(s)>>>(dy, ld, col_off, out, B, h, w, Cout);
  return check_launch("f32_unshuffle");
}

// ---------------------------------------------------------------------------------------- 3x3 convolution gradients
// data gradient for any stride (used for the stride-2 SPM convs; stride-1 layers go through b2u_f32_gemm w_mode 2):
// dx[b, iy, ix, c] = sum_{tap, n} dy[b, (iy+1-dy)/s, (ix+1-dx)/s, n] * W[n][tap*Cpad + c]   (where divisible and in range)
__global__ void f32_conv3x3_dgrad_kernel(const float* __restrict__ dy, const float* __restrict__ W, float* __restrict__ dx, int B, int H,
                                         int Wd, int Cc, int Cpad, int N, int stride) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * H * Wd * Cc;
  if (i >= total) return;
  const int c = static_cast<int>(i % Cc);
  const long long pr = i / Cc;
  const int ix = static_cast<int>(pr % Wd), iy = static_cast<int>((pr / Wd) % H);
  const long long b = pr / (static_cast<long long>(Wd) * H);
  const int Ho = H / stride, Wo = Wd / stride;
  float acc = 0.f;
  for (int dyy = 0; dyy < 3; ++dyy) {
    const int ty = iy + 1 - dyy;
    if (ty < 0 || ty % stride) continue;
    const int oy = ty / stride;
    if (oy >= Ho) continue;
    for (int dxx = 0; dxx < 3; ++dxx) {
      const int tx = ix + 1 - dxx;
      if (tx < 0 || tx % stride) continue;
      const int ox = tx / stride;
      if (ox >= Wo) continue;
      const float* g = dy + ((b * Ho + oy) * Wo + ox) * N;
      const float* wp = W + (dyy * 3 + dxx) * Cpad + c;
      for (int n = 0; n < N; ++n) acc = fmaf(g[n], wp[static_cast<long long>(n) * 9 * Cpad], acc);
    }
  }
  dx[i] = acc;
}
extern "C" int b2u_f32_conv3x3_dgrad(const float* dy, const float* W, float* dx, int32_t B, int32_t H, int32_t Wd, int32_t Cc,
                                     int32_t Cpad, int32_t N, int32_t stride, b2u_stream_t s) {
  const long long total = static_cast<long long>(B) * H * Wd * Cc;
  f32_conv3x3_dgrad_kernel<<<blocks_for(total), 256, 0, static_cast<cudaStream_t>(s)>>>(dy, W, dx, B, H, Wd, Cc, Cpad, N, stride);
  return check_launch("f32_conv3x3_dgrad");
}
// weight gradient: dW[n][tap*Cpad + c] += sum_pix dy[pix, n] * x[pix*stride + tap - 1, c].
// grid (9 taps, (N/16)*(C/16) tiles, pixel splits), block 16 x 16 = (n, c); 32 output pixels staged per iteration.
__global__ void __launch_bounds__(256) f32_conv3x3_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                                float* __restrict__ dW, int B, int H, int Wd, int Cc, int Cpad, int N,
                                                                int stride) {
  __shared__ float sg[32][17], sx[32][17];
  const int tap = blockIdx.x, dyy = tap / 3, dxx = tap - dyy * 3;
  const int ct = (Cc + 15) / 16;
  const int n0 = (blockIdx.y / ct) * 16, c0 = (blockIdx.y % ct) * 16;
  const int tn = threadIdx.x >> 4, tc = threadIdx.x & 15;
  const int Ho = H / stride, Wo = Wd / stride;
  const long long total = static_cast<long long>(B) * Ho * Wo;
  const long long per = ((total + gridDim.z - 1) / gridDim.z + 31) / 32 * 32;
  const long long lo = blockIdx.z * per, hi = lo + per < total ? lo + per : total;
  float acc = 0.f;
  for (long long p0 = lo; p0 < hi; p0 += 32) {
    for (int e = threadIdx.x; e < 32 * 16; e += 256) {
      const int pp = e >> 4, k = e & 15;
      const long long p = p0 + pp;
      float g = 0.f, xv = 0.f;
      if (p < hi) {
        if (n0 + k < N) g = dy[p * N + n0 + k];
        const int ox = static_cast<int>(p % Wo), oy = static_cast<int>((p / Wo) % Ho);
        const long long b = p / (static_cast<long long>(Wo) * Ho);
        const int iy = oy * stride + dyy - 1, ix = ox * stride + dxx - 1;
        if (c0 + k < Cc && iy >= 0 && iy < H && ix >= 0 && ix < Wd) xv = x[((b * H + iy) * Wd + ix) * Cc + c0 + k];
      }
      sg[pp][k] = g;
      sx[pp][k] = xv;
    }
    __syncthreads();
#pragma unroll
    for (int pp = 0; pp < 32; ++pp) acc = fmaf(sg[pp][tn], sx[pp][tc], acc);
    __syncthreads();
  }
  if (n0 + tn < N && c0 + tc < Cc) atomicAdd(&dW[static_cast<long long>(n0 + tn) * 9 * Cpad + tap * Cpad + c0 + tc], acc);
}
extern "C" int b2u_f32_conv3x3_wgrad(const float* x, const float* dy, float* dW, int32_t B, int32_t H, int32_t Wd, int32_t Cc,
                                     int32_t Cpad, int32_t N, int32_t stride, b2u_stream_t s) {
  const long long total = static_cast<long long>(B) * (H / stride) * (Wd / stride);
  int splits = static_cast<int>(total / 4096);
  splits = splits < 1 ? 1 : (splits > 256 ? 256 : splits);
  dim3 grid(9, ((N + 15) / 16) * ((Cc + 15) / 16), splits);
  f32_conv3x3_wgrad_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(s)>>>(x, dy, dW, B, H, Wd, Cc, Cpad, N, stride);
  return check_launch("f32_conv3x3_wgrad");
}

// ---------------------------------------------------------------------------------------- optimizer
// sum of squares (double) for the global gradient-norm clip (nnUNetTrainer.py:922: clip_grad_norm_(parameters, 12))
__global__ void __launch_bounds__(256) f32_sqsum_kernel(const float* __restrict__ g, long long n, double* __restrict__ out) {
  __shared__ double red[256];
  double s = 0.0;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x)
    s += static_cast<double>(g[i]) * g[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) atomicAdd(out, red[0]);
}
extern "C" int b2u_f32_sqsum(const float* g, int64_t n, double* out, b2u_stream_t s) {
  const unsigned grid = static_cast<unsigned>(n / 4096 < 1 ? 1 : (n / 4096 > 512 ? 512 : n / 4096));
  f32_sqsum_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(s)>>>(g, n, out);
  return check_launch("f32_sqsum");
}
// torch.optim.SGD(momentum, nesterov=True, weight_decay) step with the clip coefficient read from device memory
// (nnUNetTrainer.py:486-489, 922-923): g = g * min(1, max_norm / (norm + 1e-6)) + wd * p; buf = mom * buf + g;
// p -= lr * (g + mom * buf).  sqsum = the squared total gradient norm.
__global__ void f32_sgd_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ buf, long long n, float lr,
                               float mom, float wd, const double* __restrict__ sqsum, float max_norm, int first) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float coef = 1.f;
  if (sqsum && max_norm > 0.f) {
    const float norm = static_cast<float>(sqrt(*sqsum));
    coef = fminf(1.f, max_norm / (norm + 1e-6f));
  }
  const float gg = g[i] * coef + wd * p[i];
  const float b = first ? gg : mom * buf[i] + gg;
  buf[i] = b;
  p[i] -= lr * (gg + mom * b);
}
extern "C" int b2u_f32_sgd_nesterov(float* p, const float* g, float* buf, int64_t n, float lr, float momentum, float weight_decay,
                                    const double* sqsum, float max_norm, int32_t first_step, b2u_stream_t s) {
  f32_sgd_kernel<<<blocks_for(n), 256, 0, static_cast<cudaStream_t>(s)>>>(p, g, buf, n, lr, momentum, weight_decay, sqsum, max_norm, first_step);
  return check_launch("f32_sgd");
}

}  // namespace b2u
