// Train-mode semantics of the reference's training step (nnUNetTrainer.on_train_epoch_start -> network.train()):
// batch-statistics SyncBatchNorm with the running-statistic update (dinov3_adapter.py:239-277, 479-482), the extractors'
// DropPath(0.3) residual (dinov3_adapter.py:18-27, 148) and the frozen ViT's per-block RoPE coordinate rescaling
// (rope_position_encoding.py:93-97).  fp32 data, fp64 reductions through fixed-order partials: no atomics, so two
// identical launches give identical bits.  Layout: [rows, C] row-major (NHWC pixels or tokens), like train_bwd.cu.
#include <math.h>

#include "common.cuh"
#include "../../include/dinounet_b200.h"
#include "host_util.h"

namespace b2u {

static inline unsigned tm_blocks_for(long long n, int t = 256) { return static_cast<unsigned>((n + t - 1) / t); }

// row splits of the per-channel reductions: a function of `rows` only, so the partial layout (and the sum order) is fixed
static inline int bn_splits(long long rows) {
  const long long s = rows / 4096;
  return static_cast<int>(s < 1 ? 1 : (s > 256 ? 256 : s));
}

// grid (C/32, splits), block 32 x 8: partials[split][0][c] = sum x, partials[split][1][c] = sum x^2 over the split's rows
__global__ void __launch_bounds__(256) bn_stats_partial_kernel(const float* __restrict__ x, long long rows, int Cc,
                                                               double* __restrict__ part) {
  __shared__ double r1[8][33], r2[8][33];
  const int cx = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  const long long per = (rows + gridDim.y - 1) / gridDim.y;
  const long long lo = blockIdx.y * per, hi = lo + per < rows ? lo + per : rows;
  double s1 = 0.0, s2 = 0.0;
  if (c < Cc)
    for (long long r = lo + rg; r < hi; r += 8) {
      const double v = x[r * Cc + c];
      s1 += v;
      s2 = fma(v, v, s2);
    }
  r1[rg][cx] = s1; r2[rg][cx] = s2;
  __syncthreads();
  if (rg == 0 && c < Cc) {
    double a = 0.0, b = 0.0;
    for (int k = 0; k < 8; ++k) { a += r1[k][cx]; b += r2[k][cx]; }
    part[(2LL * blockIdx.y) * Cc + c] = a;
    part[(2LL * blockIdx.y + 1) * Cc + c] = b;
  }
}

// out[0:C], out[C:2C] = partials summed in split order; out[2C] = rows
__global__ void bn_combine_kernel(const double* __restrict__ part, int splits, int Cc, long long rows, double* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c == 0) out[2 * Cc] = static_cast<double>(rows);
  if (c >= Cc) return;
  double a = 0.0, b = 0.0;
  for (int s = 0; s < splits; ++s) { a += part[(2LL * s) * Cc + c]; b += part[(2LL * s + 1) * Cc + c]; }
  out[c] = a;
  out[Cc + c] = b;
}

__global__ void bn_finalize_kernel(const double* __restrict__ sums, int Cc, float* __restrict__ mean, float* __restrict__ var,
                                   float* __restrict__ rm, float* __restrict__ rv, long long* __restrict__ nbt, float momentum) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c == 0) *nbt += 1;
  if (c >= Cc) return;
  const double n = sums[2 * Cc];
  const double mu = sums[c] / n;
  const double v = fmax(sums[Cc + c] / n - mu * mu, 0.0);
  mean[c] = static_cast<float>(mu);
  var[c] = static_cast<float>(v);
  const double m = momentum;
  rm[c] = static_cast<float>(m * mu + (1.0 - m) * static_cast<double>(rm[c]));
  rv[c] = static_cast<float>(m * (v * n / (n - 1.0)) + (1.0 - m) * static_cast<double>(rv[c]));
}

// the forward's normalised value and ReLU mask, computed exactly as b2u_f32_bn_act computes them
__device__ __forceinline__ float bn_grad_in(float xv, float d, float mu, float rs, float g, float be, int act, float* xh) {
  *xh = (xv - mu) * rs;
  if (act == B2U_ACT_RELU && (xv - mu) * rs * g + be <= 0.f) d = 0.f;
  return d;
}

__global__ void __launch_bounds__(256) bn_bwd_partial_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta,
                                                             const float* __restrict__ mean, const float* __restrict__ var, float eps,
                                                             long long rows, int Cc, int act, double* __restrict__ part) {
  __shared__ double r1[8][33], r2[8][33];
  const int cx = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  const long long per = (rows + gridDim.y - 1) / gridDim.y;
  const long long lo = blockIdx.y * per, hi = lo + per < rows ? lo + per : rows;
  double s1 = 0.0, s2 = 0.0;
  if (c < Cc) {
    const float mu = mean[c], rs = 1.0f / sqrtf(var[c] + eps), g = gamma[c], be = beta[c];
    for (long long r = lo + rg; r < hi; r += 8) {
      float xh;
      const float d = bn_grad_in(x[r * Cc + c], dy[r * Cc + c], mu, rs, g, be, act, &xh);
      s1 += d;
      s2 = fma(static_cast<double>(d), static_cast<double>(xh), s2);
    }
  }
  r1[rg][cx] = s1; r2[rg][cx] = s2;
  __syncthreads();
  if (rg == 0 && c < Cc) {
    double a = 0.0, b = 0.0;
    for (int k = 0; k < 8; ++k) { a += r1[k][cx]; b += r2[k][cx]; }
    part[(2LL * blockIdx.y) * Cc + c] = a;
    part[(2LL * blockIdx.y + 1) * Cc + c] = b;
  }
}

__global__ void bn_bwd_params_kernel(const double* __restrict__ red, int Cc, float* __restrict__ dgamma, float* __restrict__ dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= Cc) return;
  dbeta[c] = static_cast<float>(red[c]);
  dgamma[c] = static_cast<float>(red[Cc + c]);
}

__global__ void bn_bwd_apply_kernel(const float* __restrict__ x, const float* __restrict__ dy, const float* __restrict__ gamma,
                                    const float* __restrict__ beta, const float* __restrict__ mean, const float* __restrict__ var,
                                    float eps, const double* __restrict__ red, float* __restrict__ dx, long long rows, int Cc, int act) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= rows * Cc) return;
  const int c = static_cast<int>(i % Cc);
  const float mu = mean[c], rs = 1.0f / sqrtf(var[c] + eps), g = gamma[c];
  const double n = red[2 * Cc];
  const float m1 = static_cast<float>(red[c] / n), m2 = static_cast<float>(red[Cc + c] / n);
  float xh;
  const float d = bn_grad_in(x[i], dy[i], mu, rs, g, beta[c], act, &xh);
  dx[i] = g * rs * (d - m1 - xh * m2);
}

__global__ void droppath_add_kernel(const float* __restrict__ c, const float* __restrict__ f, const float* __restrict__ s,
                                    float* __restrict__ y, long long n, int D, long long rows_per_sample) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float sc = s[(i / D) / rows_per_sample];
  const float v = sc * f[i];
  y[i] = c != nullptr ? c[i] + v : v;
}

// one thread per (block, token, column j < head_dim/2); column j and j + head_dim/2 carry the same angle (`tile(2)`)
__global__ void rope_tables_kernel(const float* __restrict__ periods, const float* __restrict__ scales, float* __restrict__ sn,
                                   float* __restrict__ cs, int depth, int h, int w, int hd) {
  const long long half = hd / 2, q = hd / 4;
  const long long total = static_cast<long long>(depth) * h * w * half;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int j = static_cast<int>(i % half);
  const long long t = (i / half) % (static_cast<long long>(h) * w);
  const int blk = static_cast<int>(i / (half * h * w));
  const int axis = static_cast<int>(j / q), k = static_cast<int>(j % q);
  const int pos = axis == 0 ? static_cast<int>(t / w) : static_cast<int>(t % w);
  const int extent = axis == 0 ? h : w;
  float coord = (static_cast<float>(pos) + 0.5f) / static_cast<float>(extent);
  coord = 2.0f * coord - 1.0f;
  coord = coord * scales[blk];
  const float ang = (6.283185307179586f * coord) / periods[k];
  const long long row = (static_cast<long long>(blk) * h * w + t) * hd;
  const float sv = sinf(ang), cv = cosf(ang);
  sn[row + j] = sv; sn[row + j + half] = sv;
  cs[row + j] = cv; cs[row + j + half] = cv;
}

}  // namespace b2u

using namespace b2u;

extern "C" int64_t b2u_f32_bn_work_doubles(int64_t rows, int32_t C) { return 2LL * bn_splits(rows) * C; }

extern "C" int b2u_f32_bn_stats(const float* x, int64_t rows, int32_t C, double* work, double* sums, b2u_stream_t s_) {
  if (rows < 1 || C < 1) return set_error(-1, "b2u_f32_bn_stats: rows %lld, C %d", static_cast<long long>(rows), C);
  cudaStream_t s = static_cast<cudaStream_t>(s_);
  const int splits = bn_splits(rows);
  bn_stats_partial_kernel<<<dim3((C + 31) / 32, splits), 256, 0, s>>>(x, rows, C, work);
  bn_combine_kernel<<<(C + 255) / 256, 256, 0, s>>>(work, splits, C, rows, sums);
  return check_launch("f32_bn_stats");
}

extern "C" int b2u_f32_bn_finalize(const double* sums, int32_t C, float* mean, float* var, float* running_mean, float* running_var,
                                   int64_t* num_batches_tracked, float momentum, b2u_stream_t s_) {
  bn_finalize_kernel<<<(C + 255) / 256, 256, 0, static_cast<cudaStream_t>(s_)>>>(
      sums, C, mean, var, running_mean, running_var, reinterpret_cast<long long*>(num_batches_tracked), momentum);
  return check_launch("f32_bn_finalize");
}

extern "C" int b2u_f32_bn_train_bwd_reduce(const float* x, const float* dy, const float* gamma, const float* beta, const float* mean,
                                           const float* var, float eps, int64_t rows, int32_t C, int32_t act, double* work, double* red,
                                           float* dgamma, float* dbeta, b2u_stream_t s_) {
  if (rows < 1 || C < 1) return set_error(-1, "b2u_f32_bn_train_bwd_reduce: rows %lld, C %d", static_cast<long long>(rows), C);
  cudaStream_t s = static_cast<cudaStream_t>(s_);
  const int splits = bn_splits(rows);
  bn_bwd_partial_kernel<<<dim3((C + 31) / 32, splits), 256, 0, s>>>(x, dy, gamma, beta, mean, var, eps, rows, C, act, work);
  bn_combine_kernel<<<(C + 255) / 256, 256, 0, s>>>(work, splits, C, rows, red);
  bn_bwd_params_kernel<<<(C + 255) / 256, 256, 0, s>>>(red, C, dgamma, dbeta);
  return check_launch("f32_bn_train_bwd_reduce");
}

extern "C" int b2u_f32_bn_train_bwd_apply(const float* x, const float* dy, const float* gamma, const float* beta, const float* mean,
                                          const float* var, float eps, const double* red, float* dx, int64_t rows, int32_t C,
                                          int32_t act, b2u_stream_t s_) {
  bn_bwd_apply_kernel<<<tm_blocks_for(rows * C), 256, 0, static_cast<cudaStream_t>(s_)>>>(x, dy, gamma, beta, mean, var, eps, red,
                                                                                        dx, rows, C, act);
  return check_launch("f32_bn_train_bwd_apply");
}

extern "C" int b2u_f32_droppath_add(const float* c, const float* f, const float* s, float* y, int64_t rows, int32_t D,
                                    int64_t rows_per_sample, b2u_stream_t s_) {
  if (rows_per_sample < 1) return set_error(-1, "b2u_f32_droppath_add: rows_per_sample %lld", static_cast<long long>(rows_per_sample));
  droppath_add_kernel<<<tm_blocks_for(rows * D), 256, 0, static_cast<cudaStream_t>(s_)>>>(c, f, s, y, rows * D, D, rows_per_sample);
  return check_launch("f32_droppath_add");
}

extern "C" int b2u_rope_tables(const float* periods, const float* scales, float* sin, float* cos, int32_t depth, int32_t h, int32_t w,
                               int32_t head_dim, b2u_stream_t s_) {
  if (head_dim % 4 != 0 || depth < 1 || h < 1 || w < 1)
    return set_error(-1, "b2u_rope_tables: head_dim %d (multiple of 4), depth %d, %dx%d", head_dim, depth, h, w);
  const long long total = static_cast<long long>(depth) * h * w * (head_dim / 2);
  rope_tables_kernel<<<tm_blocks_for(total), 256, 0, static_cast<cudaStream_t>(s_)>>>(periods, scales, sin, cos, depth, h, w, head_dim);
  return check_launch("rope_tables");
}
