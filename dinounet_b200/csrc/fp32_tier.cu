// fp32 parity tier: the whole Dino U-Net forward in IEEE fp32 (FMA accumulation, exact erf/exp), one plain SIMT kernel per
// operator.  It exists for ONE purpose: north_star's "within 1e-5 of the reference PyTorch forward in fp32" - the
// reference's fp32 regime is its CPU forward (autocast('cuda') self-disables, dinov3_adapter.py:422), which the 16-bit
// tensor-core path cannot meet by construction (BASELINE.md section 5: bf16-ViT noise floor 2.5e-2).  These kernels are
// deliberately simple (no tensor cores: TF32 keeps 10 mantissa bits, and the bf16x3 split accumulates with
// truncation) and are NOT the benchmarked path; `DinoUNet.precision = "fp32"` selects them.
// Layout: tokens [rows, C] / images NHWC fp32, same as the 16-bit engine.  Weights: [N, K] K-major fp32
// (conv: k = tap * Cpad + c), packed by ForwardEngine.pack with dtype float32.
#include <math.h>

#include "common.cuh"
#include "../../include/dinounet_b200.h"
#include "host_util.h"

namespace b2u {

__device__ __forceinline__ float f32_act(float v, int act) {
  if (act == B2U_ACT_GELU) return 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f));
  if (act == B2U_ACT_RELU) return fmaxf(v, 0.f);
  if (act == B2U_ACT_LRELU) return v > 0.f ? v : 0.01f * v;
  return v;
}

// ------------------------------------------------------------------------------------------------ GEMM / conv3x3
// acc[m, n] = sum_k A(m, k) * W'(n, k).  A(m, k): plain rows (optional batch row remap), transposed rows, or the 3x3 / pad 1
// window of an NHWC image; W'(n, k): plain [N, K] rows, transposed, the flipped 3x3 weights of the conv data gradient, or
// the 3x3 window of an image (conv weight gradient: k = output pixel).  Epilogue identical in meaning to b2u_epilogue.
// 128 x 128 tile, BK 8, 256 threads, 8 x 8 outputs per thread (two 4-wide groups 64 apart), k ascending (one fmaf chain
// per output: the accumulation order within a K slice does not depend on the tiling).
constexpr int FT = 128, FK = 8;

struct F32RowAddr {      // per-thread loader state for one row of the A / W' operand
  long long row;         // plain row index (after remap) or -1 when out of range
  int cb, cy, cx;        // conv: batch, output y, output x of the pixel this row / column stands for
};

__device__ __forceinline__ float f32_conv_window(const float* img, int Hin, int Win, int Cc, int stride, int cb, int cy, int cx, int tap,
                                                 int c) {
  const int dy = tap / 3, dx = tap - dy * 3;
  const int iy = cy * stride + dy - 1, ix = cx * stride + dx - 1;
  if (c < Cc && iy >= 0 && iy < Hin && ix >= 0 && ix < Win) return img[((static_cast<long long>(cb) * Hin + iy) * Win + ix) * Cc + c];
  return 0.f;
}

__global__ void __launch_bounds__(256) f32_gemm_kernel(const b2u_f32_gemm_params p) {
  __shared__ __align__(16) float sA[FK][FT + 4];
  __shared__ __align__(16) float sW[FK][FT + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const long long m0 = static_cast<long long>(blockIdx.x) * FT;   // rows on grid.x (up to 2^31 tiles: 64 x 512^2 pixels)
  const int n0 = blockIdx.y * FT;
  const float* A = p.A;
  const float* W = p.W;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  // loader: thread -> (tile row lr = tid / 2 (0..127), 4 consecutive k's lk = (tid & 1) * 4) of both operands
  const int lr = tid >> 1, lk = (tid & 1) * 4;
  const long long am = m0 + lr;
  const int wn = n0 + lr;
  const int stride = p.conv == B2U_CONV3X3_S2 ? 2 : 1;
  const int Ho = p.conv ? p.Hin / stride : 0, Wo = p.conv ? p.Win / stride : 0;
  int acb = 0, acy = 0, acx = 0;
  if (p.conv && p.w_mode != 3 && am < p.M) {                     // A side = conv window (forward / data gradient)
    acb = static_cast<int>(am / (static_cast<long long>(Ho) * Wo));
    const int r = static_cast<int>(am - static_cast<long long>(acb) * Ho * Wo);
    acy = r / Wo;
    acx = r - acy * Wo;
  }
  long long arow = am;
  if (!p.conv && p.a_rows_in > 0 && am < p.M) arow = (am / p.a_rows_in) * p.a_rows_out + p.a_row_off + am % p.a_rows_in;
  // w_mode 3: W'(n, k) = window(pixel k, tap = n / Cpad, c = n % Cpad)
  const int wtap = p.w_mode == 3 ? wn / p.Cpad : 0, wc = p.w_mode == 3 ? wn - wtap * p.Cpad : 0;
  // split-K (backward weight gradients: K = number of rows / pixels): slice blockIdx.z of the K range, atomic epilogue
  int k_lo = 0, k_hi = p.K;
  if (p.ksplit > 1) {
    const int per = ((p.K + p.ksplit - 1) / p.ksplit + FK - 1) / FK * FK;
    k_lo = blockIdx.z * per;
    k_hi = min(p.K, k_lo + per);
  }
  const bool a_vec = !p.conv && !p.a_trans && (p.lda & 3) == 0 && ((reinterpret_cast<uintptr_t>(A) & 15) == 0);
  const bool w_vec = p.w_mode == 0 && (p.ldw & 3) == 0 && ((reinterpret_cast<uintptr_t>(W) & 15) == 0);
  for (int k0 = k_lo; k0 < k_hi; k0 += FK) {
    float a4[4] = {0.f, 0.f, 0.f, 0.f}, w4[4] = {0.f, 0.f, 0.f, 0.f};
    const int kb = k0 + lk;
    if (am < p.M) {
      if (a_vec && kb + 3 < k_hi) {
        const float4 t = *reinterpret_cast<const float4*>(A + arow * p.lda + kb);
        a4[0] = t.x; a4[1] = t.y; a4[2] = t.z; a4[3] = t.w;
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int k = kb + e;
          if (k >= k_hi) break;
          if (p.a_trans) a4[e] = A[static_cast<long long>(k) * p.lda + am];            // A'(m, k) = A[k][m]
          else if (!p.conv || p.w_mode == 3) a4[e] = A[arow * p.lda + k];
          else {
            const int tap = k / p.Cpad, c = k - tap * p.Cpad;
            a4[e] = f32_conv_window(A, p.Hin, p.Win, p.C, stride, acb, acy, acx, tap, c);
          }
        }
      }
    }
    if (wn < p.N) {
      if (w_vec && kb + 3 < k_hi) {
        const float4 t = *reinterpret_cast<const float4*>(W + static_cast<long long>(wn) * p.ldw + kb);
        w4[0] = t.x; w4[1] = t.y; w4[2] = t.z; w4[3] = t.w;
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int k = kb + e;
          if (k >= k_hi) break;
          if (p.w_mode == 0) w4[e] = W[static_cast<long long>(wn) * p.ldw + k];
          else if (p.w_mode == 1) w4[e] = W[static_cast<long long>(k) * p.ldw + wn];   // W'(n, k) = W[k][n]
          else if (p.w_mode == 2) {
            // 3x3 data gradient: this call convolves dY (C = Cout channels) with W'(c, (tap', n)) = W[n][(8 - tap')*w_cpad + c]
            const int tap = k / p.Cpad, nn = k - tap * p.Cpad;
            if (nn < p.C) w4[e] = W[static_cast<long long>(nn) * p.ldw + (8 - tap) * p.w_cpad + wn];
          } else {
            // 3x3 weight gradient: k = output pixel of the image W (the layer input), window element (wtap, wc)
            const int cb = k / (Ho * Wo), r = k - cb * (Ho * Wo);
            const int cy = r / Wo, cx = r - cy * Wo;
            w4[e] = f32_conv_window(W, p.Hin, p.Win, p.C, stride, cb, cy, cx, wtap, wc);
          }
        }
      }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) { sA[lk + e][lr] = a4[e]; sW[lk + e][lr] = w4[e]; }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < FK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&sA[k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&sA[k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&sW[k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&sW[k][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float w[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const long long m = m0 + (i >> 2) * 64 + ty * 4 + (i & 3);
    if (m >= p.M) continue;
    long long orow = m;
    if (p.ps_cout > 0) {
      const long long hw = static_cast<long long>(p.ps_h) * p.ps_w;
      const long long pb = m / hw;
      const long long rem = m - pb * hw;
      const long long pi = rem / p.ps_w, pj = rem - pi * p.ps_w;
      orow = (pb * (2 * p.ps_h) + 2 * pi) * (2 * p.ps_w) + 2 * pj;
    } else if (p.rows_in > 0) {
      orow = (m / p.rows_in) * p.rows_out + p.row_off + m % p.rows_in;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = n0 + (j >> 2) * 64 + tx * 4 + (j & 3);
      if (n >= p.N) continue;
      long long r = orow;
      int oc = n;
      if (p.ps_cout > 0) {
        const int q = n / p.ps_cout;
        oc = n - q * p.ps_cout;
        r += static_cast<long long>(q >> 1) * (2 * p.ps_w) + (q & 1);
      }
      oc += p.col_off;
      float v = acc[i][j];
      if (p.bias) v += p.bias[n];
      v = f32_act(v, p.act1);
      if (p.scale) v *= p.scale[n];
      if (p.shift) v += p.shift[n];
      v = f32_act(v, p.act2);
      if (p.residual) v += p.residual[r * p.ldres + oc];
      if (p.ksplit > 1 || p.accumulate) atomicAdd(&p.out[r * p.ldc + oc], v);
      else p.out[r * p.ldc + oc] = v;
    }
  }
}

extern "C" int b2u_f32_gemm(const b2u_f32_gemm_params* p, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!p || !p->A || !p->W || !p->out) return set_error(-1, "b2u_f32_gemm: null pointer");
  if (p->M <= 0 || p->N <= 0 || p->K <= 0) return set_error(-1, "b2u_f32_gemm: bad shape");
  if (p->conv && p->w_mode != 3 && (p->Cpad < p->C || p->K != 9 * p->Cpad)) return set_error(-1, "b2u_f32_gemm: conv needs K = 9 * Cpad");
  if (p->w_mode == 3 && (!p->conv || p->N != 9 * p->Cpad)) return set_error(-1, "b2u_f32_gemm: conv weight gradient needs N = 9 * Cpad");
  if (p->ksplit > 1 && (p->bias || p->scale || p->shift || p->act1 || p->act2 || p->residual))
    return set_error(-1, "b2u_f32_gemm: split-K accumulates raw products only");
  dim3 grid(static_cast<unsigned>((p->M + FT - 1) / FT), (p->N + FT - 1) / FT, p->ksplit > 1 ? p->ksplit : 1);
  f32_gemm_kernel<<<grid, 256, 0, stream>>>(*p);
  return check_launch("f32_gemm");
}

// ------------------------------------------------------------------------------------------------ LayerNorm
// one warp per row; exact two-pass mean / variance; in row = (r / rows_out_per_b) * rows_in_per_b + in_off + r % rows_out_per_b
__global__ void f32_layernorm_kernel(const float* __restrict__ in, float* __restrict__ out, const float* __restrict__ w,
                                     const float* __restrict__ b, long long rows, int D, float eps, int in_per_b,
                                     int out_per_b, int in_off) {
  const long long r = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  long long ir = r;
  if (in_per_b > 0) ir = (r / out_per_b) * in_per_b + in_off + r % out_per_b;
  const float* x = in + ir * D;
  float s = 0.f;
  for (int c = lane; c < D; c += 32) s += x[c];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / D;
  float q = 0.f;
  for (int c = lane; c < D; c += 32) { const float d = x[c] - mean; q = fmaf(d, d, q); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = 1.0f / sqrtf(q / D + eps);
  float* y = out + r * D;
  for (int c = lane; c < D; c += 32) y[c] = (x[c] - mean) * rstd * w[c] + b[c];
}

extern "C" int b2u_f32_layernorm(const float* in, float* out, const float* w, const float* b, int64_t rows, int32_t D,
                                 float eps, int32_t in_per_b, int32_t out_per_b, int32_t in_off, b2u_stream_t stream_) {
  if (!in || !out || !w || !b) return set_error(-1, "b2u_f32_layernorm: null pointer");
  const long long threads = rows * 32;
  f32_layernorm_kernel<<<static_cast<unsigned>((threads + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream_)>>>(
      in, out, w, b, rows, D, eps, in_per_b, out_per_b, in_off);
  return check_launch("f32_layernorm");
}

// ------------------------------------------------------------------------------------------------ input reshapes
// x NCHW [B,3,S,S] -> patch rows [B*P, 768], k = c*256 + ky*16 + kx (== proj.weight.reshape(D, -1), patch_embed.py:64-76)
__global__ void f32_patchify_kernel(const float* __restrict__ x, float* __restrict__ out, int B, int S) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int h = S / 16;
  const long long total = static_cast<long long>(B) * h * h * 768;
  if (i >= total) return;
  const int k = static_cast<int>(i % 768);
  const long long pr = i / 768;
  const int px = static_cast<int>(pr % h), py = static_cast<int>((pr / h) % h), b = static_cast<int>(pr / (h * h));
  const int c = k >> 8, ky = (k >> 4) & 15, kx = k & 15;
  out[i] = x[((static_cast<long long>(b) * 3 + c) * S + py * 16 + ky) * S + px * 16 + kx];
}
__global__ void f32_nchw_to_nhwc_kernel(const float* __restrict__ x, float* __restrict__ out, int B, int Cc, long long HW) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= B * HW * Cc) return;
  const int c = static_cast<int>(i % Cc);
  const long long p = (i / Cc) % HW, b = i / (Cc * HW);
  out[i] = x[(b * Cc + c) * HW + p];
}
extern "C" int b2u_f32_patchify(const float* x, float* out, int32_t B, int32_t S, b2u_stream_t stream_) {
  const long long total = static_cast<long long>(B) * (S / 16) * (S / 16) * 768;
  f32_patchify_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream_)>>>(x, out, B, S);
  return check_launch("f32_patchify");
}
extern "C" int b2u_f32_nchw_to_nhwc(const float* x, float* out, int32_t B, int32_t Cc, int64_t HW, b2u_stream_t stream_) {
  const long long total = static_cast<long long>(B) * HW * Cc;
  f32_nchw_to_nhwc_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream_)>>>(x, out, B, Cc, HW);
  return check_launch("f32_nchw_to_nhwc");
}

// lin [B*HW, ncls] -> logits NCHW fp32 [B, ncls, HW] + first-maximum argmax labels (nnUNetTrainer.py:977)
__global__ void f32_seg_out_kernel(const float* __restrict__ lin, float* __restrict__ logits, uint8_t* __restrict__ labels,
                                   int B, long long HW, int ncls) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= B * HW) return;
  const long long b = i / HW, p = i - b * HW;
  float best = lin[i * ncls];
  int arg = 0;
  for (int c = 0; c < ncls; ++c) {
    const float v = lin[i * ncls + c];
    logits[(b * ncls + c) * HW + p] = v;
    if (v > best) { best = v; arg = c; }
  }
  labels[i] = static_cast<uint8_t>(arg);
}
extern "C" int b2u_f32_seg_out(const float* lin, float* logits, uint8_t* labels, int32_t B, int64_t HW, int32_t ncls,
                               b2u_stream_t stream_) {
  // labels are uint8: class 255 is the largest one they hold
  if (ncls < 1 || ncls > 256) return set_error(-1, "b2u_f32_seg_out: 1 <= ncls <= 256");
  const long long total = static_cast<long long>(B) * HW;
  f32_seg_out_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream_)>>>(lin, logits, labels, B, HW, ncls);
  return check_launch("f32_seg_out");
}

// ------------------------------------------------------------------------------------------------ pooling / depthwise
__global__ void f32_maxpool_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int H, int W, int Cc) {
  const int Ho = H / 2, Wo = W / 2;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * Ho * Wo * Cc;
  if (i >= total) return;
  const int c = static_cast<int>(i % Cc);
  const long long pr = i / Cc;
  const int x = static_cast<int>(pr % Wo), y = static_cast<int>((pr / Wo) % Ho), b = static_cast<int>(pr / (static_cast<long long>(Wo) * Ho));
  float m = -INFINITY;
  for (int dy = -1; dy <= 1; ++dy)
    for (int dx = -1; dx <= 1; ++dx) {
      const int iy = 2 * y + dy, ix = 2 * x + dx;
      if (iy >= 0 && iy < H && ix >= 0 && ix < W) m = fmaxf(m, in[((static_cast<long long>(b) * H + iy) * W + ix) * Cc + c]);
    }
  out[i] = m;
}
extern "C" int b2u_f32_maxpool3x3s2(const float* in, float* out, int32_t B, int32_t H, int32_t W, int32_t Cc, b2u_stream_t stream_) {
  const long long total = static_cast<long long>(B) * (H / 2) * (W / 2) * Cc;
  f32_maxpool_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream_)>>>(in, out, B, H, W, Cc);
  return check_launch("f32_maxpool");
}

// depthwise 3x3 / pad 1 + bias (+ GELU) on token-major planes.  planes == 1: one H x W image per batch item;
// planes == 3: the ConvFFN layout (dinov3_adapter.py:99-109): tokens [16n | 4n | n] = planes 2Hx2W, HxW, H/2xW/2.
__global__ void f32_dwconv_kernel(const float* __restrict__ in, float* __restrict__ out, const float* __restrict__ w9,
                                  const float* __restrict__ bias, int B, int H, int W, int Cc, int planes, int act) {
  const long long per_b = planes == 3 ? static_cast<long long>(H) * W * 21 / 4 : static_cast<long long>(H) * W;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= B * per_b * Cc) return;
  const int c = static_cast<int>(i % Cc);
  const long long t = (i / Cc) % per_b, b = i / (Cc * per_b);
  long long base = 0;
  int ph = H, pw = W;
  long long local = t;
  if (planes == 3) {
    const long long n16 = static_cast<long long>(H) * W * 4, n4 = static_cast<long long>(H) * W;
    if (t < n16) { ph = 2 * H; pw = 2 * W; }
    else if (t < n16 + n4) { base = n16; local = t - n16; }
    else { base = n16 + n4; local = t - n16 - n4; ph = H / 2; pw = W / 2; }
  }
  const int y = static_cast<int>(local / pw), x = static_cast<int>(local - static_cast<long long>(y) * pw);
  float acc = 0.f;
  for (int dy = 0; dy < 3; ++dy)
    for (int dx = 0; dx < 3; ++dx) {
      const int iy = y + dy - 1, ix = x + dx - 1;
      if (iy >= 0 && iy < ph && ix >= 0 && ix < pw)
        acc = fmaf(in[(b * per_b + base + static_cast<long long>(iy) * pw + ix) * Cc + c], w9[(dy * 3 + dx) * Cc + c], acc);
    }
  acc += bias[c];
  out[i] = f32_act(acc, act);
}
extern "C" int b2u_f32_dwconv3x3(const float* in, float* out, const float* w9, const float* bias, int32_t B, int32_t H,
                                 int32_t W, int32_t Cc, int32_t planes, int32_t act, b2u_stream_t stream_) {
  const long long per_b = planes == 3 ? static_cast<long long>(H) * W * 21 / 4 : static_cast<long long>(H) * W;
  const long long total = B * per_b * Cc;
  f32_dwconv_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream_)>>>(in, out, w9, bias, B, H, W, Cc, planes, act);
  return check_launch("f32_dwconv");
}

// ------------------------------------------------------------------------------------------------ attention (+ RoPE)
// qkv [B*N, 3D] (q | k | v, head-major inside each) -> out [B*N, D].  One block = 8 query rows of one (batch, head);
// rope (attention.py:16-27,66-85) is applied while loading q and k rows: x*cos + rotate_half(x)*sin on tokens >= prefix.
constexpr int FQ = 8;
__device__ __forceinline__ float f32_rope_elem(const float* row, int d, int hd, int tok, int prefix, const float* sin,
                                               const float* cos) {
  const float x = row[d];
  if (tok < prefix) return x;
  const int half = hd >> 1;
  const float other = d < half ? -row[d + half] : row[d - half];
  const long long t = static_cast<long long>(tok - prefix) * hd + d;
  return x * cos[t] + other * sin[t];
}
__global__ void __launch_bounds__(256) f32_attention_kernel(const float* __restrict__ qkv, const float* __restrict__ sin,
                                                            const float* __restrict__ cos, float* __restrict__ out, int N,
                                                            int heads, int hd, int prefix, float scale) {
  extern __shared__ float sm[];
  float* sq = sm;                         // [FQ][hd]
  float* sp = sq + FQ * hd;               // [FQ][N]
  float* red = sp + static_cast<size_t>(FQ) * N;   // [FQ][8]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int q0 = blockIdx.x * FQ, h = blockIdx.y, b = blockIdx.z;
  const int D = heads * hd;
  const int nq = min(FQ, N - q0);
  const float* base = qkv + static_cast<long long>(b) * N * 3 * D;
  for (int i = tid; i < nq * hd; i += 256) {
    const int r = i / hd, d = i - r * hd;
    sq[i] = f32_rope_elem(base + static_cast<long long>(q0 + r) * 3 * D + h * hd, d, hd, q0 + r, prefix, sin, cos);
  }
  __syncthreads();
  // scores: one warp per key, lanes over head dims
  for (int key = warp; key < N; key += 8) {
    const float* krow = base + static_cast<long long>(key) * 3 * D + D + h * hd;
    float kv[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) kv[e] = (lane + 32 * e) < hd ? f32_rope_elem(krow, lane + 32 * e, hd, key, prefix, sin, cos) : 0.f;
    for (int r = 0; r < nq; ++r) {
      float s = 0.f;
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (lane + 32 * e < hd) s = fmaf(sq[r * hd + lane + 32 * e], kv[e], s);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) sp[static_cast<size_t>(r) * N + key] = s * scale;
    }
  }
  __syncthreads();
  // exact softmax per row: warp r handles row r
  if (warp < nq) {
    float* prow = sp + static_cast<size_t>(warp) * N;
    float mx = -INFINITY;
    for (int k = lane; k < N; k += 32) mx = fmaxf(mx, prow[k]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float s = 0.f;
    for (int k = lane; k < N; k += 32) { const float e = expf(prow[k] - mx); prow[k] = e; s += e; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) red[warp] = s;
  }
  __syncthreads();
  // out[r][d] = sum_k p[r][k] v[k][d] / l[r]
  for (int i = tid; i < nq * hd; i += 256) {
    const int r = i / hd, d = i - r * hd;
    const float* prow = sp + static_cast<size_t>(r) * N;
    const float* vcol = base + 2 * D + h * hd + d;
    float acc = 0.f;
    for (int k = 0; k < N; ++k) acc = fmaf(prow[k], vcol[static_cast<long long>(k) * 3 * D], acc);
    out[(static_cast<long long>(b) * N + q0 + r) * D + h * hd + d] = acc / red[r];
  }
}
extern "C" int b2u_f32_attention(const float* qkv, const float* sin, const float* cos, float* out, int32_t B, int32_t N,
                                 int32_t heads, int32_t hd, int32_t prefix, float scale, b2u_stream_t stream_) {
  if (hd > 128) return set_error(-1, "b2u_f32_attention: head_dim <= 128");
  const size_t smem = (static_cast<size_t>(FQ) * hd + static_cast<size_t>(FQ) * N + FQ * 8) * sizeof(float);
  if (smem > 200 * 1024) return set_error(-1, "b2u_f32_attention: too many tokens for the shared-memory score rows");
  static bool configured_dev[64] = {};
  bool& configured = configured_dev[current_device_index()];
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(f32_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) return set_error(-2, "cudaFuncSetAttribute(f32_attention): %s", cudaGetErrorString(e));
    configured = true;
  }
  dim3 grid((N + FQ - 1) / FQ, heads, B);
  f32_attention_kernel<<<grid, 256, smem, static_cast<cudaStream_t>(stream_)>>>(qkv, sin, cos, out, N, heads, hd, prefix, scale);
  return check_launch("f32_attention");
}

// ------------------------------------------------------------------------------------------------ MSDA (fused prologue)
// value [B, Hv*Wv, heads, dh], offaw [B*Lq, heads*8 + heads*4] (offsets | attention logits) -> out [B*Lq, heads*dh].
// Lq = 21 * Hv*Wv / 4 queries = cell centres of the (2Hv x 2Wv), (Hv x Wv), (Hv/2 x Wv/2) grids (dinov3_adapter.py:40-70);
// loc = ref + off / (Wv, Hv) (ms_deform_attn.py:193-197); weights = softmax over the 4 points; bilinear, zero padding,
// align_corners = False (ms_deform_im2col_cuda.cuh:242-304).
__global__ void f32_msda_kernel(const float* __restrict__ value, const float* __restrict__ offaw, float* __restrict__ out,
                                int B, int Hv, int Wv, int heads, int dh) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int HW = Hv * Wv;
  const long long Lq = static_cast<long long>(HW) * 21 / 4;
  const long long total = B * Lq * heads * dh;
  if (i >= total) return;
  const int c = static_cast<int>(i % dh);
  const int m = static_cast<int>((i / dh) % heads);
  const long long bq = i / (static_cast<long long>(dh) * heads);
  const long long q = bq % Lq, b = bq / Lq;
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
#pragma unroll
  for (int p = 0; p < 4; ++p) { e[p] = expf(a[p] - mx); s += e[p]; }
  const float* vb = value + (b * HW) * heads * dh + m * dh + c;
  const long long rs = static_cast<long long>(heads) * dh;
  float acc = 0.f;
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const float lx = refx + o[2 * p] / Wv, ly = refy + o[2 * p + 1] / Hv;
    const float px = lx * Wv - 0.5f, py = ly * Hv - 0.5f;
    if (py > -1 && px > -1 && py < Hv && px < Wv) {
      const float fx = floorf(px), fy = floorf(py);
      const int x0 = static_cast<int>(fx), y0 = static_cast<int>(fy);
      const float ax = px - fx, ay = py - fy;
      float v = 0.f;
      if (y0 >= 0 && x0 >= 0) v += (1.f - ay) * (1.f - ax) * vb[static_cast<long long>(y0 * Wv + x0) * rs];
      if (y0 >= 0 && x0 + 1 < Wv) v += (1.f - ay) * ax * vb[static_cast<long long>(y0 * Wv + x0 + 1) * rs];
      if (y0 + 1 < Hv && x0 >= 0) v += ay * (1.f - ax) * vb[static_cast<long long>((y0 + 1) * Wv + x0) * rs];
      if (y0 + 1 < Hv && x0 + 1 < Wv) v += ay * ax * vb[static_cast<long long>((y0 + 1) * Wv + x0 + 1) * rs];
      acc += (e[p] / s) * v;
    }
  }
  out[i] = acc;
}
extern "C" int b2u_f32_msda(const float* value, const float* offaw, float* out, int32_t B, int32_t Hv, int32_t Wv,
                            int32_t heads, int32_t dh, b2u_stream_t stream_) {
  const long long total = static_cast<long long>(B) * (static_cast<long long>(Hv) * Wv * 21 / 4) * heads * dh;
  f32_msda_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream_)>>>(value, offaw, out, B, Hv, Wv, heads, dh);
  return check_launch("f32_msda");
}

// ------------------------------------------------------------------------------------------------ InstanceNorm / SE / FiLM
// per-(n, c) mean and biased variance over HW rows (fp64 accumulation, two passes: mean first, then centred squares), then
// y = (x-mean)*rstd*w + b (+ LeakyReLU).  The rows of one image are split over gridDim.z blocks (a 512^2 image with 32
// channels would otherwise be ONE block): partial sums meet in fp64 atomics on work[2][B][C]; stats[B][C][2] = (mean, rstd)
// is also what the backward needs.
__global__ void __launch_bounds__(256) f32_in_sum_kernel(const float* __restrict__ x, long long ld, long long HW, int Cc, int pass,
                                                         double* __restrict__ work, int B) {
  __shared__ double red[8][33];
  const int cx = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  const long long b = blockIdx.y;
  const long long per = (HW + gridDim.z - 1) / gridDim.z;
  const long long lo = blockIdx.z * per, hi = lo + per < HW ? lo + per : HW;
  const float* xb = x + b * HW * ld;
  double s = 0.0;
  if (c < Cc) {
    if (pass == 0) {
      for (long long r = lo + rg; r < hi; r += 8) s += xb[r * ld + c];
    } else {
      const double mean = work[b * Cc + c] / static_cast<double>(HW);
      for (long long r = lo + rg; r < hi; r += 8) { const double d = static_cast<double>(xb[r * ld + c]) - mean; s += d * d; }
    }
  }
  red[rg][cx] = s;
  __syncthreads();
  if (rg == 0 && c < Cc) {
    double t = 0.0;
    for (int k = 0; k < 8; ++k) t += red[k][cx];
    atomicAdd(&work[(static_cast<long long>(pass) * B + b) * Cc + c], t);
  }
}
__global__ void f32_in_finish_kernel(const double* __restrict__ work, float* __restrict__ stats, int B, int Cc, long long HW, float eps) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * Cc) return;
  stats[2 * i] = static_cast<float>(work[i] / static_cast<double>(HW));
  stats[2 * i + 1] = 1.0f / sqrtf(static_cast<float>(work[static_cast<long long>(B) * Cc + i] / static_cast<double>(HW)) + eps);
}
__global__ void f32_in_apply_kernel(const float* __restrict__ x, long long ldx, float* __restrict__ out, long long ldo,
                                    const float* __restrict__ stats, const float* __restrict__ w, const float* __restrict__ bb, int B,
                                    long long HW, int Cc, int lrelu) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= B * HW * Cc) return;
  const int c = static_cast<int>(i % Cc);
  const long long r = i / Cc, b = r / HW;
  const float mean = stats[2 * (b * Cc + c)], rstd = stats[2 * (b * Cc + c) + 1];
  float v = (x[r * ldx + c] - mean) * rstd * w[c] + bb[c];
  if (lrelu) v = v > 0.f ? v : 0.01f * v;
  out[r * ldo + c] = v;
}
static int in_splits(long long HW) { return static_cast<int>(HW >= 65536 ? 32 : (HW >= 4096 ? 8 : 1)); }

extern "C" int b2u_f32_instnorm(const float* in, int64_t ld_in, float* out, int64_t ld_out, const float* w, const float* b,
                                double* work, float* stats, int32_t B, int64_t HW, int32_t Cc, float eps, int32_t lrelu,
                                b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!in || !out || !w || !b || !work || !stats) return set_error(-1, "b2u_f32_instnorm: null pointer");
  cudaError_t e = cudaMemsetAsync(work, 0, sizeof(double) * 2 * B * Cc, stream);
  if (e != cudaSuccess) return set_error(-2, "b2u_f32_instnorm: memset: %s", cudaGetErrorString(e));
  dim3 grid((Cc + 31) / 32, B, in_splits(HW));
  f32_in_sum_kernel<<<grid, 256, 0, stream>>>(in, ld_in, HW, Cc, 0, work, B);
  f32_in_sum_kernel<<<grid, 256, 0, stream>>>(in, ld_in, HW, Cc, 1, work, B);
  f32_in_finish_kernel<<<(B * Cc + 255) / 256, 256, 0, stream>>>(work, stats, B, Cc, HW, eps);
  const long long total = static_cast<long long>(B) * HW * Cc;
  f32_in_apply_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(in, ld_in, out, ld_out, stats, w, b, B, HW, Cc, lrelu);
  return check_launch("f32_instnorm");
}

// SqueezeExcitation + shortcut (dinounet_training.py:222-225, 438-441): out = t * sigmoid(W2 relu(W1 mean_hw(t) + b1) + b2) + sc
// kernel 1: pooled[b, c] = mean over HW (fp64); kernel 2: per block recompute the gate of its batch item, then apply.
__global__ void __launch_bounds__(256) f32_colmean_kernel(const float* __restrict__ in, float* __restrict__ pooled, long long HW, int Cc) {
  __shared__ double red[8][33];
  const int cx = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  const long long b = blockIdx.y;
  double s = 0.0;
  if (c < Cc)
    for (long long r = rg; r < HW; r += 8) s += in[(b * HW + r) * Cc + c];
  red[rg][cx] = s;
  __syncthreads();
  if (rg == 0 && c < Cc) {
    double t = 0.0;
    for (int k = 0; k < 8; ++k) t += red[k][cx];
    pooled[b * Cc + c] = static_cast<float>(t / HW);
  }
}
__global__ void __launch_bounds__(256) f32_se_apply_kernel(const float* __restrict__ t, const float* __restrict__ sc, long long ldsc,
                                                           const float* __restrict__ pooled, const float* __restrict__ w1,
                                                           const float* __restrict__ b1, const float* __restrict__ w2,
                                                           const float* __restrict__ b2, float* __restrict__ out, long long HW,
                                                           int Cc, int hid) {
  __shared__ float s_h[64], s_gate[256];
  const long long b = blockIdx.y;
  for (int j = threadIdx.x; j < hid; j += 256) {
    float a = b1[j];
    for (int c = 0; c < Cc; ++c) a = fmaf(w1[j * Cc + c], pooled[b * Cc + c], a);
    s_h[j] = fmaxf(a, 0.f);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < Cc; c += 256) {
    float a = b2[c];
    for (int j = 0; j < hid; ++j) a = fmaf(w2[c * hid + j], s_h[j], a);
    s_gate[c] = 1.0f / (1.0f + expf(-a));
  }
  __syncthreads();
  const long long per_block = (HW * Cc + gridDim.x - 1) / gridDim.x;
  const long long lo = blockIdx.x * per_block;
  const long long hi = lo + per_block < HW * Cc ? lo + per_block : HW * Cc;
  for (long long i = lo + threadIdx.x; i < hi; i += 256) {
    const int c = static_cast<int>(i % Cc);
    const long long r = i / Cc;
    out[(b * HW) * Cc + i] = t[(b * HW) * Cc + i] * s_gate[c] + sc[(b * HW + r) * ldsc + c];
  }
}
extern "C" int b2u_f32_se(const float* t, const float* sc, int64_t ldsc, float* pooled, const float* w1, const float* b1,
                          const float* w2, const float* b2, float* out, int32_t B, int64_t HW, int32_t Cc, int32_t hid,
                          b2u_stream_t stream_) {
  if (Cc > 256 || hid > 64) return set_error(-1, "b2u_f32_se: at most 256 channels / 64 hidden");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  f32_colmean_kernel<<<dim3((Cc + 31) / 32, B), 256, 0, stream>>>(t, pooled, HW, Cc);
  int rc = check_launch("f32_colmean");
  if (rc) return rc;
  long long nb = (static_cast<long long>(HW) * Cc + 4095) / 4096;
  const int bx = static_cast<int>(nb > 1024 ? 1024 : (nb < 1 ? 1 : nb));
  f32_se_apply_kernel<<<dim3(bx, B), 256, 0, stream>>>(t, sc, ldsc, pooled, w1, b1, w2, b2, out, HW, Cc, hid);
  return check_launch("f32_se_apply");
}

// FiLM (dinounet_training.py:430-432): z = gamma * zp + beta; gb [px, 2R] = (gamma | beta), zz [px, 2R] = (zs | zp)
__global__ void f32_film_kernel(const float* __restrict__ gb, const float* __restrict__ zz, float* __restrict__ z, long long px, int R) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= px * R) return;
  const long long r = i / R;
  const int c = static_cast<int>(i - r * R);
  z[i] = gb[r * 2 * R + c] * zz[r * 2 * R + R + c] + gb[r * 2 * R + R + c];
}
extern "C" int b2u_f32_film(const float* gb, const float* zz, float* z, int64_t px, int32_t R, b2u_stream_t stream_) {
  f32_film_kernel<<<static_cast<unsigned>((px * R + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream_)>>>(gb, zz, z, px, R);
  return check_launch("f32_film");
}

// ------------------------------------------------------------------------------------------------ adapter tail
// out[b, y, x, :] = (c[b, y, x, :] + bilinear(tap[b])(y, x, :)) * sc + sh   (dinov3_adapter.py:468-482: F.interpolate
// bilinear align_corners=False of the [h x w] ViT tap to [r x r], add, eval-mode SyncBatchNorm folded into sc/sh).
// c rows: b * c_rows_per_b + c_off + y * r + x (a slice of the query stream, or a dense [B*r*r, D] buffer).
__global__ void f32_tail_kernel(const float* __restrict__ cs, long long c_per_b, long long c_off, const float* __restrict__ tap,
                                float* __restrict__ out, const float* __restrict__ sc, const float* __restrict__ sh, int B,
                                int r, int h, int D) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * r * r * D;
  if (i >= total) return;
  const int c = static_cast<int>(i % D);
  const long long pr = i / D;
  const int x = static_cast<int>(pr % r), y = static_cast<int>((pr / r) % r);
  const long long b = pr / (static_cast<long long>(r) * r);
  const float scale = static_cast<float>(h) / r;      // area_pixel_compute_scale(in, out, align_corners=False)
  float sy = scale * (y + 0.5f) - 0.5f, sx = scale * (x + 0.5f) - 0.5f;
  if (sy < 0.f) sy = 0.f;
  if (sx < 0.f) sx = 0.f;
  const int y0 = static_cast<int>(sy), x0 = static_cast<int>(sx);
  const int y1 = y0 + (y0 < h - 1 ? 1 : 0), x1 = x0 + (x0 < h - 1 ? 1 : 0);
  const float ly = sy - y0, lx = sx - x0;
  const float* t = tap + b * h * h * D + c;
  const float v = (1.f - ly) * ((1.f - lx) * t[static_cast<long long>(y0 * h + x0) * D] + lx * t[static_cast<long long>(y0 * h + x1) * D]) +
                  ly * ((1.f - lx) * t[static_cast<long long>(y1 * h + x0) * D] + lx * t[static_cast<long long>(y1 * h + x1) * D]);
  const float cv = cs[(b * c_per_b + c_off + static_cast<long long>(y) * r + x) * D + c];
  out[i] = (cv + v) * sc[c] + sh[c];
}
extern "C" int b2u_f32_tail(const float* cs, int64_t c_rows_per_b, int64_t c_off, const float* tap, float* out,
                            const float* sc, const float* sh, int32_t B, int32_t r, int32_t h, int32_t D, b2u_stream_t stream_) {
  const long long total = static_cast<long long>(B) * r * r * D;
  f32_tail_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream_)>>>(cs, c_rows_per_b, c_off, tap, out, sc, sh, B, r, h, D);
  return check_launch("f32_tail");
}

}  // namespace b2u
