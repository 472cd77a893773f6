// Addressing of the TF32 wgmma GEMM (gemm_tf32.cu), as host/device inline functions: which operand element every
// loader thread fetches in every mode of b2u_f32_gemm_params, where it lands in the 128B-swizzled k-block tile, how the
// K range is sliced, and where an accumulator element goes in the epilogue.  The kernel is the composition of these
// functions with the wgmma plumbing; tests/test_tf32_gemm_hostsim_cpu.py compiles the SAME functions for the
// host (csrc/gemm_tf32_hostsim.cpp: a software model of the 256 threads of a CTA + the SWIZZLE_128B K-major read-out of
// the MMA) and checks every mode against torch without a GPU.
#pragma once
#include <math.h>
#include <stdint.h>
#include <vector_functions.h>
#include <vector_types.h>

#include "../../include/dinounet_b200.h"

#if defined(__CUDACC__)
#define TF_HD __host__ __device__ __forceinline__
#else
#define TF_HD inline
#endif
#if defined(__CUDA_ARCH__)
#define TF_LDG(ptr) __ldg(ptr)
#else
#define TF_LDG(ptr) (*(ptr))
#endif

namespace b2u {
namespace tf32 {

constexpr int kTM = 128;      // UMMA M: rows of an output tile
constexpr int kTK = 32;       // k-block: 32 fp32 = one 128-byte swizzle row
constexpr int kTStages = 3;
constexpr int kTThreads = 256;

enum { kAPlain = 0, kATrans = 1, kAWindow = 2 };

struct Row {              // what one loader thread knows about "its" operand row for the whole CTA
  bool ok;                // row inside the matrix
  long long idx;          // A: m (transposed mode) / remapped row (plain); W: n
  int cb, cy, cx;         // A window mode: output pixel of this row
  int tap, c;             // W window mode (w_mode 3): window element of this row
};

// Loader role of one thread, per operand one of two shapes:
//   row mode   (operand contiguous along K, or no alignment guarantees): ONE tile row, a run of 16-byte chunks of it
//              (A: row tid / 2, 4 chunks; W: BN / 32 chunks) - each chunk is 4 consecutive k's, one LDG.128 where allowed;
//   block mode (operand contiguous along its ROW index: A[k][m], W[k][n], the flipped 3x3 weights, the pixel-indexed window
//              of a weight gradient): a 4 x 4 block = 4 consecutive rows x one chunk, fetched as four LDG.128 ALONG THE ROWS
//              (one per k) and transposed in registers into the four 16-byte chunks the K-major tile wants.  Row mode needs
//              16 scalar loads with 16 address computations for the same 16 elements, integer work that bounds the
//              weight-gradient GEMMs.
struct Roles {
  int amode, stride, Ho, Wo;
  bool a_blk, w_blk;
  int a_r, a_c0;          // row mode: row tid / 2, chunks a_c0 .. a_c0 + 3; block mode: first row 4 * (tid / 8), chunk tid % 8
  int w_r, w_c0, w_n;     // row mode: BN / 32 = w_n chunks of one row; block mode: first row, chunk, w_n = 4 loads (0: idle thread)
  Row ar, wr;             // block mode: the FIRST row of the group
  bool a_vec, w_vec;      // row mode: 16-byte global loads allowed (K-contiguous, aligned base and leading dimension)
};

// byte offset of 16-byte chunk `chunk` (0..7) of row `row` inside a K-major SWIZZLE_128B tile whose base is 1024-aligned
TF_HD uint32_t smem_off(int row, int chunk) { return static_cast<uint32_t>(row) * 128u + (static_cast<uint32_t>(chunk ^ (row & 7)) << 4); }

// output tile of linear block index `tile` (grid.x): the n tiles of one row tile are NEIGHBOURS in launch order, so the CTAs
// that share an A row tile run together and A streams from HBM once (the other order re-read A once per n tile: measured
// 1.65 TB/s of DRAM traffic on the 768-wide linears); W' (weights, or the small dy^T / x slices of a weight gradient) is
// L2-resident either way
TF_HD void tile_origin(const b2u_f32_gemm_params& p, int BN, long long tile, long long& m0, int& n0) {
  const int n_tiles = (p.N + BN - 1) / BN;
  m0 = (tile / n_tiles) * kTM;
  n0 = static_cast<int>(tile % n_tiles) * BN;
}

// K slice [k_lo, k_hi) of grid.z index z: whole k-blocks, so every chunk of four k's stays 16-byte aligned; may be empty
TF_HD void k_slice(const b2u_f32_gemm_params& p, int z, int& k_lo, int& k_hi) {
  k_lo = 0;
  k_hi = p.K;
  if (p.ksplit > 1) {
    const int per = ((p.K + p.ksplit - 1) / p.ksplit + kTK - 1) / kTK * kTK;
    const long long lo = static_cast<long long>(z) * per;
    k_lo = lo < p.K ? static_cast<int>(lo) : p.K;
    k_hi = (lo + per) < p.K ? static_cast<int>(lo + per) : p.K;
  }
}

TF_HD float act(float v, int a) {
  if (a == B2U_ACT_GELU) return 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f));
  if (a == B2U_ACT_RELU) return fmaxf(v, 0.f);
  if (a == B2U_ACT_LRELU) return v > 0.f ? v : 0.01f * v;
  return v;
}

// element (tap, c) of the 3x3 / pad 1 window of output pixel (cb, cy, cx) of an NHWC image with Cc channels
TF_HD float window(const float* img, int Hin, int Win, int Cc, int stride, int cb, int cy, int cx, int tap, int c) {
  const int dy = tap / 3, dx = tap - dy * 3;
  const int iy = cy * stride + dy - 1, ix = cx * stride + dx - 1;
  if (c < Cc && iy >= 0 && iy < Hin && ix >= 0 && ix < Win) return TF_LDG(img + ((static_cast<long long>(cb) * Hin + iy) * Win + ix) * Cc + c);
  return 0.f;
}

// Which staging shape each operand gets.  Block mode needs the row-contiguous addressing AND 16-byte alignment of every row
// group; it is used for the CONVOLUTION gradients only (weight gradient: both operands; data gradient: the flipped weights):
// block mode replaces 16 scalar loads and address computations per 4 x 4 block by four 16-byte loads, which is what the
// 3x3 weight and data gradients are bound by; the plain linears' transposed operands are small, L2-resident weight / dy^T
// slices, for which scalar row-mode loads are kept.
TF_HD void pick_modes(const b2u_f32_gemm_params& p, bool& a_blk, bool& w_blk) {
  const bool a_al = (reinterpret_cast<uintptr_t>(p.A) & 15) == 0, w_al = (reinterpret_cast<uintptr_t>(p.W) & 15) == 0;
  w_blk = p.conv != 0 && w_al &&
          ((p.w_mode == 2 && (p.ldw & 3) == 0 && (p.w_cpad & 3) == 0 && (p.N & 3) == 0) || (p.w_mode == 3 && (p.Cpad & 3) == 0 && (p.C & 3) == 0));
  a_blk = w_blk && p.a_trans && a_al && (p.lda & 3) == 0 && (p.M & 3) == 0;
}

TF_HD Roles make_roles(const b2u_f32_gemm_params& p, int tid, long long m0, int n0, int BN, bool a_blk, bool w_blk) {
  Roles r;
  r.stride = p.conv == B2U_CONV3X3_S2 ? 2 : 1;
  r.Ho = p.conv ? p.Hin / r.stride : 0;
  r.Wo = p.conv ? p.Win / r.stride : 0;
  r.amode = p.a_trans ? kATrans : ((!p.conv || p.w_mode == 3) ? kAPlain : kAWindow);
  const bool a_al = (reinterpret_cast<uintptr_t>(p.A) & 15) == 0, w_al = (reinterpret_cast<uintptr_t>(p.W) & 15) == 0;
  r.a_blk = a_blk;
  r.w_blk = w_blk;
  // ---- A operand
  // block mode: chunk = tid % 8, row group = tid / 8: the 8 lanes of a shared-memory store phase hold the 8 chunks of ONE row,
  // which the swizzle spreads over all 32 banks (conflict-free STS.128); a warp-wide load covers 16 consecutive rows (64
  // contiguous bytes) at 8 different k
  if (a_blk) { r.a_r = 4 * (tid >> 3); r.a_c0 = tid & 7; }
  else { r.a_r = tid >> 1; r.a_c0 = (tid & 1) * 4; }
  const long long am = m0 + r.a_r;
  r.ar.ok = am < p.M;
  r.ar.idx = am;
  r.ar.cb = r.ar.cy = r.ar.cx = r.ar.tap = r.ar.c = 0;
  if (r.ar.ok && r.amode == kAWindow) {
    const long long hw = static_cast<long long>(r.Ho) * r.Wo;
    r.ar.cb = static_cast<int>(am / hw);
    const int rem = static_cast<int>(am - static_cast<long long>(r.ar.cb) * hw);
    r.ar.cy = rem / r.Wo;
    r.ar.cx = rem - r.ar.cy * r.Wo;
  }
  if (r.ar.ok && r.amode == kAPlain && p.a_rows_in > 0) r.ar.idx = (am / p.a_rows_in) * p.a_rows_out + p.a_row_off + am % p.a_rows_in;
  // ---- W operand
  if (w_blk) {
    r.w_r = 4 * (tid >> 3);                          // BN / 4 row groups x 8 chunks = 2 * BN block slots, the other threads idle
    r.w_c0 = tid & 7;
    r.w_n = (tid >> 3) < BN / 4 ? 4 : 0;
  } else {
    r.w_n = BN / 32;
    r.w_r = (tid * r.w_n) >> 3;
    r.w_c0 = (tid * r.w_n) & 7;
  }
  const int wn = n0 + r.w_r;
  r.wr.ok = wn < p.N;
  r.wr.idx = wn;
  r.wr.cb = r.wr.cy = r.wr.cx = 0;
  r.wr.tap = 0;
  r.wr.c = 0;
  if (p.w_mode == 3) { r.wr.tap = wn / p.Cpad; r.wr.c = wn - r.wr.tap * p.Cpad; }
  r.a_vec = r.amode == kAPlain ? ((p.lda & 3) == 0 && a_al) : (r.amode == kAWindow && (p.C & 3) == 0 && a_al);
  r.w_vec = p.w_mode == 0 && (p.ldw & 3) == 0 && w_al;
  return r;
}

// four consecutive k's (k % 4 == 0) of this thread's row of A'
TF_HD float4 load_a(const b2u_f32_gemm_params& p, const Roles& R, int k, int k_hi) {
  const Row& r = R.ar;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!r.ok || k >= k_hi) return v;
  if (R.amode == kAPlain) {
    const float* src = p.A + r.idx * p.lda + k;
    if (R.a_vec && k + 3 < k_hi) return TF_LDG(reinterpret_cast<const float4*>(src));
    v.x = TF_LDG(src);
    if (k + 1 < k_hi) v.y = TF_LDG(src + 1);
    if (k + 2 < k_hi) v.z = TF_LDG(src + 2);
    if (k + 3 < k_hi) v.w = TF_LDG(src + 3);
  } else if (R.amode == kATrans) {
    const float* src = p.A + static_cast<long long>(k) * p.lda + r.idx;    // A'(m, k) = A[k][m]
    v.x = TF_LDG(src);
    if (k + 1 < k_hi) v.y = TF_LDG(src + p.lda);
    if (k + 2 < k_hi) v.z = TF_LDG(src + 2 * p.lda);
    if (k + 3 < k_hi) v.w = TF_LDG(src + 3 * p.lda);
  } else if ((p.Cpad & 3) == 0) {                 // window; the four k's share one tap
    const int tap = k / p.Cpad, c = k - tap * p.Cpad;
    const int dy = tap / 3, dx = tap - dy * 3;
    const int iy = r.cy * R.stride + dy - 1, ix = r.cx * R.stride + dx - 1;
    if (iy >= 0 && iy < p.Hin && ix >= 0 && ix < p.Win) {
      const float* src = p.A + ((static_cast<long long>(r.cb) * p.Hin + iy) * p.Win + ix) * p.C + c;
      if (R.a_vec && c + 3 < p.C && k + 3 < k_hi) return TF_LDG(reinterpret_cast<const float4*>(src));
      if (c < p.C) v.x = TF_LDG(src);
      if (c + 1 < p.C && k + 1 < k_hi) v.y = TF_LDG(src + 1);
      if (c + 2 < p.C && k + 2 < k_hi) v.z = TF_LDG(src + 2);
      if (c + 3 < p.C && k + 3 < k_hi) v.w = TF_LDG(src + 3);
    }
  } else {
    float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int kk = k + e;
      if (kk < k_hi) {
        const int tap = kk / p.Cpad;
        t[e] = window(p.A, p.Hin, p.Win, p.C, R.stride, r.cb, r.cy, r.cx, tap, kk - tap * p.Cpad);
      }
    }
    v = make_float4(t[0], t[1], t[2], t[3]);
  }
  return v;
}

// four consecutive k's of this thread's row (= output column n) of W'
TF_HD float4 load_w(const b2u_f32_gemm_params& p, const Roles& R, int k, int k_hi) {
  const Row& r = R.wr;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!r.ok || k >= k_hi) return v;
  if (p.w_mode == 0) {
    const float* src = p.W + r.idx * p.ldw + k;
    if (R.w_vec && k + 3 < k_hi) return TF_LDG(reinterpret_cast<const float4*>(src));
    v.x = TF_LDG(src);
    if (k + 1 < k_hi) v.y = TF_LDG(src + 1);
    if (k + 2 < k_hi) v.z = TF_LDG(src + 2);
    if (k + 3 < k_hi) v.w = TF_LDG(src + 3);
  } else if (p.w_mode == 1) {
    const float* src = p.W + static_cast<long long>(k) * p.ldw + r.idx;    // W'(n, k) = W[k][n]
    v.x = TF_LDG(src);
    if (k + 1 < k_hi) v.y = TF_LDG(src + p.ldw);
    if (k + 2 < k_hi) v.z = TF_LDG(src + 2 * p.ldw);
    if (k + 3 < k_hi) v.w = TF_LDG(src + 3 * p.ldw);
  } else if (p.w_mode == 2) {
    // 3x3 data gradient: W'(c, (tap', n)) = W[n][(8 - tap') * w_cpad + c]; here r.idx = c and k = tap' * Cpad + n
    float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int kk = k + e;
      if (kk < k_hi) {
        const int tap = kk / p.Cpad, nn = kk - tap * p.Cpad;
        if (nn < p.C) t[e] = TF_LDG(p.W + static_cast<long long>(nn) * p.ldw + (8 - tap) * p.w_cpad + r.idx);
      }
    }
    v = make_float4(t[0], t[1], t[2], t[3]);
  } else {
    // 3x3 weight gradient: k = output pixel of the image W (the layer input), this row = window element (r.tap, r.c)
    const int hw = R.Ho * R.Wo;
    int cb = k / hw;
    const int rem = k - cb * hw;
    int cy = rem / R.Wo, cx = rem - cy * R.Wo;
    float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (k + e < k_hi) t[e] = window(p.W, p.Hin, p.Win, p.C, R.stride, cb, cy, cx, r.tap, r.c);
      if (++cx == R.Wo) { cx = 0; if (++cy == R.Ho) { cy = 0; ++cb; } }
    }
    v = make_float4(t[0], t[1], t[2], t[3]);
  }
  return v;
}

TF_HD float4 ldg4(const float* src) { return TF_LDG(reinterpret_cast<const float4*>(src)); }

// this thread's share of the A' k-block that starts at kbase, as up to four float4:
//   row mode: v[j] = chunk a_c0 + j of the thread's row (four consecutive k's);
//   block mode: v[i] = rows a_r .. a_r + 3 at k = kbase + 4 * a_c0 + i (four consecutive ROWS: the memory-contiguous direction)
template <bool BLK> TF_HD void fetch_a(const b2u_f32_gemm_params& p, const Roles& R, int kbase, int k_hi, float4 (&v)[4]) {
  if constexpr (!BLK) {
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = load_a(p, R, kbase + (R.a_c0 + j) * 4, k_hi);
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int k = kbase + R.a_c0 * 4 + i;
      v[i] = (R.ar.ok && k < k_hi) ? ldg4(p.A + static_cast<long long>(k) * p.lda + R.ar.idx) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}

// WN: float4 per thread in row mode (BN / 32, a compile-time constant in the kernel)
template <bool BLK, int WN> TF_HD void fetch_w(const b2u_f32_gemm_params& p, const Roles& R, int kbase, int k_hi, float4 (&v)[4]) {
  if constexpr (!BLK) {
#pragma unroll
    for (int j = 0; j < WN; ++j) v[j] = load_w(p, R, kbase + (R.w_c0 + j) * 4, k_hi);
    return;
  }
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = zero;
  if (R.w_n == 0 || !R.wr.ok) return;
  const int k0 = kbase + R.w_c0 * 4;
  if (p.w_mode == 1) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (k0 + i < k_hi) v[i] = ldg4(p.W + static_cast<long long>(k0 + i) * p.ldw + R.wr.idx);          // W'(n, k) = W[k][n]
  } else if (p.w_mode == 2) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int kk = k0 + i;
      if (kk < k_hi) {
        const int tap = kk / p.Cpad, nn = kk - tap * p.Cpad;                                              // W'(c, (tap', n)) = W[n][(8 - tap') w_cpad + c]
        if (nn < p.C) v[i] = ldg4(p.W + static_cast<long long>(nn) * p.ldw + (8 - tap) * p.w_cpad + R.wr.idx);
      }
    }
  } else {
    const int hw = R.Ho * R.Wo;
    int cb = k0 / hw;
    const int rem = k0 - cb * hw;
    int cy = rem / R.Wo, cx = rem - cy * R.Wo;
    const int dy = R.wr.tap / 3, dx = R.wr.tap - dy * 3;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (k0 + i < k_hi) {
        const int iy = cy * R.stride + dy - 1, ix = cx * R.stride + dx - 1;
        if (R.wr.c < p.C && iy >= 0 && iy < p.Hin && ix >= 0 && ix < p.Win)                               // c >= C: channel padding rows
          v[i] = ldg4(p.W + ((static_cast<long long>(cb) * p.Hin + iy) * p.Win + ix) * p.C + R.wr.c);    // channels c .. c + 3 of that pixel
      }
      if (++cx == R.Wo) { cx = 0; if (++cy == R.Ho) { cy = 0; ++cb; } }
    }
  }
}

// write the fetched values into the k-block tile: put(byte offset inside the operand's tile, 16 bytes)
#if defined(__CUDACC__)
#pragma nv_exec_check_disable
#endif
// row mode: N chunks of one row (compile-time); block mode: `active` threads write the 4 x 4 transpose
template <bool BLK, int N, class Put> TF_HD void stage(int row, int c0, bool active, const float4 (&v)[4], Put put) {
  if constexpr (!BLK) {
#pragma unroll
    for (int j = 0; j < N; ++j) put(smem_off(row, c0 + j), v[j]);
    return;
  }
  if (!active) return;
  put(smem_off(row, c0), make_float4(v[0].x, v[1].x, v[2].x, v[3].x));          // the 4 x 4 register transpose
  put(smem_off(row + 1, c0), make_float4(v[0].y, v[1].y, v[2].y, v[3].y));
  put(smem_off(row + 2, c0), make_float4(v[0].z, v[1].z, v[2].z, v[3].z));
  put(smem_off(row + 3, c0), make_float4(v[0].w, v[1].w, v[2].w, v[3].w));
}

struct EpiRow {           // epilogue state of one thread = one accumulator row
  bool mok, atomic, vec_out;
  long long orow;
};

TF_HD EpiRow make_epi_row(const b2u_f32_gemm_params& p, long long m) {
  EpiRow e;
  e.mok = m < p.M;
  e.orow = m;
  if (e.mok) {
    if (p.ps_cout > 0) {
      const long long hw = static_cast<long long>(p.ps_h) * p.ps_w;
      const long long pb = m / hw;
      const long long rem = m - pb * hw;
      const long long pi = rem / p.ps_w, pj = rem - pi * p.ps_w;
      e.orow = (pb * (2 * p.ps_h) + 2 * pi) * (2 * p.ps_w) + 2 * pj;
    } else if (p.rows_in > 0) {
      e.orow = (m / p.rows_in) * p.rows_out + p.row_off + m % p.rows_in;
    }
  }
  e.atomic = p.ksplit > 1 || p.accumulate;
  e.vec_out = p.ps_cout == 0 && !e.atomic && (p.ldc & 3) == 0 && (p.col_off & 3) == 0 && (reinterpret_cast<uintptr_t>(p.out) & 15) == 0 &&
              (!p.residual || ((p.ldres & 3) == 0 && (reinterpret_cast<uintptr_t>(p.residual) & 15) == 0));
  return e;
}

TF_HD void out_add(float* dst, float v) {
#if defined(__CUDA_ARCH__)
  atomicAdd(dst, v);
#else
  *dst += v;
#endif
}

// four consecutive accumulator columns nb .. nb + 3 (nb % 4 == 0) of the row described by `e`
TF_HD void emit4(const b2u_f32_gemm_params& p, const EpiRow& e, int nb, const float (&acc)[4]) {
  if (!e.mok || nb >= p.N) return;
  float f[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int n = nb + j;
    float t = acc[j];
    if (n < p.N) {
      if (p.bias) t += TF_LDG(p.bias + n);
      t = act(t, p.act1);
      if (p.scale) t *= TF_LDG(p.scale + n);
      if (p.shift) t += TF_LDG(p.shift + n);
      t = act(t, p.act2);
    }
    f[j] = t;
  }
  if (e.vec_out && nb + 3 < p.N) {
    const int oc = nb + p.col_off;
    if (p.residual) {
      const float4 r4 = *reinterpret_cast<const float4*>(p.residual + e.orow * p.ldres + oc);
      f[0] += r4.x; f[1] += r4.y; f[2] += r4.z; f[3] += r4.w;
    }
    *reinterpret_cast<float4*>(p.out + e.orow * p.ldc + oc) = make_float4(f[0], f[1], f[2], f[3]);
    return;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int n = nb + j;
    if (n >= p.N) continue;
    long long r = e.orow;
    int oc = n;
    if (p.ps_cout > 0) {
      const int q = n / p.ps_cout;
      oc = n - q * p.ps_cout;
      r += static_cast<long long>(q >> 1) * (2 * p.ps_w) + (q & 1);
    }
    oc += p.col_off;
    float t = f[j];
    if (p.residual) t += p.residual[r * p.ldres + oc];
    if (e.atomic) out_add(&p.out[r * p.ldc + oc], t);
    else p.out[r * p.ldc + oc] = t;
  }
}

// argument checks shared by the GPU entry point and the host model; returns nullptr when the block is valid
inline const char* validate(const b2u_f32_gemm_params* p) {
  if (!p || !p->A || !p->W || !p->out) return "null pointer";
  if (p->M <= 0 || p->N <= 0 || p->K <= 0) return "bad shape";
  if (p->conv && p->w_mode != 3 && (p->Cpad < p->C || p->K != 9 * p->Cpad)) return "conv needs K = 9 * Cpad";
  if (p->w_mode == 3 && (!p->conv || p->N != 9 * p->Cpad)) return "conv weight gradient needs N = 9 * Cpad";
  if (p->w_mode == 2 && !p->conv) return "w_mode 2 is the conv data gradient";
  if (p->ksplit > 1 && (p->bias || p->scale || p->shift || p->act1 || p->act2 || p->residual)) return "split-K accumulates raw products only";
  if (p->ksplit > 65535) return "ksplit too large";
  return nullptr;
}
inline int pick_bn(int N) { return N <= 32 ? 32 : (N <= 64 ? 64 : 128); }

}  // namespace tf32
}  // namespace b2u
