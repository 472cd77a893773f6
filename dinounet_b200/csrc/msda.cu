// MultiScaleDeformableAttention forward for sm_90a.
//
// b2u_msda_forward — the hot-path kernel: one warp per query, lane = (head = lane/2, channel half = lane&1).  The
//   per-head prologue the reference runs as separate torch ops (softmax over the points, reference point + offset /
//   (W,H), ms_deform_attn.py:185-197) is fused: each lane loads its head's 8 offsets + 4 logits as three float4.
//   The value map of one image (Hv*Wv x D/2, 16-bit, <= 1 MB for ViT-L) stays L2/L1 resident; the kernel is bound by
//   the streaming read of the offset/logit rows and the write of the sampled rows.
// b2u_msda_forward_f32 — signature-compatible (in meaning) with the reference pybind op `ms_deform_attn_forward`
//   (ops/src/vision.cpp:18, ms_deform_attn_cuda.cu:25-85, ms_deform_im2col_cuda.cuh:242-304): fp32, multi-level.
#include <algorithm>

#include "common.cuh"
#include "../../include/dinounet_b200.h"
#include "host_util.h"
#include "gemm_common.h"

namespace b2u {

template <typename T, int HALF>  // HALF = channels per lane (dh / 2), even
__global__ void __launch_bounds__(256) msda_fwd_kernel(const T* __restrict__ value, const float* __restrict__ offaw,
                                                       T* __restrict__ out, int B, int Hv, int Wv, int heads) {
  pdl_begin();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int HW = Hv * Wv;
  const int Lq = (HW * 21) / 4;
  const long long qg = static_cast<long long>(blockIdx.x) * 8 + warp;  // global query index in [0, B*Lq)
  if (qg >= static_cast<long long>(B) * Lq) return;
  const int b = static_cast<int>(qg / Lq);
  int q = static_cast<int>(qg - static_cast<long long>(b) * Lq);
  // reference point = cell centre of the query in its own pyramid level (dinov3_adapter.py:40-53,65-68)
  int gh = 2 * Hv, gw = 2 * Wv;
  if (q >= 4 * HW) { q -= 4 * HW; gh = Hv; gw = Wv; if (q >= HW) { q -= HW; gh = Hv / 2; gw = Wv / 2; } }
  const int qy = q / gw, qx = q - qy * gw;
  const float refx = (qx + 0.5f) / gw, refy = (qy + 0.5f) / gh;

  const int head = lane >> 1, half = lane & 1;
  const int dh = 2 * HALF;
  const float* row = offaw + qg * (heads * 12);
  const float4 o0 = *reinterpret_cast<const float4*>(row + head * 8);
  const float4 o1 = *reinterpret_cast<const float4*>(row + head * 8 + 4);
  const float4 lg = *reinterpret_cast<const float4*>(row + heads * 8 + head * 4);
  // softmax over the 4 points (fp32, ms_deform_attn.py:189-190)
  const float mx = fmaxf(fmaxf(lg.x, lg.y), fmaxf(lg.z, lg.w));
  float w[4] = {__expf(lg.x - mx), __expf(lg.y - mx), __expf(lg.z - mx), __expf(lg.w - mx)};
  const float inv = 1.f / (w[0] + w[1] + w[2] + w[3]);
  const float ox[4] = {o0.x, o0.z, o1.x, o1.z}, oy[4] = {o0.y, o0.w, o1.y, o1.w};

  float acc[HALF];
#pragma unroll
  for (int j = 0; j < HALF; ++j) acc[j] = 0.f;
  const T* vb = value + (static_cast<long long>(b) * HW * heads + head) * dh + half * HALF;
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const float aw = w[p] * inv;
    // loc = ref + off / (W, H);  pixel = loc * (W, H) - 0.5   (grid_sample align_corners=False)
    const float px = (refx + ox[p] / Wv) * Wv - 0.5f;
    const float py = (refy + oy[p] / Hv) * Hv - 0.5f;
    const float fx = floorf(px), fy = floorf(py);
    const int x0 = static_cast<int>(fx), y0 = static_cast<int>(fy);
    const float lx = px - fx, ly = py - fy;
    const float cw[4] = {(1.f - ly) * (1.f - lx), (1.f - ly) * lx, ly * (1.f - lx), ly * lx};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int yy = y0 + (c >> 1), xx = x0 + (c & 1);
      if (yy < 0 || yy >= Hv || xx < 0 || xx >= Wv) continue;  // zero padding
      const float wt = aw * cw[c];
      const T* src = vb + static_cast<long long>(yy * Wv + xx) * heads * dh;
#pragma unroll
      for (int j = 0; j < HALF; j += 2) {
        const float2 v2 = T16<T>::unpack2(*reinterpret_cast<const uint32_t*>(src + j));
        acc[j] = fmaf(wt, v2.x, acc[j]);
        acc[j + 1] = fmaf(wt, v2.y, acc[j + 1]);
      }
    }
  }
  T* dst = out + qg * (heads * dh) + head * dh + half * HALF;
#pragma unroll
  for (int j = 0; j < HALF; j += 2) *reinterpret_cast<uint32_t*>(dst + j) = T16<T>::pack2(acc[j], acc[j + 1]);
}

// ---- v2: value slab of HPC heads of one image staged in shared memory -------------------------------------------------
// CTA = (query slice, head group, image).  The HPC heads' value maps ([Hv*Wv, dh] each, 16-bit) are copied once into
// smem (coalesced 16 B loads), then every thread owns one (query, head) pair: it reads its 8 offsets + 4 logits
// (three float4 from the fp32 offaw row), runs the softmax / location prologue, gathers 4 points x 4 corners x dh
// channels from SHARED memory with 16-byte loads and writes dh contiguous 16-bit outputs.  HBM traffic is the
// algorithmic minimum (offaw + out + value once per CTA); the random gather never leaves the SM.
template <typename T, int DH, int HPC, int PITCH = HPC * DH>
__global__ void __launch_bounds__(256) msda_smem_kernel(const T* __restrict__ value, const float* __restrict__ offaw,
                                                        T* __restrict__ out, int Hv, int Wv, int heads, int qsplit) {
  pdl_begin();
  extern __shared__ __align__(16) uint8_t sm_raw[];
  T* slab = reinterpret_cast<T*>(sm_raw);                 // [HW][PITCH]
  const int HW = Hv * Wv;
  const int Lq = (HW * 21) / 4;
  const int b = blockIdx.z, hg = blockIdx.y;
  constexpr int ROW = HPC * DH;                           // payload elements per position
  // PITCH (elements between positions) >= ROW.  One-head layouts pad the row to a power of two so that many small CTAs
  // fit an SM (dh 32 / 24: 64 B rows = 64 KB slab, 3 CTAs per SM; dh 12: 32 B rows = 32 KB slab, 6 CTAs per SM).
  // SWZ (64 B rows): 16-byte chunk c of position pos lives at c ^ ((pos >> 1) & 3), so the 8 lanes of a quarter-warp
  // that sample 8 neighbouring positions (neighbouring queries do) hit 8 distinct bank groups instead of 2.
  constexpr bool SWZ = (HPC == 1 && PITCH == 32);
  // ---- stage the slab: value[b, pos, hg*HPC .. +HPC, :] -> slab[pos][0 .. ROW)  (8-byte granules)
  {
    constexpr int V8 = ROW * 2 / 8;                       // 8-byte granules per position
    const uint2* src = reinterpret_cast<const uint2*>(value + (static_cast<long long>(b) * HW * heads + hg * HPC) * DH);
    const int src_stride = heads * DH * 2 / 8;            // granules between consecutive positions
    for (int i = threadIdx.x; i < HW * V8; i += 256) {
      const int pos = i / V8, v = i - pos * V8;
      int off = v * 8;                                    // byte offset inside the row
      if (SWZ) off = (((off >> 4) ^ ((pos >> 1) & 3)) << 4) | (off & 15);
      *reinterpret_cast<uint2*>(sm_raw + static_cast<size_t>(pos) * (PITCH * 2) + off) =
          __ldg(src + static_cast<long long>(pos) * src_stride + v);
    }
  }
  __syncthreads();
  const int per = (Lq + qsplit - 1) / qsplit;
  const int q_begin = blockIdx.x * per;
  const int q_end = min(Lq, q_begin + per);
  for (int w = q_begin * HPC + threadIdx.x; w < q_end * HPC; w += 256) {
    const int q = w / HPC, hl = w - q * HPC;
    const int head = hg * HPC + hl;
    int qq = q, gh = 2 * Hv, gw = 2 * Wv;
    if (qq >= 4 * HW) { qq -= 4 * HW; gh = Hv; gw = Wv; if (qq >= HW) { qq -= HW; gh = Hv / 2; gw = Wv / 2; } }
    const int qy = qq / gw, qx = qq - qy * gw;
    const float refx = (qx + 0.5f) / gw, refy = (qy + 0.5f) / gh;
    const long long qg = static_cast<long long>(b) * Lq + q;
    const float* row = offaw + qg * (heads * 12);
    const float4 o0 = __ldg(reinterpret_cast<const float4*>(row + head * 8));
    const float4 o1 = __ldg(reinterpret_cast<const float4*>(row + head * 8 + 4));
    const float4 lg = __ldg(reinterpret_cast<const float4*>(row + heads * 8 + head * 4));
    const float mx = fmaxf(fmaxf(lg.x, lg.y), fmaxf(lg.z, lg.w));
    float wgt[4] = {__expf(lg.x - mx), __expf(lg.y - mx), __expf(lg.z - mx), __expf(lg.w - mx)};
    const float inv = 1.f / (wgt[0] + wgt[1] + wgt[2] + wgt[3]);
    const float ox[4] = {o0.x, o0.z, o1.x, o1.z}, oy[4] = {o0.y, o0.w, o1.y, o1.w};
    float acc[DH];
#pragma unroll
    for (int j = 0; j < DH; ++j) acc[j] = 0.f;
    const T* hb = slab + hl * DH;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const float aw = wgt[p] * inv;
      const float px = (refx + ox[p] / Wv) * Wv - 0.5f;
      const float py = (refy + oy[p] / Hv) * Hv - 0.5f;
      const float fx = floorf(px), fy = floorf(py);
      const int x0 = static_cast<int>(fx), y0 = static_cast<int>(fy);
      const float lx = px - fx, ly = py - fy;
      const float cw[4] = {(1.f - ly) * (1.f - lx), (1.f - ly) * lx, ly * (1.f - lx), ly * lx};
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int yy = y0 + (c >> 1), xx = x0 + (c & 1);
        if (yy < 0 || yy >= Hv || xx < 0 || xx >= Wv) continue;
        const float wt = aw * cw[c];
        const int pos = yy * Wv + xx;
        const T* src = hb + pos * PITCH;
        const int sw = SWZ ? ((pos >> 1) & 3) : 0;
        if constexpr (DH % 8 == 0) {
#pragma unroll
          for (int j = 0; j < DH; j += 8) {
            const uint4 u = *reinterpret_cast<const uint4*>(src + (SWZ ? (((j >> 3) ^ sw) << 3) : j));
            const float2 a0 = T16<T>::unpack2(u.x), a1 = T16<T>::unpack2(u.y), a2 = T16<T>::unpack2(u.z), a3 = T16<T>::unpack2(u.w);
            acc[j] = fmaf(wt, a0.x, acc[j]); acc[j + 1] = fmaf(wt, a0.y, acc[j + 1]);
            acc[j + 2] = fmaf(wt, a1.x, acc[j + 2]); acc[j + 3] = fmaf(wt, a1.y, acc[j + 3]);
            acc[j + 4] = fmaf(wt, a2.x, acc[j + 4]); acc[j + 5] = fmaf(wt, a2.y, acc[j + 5]);
            acc[j + 6] = fmaf(wt, a3.x, acc[j + 6]); acc[j + 7] = fmaf(wt, a3.y, acc[j + 7]);
          }
        } else {   // DH = 12: 8-byte loads
#pragma unroll
          for (int j = 0; j < DH; j += 4) {
            const uint2 u = *reinterpret_cast<const uint2*>(src + j);
            const float2 a0 = T16<T>::unpack2(u.x), a1 = T16<T>::unpack2(u.y);
            acc[j] = fmaf(wt, a0.x, acc[j]); acc[j + 1] = fmaf(wt, a0.y, acc[j + 1]);
            acc[j + 2] = fmaf(wt, a1.x, acc[j + 2]); acc[j + 3] = fmaf(wt, a1.y, acc[j + 3]);
          }
        }
      }
    }
    T* dst = out + qg * (heads * DH) + head * DH;
    if constexpr (DH % 8 == 0) {
#pragma unroll
      for (int j = 0; j < DH; j += 8)
        *reinterpret_cast<uint4*>(dst + j) = make_uint4(T16<T>::pack2(acc[j], acc[j + 1]), T16<T>::pack2(acc[j + 2], acc[j + 3]),
                                                        T16<T>::pack2(acc[j + 4], acc[j + 5]), T16<T>::pack2(acc[j + 6], acc[j + 7]));
    } else {
#pragma unroll
      for (int j = 0; j < DH; j += 4)
        *reinterpret_cast<uint2*>(dst + j) = make_uint2(T16<T>::pack2(acc[j], acc[j + 1]), T16<T>::pack2(acc[j + 2], acc[j + 3]));
    }
  }
}

template <typename T, int DH, int HPC, int PITCH = HPC * DH>
static int launch_msda_smem(const void* value, const float* offaw, void* out, int B, int Hv, int Wv, int heads,
                            cudaStream_t stream) {
  const size_t smem = static_cast<size_t>(Hv) * Wv * PITCH * 2;
  auto kern = msda_smem_kernel<T, DH, HPC, PITCH>;
  static size_t configured_dev[64] = {};
  size_t& configured = configured_dev[current_device_index()];
  if (smem > configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return set_error(-2, "cudaFuncSetAttribute(msda_smem): %s", cudaGetErrorString(e));
    configured = smem;
  }
  const int groups = heads / HPC;
  // enough CTAs for several waves of (CTAs that fit an SM) x 132 SMs; each re-stages its slab from L2
  const int per_sm = static_cast<int>(std::min<size_t>(8, std::max<size_t>(1, (200 * 1024) / std::max<size_t>(smem, 1))));
  int qsplit = ((per_sm > 1 ? 6 : 2) * per_sm * num_sms() + B * groups - 1) / (B * groups);
  if (qsplit < 1) qsplit = 1;
  dim3 grid(qsplit, groups, B);
  launch_pdl(kern, grid, 256, smem, stream, static_cast<const T*>(value), offaw, static_cast<T*>(out), Hv, Wv, heads, qsplit);
  return check_launch("msda_forward(smem)");
}

extern "C" int b2u_msda_forward(const void* value, const float* offaw, void* out, int32_t B, int32_t Hv, int32_t Wv,
                                int32_t heads, int32_t dh, int32_t points, int32_t dtype, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (heads != 16 || points != 4) return set_error(-1, "b2u_msda_forward: built for 16 heads x 4 points (dinounet_training.py:758-759)");
  if ((Hv & 1) || (Wv & 1)) return set_error(-1, "b2u_msda_forward: value map must have even size");
  // shared-memory slab path (default): per CTA HPC heads x Hv*Wv positions x dh channels must fit in 200 KB
  if (get_option(1) != 1) {
#define B2U_MSDA_SMEM(DH_, HPC_, PITCH_)                                                                                  \
    if (dh == DH_ && static_cast<size_t>(Hv) * Wv * PITCH_ * 2 <= 200 * 1024)                                              \
      return dtype == B2U_BF16 ? launch_msda_smem<__nv_bfloat16, DH_, HPC_, PITCH_>(value, offaw, out, B, Hv, Wv, heads, stream) \
                               : launch_msda_smem<__half, DH_, HPC_, PITCH_>(value, offaw, out, B, Hv, Wv, heads, stream);
    // one head per CTA with power-of-two padded rows (many small CTAs per SM); option 1 == 2 keeps the multi-head layouts
    if (get_option(1) != 2) { B2U_MSDA_SMEM(32, 1, 32) B2U_MSDA_SMEM(24, 1, 32) B2U_MSDA_SMEM(12, 1, 16) }
    B2U_MSDA_SMEM(12, 8, 96) B2U_MSDA_SMEM(24, 4, 96) B2U_MSDA_SMEM(32, 2, 64) B2U_MSDA_SMEM(12, 2, 24) B2U_MSDA_SMEM(24, 1, 24)
    B2U_MSDA_SMEM(32, 1, 32)
#undef B2U_MSDA_SMEM
  }
  const long long nq = static_cast<long long>(B) * ((Hv * Wv * 21) / 4);
  const int grid = static_cast<int>((nq + 7) / 8);
#define B2U_MSDA(HALF_)                                                                                               \
  case 2 * HALF_:                                                                                                     \
    if (dtype == B2U_BF16)                                                                                            \
      launch_pdl(msda_fwd_kernel<__nv_bfloat16, HALF_>, grid, 256, 0, stream, static_cast<const __nv_bfloat16*>(value), offaw,  \
                                                                      static_cast<__nv_bfloat16*>(out), B, Hv, Wv, heads); \
    else                                                                                                              \
      launch_pdl(msda_fwd_kernel<__half, HALF_>, grid, 256, 0, stream, static_cast<const __half*>(value), offaw,               \
                                                               static_cast<__half*>(out), B, Hv, Wv, heads);          \
    break;
  switch (dh) {
    B2U_MSDA(6) B2U_MSDA(12) B2U_MSDA(16) B2U_MSDA(64)
    default: return set_error(-1, "b2u_msda_forward: per-head dim %d not in {12,24,32,128}", dh);
  }
#undef B2U_MSDA
  return check_launch("msda_forward");
}

// ------------------------------------------------------------------------------------------------ reference-op drop-in
__global__ void msda_f32_kernel(const float* __restrict__ value, const int64_t* __restrict__ shapes,
                                const int64_t* __restrict__ lsi, const float* __restrict__ loc,
                                const float* __restrict__ attw, float* __restrict__ out, int B, int S, int Lq, int M,
                                int D, int L, int P) {
  pdl_begin();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * Lq * M * D;
  if (i >= total) return;
  const int c = static_cast<int>(i % D);
  const int m = static_cast<int>((i / D) % M);
  const int q = static_cast<int>((i / (static_cast<long long>(D) * M)) % Lq);
  const int b = static_cast<int>(i / (static_cast<long long>(D) * M * Lq));
  const long long wbase = ((static_cast<long long>(b) * Lq + q) * M + m) * L * P;
  float acc = 0.f;
  for (int l = 0; l < L; ++l) {
    const int H = static_cast<int>(shapes[2 * l]), W = static_cast<int>(shapes[2 * l + 1]);
    const float* vl = value + ((static_cast<long long>(b) * S + lsi[l]) * M + m) * D + c;
    for (int p = 0; p < P; ++p) {
      const float lx = loc[(wbase + l * P + p) * 2], ly = loc[(wbase + l * P + p) * 2 + 1];
      const float aw = attw[wbase + l * P + p];
      const float px = lx * W - 0.5f, py = ly * H - 0.5f;
      if (py > -1 && px > -1 && py < H && px < W) {
        const float fx = floorf(px), fy = floorf(py);
        const int x0 = static_cast<int>(fx), y0 = static_cast<int>(fy);
        const float ax = px - fx, ay = py - fy;
        float v = 0.f;
        if (y0 >= 0 && x0 >= 0) v += (1.f - ay) * (1.f - ax) * vl[static_cast<long long>(y0 * W + x0) * M * D];
        if (y0 >= 0 && x0 + 1 < W) v += (1.f - ay) * ax * vl[static_cast<long long>(y0 * W + x0 + 1) * M * D];
        if (y0 + 1 < H && x0 >= 0) v += ay * (1.f - ax) * vl[static_cast<long long>((y0 + 1) * W + x0) * M * D];
        if (y0 + 1 < H && x0 + 1 < W) v += ay * ax * vl[static_cast<long long>((y0 + 1) * W + x0 + 1) * M * D];
        acc += aw * v;
      }
    }
  }
  out[i] = acc;
}

extern "C" int b2u_msda_forward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                                    const float* loc, const float* attw, float* out, int32_t B, int32_t S, int32_t Lq,
                                    int32_t heads, int32_t dh, int32_t levels, int32_t points, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!value || !spatial_shapes || !level_start_index || !loc || !attw || !out)
    return set_error(-1, "b2u_msda_forward_f32: null pointer");
  const long long total = static_cast<long long>(B) * Lq * heads * dh;
  launch_pdl(msda_f32_kernel, static_cast<int>((total + 255) / 256), 256, 0, stream, value, spatial_shapes, level_start_index, loc,
                                                                            attw, out, B, S, Lq, heads, dh, levels, points);
  return check_launch("msda_forward_f32");
}
// Backward of the op above == the reference pybind op `ms_deform_attn_backward` (the one native kernel the reference's
// training step executes, ms_deform_attn.py:58-66).  One warp per (b, q, head); lanes stride the channels, so the
// per-sample scalars (grad of the location / attention weight) are warp-shuffle reductions and the scatter into
// grad_value is a coalesced row of `red.global.add.f32` per bilinear corner (value maps are L2-resident: 32x32xD).
__global__ void msda_bwd_f32_kernel(const float* __restrict__ value, const int64_t* __restrict__ shapes,
                                    const int64_t* __restrict__ lsi, const float* __restrict__ loc,
                                    const float* __restrict__ attw, const float* __restrict__ gout,
                                    float* __restrict__ gvalue, float* __restrict__ gloc, float* __restrict__ gattw,
                                    int B, int S, int Lq, int M, int D, int L, int P) {
  pdl_begin();
  const long long warp = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const long long total = static_cast<long long>(B) * Lq * M;
  if (warp >= total) return;
  const int m = static_cast<int>(warp % M);
  const long long bq = warp / M;
  const int b = static_cast<int>(bq / Lq);
  const long long wbase = warp * L * P;
  const float* go = gout + (bq * M + m) * D;
  const long long rs = static_cast<long long>(M) * D;  // stride between spatial positions of one head
  for (int l = 0; l < L; ++l) {
    const int H = static_cast<int>(shapes[2 * l]), W = static_cast<int>(shapes[2 * l + 1]);
    const long long lbase = ((static_cast<long long>(b) * S + lsi[l]) * M + m) * D;
    const float* vl = value + lbase;
    float* gvl = gvalue + lbase;
    for (int p = 0; p < P; ++p) {
      const long long wi = wbase + l * P + p;
      const float lx = loc[wi * 2], ly = loc[wi * 2 + 1], aw = attw[wi];
      const float px = lx * W - 0.5f, py = ly * H - 0.5f;
      float g_aw = 0.f, g_x = 0.f, g_y = 0.f;
      if (py > -1 && px > -1 && py < H && px < W) {
        const float fx = floorf(px), fy = floorf(py);
        const int x0 = static_cast<int>(fx), y0 = static_cast<int>(fy);
        const float ax = px - fx, ay = py - fy;
        const bool t = y0 >= 0, bt = y0 + 1 < H, lf = x0 >= 0, rt = x0 + 1 < W;
        const long long o00 = static_cast<long long>(y0 * W + x0) * rs, o01 = o00 + rs,
                        o10 = o00 + static_cast<long long>(W) * rs, o11 = o10 + rs;
        const float w00 = (1.f - ay) * (1.f - ax), w01 = (1.f - ay) * ax, w10 = ay * (1.f - ax), w11 = ay * ax;
        for (int c = lane; c < D; c += 32) {
          const float g = go[c];
          const float v00 = (t && lf) ? vl[o00 + c] : 0.f, v01 = (t && rt) ? vl[o01 + c] : 0.f;
          const float v10 = (bt && lf) ? vl[o10 + c] : 0.f, v11 = (bt && rt) ? vl[o11 + c] : 0.f;
          g_aw += g * (w00 * v00 + w01 * v01 + w10 * v10 + w11 * v11);
          g_x += g * ((1.f - ay) * (v01 - v00) + ay * (v11 - v10));
          g_y += g * ((1.f - ax) * (v10 - v00) + ax * (v11 - v01));
          const float ga = g * aw;
          if (t && lf) atomicAdd(gvl + o00 + c, ga * w00);
          if (t && rt) atomicAdd(gvl + o01 + c, ga * w01);
          if (bt && lf) atomicAdd(gvl + o10 + c, ga * w10);
          if (bt && rt) atomicAdd(gvl + o11 + c, ga * w11);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          g_aw += __shfl_xor_sync(0xffffffffu, g_aw, o);
          g_x += __shfl_xor_sync(0xffffffffu, g_x, o);
          g_y += __shfl_xor_sync(0xffffffffu, g_y, o);
        }
      }
      if (lane == 0) {
        gattw[wi] = g_aw;
        gloc[wi * 2] = g_x * aw * W;
        gloc[wi * 2 + 1] = g_y * aw * H;
      }
    }
  }
}

extern "C" int b2u_msda_backward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                                     const float* loc, const float* attw, const float* grad_out, float* grad_value,
                                     float* grad_loc, float* grad_attw, int32_t B, int32_t S, int32_t Lq, int32_t heads,
                                     int32_t dh, int32_t levels, int32_t points, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!value || !spatial_shapes || !level_start_index || !loc || !attw || !grad_out || !grad_value || !grad_loc ||
      !grad_attw)
    return set_error(-1, "b2u_msda_backward_f32: null pointer");
  if (B <= 0 || S <= 0 || Lq <= 0 || heads <= 0 || dh <= 0 || levels <= 0 || points <= 0)
    return set_error(-1, "b2u_msda_backward_f32: non-positive dimension");
  cudaError_t e = cudaMemsetAsync(grad_value, 0, sizeof(float) * static_cast<size_t>(B) * S * heads * dh, stream);
  if (e != cudaSuccess) return set_error(-2, "b2u_msda_backward_f32: memset: %s", cudaGetErrorString(e));
  const long long warps = static_cast<long long>(B) * Lq * heads;
  launch_pdl(msda_bwd_f32_kernel, static_cast<int>((warps * 32 + 255) / 256), 256, 0, stream, 
      value, spatial_shapes, level_start_index, loc, attw, grad_out, grad_value, grad_loc, grad_attw, B, S, Lq, heads,
      dh, levels, points);
  return check_launch("msda_backward_f32");
}

}  // namespace b2u
