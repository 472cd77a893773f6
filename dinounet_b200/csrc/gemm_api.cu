// Host side of the tensor-core GEMM / implicit-GEMM convolution entry points (b2u_gemm, b2u_qkv_rope): shape checks, tile
// choice, TMA tensor maps, dispatch to the persistent wgmma kernel family of gemm_tc2.cu.
#include "common.cuh"
#include "../../include/dinounet_b200.h"
#include "host_util.h"
#include "gemm_common.h"

namespace b2u {

// BLOCK_N: the fp32 accumulator tile (128 x BN) and the TMA ring share the 227 KB of shared memory, so tiles stop at 128
static int pick_bn(int N) {
  if (N <= 32) return 32;
  if (N <= 64) return 64;
  return 128;
}

static int run_gemm(bool qkv, int bn, int dtype, const GemmMaps& maps, const GemmArgs& args, cudaStream_t stream) {
  return gemm_v2_dispatch(qkv, bn, dtype, maps, args, stream);
}

// 2-D K-major operand map: dims {K, rows}, box {64, box_rows}, 128B swizzle, OOB zero fill.
static int make_map_2d(CUtensorMap* map, const void* base, int64_t rows, int64_t K, int64_t ld, int box_rows,
                       int dtype) {
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(K), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 2};
  cuuint32_t box[2] = {BK, static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  return encode_tensor_map(map, dtype, 2, base, dims, strides, box, estr);
}

extern "C" int b2u_gemm(const b2u_gemm_params* p, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!p || !p->A || !p->Wp || !p->epi.out) return set_error(-1, "b2u_gemm: null pointer");
  if (p->N % 32 || p->lda % 8 || p->ldw % 8) return set_error(-1, "b2u_gemm: N must be a multiple of 32; lda, ldw multiples of 8");
  const b2u_epilogue& e = p->epi;
  if ((e.ldc % 8) || (e.col_off % 8)) return set_error(-1, "b2u_gemm: ldc/col_off must be multiples of 8");
  if (e.ps_cout > 0 && (e.ps_cout % 32)) return set_error(-1, "b2u_gemm: ps_cout must be a multiple of 32");
  GemmMaps maps;
  GemmArgs a{};
  a.N = p->N;
  a.epi = p->epi;
  a.conv = p->conv;
  if (e.act1 == B2U_ACT_SWIGLU && (p->N % 64 || p->conv != B2U_CONV_NONE))
    return set_error(-1, "b2u_gemm: SwiGLU epilogue needs N %% 64 == 0 and a plain GEMM");
  const int bn = e.act1 == B2U_ACT_SWIGLU ? 128 : pick_bn(p->N);
  a.n_tiles = (p->N + bn - 1) / bn;
  long long m_tiles;
  int rc;
  if (p->conv == B2U_CONV_NONE) {
    a.M = p->M;
    a.num_kb = (p->K + BK - 1) / BK;
    m_tiles = (static_cast<long long>(p->M) + BM - 1) / BM;
    a.res_prefetch = (get_option(7) != 1 && a.num_kb <= 8) ? 1 : 0;   // short K only: measured +3 % there, nothing (or worse) at K >= 1024
    if ((rc = make_map_2d(&maps.a[0], p->A, p->M, p->K, p->lda, BM, p->dtype))) return rc;
    if ((rc = make_map_2d(&maps.b, p->Wp, p->N, p->K, p->ldw, bn, p->dtype))) return rc;
  } else {
    const int stride = p->conv == B2U_CONV3X3_S2 ? 2 : 1;
    if (p->C % 8) return set_error(-1, "b2u_gemm(conv): C must be a multiple of 8");
    if (stride == 2 && ((p->Hin | p->Win) & 1)) return set_error(-1, "b2u_gemm(conv s2): odd image size");
    a.Ho = p->Hin / stride;
    a.Wo = p->Win / stride;
    a.cb = (p->C + BK - 1) / BK;
    a.num_kb = 9 * a.cb;
    // tile = TH x TW = 128 output pixels; TW = the largest power of two (<= 128) that divides the output width, so any
    // width that is a multiple of 4 tiles exactly in x (rows past the image are masked in the epilogue, OOB = zero fill)
    a.TW = 128;
    while (a.TW > 1 && (a.Wo % a.TW)) a.TW >>= 1;
    if (a.TW < 4) return set_error(-1, "b2u_gemm(conv): output width must be a multiple of 4");
    a.TH = BM / a.TW;
    a.tiles_x = a.Wo / a.TW;
    a.tiles_y = (a.Ho + a.TH - 1) / a.TH;
    m_tiles = static_cast<long long>(p->B) * a.tiles_x * a.tiles_y;
    a.M = p->B * a.Ho * a.Wo;
    const int64_t C = p->C;
    if (stride == 1) {
      cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)p->Win, (cuuint64_t)p->Hin, (cuuint64_t)p->B};
      cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)C * p->Win * 2, (cuuint64_t)C * p->Win * p->Hin * 2};
      cuuint32_t box[4] = {BK, (cuuint32_t)a.TW, (cuuint32_t)a.TH, 1};
      cuuint32_t estr[4] = {1, 1, 1, 1};
      if ((rc = encode_tensor_map(&maps.a[0], p->dtype, 4, p->A, dims, strides, box, estr))) return rc;
    } else {
      for (int py = 0; py < 2; ++py)
        for (int px = 0; px < 2; ++px) {
          const char* base = static_cast<const char*>(p->A) + (static_cast<int64_t>(py) * p->Win + px) * C * 2;
          cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)(p->Win / 2), (cuuint64_t)(p->Hin / 2), (cuuint64_t)p->B};
          cuuint64_t strides[3] = {(cuuint64_t)C * 4, (cuuint64_t)C * p->Win * 4, (cuuint64_t)C * p->Win * p->Hin * 2};
          cuuint32_t box[4] = {BK, (cuuint32_t)a.TW, (cuuint32_t)a.TH, 1};
          cuuint32_t estr[4] = {1, 1, 1, 1};
          if ((rc = encode_tensor_map(&maps.a[py * 2 + px], p->dtype, 4, base, dims, strides, box, estr))) return rc;
        }
    }
    if ((rc = make_map_2d(&maps.b, p->Wp, p->N, static_cast<int64_t>(a.num_kb) * BK, p->ldw, bn, p->dtype))) return rc;
  }
  if (m_tiles <= 0 || m_tiles > 0x7FFFFFFFLL) return set_error(-1, "b2u_gemm: bad grid");
  a.m_tiles = static_cast<int>(m_tiles);
  return run_gemm(false, bn, p->dtype, maps, a, stream);
}

extern "C" int b2u_qkv_rope(const b2u_qkv_params* p, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!p || !p->A || !p->Wp || !p->q || !p->k || !p->v) return set_error(-1, "b2u_qkv_rope: null pointer");
  const int head_dim = p->heads > 0 ? p->D / p->heads : 0;
  if (p->D != p->heads * head_dim || (head_dim != 64 && head_dim != 128))
    return set_error(-1, "b2u_qkv_rope: head_dim must be 64 or 128");
  GemmMaps maps;
  GemmArgs a{};
  a.M = p->B * p->ntok;
  a.N = 3 * p->D;
  a.num_kb = (p->D + BK - 1) / BK;
  const int bn = pick_bn(a.N);
  a.n_tiles = (a.N + bn - 1) / bn;
  a.conv = 0;
  a.epi.bias = p->bias;
  a.ntok = p->ntok; a.D = p->D; a.heads = p->heads; a.prefix = p->prefix; a.head_dim = head_dim;
  a.rope_sin = p->rope_sin; a.rope_cos = p->rope_cos;
  a.q = p->q; a.k = p->k; a.v = p->v;
  a.npad = p->v_transposed ? p->npad : 0;
  if (p->rope_w > 0) {
    a.rope_w = p->rope_w;
    a.rope_h = (p->ntok - p->prefix) / p->rope_w;
    if (a.rope_h * a.rope_w != p->ntok - p->prefix || (a.rope_h + a.rope_w) * (head_dim * 2 + 16) > 128 * 32 * 2 * 4)
      return set_error(-1, "b2u_qkv_rope: rope grid %d x %d does not match ntok/prefix or is too large", a.rope_h, a.rope_w);
  }
  if (a.npad && (a.npad % 8 || a.npad < p->ntok)) return set_error(-1, "b2u_qkv_rope: bad npad");
  int rc;
  a.m_tiles = static_cast<int>((static_cast<long long>(a.M) + BM - 1) / BM);
  if ((rc = make_map_2d(&maps.a[0], p->A, a.M, p->D, p->lda, BM, p->dtype))) return rc;
  if ((rc = make_map_2d(&maps.b, p->Wp, a.N, p->D, p->ldw, bn, p->dtype))) return rc;
  return run_gemm(true, bn, p->dtype, maps, a, stream);
}

}  // namespace b2u
