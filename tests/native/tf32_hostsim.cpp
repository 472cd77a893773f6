// Host model of gemm_tf32_kernel (dinounet_b200/csrc/gemm_tf32.cu) for the CPU test suite: the kernel's own addressing
// functions (csrc/gemm_tf32_addr.h, compiled for the host) are executed for all 256 threads of every CTA, writing the
// 128B-swizzled k-block tiles into a byte array that stands for shared memory; the tensor core is modelled by reading those
// tiles back the way the tensor-core MMA reads a K-major SWIZZLE_128B operand (row r, element k of the k-block at byte
// r*128 + k*4 with address bits [4,7) XORed by bits [7,10)), accumulating in double; the epilogue walks the accumulator-tile row /
// column assignment of the 8 warps.  What this does NOT model: descriptors, barriers, the hardware itself - those are
// checked by tests/test_gpu_tf32_gemm.py on the GPU.  Test infrastructure only.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../../dinounet_b200/csrc/gemm_tf32_addr.h"

using namespace b2u::tf32;

static float round_tf32(float v) {   // cvt.rna.tf32.f32
  uint32_t u;
  memcpy(&u, &v, 4);
  const uint32_t mag = ((u & 0x7fffffffu) + 0x1000u) & 0x7fffe000u;
  u = (u & 0x80000000u) | mag;
  memcpy(&v, &u, 4);
  return v;
}

struct HostPut {             // tf32::stage's sink on the host: round to TF32, 16 bytes into the modelled shared memory
  uint8_t* tile;
  void operator()(uint32_t off, float4 v) const {
    const float t[4] = {round_tf32(v.x), round_tf32(v.y), round_tf32(v.z), round_tf32(v.w)};
    memcpy(tile + off, t, 16);
  }
};

// element (row, k) of a K-major SWIZZLE_128B tile with a 1024-byte aligned base, as the tensor core addresses it
static float get(const uint8_t* tile, int row, int k) {
  uint32_t addr = static_cast<uint32_t>(row) * 128u + static_cast<uint32_t>(k) * 4u;
  addr ^= ((addr >> 7) & 7u) << 4;
  float v;
  memcpy(&v, tile + addr, 4);
  return v;
}

static int g_modes = 0;   // bit 0 / 1: A / W operand staged in row mode, bit 2 / 3: in block mode (since the last reset)
extern "C" int tf32_hostsim_modes(int reset) {
  const int m = g_modes;
  if (reset) g_modes = 0;
  return m;
}

template <int BN, bool ABLK, bool WBLK> static void run(const b2u_f32_gemm_params& p);

extern "C" const char* tf32_hostsim_gemm(const b2u_f32_gemm_params* pp) {
  if (const char* why = validate(pp)) return why;
  bool a_blk, w_blk;
  pick_modes(*pp, a_blk, w_blk);
  const int mode = a_blk ? 2 : (w_blk ? 1 : 0);        // the same dispatch as b2u_tf32_gemm
  switch (pick_bn(pp->N) + mode) {
    case 32: run<32, false, false>(*pp); break;
    case 33: run<32, false, true>(*pp); break;
    case 34: run<32, true, true>(*pp); break;
    case 64: run<64, false, false>(*pp); break;
    case 65: run<64, false, true>(*pp); break;
    case 66: run<64, true, true>(*pp); break;
    case 128: run<128, false, false>(*pp); break;
    case 129: run<128, false, true>(*pp); break;
    default: run<128, true, true>(*pp); break;
  }
  return nullptr;
}

template <int BN, bool ABLK, bool WBLK> static void run(const b2u_f32_gemm_params& p) {
  const long long tiles = ((p.M + kTM - 1) / kTM) * ((p.N + BN - 1) / BN);
  const int nz = p.ksplit > 1 ? p.ksplit : 1;
  const int a_bytes = kTM * 128, w_bytes = BN * 128;
  std::vector<uint8_t> tile(a_bytes + w_bytes);
  std::vector<double> acc(static_cast<size_t>(kTM) * BN);
  for (int bz = 0; bz < nz; ++bz)
      for (long long bx = 0; bx < tiles; ++bx) {
        int k_lo, k_hi;
        k_slice(p, bz, k_lo, k_hi);
        if (k_lo >= k_hi) continue;
        const int nkb = (k_hi - k_lo + kTK - 1) / kTK;
        long long m0;
        int n0;
        tile_origin(p, BN, bx, m0, n0);
        std::fill(acc.begin(), acc.end(), 0.0);
        for (int kb = 0; kb < nkb; ++kb) {
          memset(tile.data(), 0xff, tile.size());                 // NaN pattern: an unwritten chunk poisons the tile
          const int k0 = k_lo + kb * kTK;
          for (int tid = 0; tid < kTThreads; ++tid) {
            const Roles R = make_roles(p, tid, m0, n0, BN, ABLK, WBLK);
            g_modes |= (R.a_blk ? 4 : 1) | (R.w_blk ? 8 : 2);
            float4 va[4], vw[4];
            fetch_a<ABLK>(p, R, k0, k_hi, va);
            fetch_w<WBLK, BN / 32>(p, R, k0, k_hi, vw);
            stage<ABLK, 4>(R.a_r, R.a_c0, true, va, HostPut{tile.data()});
            stage<WBLK, BN / 32>(R.w_r, R.w_c0, R.w_n != 0, vw, HostPut{tile.data() + a_bytes});
          }
          for (int r = 0; r < kTM; ++r)
            for (int n = 0; n < BN; ++n) {
              double s = 0.0;
              for (int k = 0; k < kTK; ++k) s += static_cast<double>(get(tile.data(), r, k)) * static_cast<double>(get(tile.data() + a_bytes, n, k));
              acc[static_cast<size_t>(r) * BN + n] += s;
            }
        }
        const int cols = BN / 2;
        for (int warp = 0; warp < 8; ++warp)
          for (int lane = 0; lane < 32; ++lane) {
            const int q = warp & 3, half = warp >> 2;
            const int row = q * 32 + lane;
            const EpiRow e = make_epi_row(p, m0 + row);
            for (int c0 = 0; c0 < cols; c0 += 16)
              for (int g = 0; g < 4; ++g) {
                const int col = half * cols + c0 + g * 4;
                const float a4[4] = {static_cast<float>(acc[static_cast<size_t>(row) * BN + col]), static_cast<float>(acc[static_cast<size_t>(row) * BN + col + 1]),
                                     static_cast<float>(acc[static_cast<size_t>(row) * BN + col + 2]), static_cast<float>(acc[static_cast<size_t>(row) * BN + col + 3])};
                emit4(p, e, n0 + col, a4);
              }
          }
      }
}
