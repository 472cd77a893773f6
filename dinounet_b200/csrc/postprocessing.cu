// Keep-the-largest-component postprocessing on the device (reference: postprocessing/remove_connected_components.py:22-34
// `remove_all_but_largest_component_from_segmentation`, with acvl-utils' `remove_all_but_largest_component`:
// skimage's `label(mask, connectivity=None)`, a bincount, and every component whose size equals the largest kept).
//
// One call labels the union mask of a sorted label list with full connectivity (26 neighbours on the [Z, Y, X] volume;
// a lower-rank mask is padded with leading unit axes, where this is skimage's 8 / 2 neighbours) by block-based
// union-find, then writes the copy of the volume with every masked voxel outside the largest components set to the
// background value:
//   local_kernel    one block per 4x8x32 tile: the mask from the stored dtype (label_compare.cuh), a union-find over
//                   the tile's 13 backward neighbours in shared memory, and every masked voxel's global parent set to
//                   the linear index of its tile-local root (the smallest index of the tile component).
//   merge_kernel    the same tiles: every masked voxel unites with its backward neighbours in another tile, in global
//                   memory.  A union always links the larger root under the smaller with atomicMin, so parent[i] <= i
//                   holds throughout and every union terminates whatever the interleaving.
//   count_kernel    one thread per voxel: parent[i] = root, and the component sizes size[root] summed per warp over
//                   the lanes that share a root (__match_any_sync) before one atomic per root and warp.
//   max_kernel      the largest size (block reduction, one atomicMax per block).
//   apply_kernel    out = seg, with background where the voxel is masked and its component is not of the largest size.
// Scratch: parent and size, two int32 volumes, plus one int32 for the largest size.
#include <algorithm>

#include "../../include/dinounet_b200.h"
#include "gemm_common.h"
#include "host_util.h"
#include "label_compare.cuh"

namespace b2u {

constexpr int kTX = 32, kTY = 8, kTZ = 4;    // tile: a warp spans a row, a thread walks the tile's depth
constexpr int kTileThreads = kTX * kTY;      // 256
constexpr int kTile = kTX * kTY * kTZ;       // 1024 voxels
constexpr int kFlatThreads = 256;

// The 13 neighbours (dz, dy, dx) that precede a voxel in C order, out of its 26.
__constant__ signed char kBack[13][3] = {{-1, -1, -1}, {-1, -1, 0}, {-1, -1, 1}, {-1, 0, -1}, {-1, 0, 0},
                                         {-1, 0, 1},   {-1, 1, -1}, {-1, 1, 0},  {-1, 1, 1},  {0, -1, -1},
                                         {0, -1, 0},   {0, -1, 1},  {0, 0, -1}};

struct Tiles {
  int Z, Y, X, tx, ty;  // tx, ty: tiles along x and y
  __device__ __forceinline__ void origin(long long b, int& z0, int& y0, int& x0) const {
    x0 = static_cast<int>(b % tx) * kTX;
    const long long r = b / tx;
    y0 = static_cast<int>(r % ty) * kTY;
    z0 = static_cast<int>(r / ty) * kTZ;
  }
  __device__ __forceinline__ int index(int z, int y, int x) const { return (z * Y + y) * X + x; }
};

// Root of i: parents only ever decrease, and a root is its own parent.  Volatile reads: other threads relink roots.
__device__ __forceinline__ int find_root(const volatile int* parent, int i) {
  int p;
  while ((p = parent[i]) != i) i = p;
  return i;
}

// Joins the trees of a and b (both masked).  atomicMin on the larger root either links it (it was still a root) or
// returns the parent another thread gave it meanwhile, which is smaller; the loop then joins that one.
__device__ __forceinline__ void unite(int* parent, int a, int b) {
  while (true) {
    a = find_root(parent, a);
    b = find_root(parent, b);
    if (a == b) return;
    if (a > b) {
      const int t = a;
      a = b;
      b = t;
    }
    const int old = atomicMin(parent + b, a);
    if (old == b) return;
    b = old;
  }
}

__global__ void __launch_bounds__(kTileThreads) local_kernel(const void* __restrict__ seg, int dtype, Tiles T,
                                                             const long long* __restrict__ labels, int n_labels,
                                                             int* __restrict__ parent) {
  __shared__ int sp[kTile];  // tile-local parent, -1 outside the mask or the volume
  int z0, y0, x0;
  T.origin(blockIdx.x, z0, y0, x0);
  const int dx = threadIdx.x % kTX, dy = threadIdx.x / kTX;
  const int x = x0 + dx, y = y0 + dy;
#pragma unroll
  for (int dz = 0; dz < kTZ; ++dz) {
    const int l = dz * kTileThreads + threadIdx.x, z = z0 + dz;
    const bool in = x < T.X && y < T.Y && z < T.Z;
    sp[l] = in && in_sorted_labels(seg, dtype, T.index(z, y, x), labels, n_labels) ? l : -1;
  }
  __syncthreads();
#pragma unroll
  for (int dz = 0; dz < kTZ; ++dz) {
    const int l = dz * kTileThreads + threadIdx.x;
    if (sp[l] < 0) continue;
    for (int k = 0; k < 13; ++k) {
      const int nz = dz + kBack[k][0], ny = dy + kBack[k][1], nx = dx + kBack[k][2];
      if (nz < 0 || ny < 0 || ny >= kTY || nx < 0 || nx >= kTX) continue;
      const int nl = (nz * kTY + ny) * kTX + nx;
      if (sp[nl] >= 0) unite(sp, l, nl);
    }
  }
  __syncthreads();
#pragma unroll
  for (int dz = 0; dz < kTZ; ++dz) {
    const int l = dz * kTileThreads + threadIdx.x, z = z0 + dz;
    if (x >= T.X || y >= T.Y || z >= T.Z) continue;
    int r = -1;
    if (sp[l] >= 0) {
      r = find_root(sp, l);
      r = T.index(z0 + r / kTileThreads, y0 + (r / kTX) % kTY, x0 + r % kTX);
    }
    parent[T.index(z, y, x)] = r;
  }
}

__global__ void __launch_bounds__(kTileThreads) merge_kernel(Tiles T, int* __restrict__ parent) {
  int z0, y0, x0;
  T.origin(blockIdx.x, z0, y0, x0);
  const int dx = threadIdx.x % kTX, dy = threadIdx.x / kTX;
  const int x = x0 + dx, y = y0 + dy;
  if (x >= T.X || y >= T.Y) return;
  for (int dz = 0; dz < kTZ; ++dz) {
    const int z = z0 + dz;
    if (z >= T.Z) break;
    const int i = T.index(z, y, x);
    if (parent[i] < 0) continue;
    for (int k = 0; k < 13; ++k) {
      const int ez = dz + kBack[k][0], ey = dy + kBack[k][1], ex = dx + kBack[k][2];
      if (ez >= 0 && ey >= 0 && ey < kTY && ex >= 0 && ex < kTX) continue;  // same tile: joined by local_kernel
      const int nz = z + kBack[k][0], ny = y + kBack[k][1], nx = x + kBack[k][2];
      if (nz < 0 || ny < 0 || ny >= T.Y || nx < 0 || nx >= T.X) continue;
      const int j = T.index(nz, ny, nx);
      if (parent[j] >= 0) unite(parent, i, j);
    }
  }
}

// One voxel per thread and no early exit before the ballot: the warp's lanes must all reach it.
__global__ void __launch_bounds__(kFlatThreads) count_kernel(int n, int* __restrict__ parent, int* __restrict__ size) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  int r = -1;
  if (i < n && parent[i] >= 0) {
    r = find_root(parent, static_cast<int>(i));
    parent[i] = r;
  }
  const unsigned active = __ballot_sync(0xffffffffu, r >= 0);
  if (r >= 0) {
    const unsigned peers = __match_any_sync(active, r);
    if ((threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(size + r, __popc(peers));
  }
}

__global__ void __launch_bounds__(kFlatThreads) max_kernel(int n, const int* __restrict__ size, int* __restrict__ best) {
  __shared__ int red[kFlatThreads / 32];
  int m = 0;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    m = max(m, size[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_down_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x / 32] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    m = threadIdx.x < kFlatThreads / 32 ? red[threadIdx.x] : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_down_sync(0xffffffffu, m, o));
    if (threadIdx.x == 0 && m > 0) atomicMax(best, m);
  }
}

// T: the stored element's bits (1, 2 or 4 bytes); background: the background value in those bits.
template <typename T>
__global__ void __launch_bounds__(kFlatThreads) apply_kernel(int n, const T* __restrict__ seg,
                                                             const int* __restrict__ parent,
                                                             const int* __restrict__ size,
                                                             const int* __restrict__ best, T background,
                                                             T* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = parent[i];
  out[i] = r >= 0 && size[r] != *best ? background : seg[i];
}

}  // namespace b2u

using namespace b2u;

extern "C" int b2u_pp_largest_component(const void* seg, int32_t dtype, int32_t Z, int32_t Y, int32_t X,
                                        const int64_t* labels, int32_t n_labels, int64_t background, void* out,
                                        int32_t* work, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!seg || !out || !work || (n_labels > 0 && !labels))
    return set_error(-1, "b2u_pp_largest_component: null pointer");
  if (Z <= 0 || Y <= 0 || X <= 0 || static_cast<long long>(Z) * Y * X > 0x7fffffffLL)
    return set_error(-1, "b2u_pp_largest_component: bad shape %dx%dx%d (1 to 2^31 - 1 voxels)", Z, Y, X);
  if (dtype < B2U_EVAL_U8 || dtype > B2U_EVAL_F32)
    return set_error(-1, "b2u_pp_largest_component: dtype code %d", dtype);
  if (n_labels < 0) return set_error(-1, "b2u_pp_largest_component: %d labels", n_labels);
  const int n = Z * Y * X;
  int* parent = work;
  int* size = work + n;
  int* best = work + 2LL * n;
  if (cudaMemsetAsync(size, 0, (static_cast<size_t>(n) + 1) * sizeof(int), stream) != cudaSuccess)
    return set_error(-1, "b2u_pp_largest_component: cudaMemsetAsync failed");
  Tiles T{Z, Y, X, (X + kTX - 1) / kTX, (Y + kTY - 1) / kTY};
  const long long tiles = static_cast<long long>(T.tx) * T.ty * ((Z + kTZ - 1) / kTZ);
  local_kernel<<<static_cast<unsigned>(tiles), kTileThreads, 0, stream>>>(
      seg, dtype, T, reinterpret_cast<const long long*>(labels), n_labels, parent);
  int rc = check_launch("pp_local");
  if (rc) return rc;
  merge_kernel<<<static_cast<unsigned>(tiles), kTileThreads, 0, stream>>>(T, parent);
  if ((rc = check_launch("pp_merge"))) return rc;
  const unsigned flat = static_cast<unsigned>((static_cast<long long>(n) + kFlatThreads - 1) / kFlatThreads);
  count_kernel<<<flat, kFlatThreads, 0, stream>>>(n, parent, size);
  if ((rc = check_launch("pp_count"))) return rc;
  const unsigned red_blocks = std::min<unsigned>(flat, static_cast<unsigned>(num_sms()) * 8);
  max_kernel<<<red_blocks, kFlatThreads, 0, stream>>>(n, size, best);
  if ((rc = check_launch("pp_max"))) return rc;
  switch (dtype) {
    case B2U_EVAL_U8:
    case B2U_EVAL_I8:
      apply_kernel<uint8_t><<<flat, kFlatThreads, 0, stream>>>(n, static_cast<const uint8_t*>(seg), parent, size, best,
                                                                static_cast<uint8_t>(background),
                                                                static_cast<uint8_t*>(out));
      break;
    case B2U_EVAL_I16:
    case B2U_EVAL_U16:
      apply_kernel<uint16_t><<<flat, kFlatThreads, 0, stream>>>(n, static_cast<const uint16_t*>(seg), parent, size,
                                                                 best, static_cast<uint16_t>(background),
                                                                 static_cast<uint16_t*>(out));
      break;
    default:
      apply_kernel<uint32_t><<<flat, kFlatThreads, 0, stream>>>(n, static_cast<const uint32_t*>(seg), parent, size,
                                                                 best, static_cast<uint32_t>(background),
                                                                 static_cast<uint32_t*>(out));
  }
  return check_launch("pp_apply");
}
