// Host-side helpers shared by the C-ABI translation units: error reporting, launch accounting, TMA descriptor encode.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2u {

int set_error(int code, const char* fmt, ...);
// Index of the current CUDA device (0..63): cudaFuncSetAttribute is PER DEVICE, so "already configured" flags are arrays.
int current_device_index();
// cudaGetLastError() after a launch; bumps the launch counter on success.
int check_launch(const char* what);
// cuTensorMapEncodeTiled through cudaGetDriverEntryPoint (no link-time libcuda dependency): 16-bit elements,
// 128B swizzle, zero OOB fill.  `strides` are byte strides of dims 1..rank-1.
int encode_tensor_map(CUtensorMap* map, int dtype, int rank, const void* base, const cuuint64_t* dims,
                      const cuuint64_t* strides, const cuuint32_t* box, const cuuint32_t* elem_strides);

int get_option(int key);

// numpy's pairwise sum of a contiguous float64 x[n] (preprocess.cu's tree, shared with the float32 ZScore statistics):
// the sum lands in work[0].  work: ceil(n / 8) doubles.
int pairwise_sum_f64(const double* x, long long n, double* work, cudaStream_t stream);
// numpy's float32 pairwise sum of each of `planes` contiguous runs of n (run p at x + p * n) into work[p * ws]; sq: of
// (x - mean[p])^2.  work: planes * ws floats, ws >= ceil(n / 8).
int pairwise_sum_planes_f32(const float* x, long long n, int planes, int sq, const float* mean, float* work,
                            long long ws, cudaStream_t stream);
// Exact min / max of each of `planes` contiguous runs of n into lo[p], hi[p].
int minmax_planes_f32(const float* x, long long n, int planes, float* lo, float* hi, cudaStream_t stream);

// Programmatic dependent launch (PDL), OPT-IN (option 5 = 1): every kernel of the forward plan can be launched with
// cudaLaunchAttributeProgrammaticStreamSerialization; each calls `griddepcontrol.wait` before it touches global memory
// (after its barrier-init / tensormap-prefetch prologue where it has one) and the persistent GEMM / attention
// kernels call `griddepcontrol.launch_dependents` when a CTA has finished its tiles.  Default off (the plan's persistent
// kernels hold most of an SM's shared memory, so a dependent cannot become resident before its predecessor's CTAs exit);
// with the attribute off `griddepcontrol.wait` is a no-op.
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = get_option(5) == 1 ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

}  // namespace b2u
