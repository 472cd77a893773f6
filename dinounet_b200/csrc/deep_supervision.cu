// Deep-supervision targets on the device: nnU-Net's DownsampleSegForDSTransform2(scales, order=0)
// (batchgenerators resize_segmentation -> skimage.transform.resize(seg.astype(float), round(shape * s), order=0,
// mode="edge", anti_aliasing=False), cast back).  skimage's resize maps output index o of an axis shrunk by an integer
// factor f to the input coordinate (o + 0.5) * f - 0.5 and takes the nearest sample with ties rounded up (ndimage's
// order-0 floor(x + 0.5)), i.e. input index f*o + f/2: 2o+1 at f = 2, 4o+2 at f = 4.  Only integer factors that divide
// the extent are taken (np.round(shape * s) is then exact); anything else is rejected before the launch.
// One launch writes every scale: thread per output element over the concatenated outputs, consecutive threads
// consecutive output columns (coalesced stores; the gathers read every f-th element of an input row).
#include <algorithm>

#include "../../include/dinounet_b200.h"
#include "gemm_common.h"
#include "host_util.h"

namespace b2u {
namespace {

constexpr int kT = 256;

struct DsScales {
  long long end[B2U_DS_MAX_SCALES];   // exclusive prefix end of each scale's outputs in the concatenated index space
  int fy[B2U_DS_MAX_SCALES], fx[B2U_DS_MAX_SCALES];
  void* dst[B2U_DS_MAX_SCALES];
  int n;
};

template <typename T>
__global__ void __launch_bounds__(kT) ds_targets_kernel(const T* __restrict__ src, int H, int W, DsScales sc, long long total) {
  for (long long i = blockIdx.x * static_cast<long long>(kT) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kT) {
    int s = 0;
    while (i >= sc.end[s]) ++s;
    const long long j = i - (s ? sc.end[s - 1] : 0);
    const int fy = sc.fy[s], fx = sc.fx[s];
    const int w = W / fx, h = H / fy;
    const int ox = static_cast<int>(j % w);
    const long long r = j / w;
    const int oy = static_cast<int>(r % h);
    const long long plane = r / h;
    const T v = src[(plane * H + static_cast<long long>(oy) * fy + fy / 2) * W + static_cast<long long>(ox) * fx + fx / 2];
    static_cast<T*>(sc.dst[s])[j] = v;
  }
}

}  // namespace
}  // namespace b2u

using namespace b2u;

extern "C" int b2u_ds_targets(const b2u_ds_targets_params* p, b2u_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!p || !p->src) return set_error(-1, "b2u_ds_targets: null pointer");
  if (p->dtype != B2U_DS_INT16 && p->dtype != B2U_DS_FP32) return set_error(-1, "b2u_ds_targets: dtype %d", p->dtype);
  if (p->B <= 0 || p->C <= 0 || p->H <= 0 || p->W <= 0)
    return set_error(-1, "b2u_ds_targets: bad shape B=%d C=%d %dx%d", p->B, p->C, p->H, p->W);
  if (p->nscales < 1 || p->nscales > B2U_DS_MAX_SCALES)
    return set_error(-1, "b2u_ds_targets: 1 <= nscales <= %d, got %d", B2U_DS_MAX_SCALES, p->nscales);
  DsScales sc = {};
  sc.n = p->nscales;
  long long total = 0;
  const long long planes = static_cast<long long>(p->B) * p->C;
  for (int s = 0; s < p->nscales; ++s) {
    const int fy = p->fy[s], fx = p->fx[s];
    if (fy < 1 || fx < 1 || p->H % fy || p->W % fx)
      return set_error(-1, "b2u_ds_targets: scale %d: factors %dx%d do not divide %dx%d", s, fy, fx, p->H, p->W);
    if (!p->dst[s]) return set_error(-1, "b2u_ds_targets: scale %d: null output", s);
    total += planes * (p->H / fy) * (p->W / fx);
    sc.end[s] = total;
    sc.fy[s] = fy;
    sc.fx[s] = fx;
    sc.dst[s] = p->dst[s];
  }
  const long long blocks = std::min<long long>((total + kT - 1) / kT, 132LL * 16);
  if (p->dtype == B2U_DS_INT16)
    ds_targets_kernel<int16_t><<<static_cast<unsigned>(blocks), kT, 0, stream>>>(static_cast<const int16_t*>(p->src), p->H,
                                                                                 p->W, sc, total);
  else
    ds_targets_kernel<float><<<static_cast<unsigned>(blocks), kT, 0, stream>>>(static_cast<const float*>(p->src), p->H, p->W,
                                                                               sc, total);
  return check_launch("ds_targets");
}
