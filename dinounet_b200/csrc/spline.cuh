// scipy.ndimage's order-3 B-spline arithmetic, operation for operation (every product and sum an explicit _rn
// intrinsic, so nvcc forms no FMA), shared by the case resampling (preprocess.cu) and the training augmentation
// (augmentation.cu).
#pragma once

namespace b2u {

constexpr int kPad = 12;  // scipy's _prepad_for_spline_filter for mode 'nearest'

// Reflect boundaries (mode 'nearest' after scipy's edge pre-padding): {pole, z^n, gain, z / (1 - z^2n), z / (z - 1)}.
// Mirror boundaries (mode 'constant' / 'mirror', no pre-padding): {pole, z^(n-1), gain, unused, z^2 - 1}.
struct FilterConsts {
  double z, zn, gain, f_causal, f_anti;
};

// scipy's NI_SplineFilter1D on one line of n samples at stride st (ni_splines.c: gain, causal init, causal pass,
// anti-causal init, anti-causal pass).  kMirror selects _init_causal_mirror / _init_anticausal_mirror, otherwise the
// reflect pair.
template <bool kMirror>
__device__ __forceinline__ void spline_filter_line(double* p, long long st, int n, const FilterConsts& k) {
  if (kMirror && n == 1) return;
  for (int i = 0; i < n; ++i) p[i * st] = __dmul_rn(p[i * st], k.gain);
  const double c0 = p[0];
  double s = __dadd_rn(c0, __dmul_rn(k.zn, p[(n - 1) * st]));
  double zi = k.z;
  for (int i = 1; i < (kMirror ? n - 1 : n); ++i) {
    s = __dadd_rn(s, __dmul_rn(zi, __dadd_rn(p[i * st], __dmul_rn(k.zn, p[(n - 1 - i) * st]))));
    zi = __dmul_rn(zi, k.z);
  }
  if (kMirror)
    p[0] = __ddiv_rn(s, __dsub_rn(1.0, __dmul_rn(k.zn, k.zn)));
  else
    p[0] = __dadd_rn(__dmul_rn(s, k.f_causal), c0);
  double prev = p[0];
  for (int i = 1; i < n; ++i) {
    prev = __dadd_rn(p[i * st], __dmul_rn(k.z, prev));
    p[i * st] = prev;
  }
  double next;
  if (kMirror)
    next = __ddiv_rn(__dmul_rn(k.z, __dadd_rn(__dmul_rn(k.z, p[(n - 2) * st]), p[(n - 1) * st])), k.f_anti);
  else
    next = __dmul_rn(p[(n - 1) * st], k.f_anti);
  p[(n - 1) * st] = next;
  for (int i = n - 2; i >= 0; --i) {
    next = __dmul_rn(k.z, __dsub_rn(next, p[i * st]));
    p[i * st] = next;
  }
}

struct Taps3 {
  int start;  // first tap
  double w[4];
};

// get_spline_interpolation_weights(order 3) at coordinate cc: taps floor(cc) - 1 .. + 2.
__device__ __forceinline__ Taps3 cubic_taps_at(double cc) {
  const double fl = floor(cc);
  const double y = __dsub_rn(cc, fl), z = __dsub_rn(1.0, y);
  Taps3 t;
  t.start = static_cast<int>(fl) - 1;
  t.w[0] = __ddiv_rn(__dmul_rn(__dmul_rn(z, z), z), 6.0);
  t.w[1] = __ddiv_rn(__dadd_rn(__dmul_rn(__dmul_rn(__dmul_rn(y, y), __dsub_rn(y, 2.0)), 3.0), 4.0), 6.0);
  t.w[2] = __ddiv_rn(__dadd_rn(__dmul_rn(__dmul_rn(__dmul_rn(z, z), __dsub_rn(z, 2.0)), 3.0), 4.0), 6.0);
  t.w[3] = __dsub_rn(__dsub_rn(__dsub_rn(1.0, t.w[0]), t.w[1]), t.w[2]);
  return t;
}

// NI_ZoomShift with grid_mode on an edge-padded axis: cc = ((k + 0.5) * zoom - 0.5) + 12.
__device__ __forceinline__ Taps3 cubic_taps(int k, double zoom) {
  return cubic_taps_at(__dadd_rn(__dsub_rn(__dmul_rn(__dadd_rn(static_cast<double>(k), 0.5), zoom), 0.5),
                                 static_cast<double>(kPad)));
}

// The 16-tap sum of a 2-D zoom on a padded coefficient plane (row pitch Wp): t += coef * w_y * w_x, x fastest.
__device__ __forceinline__ double cubic16(const double* plane, long long Wp, const Taps3& ty, const Taps3& tx) {
  double t = 0.0;
#pragma unroll
  for (int b = 0; b < 4; ++b) {
    const double* row = plane + (ty.start + b) * Wp + tx.start;
#pragma unroll
    for (int c = 0; c < 4; ++c) t = __dadd_rn(t, __dmul_rn(__dmul_rn(row[c], ty.w[b]), tx.w[c]));
  }
  return t;
}

}  // namespace b2u
