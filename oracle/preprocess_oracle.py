"""Restatement of the reference's case preprocessing for 2D configurations (`DefaultPreprocessor.run_case_npy`,
preprocessing/preprocessors/default_preprocessor.py:40-118) on the host:

    np.copy, transpose_forward, crop_to_nonzero      the crop is the whole volume (cropping.py:34 sets every voxel of the
                                                    nonzero mask), so the bbox is [[0, s], ...] and the seg all zeros
    per-channel normalization (float32)              default_normalization_schemes.py
    resample_data_or_seg_to_shape(order=3)           default_resampling.py:77-216, Z unchanged; per slice (separate z
                                                    along axis 0) or one 3-D resize per channel

Three pieces are restated so that the GPU tests need neither scipy nor numpy's reduction internals:

* `zoom_order3_torch64`: scipy `ndimage.zoom(order=3, mode='nearest', grid_mode=True)` on float64 in torch float64,
  bit for bit: np.pad(12, 'edge') on every axis, the order-3 spline prefilter per axis (axis 0 first) with scipy's
  initial conditions for mode 'nearest' and the correctly rounded pole, then NI_ZoomShift's coordinates (shifted by the
  12 padded samples), weights and tap order.  `tests/test_preprocess_cpu.py` pins it to scipy.
* `pairwise_sum_f32`: numpy's float32 `add.reduce` over one run, its pairwise_sum tree (leaves of <= 128 elements in 8
  lanes, splits at n/2 rounded down to a multiple of 8); `mean_std_f32` forms `mean()` / `std()` from it as numpy's
  _methods does (float32 sum / intp count in float64, rounded to float32; sqrt in float32).
* the five normalization schemes, elementwise in numpy float32.

skimage's `resize(order=3, mode='edge', anti_aliasing=False)` on float64 is taken to be the scipy call followed by a clip
to the input's [min, max] (skimage >= 0.19.3, `_clip_warp_output` with clip=True): that is read from skimage's source;
skimage is not a dependency here and the equivalence is not checked by this repository's tests.  The same clip applies
to skimage's order-1 resize in the export (oracle/export_oracle.py), where it can change a value only by a rounding of
the float64 interpolation, which the fp16 cast hides; the export is left as it is.
"""
import math
from typing import List, Sequence

import numpy as np
import torch

NPAD = 12                                     # scipy's _prepad_for_spline_filter for mode 'nearest'
POLE = -0.267949192431122706472553658494127633  # the order-3 pole sqrt(3) - 2, correctly rounded (as scipy has it)
ANISO_THRESHOLD = 3
SCHEMES = ("ZScoreNormalization", "CTNormalization", "NoNormalization", "RescaleTo01Normalization",
           "RGBTo01Normalization")


def filter_consts(n: int) -> List[float]:
    """{pole, pole^n, gain, pole / (1 - pole^2n), pole / (pole - 1)} for a line of n samples (host libm pow)."""
    z = POLE
    zn = math.pow(z, n)
    return [z, zn, (1.0 - z) * (1.0 - 1.0 / z), z / (1 - zn * zn), z / (z - 1)]


def spline_filter_axis(c: torch.Tensor, axis: int) -> torch.Tensor:
    """scipy's order-3 spline_filter1d(mode='nearest') along `axis` of a float64 tensor (all lines at once)."""
    c = c.movedim(axis, -1).clone()
    n = c.shape[-1]
    z, zn, gain, f_causal, f_anti = filter_consts(n)
    c = c * gain
    c0 = c[..., 0].clone()
    s = c0 + zn * c[..., n - 1]
    zi = z
    for i in range(1, n):
        s = s + zi * (c[..., i] + zn * c[..., n - 1 - i])
        zi = zi * z
    c[..., 0] = s * f_causal + c0
    for i in range(1, n):
        c[..., i] = c[..., i] + z * c[..., i - 1]
    c[..., n - 1] = c[..., n - 1] * f_anti
    for i in range(n - 2, -1, -1):
        c[..., i] = z * (c[..., i + 1] - c[..., i])
    return c.movedim(-1, axis)


def _cubic_taps(n_in: int, n_out: int):
    """NI_ZoomShift along one axis: first tap (index into the padded axis) and the 4 weights per output sample."""
    k = torch.arange(n_out, dtype=torch.float64)
    cc = (k + 0.5) * (n_in / n_out) - 0.5 + float(NPAD)
    fl = torch.floor(cc)
    y = cc - fl
    z = 1.0 - y
    w0 = z * z * z / 6.0
    w1 = (y * y * (y - 2.0) * 3.0 + 4.0) / 6.0
    w2 = (z * z * (z - 2.0) * 3.0 + 4.0) / 6.0
    w3 = 1.0 - w0 - w1 - w2
    return fl.long() - 1, (w0, w1, w2, w3)


def zoom_order3_torch64(x: torch.Tensor, out_shape: Sequence[int]) -> torch.Tensor:
    """scipy.ndimage.zoom(x, order=3, mode='nearest', grid_mode=True) of a 2-D or 3-D float64 array, in torch."""
    x = torch.as_tensor(x, dtype=torch.float64)
    c = torch.from_numpy(np.pad(x.numpy(), NPAD, mode="edge"))
    for axis in range(c.ndim):
        c = spline_filter_axis(c, axis)
    taps = [_cubic_taps(i, o) for i, o in zip(x.shape, out_shape)]
    t = torch.zeros(tuple(int(o) for o in out_shape), dtype=torch.float64)
    if x.ndim == 2:
        (sy, wy), (sx, wx) = taps
        for a in range(4):
            rows = c[sy + a]
            for b in range(4):
                t = t + rows[:, sx + b] * wy[a][:, None] * wx[b][None, :]
        return t
    (sz, wz), (sy, wy), (sx, wx) = taps
    for a in range(4):
        planes = c[sz + a]
        for b in range(4):
            rows = planes[:, sy + b]
            for d in range(4):
                t = t + rows[:, :, sx + d] * wz[a][:, None, None] * wy[b][None, :, None] * wx[d][None, None, :]
    return t


def resize_order3(x: torch.Tensor, out_shape: Sequence[int]) -> torch.Tensor:
    """skimage resize(order=3, mode='edge', anti_aliasing=False) on float64: the zoom clipped to x's [min, max]."""
    x = torch.as_tensor(x, dtype=torch.float64)
    return zoom_order3_torch64(x, out_shape).clamp(float(x.min()), float(x.max()))


def resample_channel(x32, H: int, W: int, three_d: bool) -> torch.Tensor:
    """float32 [Z, h, w] -> float32 [Z, H, W] as resample_data_or_seg (Z unchanged): per slice or one 3-D resize."""
    x = torch.as_tensor(np.ascontiguousarray(x32), dtype=torch.float64)
    if three_d:
        return resize_order3(x, (x.shape[0], H, W)).float()
    return torch.stack([resize_order3(x[z], (H, W)) for z in range(x.shape[0])]).float()


# ---- numpy's float32 reductions


def _leaves(n: int):
    out = []

    def rec(o, m):
        if m <= 128:
            out.append((o, m))
            return
        m2 = m // 2
        m2 -= m2 % 8
        rec(o, m2)
        rec(o + m2, m - m2)

    rec(0, n)
    return out


def pairwise_sum_f32(a) -> np.float32:
    """numpy's float32 sum of a 1-D run (pairwise_sum in numpy's loops_utils)."""
    a = np.ascontiguousarray(a, dtype=np.float32).ravel()
    n = a.size
    if n < 8:
        res = np.float32(0)
        for v in a:
            res = np.float32(res + v)
        return res
    leaves = _leaves(n)
    sums = {}
    by_len = {}
    for o, m in leaves:
        by_len.setdefault(m, []).append(o)
    for m, offs in by_len.items():
        offs = np.asarray(offs)
        vals = a[offs[:, None] + np.arange(m)[None, :]]
        r = vals[:, :8].copy()
        end = m - m % 8
        for i in range(8, end, 8):
            r += vals[:, i:i + 8]
        res = ((r[:, 0] + r[:, 1]) + (r[:, 2] + r[:, 3])) + ((r[:, 4] + r[:, 5]) + (r[:, 6] + r[:, 7]))
        for i in range(end, m):
            res = res + vals[:, i]
        sums.update(zip(offs.tolist(), res.tolist()))

    def comb(o, m):
        if m <= 128:
            return np.float32(sums[o])
        m2 = m // 2
        m2 -= m2 % 8
        return np.float32(comb(o, m2) + comb(o + m2, m - m2))

    return comb(0, n)


def mean_std_f32(a):
    """numpy's float32 `a.mean()` and `a.std()` of the elements of `a` in the given (flattened C) order."""
    a = np.ascontiguousarray(a, dtype=np.float32).ravel()
    n = a.size
    mean = np.float32(np.float64(pairwise_sum_f32(a)) / np.float64(n))
    d = a - mean
    ss = pairwise_sum_f32(d * d)
    std = np.sqrt(np.float32(np.float64(ss) / np.float64(n)))
    return mean, std


def memory_order(view: np.ndarray) -> np.ndarray:
    """The elements of a view of a C-contiguous array in memory order (numpy's reduction order without a mask)."""
    order = np.argsort([-s for s in view.strides], kind="stable")
    return np.ascontiguousarray(view.transpose(order)).ravel()


# ---- normalization (default_normalization_schemes.py), on a float32 view, as the reference writes it


def normalize_channel(image: np.ndarray, scheme: str, use_mask: bool, props: dict) -> np.ndarray:
    """float32 result of the reference's normalizer on the channel view `image` (transposed; memory of the copy)."""
    image = np.asarray(image, dtype=np.float32)
    if scheme == "ZScoreNormalization":
        mean, std = mean_std_f32(image.ravel() if use_mask else memory_order(image))
        d = np.float32(1e-8) if np.float32(1e-8) > std else std
        return (image - mean) / d
    if scheme == "CTNormalization":
        out = np.clip(image, np.float32(props["percentile_00_5"]), np.float32(props["percentile_99_5"]))
        out = out - np.float32(props["mean"])
        return out / np.float32(max(props["std"], 1e-8))
    if scheme == "NoNormalization":
        return image.copy()
    if scheme == "RescaleTo01Normalization":
        out = image - image.min()
        return out / max(out.max(), np.float32(1e-8))
    if scheme == "RGBTo01Normalization":
        assert image.min() >= 0 and image.max() <= 255
        return image / np.float32(255.0)
    raise NotImplementedError(scheme)


# ---- the case


def lowres_axis(spacing) -> np.ndarray:
    spacing = np.asarray(spacing, dtype=float)
    return np.where(max(spacing) / spacing == 1)[0]


def separate_z_axis(current_spacing, new_spacing):
    """resample_data_or_seg_to_shape(force_separate_z=None): the separate-z axis, or None for one 3-D resize."""
    for sp in (current_spacing, new_spacing):
        sp = np.asarray(sp, dtype=float)
        if np.max(sp) / np.min(sp) > ANISO_THRESHOLD:
            axis = lowres_axis(sp)
            return int(axis[0]) if len(axis) == 1 else None
    return None


def compute_new_shape(old_shape, old_spacing, new_spacing):
    return [int(round(i / j * k)) for i, j, k in zip(old_spacing, new_spacing, old_shape)]


def preprocess_case(data: np.ndarray, spacing: Sequence[float], transpose_forward: Sequence[int],
                    config_spacing: Sequence[float], schemes: Sequence[str], use_mask: Sequence[bool],
                    intensity_props: dict):
    """run_case_npy for a 2D configuration with the restated normalizers and resampler.  Returns the float32 data
    [C, *new_shape] and the three properties run_case_npy adds."""
    data = np.copy(data).astype(np.float32)
    tf = list(transpose_forward)
    view = data.transpose([0, *[i + 1 for i in tf]])
    original_spacing = [spacing[i] for i in tf]
    shape = tuple(int(s) for s in view.shape[1:])
    target_spacing = [original_spacing[0], *config_spacing] if len(config_spacing) < 3 else list(config_spacing)
    new_shape = compute_new_shape(shape, original_spacing, target_spacing)
    normed = np.stack([normalize_channel(view[c], schemes[c], bool(use_mask[c]), intensity_props.get(str(c), {}))
                       for c in range(view.shape[0])])
    props = {"shape_before_cropping": shape, "bbox_used_for_cropping": [[0, s] for s in shape],
             "shape_after_cropping_and_before_resampling": shape}
    if tuple(new_shape) == shape:
        return normed, props
    assert new_shape[0] == shape[0]
    axis = separate_z_axis(original_spacing, target_spacing)
    assert axis in (None, 0)
    out = np.stack([resample_channel(normed[c], new_shape[1], new_shape[2], axis is None).numpy()
                    for c in range(normed.shape[0])])
    return out, props
