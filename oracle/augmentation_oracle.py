"""CPU restatement of nnU-Net's 2-D training augmentation (`nnUNetTrainer.get_training_transforms`,
nnUNetTrainer.py:684-775, batchgenerators 0.25), for tests only.  batchgenerators is not needed.

The transforms are driven by a parameter record of `dinounet_b200.augmentation.sample_augmentation_params` (every
random decision of the pipeline) and by the Gaussian noise field as an array, so that the device pipeline and this
restatement see the same draws.  `draw_decisions` replays batchgenerators' loops on a RandomState and records what
each transform decided, for the tests that pin the sampler's draw order.

Pieces restated bit for bit in torch float64 (pinned to scipy by tests/test_augmentation_cpu.py):
* `map_coordinates_torch64`: scipy `ndimage.map_coordinates(x, coords, order=1 or 3, mode='constant', cval)`:
  the order-3 spline prefilter along axis 0 then 1 with the mirror initial conditions (scipy uses them for 'constant',
  with no pre-padding), then NI_GeometricTransform: cval where a coordinate lies outside [0, n-1], otherwise the taps
  floor(c) - 1 .. + 2 (order 3) or floor(c) .. + 1 (order 1), mirrored at the edges, summed with the last axis fastest.
* `gaussian_filter1d_torch64`: scipy `gaussian_filter1d(x32, sigma, axis)` (mode 'reflect', truncate 4) on a float32
  array: the symmetric correlation of NI_Correlate1D, x[i] w[0] + sum over k = r .. 1 of (x[i-k] + x[i+k]) w[k], in
  float64, rounded once to float32.
The rest is numpy on float32 arrays as batchgenerators writes it (python floats are weak scalars under NEP 50), and the
low-resolution step reuses oracle/preprocess_oracle.py's skimage resize (order-3 zoom clipped to the input's range).

The coordinates of the spatial transform are formed elementwise, c0 cos + c1 sin and c1 cos - c0 sin, each product
and sum rounded once; batchgenerators forms them with `np.dot`, where a BLAS may fuse a multiply-add.
"""
import math

import numpy as np
import torch

from . import preprocess_oracle as PRE

POLE = PRE.POLE


# ---- scipy.ndimage restatements -------------------------------------------------------------------------------------


def mirror_filter_consts(n: int):
    """{pole, pole^(n-1) (host libm), gain, pole^2 - 1} of scipy's order-3 filter with mirror boundaries."""
    z = POLE
    return [z, math.pow(z, n - 1), (1.0 - z) * (1.0 - 1.0 / z), z * z - 1.0]


def spline_filter_mirror_axis(c: torch.Tensor, axis: int) -> torch.Tensor:
    """scipy's order-3 spline_filter1d along `axis` for mode 'constant' / 'mirror' (float64, all lines at once)."""
    c = c.movedim(axis, -1).clone()
    n = c.shape[-1]
    if n == 1:
        return c.movedim(-1, axis)
    z, zn1, gain, zz1 = mirror_filter_consts(n)
    c = c * gain
    s = c[..., 0] + zn1 * c[..., n - 1]
    zi = z
    for i in range(1, n - 1):
        s = s + zi * (c[..., i] + zn1 * c[..., n - 1 - i])
        zi = zi * z
    c[..., 0] = s / (1.0 - zn1 * zn1)
    for i in range(1, n):
        c[..., i] = c[..., i] + z * c[..., i - 1]
    c[..., n - 1] = z * (z * c[..., n - 2] + c[..., n - 1]) / zz1
    for i in range(n - 2, -1, -1):
        c[..., i] = z * (c[..., i + 1] - c[..., i])
    return c.movedim(-1, axis)


def _mirror_index(idx: torch.Tensor, n: int) -> torch.Tensor:
    if n <= 1:
        return torch.zeros_like(idx)
    s2 = 2 * n - 2
    idx = idx.clone()
    neg = idx < 0
    i = s2 * torch.div(-idx, s2, rounding_mode="trunc") + idx
    idx = torch.where(neg, torch.where(i <= 1 - n, i + s2, -i), idx)
    big = idx >= n
    i = idx - s2 * torch.div(idx, s2, rounding_mode="trunc")
    i = torch.where(i >= n, s2 - i, i)
    return torch.where(big, i, idx)


def _weights(cc: torch.Tensor, order: int):
    """get_spline_interpolation_weights: (first tap, [w0 .. w_order]) per coordinate."""
    fl = torch.floor(cc)
    y = cc - fl
    if order == 1:
        w0 = 1.0 - y
        return fl.long(), [w0, 1.0 - w0]
    z = 1.0 - y
    w1 = (y * y * (y - 2.0) * 3.0 + 4.0) / 6.0
    w2 = (z * z * (z - 2.0) * 3.0 + 4.0) / 6.0
    w0 = z * z * z / 6.0
    w3 = 1.0 - w0 - w1 - w2
    return fl.long() - 1, [w0, w1, w2, w3]


def map_coordinates_torch64(x, c0, c1, order: int, cval: float = 0.0, prefiltered: bool = False) -> torch.Tensor:
    """scipy.ndimage.map_coordinates(x, [c0, c1], order, mode='constant', cval) of a 2-D array, in torch float64.
    prefiltered: x already holds the spline coefficients (order 3)."""
    x = torch.as_tensor(np.asarray(x), dtype=torch.float64) if not isinstance(x, torch.Tensor) else x.double()
    c0 = torch.as_tensor(np.asarray(c0), dtype=torch.float64)
    c1 = torch.as_tensor(np.asarray(c1), dtype=torch.float64)
    h, w = x.shape
    coef = x
    if order == 3 and not prefiltered:
        coef = spline_filter_mirror_axis(spline_filter_mirror_axis(x, 0), 1)
    s0, w0 = _weights(c0, order)
    s1, w1 = _weights(c1, order)
    t = torch.zeros(c0.shape, dtype=torch.float64)
    for a in range(order + 1):
        ia = _mirror_index(s0 + a, h)
        for b in range(order + 1):
            ib = _mirror_index(s1 + b, w)
            t = t + coef[ia, ib] * w0[a] * w1[b]
    inside = (c0 >= 0) & (c0 <= h - 1) & (c1 >= 0) & (c1 <= w - 1)
    return torch.where(inside, t, torch.full_like(t, cval))


def gaussian_kernel1d(sigma: float):
    """scipy's _gaussian_kernel1d(sigma, 0, radius) with radius int(4 sigma + 0.5): the float64 weights."""
    radius = int(4.0 * float(sigma) + 0.5)
    x = np.arange(-radius, radius + 1)
    phi = np.exp(-0.5 / (sigma * sigma) * x ** 2)
    return phi / phi.sum()


def gaussian_filter1d_torch64(x32, sigma: float, axis: int) -> np.ndarray:
    """scipy.ndimage.gaussian_filter1d(x32, sigma, axis) of a float32 array (mode 'reflect'): float32 result."""
    wts = torch.from_numpy(gaussian_kernel1d(sigma)[::-1].copy())
    r = (wts.numel() - 1) // 2
    x = torch.as_tensor(np.asarray(x32, dtype=np.float32)).double().movedim(axis, -1)
    n = x.shape[-1]
    idx = torch.arange(-r, n + r)
    while bool(((idx < 0) | (idx >= n)).any()):   # half-sample symmetric, repeated for lines shorter than r
        idx = torch.where(idx < 0, -idx - 1, idx)
        idx = torch.where(idx >= n, 2 * n - idx - 1, idx)
    ext = x[..., idx]
    out = ext[..., r:r + n] * wts[r]
    for k in range(r, 0, -1):
        out = out + (ext[..., r - k:r - k + n] + ext[..., r + k:r + k + n]) * wts[r - k]
    return out.float().movedim(-1, axis).numpy()


def gaussian_filter_2d(x32, sigma: float) -> np.ndarray:
    """scipy.ndimage.gaussian_filter(x32, sigma) of a 2-D float32 array: axis 0, then axis 1, float32 in between."""
    return gaussian_filter1d_torch64(gaussian_filter1d_torch64(x32, sigma, 0), sigma, 1)


# ---- batchgenerators' transforms on the parameter record ---------------------------------------------------------


def spatial_coords(p, b: int, in_shape, out_shape):
    """augment_spatial's coordinates for sample b (create_zero_centered_coordinate_mesh, rotate, scale, centre)."""
    H, W = out_shape
    c0 = np.arange(H, dtype=np.float64)[:, None] - (H - 1) / 2.0 + np.zeros((1, W))
    c1 = np.arange(W, dtype=np.float64)[None, :] - (W - 1) / 2.0 + np.zeros((H, 1))
    if p.rotate[b]:
        cs, sn = p.cos[b], p.sin[b]
        c0, c1 = c0 * cs + c1 * sn, c1 * cs - c0 * sn
    if p.scale_on[b]:
        c0, c1 = c0 * p.scale[b], c1 * p.scale[b]
    return c0 + (in_shape[0] / 2.0 - 0.5), c1 + (in_shape[1] / 2.0 - 0.5)


def interpolate_seg(seg, c0, c1) -> np.ndarray:
    """interpolate_img(is_seg=True, order=1, mode='constant', cval=-1): one order-1 map per label, ascending."""
    result = np.zeros(c0.shape, seg.dtype)
    for c in np.unique(seg):
        m = map_coordinates_torch64((seg == c).astype(float), c0, c1, 1, -1.0).numpy()
        result[m >= 0.5] = c
    return result


def spatial(data, seg, p, out_shape):
    B, C = data.shape[:2]
    H, W = out_shape
    d_out = np.zeros((B, C, H, W), np.float32)
    s_out = np.zeros((B, seg.shape[1], H, W), np.float32)
    in_shape = data.shape[2:]
    for b in range(B):
        if p.spatial[b]:
            c0, c1 = spatial_coords(p, b, in_shape, out_shape)
            for c in range(C):
                d_out[b, c] = map_coordinates_torch64(data[b, c].astype(float), c0, c1, 3, 0.0).numpy().astype(
                    np.float32)
            for c in range(seg.shape[1]):
                s_out[b, c] = interpolate_seg(seg[b, c], c0, c1)
        else:   # center_crop_aug
            o0, o1 = (in_shape[0] - H) // 2, (in_shape[1] - W) // 2
            d_out[b] = data[b, :, o0:o0 + H, o1:o1 + W]
            s_out[b] = seg[b, :, o0:o0 + H, o1:o1 + W]
    return d_out, s_out


def lowres_channel(x32, target) -> np.ndarray:
    """augment_linear_downsampling_scipy on one channel: skimage resize order 0 down, order 3 up (mode 'edge')."""
    H, W = x32.shape
    th, tw = (int(v) for v in target)
    x = x32.astype(np.float64)
    i0 = np.floor(((np.arange(th) + 0.5) * (H / th) - 0.5) + 0.5).astype(int)   # ndimage.zoom order 0, grid_mode
    i1 = np.floor(((np.arange(tw) + 0.5) * (W / tw) - 0.5) + 0.5).astype(int)
    down = x[np.clip(i0, 0, H - 1)][:, np.clip(i1, 0, W - 1)]
    return PRE.resize_order3(torch.from_numpy(down), (H, W)).numpy().astype(np.float32)


def gamma_channel(x, gamma, eps=1e-7):
    """augment_gamma's per-channel body with retain_stats (mean / std as numpy's float32 reductions)."""
    mn, sd = PRE.mean_std_f32(x)
    minm = x.min()
    rnge = x.max() - minm
    r = float(rnge + eps)                       # float32 + weak python float
    x = np.power((x - minm) / r, np.float32(gamma)) * r + minm
    m2, s2 = PRE.mean_std_f32(x)
    x = x - m2
    x = x / (s2 + 1e-8) * sd
    return x + mn


def augment(data, seg, p, noise, out_shape, use_mask_for_norm=None, regions=None, ignore_label=None):
    """The whole pipeline: float32 data [B, C, h, w] and integer seg [B, 1, h, w] at the initial patch size, the record
    `p`, the standard-normal noise field [B, C, H, W] (float64) -> float32 data [B, C, H, W] and the float32 target
    ([B, 1, H, W], or [B, R (+1), H, W] for regions)."""
    data = np.asarray(data, np.float32)
    seg = np.asarray(seg)
    B, C = data.shape[:2]
    x, s = spatial(data, seg, p, out_shape)
    for b in range(B):
        for c in range(C):
            if p.noise[b, c]:
                x[b, c] = x[b, c].astype(np.float64) + p.noise_std[b] * noise[b, c]
    for b in range(B):
        for c in range(C):
            if p.blur_sigma[b, c] > 0:
                x[b, c] = gaussian_filter_2d(x[b, c], float(p.blur_sigma[b, c]))
    for b in range(B):
        if p.brightness_on[b]:
            for c in range(C):
                x[b, c] *= float(p.brightness[b, c])
    for b in range(B):
        for c in range(C):
            if p.contrast_on[b, c]:
                xc = x[b, c]
                mn = PRE.mean_std_f32(xc)[0]
                lo, hi = xc.min(), xc.max()
                xc = (xc - mn) * float(p.contrast[b, c]) + mn
                xc[xc < lo] = lo
                xc[xc > hi] = hi
                x[b, c] = xc
    for b in range(B):
        for c in range(C):
            if p.lowres_shape[b, c, 0] > 0:
                x[b, c] = lowres_channel(x[b, c], p.lowres_shape[b, c])
    for on, gam, invert in ((p.gamma_inv_on, p.gamma_inv, True), (p.gamma_on, p.gamma, False)):
        for b in range(B):
            if on[b]:
                xs = -x[b] if invert else x[b]
                for c in range(C):
                    xs[c] = gamma_channel(xs[c], gam[b, c])
                x[b] = -xs if invert else xs
    for b in range(B):
        if p.flip[b, 0]:
            x[b] = x[b, :, ::-1]
            s[b] = s[b, :, ::-1]
        if p.flip[b, 1]:
            x[b] = x[b, :, :, ::-1]
            s[b] = s[b, :, :, ::-1]
    if use_mask_for_norm is not None:
        mask = s[:, 0] < 0
        for c in range(C):
            if use_mask_for_norm[c]:
                x[:, c][mask] = 0
    s[s == -1] = 0
    if regions is not None:
        regs = list(regions) + ([ignore_label] if ignore_label is not None else [])
        t = np.zeros((B, len(regs), *out_shape), np.float32)
        for b in range(B):
            for r, labels in enumerate(regs):
                for v in (labels if isinstance(labels, (list, tuple)) else (labels,)):
                    t[b, r][s[b, 0] == v] = 1
        s = t
    return x, s


# ---- seeded inputs ----------------------------------------------------------------------------------------------


def ct_like(B, C, h, w, pad, seed, labels=3):
    """Seeded CT-like data (float32 [B, C, h, w]) and labels (int16 [B, 1, h, w]); `pad` border rows (top) and
    columns (right) of every sample are padding, as nnUNetDataLoader2D pads: data 0, seg -1."""
    rng = np.random.RandomState(seed)
    yy, xx = np.meshgrid(np.linspace(-1, 1, h), np.linspace(-1, 1, w), indexing="ij")
    data = np.zeros((B, C, h, w), np.float32)
    seg = np.zeros((B, 1, h, w), np.int16)
    for b in range(B):
        r = np.sqrt((yy - rng.uniform(-.3, .3)) ** 2 + (xx - rng.uniform(-.3, .3)) ** 2)
        seg[b, 0] = np.minimum((r < 0.7).astype(int) + (r < 0.4) + (r < 0.15) * rng.randint(0, 2), labels - 1)
        for c in range(C):
            data[b, c] = (seg[b, 0] * 80.0 - 500 + rng.normal(0, 40, (h, w))) / 300.0 + c
        if pad:
            seg[b, :, :pad] = -1
            seg[b, :, :, -pad:] = -1
            data[b, :, :pad] = 0
            data[b, :, :, -pad:] = 0
    return data, seg


# ---- batchgenerators' draws, transform by transform ---------------------------------------------------------------


def draw_decisions(B, C, patch_size, rng, rot_range, noise_from=None):
    """Replays the random draws of the training pipeline's transforms on `rng`, loop by loop as batchgenerators 0.25
    writes them, and returns every decision as a list of (transform, sample, channel, value) tuples.  The values
    batchgenerators takes from python's `random` (get_range_val: the noise std, the blur sigma) are taken from `rng`
    at the same place."""
    U = rng.uniform
    out = []
    for b in range(B):                                    # SpatialTransform (augment_spatial)
        if U() < 0.2:
            a = U(rot_range[0], rot_range[1]) if U() <= 1 else 0.0
            out.append(("rot", b, -1, a))
        if U() < 0.2:
            sc = U(0.7, 1) if rng.random_sample() < 0.5 else U(1, 1.4)
            out.append(("scale", b, -1, sc))
    for b in range(B):                                    # GaussianNoiseTransform
        if U() < 0.1:
            std = U(0, 0.1)
            out.append(("noise_std", b, -1, std))
            for c in range(C):
                if U() < 1:
                    out.append(("noise", b, c, 1))
    for b in range(B):                                    # GaussianBlurTransform
        if U() < 0.2:
            for c in range(C):
                if U() <= 0.5:
                    out.append(("blur", b, c, U(0.5, 1)))
    for b in range(B):                                    # BrightnessMultiplicativeTransform
        if U() < 0.15:
            U(0.75, 1.25)
            for c in range(C):
                out.append(("brightness", b, c, U(0.75, 1.25)))
    for b in range(B):                                    # ContrastAugmentationTransform
        if U() < 0.15:
            for c in range(C):
                if U() < 1:
                    f = U(0.75, 1) if rng.random_sample() < 0.5 else U(1, 1.25)
                    out.append(("contrast", b, c, f))
    for b in range(B):                                    # SimulateLowResolutionTransform
        if U() < 0.25:
            for c in range(C):
                if U() < 0.5:
                    zoom = U(0.5, 1)
                    out.append(("lowres", b, c, tuple(np.round(np.array(patch_size) * zoom).astype(int))))
    for name, p in (("gamma_inv", 0.1), ("gamma", 0.3)):  # GammaTransform x 2
        for b in range(B):
            if U() < p:
                for c in range(C):
                    g = U(0.7, 1) if rng.random_sample() < 0.5 else U(1, 1.5)
                    out.append((name, b, c, g))
    for b in range(B):                                    # MirrorTransform
        if U() < 1:
            for ax in (0, 1):
                if U() < 0.5:
                    out.append(("flip", b, ax, 1))
    return out
