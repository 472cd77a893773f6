"""nnU-Net's 2-D training augmentation on the device (reference: `nnUNetTrainer.get_training_transforms`,
nnUNetTrainer.py:684-775, batchgenerators 0.25), for the Dino U-Net trainer (no deep supervision, no cascade).

    aug = DeviceTrainingAugmentation(patch_size, rotation_for_DA, mirror_axes, use_mask_for_norm, regions, ignore_label)
    data, target = aug(data, seg)   # CUDA: fp32 [B, C, *initial patch], int16 [B, 1, *initial patch] -> fp32 at patch

`sample_augmentation_params` draws every decision of the transforms on the host, on a `np.random.RandomState`, in
batchgenerators' order: spatial (rotation, scale), Gaussian noise, Gaussian blur, multiplicative brightness, contrast,
low-resolution simulation, gamma on the inverted image, gamma, mirroring.  It differs from batchgenerators in two
documented ways: the values batchgenerators takes from python's `random` through `get_range_val` (the noise std and
the blur sigma) are drawn from the same RandomState at the same place, and the per-pixel normal draws of the noise are
not taken from it (the device generates them with Philox, keyed by (seed, sample, channel, pixel):
`noise_field`).  The record is uploaded once; `b2u_aug_apply` (csrc/augmentation.cu) runs the whole pipeline in one
stream with no host synchronisation.

On the same record and noise field the device reproduces oracle/augmentation_oracle.py (the numpy / scipy
restatement): the spatial transform, blur, brightness, contrast, low-resolution simulation, mirroring, mask, label
removal and regions bit for bit; the gamma steps use CUDA's `powf` where numpy uses libm's (a few ulp).
"""
from __future__ import annotations

import ctypes
import math
from dataclasses import dataclass, fields
from typing import Optional, Sequence

import numpy as np
import torch

from . import lib as L

POLE = -0.267949192431122706472553658494127633  # sqrt(3) - 2, correctly rounded
NPAD = 12
REC = 40
# record fields, as csrc/augmentation.cu reads them
(F_SPATIAL, F_ROT, F_COS, F_SIN, F_SCALE_ON, F_SCALE, F_NOISE, F_NOISE_STD, F_BLUR_R, F_BLUR_W) = range(10)
F_BRIGHT, F_BRIGHT_M, F_CONTRAST, F_CONTRAST_F, F_LOW_H, F_LOW_W, F_LOW_Y, F_LOW_X = 14, 15, 16, 17, 18, 19, 20, 25
F_GAMINV_ON, F_GAMINV, F_GAM_ON, F_GAM, F_FLIP0, F_FLIP1, F_MASK = 30, 31, 32, 33, 34, 35, 36


def rotation_for_da_2d(patch_size) -> dict:
    """configure_rotation_dummyDA_mirroring_and_inital_patch_size for 2-D: +-15 deg when max/min of the patch exceeds
    1.5, else +-180 deg (in radians, about 'x')."""
    a = 15. if max(patch_size) / min(patch_size) > 1.5 else 180.
    return {"x": (-a / 360 * 2. * np.pi, a / 360 * 2. * np.pi), "y": (0, 0), "z": (0, 0)}


def initial_patch_size_2d(patch_size) -> np.ndarray:
    """get_patch_size(patch_size, *rotation_for_da_2d(patch_size).values(), (0.85, 1.25)) for 2-D patches
    (compute_initial_patch_size.py with batchgenerators' rotate_coords_2d)."""
    rot = min(90 / 360 * 2. * np.pi, max(np.abs(rotation_for_da_2d(patch_size)["x"])))
    coords = np.array(patch_size)
    rm = np.array([[np.cos(rot), -np.sin(rot)], [np.sin(rot), np.cos(rot)]])
    rotated = np.dot(coords.reshape(len(coords), -1).transpose(), rm).transpose().reshape(coords.shape)
    final_shape = np.max(np.vstack((np.abs(rotated), np.copy(coords))), 0)
    final_shape = final_shape / 0.85
    return final_shape.astype(int)


@dataclass
class AugmentationParams:
    """Every decision of one batch's training transforms (B samples, C channels)."""
    spatial: np.ndarray        # bool [B]: rotated and / or scaled (else the centre crop)
    rotate: np.ndarray         # bool [B]
    angle: np.ndarray          # float64 [B]
    cos: np.ndarray            # float64 [B]: np.cos(angle)
    sin: np.ndarray            # float64 [B]
    scale_on: np.ndarray       # bool [B]
    scale: np.ndarray          # float64 [B]
    noise: np.ndarray          # bool [B, C]
    noise_std: np.ndarray      # float64 [B]
    blur_sigma: np.ndarray     # float64 [B, C], 0 = no blur
    brightness_on: np.ndarray  # bool [B]
    brightness: np.ndarray     # float64 [B, C]
    contrast_on: np.ndarray    # bool [B, C]
    contrast: np.ndarray       # float64 [B, C]
    lowres_shape: np.ndarray   # int64 [B, C, 2], 0 = no low-resolution simulation
    gamma_inv_on: np.ndarray   # bool [B]
    gamma_inv: np.ndarray      # float64 [B, C]
    gamma_on: np.ndarray       # bool [B]
    gamma: np.ndarray          # float64 [B, C]
    flip: np.ndarray           # bool [B, 2]

    @classmethod
    def identity(cls, B: int, C: int) -> "AugmentationParams":
        """Centre crop only: every transform off."""
        z = lambda *s: np.zeros(s, bool)  # noqa: E731
        f = lambda *s: np.zeros(s)  # noqa: E731
        return cls(z(B), z(B), f(B), np.ones(B), f(B), z(B), np.ones(B), z(B, C), f(B), f(B, C), z(B), np.ones((B, C)),
                   z(B, C), np.ones((B, C)), np.zeros((B, C, 2), np.int64), z(B), np.ones((B, C)), z(B),
                   np.ones((B, C)), z(B, 2))

    @property
    def batch_size(self) -> int:
        return int(self.spatial.shape[0])

    @property
    def num_channels(self) -> int:
        return int(self.noise.shape[1])

    def copy(self) -> "AugmentationParams":
        return AugmentationParams(**{f.name: np.array(getattr(self, f.name)) for f in fields(self)})


def _half_split(rng, lo, hi):
    """batchgenerators' `np.random.random() < 0.5 and lo < 1` split of a range around 1."""
    return rng.uniform(lo, 1) if rng.random_sample() < 0.5 and lo < 1 else rng.uniform(max(lo, 1), hi)


def sample_augmentation_params(batch_size: int, num_channels: int, patch_size: Sequence[int],
                               rng: np.random.RandomState, rotation_for_DA: Optional[dict] = None,
                               mirror_axes: Sequence[int] = (0, 1)) -> AugmentationParams:
    """The draws of the 2-D training pipeline for one batch, in batchgenerators' order (module docstring)."""
    B, C = int(batch_size), int(num_channels)
    rot = (rotation_for_DA or rotation_for_da_2d(patch_size))["x"]
    p = AugmentationParams.identity(B, C)
    U = rng.uniform
    for b in range(B):                              # SpatialTransform
        if U() < 0.2:
            p.rotate[b] = True
            p.angle[b] = U(rot[0], rot[1]) if U() <= 1 else 0.0
            p.cos[b], p.sin[b] = np.cos(p.angle[b]), np.sin(p.angle[b])
        if U() < 0.2:
            p.scale_on[b] = True
            p.scale[b] = _half_split(rng, 0.7, 1.4)
        p.spatial[b] = p.rotate[b] or p.scale_on[b]
    for b in range(B):                              # GaussianNoiseTransform(p_per_sample=0.1)
        if U() < 0.1:
            p.noise_std[b] = U(0, 0.1)
            for c in range(C):
                p.noise[b, c] = U() < 1
    for b in range(B):                              # GaussianBlurTransform((0.5, 1), p 0.2, p_per_channel 0.5)
        if U() < 0.2:
            for c in range(C):
                if U() <= 0.5:
                    p.blur_sigma[b, c] = U(0.5, 1)
    for b in range(B):                              # BrightnessMultiplicativeTransform((0.75, 1.25), p 0.15)
        if U() < 0.15:
            p.brightness_on[b] = True
            U(0.75, 1.25)
            for c in range(C):
                p.brightness[b, c] = U(0.75, 1.25)
    for b in range(B):                              # ContrastAugmentationTransform(p 0.15)
        if U() < 0.15:
            for c in range(C):
                if U() < 1:
                    p.contrast_on[b, c] = True
                    p.contrast[b, c] = _half_split(rng, 0.75, 1.25)
    shp = np.array(patch_size)
    for b in range(B):                              # SimulateLowResolutionTransform((0.5, 1), p 0.25, p_per_channel 0.5)
        if U() < 0.25:
            for c in range(C):
                if U() < 0.5:
                    p.lowres_shape[b, c] = np.round(shp * U(0.5, 1)).astype(int)
    for on, g, prob in ((p.gamma_inv_on, p.gamma_inv, 0.1), (p.gamma_on, p.gamma, 0.3)):   # GammaTransform x 2
        for b in range(B):
            if U() < prob:
                on[b] = True
                for c in range(C):
                    g[b, c] = _half_split(rng, 0.7, 1.5)
    if len(mirror_axes):
        for b in range(B):                          # MirrorTransform
            if U() < 1:
                for ax in (0, 1):
                    if ax in mirror_axes and U() < 0.5:
                        p.flip[b, ax] = True
    return p


def _reflect_consts(n: int):
    z = POLE
    zn = math.pow(z, n)
    return [z, zn, (1.0 - z) * (1.0 - 1.0 / z), z / (1 - zn * zn), z / (z - 1)]


def gaussian_weights(sigma: float) -> np.ndarray:
    """scipy's _gaussian_kernel1d(sigma, 0, int(4 sigma + 0.5)), float64."""
    radius = int(4.0 * float(sigma) + 0.5)
    x = np.arange(-radius, radius + 1)
    phi = np.exp(-0.5 / (sigma * sigma) * x ** 2)
    return phi / phi.sum()


def pack_record(p: AugmentationParams, patch_size, use_mask_for_norm=None) -> np.ndarray:
    """The device record: float64 [B*C, REC] (csrc/augmentation.cu)."""
    B, C = p.batch_size, p.num_channels
    r = np.zeros((B, C, REC))
    r[..., F_SPATIAL] = p.spatial[:, None]
    r[..., F_ROT] = p.rotate[:, None]
    r[..., F_COS] = p.cos[:, None]
    r[..., F_SIN] = p.sin[:, None]
    r[..., F_SCALE_ON] = p.scale_on[:, None]
    r[..., F_SCALE] = p.scale[:, None]
    r[..., F_NOISE] = p.noise
    r[..., F_NOISE_STD] = p.noise_std[:, None]
    r[..., F_BRIGHT] = p.brightness_on[:, None]
    r[..., F_BRIGHT_M] = p.brightness
    r[..., F_CONTRAST] = p.contrast_on
    r[..., F_CONTRAST_F] = p.contrast
    r[..., F_GAMINV_ON] = p.gamma_inv_on[:, None]
    r[..., F_GAMINV] = p.gamma_inv
    r[..., F_GAM_ON] = p.gamma_on[:, None]
    r[..., F_GAM] = p.gamma
    r[..., F_FLIP0] = p.flip[:, 0:1]
    r[..., F_FLIP1] = p.flip[:, 1:2]
    if use_mask_for_norm is not None:
        r[..., F_MASK] = np.asarray([bool(v) for v in use_mask_for_norm], dtype=float)[None, :C]
    for b in range(B):
        for c in range(C):
            s = float(p.blur_sigma[b, c])
            if s > 0:
                w = gaussian_weights(s)[::-1]
                rad = (len(w) - 1) // 2
                r[b, c, F_BLUR_R] = rad
                r[b, c, F_BLUR_W:F_BLUR_W + rad + 1] = w[rad:]
            th, tw = (int(v) for v in p.lowres_shape[b, c])
            if th > 0:
                r[b, c, F_LOW_H], r[b, c, F_LOW_W] = th, tw
                r[b, c, F_LOW_Y:F_LOW_Y + 5] = _reflect_consts(th + 2 * NPAD)
                r[b, c, F_LOW_X:F_LOW_X + 5] = _reflect_consts(tw + 2 * NPAD)
    return r.reshape(B * C, REC)


def noise_field(seed: int, B: int, C: int, shape, device=None) -> torch.Tensor:
    """The standard-normal field the noise step scales by its std: float64 [B, C, *shape] on the device."""
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    n = int(np.prod(shape))
    out = torch.empty((B, C, *shape), dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        L.check(L.load().b2u_aug_noise_field(int(seed) & (2 ** 64 - 1), B, C, n, out.data_ptr(), stream),
                "b2u_aug_noise_field")
    return out


def _region_table(regions, ignore_label):
    """int32 [R + 1 offsets, labels] of ConvertSegmentationToRegionsTransform(regions (+ [ignore_label]))."""
    regs = list(regions) + ([ignore_label] if ignore_label is not None else [])
    offs, labels = [0], []
    for r in regs:
        vals = list(r) if isinstance(r, (list, tuple)) else [r]
        for v in vals:
            if not isinstance(v, (int, np.integer)) or isinstance(v, (bool, np.bool_)) or not -2 ** 15 <= int(v) < 2 ** 15:
                raise ValueError(f"region label {v!r} of {r!r} is not an int16 label")
            labels.append(int(v))
        offs.append(len(labels))
    return len(regs), np.asarray(offs + labels, dtype=np.int32)


class DeviceTrainingAugmentation:
    """The trainer's 2-D training transforms on CUDA tensors at the initial patch size (module docstring)."""

    def __init__(self, patch_size, rotation_for_DA: Optional[dict] = None, mirror_axes=(0, 1), use_mask_for_norm=None,
                 regions=None, ignore_label=None, seed: Optional[int] = None):
        self.patch_size = tuple(int(v) for v in patch_size)
        if len(self.patch_size) != 2 or min(self.patch_size) < 2:
            raise ValueError(f"device augmentation is 2-D only, with patch sides >= 2; got patch_size {patch_size}")
        self.rotation_for_DA = rotation_for_DA or rotation_for_da_2d(self.patch_size)
        self.mirror_axes = tuple(int(a) for a in (mirror_axes or ()))
        if any(a not in (0, 1) for a in self.mirror_axes):
            raise ValueError(f"mirror axes {mirror_axes} are not 2-D axes")
        self.use_mask_for_norm = None if use_mask_for_norm is None or not any(use_mask_for_norm) else \
            [bool(v) for v in use_mask_for_norm]
        self.regions = list(regions) if regions is not None else None
        self.ignore_label = ignore_label
        self._R, self._table = (0, None) if self.regions is None else _region_table(self.regions, ignore_label)
        self.rng = np.random.RandomState(seed)
        self._seed_rng = np.random.RandomState(None if seed is None else (int(seed) + 1) % 2 ** 32)
        self._cache = {}

    @property
    def num_target_channels(self) -> int:
        return self._R if self.regions is not None else 1

    def _check(self, data: torch.Tensor, seg: torch.Tensor):
        if not isinstance(data, torch.Tensor) or not isinstance(seg, torch.Tensor):
            raise TypeError("data and seg must be tensors")
        if not data.is_cuda or seg.device != data.device:
            raise ValueError(f"data and seg must be on the same CUDA device, got {data.device} and {seg.device}")
        if data.dtype != torch.float32:
            raise TypeError(f"data must be float32, got {data.dtype}")
        if seg.dtype != torch.int16:
            raise TypeError(f"seg must be int16 (the data loader's label dtype), got {seg.dtype}")
        if data.ndim != 4 or seg.ndim != 4:
            raise ValueError(f"data and seg must be [B, C, X, Y], got {tuple(data.shape)} and {tuple(seg.shape)}")
        B, C, h, w = data.shape
        if tuple(seg.shape) != (B, 1, h, w):
            raise ValueError(f"seg must be [B, 1, X, Y] = {(B, 1, h, w)}, got {tuple(seg.shape)}")
        if h < self.patch_size[0] or w < self.patch_size[1]:
            raise ValueError(f"the input {(h, w)} is smaller than the patch {self.patch_size}")
        if B < 1 or C < 1 or B * C > 65535:
            raise ValueError(f"B={B}, C={C}: need 1 <= B*C <= 65535")
        if self.use_mask_for_norm is not None and len(self.use_mask_for_norm) != C:
            raise ValueError(f"use_mask_for_norm has {len(self.use_mask_for_norm)} entries for {C} channels")

    def sample(self, batch_size: int, num_channels: int) -> AugmentationParams:
        return sample_augmentation_params(batch_size, num_channels, self.patch_size, self.rng, self.rotation_for_DA,
                                          self.mirror_axes)

    def __call__(self, data: torch.Tensor, seg: torch.Tensor):
        self._check(data, seg)
        params = self.sample(data.shape[0], data.shape[1])
        return self.apply(data, seg, params, int(self._seed_rng.randint(0, 2 ** 63, dtype=np.int64)))

    def apply(self, data: torch.Tensor, seg: torch.Tensor, params: AugmentationParams, noise_seed: int):
        """The pipeline with the given decisions and noise seed: (fp32 [B, C, *patch], fp32 target)."""
        self._check(data, seg)
        B, C, h, w = (int(v) for v in data.shape)
        H, W = self.patch_size
        if params.batch_size != B or params.num_channels != C:
            raise ValueError(f"the parameters are for B={params.batch_size}, C={params.num_channels}; the batch is "
                             f"B={B}, C={C}")
        dev = data.device
        lib = L.load()
        rec = torch.from_numpy(pack_record(params, self.patch_size, self.use_mask_for_norm)).to(dev, non_blocking=True)
        key = (dev, B, C, h, w)
        if key not in self._cache:
            nbytes = int(lib.b2u_aug_work_bytes(B, C, h, w, H, W))
            table = None if self._table is None else torch.from_numpy(self._table).to(dev)
            self._cache = {key: (torch.empty(nbytes, dtype=torch.uint8, device=dev), table)}
        work, table = self._cache[key]
        z = POLE
        consts = (ctypes.c_double * 5)(z, math.pow(z, h - 1), math.pow(z, w - 1), (1.0 - z) * (1.0 - 1.0 / z),
                                       z * z - 1.0)
        out = torch.empty((B, C, H, W), dtype=torch.float32, device=dev)
        target = torch.empty((B, self.num_target_channels, H, W), dtype=torch.float32, device=dev)
        data, seg = data.contiguous(), seg.contiguous()
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            L.check(lib.b2u_aug_apply(data.data_ptr(), seg.data_ptr(), B, C, h, w, H, W, rec.data_ptr(),
                                      ctypes.addressof(consts), int(noise_seed) & (2 ** 64 - 1),
                                      table.data_ptr() if table is not None else None, self._R, work.data_ptr(),
                                      out.data_ptr(), target.data_ptr(), stream), "b2u_aug_apply")
        return out, target
