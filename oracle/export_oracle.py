"""Restatement of the reference's logits -> segmentation export for 2D configurations
(`convert_predicted_logits_to_segmentation_with_correct_shape`, inference/export_prediction.py:15-68):

    resample_data_or_seg_to_shape(order=1)   (default_resampling.py)   data.astype(float); per channel
        skimage resize(order=1, mode='edge', anti_aliasing=False) == scipy ndimage.zoom(order=1, mode='nearest',
        grid_mode=True) on [Z, h, w], Z unchanged; .astype(float16).  The array is returned as is when shapes are equal.
    apply_inference_nonlin                    .float(), softmax(0) (label maps) / sigmoid (regions)
    convert_probabilities_to_segmentation     argmax(0) / seg[p[i] > 0.5] = regions_class_order[i] in order
    revert cropping + transpose               uint8 (< 255 foreground labels) else uint16; probabilities as
                                              revert_cropping_on_probabilities + transpose [0] + [i + 1 ...]

Two resamplers: `resample_scipy` calls scipy (the reference's own arithmetic), and `resample_torch64` restates scipy's
order-1 zoom (NI_ZoomShift: coordinates, spline weights, tap order) in torch float64, bit for bit, so the GPU tests
need no scipy.  That skimage >= 0.19's resize on float64 equals the scipy call is taken from skimage's source: skimage
is not a dependency here and that equivalence is not checked by this repository's tests.
"""
from typing import Sequence

import numpy as np
import torch


def resample_scipy(logits16: np.ndarray, new_shape: Sequence[int]) -> np.ndarray:
    """fp16 [C, Z, h, w] -> fp16 [C, *new_shape] the reference's way (scipy float64 zoom per channel)."""
    import scipy.ndimage as ndi
    logits16 = np.asarray(logits16)
    new_shape = tuple(int(s) for s in new_shape)
    if logits16.shape[1:] == new_shape:
        return logits16
    data = logits16.astype(float)
    factors = [n / o for n, o in zip(new_shape, data.shape[1:])]
    out = np.stack([ndi.zoom(data[c], factors, order=1, mode="nearest", grid_mode=True) for c in range(data.shape[0])])
    assert out.shape[1:] == new_shape, (out.shape, new_shape)
    return out.astype(logits16.dtype)


def _axis_taps(n_in: int, n_out: int):
    """scipy's order-1 zoom along one axis: cc = (k + 0.5) * (n_in / n_out) - 0.5 (not clamped for mode 'nearest'),
    weights 1 - (cc - floor(cc)) and 1 - that, tap indices floor(cc), floor(cc) + 1 clamped to the array."""
    k = torch.arange(n_out, dtype=torch.float64)
    cc = (k + 0.5) * (n_in / n_out) - 0.5
    fl = torch.floor(cc)
    w0 = 1.0 - (cc - fl)
    w1 = 1.0 - w0
    i0 = fl.long()
    return i0.clamp(0, n_in - 1), (i0 + 1).clamp(0, n_in - 1), w0, w1


def resample_torch64(logits16: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """float64 [C, Z, H, W] of scipy's zoom of fp16 [C, Z, h, w] to [H, W] (before the fp16 rounding)."""
    x = logits16.detach().cpu().double()
    y0, y1, wy0, wy1 = _axis_taps(x.shape[2], H)
    x0, x1, wx0, wx1 = _axis_taps(x.shape[3], W)
    t = torch.zeros((*x.shape[:2], H, W), dtype=torch.float64)
    for yi, wy in ((y0, wy0), (y1, wy1)):
        rows = x[:, :, yi]
        for xi, wx in ((x0, wx0), (x1, wx1)):
            t = t + rows[:, :, :, xi] * wy[:, None] * wx[None, :]
    return t


def to_f16(t64: torch.Tensor) -> torch.Tensor:
    """float64 -> float16 rounded once to nearest even, as numpy's astype (torch's CPU cast goes through fp32)."""
    return torch.from_numpy(t64.numpy().astype(np.float16))


def resample_f16(logits16: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """The reference's resampling of fp16 logits [C, Z, h, w] to [C, Z, H, W], through the torch restatement."""
    logits16 = logits16.detach().cpu()
    if tuple(logits16.shape[2:]) == (H, W):
        return logits16
    return to_f16(resample_torch64(logits16, H, W))


def nonlin_and_segment(logits16: torch.Tensor, has_regions: bool, regions_class_order=None):
    """apply_inference_nonlin + convert_probabilities_to_segmentation (label_handling.py:128-175)."""
    logits = logits16.detach().cpu().float()
    if has_regions:
        probs = torch.sigmoid(logits)
        seg = torch.zeros(probs.shape[1:], dtype=torch.int16)
        for i, c in enumerate(regions_class_order):
            seg[probs[i] > 0.5] = c
    else:
        probs = torch.softmax(logits, 0)
        seg = probs.argmax(0)
    return probs, seg


def revert_geometry(seg, probs, properties: dict, transpose_backward: Sequence[int], n_foreground: int,
                    has_regions: bool):
    """export_prediction.py:43-62 with revert_cropping_on_probabilities (label_handling.py:200-212)."""
    slicer = tuple(slice(int(lo), int(hi)) for lo, hi in properties["bbox_used_for_cropping"])
    out = np.zeros(properties["shape_before_cropping"], dtype=np.uint8 if n_foreground < 255 else np.uint16)
    out[slicer] = np.asarray(seg)
    out = out.transpose(list(transpose_backward))
    if probs is None:
        return out, None
    p = np.zeros((probs.shape[0], *properties["shape_before_cropping"]), dtype=np.float32)
    if not has_regions:
        p[0] = 1
    p[(slice(None), *slicer)] = np.asarray(probs)
    return out, p.transpose([0] + [i + 1 for i in transpose_backward])


def convert(logits16, properties: dict, transpose_backward, n_foreground: int, has_regions: bool,
            regions_class_order=None, return_probabilities: bool = False, resampler: str = "torch"):
    """The whole chain.  Returns (resampled fp16 tensor, segmentation, probabilities or None)."""
    logits16 = torch.as_tensor(np.asarray(logits16.cpu() if isinstance(logits16, torch.Tensor) else logits16))
    _, H, W = (int(s) for s in properties["shape_after_cropping_and_before_resampling"])
    if resampler == "scipy":
        r = torch.from_numpy(resample_scipy(logits16.numpy(), properties["shape_after_cropping_and_before_resampling"]))
    else:
        r = resample_f16(logits16, H, W)
    probs, seg = nonlin_and_segment(r, has_regions, regions_class_order)
    seg, p = revert_geometry(seg.numpy(), probs.numpy() if return_probabilities else None, properties,
                             transpose_backward, n_foreground, has_regions)
    return r, seg, p


# ---- golden cases (oracle/make_golden_export.py -> tests/golden/export_cases.npz)

# (name, C, has_regions, regions_class_order, cropped [Z, h, w] of the logits, target [Z, H, W],
#  shape_before_cropping, bbox, transpose_backward, save_probabilities)
GOLDEN_CASES = [
    ("lab2_up", 2, False, None, (2, 24, 20), (2, 41, 37), (3, 50, 45), [[1, 3], [4, 45], [2, 39]], (0, 1, 2), False),
    ("lab4_down", 4, False, None, (2, 48, 52), (2, 30, 26), (2, 33, 30), [[0, 2], [3, 33], [1, 27]], (0, 2, 1), True),
    ("lab2_mixed", 2, False, None, (1, 96, 96), (1, 57, 131), (2, 58, 133), [[1, 2], [1, 58], [2, 133]], (2, 0, 1), False),
    ("lab4_identity", 4, False, None, (3, 20, 24), (3, 20, 24), (3, 26, 30), [[0, 3], [6, 26], [2, 26]], (1, 0, 2), False),
    ("reg3_up", 3, True, (2, 1, 3), (2, 20, 28), (2, 33, 45), (2, 40, 45), [[0, 2], [5, 38], [0, 45]], (0, 2, 1), True),
    ("reg3_mixed", 3, True, (1, 3, 2), (2, 64, 40), (2, 39, 71), (5, 39, 80), [[1, 3], [0, 39], [4, 75]], (2, 1, 0), False),
]


def golden_logits(C: int, shape, seed: int) -> torch.Tensor:
    """fp16 logits whose classes compete (so argmax and the 0.5 threshold both flip inside every case)."""
    g = torch.Generator().manual_seed(seed)
    z, h, w = shape
    base = torch.randn(C, z, h // 4 + 2, w // 4 + 2, generator=g, dtype=torch.float64) * 3
    smooth = torch.nn.functional.interpolate(base, size=(h, w), mode="bilinear", align_corners=False)
    return (smooth + 0.3 * torch.randn(C, z, h, w, generator=g, dtype=torch.float64)).to(torch.float32).half()


def golden_properties(case) -> dict:
    _, _, _, _, _, target, before, bbox, _, _ = case
    return {"shape_after_cropping_and_before_resampling": list(target), "shape_before_cropping": list(before),
            "bbox_used_for_cropping": [list(b) for b in bbox], "spacing": [1.0, 1.0, 1.0]}
