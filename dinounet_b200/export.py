"""Prediction export: logits -> the segmentation file nnU-Net writes (reference: `dinounet/inference/export_prediction.py`).

Two routes:

* `labels_to_original_geometry`: the uint8 label maps that `b2u_seg_head` writes, when no resampling is needed (the case
  was not rescaled at preprocessing: `shape_after_cropping_and_before_resampling == labels.shape`).  Softmax does not
  change an argmax, so only the labels leave the GPU:

      seg = labels_to_original_geometry(labels, properties_dict, plans_manager.transpose_backward)
      rw.write_seg(seg, output_file_truncated + file_ending, properties_dict)        # the reference's writer, unchanged

* `convert_predicted_logits_to_segmentation_with_correct_shape` / `export_prediction_from_logits`: drop-ins with the
  reference's signatures for the fp16 logits `SlidingWindowPredictor` returns, label maps or regions, with or without
  resampling.  The resampling to the original spacing and the softmax / sigmoid + argmax / region painting run on the
  device (`b2u_export_resample_f16`, `b2u_export_segment`); only the labels (and the probabilities, when asked) are
  copied to the host, where the paste into the pre-crop box and the transpose stay in numpy.
"""
import json
import pickle
from typing import Sequence

import numpy as np
import torch

from . import lib as L

# The planner's `resampling_fn_probabilities` for every configuration (default_experiment_planner.py:146-160).
DEFAULT_RESAMPLING_FN = "resample_data_or_seg_to_shape"
DEFAULT_RESAMPLING_KWARGS = {"is_seg": False, "order": 1, "order_z": 0, "force_separate_z": None}
ANISO_THRESHOLD = 3  # dinounet/configuration.py, the default `separate_z_anisotropy_threshold`
MAX_EXPORT_CHANNELS = 32  # b2u_export_segment keeps the channels in registers


def needs_resampling(label_shape: Sequence[int], properties_dict: dict) -> bool:
    """True when the reference's `resampling_fn_probabilities` would change the grid (export_prediction.py:26-33)."""
    return tuple(int(s) for s in label_shape) != tuple(int(s) for s in properties_dict["shape_after_cropping_and_before_resampling"])


def labels_to_original_geometry(labels, properties_dict: dict, transpose_backward: Sequence[int],
                                num_foreground_labels: int = 1) -> np.ndarray:
    """export_prediction.py:43-52: paste the predicted label volume into the pre-crop bounding box (background 0 outside)
    and revert the plans' transpose.  `labels`: integer array / tensor shaped like the cropped case [z, y, x] (for a 2D
    configuration the slice stack the sliding-window predictor returns)."""
    if hasattr(labels, "detach"):
        labels = labels.detach().cpu().numpy()
    labels = np.asarray(labels)
    if needs_resampling(labels.shape, properties_dict):
        raise ValueError("this case needs resampling to its original spacing: export it through the logits route "
                         "(convert_predicted_logits_to_segmentation_with_correct_shape)")
    dtype = np.uint8 if num_foreground_labels < 255 else np.uint16
    out = np.zeros(properties_dict["shape_before_cropping"], dtype=dtype)
    slicer = tuple(slice(int(lo), int(hi)) for lo, hi in properties_dict["bbox_used_for_cropping"])   # bounding_box_to_slice
    out[slicer] = labels.astype(dtype, copy=False)
    return out.transpose(list(transpose_backward))


def probabilities_to_original_geometry(probs: np.ndarray, properties_dict: dict, transpose_backward: Sequence[int],
                                       has_regions: bool) -> np.ndarray:
    """`LabelManager.revert_cropping_on_probabilities` (label_handling.py:200-212: channel 0 is 1 outside the box for
    label maps, 0 for regions) followed by the transpose `[0] + [i + 1 ...]` (export_prediction.py:54-62)."""
    out = np.zeros((probs.shape[0], *properties_dict["shape_before_cropping"]), dtype=probs.dtype)
    if not has_regions:
        out[0] = 1
    slicer = tuple(slice(int(lo), int(hi)) for lo, hi in properties_dict["bbox_used_for_cropping"])
    out[(slice(None), *slicer)] = probs
    return out.transpose([0] + [i + 1 for i in transpose_backward])


def _current_spacing(configuration_manager, properties_dict) -> list:
    """export_prediction.py:26-29."""
    spacing = list(configuration_manager.spacing)
    if len(spacing) == len(properties_dict["shape_after_cropping_and_before_resampling"]):
        return spacing
    return [properties_dict["spacing"][0], *spacing]


def _lowres_axis(spacing) -> np.ndarray:
    """default_resampling.get_lowres_axis."""
    spacing = np.asarray(spacing, dtype=float)
    return np.where(max(spacing) / spacing == 1)[0]


def _separate_z_axis(current_spacing, new_spacing):
    """The anisotropic axis along which `resample_data_or_seg_to_shape(force_separate_z=None)` resamples with order 0,
    or None (default_resampling.py: get_do_separate_z / get_lowres_axis; 2 or 3 lowres axes disable separate z)."""
    for sp in (current_spacing, new_spacing):
        sp = np.asarray(sp, dtype=float)
        if np.max(sp) / np.min(sp) > ANISO_THRESHOLD:
            axis = _lowres_axis(sp)
            return int(axis[0]) if len(axis) == 1 else None
    return None


def _check_resampling(configuration_manager, properties_dict, in_shape, out_shape):
    """Raise NotImplementedError unless the reference's resampling of this case is what b2u_export_resample_f16 computes:
    the planner's default function and kwargs, Z unchanged, and no order-0 resampling along an in-plane axis."""
    conf = getattr(configuration_manager, "configuration", None)
    if not isinstance(conf, dict) or conf.get("resampling_fn_probabilities") != DEFAULT_RESAMPLING_FN or \
            dict(conf.get("resampling_fn_probabilities_kwargs") or {}) != DEFAULT_RESAMPLING_KWARGS:
        raise NotImplementedError(
            f"device export implements resampling_fn_probabilities = {DEFAULT_RESAMPLING_FN}(**{DEFAULT_RESAMPLING_KWARGS}) "
            "only (the planner's default)")
    if len(out_shape) != 3:
        raise NotImplementedError(f"device export handles 2D configurations' [Z, H, W] cases, got target {tuple(out_shape)}")
    if in_shape == out_shape:
        return
    if in_shape[0] != out_shape[0]:
        raise NotImplementedError(f"device export resamples in-plane only; the target shape {tuple(out_shape)} changes Z "
                                  f"({in_shape[0]} slices)")
    axis = _separate_z_axis(_current_spacing(configuration_manager, properties_dict), properties_dict["spacing"])
    if axis in (1, 2) and in_shape[axis] != out_shape[axis]:
        raise NotImplementedError(f"the low-resolution axis {axis} is in-plane and changes size ({in_shape[axis]} -> "
                                  f"{out_shape[axis]}): the reference resamples it with order 0, which the device export "
                                  "does not implement")


def _to_device(predicted_logits: torch.Tensor) -> torch.Tensor:
    """Contiguous logits on their CUDA device; host input goes to the current device."""
    dev = predicted_logits.device if predicted_logits.is_cuda else torch.device("cuda", torch.cuda.current_device())
    return predicted_logits.to(dev).contiguous()


def convert_predicted_logits_to_segmentation_with_correct_shape(predicted_logits, plans_manager, configuration_manager,
                                                                label_manager, properties_dict: dict,
                                                                return_probabilities: bool = False,
                                                                num_threads_torch: int = 8):
    """Drop-in for export_prediction.py:15-68 on fp16 logits [C, Z, h, w]: a CUDA tensor (any strides, e.g. the
    un-padded view `SlidingWindowPredictor` returns), or a host tensor / ndarray, which is uploaded to the current device.
    Returns the segmentation (uint8, or uint16 for >= 255 foreground labels) in the original geometry, and with
    `return_probabilities` also the fp32 probabilities [C, *original shape].  `num_threads_torch` is accepted for the
    reference's signature; the host work here is numpy."""
    if isinstance(predicted_logits, np.ndarray):
        predicted_logits = torch.from_numpy(predicted_logits)
    if not isinstance(predicted_logits, torch.Tensor) or predicted_logits.ndim != 4:
        raise ValueError("predicted_logits must be a [C, Z, H, W] tensor or ndarray")
    if predicted_logits.dtype != torch.float16:
        raise NotImplementedError(f"device export takes the predictor's fp16 logits, got {predicted_logits.dtype}")
    has_regions = bool(label_manager.has_regions)
    if has_regions:
        assert label_manager.regions_class_order is not None, 'if region-based training is requested then you need to ' \
                                                              'define regions_class_order!'
    C = int(predicted_logits.shape[0])
    assert C == label_manager.num_segmentation_heads, \
        f'unexpected number of channels in predicted_probabilities. Expected {label_manager.num_segmentation_heads}, ' \
        f'got {C}. Remember that predicted_probabilities should have shape (c, x, y(, z)).'
    if C > MAX_EXPORT_CHANNELS:
        raise NotImplementedError(f"device export handles up to {MAX_EXPORT_CHANNELS} channels, got {C}")
    in_shape = tuple(int(s) for s in predicted_logits.shape[1:])
    out_shape = tuple(int(s) for s in properties_dict["shape_after_cropping_and_before_resampling"])
    _check_resampling(configuration_manager, properties_dict, in_shape, out_shape)
    n_fg = len(label_manager.foreground_labels)
    label_bytes = 1 if n_fg < 255 else 2

    lib = L.load()
    logits = _to_device(predicted_logits)
    dev = logits.device
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        Z, h, w = in_shape
        _, H, W = out_shape
        if (h, w) != (H, W):
            resampled = torch.empty((C, Z, H, W), dtype=torch.float16, device=dev)
            L.check(lib.b2u_export_resample_f16(logits.data_ptr(), resampled.data_ptr(), C, Z, h, w, H, W, stream),
                    "b2u_export_resample_f16")
            logits = resampled
        voxels = Z * H * W
        labels = torch.empty(out_shape, dtype=torch.uint8 if label_bytes == 1 else torch.int16, device=dev)
        probs = torch.empty((C, *out_shape), dtype=torch.float32, device=dev) if return_probabilities else None
        region_labels = None
        if has_regions:
            region_labels = torch.tensor([int(c) for c in label_manager.regions_class_order], dtype=torch.int32, device=dev)
        L.check(lib.b2u_export_segment(logits.data_ptr(), C, voxels, int(has_regions),
                                       None if region_labels is None else region_labels.data_ptr(), labels.data_ptr(),
                                       label_bytes, None if probs is None else probs.data_ptr(), stream),
                "b2u_export_segment")
        seg = labels.cpu().numpy()
        probs_host = probs.cpu().numpy() if probs is not None else None
    if label_bytes == 2:
        seg = seg.view(np.uint16)
    seg = labels_to_original_geometry(seg, properties_dict, plans_manager.transpose_backward, n_fg)
    if not return_probabilities:
        return seg
    return seg, probabilities_to_original_geometry(probs_host, properties_dict, plans_manager.transpose_backward,
                                                   has_regions)


def export_prediction_from_logits(predicted_array_or_file, properties_dict: dict, configuration_manager, plans_manager,
                                  dataset_json_dict_or_file, output_file_truncated: str, save_probabilities: bool = False):
    """Drop-in for export_prediction.py:70-104: the segmentation through `plans_manager.image_reader_writer_class()`,
    and with `save_probabilities` the probabilities as `<output>.npz` (key `probabilities`) next to a pickle of
    `properties_dict` (`<output>.pkl`)."""
    if isinstance(dataset_json_dict_or_file, str):
        with open(dataset_json_dict_or_file) as f:
            dataset_json_dict_or_file = json.load(f)
    label_manager = plans_manager.get_label_manager(dataset_json_dict_or_file)
    ret = convert_predicted_logits_to_segmentation_with_correct_shape(
        predicted_array_or_file, plans_manager, configuration_manager, label_manager, properties_dict,
        return_probabilities=save_probabilities)
    if save_probabilities:
        segmentation_final, probabilities_final = ret
        np.savez_compressed(output_file_truncated + ".npz", probabilities=probabilities_final)
        with open(output_file_truncated + ".pkl", "wb") as f:
            pickle.dump(properties_dict, f)
    else:
        segmentation_final = ret
    rw = plans_manager.image_reader_writer_class()
    rw.write_seg(segmentation_final, output_file_truncated + dataset_json_dict_or_file["file_ending"], properties_dict)
