"""Scoring predictions against the ground truth on the device (reference: `dinounet/evaluation/evaluate_predictions.py`).

`compute_metrics_arrays` scores one case given as arrays or tensors shaped `(1, *spatial)`; `compute_metrics` and
`compute_metrics_on_folder` are drop-ins with the reference's signatures that read the files with the caller's
reader-writer.  Per label or region the device computes (csrc/evaluation.cu):

* the masks `seg == r` (or their union over a region's labels) straight from the stored dtypes (uint8, int8, int16,
  uint16, int32, float32; the two operands may differ), their face-connectivity borders and the exact int64
  TP / FP / FN / TN over the voxels whose reference is not the ignore label (`b2u_eval_masks`);
* when both masks are non-empty, medpy's surface distances (`hd95` / `asd`, medpy 0.4/0.5): the exact anisotropic
  Euclidean distance transform of each border (`b2u_eval_edt`, scipy's arithmetic: bit-identical at integer spacings),
  the distances gathered at the other mask's border in C order, ASD as numpy's pairwise float64 mean
  (`b2u_eval_sum_f64`) and HD95 from the two order statistics numpy's linear percentile interpolates.

Only scalars come back to the host: the six counts, one sum and two order statistics per label or region.  The ratios
are computed there with the reference's expressions, so keys, order, NaN rules and value types are the reference's.
As in the reference, every foreground voxel on the first or last slice along an axis is surface (erosion uses border
value 0), and the ignore label changes the counts only.

Peak extra device memory per case: the two label volumes as stored, two uint8 border masks, and while surface distances
are computed two float64 volumes, one int32 volume and the gathered distances.
"""
from __future__ import annotations

import ctypes
import json
import math
import os
from concurrent.futures import ThreadPoolExecutor
from copy import deepcopy

import numpy as np
import torch

from . import lib as L

METRIC_KEYS = ("Dice", "IoU", "Sensitivity", "Specificity", "Precision", "HD95", "ASD", "FP", "TP", "FN", "TN",
               "n_pred", "n_ref")
MAX_REGION_LABELS = 8  # B2U_EVAL_MAX_REGION_LABELS: a region's label values travel to the kernel by value
DTYPE_CODES = {torch.uint8: 0, torch.int8: 1, torch.int16: 2, torch.uint16: 3, torch.int32: 4, torch.float32: 5}
# dinounet/configuration.py's default_num_processes
DEFAULT_NUM_PROCESSES = int(os.environ.get("nnUNet_def_n_proc", 8))


# ---- host-side restatements ------------------------------------------------------------------------------------------


def surface_spacing(spacing, ndim: int):
    """The spacing medpy receives for a mask of rank `ndim` (evaluate_predictions.py:123-136).  None when its length
    still differs from the rank: medpy then raises, and the reference reports NaN."""
    spacing = tuple(float(s) for s in spacing)
    if len(spacing) > ndim:
        spacing = spacing[-ndim:]
    elif len(spacing) < ndim - 1:
        spacing = spacing + (1.0,) * (ndim - len(spacing))
    return spacing if len(spacing) == ndim else None


def percentile95_indices(n: int):
    """numpy's linear `percentile(x, 95)` over n values: the two order statistics it reads and its interpolation weight
    (numpy 2.x `_quantile`: virtual index (n - 1) * q with q = 95 / 100, `_get_indexes`, `_get_gamma`)."""
    q = np.true_divide(95, np.float64(100))
    v = np.float64(n - 1) * q
    if v >= n - 1:
        return n - 1, n - 1, v + 1.0  # numpy reads the last element twice (its index -1)
    lo = int(np.floor(v))
    return lo, lo + 1, v - np.float64(lo)


def lerp(a, b, t):
    """numpy's `_lerp` on float64 scalars: a + (b - a) t, or b - (b - a)(1 - t) where t >= 0.5."""
    a, b, t = np.float64(a), np.float64(b), np.float64(t)
    d = b - a
    return b - d * (1 - t) if t >= 0.5 else a + d * t


def percentile95(order_statistic, n: int):
    """`np.percentile(x, 95)` of n values given `order_statistic(k)`, the k-th smallest (0-based)."""
    lo, hi, t = percentile95_indices(n)
    return lerp(order_statistic(lo), order_statistic(hi), t)


def ratios(tp, fp, fn, tn, hd95, asd) -> dict:
    """The reference's per-case metric dict from int64 counts (evaluate_predictions.py:186-229)."""
    m = {}
    if tp + fp + fn == 0:
        m["Dice"] = np.nan
        m["IoU"] = np.nan
    else:
        m["Dice"] = 2 * tp / (2 * tp + fp + fn)
        m["IoU"] = tp / (tp + fp + fn)
    m["Sensitivity"] = tp / (tp + fn) if tp + fn > 0 else np.nan
    m["Specificity"] = tn / (tn + fp) if tn + fp > 0 else np.nan
    m["Precision"] = tp / (tp + fp) if tp + fp > 0 else np.nan
    m["HD95"] = hd95
    m["ASD"] = asd
    m["FP"] = fp
    m["TP"] = tp
    m["FN"] = fn
    m["TN"] = tn
    m["n_pred"] = fp + tp
    m["n_ref"] = fn + tp
    return m


def _region_values(r) -> list:
    values = [r] if np.isscalar(r) else list(r)
    for v in values:
        if not isinstance(v, (int, np.integer)) or isinstance(v, (bool, np.bool_)):
            raise NotImplementedError(f"label {v!r} of {r!r}: only integer labels are supported")
        if not -2 ** 63 <= int(v) < 2 ** 63:
            raise NotImplementedError(f"label {v!r} of {r!r} does not fit in int64")
    if not 1 <= len(values) <= MAX_REGION_LABELS:
        raise NotImplementedError(f"region {r!r} has {len(values)} label values; the kernel takes 1 to "
                                  f"{MAX_REGION_LABELS}")
    return [int(v) for v in values]


def _as_tensor(seg, what: str) -> torch.Tensor:
    t = torch.from_numpy(np.ascontiguousarray(seg)) if isinstance(seg, np.ndarray) else seg
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{what}: expected a numpy array or a torch tensor, got {type(seg).__name__}")
    if t.dtype not in DTYPE_CODES:
        raise NotImplementedError(f"{what}: dtype {t.dtype} is not supported (uint8, int8, int16, uint16, int32, "
                                  "float32)")
    return t


def _device(ref: torch.Tensor, pred: torch.Tensor) -> torch.device:
    """The operands' CUDA device, else the current one (host data is uploaded there)."""
    for t in (ref, pred):
        if t.is_cuda:
            return t.device
    return torch.device("cuda", torch.cuda.current_device())


def _to_device(t: torch.Tensor, device) -> torch.Tensor:
    return t.to(device, non_blocking=False).contiguous()


# ---- one case ----------------------------------------------------------------------------------------------------------


def compute_metrics_arrays(seg_ref, seg_pred, labels_or_regions, ignore_label=None, spacing=None) -> dict:
    """The reference's per-case `results['metrics']` for two segmentations shaped `(1, *spatial)` (numpy arrays or
    tensors; CUDA tensors are read in place on their device, host data is uploaded to the current device).  `spacing`
    is the reader's spacing of the spatial axes (default isotropic 1).  Keys in `labels_or_regions` order, each holding
    METRIC_KEYS in that order with the reference's value types."""
    ref = _as_tensor(seg_ref, "seg_ref")
    pred = _as_tensor(seg_pred, "seg_pred")
    if tuple(ref.shape) != tuple(pred.shape):
        raise ValueError(f"seg_ref {tuple(ref.shape)} and seg_pred {tuple(pred.shape)} differ in shape")
    if ref.dim() < 2 or ref.dim() > 4 or ref.shape[0] != 1:
        raise NotImplementedError(f"segmentations shaped {tuple(ref.shape)}: expected (1, *spatial) with 1 to 3 spatial "
                                  "axes")
    spatial = tuple(int(s) for s in ref.shape[1:])
    if min(spatial) <= 0:
        raise ValueError(f"empty segmentation {tuple(ref.shape)}")
    ndim = len(spatial)
    if spacing is None:
        spacing = (1.0,) * ndim
    sp = surface_spacing(spacing, ndim)
    if sp is not None and not all(math.isfinite(s) and s > 0 for s in sp):
        raise ValueError(f"spacing {tuple(spacing)} must be positive and finite")
    regions = [(r, _region_values(r)) for r in labels_or_regions]
    if ignore_label is not None:
        _region_values(ignore_label)
    Z, Y, X = (1,) * (3 - ndim) + spatial
    n = Z * Y * X

    device = _device(ref, pred)
    lib = L.load()
    out = {}
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device).cuda_stream
        ref_d, pred_d = _to_device(ref, device), _to_device(pred, device)
        border_ref = torch.empty(n, dtype=torch.uint8, device=device)
        border_pred = torch.empty(n, dtype=torch.uint8, device=device)
        counts = torch.empty(6, dtype=torch.int64, device=device)
        edt = None
        for r, values in regions:
            arr = (ctypes.c_int64 * len(values))(*values)
            L.check(lib.b2u_eval_masks(ref_d.data_ptr(), DTYPE_CODES[ref.dtype], pred_d.data_ptr(),
                                       DTYPE_CODES[pred.dtype], ndim, Z, Y, X, arr, len(values),
                                       int(ignore_label is not None), 0 if ignore_label is None else int(ignore_label),
                                       border_ref.data_ptr(), border_pred.data_ptr(), counts.data_ptr(), stream),
                    "b2u_eval_masks")
            tp, fp, fn, tn, n_ref, n_pred = (np.int64(c) for c in counts.cpu().numpy())
            hd95 = asd = np.nan
            if n_ref > 0 and n_pred > 0 and sp is not None:
                if edt is None:
                    edt = (torch.empty(n, dtype=torch.float64, device=device),
                           torch.empty(n, dtype=torch.float64, device=device),
                           torch.empty(n, dtype=torch.int32, device=device))
                hd95, asd = _surface_metrics(lib, border_ref, border_pred, (Z, Y, X), (1.0,) * (3 - ndim) + sp, edt,
                                             stream)
            out[r] = ratios(tp, fp, fn, tn, hd95, asd)
    return out


def _surface_metrics(lib, border_ref, border_pred, shape, sp, edt, stream):
    """medpy's hd95(pred, ref) and asd(pred, ref) as Python floats (the reference stores float(...))."""
    dt, tmp, scratch = edt

    def distances_to(border, at):
        L.check(lib.b2u_eval_edt(border.data_ptr(), *shape, *sp, tmp.data_ptr(), scratch.data_ptr(), dt.data_ptr(),
                                 stream), "b2u_eval_edt")
        return dt.masked_select(at.view(torch.bool))  # C order, as numpy's boolean indexing gathers

    pred_to_ref = distances_to(border_ref, border_pred)   # medpy's __surface_distances(pred, ref)
    ref_to_pred = distances_to(border_pred, border_ref)   # ... (ref, pred)
    n_a = pred_to_ref.numel()
    work = torch.empty(max(1, (n_a + 7) // 8), dtype=torch.float64, device=dt.device)
    L.check(lib.b2u_eval_sum_f64(pred_to_ref.data_ptr(), n_a, work.data_ptr(), stream), "b2u_eval_sum_f64")
    both = torch.cat((pred_to_ref, ref_to_pred))
    lo, hi, t = percentile95_indices(both.numel())
    stats = torch.stack((work[0], both.kthvalue(lo + 1).values, both.kthvalue(hi + 1).values)).cpu().numpy()
    asd = np.float64(stats[0]) / np.intp(n_a)  # numpy's mean: the pairwise sum over the count
    return float(lerp(stats[1], stats[2], t)), float(asd)


# ---- files and folders -------------------------------------------------------------------------------------------------


def _case_spacing(seg_ref, seg_ref_dict, seg_pred_dict):
    """evaluate_predictions.py:159-172."""
    spacing = seg_ref_dict.get("spacing", None)
    if spacing is None:
        spacing = seg_pred_dict.get("spacing", None)
    if spacing is None:
        spacing = tuple([1.0] * (np.ndim(seg_ref) - 1))
        print(f"Warning: No spacing information found, using default isotropic spacing: {spacing}")
    return spacing


def _score(reference_file, prediction_file, loaded, labels_or_regions, ignore_label) -> dict:
    (seg_ref, seg_ref_dict), (seg_pred, seg_pred_dict) = loaded
    spacing = _case_spacing(seg_ref, seg_ref_dict, seg_pred_dict)
    return {"reference_file": reference_file, "prediction_file": prediction_file,
            "metrics": compute_metrics_arrays(seg_ref, seg_pred, labels_or_regions, ignore_label, spacing)}


def compute_metrics(reference_file: str, prediction_file: str, image_reader_writer, labels_or_regions,
                    ignore_label: int = None) -> dict:
    """Drop-in for the reference's `compute_metrics`: reads both files with `image_reader_writer.read_seg` and scores
    them on the current device."""
    loaded = (image_reader_writer.read_seg(reference_file), image_reader_writer.read_seg(prediction_file))
    return _score(reference_file, prediction_file, loaded, labels_or_regions, ignore_label)


def _subfiles(folder: str, suffix: str) -> list:
    """batchgenerators' `subfiles(folder, suffix=..., join=False)`: sorted file names ending in suffix."""
    return sorted(f for f in os.listdir(folder) if os.path.isfile(os.path.join(folder, f)) and f.endswith(suffix))


def fix_for_json_export(obj):
    """In place, what the reference's `recursive_fix_for_json_export` does to these results: numpy integer keys become
    int, numpy bools / integers / floats become Python values, inside dicts, lists and tuples."""
    def value(v):
        if isinstance(v, dict):
            fix_for_json_export(v)
            return v
        if isinstance(v, np.bool_):
            return bool(v)
        if isinstance(v, np.integer):
            return int(v)
        if isinstance(v, np.floating):
            return float(v)
        if isinstance(v, (list, tuple)):
            return type(v)(value(i) for i in v)
        return v
    for k in list(obj.keys()):
        v = obj.pop(k) if isinstance(k, np.integer) else obj[k]
        obj[int(k) if isinstance(k, np.integer) else k] = value(v)
    return obj


def aggregate(results: list, regions_or_labels) -> dict:
    """The reference's summary over per-case results (evaluate_predictions.py:269-295): np.nanmean per label or region
    and metric, the plain mean over every key but 0 as `foreground_mean`, then the JSON fix-up."""
    metric_list = list(results[0]["metrics"][regions_or_labels[0]].keys())
    means = {}
    for r in regions_or_labels:
        means[r] = {m: np.nanmean([i["metrics"][r][m] for i in results]) for m in metric_list}
    foreground_mean = {}
    for m in metric_list:
        foreground_mean[m] = np.mean([means[k][m] for k in means.keys() if not (k == 0 or k == "0")])
    for i in results:
        fix_for_json_export(i)
    fix_for_json_export(means)
    fix_for_json_export(foreground_mean)
    return {"metric_per_case": results, "mean": means, "foreground_mean": foreground_mean}


def save_summary_json(results: dict, output_file: str):
    """The reference's `save_summary_json`: label / region keys as `str(key)`, written by `json` with indent 4 and
    sorted keys."""
    converted = deepcopy(results)
    converted["mean"] = {str(k): results["mean"][k] for k in results["mean"].keys()}
    for i in range(len(converted["metric_per_case"])):
        converted["metric_per_case"][i]["metrics"] = {str(k): v for k, v in
                                                      results["metric_per_case"][i]["metrics"].items()}
    with open(output_file, "w") as f:
        json.dump(converted, f, sort_keys=True, indent=4)


def compute_metrics_on_folder(folder_ref: str, folder_pred: str, output_file: str, image_reader_writer,
                              file_ending: str, regions_or_labels, ignore_label: int = None,
                              num_processes: int = DEFAULT_NUM_PROCESSES, chill: bool = True) -> dict:
    """Drop-in for the reference's `compute_metrics_on_folder` (same file selection, summary and JSON).  Cases are
    scored one after another on the current device; `num_processes` threads read the next cases meanwhile."""
    if output_file is not None:
        assert output_file.endswith(".json"), "output_file should end with .json"
    files_pred = _subfiles(folder_pred, file_ending)
    if not chill:
        present = [os.path.isfile(os.path.join(folder_ref, i)) for i in files_pred]
        if not all(present):
            missing = [f for f, p in zip(files_pred, present) if not p]
            print(f"Warning: {len(missing)}/{len(files_pred)} prediction files have no reference and are skipped:")
            for f in missing:
                print(f"  - {f}")
            files_pred = [f for f, p in zip(files_pred, present) if p]
    files_ref = [os.path.join(folder_ref, i) for i in files_pred]
    files_pred = [os.path.join(folder_pred, i) for i in files_pred]

    def read(i):
        return image_reader_writer.read_seg(files_ref[i]), image_reader_writer.read_seg(files_pred[i])

    window = max(1, int(num_processes))
    results = []
    with ThreadPoolExecutor(window) as pool:
        pending = [pool.submit(read, i) for i in range(min(window, len(files_pred)))]
        for i in range(len(files_pred)):
            loaded = pending[i].result()
            if i + window < len(files_pred):
                pending.append(pool.submit(read, i + window))
            pending[i] = None
            results.append(_score(files_ref[i], files_pred[i], loaded, regions_or_labels, ignore_label))
    result = aggregate(results, regions_or_labels)
    if output_file is not None:
        save_summary_json(result, output_file)
    return result
