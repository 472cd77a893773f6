"""Case preprocessing on the device (reference: `DefaultPreprocessor.run_case_npy`,
preprocessing/preprocessors/default_preprocessor.py:40-118), for 2D configurations.

`DevicePreprocessor.run_case_npy` is a drop-in with the reference's signature.  The case is uploaded once; the
normalization (csrc/preprocess.cu: `b2u_pre_zscore`, `b2u_pre_normalize`, `b2u_pre_minmax_f32`) and the order-3
resampling to the configuration's spacing (`b2u_pre_resample3`) run on the device, and the data stay there:

    data, seg = DevicePreprocessor().run_case_npy(image, None, {"spacing": sp}, plans_manager, configuration_manager,
                                                  dataset_json)           # data: fp32 [C, Z, H, W] on the device

Results are bit-identical to the reference for finite input:
* the crop is the whole volume (cropping.py:34 marks every voxel of the nonzero mask), so `properties` gets
  `shape_before_cropping` = `shape_after_cropping_and_before_resampling` = the transposed shape and the bbox
  `[[0, s], ...]`; the returned seg is the reference's all-zero int8 `[1, *new_shape]` (a host array);
* ZScore reproduces numpy's float32 pairwise summation, in memory order, or with `use_mask_for_norm` in the order of the
  transposed view, which is how the reference's boolean mask gathers;
* the resampling is scipy's order-3 zoom in fp64 with skimage's clip, per slice (separate z along axis 0) or as one
  3-D resize per channel, exactly as `resample_data_or_seg_to_shape` chooses.

Input of another dtype is cast to float32 on the device first, as the reference's image readers deliver it (for such
input the reference's `run_case_npy` would write the normalized values back into the input's dtype).  The case is
copied into a private device buffer first, as the reference copies its input: the caller's array or tensor is never
written.  That copy keeps the input's memory layout (numpy's order 'K', `memory_axes`), because ZScore without the mask
sums in memory order, so C-ordered, Fortran-ordered and transposed inputs each give the reference's bits.  Non-finite input raises ValueError after one read of a device flag (the reference's
NaN-aware clip is not reproduced).  Cases outside this scope raise NotImplementedError before any launch.

Peak extra device memory, besides the private copy (in the input's dtype, and fp32) and the fp32 output: one channel's edge-padded fp64
spline coefficients, 8 * Z * (h + 24) * (w + 24) bytes (8 * (Z + 24) * ... on the 3-D path), plus n / 8 floats of
ZScore tree slots.
"""
import ctypes
import math
from typing import Sequence

import numpy as np
import torch

from . import lib as L

DEFAULT_PREPROCESSOR = "DefaultPreprocessor"
# The planner's `resampling_fn_data` (default_experiment_planner.py:146-160).
DEFAULT_RESAMPLING_FN = "resample_data_or_seg_to_shape"
DEFAULT_RESAMPLING_KWARGS = {"is_seg": False, "order": 3, "order_z": 0, "force_separate_z": None}
ANISO_THRESHOLD = 3  # dinounet/configuration.py
NPAD = 12            # scipy's pre-padding for the spline filter in mode 'nearest'
POLE = -0.267949192431122706472553658494127633  # sqrt(3) - 2, correctly rounded
SCHEME_IDS = {"CTNormalization": 1, "RescaleTo01Normalization": 2, "RGBTo01Normalization": 3}
SCHEMES = ("ZScoreNormalization", "NoNormalization", *SCHEME_IDS)


def filter_consts(n: int):
    """The spline prefilter's constants for a line of n samples: pole, pole^n (host libm), gain, causal and anti-causal
    factors."""
    z = POLE
    zn = math.pow(z, n)
    return [z, zn, (1.0 - z) * (1.0 - 1.0 / z), z / (1 - zn * zn), z / (z - 1)]


def compute_new_shape(old_shape, old_spacing, new_spacing) -> tuple:
    """default_resampling.compute_new_shape."""
    return tuple(int(round(i / j * k)) for i, j, k in zip(old_spacing, new_spacing, old_shape))


def _separate_z_axis(current_spacing, new_spacing):
    """default_resampling: the separate-z low-resolution axis, or None (2 or 3 low-resolution axes disable it)."""
    for sp in (current_spacing, new_spacing):
        sp = np.asarray(sp, dtype=float)
        if np.max(sp) / np.min(sp) > ANISO_THRESHOLD:
            axis = np.where(max(sp) / sp == 1)[0]
            return int(axis[0]) if len(axis) == 1 else None
    return None


def resampling_path(shape, new_shape, original_spacing, target_spacing):
    """None (shapes equal: no resampling), "slices" (separate z along axis 0) or "3d"; NotImplementedError otherwise."""
    if tuple(shape) == tuple(new_shape):
        return None
    if shape[0] != new_shape[0]:
        raise NotImplementedError(f"device preprocessing resamples in-plane only; the target shape {tuple(new_shape)} "
                                  f"changes Z ({shape[0]} slices)")
    axis = _separate_z_axis(original_spacing, target_spacing)
    if axis in (1, 2):
        raise NotImplementedError(f"the low-resolution axis {axis} is in-plane: the reference resamples it separately "
                                  "with order 0, which device preprocessing does not implement")
    return "slices" if axis == 0 else "3d"


def check_configuration(configuration_manager):
    """NotImplementedError unless this is a 2D configuration with the planner's preprocessor and data resampling."""
    conf = getattr(configuration_manager, "configuration", None)
    if not isinstance(conf, dict):
        raise NotImplementedError("device preprocessing needs the configuration dict (ConfigurationManager.configuration)")
    if conf.get("preprocessor_name") != DEFAULT_PREPROCESSOR:
        raise NotImplementedError(f"device preprocessing implements {DEFAULT_PREPROCESSOR} only, got "
                                  f"{conf.get('preprocessor_name')}")
    if conf.get("resampling_fn_data") != DEFAULT_RESAMPLING_FN or \
            dict(conf.get("resampling_fn_data_kwargs") or {}) != DEFAULT_RESAMPLING_KWARGS:
        raise NotImplementedError(f"device preprocessing implements resampling_fn_data = {DEFAULT_RESAMPLING_FN}"
                                  f"(**{DEFAULT_RESAMPLING_KWARGS}) only (the planner's default)")
    if len(configuration_manager.spacing) != 2:
        raise NotImplementedError("device preprocessing handles 2D configurations only, got spacing "
                                  f"{list(configuration_manager.spacing)}")


class DevicePreprocessor:
    """Drop-in for the reference's DefaultPreprocessor at inference (`run_case_npy` with seg None)."""

    def __init__(self, verbose: bool = True, device: torch.device = None):
        self.verbose = verbose
        self.device = device

    def run_case_npy(self, data, seg, properties: dict, plans_manager, configuration_manager, dataset_json):
        """data [C, X, Y, Z] (numpy, or a host or device tensor) -> (fp32 [C, *new_shape] on the device, int8 zeros [1, *new_shape]),
        filling `properties` as the reference does."""
        if seg is not None:
            raise NotImplementedError("device preprocessing covers inference (seg None); training-set preprocessing and "
                                      "the cascade's previous-stage segmentation are not implemented")
        check_configuration(configuration_manager)
        if not isinstance(data, torch.Tensor):
            data = np.asarray(data)
        if data.ndim != 4:
            raise ValueError(f"data must be [C, X, Y, Z], got shape {data.shape}")
        C = data.shape[0]
        schemes = list(configuration_manager.normalization_schemes)
        use_mask = list(configuration_manager.use_mask_for_norm)
        for c in range(C):
            if schemes[c] not in SCHEMES:
                raise NotImplementedError(f"normalization scheme {schemes[c]!r} of channel {c} is not implemented on the "
                                          f"device (implemented: {', '.join(SCHEMES)})")
        tf = [int(i) for i in plans_manager.transpose_forward]
        original_spacing = [properties["spacing"][i] for i in tf]
        shape = tuple(int(data.shape[1 + i]) for i in tf)
        target_spacing = [original_spacing[0], *configuration_manager.spacing]
        new_shape = compute_new_shape(shape, original_spacing, target_spacing)
        path = resampling_path(shape, new_shape, original_spacing, target_spacing)
        intensity = plans_manager.foreground_intensity_properties_per_channel
        ct = {}
        for c in range(C):
            if schemes[c] == "CTNormalization":
                p = intensity[str(c)]
                ct[c] = (np.float32(p["percentile_00_5"]), np.float32(p["percentile_99_5"]), np.float32(p["mean"]),
                         np.float32(max(p["std"], 1e-8)))

        properties["shape_before_cropping"] = shape
        properties["bbox_used_for_cropping"] = [[0, s] for s in shape]
        properties["shape_after_cropping_and_before_resampling"] = shape

        lib = L.load()
        dev = self.device or torch.device("cuda", torch.cuda.current_device())
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            x, axes = _private_copy(data, dev)
            n = int(np.prod(data.shape[1:]))
            d = [int(v) for v in data.shape[1:]]
            # element strides of the logical axes (X, Y, Z) in the private copy, whose channels are laid out in `axes`
            dev_dims = [d[i] for i in axes]
            dev_strides = [dev_dims[1] * dev_dims[2], dev_dims[2], 1]
            mem_strides = [dev_strides[axes.index(i)] for i in range(3)]
            # per-channel exact [min, max] and one non-finite flag, read once
            groups = (n + 65535) // 65536
            mm_work = torch.empty(2 * groups, dtype=torch.float32, device=dev)
            lohi = torch.zeros((C, 2), dtype=torch.float32, device=dev)
            flag = torch.zeros(1, dtype=torch.int32, device=dev)
            for c in range(C):
                L.check(lib.b2u_pre_minmax_f32(x[c].data_ptr(), n, mm_work.data_ptr(), lohi[c].data_ptr(),
                                               flag.data_ptr(), stream), "b2u_pre_minmax_f32")
            lohi_host = lohi.cpu().numpy()
            if int(flag.cpu()[0]):
                raise ValueError("the case holds NaN or infinite values; device preprocessing takes finite input only")
            for c in range(C):
                if schemes[c] == "RGBTo01Normalization":
                    assert lohi_host[c, 0] >= 0, "RGB images are uint 8, for whatever reason I found pixel values " \
                                                 "smaller than 0. Your images do not seem to be RGB images"
                    assert lohi_host[c, 1] <= 255, "RGB images are uint 8, for whatever reason I found pixel values " \
                                                   "greater than 255. Your images do not seem to be RGB images"
            tree = None
            stats = torch.empty(2, dtype=torch.float32, device=dev)
            for c in range(C):
                xc, s = x[c], schemes[c]
                if s == "ZScoreNormalization":
                    tree = torch.empty((n + 7) // 8, dtype=torch.float32, device=dev) if tree is None else tree
                    if use_mask[c]:   # image[mask] gathers in the transposed view's (logical) order
                        o = [int(d[i]) for i in tf] + [int(mem_strides[i]) for i in tf]
                    else:             # memory order
                        o = [1, 1, n, 0, 0, 1]
                    L.check(lib.b2u_pre_zscore(xc.data_ptr(), n, *o, tree.data_ptr(), stats.data_ptr(), stream),
                            "b2u_pre_zscore")
                elif s in SCHEME_IDS:
                    a, b, cc, dd = ct.get(c, (0.0, 0.0, 0.0, 1.0))
                    L.check(lib.b2u_pre_normalize(xc.data_ptr(), n, SCHEME_IDS[s], lohi[c].data_ptr(), float(a),
                                                  float(b), float(cc), float(dd), stream), "b2u_pre_normalize")
            Z, H, W = new_shape
            out = torch.empty((C, Z, H, W), dtype=torch.float32, device=dev)
            if path is None:
                logical = x.permute(0, *[1 + axes.index(i) for i in range(3)])
                out.copy_(logical.permute(0, *[i + 1 for i in tf]))
            else:
                three_d = int(path == "3d")
                z_in, h, w = shape
                consts = (ctypes.c_double * 15)(*(filter_consts(z_in + 2 * NPAD) + filter_consts(h + 2 * NPAD) +
                                                  filter_consts(w + 2 * NPAD)))
                work = torch.empty(int(lib.b2u_pre_resample3_work_doubles(z_in, h, w, three_d)), dtype=torch.float64,
                                   device=dev)
                sz, sy, sx = (mem_strides[i] for i in tf)
                for c in range(C):
                    L.check(lib.b2u_pre_resample3(x[c].data_ptr(), z_in, h, w, sz, sy, sx, H, W, three_d,
                                                  ctypes.addressof(consts), work.data_ptr(), out[c].data_ptr(),
                                                  stream), "b2u_pre_resample3")
        seg_out = np.zeros((1, *new_shape), dtype=np.int8)
        return out, seg_out


def memory_axes(data) -> list:
    """The spatial axes of a case [C, X, Y, Z] in the memory order of the reference's `np.copy(data)` (order 'K': the
    input's layout, with negative strides made positive), outermost first.  numpy reduces a channel in this order."""
    strides = data.stride() if isinstance(data, torch.Tensor) else data.strides
    return sorted(range(3), key=lambda i: -abs(int(strides[i + 1])))


def _private_copy(data, dev):
    """The case as a new fp32 device buffer [C, *spatial axes in memory_axes order] (contiguous; the caller's array or
    tensor is never written), and those axes."""
    axes = memory_axes(data)
    order = (0, *[i + 1 for i in axes])
    if isinstance(data, torch.Tensor) and data.is_cuda:
        x = torch.empty([int(data.shape[i]) for i in order], dtype=torch.float32, device=dev)
        x.copy_(data.detach().permute(*order))
        return x, axes
    if isinstance(data, torch.Tensor):
        host = data.detach().permute(*order).contiguous()
    else:
        host = torch.from_numpy(np.ascontiguousarray(data.transpose(order)))
    up = host.to(dev)                  # a new device tensor: one upload in the input's dtype
    return up.to(torch.float32), axes  # cast on the device (returns `up` itself for fp32 input)


def ensemble_logits(runs, n_folds: int, add_fn) -> torch.Tensor:
    """Fold ensemble of the reference (predict_from_raw_data.py:479-496) on the device: `runs` yields each fold's fp16
    logits; the first is copied, the others added in fp16, then divided by the number of folds, as torch's CPU fp16
    ops do it.  `add_fn(acc, x_or_None, divisor)` is the native step."""
    acc = None
    for logits in runs:
        if acc is None:
            acc = logits.contiguous().clone() if logits.is_contiguous() else logits.contiguous()
        else:
            add_fn(acc, logits.contiguous(), 0)
    if n_folds > 1:
        add_fn(acc, None, n_folds)
    return acc
