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

With a training seg (training-set preprocessing; `run_case` / `run_case_save` read the case and write the trainer's
npz / pkl), the seg is checked once on the device (integer labels in [0, 32767], else NotImplementedError; the
reference's normalization mask `seg >= 0` is then all true, so the data are computed exactly as above), resampled by
batchgenerators' `resize_segmentation(order=1)` in one pass (csrc/preprocess_seg.cu: `b2u_pre_resample_seg`) and
returned as an int8 / int16 device tensor by the reference's `np.max(seg) > 127` rule, and
`properties["class_locations"]` gets `_sample_foreground_locations`' keys and rows (`b2u_pre_seg_count`,
`b2u_pre_seg_compact`, `b2u_pre_seg_gather`; the RandomState draws stay on the host).  `run` is the dataset loop
(default_preprocessor.py:197-260) without the spawn pool: the cases run in order on the current device while threads
read the next cases and compress and write the finished ones.  Not implemented: the `modify_seg_fn` hook and the
cascade's previous-stage segmentation.

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
import json
import math
import os
import pickle
import shutil
from concurrent.futures import ThreadPoolExecutor
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


# The planner's `resampling_fn_seg` kwargs; the seg's dtype codes (B2U_EVAL_*: uint16 travels as int16 bits).
DEFAULT_RESAMPLING_SEG_KWARGS = {"is_seg": True, "order": 1, "order_z": 0, "force_separate_z": None}
SEG_DTYPE_CODES = {np.dtype(np.uint8): 0, np.dtype(np.int8): 1, np.dtype(np.int16): 2, np.dtype(np.uint16): 3,
                   np.dtype(np.int32): 4, np.dtype(np.float32): 5}
_TORCH_SEG_DTYPES = {torch.uint8: np.uint8, torch.int8: np.int8, torch.int16: np.int16, torch.int32: np.int32,
                     torch.float32: np.float32, torch.uint16: np.uint16}
MAX_LABEL = 32767
# _sample_foreground_locations (default_preprocessor.py:156-181)
LOCATIONS_SEED, NUM_SAMPLES, MIN_PERCENT_COVERAGE = 1234, 10000, 0.01


def sample_count(n: int) -> int:
    """The rows `_sample_foreground_locations` draws from a class of n voxels."""
    return max(min(NUM_SAMPLES, n), int(np.ceil(n * MIN_PERCENT_COVERAGE)))


def foreground_classes(label_manager) -> list:
    """The classes run_case_npy collects locations for, as (key, sorted distinct labels): the foreground regions or
    labels, and all labels when the dataset has an ignore label.  The label manager's lists are not modified."""
    classes = list(label_manager.foreground_regions if label_manager.has_regions else label_manager.foreground_labels)
    if label_manager.has_ignore_label:
        classes.append(label_manager.all_labels)
    return [(c if not isinstance(c, list) else tuple(c),
             sorted({int(v) for v in c}) if isinstance(c, (tuple, list)) else [int(c)]) for c in classes]


def check_training_seg(data, seg, plans_manager, configuration_manager, dataset_json):
    """Rejects, before any launch, what the device does not implement for a training seg; returns the seg (a numpy
    array or a tensor) and foreground_classes()."""
    conf = configuration_manager.configuration
    if conf.get("resampling_fn_seg") != DEFAULT_RESAMPLING_FN or \
            dict(conf.get("resampling_fn_seg_kwargs") or {}) != DEFAULT_RESAMPLING_SEG_KWARGS:
        raise NotImplementedError(f"device preprocessing of a seg implements resampling_fn_seg = {DEFAULT_RESAMPLING_FN}"
                                  f"(**{DEFAULT_RESAMPLING_SEG_KWARGS}) only (the planner's default); the cascade's "
                                  "previous-stage segmentation is not implemented")
    if not callable(getattr(plans_manager, "get_label_manager", None)):
        raise NotImplementedError("device preprocessing of a seg needs plans_manager.get_label_manager")
    if isinstance(seg, torch.Tensor):
        if seg.dtype not in _TORCH_SEG_DTYPES:
            raise NotImplementedError(f"seg dtype {seg.dtype} is not implemented on the device (implemented: uint8, "
                                      "int8, int16, uint16, int32, float32)")
    else:
        seg = np.asarray(seg)
        if seg.dtype not in SEG_DTYPE_CODES:
            raise NotImplementedError(f"seg dtype {seg.dtype} is not implemented on the device (implemented: uint8, "
                                      "int8, int16, uint16, int32, float32)")
    if tuple(data.shape[1:]) != tuple(seg.shape[1:]):
        raise AssertionError("Shape mismatch between image and segmentation. Please fix your dataset and make use of "
                             "the --verify_dataset_integrity flag to ensure everything is correct")
    if seg.ndim != 4 or seg.shape[0] != 1:
        raise NotImplementedError(f"device preprocessing takes a seg of one channel [1, X, Y, Z], got {tuple(seg.shape)}")
    classes = foreground_classes(plans_manager.get_label_manager(dataset_json))
    if len(classes) > 4096:
        raise NotImplementedError(f"{len(classes)} classes: at most 4096 are implemented on the device")
    return seg, classes


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
    """Drop-in for the reference's DefaultPreprocessor: `run_case_npy` at inference (seg None) and for training cases,
    `run_case` and `run_case_save`."""

    def __init__(self, verbose: bool = True, device: torch.device = None):
        self.verbose = verbose
        self.device = device

    def run_case_npy(self, data, seg, properties: dict, plans_manager, configuration_manager, dataset_json):
        """data [C, X, Y, Z] (numpy, or a host or device tensor) -> (fp32 [C, *new_shape] on the device, seg), filling
        `properties` as the reference does.  Without a seg, seg is the reference's int8 zeros [1, *new_shape] (a host
        array); with a training seg [1, X, Y, Z] it is the resampled label map as an int8 / int16 device tensor and
        `properties["class_locations"]` holds the foreground locations."""
        check_configuration(configuration_manager)
        if not isinstance(data, torch.Tensor):
            data = np.asarray(data)
        if data.ndim != 4:
            raise ValueError(f"data must be [C, X, Y, Z], got shape {data.shape}")
        classes = None
        if seg is not None:
            seg, classes = check_training_seg(data, seg, plans_manager, configuration_manager, dataset_json)
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

        if seg is not None and int(np.prod(new_shape)) >= 2 ** 31:
            raise NotImplementedError(f"the resampled seg {tuple(new_shape)} has 2^31 voxels or more")

        properties["shape_before_cropping"] = shape
        properties["bbox_used_for_cropping"] = [[0, s] for s in shape]
        properties["shape_after_cropping_and_before_resampling"] = shape

        lib = L.load()
        dev = self.device or torch.device("cuda", torch.cuda.current_device())
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            if seg is not None:   # labels are checked before the data are touched
                seg_dev, seg_code, seg_max = _checked_seg_copy(seg, tf, dev, lib, stream)
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
            if seg is not None:
                seg_out, properties["class_locations"] = _training_seg(seg_dev, seg_code, seg_max, path, new_shape,
                                                                       classes, dev, lib, stream)
                return out, seg_out
        seg_out = np.zeros((1, *new_shape), dtype=np.int8)
        return out, seg_out

    def run_case(self, image_files, seg_file, plans_manager, configuration_manager, dataset_json):
        """DefaultPreprocessor.run_case (default_preprocessor.py:120-146): reads the images (and the seg, if any) with
        the plans' reader on the host and preprocesses them on the device.  Returns (data, seg, properties)."""
        if isinstance(dataset_json, str):
            with open(dataset_json) as f:
                dataset_json = json.load(f)
        data, seg, data_properties = _read_case(image_files, seg_file, plans_manager)
        data, seg = self.run_case_npy(data, seg, data_properties, plans_manager, configuration_manager, dataset_json)
        return data, seg, data_properties

    def run_case_save(self, output_filename_truncated: str, image_files, seg_file, plans_manager, configuration_manager,
                      dataset_json):
        """DefaultPreprocessor.run_case_save (lines 148-154): `<name>.npz` (data, seg as host arrays, compressed) and the
        properties pickled to `<name>.pkl`, the files the trainer loads."""
        data, seg, properties = self.run_case(image_files, seg_file, plans_manager, configuration_manager, dataset_json)
        _save_case(output_filename_truncated, _host(data), _host(seg), properties)

    def run(self, dataset_name_or_id, configuration_name: str, plans_identifier: str, num_processes: int):
        """DefaultPreprocessor.run (default_preprocessor.py:197-260): the plans and dataset.json of the preprocessed
        folder, a fresh `<data_identifier>/` and one `<case>.npz` / `<case>.pkl` per training case, each what
        `run_case_save` writes.  The cases run in order on the current device; `num_processes` threads read the next
        cases ahead and as many compress and write the finished ones."""
        dataset_name = _dataset_name(dataset_name_or_id)
        raw, preprocessed = _raw_and_preprocessed()
        assert os.path.isdir(os.path.join(raw, dataset_name)), "The requested dataset could not be found in nnUNet_raw"
        plans_file = os.path.join(preprocessed, dataset_name, plans_identifier + ".json")
        assert os.path.isfile(plans_file), "Expected plans file (%s) not found. Run corresponding " \
                                           "nnUNet_plan_experiment first." % plans_file
        with open(plans_file) as f:
            plans_manager = _plans_manager(json.load(f))
        configuration_manager = plans_manager.get_configuration(configuration_name)
        if self.verbose:
            print(f"Preprocessing the following configuration: {configuration_name}")
            print(configuration_manager)
        with open(os.path.join(preprocessed, dataset_name, "dataset.json")) as f:
            dataset_json = json.load(f)
        output_directory = os.path.join(preprocessed, dataset_name, configuration_manager.data_identifier)
        if os.path.isdir(output_directory):
            shutil.rmtree(output_directory)
        os.makedirs(output_directory, exist_ok=True)
        dataset = _get_filenames_of_train_images_and_targets(os.path.join(raw, dataset_name), dataset_json)
        keys = list(dataset.keys())
        workers = max(1, int(num_processes))
        with ThreadPoolExecutor(workers) as readers, ThreadPoolExecutor(workers) as writers:
            reads = [readers.submit(_read_case, dataset[k]["images"], dataset[k]["label"], plans_manager)
                     for k in keys[:workers]]
            writes = []
            for i, k in enumerate(keys):
                data, seg, properties = reads[i].result()
                if i + workers < len(keys):
                    nk = keys[i + workers]
                    reads.append(readers.submit(_read_case, dataset[nk]["images"], dataset[nk]["label"], plans_manager))
                data, seg = self.run_case_npy(data, seg, properties, plans_manager, configuration_manager,
                                              dataset_json)
                writes.append(writers.submit(_save_case, os.path.join(output_directory, k), _host(data), _host(seg),
                                             properties))
                reads[i] = None
                while len([w for w in writes if not w.done()]) > workers:   # bound the host copies held for writing
                    next(w for w in writes if not w.done()).result()
            for w in writes:
                w.result()


def _read_case(image_files, seg_file, plans_manager):
    """The case as the plans' reader delivers it: (images, seg or None, properties)."""
    rw = plans_manager.image_reader_writer_class()
    data, data_properties = rw.read_images(image_files)
    seg = rw.read_seg(seg_file)[0] if seg_file is not None else None
    return data, seg, data_properties


def _save_case(output_filename_truncated: str, data: np.ndarray, seg: np.ndarray, properties: dict):
    np.savez_compressed(output_filename_truncated + ".npz", data=data, seg=seg)
    with open(output_filename_truncated + ".pkl", "wb") as f:
        pickle.dump(properties, f)


# ---- the host nnU-Net's dataset helpers, which the dataset loops are called from (tests substitute them) -------------


def _dataset_name(dataset_name_or_id) -> str:
    from dinounet.utilities.dataset_name_id_conversion import maybe_convert_to_dataset_name
    return maybe_convert_to_dataset_name(dataset_name_or_id)


def _raw_and_preprocessed():
    """(nnUNet_raw, nnUNet_preprocessed)."""
    from dinounet import paths
    return paths.nnUNet_raw, paths.nnUNet_preprocessed


def _plans_manager(plans: dict):
    from dinounet.utilities.plans_handling.plans_handler import PlansManager
    return PlansManager(plans)


def _get_filenames_of_train_images_and_targets(raw_dataset_folder: str, dataset_json: dict) -> dict:
    from dinounet.utilities.utils import get_filenames_of_train_images_and_targets
    return get_filenames_of_train_images_and_targets(raw_dataset_folder, dataset_json)


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


def _seg_dtype_code(seg) -> int:
    dt = _TORCH_SEG_DTYPES[seg.dtype] if isinstance(seg, torch.Tensor) else seg.dtype
    return SEG_DTYPE_CODES[np.dtype(dt)]


def _checked_seg_copy(seg, tf, dev, lib, stream):
    """seg[0] as a new C-contiguous device tensor [Z, h, w] in the transposed order, in its stored bits (the caller's
    array or tensor is never written), after one read of the label check: NotImplementedError for labels that are
    negative, above 32767 or not integers.  Returns (copy, dtype code, largest label)."""
    code = _seg_dtype_code(seg)
    if isinstance(seg, torch.Tensor):
        s = seg.detach()[0]
        s = s.view(torch.int16) if code == 3 else s
        x = torch.empty([int(s.shape[i]) for i in tf], dtype=s.dtype, device=dev)
        x.copy_(s.permute(*tf))
    else:
        s = seg[0].view(np.int16) if code == 3 else seg[0]
        axes = memory_axes(seg)
        up = torch.from_numpy(np.ascontiguousarray(s.transpose(axes))).to(dev)   # one upload in the stored dtype
        x = up.permute(*[axes.index(i) for i in range(3)]).permute(*tf).contiguous()
    chk = torch.zeros(3, dtype=torch.int32, device=dev)
    L.check(lib.b2u_pre_seg_check(x.data_ptr(), code, x.numel(), chk.data_ptr(), stream), "b2u_pre_seg_check")
    lo, hi, bad = (int(v) for v in chk.cpu())
    if bad:
        raise NotImplementedError("the seg holds non-integer or non-finite labels; device preprocessing takes integer "
                                  "labels only")
    if lo < 0 or hi > MAX_LABEL:
        raise NotImplementedError(f"seg labels span [{lo}, {hi}]: device preprocessing takes labels in [0, {MAX_LABEL}] "
                                  "(negative labels would change the normalization mask)")
    return x, code, hi


def _training_seg(seg, code, seg_max, path, new_shape, classes, dev, lib, stream):
    """Resamples the checked seg copy [Z, h, w] to new_shape and samples the foreground locations.  Returns (int8 /
    int16 seg [1, *new_shape] on the device, class_locations)."""
    Z, H, W = (int(v) for v in new_shape)
    K = len(classes)
    info = torch.zeros(1 + K, dtype=torch.int64, device=dev)   # the resampled maximum, then the class counts
    if path is not None:
        out = torch.empty((Z, H, W), dtype=seg.dtype, device=dev)
        L.check(lib.b2u_pre_resample_seg(seg.data_ptr(), code, Z, int(seg.shape[1]), int(seg.shape[2]), H, W,
                                         out.data_ptr(), info.data_ptr(), stream), "b2u_pre_resample_seg")
        seg = out
    n = Z * H * W
    offsets = np.cumsum([0] + [len(labels) for _, labels in classes]).astype(np.int32)
    if K:
        labels = torch.tensor([v for _, lab in classes for v in lab], dtype=torch.int64).to(dev)
        offs = torch.from_numpy(offsets).to(dev)
        L.check(lib.b2u_pre_seg_count(seg.data_ptr(), code, n, labels.data_ptr(), offs.data_ptr(), K,
                                      info[1:].data_ptr(), stream), "b2u_pre_seg_count")
    info = info.cpu().numpy()
    out_max = seg_max if path is None else int(info[0])
    counts = [int(c) for c in info[1:]]
    locations = {key: [] for key, _ in classes}
    pending = []
    if any(counts):
        idx = torch.empty(max(counts), dtype=torch.int32, device=dev)
        work = torch.empty(int(lib.b2u_pre_seg_compact_work_ints(n)), dtype=torch.int32, device=dev)
        rndst = np.random.RandomState(LOCATIONS_SEED)
        for k, (key, lab) in enumerate(classes):
            if counts[k] == 0:
                continue
            L.check(lib.b2u_pre_seg_compact(seg.data_ptr(), code, n, labels.data_ptr() + 8 * int(offsets[k]), len(lab),
                                            work.data_ptr(), idx.data_ptr(), stream), "b2u_pre_seg_compact")
            # the reference's draw (legacy choice without replacement: permutation(n)[:t]), while the device compacts
            ranks = torch.from_numpy(rndst.choice(counts[k], sample_count(counts[k]), replace=False)).to(dev)
            rows = torch.empty((ranks.numel(), 4), dtype=torch.int64, device=dev)
            L.check(lib.b2u_pre_seg_gather(idx.data_ptr(), ranks.data_ptr(), ranks.numel(), H, W, rows.data_ptr(),
                                           stream), "b2u_pre_seg_gather")
            pending.append((key, rows))
    for key, rows in pending:
        locations[key] = rows.cpu().numpy()
    seg_out = seg.to(torch.int16 if out_max > 127 else torch.int8)   # exact: the labels lie in [0, 32767]
    return seg_out.reshape(1, Z, H, W), locations


def _host(x) -> np.ndarray:
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


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
