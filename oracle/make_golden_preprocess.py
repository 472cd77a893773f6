"""Writes tests/golden/preprocess_cases.npz: the reference's own `DefaultPreprocessor.run_case_npy`
(default_preprocessor.py:40-118), `crop_to_nonzero` (cropping.py), normalization classes
(default_normalization_schemes.py) and `resample_data_or_seg_to_shape` (default_resampling.py) on the cases of
`CASES`, with the plans' default resampling kwargs.

Stand-ins only for modules that are not installed here: skimage's `resize` (as skimage >= 0.19.3 computes it for
order 3 / mode 'edge' / no anti-aliasing on float64: scipy's zoom with grid_mode=True, then the clip to the input's
range), batchgenerators' `resize_segmentation` (called on the all-zero seg only) and file helpers, the acvl_utils bbox
helpers, and the plans-handling / path modules that default_preprocessor.py imports but `run_case_npy` does not use.

    python oracle/make_golden_preprocess.py
"""
import importlib
import os
import sys
import types
from types import SimpleNamespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "preprocess_cases.npz")

# name, C x (X, Y, Z) input shape and dtype, spacing, transpose_forward, configuration spacing, schemes, use_mask
CASES = [
    # separate z (spacing ratio > 3, low-resolution axis 0): per-slice 2-D resizes; up-sampling, ZScore memory order
    ("slices_up_zscore", (1, 3, 37, 29), "float32", [5.0, 0.8, 0.8], [0, 1, 2], [0.5, 0.5], ["ZScoreNormalization"],
     [False]),
    # non-identity transpose_forward, ZScore with and without the mask, down-sampling
    ("slices_down_tf_mask", (2, 45, 2, 52), "float32", [0.7, 4.0, 0.7], [1, 0, 2], [1.1, 0.9],
     ["ZScoreNormalization", "ZScoreNormalization"], [True, False]),
    # near-isotropic spacing: one 3-D resize per channel (Z factor 1); mixed factors; CT + RescaleTo01
    ("volume_mixed_ct_rescale", (2, 3, 31, 40), "float32", [1.0, 0.9, 1.1], [0, 1, 2], [1.3, 0.7],
     ["CTNormalization", "RescaleTo01Normalization"], [False, False]),
    # 2 low-resolution axes (separate z disabled): 3-D path with axes of length 1 and 2 in plane
    ("volume_thin_axes", (1, 2, 1, 33), "float32", [2.0, 2.0, 0.5], [0, 1, 2], [0.7, 0.4], ["ZScoreNormalization"],
     [False]),
    # RGB natural image (uint8 values, the readers deliver float32), 3 channels, in-plane resampling per slice
    ("rgb_slices", (3, 1, 48, 64), "uint8", [999.0, 1.0, 1.0], [0, 1, 2], [1.5, 1.5], ["RGBTo01Normalization"] * 3,
     [False] * 3),
    # identity shape: returned as normalized, no resampling; constant channel (std 0, divisor 1e-8) and NoNormalization
    ("identity_const", (2, 2, 9, 11), "float32", [4.0, 1.0, 1.0], [0, 2, 1], [1.0, 1.0],
     ["ZScoreNormalization", "NoNormalization"], [False, False]),
    # a channel above numpy's 8192-element buffer, mask under transpose, 3-D path
    ("volume_large_mask", (1, 4, 70, 90), "float32", [1.2, 1.0, 1.0], [0, 2, 1], [0.8, 0.8], ["ZScoreNormalization"],
     [True]),
]
INTENSITY = {"0": {"mean": 37.5, "std": 21.25, "percentile_00_5": -40.0, "percentile_99_5": 95.5},
             "1": {"mean": 0.0, "std": 1.0, "percentile_00_5": -1.0, "percentile_99_5": 1.0},
             "2": {"mean": 0.0, "std": 1.0, "percentile_00_5": -1.0, "percentile_99_5": 1.0}}


def case_input(case, seed):
    name, shape, dtype, *_ = case
    rng = np.random.default_rng(seed)
    if dtype == "uint8":
        return rng.integers(0, 256, size=shape).astype(np.uint8)
    x = (rng.standard_normal(shape) * 30 + 10).astype(np.float32)
    if name == "identity_const":
        x[0] = 7.25
    return x


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def _skimage_resize(image, output_shape, order=1, mode="edge", anti_aliasing=False, **kw):
    import scipy.ndimage as ndi
    assert order == 3 and mode == "edge" and not anti_aliasing and image.dtype == np.float64
    factors = np.divide(image.shape, output_shape)
    out = ndi.zoom(image, [1 / f for f in factors], order=order, mode="nearest", grid_mode=True)
    return np.clip(out, image.min(), image.max())


def reference_preprocessor():
    from oracle import ref_loader
    ref_loader.load_reference_module()
    _stub("skimage").__path__ = []
    _stub("skimage.transform", resize=_skimage_resize)
    for n in ("batchgenerators", "batchgenerators.augmentations", "batchgenerators.utilities"):
        sys.modules.setdefault(n, types.ModuleType(n)).__path__ = []
    _stub("batchgenerators.augmentations.utils",
          resize_segmentation=lambda seg, new_shape, order=3: np.zeros(new_shape, dtype=seg.dtype))
    fo = _stub("batchgenerators.utilities.file_and_folder_operations", join=os.path.join, load_json=None,
               maybe_mkdir_p=None, isfile=os.path.isfile, subfiles=None, List=list)
    fo.__all__ = ["join", "load_json", "maybe_mkdir_p", "isfile", "subfiles", "List"]
    for n in ("acvl_utils", "acvl_utils.cropping_and_padding"):
        sys.modules.setdefault(n, types.ModuleType(n)).__path__ = []

    def get_bbox_from_mask(mask):
        return [[int(np.nonzero(mask.any(axis=tuple(a for a in range(mask.ndim) if a != d)))[0][0]),
                 int(np.nonzero(mask.any(axis=tuple(a for a in range(mask.ndim) if a != d)))[0][-1]) + 1]
                for d in range(mask.ndim)]

    bb = sys.modules.get("acvl_utils.cropping_and_padding.bounding_boxes") or \
        _stub("acvl_utils.cropping_and_padding.bounding_boxes")
    bb.get_bbox_from_mask = get_bbox_from_mask
    bb.crop_to_bbox = None
    bb.bounding_box_to_slice = lambda bbox: tuple(slice(*i) for i in bbox)
    norm = importlib.import_module("dinounet.preprocessing.normalization.default_normalization_schemes")
    _stub("dinounet.utilities.plans_handling").__path__ = []
    _stub("dinounet.utilities.plans_handling.plans_handler", PlansManager=object, ConfigurationManager=object)
    _stub("dinounet.utilities.dataset_name_id_conversion", maybe_convert_to_dataset_name=None)
    _stub("dinounet.utilities.find_class_by_name",
          recursive_find_python_class=lambda folder, name, current_module: getattr(norm, name))
    _stub("dinounet.utilities.utils", get_identifiers_from_splitted_dataset_folder=None,
          create_lists_from_splitted_dataset_folder=None, get_filenames_of_train_images_and_targets=None)
    pre = importlib.import_module("dinounet.preprocessing.preprocessors.default_preprocessor")
    res = importlib.import_module("dinounet.preprocessing.resampling.default_resampling")
    return pre.DefaultPreprocessor, res


def run_reference(case, data):
    from functools import partial
    DefaultPreprocessor, res = reference_preprocessor()
    _, _, _, spacing, tf, cfg_spacing, schemes, use_mask = case
    kwargs = {"is_seg": False, "order": 3, "order_z": 0, "force_separate_z": None}
    cm = SimpleNamespace(spacing=list(cfg_spacing), normalization_schemes=list(schemes), use_mask_for_norm=list(use_mask),
                         resampling_fn_data=partial(res.resample_data_or_seg_to_shape, **kwargs),
                         resampling_fn_seg=partial(res.resample_data_or_seg_to_shape,
                                                   **{**kwargs, "is_seg": True, "order": 1}))
    pm = SimpleNamespace(transpose_forward=list(tf), foreground_intensity_properties_per_channel=INTENSITY)
    props = {"spacing": list(spacing)}
    out, seg = DefaultPreprocessor(verbose=False).run_case_npy(data.astype(np.float32), None, props, pm, cm, {})
    return out, seg, props


def main():
    import scipy
    arrays = {"versions": np.array([f"numpy {np.__version__}", f"scipy {scipy.__version__}"])}
    for seed, case in enumerate(CASES):
        name = case[0]
        data = case_input(case, seed)
        out, seg, props = run_reference(case, data)
        assert out.dtype == np.float32 and seg.dtype == np.int8 and not seg.any(), (out.dtype, seg.dtype)
        arrays[f"{name}_input"] = data
        arrays[f"{name}_output"] = out
        arrays[f"{name}_seg_shape"] = np.array(seg.shape)
        arrays[f"{name}_shape_before_cropping"] = np.array(props["shape_before_cropping"])
        arrays[f"{name}_bbox"] = np.array(props["bbox_used_for_cropping"])
        arrays[f"{name}_shape_after"] = np.array(props["shape_after_cropping_and_before_resampling"])
        print(name, data.shape, "->", out.shape)
    np.savez_compressed(OUT, **arrays)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
