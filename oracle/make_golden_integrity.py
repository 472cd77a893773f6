"""Writes tests/golden/integrity_cases.npz: the reference's own `verify_dataset_integrity`
(experiment_planning/verify_dataset_integrity.py) and, for the datasets it accepts, its `DatasetFingerprintExtractor`
run as `extract_fingerprint_dataset` runs them (plan_and_preprocess_api.py:25-32: the name, the check, then
`run(overwrite_existing=clean)`), on the small seeded raw datasets of `DATASETS`.

Stored per dataset: the cases' arrays and spacings; the stdout of `verify_dataset_integrity` and of
`extract_fingerprint_dataset(check_dataset_integrity=True)`, the exception's type and message (with the raw folder
written as RAW_TOKEN), and for the accepted datasets the fingerprint JSON text.

Stand-ins only for what is not installed here, as oracle/make_golden_fingerprint.py has them: batchgenerators' file
helpers, the reader registry (`NpyGeoReader`: one `.npy` file per channel, the spacing and the optional nibabel / sitk
geometry from class tables), the dataset-name conversion, and a serial map for the spawn pool (its workers cannot
import the stand-ins).  `get_filenames_of_train_images_and_targets` and the LabelManager are the reference's own.

    python oracle/make_golden_integrity.py
"""
import contextlib
import importlib
import io
import json
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "integrity_cases.npz")
RAW_TOKEN = "<raw>"
CHANNELS = {"0": "CT", "1": "aux"}
LABELS = {"background": 0, "a": 1, "b": 2, "c": 3}

# A case: (key, (X, Y, Z), seg dtype, defect).  A dataset: (name, folder style, labels, cases, dataset.json edits).
# Defects: see case_arrays and write_dataset.
DATASETS = [
    ("Dataset911_Clean", "folder", LABELS, [
        ("c0", (3, 10, 12), "int16", None), ("c1", (2, 9, 14), "int8", None), ("c2", (4, 8, 8), "float32", None)], {}),
    ("Dataset912_RegionsIgnore", "dataset", {"background": 0, "liver": [1, 2], "tumor": 2, "ignore": 3}, [
        ("r0", (2, 11, 10), "int32", "ignore"), ("r1", (3, 9, 9), "int16", "ignore")], {"regions_class_order": [1, 2]}),
    ("Dataset913_UnexpectedU8", "folder", LABELS, [
        ("u0", (2, 8, 9), "uint8", None), ("u1", (2, 10, 7), "uint8", None), ("u2", (3, 6, 8), "uint8", "label7")],
     {}),
    ("Dataset914_NegativeI16", "folder", LABELS, [
        ("n0", (2, 8, 9), "int16", "negative"), ("n1", (2, 7, 7), "int16", "nan_image")], {}),
    ("Dataset915_FloatSeg", "folder", LABELS, [
        ("f0", (2, 9, 8), "float32", "float_nan"), ("f1", (2, 8, 8), "float32", "minus_zero")], {}),
    ("Dataset916_NaNImage", "folder", LABELS, [
        ("i0", (2, 8, 9), "int16", "affine"), ("i1", (2, 7, 10), "int16", "nan_image")], {}),
    ("Dataset917_Shape", "folder", LABELS, [
        ("s0", (2, 8, 9), "int16", "shape"), ("s1", (2, 7, 8), "int16", "origin")], {}),
    ("Dataset918_SpacingOut", "folder", LABELS, [
        ("p0", (2, 8, 9), "int16", "spacing_in"), ("p1", (2, 7, 8), "int16", "spacing_out")], {}),
    ("Dataset919_SpacingIn", "folder", LABELS, [
        ("q0", (2, 8, 9), "int16", "spacing_in"), ("q1", (3, 7, 8), "float32", None)], {}),
    ("Dataset920_Channels", "folder", LABELS, [
        ("h0", (2, 8, 9), "int16", "channels"), ("h1", (2, 7, 8), "int16", None)], {}),
    ("Dataset921_Geometry", "folder", LABELS, [
        ("g0", (2, 8, 9), "int16", "affine"), ("g1", (2, 7, 8), "int32", "origin"),
        ("g2", (3, 6, 7), "int8", "direction")], {}),
    ("Dataset922_MissingLabelFolder", "folder", LABELS, [
        ("m0", (2, 8, 9), "int16", None), ("m1", (2, 7, 8), "int16", "no_label")], {}),
    ("Dataset923_MissingLabelDataset", "dataset", LABELS, [
        ("d0", (2, 8, 9), "int16", "no_label"), ("d1", (2, 7, 8), "int16", None)], {}),
    ("Dataset924_NumTraining", "folder", LABELS, [
        ("t0", (2, 8, 9), "int16", None), ("t1", (2, 7, 8), "int16", None)], {"numTraining": 3}),
    ("Dataset925_NonConsecutive", "folder", {"background": 0, "a": 1, "b": 3}, [
        ("k0", (2, 8, 9), "int16", None)], {}),
    ("Dataset926_MissingKey", "folder", LABELS, [("y0", (2, 8, 9), "int16", None)], {"drop": "channel_names"}),
    ("Dataset927_LastBad", "folder", LABELS, [
        ("z0", (2, 8, 9), "int16", "origin"), ("z1", (2, 7, 8), "uint16", None), ("z2", (2, 9, 8), "int32", None),
        ("z3", (3, 6, 7), "uint16", "label7")], {}),
]
BASE_SPACING = [2.5, 0.75, 0.75]


def case_arrays(index: int, shape, dtype: str, defect):
    """(images fp32 [C, X, Y, Z], seg [X, Y, Z] of `dtype`, seg shape override or None): integer HU and labels 0..3
    (0..3 with 3 the ignore label for "ignore"), with the defect applied."""
    rng = np.random.default_rng(2000 + index)
    c = 3 if defect == "channels" else 2
    img = np.stack([rng.integers(-120, 161, size=shape) for _ in range(c)]).astype(np.float32)
    seg = rng.integers(0, 4 if defect == "ignore" else 3, size=shape).astype(np.float64)
    seg.reshape(-1)[0] = 0
    if defect == "label7":
        seg.reshape(-1)[-1] = 7
    elif defect == "negative":
        seg.reshape(-1)[5] = -1
    elif defect == "float_nan":
        seg.reshape(-1)[[3, 9]] = (1.5, np.nan)
        seg.reshape(-1)[11] = np.nan
    elif defect == "minus_zero":
        seg.reshape(-1)[seg.reshape(-1) == 0] = -0.0
    elif defect == "nan_image":
        img[1, 1, 2, 3] = np.nan
    elif defect == "shape":
        seg = seg[:, :-1]
    return img, seg.astype(dtype)


class NpyGeoReader:
    """One `.npy` file per channel; the spacing and the optional geometry properties come from the class tables,
    keyed by file."""
    SPACINGS = {}
    GEOMETRY = {}

    def read_images(self, image_fnames):
        images = np.stack([np.load(f) for f in image_fnames]).astype(np.float32)
        return images, {"spacing": list(self.SPACINGS[image_fnames[0]]), **self.GEOMETRY.get(image_fnames[0], {})}

    def read_seg(self, seg_fname):
        return np.load(seg_fname)[None], {"spacing": list(self.SPACINGS[seg_fname]), **self.GEOMETRY.get(seg_fname, {})}


def _geometry(defect, seg: bool):
    if defect == "affine":
        a = np.diag([2.5, 0.75, 0.75, 1.0])
        if seg:
            a[0, 3] = 0.5
        return {"nibabel_stuff": {"original_affine": a}}
    if defect in ("origin", "direction"):
        origin = (0.0, -10.0, 4.5) if seg and defect == "origin" else (0.0, -10.0, 4.0)
        direction = (1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0)
        if seg and defect == "direction":
            direction = (1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 1.0, 0.0)
        return {"sitk_stuff": {"origin": origin, "direction": direction, "spacing": tuple(BASE_SPACING)}}
    return {}


def dataset_arrays(dataset, first_index: int) -> dict:
    name, _, _, cases, _ = dataset
    arrays = {}
    for i, (key, shape, dtype, defect) in enumerate(cases):
        img, seg = case_arrays(first_index + i, shape, dtype, defect)
        arrays[f"{name}_{key}_images"] = img
        arrays[f"{name}_{key}_seg"] = seg
    return arrays


def write_dataset(raw: str, dataset, arrays: dict) -> str:
    """Writes the dataset under raw/<name>/ (imagesTr / labelsTr, or the `dataset` key of dataset.json), registers its
    files with NpyGeoReader, and returns its folder."""
    name, style, labels, cases, edits = dataset
    folder = os.path.join(raw, name)
    os.makedirs(os.path.join(folder, "imagesTr"), exist_ok=True)
    os.makedirs(os.path.join(folder, "labelsTr"), exist_ok=True)
    dj = {"channel_names": dict(CHANNELS), "labels": labels, "file_ending": ".npy", "numTraining": len(cases)}
    entries = {}
    for key, shape, dtype, defect in cases:
        images, seg = arrays[f"{name}_{key}_images"], arrays[f"{name}_{key}_seg"]
        files = [os.path.join(folder, "imagesTr", f"{key}_{c:04d}.npy") for c in range(images.shape[0])]
        for c, f in enumerate(files):
            np.save(f, images[c])
        label = os.path.join(folder, "labelsTr", f"{key}.npy")
        if defect != "no_label":
            np.save(label, seg)
        spacing = list(BASE_SPACING)
        seg_spacing = list(spacing)
        if defect == "spacing_out":
            seg_spacing[1] += 1e-5 * spacing[1] + 2e-6
        elif defect == "spacing_in":
            seg_spacing[1] += 0.5e-5 * spacing[1]
        for f in files:
            NpyGeoReader.SPACINGS[f] = spacing
            NpyGeoReader.GEOMETRY[f] = _geometry(defect, False)
        NpyGeoReader.SPACINGS[label] = seg_spacing
        NpyGeoReader.GEOMETRY[label] = _geometry(defect, True)
        entries[key] = {"images": [os.path.relpath(f, folder) for f in files], "label": os.path.relpath(label, folder)}
    if style == "dataset":
        dj["dataset"] = entries
    for k, v in edits.items():
        if k == "drop":
            del dj[v]
        else:
            dj[k] = v
    with open(os.path.join(folder, "dataset.json"), "w") as f:
        json.dump(dj, f)
    return folder


class _SerialPool:
    def __init__(self, n):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False

    def starmap(self, fn, args):
        return [fn(*a) for a in args]


def reference_modules(raw: str, preprocessed: str):
    """(the reference's verify_dataset_integrity module, its DatasetFingerprintExtractor) with the stand-ins above."""
    from oracle import make_golden_fingerprint as MF
    from oracle import make_golden_preprocess as MG
    MF.reference_extractor(raw, preprocessed, {})
    fo = sys.modules["batchgenerators.utilities.file_and_folder_operations"]

    def subfiles(folder, join=True, prefix=None, suffix=None, sort=True):
        res = [os.path.join(folder, i) if join else i for i in os.listdir(folder)
               if os.path.isfile(os.path.join(folder, i)) and (prefix is None or i.startswith(prefix))
               and (suffix is None or i.endswith(suffix))]
        return sorted(res) if sort else res

    fo.subfiles, fo.isdir = subfiles, os.path.isdir
    fo.__all__ = sorted(set(fo.__all__) | {"subfiles", "isdir", "save_json", "load_json", "maybe_mkdir_p"})
    MG._stub("dinounet.paths", nnUNet_raw=raw, nnUNet_preprocessed=preprocessed, nnUNet_results=None)
    sys.modules.pop("dinounet.utilities.utils", None)
    utils = importlib.import_module("dinounet.utilities.utils")
    MG._stub("dinounet.imageio.reader_writer_registry",
             determine_reader_writer_from_dataset_json=lambda dataset_json, example_file=None, *a, **k: NpyGeoReader)
    MG._stub("dinounet.imageio.base_reader_writer", BaseReaderWriter=object)
    lh = importlib.import_module("dinounet.utilities.label_handling.label_handling")
    vdi = importlib.import_module("dinounet.experiment_planning.verify_dataset_integrity")
    vdi.multiprocessing = types.SimpleNamespace(get_context=lambda kind: types.SimpleNamespace(Pool=_SerialPool))
    vdi.LabelManager = lh.LabelManager
    fe = sys.modules["dinounet.experiment_planning.dataset_fingerprint.fingerprint_extractor"]
    fe.nnUNet_raw, fe.nnUNet_preprocessed = raw, preprocessed
    fe.get_filenames_of_train_images_and_targets = utils.get_filenames_of_train_images_and_targets
    fe.determine_reader_writer_from_dataset_json = lambda dataset_json, example_file=None, *a, **k: NpyGeoReader
    return vdi, fe.DatasetFingerprintExtractor


def capture(fn, *args, **kwargs):
    """(stdout, exception or None) of fn(*args, **kwargs)."""
    out = io.StringIO()
    exc = None
    with contextlib.redirect_stdout(out):
        try:
            fn(*args, **kwargs)
        except Exception as e:   # noqa: BLE001 - the exception is the recorded result
            exc = e
    return out.getvalue(), exc


def main():
    arrays = {"versions": np.array([f"numpy {np.__version__}", f"pandas {__import__('pandas').__version__}"])}
    first = 0
    for ds in DATASETS:
        arrays.update(dataset_arrays(ds, first))
        first += len(ds[3])
    with tempfile.TemporaryDirectory() as tmp:
        raw, pre = os.path.join(tmp, "raw"), os.path.join(tmp, "preprocessed")
        for ds in DATASETS:
            write_dataset(raw, ds, arrays)
        vdi, Extractor = reference_modules(raw, pre)

        def extract_fingerprint_dataset(name, num_processes, clean):
            """plan_and_preprocess_api.py:25-32 with check_dataset_integrity=True."""
            print(name)
            vdi.verify_dataset_integrity(os.path.join(raw, name), num_processes)
            fpe = Extractor(name, num_processes, verbose=True)
            return fpe.run(overwrite_existing=clean)

        for name, *_ in DATASETS:
            text, exc = capture(vdi.verify_dataset_integrity, os.path.join(raw, name), 2)
            fused, exc2 = capture(extract_fingerprint_dataset, name, 2, True)
            assert type(exc) is type(exc2) and str(exc) == str(exc2), (exc, exc2)
            arrays[f"{name}_stdout"] = np.array(text.replace(raw, RAW_TOKEN))
            arrays[f"{name}_fused_stdout"] = np.array(fused.replace(raw, RAW_TOKEN))
            arrays[f"{name}_exc_type"] = np.array("" if exc is None else type(exc).__name__)
            arrays[f"{name}_exc_msg"] = np.array("" if exc is None else str(exc).replace(raw, RAW_TOKEN))
            fp = os.path.join(pre, name, "dataset_fingerprint.json")
            if exc is None:
                with open(fp) as f:
                    arrays[f"{name}_json"] = np.array(f.read())
            assert (exc is None) == os.path.isfile(fp), name
            print(name, type(exc).__name__ if exc else "ok", len(text))
    np.savez_compressed(OUT, **arrays)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
