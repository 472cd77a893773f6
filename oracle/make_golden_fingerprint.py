"""Writes tests/golden/fingerprint_cases.npz: the reference's own `DatasetFingerprintExtractor`
(experiment_planning/dataset_fingerprint/fingerprint_extractor.py) with its `crop_to_nonzero` (cropping.py) on two small
seeded datasets of `.npy` cases:
* DATASET_A: six cases, one per seg dtype, two channels of integer-valued "HU" data with heavy ties, negatives and
  zeros; one case without foreground (its `[]` promotes the concatenation, so every statistic is float64) and one with
  fewer foreground voxels than the small budget's per-case sample count;
* DATASET_B: four cases, all with foreground (float32 statistics).

Stored per dataset: the inputs and spacings; `run()`'s JSON text at the default budget of 10e7 samples; each case's
`collect_foreground_intensities` (num_samples 10000: the samples and the six statistics, NaN without foreground); the
dataset vectors at a budget of 1000 samples, element for element; the SHA-256 of each channel's vector at the default
budget (the bytes of the concatenation, in its dtype).

Stand-ins only for what is not installed here: batchgenerators' file helpers and `save_json` (json.dump with
sort_keys=True, indent=4, as batchgenerators writes it), acvl_utils' bounding-box helpers
(oracle/make_golden_preprocess), the reader registry (a `.npy` reader: one file per channel, spacing from SPACINGS),
the dataset-name conversion and `get_filenames_of_train_images_and_targets`, and an in-process stand-in for the spawn
pool.

numpy 2 refuses the reference's `seg[(seg == 0) & ~nonzero_mask] = -1` (cropping.py:46) on an unsigned seg with an
OverflowError, although the mask selects no voxel.  The reader therefore hands the reference the uint8 / uint16 cases'
labels as int16 / int32; the foreground `seg > 0` and so every output depends on the label values only.

    python oracle/make_golden_fingerprint.py
"""
import hashlib
import importlib
import json
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden_preprocess as MG  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "fingerprint_cases.npz")
SMALL_BUDGET = 1000
CASE_SAMPLES = 10000

# name, cases: (key, (X, Y, Z), seg dtype, spacing, foreground kind)
DATASET_A = ("Dataset901_FpPromoted", [
    ("a_u8", (3, 20, 24), "uint8", [2.5, 0.75, 0.75], "blob"),
    ("a_i8", (2, 17, 31), "int8", [3.0, 0.8, 0.8], "blob"),
    ("a_i16", (4, 15, 18), "int16", [2.5, 0.7, 0.7], "blob"),
    ("a_u16_empty", (2, 21, 16), "uint16", [2.5, 0.75, 0.75], "none"),
    ("a_i32_sparse", (3, 12, 14), "int32", [2.0, 0.9, 0.9], "sparse"),
    ("a_f32", (2, 25, 22), "float32", [2.5, 0.6, 0.6], "blob"),
])
DATASET_B = ("Dataset902_FpFloat32", [
    ("b_f32", (3, 19, 23), "float32", [1.5, 1.0, 1.0], "blob"),
    ("b_i16", (2, 30, 20), "int16", [1.5, 1.0, 1.0], "blob"),
    ("b_u8_sparse", (2, 11, 13), "uint8", [1.5, 1.1, 1.1], "sparse"),
    ("b_i32", (3, 16, 16), "int32", [1.5, 0.9, 0.9], "blob"),
])
DATASETS = (DATASET_A, DATASET_B)
CHANNELS = 2


def case_arrays(index: int, shape, dtype: str, kind: str):
    """(images fp32 [2, X, Y, Z], seg [1, X, Y, Z] of `dtype`): channel 0 integer HU in [-120, 160] (ties, zeros,
    negatives), channel 1 integers in [-3, 3] scaled by 0.5; labels 0..3."""
    rng = np.random.default_rng(1000 + index)
    img = np.stack([rng.integers(-120, 161, size=shape), rng.integers(-3, 4, size=shape) * 0.5]).astype(np.float32)
    seg = np.zeros(shape, np.int32)
    if kind == "blob":
        X, Y, Z = shape
        seg[:, Y // 4: 3 * Y // 4, Z // 5: 4 * Z // 5] = rng.integers(0, 4, size=(X, 3 * Y // 4 - Y // 4,
                                                                                4 * Z // 5 - Z // 5))
    elif kind == "sparse":   # 12 foreground voxels: fewer than the small budget's per-case samples
        flat = seg.reshape(-1)
        flat[rng.choice(flat.size, 12, replace=False)] = rng.integers(1, 4, size=12)
    return img, seg[None].astype(dtype)


class NpyReader:
    """One `.npy` file per channel; the spacing comes from SPACINGS[case file]."""
    SPACINGS = {}
    REFERENCE_VIEW = False   # hand the reference unsigned labels as the next wider signed dtype (see above)

    def read_images(self, image_fnames):
        images = np.stack([np.load(f) for f in image_fnames]).astype(np.float32)
        return images, {"spacing": list(self.SPACINGS[image_fnames[0]])}

    def read_seg(self, seg_fname):
        seg = np.load(seg_fname)[None]
        if self.REFERENCE_VIEW and seg.dtype in (np.uint8, np.uint16):
            seg = seg.astype(np.int16 if seg.dtype == np.uint8 else np.int32)
        return seg, {"spacing": list(self.SPACINGS[seg_fname])}


def write_dataset(raw: str, dataset, arrays: dict) -> dict:
    """Writes the dataset's `.npy` files under raw/<name>/ and returns the dataset dict of
    `get_filenames_of_train_images_and_targets`."""
    name, cases = dataset
    folder = os.path.join(raw, name)
    os.makedirs(folder, exist_ok=True)
    with open(os.path.join(folder, "dataset.json"), "w") as f:
        json.dump({"channel_names": {"0": "CT", "1": "aux"}, "labels": {"background": 0, "a": 1, "b": 2, "c": 3},
                   "file_ending": ".npy", "numTraining": len(cases)}, f)
    ds = {}
    for key, *_ in cases:
        images, seg = arrays[f"{name}_{key}_images"], arrays[f"{name}_{key}_seg"]
        files = []
        for c in range(images.shape[0]):
            files.append(os.path.join(folder, f"{key}_{c:04d}.npy"))
            np.save(files[-1], images[c])
        label = os.path.join(folder, f"{key}.npy")
        np.save(label, seg[0])
        for f in files + [label]:
            NpyReader.SPACINGS[f] = [float(v) for v in arrays[f"{name}_{key}_spacing"]]
        ds[key] = {"images": files, "label": label}
    return ds


def dataset_arrays(dataset, first_index: int) -> dict:
    name, cases = dataset
    arrays = {f"{name}_keys": np.array([c[0] for c in cases])}
    for i, (key, shape, dtype, spacing, kind) in enumerate(cases):
        img, seg = case_arrays(first_index + i, shape, dtype, kind)
        arrays[f"{name}_{key}_images"] = img
        arrays[f"{name}_{key}_seg"] = seg
        arrays[f"{name}_{key}_spacing"] = np.array(spacing, dtype=np.float64)
    return arrays


class _InlinePool:
    """multiprocessing.get_context("spawn").Pool(n) run in this process."""

    class _Result:
        def __init__(self, value):
            self.value = value

        def ready(self):
            return True

        def get(self):
            return self.value

    def __init__(self, n):
        self._pool = []

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False

    def starmap_async(self, fn, args):
        return self._Result([fn(*a) for a in args])


def reference_extractor(raw: str, preprocessed: str, datasets: dict):
    """The reference's fingerprint_extractor module with the stand-ins above."""
    MG.reference_preprocessor()   # the reference on sys.path, batchgenerators / acvl_utils stand-ins
    fo = sys.modules["batchgenerators.utilities.file_and_folder_operations"]

    def save_json(obj, file, indent=4, sort_keys=True):
        with open(file, "w") as f:
            json.dump(obj, f, sort_keys=sort_keys, indent=indent)

    def load_json(file):
        with open(file) as f:
            return json.load(f)

    fo.save_json, fo.load_json = save_json, load_json
    fo.maybe_mkdir_p = lambda d: os.makedirs(d, exist_ok=True)
    sys.modules["dinounet.utilities.dataset_name_id_conversion"].maybe_convert_to_dataset_name = lambda x: x
    sys.modules["dinounet.utilities.utils"].get_filenames_of_train_images_and_targets = \
        lambda folder, dataset_json=None: datasets[os.path.basename(folder)]
    MG._stub("dinounet.imageio.reader_writer_registry",
             determine_reader_writer_from_dataset_json=lambda dataset_json, example_file=None, *a, **k: NpyReader)
    fe = importlib.import_module("dinounet.experiment_planning.dataset_fingerprint.fingerprint_extractor")
    fe.nnUNet_raw, fe.nnUNet_preprocessed = raw, preprocessed
    fe.multiprocessing = types.SimpleNamespace(get_context=lambda kind: types.SimpleNamespace(Pool=_InlinePool))
    return fe.DatasetFingerprintExtractor


def vector_hash(parts) -> str:
    """SHA-256 of np.concatenate(parts)'s bytes, without building it."""
    promoted = any(isinstance(p, list) for p in parts)
    h = hashlib.sha256()
    for p in parts:
        if not isinstance(p, list):
            h.update(np.ascontiguousarray(p, dtype=np.float64 if promoted else p.dtype).tobytes())
    return h.hexdigest()


def main():
    import scipy
    arrays = {"versions": np.array([f"numpy {np.__version__}", f"scipy {scipy.__version__}"])}
    first = 0
    for ds in DATASETS:
        arrays.update(dataset_arrays(ds, first))
        first += len(ds[1])
    NpyReader.REFERENCE_VIEW = True
    with tempfile.TemporaryDirectory() as tmp:
        raw, pre = os.path.join(tmp, "raw"), os.path.join(tmp, "preprocessed")
        datasets = {ds[0]: write_dataset(raw, ds, arrays) for ds in DATASETS}
        Extractor = reference_extractor(raw, pre, datasets)
        for name, cases in DATASETS:
            ext = Extractor(name, num_processes=2)
            fp = ext.run(overwrite_existing=True)
            with open(os.path.join(pre, name, "dataset_fingerprint.json")) as f:
                arrays[f"{name}_json"] = np.array(f.read())
            print(name, json.dumps(fp["foreground_intensity_properties_per_channel"])[:200])
            for budget, tag in ((SMALL_BUDGET, "small"), (10e7, "default")):
                per_case = [Extractor.analyze_case(ext.dataset[k]["images"], ext.dataset[k]["label"], NpyReader,
                                                   int(budget // len(cases)))[2] for k, *_ in cases]
                for c in range(CHANNELS):
                    parts = [r[c] for r in per_case]
                    if tag == "small":
                        arrays[f"{name}_samples_small_{c}"] = np.concatenate(parts)
                    else:
                        arrays[f"{name}_sha256_{c}"] = np.array(vector_hash(parts))
            for key, *_ in cases:
                rw = NpyReader()
                seg, _ = rw.read_seg(ext.dataset[key]["label"])
                images, _ = rw.read_images(ext.dataset[key]["images"])
                samples, stats = Extractor.collect_foreground_intensities(seg, images, num_samples=CASE_SAMPLES)
                for c in range(CHANNELS):
                    arrays[f"{name}_{key}_case_samples_{c}"] = np.asarray(samples[c], dtype=np.float32)
                    arrays[f"{name}_{key}_case_stats_{c}"] = np.array(
                        [stats[c][k] for k in STAT_KEYS], dtype=np.float32)
    np.savez_compressed(OUT, **arrays)
    print(OUT, os.path.getsize(OUT), "bytes")


STAT_KEYS = ("mean", "median", "min", "max", "percentile_99_5", "percentile_00_5")

if __name__ == "__main__":
    main()
