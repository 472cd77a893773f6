"""Writes tests/golden/dataloader_cases.npz: batches of the reference's own `nnUNetDataLoader2D.generate_train_batch`
(data_loader_2d.py:7-91, base_data_loader.py) with `np.random.seed(seed)`, over seeded cases saved in the reference's
format (`<key>.npz` with data and seg, `<key>.pkl` with the properties) and read by the reference's `nnUNetDataset`.

The inputs are not stored: `oracle.dataloader_oracle.ct_like_case` regenerates them from the seeds below, and the file
keeps a checksum of every case so that a change in the generator is caught.

Stand-ins for what is not installed here:
* batchgenerators 0.25's `DataLoader` base: its constructor's fields and, for `infinite=True`, `get_indices`:

      return np.random.choice(self.indices, self.batch_size, replace=True, p=self.sampling_probabilities)

  That restatement is batchgenerators' code as read from its source; no test here checks it against the library, which
  is not installed.  `batchgenerators.utilities.file_and_folder_operations` gets the five helpers the dataset imports.
* `blosc2`: the `Filter` / `Codec` attributes read when nnunet_dataset.py defines its classes (no case uses blosc2).
* `dinounet.utilities.label_handling.label_handling`: only the `LabelManager` name of an annotation; the loader reads
  `all_labels` and `has_ignore_label`, given here by a namespace.

    python oracle/make_golden_dataloader.py
"""
import importlib
import os
import pickle
import sys
import tempfile
import types
from types import SimpleNamespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import dataloader_oracle as DO  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "dataloader_cases.npz")

# name: C, case shapes [(Z, X, Y)], labels, ignore label, regions, seg dtype, empty case indices, patch, final patch,
#       B, oversample, seed, batches, val (regions / label-map target of the validation transforms)
CASES = {
    "labels_b2": (1, [(3, 30, 44), (2, 52, 36), (4, 40, 40)], [1, 2], None, None, "int8", [], (48, 40), (40, 32),
                  2, 0.33, 0, 3, False),
    "ignore_b3": (1, [(3, 34, 50), (2, 56, 30), (3, 40, 38)], [1, 2], 3, None, "int8", [], (40, 44), (32, 36),
                  3, 0.33, 1, 3, False),
    "regions_b5": (1, [(3, 40, 44), (2, 30, 50), (4, 36, 36)], [1, 2, 3], 4, [(1, 2, 3), (2, 3), (3,)], "int8", [],
                   (32, 32), (32, 32), 5, 0.33, 2, 2, True),
    "round_b5": (1, [(2, 28, 30), (3, 44, 40), (2, 36, 52)], [1, 2], None, None, "int8", [], (40, 40), (32, 32),
                 5, 0.5, 3, 3, False),
    "empty_nonsquare": (1, [(3, 30, 60), (2, 26, 40), (3, 44, 70)], [1], None, None, "int8", [1], (24, 56), (20, 48),
                        3, 0.33, 4, 4, False),
    "c2_int16": (2, [(2, 36, 36), (3, 30, 42)], [1, 200], None, None, "int16", [], (44, 36), (36, 28),
                 3, 0.33, 5, 3, False),
    "val_labels": (1, [(3, 40, 44), (2, 24, 30), (3, 36, 36)], [1, 2], None, None, "int8", [], (32, 32), (32, 32),
                   2, 0.33, 6, 3, True),
}


def label_manager(case):
    _, _, labels, ignore, *_ = case
    return SimpleNamespace(all_labels=[0] + list(labels), has_ignore_label=ignore is not None)


def case_arrays(name):
    """{key: (data, seg, properties)} of a golden case, regenerated from its seeds."""
    C, shapes, labels, ignore, regions, dtype, empty, *_, seed, _, _ = CASES[name]
    out = {}
    for i, (Z, X, Y) in enumerate(shapes):
        out[f"{name}_{i:02d}"] = DO.ct_like_case(C, Z, X, Y, labels, 1000 * seed + i, getattr(np, dtype),
                                                 empty=i in empty, ignore_label=ignore, regions=regions)
    return out


def checksum(cases):
    return np.array([float(np.float64(d.astype(np.float64).sum())) + float(s.astype(np.int64).sum())
                     for d, s, _ in cases.values()])


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


class _DataLoader:
    """batchgenerators 0.25 `DataLoader`: the constructor's fields and the infinite `get_indices`."""

    def __init__(self, data, batch_size, num_threads_in_multithreaded=1, seed_for_shuffle=None,
                 return_incomplete=False, shuffle=True, infinite=False, sampling_probabilities=None):
        self._data = data
        self.batch_size = batch_size
        self.thread_id = 0
        self.number_of_threads_in_multithreaded = num_threads_in_multithreaded
        self.rs = np.random.RandomState(seed_for_shuffle)
        self.return_incomplete = return_incomplete
        self.shuffle = shuffle
        self.infinite = infinite
        self.sampling_probabilities = sampling_probabilities
        self.indices = None

    def get_indices(self):
        assert self.infinite
        return np.random.choice(self.indices, self.batch_size, replace=True, p=self.sampling_probabilities)


def reference():
    """(nnUNetDataLoader2D, nnUNetDataset) of the reference, with the stand-ins above."""
    from oracle import ref_loader
    ref_loader.load_reference_module()
    for n in ("batchgenerators", "batchgenerators.dataloading", "batchgenerators.utilities"):
        sys.modules.setdefault(n, types.ModuleType(n)).__path__ = []
    _stub("batchgenerators.dataloading.data_loader", DataLoader=_DataLoader)

    def load_pickle(f, mode="rb"):
        with open(f, mode) as fh:
            return pickle.load(fh)
    fo = sys.modules.get("batchgenerators.utilities.file_and_folder_operations") or \
        _stub("batchgenerators.utilities.file_and_folder_operations")
    for k, v in dict(join=os.path.join, load_pickle=load_pickle, isfile=os.path.isfile, write_pickle=None,
                     subfiles=None, List=list).items():
        setattr(fo, k, v)
    fo.__all__ = sorted(set(getattr(fo, "__all__", [])) | {"join", "load_pickle", "isfile", "write_pickle",
                                                              "subfiles", "List"})
    _stub("blosc2", Filter=SimpleNamespace(SHUFFLE=1), Codec=SimpleNamespace(ZSTD=5), set_nthreads=None)
    ref = os.path.join(ref_loader.REF_ROOT, "dinounet")
    if "dinounet.utilities" not in sys.modules:   # a bare package: its modules import on their own
        _stub("dinounet.utilities").__path__ = [os.path.join(ref, "utilities")]
    if "dinounet.utilities.label_handling" not in sys.modules:
        _stub("dinounet.utilities.label_handling").__path__ = []
    _stub("dinounet.utilities.label_handling.label_handling", LabelManager=object)
    dl = sys.modules.get("dinounet.training.dataloading")
    if dl is None or not getattr(dl, "__path__", None):
        _stub("dinounet.training.dataloading").__path__ = [os.path.join(ref, "training", "dataloading")]
    d2 = importlib.import_module("dinounet.training.dataloading.data_loader_2d")
    ds = importlib.import_module("dinounet.training.dataloading.nnunet_dataset")
    return d2.nnUNetDataLoader2D, ds.nnUNetDataset


def run_reference(name, folder):
    Loader, Dataset = reference()
    case = CASES[name]
    patch, final, B, osp, seed, nb = case[7:13]
    cases = case_arrays(name)
    for k, (d, s, p) in cases.items():
        np.savez(os.path.join(folder, k + ".npz"), data=d, seg=s)
        with open(os.path.join(folder, k + ".pkl"), "wb") as f:
            pickle.dump(p, f)
    ds = Dataset(folder, sorted(cases), num_images_properties_loading_threshold=0)
    np.random.seed(seed)
    dl = Loader(ds, B, list(patch), list(final), label_manager(case), oversample_foreground_percent=osp,
                sampling_probabilities=None, pad_sides=None)
    return cases, [dl.generate_train_batch() for _ in range(nb)]


def main():
    arrays = {"versions": np.array([f"numpy {np.__version__}"])}
    for name in CASES:
        with tempfile.TemporaryDirectory() as tmp:
            cases, batches = run_reference(name, tmp)
        arrays[f"{name}_checksum"] = checksum(cases)
        for i, b in enumerate(batches):
            arrays[f"{name}_{i}_keys"] = np.asarray(b["keys"]).astype(str)
            arrays[f"{name}_{i}_data"] = b["data"]
            arrays[f"{name}_{i}_seg"] = b["seg"]
        print(name, [list(b["keys"]) for b in batches], batches[0]["data"].shape)
    np.savez_compressed(OUT, **arrays)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
