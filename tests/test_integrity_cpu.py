"""-m "not gpu": the dataset integrity check's host side.  The numpy / pandas restatement (oracle/integrity_oracle.py)
reproduces the reference's own verify_dataset_integrity (tests/golden/integrity_cases.npz, written by
oracle/make_golden_integrity.py); the host-only failures and the scope rejections are raised before the native library
is reached; the drop-ins keep the reference's signatures."""
import contextlib
import inspect
import io
import os

import numpy as np
import pytest

from dinounet_b200 import fingerprint as F
from dinounet_b200 import integrity as I
from dinounet_b200 import preprocess as PP
from oracle import integrity_oracle as IO
from oracle import make_golden_integrity as MI

REF = np.load(os.path.join(os.path.dirname(__file__), "golden", "integrity_cases.npz"))
NAMES = [d[0] for d in MI.DATASETS]
HOST_FAILURES = [n for n in NAMES if str(REF[f"{n}_exc_type"]) in ("AssertionError", "FileNotFoundError")]


def golden(name: str, raw: str, key: str) -> str:
    return str(REF[f"{name}_{key}"]).replace(MI.RAW_TOKEN, raw)


@pytest.fixture
def raw(tmp_path, monkeypatch):
    """Every golden dataset under tmp_path/raw, with the module seams pointed at the oracle's restatements."""
    arrays = {k: REF[k] for k in REF.files}
    raw = str(tmp_path / "raw")
    for ds in MI.DATASETS:
        MI.write_dataset(raw, ds, arrays)
    monkeypatch.setattr(PP, "_dataset_name", lambda x: x)
    monkeypatch.setattr(PP, "_raw_and_preprocessed", lambda: (raw, str(tmp_path / "preprocessed")))
    monkeypatch.setattr(PP, "_get_filenames_of_train_images_and_targets", IO.get_filenames_of_train_images_and_targets)
    monkeypatch.setattr(F, "_determine_reader_writer", lambda dj, f: MI.NpyGeoReader)
    monkeypatch.setattr(I, "_label_manager", IO.LabelManager)
    return raw


@pytest.mark.parametrize("name", NAMES)
def test_oracle_equals_reference(name, raw):
    text, exc = IO.verify(os.path.join(raw, name), MI.NpyGeoReader)
    assert text == golden(name, raw, "stdout")
    assert ("" if exc is None else type(exc).__name__) == str(REF[f"{name}_exc_type"])
    assert ("" if exc is None else str(exc)) == golden(name, raw, "exc_msg")


class _Recorder:
    """A stand-in for the native library that records every entry point asked for."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        self.calls.append(name)
        raise AssertionError(f"{name} was reached")


def _no_native(monkeypatch):
    rec = _Recorder()
    monkeypatch.setattr(I.L, "load", lambda: rec)
    monkeypatch.setattr(F.L, "load", lambda: rec)
    return rec


def _run(fn, *args):
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        try:
            fn(*args)
        except Exception as e:   # noqa: BLE001 - compared below
            return out.getvalue(), e
    return out.getvalue(), None


@pytest.mark.parametrize("name", HOST_FAILURES)
def test_host_failures_issue_no_launch(name, raw, monkeypatch):
    rec = _no_native(monkeypatch)
    text, exc = _run(I.verify_dataset_integrity, os.path.join(raw, name), 2)
    assert text == "" and type(exc).__name__ == str(REF[f"{name}_exc_type"])
    assert str(exc) == golden(name, raw, "exc_msg")
    text, exc2 = _run(I.extract_fingerprint_dataset, name, F.DeviceFingerprintExtractor, 2, True, True, True)
    assert text == name + "\n" and type(exc2) is type(exc) and str(exc2) == str(exc)
    assert rec.calls == []


def test_seg_dtype_rejected_before_any_launch(raw, monkeypatch):
    rec = _no_native(monkeypatch)
    name = "Dataset911_Clean"
    label = os.path.join(raw, name, "labelsTr", "c0.npy")
    np.save(label, np.load(label).astype(np.int64))
    with pytest.raises(NotImplementedError, match="int64"):
        I.verify_dataset_integrity(os.path.join(raw, name), 2)
    assert rec.calls == []


def test_too_many_voxels_rejected_before_any_launch(raw, monkeypatch):
    rec = _no_native(monkeypatch)

    class Huge(MI.NpyGeoReader):   # 2^31 voxels as zero-stride views: nothing is allocated
        def read_images(self, files):
            return np.broadcast_to(np.float32(0), (2, 2048, 1024, 1024)), {"spacing": [1.0, 1.0, 1.0]}

        def read_seg(self, f):
            return np.broadcast_to(np.uint8(0), (1, 2048, 1024, 1024)), {"spacing": [1.0, 1.0, 1.0]}

    monkeypatch.setattr(F, "_determine_reader_writer", lambda dj, f: Huge)
    with pytest.raises(NotImplementedError, match="2\\^31"):
        I.verify_dataset_integrity(os.path.join(raw, "Dataset911_Clean"), 2)
    assert rec.calls == []


def test_signatures_match_the_reference():
    def params(fn):
        return [(p.name, p.default) for p in inspect.signature(fn).parameters.values()]

    assert params(I.verify_dataset_integrity) == [("folder", inspect.Parameter.empty), ("num_processes", 8)]
    n = I.DEFAULT_NUM_PROCESSES
    assert params(I.extract_fingerprint_dataset) == [
        ("dataset_id", inspect.Parameter.empty), ("fingerprint_extractor_class", F.DeviceFingerprintExtractor),
        ("num_processes", n), ("check_dataset_integrity", False), ("clean", True), ("verbose", True)]
    assert params(I.extract_fingerprints) == [
        ("dataset_ids", inspect.Parameter.empty), ("fingerprint_extractor_class_name", "DatasetFingerprintExtractor"),
        ("num_processes", n), ("check_dataset_integrity", False), ("clean", True), ("verbose", True)]
    assert I._find_extractor_class("DeviceFingerprintExtractor") is F.DeviceFingerprintExtractor
