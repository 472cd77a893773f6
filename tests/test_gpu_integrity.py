"""-m gpu: the dataset integrity check on the device against the reference's own verify_dataset_integrity and
extract_fingerprint_dataset (tests/golden/integrity_cases.npz): the stdout and the exception of every dataset, the
fused route's fingerprint JSON byte for byte (and none for a failing dataset); the scan kernel against numpy for every
seg dtype; and the failing path's label list against np.sort(pd.unique(...))."""
import contextlib
import io
import json
import os

import numpy as np
import pandas as pd
import pytest
import torch

from dinounet_b200 import fingerprint as F
from dinounet_b200 import integrity as I
from dinounet_b200 import lib as L
from dinounet_b200 import preprocess as PP
from oracle import integrity_oracle as IO
from oracle import make_golden_integrity as MI
from tests.gpu_helpers import stream

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
REF = np.load(os.path.join(os.path.dirname(__file__), "golden", "integrity_cases.npz"))
NAMES = [d[0] for d in MI.DATASETS]
PASSING = [n for n in NAMES if str(REF[f"{n}_exc_type"]) == ""]
SEG_DTYPES = [np.uint8, np.int8, np.int16, np.uint16, np.int32, np.float32]


def golden(name: str, raw: str, key: str) -> str:
    return str(REF[f"{name}_{key}"]).replace(MI.RAW_TOKEN, raw)


@pytest.fixture
def dirs(tmp_path, monkeypatch):
    arrays = {k: REF[k] for k in REF.files}
    raw, pre = str(tmp_path / "raw"), str(tmp_path / "preprocessed")
    for ds in MI.DATASETS:
        MI.write_dataset(raw, ds, arrays)
    monkeypatch.setattr(PP, "_dataset_name", lambda x: x)
    monkeypatch.setattr(PP, "_raw_and_preprocessed", lambda: (raw, pre))
    monkeypatch.setattr(PP, "_get_filenames_of_train_images_and_targets", IO.get_filenames_of_train_images_and_targets)
    monkeypatch.setattr(F, "_determine_reader_writer", lambda dj, f: MI.NpyGeoReader)
    monkeypatch.setattr(I, "_label_manager", IO.LabelManager)
    return raw, pre


def _run(fn, *args):
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        try:
            ret = fn(*args)
        except Exception as e:   # noqa: BLE001 - compared below
            return out.getvalue(), e, None
    return out.getvalue(), None, ret


def _check_exception(name, raw, exc):
    assert ("" if exc is None else type(exc).__name__) == str(REF[f"{name}_exc_type"]), (name, exc)
    assert ("" if exc is None else str(exc)) == golden(name, raw, "exc_msg")


@pytest.mark.parametrize("name", NAMES)
def test_verify_equals_reference(name, dirs):
    raw, _ = dirs
    text, exc, ret = _run(I.verify_dataset_integrity, os.path.join(raw, name), 3)
    assert text == golden(name, raw, "stdout") and ret is None
    _check_exception(name, raw, exc)


@pytest.mark.parametrize("name", NAMES)
def test_fused_route_equals_reference(name, dirs):
    raw, pre = dirs
    text, exc, fp = _run(I.extract_fingerprint_dataset, name, F.DeviceFingerprintExtractor, 2, True, True, True)
    assert text == golden(name, raw, "fused_stdout")
    _check_exception(name, raw, exc)
    stored = os.path.join(pre, name, "dataset_fingerprint.json")
    if name not in PASSING:
        assert not os.path.isfile(stored)
        return
    with open(stored) as f:
        assert f.read() == str(REF[f"{name}_json"])
    assert json.dumps(fp, sort_keys=True, indent=4) == str(REF[f"{name}_json"])
    # clean=False with the stored fingerprint: the check still runs, then the file is loaded
    text, exc, again = _run(I.extract_fingerprint_dataset, name, F.DeviceFingerprintExtractor, 2, True, False, True)
    assert exc is None and text == golden(name, raw, "fused_stdout")
    assert json.dumps(again, sort_keys=True, indent=4) == str(REF[f"{name}_json"])


@pytest.mark.parametrize("name", PASSING)
def test_check_off_is_the_extractor(name, dirs):
    raw, pre = dirs
    text, exc, fp = _run(I.extract_fingerprint_dataset, name, F.DeviceFingerprintExtractor, 2, False, True, True)
    assert exc is None and text == name + "\n"
    with open(os.path.join(pre, name, "dataset_fingerprint.json")) as f:
        assert f.read() == str(REF[f"{name}_json"])


def test_fused_route_raises_fingerprint_errors_after_the_check(dirs):
    """+-inf passes the check (its banner is printed) and is then the fingerprint's NotImplementedError."""
    raw, pre = dirs
    name = "Dataset911_Clean"
    f = os.path.join(raw, name, "imagesTr", "c1_0001.npy")
    x = np.load(f)
    x[0, 1, 2] = np.inf
    np.save(f, x)
    text, exc, _ = _run(I.extract_fingerprint_dataset, name, F.DeviceFingerprintExtractor, 2, True, True, True)
    assert text == golden(name, raw, "fused_stdout") and isinstance(exc, NotImplementedError) and "inf" in str(exc)
    assert not os.path.isfile(os.path.join(pre, name, "dataset_fingerprint.json"))


def test_fused_route_scope_rejection_issues_no_launch(dirs):
    raw, _ = dirs
    name = "Dataset911_Clean"
    label = os.path.join(raw, name, "labelsTr", "c0.npy")
    np.save(label, np.load(label).astype(np.int64))
    before = int(L.load().b2u_launch_count())
    with pytest.raises(NotImplementedError, match="int64"):
        I.extract_fingerprint_dataset(name, F.DeviceFingerprintExtractor, 2, True, True, True)
    assert int(L.load().b2u_launch_count()) == before


# ---- the scan kernel ---------------------------------------------------------------------------------------------


def _scan(img_d, seg_d, code, lo, hi):
    out = torch.zeros(2, dtype=torch.int64, device=DEV)
    L.check(L.load().b2u_vi_scan(img_d.data_ptr() if img_d is not None else None,
                                 img_d.numel() if img_d is not None else 0, seg_d.data_ptr(), code, seg_d.numel(),
                                 lo, hi, out.data_ptr(), stream()), "b2u_vi_scan")
    r = out.cpu().numpy()
    return int(r[0]), int(r[1]) & 0xffffffff


def _on_device(seg: np.ndarray, offset: int):
    """seg as a device tensor starting `offset` elements into a larger buffer (int16 bits for uint16)."""
    s = seg.view(np.int16) if seg.dtype == np.uint16 else seg
    buf = torch.empty(s.size + offset, dtype=getattr(torch, s.dtype.name), device=DEV)
    view = buf[offset:]
    view.copy_(torch.from_numpy(np.ascontiguousarray(s).reshape(-1)))
    return view


def _random_seg(dtype, n, rng):
    info = np.iinfo(dtype) if dtype != np.float32 else None
    if info is None:
        x = rng.integers(-3, 8, n).astype(np.float32)
        x[rng.random(n) < 0.01] = 1.5
        x[rng.random(n) < 0.01] = -0.0
        if n > 3:
            x[rng.integers(0, n, 2)] = np.nan
        return x
    x = rng.integers(0, 4, n).astype(np.int64)
    bad = rng.random(n) < 0.002
    x[bad] = rng.integers(info.min, info.max, int(bad.sum()), endpoint=True)
    return x.astype(dtype)


def _want(seg, lo, hi):
    x = seg.astype(np.float64)
    offenders = int((~np.isin(x, np.arange(lo, hi + 1))).sum())
    return offenders, bool(np.isnan(x).any())


@pytest.mark.parametrize("dtype", SEG_DTYPES, ids=lambda d: np.dtype(d).name)
def test_scan_equals_numpy(dtype):
    rng = np.random.default_rng(np.dtype(dtype).num)
    code = PP.SEG_DTYPE_CODES[np.dtype(dtype)]
    for n in (1, 2, 3, 7, 15, 16, 17, 31, 33, 255, 1000, 4099, 100_003):
        for offset in (0, 1, 3):
            seg = _random_seg(dtype, n, rng)
            img = rng.standard_normal(n * 2 + offset).astype(np.float32)
            if n % 3 == 0:
                img[rng.integers(0, img.size)] = np.nan
            if n % 5 == 0:
                img[rng.integers(0, img.size)] = -np.inf
            img_d = torch.from_numpy(img).to(DEV)[offset:]
            for lo, hi in ((0, 3), (0, 0), (-1, 2), (1, 300), (-100000, 100000)):
                got, flags = _scan(img_d, _on_device(seg, offset), code, lo, hi)
                want, seg_nan = _want(seg, lo, hi)
                assert got == want, (n, offset, lo, hi)
                assert bool(flags & I.SEG_NAN) == seg_nan
                assert bool(flags & I.IMAGE_NAN) == bool(np.isnan(img[offset:]).any())
                assert bool(flags & I.IMAGE_INF) == bool(np.isinf(img[offset:]).any())


@pytest.mark.parametrize("dtype", SEG_DTYPES, ids=lambda d: np.dtype(d).name)
def test_scan_large_volume_and_repeat(dtype):
    rng = np.random.default_rng(5)
    shape = (200, 512, 512)
    seg = rng.integers(0, 4, shape, dtype=np.int32).astype(dtype)
    flat = seg.reshape(-1)
    idx = rng.integers(0, flat.size, 37)
    flat[idx] = 5
    if dtype == np.float32:
        flat[idx[:3]] = np.nan
    code = PP.SEG_DTYPE_CODES[np.dtype(dtype)]
    seg_d = _on_device(seg, 0)
    img_d = torch.zeros(seg.size, dtype=torch.float32, device=DEV)
    want = (int((~np.isin(flat, np.arange(0, 4))).sum()), dtype == np.float32)
    results = {_scan(img_d, seg_d, code, 0, 3) for _ in range(5)}
    assert len(results) == 1
    got, flags = results.pop()
    assert (got, bool(flags & I.SEG_NAN)) == want and not flags & (I.IMAGE_NAN | I.IMAGE_INF)
    assert _scan(None, seg_d, code, 0, 5)[0] == (3 if dtype == np.float32 else 0)


@pytest.mark.parametrize("dtype", SEG_DTYPES, ids=lambda d: np.dtype(d).name)
def test_found_labels_equal_pandas(dtype):
    rng = np.random.default_rng(9)
    seg = _random_seg(dtype, 5000, rng)
    cases = [seg]
    if dtype == np.float32:
        z = np.array([3.0, -0.0, 1.5, 0.0, np.nan, np.nan, 1.0], np.float32)
        cases += [z, z[[0, 3, 1, 4]], np.array([np.nan, np.nan], np.float32)]
    for s in cases:
        code = PP.SEG_DTYPE_CODES[np.dtype(dtype)]
        d = _on_device(s, 0)
        d = d.view(10, -1) if s.size % 10 == 0 else d   # a case's seg arrives as [X, Y, Z]
        got = I.found_labels(d, code, s.dtype, bool(np.isnan(s.astype(np.float64)).any()))
        want = np.sort(pd.unique(s.ravel()))
        assert got.dtype == want.dtype and "%s" % got == "%s" % want
        assert np.array_equal(got, want, equal_nan=True) and np.array_equal(np.signbit(got), np.signbit(want))
