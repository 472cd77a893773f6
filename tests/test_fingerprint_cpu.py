"""-m "not gpu": the fingerprint's host side.  The numpy restatement of the device algorithm
(oracle/fingerprint_oracle.py) reproduces the reference's own DatasetFingerprintExtractor
(tests/golden/fingerprint_cases.npz, written by oracle/make_golden_fingerprint.py); the host finishing helpers equal
numpy's median / percentile / mean / std; and every rejection is raised before anything touches a device."""
import hashlib
import os

import numpy as np
import pytest
import torch

from dinounet_b200 import fingerprint as F
from oracle import fingerprint_oracle as FO
from oracle import make_golden_fingerprint as MF

REF = np.load(os.path.join(os.path.dirname(__file__), "golden", "fingerprint_cases.npz"))
DATASET_IDS = [d[0] for d in MF.DATASETS]


def _cases(dataset):
    name, cases = dataset
    return [(REF[f"{name}_{k}_seg"], REF[f"{name}_{k}_images"]) for k, *_ in cases]


def _spacings(dataset):
    name, cases = dataset
    return [[float(v) for v in REF[f"{name}_{k}_spacing"]] for k, *_ in cases]


@pytest.mark.parametrize("dataset", MF.DATASETS, ids=DATASET_IDS)
def test_oracle_json_equals_reference(dataset):
    fp = FO.fingerprint(_cases(dataset), _spacings(dataset), MF.CHANNELS)
    assert FO.fingerprint_json(fp) == str(REF[f"{dataset[0]}_json"])


@pytest.mark.parametrize("dataset", MF.DATASETS, ids=DATASET_IDS)
def test_oracle_sample_vectors_equal_reference(dataset):
    name, cases = dataset
    small = FO.dataset_vectors(_cases(dataset), int(MF.SMALL_BUDGET // len(cases)))
    full = FO.dataset_vectors(_cases(dataset), int(10e7 // len(cases)))
    for c in range(MF.CHANNELS):
        want = REF[f"{name}_samples_small_{c}"]
        assert small[c].dtype == want.dtype and np.array_equal(small[c], want)
        assert hashlib.sha256(full[c].tobytes()).hexdigest() == str(REF[f"{name}_sha256_{c}"])
    assert small[0].dtype == (np.float64 if name == MF.DATASET_A[0] else np.float32)


@pytest.mark.parametrize("dataset", MF.DATASETS, ids=DATASET_IDS)
def test_oracle_case_statistics_equal_reference(dataset):
    name, cases = dataset
    for (key, *_), (seg, images) in zip(cases, _cases(dataset)):
        samples, stats = FO.collect_foreground_intensities(seg, images, num_samples=MF.CASE_SAMPLES)
        for c in range(MF.CHANNELS):
            assert np.array_equal(np.asarray(samples[c], dtype=np.float32), REF[f"{name}_{key}_case_samples_{c}"])
            got = np.array([stats[c][k] for k in MF.STAT_KEYS], dtype=np.float32)
            assert np.array_equal(got, REF[f"{name}_{key}_case_stats_{c}"], equal_nan=True), key
            if len(samples[c]):
                assert all(type(stats[c][k]) is np.float32 for k in MF.STAT_KEYS)


def _sweep():
    rng = np.random.default_rng(7)
    for n in (1, 2, 3, 8, 9, 128, 129, 1000, 4097, 100001):
        yield f"uniform{n}", rng.standard_normal(n) * 100
        yield f"ties{n}", rng.integers(-2048, 2048, n).astype(np.float64)
        yield f"equal{n}", np.full(n, -3.25)
    yield "ties_large", rng.integers(0, 4096, 3_000_001).astype(np.float64)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_host_finishing_equals_numpy(dtype):
    for label, x in _sweep():
        x = x.astype(dtype)
        n, s = len(x), np.sort(x)
        for q in (0.5, 50, 99.5):
            lo, hi, gamma = F.quantile_positions(n, q, dtype)
            got, want = F.lerp(s[lo], s[hi], gamma), np.percentile(x, q)
            assert got == want and got.dtype == want.dtype, (label, q)
        med = F.median_of([s[r] for r in F.median_ranks(n)], dtype)
        assert med == np.median(x) and med.dtype == np.median(x).dtype, label
        mean = F.finish_mean(np.sum(x), n, dtype)
        assert mean == np.mean(x) and mean.dtype == np.mean(x).dtype, label
        std = F.finish_std(np.sum(np.square(x - mean)), n, dtype)
        assert std == np.std(x) and std.dtype == np.std(x).dtype, label
        assert len(F.statistic_ranks(n, dtype)) <= 8


def _case():
    rng = np.random.default_rng(3)
    images = rng.integers(-5, 6, size=(2, 3, 8, 9)).astype(np.float32)
    seg = rng.integers(0, 3, size=(1, 3, 8, 9)).astype(np.int16)
    return seg, images


def _bad(kind):
    seg, images = _case()
    if kind == "images_f64":
        return seg, images.astype(np.float64), NotImplementedError
    if kind == "seg_i64":
        return seg.astype(np.int64), images, NotImplementedError
    if kind == "shape":
        return seg[:, :, :7], images, IndexError
    if kind == "inf":
        images[1, 2, 3, 4] = -np.inf
        return seg, images, NotImplementedError
    if kind == "nan_images":
        images[0, 0, 0, 0] = np.nan
        return seg, images, AssertionError
    if kind == "nan_seg":
        seg = seg.astype(np.float32)
        seg[0, 1, 1, 1] = np.nan
        return seg, images, AssertionError
    if kind == "ndim":
        return seg[0], images, AssertionError
    raise AssertionError(kind)


@pytest.mark.parametrize("kind", ["images_f64", "seg_i64", "shape", "inf", "nan_images", "nan_seg", "ndim"])
def test_rejections_before_any_launch(kind, monkeypatch):
    seg, images, exc = _bad(kind)
    seg_in, images_in = seg.copy(), images.copy()

    def no_launch(*a, **k):
        raise RuntimeError("the native library was reached")

    monkeypatch.setattr(F.L, "load", no_launch)
    with pytest.raises(exc) as e:
        F.DeviceFingerprintExtractor.collect_foreground_intensities(seg, images)
    if kind == "nan_images":
        assert str(e.value) == F.NAN_IMAGES
    if kind == "nan_seg":
        assert str(e.value) == F.NAN_SEG
    assert np.array_equal(seg, seg_in, equal_nan=True) and np.array_equal(images, images_in, equal_nan=True)


def test_too_many_voxels_rejected_before_any_launch(monkeypatch):
    monkeypatch.setattr(F.L, "load", lambda: (_ for _ in ()).throw(RuntimeError("the native library was reached")))
    images = torch.empty((1, 1 << 11, 1 << 10, 1 << 10), dtype=torch.float32, device="meta")
    seg = torch.empty((1, 1 << 11, 1 << 10, 1 << 10), dtype=torch.uint8, device="meta")
    with pytest.raises(NotImplementedError, match="2\\^31"):
        F.check_case(seg, images)
