"""-m gpu: the dataset fingerprint on the device against the reference's own DatasetFingerprintExtractor
(tests/golden/fingerprint_cases.npz): the JSON byte for byte, the dataset sample vectors, the per-case statistics; the
radix select against np.partition and the moments against numpy; the rejections; and DevicePreprocessor.run against
run_case_save."""
import ctypes
import hashlib
import json
import os
import pickle
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dinounet_b200 import fingerprint as F
from dinounet_b200 import lib as L
from dinounet_b200 import preprocess as PP
from oracle import make_golden_fingerprint as MF
from oracle import make_golden_preprocess_training as MT
from oracle import preprocess_training_oracle as PO
from tests.gpu_helpers import stream

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
REF = np.load(os.path.join(os.path.dirname(__file__), "golden", "fingerprint_cases.npz"))
DATASET_IDS = [d[0] for d in MF.DATASETS]


@pytest.fixture
def raw_datasets(tmp_path, monkeypatch):
    """The golden datasets as `.npy` files under tmp_path/raw, with the module seams pointed at them."""
    arrays = {k: REF[k] for k in REF.files}
    raw, pre = str(tmp_path / "raw"), str(tmp_path / "preprocessed")
    MF.NpyReader.REFERENCE_VIEW = False
    datasets = {ds[0]: MF.write_dataset(raw, ds, arrays) for ds in MF.DATASETS}
    monkeypatch.setattr(PP, "_dataset_name", lambda x: x)
    monkeypatch.setattr(PP, "_raw_and_preprocessed", lambda: (raw, pre))
    monkeypatch.setattr(PP, "_get_filenames_of_train_images_and_targets",
                        lambda folder, dj: datasets[os.path.basename(folder)])
    monkeypatch.setattr(F, "_determine_reader_writer", lambda dj, f: MF.NpyReader)
    return raw, pre


@pytest.mark.parametrize("dataset", MF.DATASETS, ids=DATASET_IDS)
def test_json_byte_identical(dataset, raw_datasets):
    name = dataset[0]
    fp = F.DeviceFingerprintExtractor(name, num_processes=3).run(overwrite_existing=True)
    with open(os.path.join(raw_datasets[1], name, "dataset_fingerprint.json")) as f:
        assert f.read() == str(REF[f"{name}_json"])
    assert json.dumps(fp, sort_keys=True, indent=4) == str(REF[f"{name}_json"])
    assert list(fp["foreground_intensity_properties_per_channel"]) == [0, 1]
    again = F.DeviceFingerprintExtractor(name).run(overwrite_existing=False)   # loads the file
    assert json.dumps(again, sort_keys=True, indent=4) == str(REF[f"{name}_json"])


@pytest.mark.parametrize("dataset", MF.DATASETS, ids=DATASET_IDS)
def test_sample_vectors(dataset, raw_datasets):
    name, cases = dataset
    ext = F.DeviceFingerprintExtractor(name, num_processes=2)
    keys = list(ext.dataset)
    for budget, check in ((MF.SMALL_BUDGET, "small"), (10e7, "sha")):
        _, _, vectors, total, promoted = ext._sample_dataset(keys, MF.NpyReader, int(budget // len(cases)))
        assert promoted == (name == MF.DATASET_A[0])
        host = vectors[:, :total].cpu().numpy().astype(np.float64 if promoted else np.float32)
        for c in range(MF.CHANNELS):
            if check == "small":
                want = REF[f"{name}_samples_small_{c}"]
                assert host[c].dtype == want.dtype and np.array_equal(host[c], want)
            else:
                assert hashlib.sha256(np.ascontiguousarray(host[c]).tobytes()).hexdigest() == \
                    str(REF[f"{name}_sha256_{c}"])


@pytest.mark.parametrize("as_tensor", [False, True], ids=["numpy", "cuda_tensor"])
def test_case_statistics(as_tensor):
    for name, cases in MF.DATASETS:
        for key, *_ in cases:
            seg, images = REF[f"{name}_{key}_seg"], REF[f"{name}_{key}_images"]
            if as_tensor:
                s = torch.from_numpy(seg.view(np.int16) if seg.dtype == np.uint16 else seg).to(DEV)
                s = s.view(torch.uint16) if seg.dtype == np.uint16 else s
                seg_in, img_in = s, torch.from_numpy(images).to(DEV)
            else:
                seg_in, img_in = seg, images
            samples, stats = F.DeviceFingerprintExtractor.collect_foreground_intensities(
                seg_in, img_in, num_samples=MF.CASE_SAMPLES)
            for c in range(MF.CHANNELS):
                want_s, want = REF[f"{name}_{key}_case_samples_{c}"], REF[f"{name}_{key}_case_stats_{c}"]
                if len(want_s) == 0:
                    assert samples[c] == [] and all(np.isnan(stats[c][k]) for k in MF.STAT_KEYS), key
                    continue
                if as_tensor:
                    assert samples[c].device == DEV and all(stats[c][k].device == DEV for k in MF.STAT_KEYS)
                    got_s = samples[c].cpu().numpy()
                    got = np.array([stats[c][k].item() for k in MF.STAT_KEYS], dtype=np.float32)
                else:
                    got_s = samples[c]
                    assert all(type(stats[c][k]) is np.float32 for k in MF.STAT_KEYS)
                    got = np.array([stats[c][k] for k in MF.STAT_KEYS], dtype=np.float32)
                assert got_s.dtype == np.float32 and np.array_equal(got_s, want_s), key
                assert np.array_equal(got, want), (key, got, want)


def _select(x: np.ndarray, ranks):
    lib = L.load()
    xd = torch.from_numpy(x).to(DEV)
    out = torch.empty(len(ranks), dtype=torch.float32, device=DEV)
    work = torch.empty(int(lib.b2u_fp_select_work_bytes()), dtype=torch.uint8, device=DEV)
    host = (ctypes.c_int64 * len(ranks))(*ranks)
    L.check(lib.b2u_fp_select(xd.data_ptr(), len(x), host, len(ranks), work.data_ptr(), out.data_ptr(), stream()),
            "b2u_fp_select")
    return out.cpu().numpy()


def _select_input(label: str) -> np.ndarray:
    rng = np.random.default_rng(11)
    if label == "uniform":
        return rng.random(120_000_000, dtype=np.float32)
    if label == "ties12":
        return (rng.integers(0, 4096, 30_000_001) - 2048).astype(np.float32)
    if label == "equal":
        return np.full(5_000_000, 7.5, np.float32)
    if label == "negative":
        return -rng.random(3_000_000, dtype=np.float32) * np.float32(1e30)
    if label == "denormal":
        return (rng.integers(-1000, 1000, 1_000_003) * np.float32(1e-44)).astype(np.float32)
    if label == "zeros":   # -0.0 and +0.0 mixed, and a few other values
        n = 1_000_001
        z = np.where(rng.random(n) < 0.5, np.float32(-0.0), np.float32(0.0)).astype(np.float32)
        return np.where(rng.random(n) < 0.01, rng.standard_normal(n).astype(np.float32), z)
    if label == "one":
        return np.array([-3.0], np.float32)
    return np.array([2.0, -0.0], np.float32)


@pytest.mark.parametrize("label", ["uniform", "ties12", "equal", "negative", "denormal", "zeros", "one", "two"])
def test_select_against_partition(label):
    x = _select_input(label)
    n = len(x)
    base = sorted({0, 1, n // 2, n - 2, n - 1, (n - 1) // 3, int(n * 0.995)} & set(range(n)))
    for i in range(0, len(base), 8):
        ranks = base[i:i + 8]
        want = np.partition(x, ranks)[ranks]
        assert np.array_equal(_select(x, ranks) == want, np.ones(len(ranks), bool)), (label, ranks)
    assert _select(x, [0])[0] == x.min() and _select(x, [n - 1])[0] == x.max()
    if label == "zeros":   # zeros come back as +0.0
        sel = _select(x, base)
        assert np.signbit(x).any() and (sel == 0).any() and not np.signbit(sel[sel == 0]).any()


@pytest.mark.parametrize("n", [1, 7, 129, 1_000_003, 50_000_000])
def test_moments_equal_numpy(n):
    lib = L.load()
    rng = np.random.default_rng(n)
    x = (rng.integers(-1024, 3000, n) * np.float32(0.25)).astype(np.float32)
    xd = torch.from_numpy(x).to(DEV)
    for f64 in (0, 1):
        stats = torch.empty(2, dtype=torch.float64 if f64 else torch.float32, device=DEV)
        work = torch.empty(int(lib.b2u_fp_moments_work_bytes(n, f64)), dtype=torch.uint8, device=DEV)
        L.check(lib.b2u_fp_moments(xd.data_ptr(), n, f64, 1, work.data_ptr(), stats.data_ptr(), stream()),
                "b2u_fp_moments")
        y = x.astype(np.float64) if f64 else x
        mean, std = stats.cpu().numpy()
        assert mean == np.mean(y) and std == np.std(y), (n, f64)


@pytest.mark.parametrize("kind", ["images_f64", "seg_i64", "shape", "inf", "nan_images", "nan_seg"])
def test_cuda_tensor_rejections_leave_inputs_unchanged(kind):
    from tests.test_fingerprint_cpu import _bad
    seg, images, exc = _bad(kind)
    s, im = torch.from_numpy(seg).to(DEV), torch.from_numpy(images).to(DEV)
    s0, im0 = s.clone(), im.clone()
    before = int(L.load().b2u_launch_count())
    with pytest.raises(exc):
        F.DeviceFingerprintExtractor.collect_foreground_intensities(s, im)
    assert int(L.load().b2u_launch_count()) == before
    assert torch.equal(s.isnan(), s0.isnan()) if s.is_floating_point() else torch.equal(s, s0)
    assert torch.equal(torch.nan_to_num(im), torch.nan_to_num(im0))


# ---- DevicePreprocessor.run ------------------------------------------------------------------------------------------


def _write_preprocess_dataset(raw, pre, name):
    rng = np.random.default_rng(5)
    folder = os.path.join(raw, name)
    os.makedirs(folder)
    labels = {"background": 0, "a": 1, "b": 2}
    ds = {}
    for i in range(4):
        shape = (3, 24 + i, 20)
        img = (rng.standard_normal(shape) * 30 + 10).astype(np.float32)
        seg = rng.integers(0, 3, size=shape).astype(np.uint8 if i % 2 else np.int16)
        f_img, f_seg = os.path.join(folder, f"c{i}_0000.npy"), os.path.join(folder, f"c{i}.npy")
        np.save(f_img, img)
        np.save(f_seg, seg)
        MF.NpyReader.SPACINGS[f_img] = MF.NpyReader.SPACINGS[f_seg] = [5.0, 0.8, 0.8]
        ds[f"c{i}"] = {"images": [f_img], "label": f_seg}
    os.makedirs(os.path.join(pre, name))
    with open(os.path.join(pre, name, "dataset.json"), "w") as f:
        json.dump({"labels": labels, "channel_names": {"0": "MR"}, "file_ending": ".npy"}, f)
    with open(os.path.join(pre, name, "TestPlans.json"), "w") as f:
        json.dump({"plans_name": "TestPlans"}, f)
    os.makedirs(os.path.join(pre, name, "2d"))
    with open(os.path.join(pre, name, "2d", "stale.npz"), "w") as f:
        f.write("removed by run")
    return ds


def _managers():
    conf = {"preprocessor_name": "DefaultPreprocessor", "resampling_fn_data": PP.DEFAULT_RESAMPLING_FN,
            "resampling_fn_data_kwargs": dict(PP.DEFAULT_RESAMPLING_KWARGS),
            "resampling_fn_seg": PP.DEFAULT_RESAMPLING_FN,
            "resampling_fn_seg_kwargs": dict(PP.DEFAULT_RESAMPLING_SEG_KWARGS)}
    cm = SimpleNamespace(spacing=[0.5, 0.5], normalization_schemes=["ZScoreNormalization"], use_mask_for_norm=[False],
                         configuration=conf, data_identifier="2d")
    pm = SimpleNamespace(transpose_forward=[0, 1, 2], foreground_intensity_properties_per_channel=MT.INTENSITY,
                         get_label_manager=lambda dj: PO.LabelSets(dj["labels"], dj.get("regions_class_order")),
                         image_reader_writer_class=MF.NpyReader, get_configuration=lambda name: cm)
    return pm, cm


def _same(a, b):
    if isinstance(a, dict):
        return isinstance(b, dict) and list(a) == list(b) and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, np.ndarray):
        return isinstance(b, np.ndarray) and a.dtype == b.dtype and np.array_equal(a, b)
    if isinstance(a, (list, tuple)):
        return type(a) is type(b) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return type(a) is type(b) and a == b


def test_device_preprocessor_run_writes_run_case_save_files(tmp_path, monkeypatch):
    raw, pre, name = str(tmp_path / "raw"), str(tmp_path / "pre"), "Dataset903_Pre"
    ds = _write_preprocess_dataset(raw, pre, name)
    pm, cm = _managers()
    seen = []
    monkeypatch.setattr(PP, "_dataset_name", lambda x: name)
    monkeypatch.setattr(PP, "_raw_and_preprocessed", lambda: (raw, pre))
    monkeypatch.setattr(PP, "_plans_manager", lambda plans: seen.append(plans) or pm)
    monkeypatch.setattr(PP, "_get_filenames_of_train_images_and_targets", lambda folder, dj: ds)
    PP.DevicePreprocessor(verbose=False, device=DEV).run(903, "2d", "TestPlans", 3)
    assert seen == [{"plans_name": "TestPlans"}]
    out = os.path.join(pre, name, "2d")
    assert sorted(os.listdir(out)) == sorted(f"{k}.{e}" for k in ds for e in ("npz", "pkl"))
    with open(os.path.join(pre, name, "dataset.json")) as f:
        dj = json.load(f)
    ref_dir = tmp_path / "single"
    ref_dir.mkdir()
    for k, v in ds.items():
        PP.DevicePreprocessor(verbose=False, device=DEV).run_case_save(str(ref_dir / k), v["images"], v["label"], pm,
                                                                       cm, dj)
        got, want = np.load(os.path.join(out, k + ".npz")), np.load(str(ref_dir / (k + ".npz")))
        assert sorted(got.files) == sorted(want.files) == ["data", "seg"]
        for f in ("data", "seg"):
            assert got[f].dtype == want[f].dtype and np.array_equal(got[f], want[f]), (k, f)
        with open(os.path.join(out, k + ".pkl"), "rb") as f1, open(str(ref_dir / (k + ".pkl")), "rb") as f2:
            assert _same(pickle.load(f1), pickle.load(f2)), k
