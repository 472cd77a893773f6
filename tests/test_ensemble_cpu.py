"""Ensembling without a GPU: the oracle against the golden (tests/golden/ensemble_cases.npz) and, where the reference
sources are present, against the reference's own `merge_files` / `ensemble_folders`; the drop-ins' file handling,
checks and messages, every rejection before any native call, and which C-ABI calls they make (recording stand-in for
the native library)."""
import contextlib
import json
import os
import pickle
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dinounet_b200 import ensembling as E
from dinounet_b200 import predict as PR
from oracle import ensemble_oracle as EN

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "ensemble_cases.npz"))


def _lm(C=3, regions=False):
    if regions:
        return SimpleNamespace(has_regions=True, regions_class_order=list(EN.REGION_ORDER), foreground_labels=[1, 2, 3],
                               num_segmentation_heads=C)
    return SimpleNamespace(has_regions=False, regions_class_order=None, foreground_labels=list(range(1, C)),
                           num_segmentation_heads=C)


@pytest.mark.parametrize("case", EN.GOLDEN_CASES, ids=[c[0] for c in EN.GOLDEN_CASES])
def test_oracle_reproduces_golden(case):
    name, C, regions, dtypes, _ = case
    members = [GOLDEN[f"{name}_m{k}"] for k in range(len(dtypes))]
    for k, m in enumerate(EN.golden_members(case, EN.GOLDEN_CASES.index(case))):
        assert np.array_equal(m, members[k])
    avg = EN.average_probabilities(members)
    assert np.array_equal(avg.view(np.int32), GOLDEN[f"{name}_avg"].view(np.int32))
    seg = EN.convert_logits_to_segmentation(avg, regions, EN.REGION_ORDER)
    assert np.array_equal(seg, GOLDEN[f"{name}_seg"])
    if regions and set(dtypes) == {"f4"}:   # averages on both sides of 1.5 * 2^-24 are planted and decide differently
        flat = seg.reshape(-1)
        assert flat[0] == 0 and flat[1] == 3 and flat[3] == 3


def test_torch_sigmoid_threshold():
    """Averaged region values around 1.5 * 2^-24: torch's CPU sigmoid(x) > 0.5 holds from the next float up."""
    t = np.float32(1.5 * 2.0 ** -24)
    x = np.array([np.nextafter(t, np.float32(0)), t, np.nextafter(t, np.float32(1)), 2.0 ** -23], np.float32)
    assert (torch.sigmoid(torch.from_numpy(x)) > 0.5).tolist() == [False, False, True, True]


def _reference():
    from oracle import ref_loader
    if not ref_loader.reference_available():
        pytest.skip("reference sources not present")
    return EN.load_reference_ensemble_module()


class NpyIO:
    def write_seg(self, seg, path, properties):
        np.save(path, seg)


def _write_members(folder, name, members, props=None):
    os.makedirs(folder, exist_ok=True)
    f = os.path.join(folder, name + ".npz")
    np.savez_compressed(f, probabilities=members)
    with open(os.path.join(folder, name + ".pkl"), "wb") as fh:
        pickle.dump(props if props is not None else {"folder": os.path.basename(folder)}, fh)
    return f


@pytest.mark.parametrize("case", EN.GOLDEN_CASES, ids=[c[0] for c in EN.GOLDEN_CASES])
def test_oracle_against_reference_merge_files(tmp_path, case):
    ensemble, LabelManager = _reference()
    name, C, regions, dtypes, _ = case
    members = [GOLDEN[f"{name}_m{k}"] for k in range(len(dtypes))]
    files = [_write_members(str(tmp_path / f"m{k}"), name, m) for k, m in enumerate(members)]
    label_dict = {"background": 0, "whole": [1, 2, 3], "core": [2, 3], "enh": [3]} if regions else \
        {"background": 0, **{f"c{i}": i for i in range(1, C)}}
    lm = LabelManager(label_dict, list(EN.REGION_ORDER) if regions else None)
    ensemble.merge_files(files, str(tmp_path / "ref"), ".npy", NpyIO(), lm, True)
    EN.merge_files(files, str(tmp_path / "ora"), ".npy", NpyIO(), lm, True)
    assert np.array_equal(np.load(tmp_path / "ref.npy"), np.load(tmp_path / "ora.npy"))
    assert np.array_equal(np.load(tmp_path / "ref.npz")["probabilities"], np.load(tmp_path / "ora.npz")["probabilities"])
    with open(tmp_path / "ref.pkl", "rb") as f:
        assert np.array_equal(pickle.load(f), np.load(tmp_path / "ora.npz")["probabilities"])   # probabilities, not props


class _InProcessPool:
    """multiprocessing's spawn pool run in this process."""

    def __init__(self, *a, **k):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False

    def starmap(self, fn, it):
        return [fn(*args) for args in it]


def test_oracle_against_reference_ensemble_folders(tmp_path, monkeypatch):
    ensemble, LabelManager = _reference()
    lm = LabelManager({"background": 0, "a": 1, "b": 2}, None)
    pm = SimpleNamespace(image_reader_writer_class=NpyIO, get_label_manager=lambda dj: lm)
    monkeypatch.setattr(ensemble, "PlansManager", lambda plans: pm)
    monkeypatch.setattr(ensemble.multiprocessing, "get_context", lambda kind: SimpleNamespace(Pool=_InProcessPool))
    rng = np.random.default_rng(3)
    folders = []
    for k in range(3):
        d = tmp_path / f"in{k}"
        for case in ("a", "b"):
            x = torch.from_numpy(rng.standard_normal((3, 2, 9, 11)).astype(np.float32))
            _write_members(str(d), case, torch.softmax(x, 0).numpy())
        (d / "dataset.json").write_text('{"file_ending": ".npy"}')
        (d / "plans.json").write_text("{}")
        folders.append(str(d))
    ensemble.ensemble_folders(folders, str(tmp_path / "ref"), True, 2)
    for case in ("a", "b"):
        EN.merge_files([os.path.join(f, case + ".npz") for f in folders], str(tmp_path / f"ora_{case}"), ".npy",
                       NpyIO(), lm, True)
        assert np.array_equal(np.load(tmp_path / "ref" / f"{case}.npy"), np.load(tmp_path / f"ora_{case}.npy"))
        assert np.array_equal(np.load(tmp_path / "ref" / f"{case}.npz")["probabilities"],
                              np.load(tmp_path / f"ora_{case}.npz")["probabilities"])
    assert (tmp_path / "ref" / "dataset.json").is_file() and not (tmp_path / "ref" / "plans.json").exists()


# ---- the drop-ins with a recording stand-in for the native library


class _Recorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*a):
            self.calls.append((name, a))
            return 0
        return fn


@pytest.fixture
def rec(monkeypatch):
    from dinounet_b200 import lib as L
    r = _Recorder()
    monkeypatch.setattr(L, "load", lambda: r)
    # CPU tensors stand in for device buffers: the stand-in library never reads them
    monkeypatch.setattr(E, "_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda dev=None: SimpleNamespace(cuda_stream=0))
    return r


def _folders(tmp_path, n, cases=("x", "y"), C=3, dtype=np.float32, shape=(2, 4, 5)):
    folders = []
    for k in range(n):
        d = tmp_path / f"f{k}"
        for c in cases:
            _write_members(str(d), c, np.full((C, *shape), 1.0 / C, dtype), {"case": c, "member": k})
        (d / "dataset.json").write_text(json.dumps({"file_ending": ".npy", "labels": {"background": 0}}))
        (d / "plans.json").write_text('{"plans_name": "p"}')
        folders.append(str(d))
    return folders


@pytest.fixture
def plans(monkeypatch):
    written = []

    class RW:
        def write_seg(self, seg, path, props):
            written.append((path, seg.dtype, seg.shape, props))

    lm = _lm(3)
    pm = SimpleNamespace(image_reader_writer_class=RW, get_label_manager=lambda dj: lm)
    monkeypatch.setattr(PR, "_plans_manager", lambda plans: pm)
    return SimpleNamespace(written=written, lm=lm, pm=pm)


def test_ensemble_folders_calls_and_files(tmp_path, rec, plans):
    folders = _folders(tmp_path, 3)
    out = tmp_path / "out"
    E.ensemble_folders(folders, str(out), save_merged_probabilities=False, num_processes=2)
    names = [n for n, _ in rec.calls]
    assert names == (["b2u_ensemble_accumulate"] * 3 + ["b2u_ensemble_segment"]) * 2
    firsts = [a[4] for n, a in rec.calls if n == "b2u_ensemble_accumulate"]
    assert firsts == [1, 0, 0, 1, 0, 0]
    acc = [a for n, a in rec.calls if n == "b2u_ensemble_accumulate"][0]
    assert acc[1] == 4 and acc[3] == 3 * 2 * 4 * 5
    seg = [a for n, a in rec.calls if n == "b2u_ensemble_segment"][0]
    assert seg[1:5] == (3, 2 * 4 * 5, 3, 0) and seg[5] is None and seg[7] == 1
    assert sorted(os.path.basename(p) for p, *_ in plans.written) == ["x.npy", "y.npy"]
    assert all(dt == np.uint8 and shape == (2, 4, 5) for _, dt, shape, _ in plans.written)
    assert all(props["member"] == 0 for *_, props in plans.written)          # the first member's properties
    assert (out / "dataset.json").is_file() and not (out / "plans.json").exists()
    assert not (out / "x.npz").exists()


def test_save_probabilities_pickles_the_probabilities(tmp_path, rec, plans):
    folders = _folders(tmp_path, 2, cases=("x",), dtype=np.float16)
    E.ensemble_folders(folders, str(tmp_path / "out"), save_merged_probabilities=True)
    assert [a[1] for n, a in rec.calls if n == "b2u_ensemble_accumulate"] == [2, 2]      # fp16 members
    p = np.load(tmp_path / "out" / "x.npz")["probabilities"]
    with open(tmp_path / "out" / "x.pkl", "rb") as f:
        # the stand-in library leaves the buffer as allocated: compare bits, which may hold NaNs
        assert np.array_equal(pickle.load(f).view(np.int32), p.view(np.int32))
    assert p.dtype == np.float32 and p.shape == (3, 2, 4, 5)


def test_folders_must_hold_the_same_files(tmp_path, rec, plans):
    folders = _folders(tmp_path, 2)
    os.remove(os.path.join(folders[1], "y.npz"))
    with pytest.raises(AssertionError, match="Not all folders contain the same files"):
        E.ensemble_folders(folders, str(tmp_path / "out"))
    assert rec.calls == []


@pytest.mark.parametrize("kind", ["float64", "channels", "shape", "heads"])
def test_rejections_before_any_native_call(tmp_path, rec, plans, kind):
    folders = _folders(tmp_path, 2, cases=("x",))
    bad = os.path.join(folders[1], "x.npz")
    if kind == "float64":
        np.savez_compressed(bad, probabilities=np.zeros((3, 2, 4, 5), np.float64))
        exc = NotImplementedError
    elif kind == "channels":
        plans.lm.num_segmentation_heads = 33
        for f in folders:
            np.savez_compressed(os.path.join(f, "x.npz"), probabilities=np.zeros((33, 2, 4, 5), np.float32))
        exc = NotImplementedError
    elif kind == "shape":
        np.savez_compressed(bad, probabilities=np.zeros((3, 2, 4, 6), np.float32))
        exc = ValueError
    else:
        plans.lm.num_segmentation_heads = 4
        exc = AssertionError
    with pytest.raises(exc):
        E.ensemble_folders(folders, str(tmp_path / "out"))
    assert rec.calls == []


def _model(tmp_path, name, folds, cases=("x", "y")):
    root = tmp_path / name
    for f in folds:
        d = root / f"fold_{f}" / "validation"
        os.makedirs(d)
        for c in cases:
            _write_members(str(d), c, np.full((3, 1, 2, 2), 1.0 / 3, np.float32))
    (root / "dataset.json").write_text('{"file_ending": ".npy"}')
    (root / "plans.json").write_text('{"plans_name": "p"}')
    return str(root)


def test_ensemble_crossvalidations(tmp_path, rec, plans):
    a = _model(tmp_path, "a", (0,), ("x",))
    os.makedirs(tmp_path / "a" / "fold_1" / "validation")
    _write_members(str(tmp_path / "a" / "fold_1" / "validation"), "y", np.full((3, 1, 2, 2), 1 / 3, np.float32))
    b = _model(tmp_path, "b", (0, 1), ("y",))
    os.remove(tmp_path / "b" / "fold_0" / "validation" / "y.npz")
    _write_members(str(tmp_path / "b" / "fold_0" / "validation"), "x", np.full((3, 1, 2, 2), 1 / 3, np.float32))
    out = tmp_path / "out"
    E.ensemble_crossvalidations([a, b], str(out), folds=(0, 1))
    assert sorted(os.path.basename(p) for p, *_ in plans.written) == ["x.npy", "y.npy"]
    assert (out / "plans.json").is_file() and (out / "dataset.json").is_file()
    assert len(rec.calls) == 6
    # overwrite=False skips the cases whose segmentation exists
    rec.calls.clear()
    np.save(out / "x.npy", np.zeros(1))
    E.ensemble_crossvalidations([a, b], str(out), folds=(0, 1), overwrite=False)
    assert len(rec.calls) == 3 and os.path.basename(plans.written[-1][0]) == "y.npy"


def test_ensemble_crossvalidations_errors(tmp_path, rec, plans):
    a = _model(tmp_path, "a", (0, 1))
    with pytest.raises(RuntimeError, match="Expected model output directory does not exist"):
        E.ensemble_crossvalidations([a], str(tmp_path / "o"), folds=(0, 1, 2))
    empty = _model(tmp_path, "e", (0,), ())
    with pytest.raises(RuntimeError, match="Rerun your validation with the --npz flag"):
        E.ensemble_crossvalidations([empty], str(tmp_path / "o"), folds=(0,))
    # a case in two folds of one model
    with pytest.raises(AssertionError, match="Duplicate detected"):
        E.ensemble_crossvalidations([a], str(tmp_path / "o"), folds=(0, 1))
    # a model without every case
    b = _model(tmp_path, "b", (0,), ("x",))
    c = _model(tmp_path, "c", (0,), ("x", "y"))
    with pytest.raises(RuntimeError, match="There were missing files"):
        E.ensemble_crossvalidations([b, c], str(tmp_path / "o"), folds=(0,))
    assert rec.calls == []


def test_entry_point(tmp_path, rec, plans, monkeypatch):
    folders = _folders(tmp_path, 2)
    seen = {}
    monkeypatch.setattr(E, "ensemble_folders", lambda *a: seen.setdefault("args", a))
    monkeypatch.setattr("sys.argv", ["x", "-i", *folders, "-o", str(tmp_path / "o"), "-np", "5", "--save_npz"])
    E.entry_point_ensemble_folders()
    assert seen["args"] == (folders, str(tmp_path / "o"), True, 5)


def test_average_probabilities(tmp_path, rec):
    folders = _folders(tmp_path, 2, cases=("x",))
    avg = E.average_probabilities([os.path.join(f, "x.npz") for f in folders])
    assert avg.dtype == np.float32 and avg.shape == (3, 2, 4, 5)
    assert [n for n, _ in rec.calls] == ["b2u_ensemble_accumulate", "b2u_ensemble_accumulate", "b2u_ensemble_segment"]


# ---- predict_ensemble_from_files: member checks


def _predictor(plans=None, configuration=None, regions=False, prev=None):
    lm = _lm(3, regions)
    return SimpleNamespace(plans_manager=SimpleNamespace(plans=plans or {"plans_name": "p"}),
                           configuration_manager=SimpleNamespace(configuration=configuration or {"patch": 1},
                                                                 previous_stage_name=prev),
                           label_manager=lm, dataset_json={"file_ending": ".npy"}, trainer_name="DinoUNetTrainer_s")


def test_members_must_share_setup(tmp_path):
    for other, what in ((_predictor(plans={"plans_name": "q"}), "plans"),
                        (_predictor(configuration={"patch": 2}), "configuration"),
                        (_predictor(regions=True), "label manager")):
        with pytest.raises(ValueError, match=what):
            E.predict_ensemble_from_files([_predictor(), other], str(tmp_path), str(tmp_path / "o"))
    with pytest.raises(ValueError, match="plans_name"):
        E.check_same_setup([_predictor(), _predictor(plans={"plans_name": "q"})])
    with pytest.raises(NotImplementedError):
        E.predict_ensemble_from_files([_predictor(prev="3d_lowres")], str(tmp_path), str(tmp_path / "o"))
    assert not (tmp_path / "o").exists()
