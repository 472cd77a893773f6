"""Device evaluation without a GPU: the oracle (oracle/evaluation_oracle.py) against the reference's own
`compute_metrics` / `compute_metrics_on_folder` and against an all-pairs brute force, the host-side percentile
restatement against numpy, the summary aggregation, the rejections (before any launch) and which C-ABI calls the
evaluation makes with which arguments (recording stand-in for the native library), and the golden file
(tests/golden/evaluation_cases.npz, oracle/make_golden_evaluation.py)."""
import contextlib
import copy
import ctypes
import importlib
import json
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dinounet_b200 import evaluation as EV
from oracle import evaluation_oracle as EO

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "evaluation_cases.npz"))
CASES = {c[0]: c for c in EO.GOLDEN_CASES}


def _same_metrics(got: dict, want: dict):
    """Same keys in the same order, same value types, equal values with NaN in the same places."""
    assert list(got) == list(want)
    for r in want:
        assert list(got[r]) == list(want[r]) == list(EV.METRIC_KEYS)
        for k in want[r]:
            g, w = got[r][k], want[r][k]
            assert type(g) is type(w), (r, k, type(g), type(w))
            assert (np.isnan(g) and np.isnan(w)) or g == w, (r, k, g, w)


class _MemoryReader:
    """A reader-writer whose `read_seg` returns in-memory arrays and their spacing."""

    def __init__(self, cases):
        self.cases = cases

    def read_seg(self, name):
        seg, spacing = self.cases[os.path.basename(name)]
        return seg, ({} if spacing is None else {"spacing": spacing})


class _NpyReader:
    def __init__(self, spacing):
        self.spacing = spacing

    def read_seg(self, path):
        return np.load(path), {"spacing": self.spacing}


@pytest.fixture(scope="module")
def ref_eval():
    from oracle import ref_loader, ref_predictor_loader
    if not ref_loader.reference_available():
        pytest.skip("reference sources not present")
    # the loader's stub packages must not outlive this module: other tests install their own stand-ins
    roots, meta_path, path = {m.split(".")[0] for m in sys.modules}, list(sys.meta_path), list(sys.path)
    try:
        ref_predictor_loader.load_reference_predictor_class()
        mod = importlib.import_module("dinounet.evaluation.evaluate_predictions")
        json_export = importlib.import_module("dinounet.utilities.json_export")
    finally:
        for name in [m for m in sys.modules if m.split(".")[0] not in roots]:
            del sys.modules[name]
        sys.meta_path[:], sys.path[:] = meta_path, path
    return SimpleNamespace(module=mod, json_export=json_export)


@pytest.fixture
def medpy_oracle(ref_eval, monkeypatch):
    monkeypatch.setattr(ref_eval.module, "medpy_metric", SimpleNamespace(hd95=EO.hd95, asd=EO.asd))
    monkeypatch.setattr(ref_eval.module, "MEDPY_AVAILABLE", True)
    return ref_eval.module


@pytest.mark.parametrize("name", list(CASES))
def test_reference_compute_metrics_equals_oracle(name, medpy_oracle):
    _, _, spacing, regions, ignore, _, _ = CASES[name]
    ref, pred = EO.make_case(name)
    rw = _MemoryReader({"ref": (ref, spacing), "pred": (pred, None)})
    got = medpy_oracle.compute_metrics("ref", "pred", rw, regions, ignore)
    assert got["reference_file"] == "ref" and got["prediction_file"] == "pred"
    want = EO.compute_metrics_arrays(ref, pred, regions, ignore, spacing)
    _same_metrics(got["metrics"], want)
    rows = np.array([[float(want[r][k]) for k in EO.METRIC_KEYS] for r in regions])
    assert np.array_equal(rows, GOLDEN[f"{name}_metrics"], equal_nan=True)


def test_reference_spacing_fallbacks(medpy_oracle):
    """The prediction's spacing when the reference has none, else isotropic 1 (the 2D reader's (999, 1, 1) is just a
    spacing)."""
    ref, pred = EO.make_case("labels3_spacing311")
    for spacing_ref, spacing_pred, used in [(None, (2.0, 1.0, 1.0), (2.0, 1.0, 1.0)), (None, None, (1.0, 1.0, 1.0))]:
        rw = _MemoryReader({"ref": (ref, spacing_ref), "pred": (pred, spacing_pred)})
        got = medpy_oracle.compute_metrics("ref", "pred", rw, [1, 2], None)["metrics"]
        _same_metrics(got, EO.compute_metrics_arrays(ref, pred, [1, 2], None, used))
        assert EV._case_spacing(ref, {} if spacing_ref is None else {"spacing": spacing_ref},
                                {} if spacing_pred is None else {"spacing": spacing_pred}) == used


def test_ratios_follow_the_reference():
    """The new module's host arithmetic gives the oracle's dict from the same int64 counts (with the oracle's surface
    metrics)."""
    for name, _, spacing, regions, ignore, _, _ in EO.GOLDEN_CASES:
        ref, pred = EO.make_case(name)
        want = EO.compute_metrics_arrays(ref, pred, regions, ignore, spacing)
        got = {r: EV.ratios(*(want[r][k] for k in ("TP", "FP", "FN", "TN", "HD95", "ASD"))) for r in regions}
        _same_metrics(got, want)


def _write_folder(tmp_path, spacing):
    ref_dir, pred_dir = tmp_path / "gt", tmp_path / "pred"
    ref_dir.mkdir()
    pred_dir.mkdir()
    for i, name in enumerate(["labels3_spacing311", "empty_masks", "touching_faces"]):
        ref, pred = EO.make_case(name)
        ref, pred = ref[..., :10, :14, :16], pred[..., :10, :14, :16]
        np.save(ref_dir / f"case_{i}.npy", ref.astype(np.float32))
        np.save(pred_dir / f"case_{i}.npy", pred)
    np.save(pred_dir / "case_9.npy", pred)   # no reference: dropped unless chill
    (pred_dir / "notes.txt").write_text("not a case")
    return str(ref_dir), str(pred_dir)


def test_reference_folder_summary_equals_aggregation(tmp_path, medpy_oracle, monkeypatch):
    """The reference's compute_metrics_on_folder (serial stand-in for its spawn pool, json for batchgenerators'
    save_json) and the new module, both fed per-case results by the oracle, write the same summary and return the same
    dict."""
    spacing = (3.0, 1.0, 1.0)
    ref_dir, pred_dir = _write_folder(tmp_path, spacing)

    class _SerialPool:
        def __init__(self, n):
            pass

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False

        def starmap(self, fn, args):
            return [fn(*a) for a in args]

    monkeypatch.setattr(medpy_oracle, "multiprocessing", SimpleNamespace(get_context=lambda m: SimpleNamespace(Pool=_SerialPool)))
    monkeypatch.setattr(medpy_oracle, "subfiles", lambda folder, suffix=None, join=True:
                        [f if not join else os.path.join(folder, f) for f in EV._subfiles(folder, suffix)])
    monkeypatch.setattr(medpy_oracle, "isfile", os.path.isfile)

    def save_json(obj, file, indent=4, sort_keys=True):
        with open(file, "w") as f:
            json.dump(obj, f, sort_keys=sort_keys, indent=indent)

    monkeypatch.setattr(medpy_oracle, "save_json", save_json)
    monkeypatch.setattr(EV, "compute_metrics_arrays", EO.compute_metrics_arrays)
    rw = _NpyReader(spacing)
    regions = [1, 2, (1, 2)]
    for chill in (False, True):
        if chill:
            os.remove(os.path.join(pred_dir, "case_9.npy"))
        want = medpy_oracle.compute_metrics_on_folder(ref_dir, pred_dir, str(tmp_path / "ref.json"), rw, ".npy", regions,
                                                      None, 2, chill=chill)
        got = EV.compute_metrics_on_folder(ref_dir, pred_dir, str(tmp_path / "new.json"), rw, ".npy", regions, None, 2,
                                           chill=chill)
        assert (tmp_path / "ref.json").read_text() == (tmp_path / "new.json").read_text()
        assert repr(got) == repr(want)
        assert [os.path.basename(c["prediction_file"]) for c in got["metric_per_case"]] == ["case_0.npy", "case_1.npy",
                                                                                             "case_2.npy"]


# ---- the oracle's surface distances against an all-pairs brute force


@pytest.mark.parametrize("shape,spacing", [((5, 7, 9), (1.0, 1.0, 1.0)), ((6, 5, 8), (3.0, 1.0, 1.0)),
                                           ((1, 9, 11), (999.0, 1.0, 1.0)), ((4, 6, 7), (2.5, 0.7, 0.7)),
                                           ((7, 3, 5), (0.3, 1.7, 1.1)), ((3, 1, 12), (2.0, 5.0, 1.0))])
def test_oracle_distances_equal_brute_force(shape, spacing):
    from scipy import ndimage as ndi
    rng = np.random.default_rng(sum(shape))
    for trial in range(4):
        a = rng.random(shape) < 0.3
        b = rng.random(shape) < (0.05 if trial % 2 else 0.4)
        a.flat[0] = b.flat[-1] = True
        fp = ndi.generate_binary_structure(len(shape), 1)
        ab, bb = a ^ ndi.binary_erosion(a, fp), b ^ ndi.binary_erosion(b, fp)
        got = EO.surface_distances(a, b, spacing)
        want = EO.brute_force_distances(ab, bb, spacing)
        if all(float(s).is_integer() for s in spacing):
            assert np.array_equal(got, want)
        else:
            np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)


def test_edges_count_as_surface():
    """Erosion with border value 0: a 4x5 square in a (1, 6, 7) mask is all surface."""
    from scipy import ndimage as ndi
    m = np.zeros((1, 6, 7), bool)
    m[0, 1:5, 1:6] = True
    border = m ^ ndi.binary_erosion(m, ndi.generate_binary_structure(3, 1))
    assert border.sum() == 20


# ---- numpy's percentile, restated


@pytest.mark.parametrize("ties", [False, True])
def test_percentile_restatement_is_numpy_bit_for_bit(ties):
    rng = np.random.default_rng(7 + ties)
    for n in range(1, 3001):
        x = rng.integers(0, 6, n).astype(np.float64) * 0.7 if ties else rng.random(n) * 100
        s = np.sort(x)
        got = EV.percentile95(lambda k: s[k], n)
        want = np.percentile(x, 95)
        assert type(got) is type(want) and got.tobytes() == want.tobytes(), n


# ---- argument contract and call sequence (recording stand-in for the native library)


class _Recorder:
    def __init__(self):
        self.calls = []
        self.counts = [5, 1, 2, 7, 7, 6]

    def __getattr__(self, name):
        def fn(*a):
            self.calls.append((name, a))
            if name == "b2u_eval_masks":
                ctypes.memmove(a[14], (ctypes.c_int64 * 6)(*self.counts), 48)
                n = a[5] * a[6] * a[7]
                ctypes.memset(a[12], 1, n)
                ctypes.memset(a[13], 1, n)
            return 0
        return fn


@pytest.fixture
def rec(monkeypatch):
    from dinounet_b200 import lib as L
    r = _Recorder()
    monkeypatch.setattr(L, "load", lambda: r)
    # CPU tensors stand in for device buffers
    monkeypatch.setattr(EV, "_device", lambda ref, pred: torch.device("cpu"))
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda dev=None: SimpleNamespace(cuda_stream=0))
    return r


def test_call_sequence(rec):
    """Per label or region one mask pass with the stored dtypes, the rank and the label values; with both masks
    non-empty two EDTs at the spacing (a rank-2 mask padded with a leading unit axis) and one float64 sum."""
    ref = np.zeros((1, 4, 6, 8), np.float32)
    pred = torch.zeros((1, 4, 6, 8), dtype=torch.uint16)
    m = EV.compute_metrics_arrays(ref, pred, [3, (1, 2)], ignore_label=9, spacing=(2.0, 0.5, 0.25))
    names = [n for n, _ in rec.calls]
    assert names == ["b2u_eval_masks", "b2u_eval_edt", "b2u_eval_edt", "b2u_eval_sum_f64"] * 2
    a = rec.calls[0][1]
    assert (a[1], a[3], a[4:8], list(a[8][:a[9]]), a[9], a[10], a[11]) == (5, 3, (3, 4, 6, 8), [3], 1, 1, 9)
    assert list(rec.calls[4][1][8][:2]) == [1, 2] and rec.calls[4][1][9] == 2
    e = rec.calls[1][1]
    assert e[1:7] == (4, 6, 8, 2.0, 0.5, 0.25)
    assert rec.calls[1][1][0] == a[12] and rec.calls[2][1][0] == a[13]   # the reference's border, then the prediction's
    s = rec.calls[3][1]
    assert s[1] == 4 * 6 * 8   # every voxel is on the stand-in's prediction border
    assert m[3]["TP"] == 5 and type(m[3]["TP"]) is np.int64 and m[3]["n_pred"] == 6 and m[3]["n_ref"] == 7
    assert type(m[3]["HD95"]) is float and type(m[3]["Dice"]) is np.float64

    rec.calls.clear()
    rec.counts = [0, 0, 3, 9, 3, 0]   # empty prediction: no surface distances
    m = EV.compute_metrics_arrays(ref[:, 0], pred[:, 0], [1], spacing=(999.0, 1.0))
    assert [n for n, _ in rec.calls] == ["b2u_eval_masks"]
    assert rec.calls[0][1][4:8] == (2, 1, 6, 8) and rec.calls[0][1][10] == 0
    assert np.isnan(m[1]["HD95"]) and np.isnan(m[1]["ASD"]) and np.isnan(m[1]["Precision"])


def test_spacing_of_wrong_length_gives_nan_like_medpy(rec):
    EV.compute_metrics_arrays(np.zeros((1, 3, 4, 5), np.uint8), np.zeros((1, 3, 4, 5), np.uint8), [1],
                              spacing=(1.0, 1.0))
    assert [n for n, _ in rec.calls] == ["b2u_eval_masks"]


@pytest.mark.parametrize("kwargs,exc,match", [
    (dict(pred=np.zeros((1, 4, 6, 7), np.uint8)), ValueError, "differ in shape"),
    (dict(ref=np.zeros((1, 4, 6, 8), np.int64)), NotImplementedError, "int64"),
    (dict(pred=np.zeros((1, 4, 6, 8), np.float64)), NotImplementedError, "float64"),
    (dict(spacing=(1.0, 0.0, 1.0)), ValueError, "positive and finite"),
    (dict(spacing=(1.0, float("nan"), 1.0)), ValueError, "positive and finite"),
    (dict(spacing=(1.0, float("inf"), 1.0)), ValueError, "positive and finite"),
    (dict(regions=[tuple(range(1, 10))]), NotImplementedError, "1 to 8"),
    (dict(regions=[1.5]), NotImplementedError, "integer labels"),
    (dict(ref=np.zeros((2, 4, 6, 8), np.uint8), pred=np.zeros((2, 4, 6, 8), np.uint8)), NotImplementedError,
     r"\(1, \*spatial\)"),
])
def test_rejections_before_any_launch(rec, kwargs, exc, match):
    ref = kwargs.get("ref", np.zeros((1, 4, 6, 8), np.uint8))
    pred = kwargs.get("pred", np.zeros((1, 4, 6, 8), np.uint8))
    with pytest.raises(exc, match=match):
        EV.compute_metrics_arrays(ref, pred, kwargs.get("regions", [1]), spacing=kwargs.get("spacing", (1.0, 1.0, 1.0)))
    assert rec.calls == []


def test_json_fix_matches_reference(ref_eval):
    recursive_fix_for_json_export = ref_eval.json_export.recursive_fix_for_json_export
    d = {np.int64(1): {"a": np.float64(0.5), "b": np.int64(3), "c": [np.float32(1.5), (np.int64(2), "x")],
                       "d": np.bool_(True), "e": float("nan")}, (1, 2): {"f": np.float16(2.0)}, "g": 1.0}
    want, got = copy.deepcopy(d), copy.deepcopy(d)
    recursive_fix_for_json_export(want)
    EV.fix_for_json_export(got)
    assert repr(got) == repr(want)


def test_golden_reproduces_from_generator():
    from oracle.make_golden_evaluation import golden_arrays
    arrays = golden_arrays()
    assert sorted(arrays) == sorted(GOLDEN.files)
    for k, v in arrays.items():
        assert v.dtype == GOLDEN[k].dtype and np.array_equal(v, GOLDEN[k], equal_nan=v.dtype.kind == "f"), k
