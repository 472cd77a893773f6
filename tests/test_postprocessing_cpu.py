"""Device postprocessing without a GPU: the oracle (oracle/postprocessing_oracle.py) and this package's folder logic
against the reference's own `remove_connected_components` module on .npy folders, the rejections (before any launch)
and the C-ABI call (recording stand-in for the native library), and the golden file
(tests/golden/postprocessing_cases.npz, oracle/make_golden_postprocessing.py)."""
import contextlib
import ctypes
import importlib
import json
import os
import pickle
import shutil
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dinounet_b200 import evaluation as EV
from dinounet_b200 import postprocessing as PP
from oracle import evaluation_oracle as EO
from oracle import postprocessing_oracle as PO

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "postprocessing_cases.npz"))


def remove_all_but_largest_component_from_segmentation(segmentation, labels_or_regions, background_label=0):
    """The oracle in the device function's place (module level, so a pkl can name it)."""
    if isinstance(segmentation, torch.Tensor):
        segmentation = segmentation.numpy()
    return PO.remove_all_but_largest_component_from_segmentation(segmentation, labels_or_regions, background_label)


class _NpyRW:
    """A reader-writer on .npy files: read_seg gives (1, *spatial) and a fixed spacing."""

    def read_seg(self, path):
        return np.load(path), {"spacing": (2.0, 1.0, 1.0)}

    def write_seg(self, seg, path, props):
        np.save(path, seg[None])


class _SerialPool:
    def __init__(self, n):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False

    def starmap(self, fn, args):
        return [fn(*a) for a in args]


def _plans(scenario):
    lm = SimpleNamespace(has_regions=scenario["regions"] is not None, foreground_regions=scenario["regions"],
                         foreground_labels=list(scenario["foreground_labels"]), ignore_label=scenario["ignore_label"])
    return SimpleNamespace(image_reader_writer_class=_NpyRW, get_label_manager=lambda dj: lm)


def _write_scenario(root, scenario):
    pred_dir, ref_dir = os.path.join(root, "pred"), os.path.join(root, "gt")
    os.makedirs(pred_dir)
    os.makedirs(ref_dir)
    for f, ref, pred in scenario["cases"]:
        np.save(os.path.join(ref_dir, f), ref)
        np.save(os.path.join(pred_dir, f), pred)
    with open(os.path.join(pred_dir, "notes.txt"), "w") as fh:
        fh.write("not a case")
    if scenario["existing_summary"]:
        with open(os.path.join(pred_dir, "summary.json"), "w") as fh:
            fh.write(PO.existing_summary_text(scenario))
    return pred_dir, ref_dir


def _snapshot(folder):
    out = {}
    for dirpath, _, files in os.walk(folder):
        for f in files:
            p = os.path.join(dirpath, f)
            with open(p, "rb") as fh:
                out[os.path.relpath(p, folder)] = fh.read()
    return out


_SHIM_ROOTS = {"dinounet", "dinounet_training", "dynamic_network_architectures", "MultiScaleDeformableAttention"}


@pytest.fixture(scope="module")
def ref_pp():
    from oracle import ref_loader, ref_predictor_loader
    if not ref_loader.reference_available():
        pytest.skip("reference sources not present")
    # stand-ins that other tests left for the same names are set aside while the reference loads, then restored
    theirs = {m: sys.modules.pop(m) for m in list(sys.modules)
              if m.split(".")[0] in ref_predictor_loader._STUB_ROOTS | _SHIM_ROOTS}
    roots, meta_path, path = {m.split(".")[0] for m in sys.modules}, list(sys.meta_path), list(sys.path)
    try:
        ref_predictor_loader.load_reference_predictor_class()
        mod = importlib.import_module("dinounet.postprocessing.remove_connected_components")
        ev = importlib.import_module("dinounet.evaluation.evaluate_predictions")
    finally:
        loaded = {name: sys.modules.pop(name) for name in [m for m in sys.modules if m.split(".")[0] not in roots]}
        sys.meta_path[:], sys.path[:] = meta_path, path
        sys.modules.update(theirs)
    return SimpleNamespace(module=mod, evaluate_predictions=ev,
                           packages={k: v for k, v in loaded.items() if k.split(".")[0] == "dinounet"})


def _load_json(file):
    with open(file) as f:
        return json.load(f)


def _save_json(obj, file, indent=4, sort_keys=True):
    with open(file, "w") as f:
        json.dump(obj, f, sort_keys=sort_keys, indent=indent)


def _save_pickle(obj, file, mode="wb"):
    with open(file, mode) as f:
        pickle.dump(obj, f)


@pytest.fixture
def patched_reference(ref_pp, monkeypatch):
    """The reference module with the oracle for acvl-utils, a serial pool, batchgenerators' file helpers, and this
    package's folder scoring (pinned to the reference's in tests/test_evaluation_cpu.py) fed by the CPU metrics oracle."""
    m = ref_pp.module
    for name, mod in ref_pp.packages.items():   # so that pickle can name the reference's function
        monkeypatch.setitem(sys.modules, name, mod)
    monkeypatch.setattr(m, "remove_all_but_largest_component", PO.remove_all_but_largest_component)
    monkeypatch.setattr(m, "multiprocessing", SimpleNamespace(get_context=lambda k: SimpleNamespace(Pool=_SerialPool)))
    monkeypatch.setattr(m, "subfiles", lambda folder, suffix=None, join=True:
                        [f if not join else os.path.join(folder, f) for f in EV._subfiles(folder, suffix or "")])
    for name, fn in [("isfile", os.path.isfile), ("isdir", os.path.isdir), ("join", os.path.join),
                     ("maybe_mkdir_p", lambda p: os.makedirs(p, exist_ok=True)), ("load_json", _load_json),
                     ("save_json", _save_json), ("save_pickle", _save_pickle),
                     ("compute_metrics_on_folder", EV.compute_metrics_on_folder)]:
        monkeypatch.setattr(m, name, fn)
    monkeypatch.setattr(ref_pp.evaluate_predictions, "load_json", _load_json)
    monkeypatch.setattr(EV, "compute_metrics_arrays", EO.compute_metrics_arrays)
    return m


@pytest.fixture
def cpu_module(monkeypatch):
    """This package's module with the oracle in the device function's place, host arrays instead of uploads and the CPU
    metrics oracle: what remains is its folder logic."""
    monkeypatch.setattr(PP, "remove_all_but_largest_component_from_segmentation",
                        remove_all_but_largest_component_from_segmentation)
    monkeypatch.setattr(PP, "_upload", lambda seg: seg)
    monkeypatch.setattr(EV, "compute_metrics_arrays", EO.compute_metrics_arrays)
    return PP


@pytest.mark.parametrize("name", PO.SCENARIOS)
def test_determine_postprocessing_equals_reference(name, tmp_path, patched_reference, cpu_module, monkeypatch,
                                                  capsys):
    """Same messages, decisions, pkl contents, postprocessing.json and postprocessed/ folder (every byte, case paths in
    the summaries included) as the reference, and the oracle's decisions and arrays."""
    scenario = PO.make_scenario(name)
    root = str(tmp_path / "run")
    plans = _plans(scenario)
    monkeypatch.setattr(patched_reference, "PlansManager", lambda p: plans)
    monkeypatch.setattr(PP, "_plans_manager", lambda p: plans)
    dataset_json = {"file_ending": ".npy"}
    runs = {}
    for who, fn in [("reference", patched_reference.determine_postprocessing),
                    ("module", cpu_module.determine_postprocessing)]:
        if os.path.isdir(root):
            shutil.rmtree(root)
        pred_dir, ref_dir = _write_scenario(root, scenario)
        capsys.readouterr()
        ret = fn(pred_dir, ref_dir, {"plans": 1}, dataset_json, 2, True)
        printed = capsys.readouterr().out
        with open(os.path.join(pred_dir, "postprocessing.pkl"), "rb") as f:
            pkl = pickle.load(f)
        files = _snapshot(pred_dir)
        del files["postprocessing.pkl"]
        runs[who] = (ret, printed, pkl, files)
    (ret_r, printed_r, pkl_r, files_r), (ret_m, printed_m, pkl_m, files_m) = runs["reference"], runs["module"]
    assert printed_m == printed_r
    assert repr(ret_m[1]) == repr(ret_r[1])
    assert repr(pkl_m[1]) == repr(pkl_r[1])
    assert [f.__name__ for f in pkl_m[0]] == [f.__name__ for f in pkl_r[0]]
    assert sorted(files_m) == sorted(files_r)
    for k in files_r:
        assert files_m[k] == files_r[k], k

    accepted, final, _, final_summary = PO.run_scenario(name)
    assert repr(pkl_r[1]) == repr(accepted)
    for (f, _, _), want in zip(scenario["cases"], final):
        got = np.load(os.path.join(root, "pred", "postprocessed", f)) if accepted else want
        assert got.dtype == want.dtype and np.array_equal(got, want)
    summary = json.loads(files_r[os.path.join("postprocessed", "summary.json")])
    assert summary["foreground_mean"]["Dice"] == final_summary["foreground_mean"]["Dice"]


def test_scenarios_cover_the_decisions():
    """(a) foreground step accepted, (b) rejected with a better mean but one label worse, (c) per-label steps accepted
    and rejected, (d) overlapping regions, (e) a pre-existing summary.json, (f) tied largest components kept."""
    outcomes = {n: PO.run_scenario(n) for n in PO.SCENARIOS}
    assert [k["labels_or_regions"] for k in outcomes["fg_accepted"][0]] == [[1, 2], 2]
    acc, _, base, _ = outcomes["fg_rejected_one_label_worse"]
    assert [k["labels_or_regions"] for k in acc] == [1]
    s = PO.make_scenario("fg_rejected_one_label_worse")
    cases = [(ref, pred) for _, ref, pred in s["cases"]]
    fg = PO._aggregate([EO.compute_metrics_arrays(ref, PO.remove_all_but_largest_component_from_segmentation(
        pred[0], [1, 2])[None], [1, 2], None, s["spacing"]) for ref, pred in cases], [1, 2])
    assert fg["foreground_mean"]["Dice"] > base["foreground_mean"]["Dice"] and fg["mean"][2]["Dice"] < base["mean"][2]["Dice"]
    assert [k["labels_or_regions"] for k in outcomes["regions_overlapping"][0]] == [(1, 2), (2,)]
    assert outcomes["existing_summary"][0] == []
    acc, final, _, _ = outcomes["tied_components"]
    assert acc == [{"labels_or_regions": [1]}]
    for (_, ref, _), got in zip(PO.make_scenario("tied_components")["cases"], final):
        assert np.array_equal(got, ref.astype(np.uint8))   # both tied boxes kept, the blob removed


def test_reference_pkl_applies_through_this_module(tmp_path, patched_reference, cpu_module, monkeypatch):
    """A postprocessing.pkl written by the reference, applied by apply_postprocessing_to_folder: the reference's
    function is replaced by this module's, and the files equal the reference's own application."""
    scenario = PO.make_scenario("fg_rejected_one_label_worse")
    plans = _plans(scenario)
    monkeypatch.setattr(patched_reference, "PlansManager", lambda p: plans)
    monkeypatch.setattr(PP, "_plans_manager", lambda p: plans)
    pred_dir, ref_dir = _write_scenario(str(tmp_path), scenario)
    patched_reference.determine_postprocessing(pred_dir, ref_dir, {}, {"file_ending": ".npy"}, 2, False)
    with open(os.path.join(pred_dir, "postprocessing.pkl"), "rb") as f:
        fns, kwargs = pickle.load(f)
    assert fns and all(fn.__module__ == PP.REFERENCE_MODULE for fn in fns)
    assert all(PP._resolve(fn) is cpu_module.remove_all_but_largest_component_from_segmentation for fn in fns)
    patched_reference.apply_postprocessing_to_folder(pred_dir, str(tmp_path / "ref_out"), fns, kwargs, {},
                                                     {"file_ending": ".npy"}, 2)
    PP.apply_postprocessing_to_folder(pred_dir, str(tmp_path / "new_out"), fns, kwargs, {}, {"file_ending": ".npy"}, 2)
    assert _snapshot(str(tmp_path / "ref_out")) == _snapshot(str(tmp_path / "new_out"))


def test_summary_json_helpers_match_reference(ref_pp, tmp_path):
    ev = ref_pp.evaluate_predictions
    for key in ["3", "(1, 2)", "(2,)", "-4"]:
        assert EV.key_to_label_or_region(key) == ev.key_to_label_or_region(key)
    s = PO.make_scenario("regions_overlapping")
    path = str(tmp_path / "summary.json")
    with open(path, "w") as f:
        f.write(PO.existing_summary_text(s))
    want = _load_json(path)
    want["mean"] = {ev.key_to_label_or_region(k): v for k, v in want["mean"].items()}
    for c in want["metric_per_case"]:
        c["metrics"] = {ev.key_to_label_or_region(k): v for k, v in c["metrics"].items()}
    assert repr(EV.load_summary_json(path)) == repr(want)


# ---- the oracle's labelling against an independent flood fill


def _flood_fill_keep(mask):
    """Keep-the-largest by breadth-first search over the 3**ndim - 1 neighbours."""
    from collections import deque
    comp = -np.ones(mask.shape, np.int64)
    sizes = []
    offsets = [o for o in np.ndindex(*(3,) * mask.ndim) if any(v != 1 for v in o)]
    for start in zip(*np.nonzero(mask)):
        if comp[start] >= 0:
            continue
        comp[start] = len(sizes)
        q, n = deque([start]), 0
        while q:
            p = q.popleft()
            n += 1
            for o in offsets:
                nb = tuple(p[d] + o[d] - 1 for d in range(mask.ndim))
                if all(0 <= nb[d] < mask.shape[d] for d in range(mask.ndim)) and mask[nb] and comp[nb] < 0:
                    comp[nb] = len(sizes)
                    q.append(nb)
        sizes.append(n)
    if not sizes:
        return np.zeros_like(mask)
    best = max(sizes)
    return np.isin(comp, [i for i, s in enumerate(sizes) if s == best])


@pytest.mark.parametrize("shape,density", [((7,), 0.5), ((9, 13), 0.35), ((5, 7, 9), 0.2), ((4, 9, 11), 0.12),
                                           ((1, 1, 1), 1.0), ((3, 4, 5), 0.0)])
def test_oracle_keeps_what_a_flood_fill_keeps(shape, density):
    rng = np.random.default_rng(len(shape) * 100 + int(density * 100))
    for _ in range(3):
        mask = rng.random(shape) < density
        assert np.array_equal(PO.remove_all_but_largest_component(mask), _flood_fill_keep(mask))


# ---- argument contract and call sequence (recording stand-in for the native library)


class _Recorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*a):
            labels = list((ctypes.c_int64 * a[6]).from_address(a[5])) if a[6] else []
            self.calls.append((name, a, labels))
            if name == "b2u_pp_largest_component":
                ctypes.memmove(a[8], a[0], a[2] * a[3] * a[4] * _ITEMSIZE[a[1]])
            return 0
        return fn


_ITEMSIZE = {0: 1, 1: 1, 2: 2, 3: 2, 4: 4, 5: 4}


@pytest.fixture
def rec(monkeypatch):
    from dinounet_b200 import lib as L
    r = _Recorder()
    monkeypatch.setattr(L, "load", lambda: r)
    monkeypatch.setattr(EV, "_device", lambda ref, pred: torch.device("cpu"))
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda dev=None: SimpleNamespace(cuda_stream=0))
    return r


def test_call_sequence(rec):
    """One call per segmentation: the stored dtype, the shape padded to [Z, Y, X], the distinct label values of every
    label and region in ascending order, the background in the dtype's bits, and 2 n + 1 int32 of scratch."""
    seg = np.zeros((6, 7), np.int16)
    out = PP.remove_all_but_largest_component_from_segmentation(seg, [(5, 3), 9, 3, np.int64(-2)], background_label=-1)
    assert isinstance(out, np.ndarray) and out.dtype == np.int16 and out.shape == (6, 7)
    (name, a, labels), = rec.calls
    assert name == "b2u_pp_largest_component"
    assert (a[1], a[2:5], labels, a[6], a[7]) == (2, (1, 6, 7), [-2, 3, 5, 9], 4, 0xFFFF)
    rec.calls.clear()
    t = torch.zeros(11, dtype=torch.float32)
    got = PP.remove_all_but_largest_component_from_segmentation(t, 2, background_label=7)
    assert isinstance(got, torch.Tensor) and got.data_ptr() != t.data_ptr()
    (_, a, labels), = rec.calls
    assert (a[1], a[2:5], labels, a[7]) == (5, (1, 1, 11), [2], int(np.float32(7).view(np.uint32)))
    rec.calls.clear()
    PP.remove_all_but_largest_component_from_segmentation(np.zeros((2, 3, 4), np.uint8), [])
    assert rec.calls[0][1][6] == 0
    rec.calls.clear()
    assert PP.remove_all_but_largest_component_from_segmentation(np.zeros((0, 3), np.uint8), 1).shape == (0, 3)
    assert rec.calls == []


def test_apply_postprocessing_keeps_one_upload(rec, monkeypatch):
    """A chain of this module's function stays a tensor between steps; a foreign function receives numpy."""
    seen = []

    def other(seg, k):
        seen.append((type(seg), k))
        return seg

    seg = torch.zeros(3, 4, dtype=torch.uint8)
    out = PP.apply_postprocessing(seg, [PP.remove_all_but_largest_component_from_segmentation, other],
                                  [{"labels_or_regions": 1}, {"k": 5}])
    assert seen == [(np.ndarray, 5)] and isinstance(out, np.ndarray) and len(rec.calls) == 1


@pytest.mark.parametrize("seg,labels,background,exc,match", [
    (np.zeros((1, 2, 3, 4), np.uint8), 1, 0, NotImplementedError, "rank 4"),
    (np.zeros((), np.uint8), 1, 0, NotImplementedError, "rank 0"),
    (torch.zeros(1, dtype=torch.uint8).expand(2 ** 31), 1, 0, NotImplementedError, "2\\^31"),
    (np.zeros((3, 4), np.int64), 1, 0, NotImplementedError, "int64"),
    (np.zeros((3, 4), np.float64), 1, 0, NotImplementedError, "float64"),
    (np.zeros((3, 4), np.uint8), 1.5, 0, NotImplementedError, "integer labels"),
    (np.zeros((3, 4), np.uint8), [(1, True)], 0, NotImplementedError, "integer labels"),
    (np.zeros((3, 4), np.uint8), 2 ** 64, 0, NotImplementedError, "int64"),
    (np.zeros((3, 4), np.uint8), 1, 300, OverflowError, "uint8"),
    (np.zeros((3, 4), np.uint8), 1, -1, OverflowError, "uint8"),
    (np.zeros((3, 4), np.int16), 1, 2 ** 15, OverflowError, "int16"),
])
def test_rejections_before_any_launch(rec, seg, labels, background, exc, match):
    with pytest.raises(exc, match=match):
        PP.remove_all_but_largest_component_from_segmentation(seg, labels, background)
    assert rec.calls == []


def test_golden_reproduces_from_generator():
    from oracle.make_golden_postprocessing import golden_arrays
    arrays = golden_arrays()
    assert sorted(arrays) == sorted(GOLDEN.files)
    for k, v in arrays.items():
        assert v.dtype == GOLDEN[k].dtype and np.array_equal(v, GOLDEN[k], equal_nan=v.dtype.kind == "f"), k
