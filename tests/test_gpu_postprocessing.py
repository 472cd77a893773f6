"""Device postprocessing on the GPU (csrc/postprocessing.cu, dinounet_b200/postprocessing.py) against the oracle
(oracle/postprocessing_oracle.py: scipy.ndimage.label with full connectivity, acvl-utils' filter), the golden cases
(tests/golden/postprocessing_cases.npz) and, for the folder drop-ins, this module's folder logic run on the oracle (pinned
to the reference in tests/test_postprocessing_cpu.py)."""
import json
import os
import pickle
import shutil

import numpy as np
import pytest
import torch
from scipy import ndimage as ndi

from dinounet_b200 import evaluation as EV
from dinounet_b200 import postprocessing as PP
from oracle import evaluation_oracle as EO
from oracle import postprocessing_oracle as PO
from tests import test_postprocessing_cpu as CPU

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "postprocessing_cases.npz"))
DTYPES = [np.uint8, np.int8, np.int16, np.uint16, np.int32, np.float32]
SHAPES = [(1, 1, 1), (1, 7, 13), (5, 1, 9), (31, 1, 1), (31,), (1,), (13, 17), (61, 3), (7, 11, 37), (3, 37, 67),
          (9, 17, 97)]


def _check(seg, labels_or_regions, background=0):
    """Device and oracle outputs equal, for the numpy and the CUDA-tensor route; the input is left unchanged."""
    before = seg.copy()
    want = PO.remove_all_but_largest_component_from_segmentation(seg, labels_or_regions, background)
    got = PP.remove_all_but_largest_component_from_segmentation(seg, labels_or_regions, background)
    assert isinstance(got, np.ndarray) and got.dtype == seg.dtype and got.shape == seg.shape
    assert np.array_equal(got, want, equal_nan=seg.dtype.kind == "f")
    assert np.array_equal(seg, before, equal_nan=seg.dtype.kind == "f")
    t = torch.from_numpy(seg).cuda()
    got_t = PP.remove_all_but_largest_component_from_segmentation(t, labels_or_regions, background)
    assert got_t.is_cuda and got_t.device == t.device and got_t.data_ptr() != t.data_ptr()
    assert np.array_equal(got_t.cpu().numpy(), want, equal_nan=seg.dtype.kind == "f")
    assert np.array_equal(t.cpu().numpy(), before, equal_nan=seg.dtype.kind == "f")
    return want


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("shape", SHAPES, ids=str)
def test_dtypes_and_shapes(dtype, shape):
    for seed, density in enumerate([0.15, 0.3, 0.6]):
        seg = PO.random_mask_case(shape, density, seed + sum(shape), dtype)
        _check(seg, [1, 3], background=0)
        _check(seg, 2, background=5)


@pytest.mark.parametrize("density", [0.08, 0.12, 0.16, 0.2, 0.25, 0.3])
def test_percolation_densities(density):
    """Near the 26-connectivity percolation threshold: long branching components across many tiles."""
    seg = PO.random_mask_case((23, 45, 130), density, int(density * 100), np.uint8)
    kept = _check(seg, [1, 2, 3])
    assert (kept > 0).sum() > 0


def _corner_walk(shape, n, seed):
    """A random walk whose every step changes all three coordinates by one: one 26-component, many 6-components."""
    rng = np.random.default_rng(seed)
    p = np.array([s // 2 for s in shape])
    out = np.zeros(shape, np.uint8)
    for _ in range(n):
        out[tuple(p)] = 1
        step = rng.choice([-1, 1], 3)
        for d in range(3):
            if not 0 <= p[d] + step[d] < shape[d]:
                step[d] = -step[d]
        p = p + step
    return out


def test_edge_and_corner_connections_merge():
    seg = _corner_walk((21, 45, 150), 6000, 1)
    assert ndi.label(seg)[1] > 1   # face connectivity would split it
    assert ndi.label(seg, np.ones((3, 3, 3)))[1] == 1
    blob = np.zeros_like(seg)
    blob[0:3, 0:3, 0:3] = 2   # a separate smaller component of another label
    seg = np.where((seg == 0) & (blob > 0), blob, seg)
    assert np.array_equal(_check(seg, [1, 2]), PO.remove_all_but_largest_component_from_segmentation(seg, [1, 2]))
    # 2-D: diagonal (edge) steps only
    diag = np.zeros((40, 70), np.int16)
    for i in range(40):
        diag[i, i] = diag[i, 69 - i] = 1
    diag[5, 30] = 1
    _check(diag, 1)


def test_serpentine_crosses_every_tile():
    Z, Y, X = 9, 33, 97
    seg = np.zeros((Z, Y, X), np.uint8)
    for z in range(Z):
        for y in range(0, Y, 2):
            seg[z, y, :] = 1
            if y + 2 < Y:
                seg[z, y + 1, X - 1 if (y // 2) % 2 == 0 else 0] = 1
        if z + 1 < Z:
            seg[z, Y - 1, :] = 1   # the last row of a slice touches the next slice by its faces
    seg[::2, 1::2, 40] = 2
    assert ndi.label(seg > 0, np.ones((3, 3, 3)))[1] == 1
    _check(seg, 1)
    _check(seg, [1, 2])


def test_ties_empty_full_single():
    seg = np.zeros((10, 20, 40), np.uint8)
    seg[1:3, 1:4, 1:4] = 1
    seg[6:8, 12:15, 30:33] = 1
    seg[5, 5, 20] = 1
    got = _check(seg, 1)
    assert (got == 1).sum() == 36   # both tied components kept, the single voxel removed
    assert np.array_equal(_check(seg, 7), seg)                       # empty mask
    full = np.full((5, 9, 40), 3, np.int32)
    assert np.array_equal(_check(full, 3), full)
    single = np.zeros((4, 4, 4), np.float32)
    single[2, 1, 3] = 1.0
    assert np.array_equal(_check(single, 1), single)
    assert np.array_equal(_check(single, []), single)


def test_long_label_lists_regions_float_labels_and_out_of_range():
    seg = PO.random_mask_case((7, 19, 45), 0.35, 11, np.int16, labels=tuple(range(1, 26)))
    _check(seg, list(range(1, 21)))
    _check(seg, [(1, 2, 3), 9, (20, 21, 22, 23, 24, 25, 4, 5, 6, 7)])
    f = seg.astype(np.float32)
    f[0, 0, :5] = [16777216.0, np.nan, -0.0, 2.5, np.inf]
    _check(f, [16777217, 0, 3])          # 16777217 rounds to float32 16777216; -0.0 equals 0
    _check(f, [(2, 4), 16777216])
    u8 = PO.random_mask_case((5, 17, 40), 0.3, 12, np.uint8)
    _check(u8, [300, -1, 1])             # labels outside uint8 match nothing
    assert np.array_equal(_check(u8, [256, -255]), u8)
    i8 = PO.random_mask_case((5, 17, 40), 0.3, 13, np.int8, labels=(-3, 1, 2))
    _check(i8, [-3, 200])
    _check(i8, [(1, -3)], background=-128)


def test_golden_cases():
    for name, *_ in PO.GOLDEN_MASKS:
        seg, lr, bg = PO.golden_mask(name)
        assert np.array_equal(seg, GOLDEN[f"{name}_seg"])
        got = PP.remove_all_but_largest_component_from_segmentation(seg, lr, bg)
        assert np.array_equal(got, GOLDEN[f"{name}_out"]), name


def test_ct_scale_case():
    """One 200 x 512 x 512 uint8 case (tools/bench_postprocessing.py's seeded volume)."""
    from tools.bench_postprocessing import make_case
    seg = make_case((200, 512, 512))
    for lr in ([1, 2, 3], 3):
        want = PO.remove_all_but_largest_component_from_segmentation(seg, lr)
        got = PP.remove_all_but_largest_component_from_segmentation(torch.from_numpy(seg).cuda(), lr)
        assert np.array_equal(got.cpu().numpy(), want)


def test_repeat_calls_are_identical():
    seg = torch.from_numpy(PO.random_mask_case((31, 64, 200), 0.22, 3, np.uint8)).cuda()
    first = PP.remove_all_but_largest_component_from_segmentation(seg, [1, 2, 3])
    for _ in range(3):
        assert torch.equal(PP.remove_all_but_largest_component_from_segmentation(seg, [1, 2, 3]), first)


# ---- folders


@pytest.mark.parametrize("name", PO.SCENARIOS)
def test_determine_and_apply_postprocessing_on_device(name, tmp_path, monkeypatch, capsys):
    """Device run and the module's folder logic on the oracle (CPU) write the same bytes: messages, postprocessing.json,
    the postprocessed/ folder with its summary (HD95 included, spacing (2, 1, 1)); the pkl holds the oracle's decisions
    and round-trips through pickle and apply_postprocessing_to_folder."""
    scenario = PO.make_scenario(name)
    plans = CPU._plans(scenario)
    monkeypatch.setattr(PP, "_plans_manager", lambda p: plans)
    root = str(tmp_path / "run")
    runs = {}
    for who in ("device", "oracle"):
        if os.path.isdir(root):
            shutil.rmtree(root)
        pred_dir, ref_dir = CPU._write_scenario(root, scenario)
        with monkeypatch.context() as m:
            if who == "oracle":
                m.setattr(PP, "remove_all_but_largest_component_from_segmentation",
                          CPU.remove_all_but_largest_component_from_segmentation)
                m.setattr(PP, "_upload", lambda seg: seg)
                m.setattr(EV, "compute_metrics_arrays", EO.compute_metrics_arrays)
            capsys.readouterr()
            ret = PP.determine_postprocessing(pred_dir, ref_dir, {"plans": 1}, {"file_ending": ".npy"}, 2, True)
            printed = capsys.readouterr().out
        with open(os.path.join(pred_dir, "postprocessing.pkl"), "rb") as f:
            pkl = pickle.load(f)
        files = CPU._snapshot(pred_dir)
        del files["postprocessing.pkl"]
        runs[who] = (ret, printed, pkl, files)
    (ret_d, printed_d, pkl_d, files_d), (ret_o, printed_o, pkl_o, files_o) = runs["device"], runs["oracle"]
    assert printed_d == printed_o
    assert sorted(files_d) == sorted(files_o)
    for k in files_o:
        assert files_d[k] == files_o[k], k
    accepted, final, _, final_summary = PO.run_scenario(name)
    assert repr(pkl_d[1]) == repr(accepted) == str(GOLDEN[f"{name}_accepted"])
    assert all(fn is PP.remove_all_but_largest_component_from_segmentation for fn in pkl_d[0])
    summary = json.loads(files_d[os.path.join("postprocessed", "summary.json")])
    assert summary["foreground_mean"]["Dice"] == final_summary["foreground_mean"]["Dice"] == GOLDEN[f"{name}_fg_dice"]
    for i, (f, _, _) in enumerate(scenario["cases"]):
        if accepted:
            assert np.array_equal(np.load(os.path.join(root, "pred", "postprocessed", f)), final[i])
        assert np.array_equal(final[i], GOLDEN[f"{name}_final{i}"])

    # the pkl through apply_postprocessing_to_folder, and a reference-named function routed to the device one
    pred_dir = os.path.join(root, "pred")
    PP.apply_postprocessing_to_folder(pred_dir, str(tmp_path / "applied"), *pkl_d, {"plans": 1}, {"file_ending": ".npy"},
                                      3)
    for i, (f, _, _) in enumerate(scenario["cases"]):
        assert np.array_equal(np.load(str(tmp_path / "applied" / f)), final[i])

    def remove_all_but_largest_component_from_segmentation(*a, **k):
        raise AssertionError("the reference's function must run through the device one")

    remove_all_but_largest_component_from_segmentation.__module__ = PP.REFERENCE_MODULE
    PP.apply_postprocessing_to_folder(pred_dir, str(tmp_path / "applied_ref"),
                                      [remove_all_but_largest_component_from_segmentation] * len(pkl_d[1]), pkl_d[1],
                                      {"plans": 1}, {"file_ending": ".npy"}, 1)
    assert CPU._snapshot(str(tmp_path / "applied_ref")) == CPU._snapshot(str(tmp_path / "applied"))
