"""Ensembling on the device: the kernels against the reference's `merge_files` (tests/golden/ensemble_cases.npz,
oracle/make_golden_ensemble.py), the fp32 region threshold against torch's CPU sigmoid, `ensemble_folders` on files the
device export wrote against the oracle's `merge_files`, and one-pass `predict_ensemble_from_files` against predicting
every member with `save_probabilities` and then `ensemble_folders`."""
import os
import pickle
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import ensemble_oracle as EN

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "ensemble_cases.npz"))
PROB_ULP = 8


def _lm(C, regions):
    if regions:
        return SimpleNamespace(has_regions=True, regions_class_order=list(EN.REGION_ORDER), foreground_labels=[1, 2, 3],
                               num_segmentation_heads=C)
    return SimpleNamespace(has_regions=False, regions_class_order=None, foreground_labels=list(range(1, C)),
                           num_segmentation_heads=C)


def _device_ensemble(members, lm):
    from dinounet_b200 import ensembling as E
    from dinounet_b200 import lib as L
    lib = L.load()
    stream = torch.cuda.current_stream(DEV).cuda_stream
    acc = torch.empty(members[0].shape, dtype=torch.float32, device=DEV)
    for k, m in enumerate(members):
        E._accumulate(lib, acc, m, k == 0, stream)
    seg = E._segment(lib, acc, len(members), lm, stream)
    return acc.cpu().numpy(), seg


@pytest.mark.parametrize("case", EN.GOLDEN_CASES, ids=[c[0] for c in EN.GOLDEN_CASES])
def test_kernels_against_reference_golden(case):
    name, C, regions, dtypes, shape = case
    members = [GOLDEN[f"{name}_m{k}"] for k in range(len(dtypes))]
    assert [m.dtype for m in members] == [np.dtype(d) for d in dtypes]
    avg, seg = _device_ensemble(members, _lm(C, regions))
    want_avg, want_seg = GOLDEN[f"{name}_avg"], GOLDEN[f"{name}_seg"]
    assert np.array_equal(avg.view(np.int32), want_avg.view(np.int32))
    if regions:
        assert seg.dtype == np.uint8 and np.array_equal(seg, want_seg)
        return
    diff = seg.astype(np.int64) != want_seg
    ulps = EN.softmax_top2_ulps(want_avg)
    voxels = int(np.prod(shape))
    print(f"{name}: {int(diff.sum())} label differences of {voxels} voxels")
    assert (ulps[diff] <= PROB_ULP).all()
    assert int(diff.sum()) <= max(8, voxels // 10000)
    # the planted exact ties resolve to the first maximum
    flat = seg.reshape(-1)
    assert (flat[:8] == 0).all()


def test_fp32_region_threshold_against_torch_sigmoid():
    """Every fp32 value in [2^-30, 2^-18] as a one-member, one-region average: the label must be torch's CPU
    `sigmoid(x) > 0.5`."""
    lo = int(np.float32(2.0 ** -30).view(np.int32))
    hi = int(np.float32(2.0 ** -18).view(np.int32))
    lm = _lm(1, True)
    lm.regions_class_order = [1]
    lm.foreground_labels = [1]
    chunk = 1 << 24
    firsts = []
    for start in range(lo, hi + 1, chunk):
        x = np.arange(start, min(start + chunk, hi + 1), dtype=np.int32).view(np.float32)
        _, seg = _device_ensemble([x.reshape(1, -1)], lm)
        want = (torch.sigmoid(torch.from_numpy(x)) > 0.5).numpy()
        assert np.array_equal(seg.reshape(-1).astype(bool), want), f"chunk at {x[0]!r}"
        if want.any():
            firsts.append(x[np.argmax(want)])
    assert firsts[0] == np.nextafter(np.float32(1.5 * 2.0 ** -24), np.float32(1))


# ---------------------------------------------------------------------------------------------- ensemble_folders
class NpyIO:
    spacing = [3.0, 1.0, 1.0]

    def read_images(self, files):
        return np.stack([np.load(f) for f in files]).astype(np.float32), {"spacing": list(self.spacing)}

    def write_seg(self, seg, path, properties):
        np.save(path, seg)


def _export_managers(regions):
    from dinounet_b200 import export as EX
    conf = {"resampling_fn_probabilities": EX.DEFAULT_RESAMPLING_FN,
            "resampling_fn_probabilities_kwargs": dict(EX.DEFAULT_RESAMPLING_KWARGS)}
    cm = SimpleNamespace(spacing=[0.8, 0.8], configuration=conf)
    lm = _lm(3, regions)
    pm = SimpleNamespace(transpose_backward=[0, 2, 1], get_label_manager=lambda dj: lm, image_reader_writer_class=NpyIO,
                         plans={"plans_name": "test"})
    return pm, cm, lm


@pytest.mark.parametrize("regions", [False, True])
def test_ensemble_folders_on_device_export(tmp_path, monkeypatch, regions):
    from dinounet_b200 import ensembling as E
    from dinounet_b200 import export as EX
    from dinounet_b200 import predict as PR
    pm, cm, lm = _export_managers(regions)
    monkeypatch.setattr(PR, "_plans_manager", lambda plans: pm)
    dj = {"file_ending": ".npy", "labels": {"background": 0}}
    g = torch.Generator().manual_seed(5)
    cases = {"c1": ((3, 40, 50), (3, 52, 61), [[1, 4], [2, 54], [0, 61]], (5, 60, 61)),
             "c2": ((2, 30, 30), (2, 30, 30), [[0, 2], [0, 30], [3, 33]], (2, 30, 40))}
    folders = []
    for k in range(3):
        folder = tmp_path / f"member{k}"
        os.makedirs(folder)
        for case, (in_shape, after, bbox, before) in cases.items():
            logits = (torch.randn((3, *in_shape), generator=g) * 3).half()
            props = {"shape_after_cropping_and_before_resampling": list(after), "shape_before_cropping": list(before),
                     "bbox_used_for_cropping": bbox, "spacing": [3.0, 1.0, 1.0], "member": k}
            EX.export_prediction_from_logits(logits, props, cm, pm, dj, str(folder / case), True)
        (folder / "dataset.json").write_text('{"file_ending": ".npy", "labels": {"background": 0}}')
        (folder / "plans.json").write_text('{"plans_name": "test"}')
        folders.append(str(folder))
    out = tmp_path / "ens"
    E.ensemble_folders(folders, str(out), save_merged_probabilities=True, num_processes=2)
    assert (out / "dataset.json").is_file()
    for case in cases:
        files = [os.path.join(f, case + ".npz") for f in folders]
        EN.merge_files(files, str(tmp_path / ("oracle_" + case)), ".npy", NpyIO(), lm, True)
        want_p = np.load(tmp_path / f"oracle_{case}.npz")["probabilities"]
        got_p = np.load(out / f"{case}.npz")["probabilities"]
        assert np.array_equal(got_p.view(np.int32), want_p.view(np.int32))
        with open(out / f"{case}.pkl", "rb") as f:
            assert np.array_equal(pickle.load(f), want_p)         # the reference pickles the probabilities
        got, want = np.load(out / f"{case}.npy"), np.load(tmp_path / f"oracle_{case}.npy")
        if regions:
            assert np.array_equal(got, want)
        else:
            diff = got.astype(np.int64) != want
            assert (EN.softmax_top2_ulps(want_p)[diff] <= PROB_ULP).all()
            assert int(diff.sum()) <= max(8, got.size // 10000)


# ---------------------------------------------------------------------------------------------- one pass
def _model_folder(root, variant, folds):
    from oracle import dinounet_oracle as O
    os.makedirs(root)
    with open(os.path.join(root, "dataset.json"), "w") as f:
        f.write('{"channel_names": {"0": "CT", "1": "CT"}, "labels": {"background": 0}, "file_ending": ".npy"}')
    with open(os.path.join(root, "plans.json"), "w") as f:
        f.write('{"plans_name": "test"}')
    trainer = "DinoUNetTrainer_" + variant.split("_")[1]
    base = O.make_state_dict(variant, 3, seed=0)
    for k in range(folds):
        sd = {n: (t if ".dinov3_adapter.backbone." in n or not t.is_floating_point() or "running_var" in n
                  else t * (1 + 0.05 * k)) for n, t in base.items()}
        os.makedirs(os.path.join(root, f"fold_{k}"))
        torch.save({"network_weights": {"module." + n: t for n, t in sd.items()}, "trainer_name": trainer,
                    "init_args": {"configuration": "2d"}, "inference_allowed_mirroring_axes": (0, 1)},
                   os.path.join(root, f"fold_{k}", "checkpoint_final.pth"))


@pytest.mark.parametrize("regions", [False, True])
def test_predict_ensemble_from_files_equals_two_step_route(tmp_path, monkeypatch, regions):
    from dinounet_b200 import ensembling as E
    from dinounet_b200 import predict as PR
    from dinounet_b200.sliding_window import SlidingWindowPredictor
    from tests.test_gpu_predict_folds import CASES, _managers
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    pm, cm, lm = _managers(regions)
    monkeypatch.setattr(PR, "_plans_manager", lambda plans: pm)
    src = tmp_path / "in"
    os.makedirs(src)
    rng = np.random.default_rng(11)
    for case, shape in CASES:
        img = (rng.standard_normal((2, *shape)) * 30 + 40).astype(np.float32)
        for c in range(2):
            np.save(src / f"{case}_{c:04d}.npy", img[c])
    predictors = []
    for variant, folds in (("dinounet_s", 2), ("dinounet_b", 1)):
        model = str(tmp_path / variant)
        _model_folder(model, variant, folds)
        p = SlidingWindowPredictor(tile_step_size=0.5, device=DEV, tile_batch=4)
        p.initialize_from_trained_model_folder(model, None)
        assert len(p.list_of_parameters) == folds
        predictors.append(p)

    # the two-step route: every member with save_probabilities, then ensemble_folders
    members = []
    for k, p in enumerate(predictors):
        out = tmp_path / f"member{k}"
        p.predict_from_files(str(src), str(out), save_probabilities=True, num_processes_preprocessing=2,
                             num_processes_segmentation_export=2)
        members.append(str(out))
    two_step = tmp_path / "two_step"
    E.ensemble_folders(members, str(two_step), save_merged_probabilities=True, num_processes=2)

    one_pass = tmp_path / "one_pass"
    E.predict_ensemble_from_files(predictors, str(src), str(one_pass), save_probabilities=True,
                                  num_processes_preprocessing=2, num_processes_segmentation_export=2)
    again = tmp_path / "again"
    E.predict_ensemble_from_files(predictors, str(src), str(again), save_probabilities=True)
    for case, shape in CASES:
        want = np.load(two_step / f"{case}.npy")
        want_p = np.load(two_step / f"{case}.npz")["probabilities"]
        for folder in (one_pass, again):
            got = np.load(folder / f"{case}.npy")
            assert got.shape == shape and np.array_equal(got, want)
            got_p = np.load(folder / f"{case}.npz")["probabilities"]
            assert got_p.shape == want_p.shape and np.array_equal(got_p.view(np.int32), want_p.view(np.int32))
            with open(folder / f"{case}.pkl", "rb") as f:
                assert pickle.load(f)["spacing"] == list(NpyIO.spacing)
    for name in ("predict_from_raw_data_args.json", "dataset.json", "plans.json"):
        assert (one_pass / name).is_file()

    # without output names the segmentations and probabilities are returned
    res = E.predict_ensemble_from_files(predictors, str(src), None, save_probabilities=True)
    assert len(res) == len(CASES)
    for (case, _), (seg, probs) in zip(CASES, res):
        assert np.array_equal(seg, np.load(two_step / f"{case}.npy"))
        assert np.array_equal(probs.view(np.int32), np.load(two_step / f"{case}.npz")["probabilities"].view(np.int32))
