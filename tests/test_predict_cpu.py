"""Model-folder prediction without a GPU: reading a trained model folder, fold detection, the trainer-name and
architecture mapping, splitting the cases between parts, output naming, the argument / dataset / plans JSON files, the
backbone check that picks the fold-ensemble route, and the rejections."""
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dinounet_b200 import config
from dinounet_b200 import predict as PR
from dinounet_b200.sliding_window import backbones_identical

CM = SimpleNamespace(network_arch_class_name="dinounet_b200.DinoUNet", network_arch_init_kwargs=dict(config.DEFAULT_ARCHITECTURE),
                     batch_size=12, patch_size=[512, 512], spacing=[0.7, 0.7], median_image_size_in_voxels=[512, 512],
                     previous_stage_name=None)


def _folder(root, folds, trainer="DinoUNetTrainer_l", with_ckpt=None):
    os.makedirs(root, exist_ok=True)
    with open(os.path.join(root, "dataset.json"), "w") as f:
        json.dump({"channel_names": {"0": "CT"}, "labels": {"background": 0, "a": 1}, "file_ending": ".nii.gz"}, f)
    with open(os.path.join(root, "plans.json"), "w") as f:
        json.dump({"plans_name": "p", "configurations": {"2d": {}}}, f)
    for k in folds:
        d = os.path.join(root, f"fold_{k}")
        os.makedirs(d, exist_ok=True)
        if with_ckpt is None or k in with_ckpt:
            torch.save({"network_weights": {"w": torch.full((2,), float(k if k != "all" else -1))}, "trainer_name": trainer,
                        "init_args": {"configuration": "2d"}, "inference_allowed_mirroring_axes": (0, 1)},
                       os.path.join(d, "checkpoint_final.pth"))


@pytest.fixture
def plans(monkeypatch):
    seen = []

    def pm(plans):
        seen.append(plans)
        return SimpleNamespace(plans=plans, get_configuration=lambda name: (CM if name == "2d" else None))
    monkeypatch.setattr(PR, "_plans_manager", pm)
    return seen


def test_model_folder_auto_detects_folds(tmp_path, plans):
    root = str(tmp_path / "m")
    _folder(root, [0, 2, 3, "all"], with_ckpt=[0, 2, "all"])
    assert PR.auto_detect_available_folds(root, "checkpoint_final.pth") == [0, 2]
    pm, cm, dj, params, trainer, conf, axes = PR.load_model_folder(root, None)
    assert [float(p["w"][0]) for p in params] == [0.0, 2.0]
    assert trainer == "DinoUNetTrainer_l" and conf == "2d" and tuple(axes) == (0, 1) and cm is CM
    assert dj["file_ending"] == ".nii.gz" and plans[0]["plans_name"] == "p"
    _, _, _, params, *_ = PR.load_model_folder(root, "all")
    assert [float(p["w"][0]) for p in params] == [-1.0]
    _, _, _, params, *_ = PR.load_model_folder(root, (2, "0"))
    assert [float(p["w"][0]) for p in params] == [2.0, 0.0]


def test_model_folder_rejects_missing_fold(tmp_path, plans):
    root = str(tmp_path / "m")
    _folder(root, [0, 3], with_ckpt=[0])
    with pytest.raises(FileNotFoundError):
        PR.load_model_folder(root, (0, 3))
    with pytest.raises(FileNotFoundError):
        PR.load_model_folder(root, (1,))
    empty = str(tmp_path / "e")
    _folder(empty, [])
    with pytest.raises(FileNotFoundError):
        PR.load_model_folder(empty, None)


@pytest.mark.parametrize("trainer,variant", [("DinoUNetTrainer_s", "dinounet_s"), ("DinoUNetTrainer_b", "dinounet_b"),
                                             ("DinoUNetTrainer_l", "dinounet_l"), ("DinoUNetTrainer_7b", "dinounet_7b")])
def test_trainer_name_to_variant(trainer, variant):
    assert PR.variant_from_trainer_name(trainer) == variant


@pytest.mark.parametrize("name", ["nnUNetTrainer", "DinoUNetTrainer", "DinoUNetTrainer_xl", ""])
def test_unknown_trainer_raises(name):
    with pytest.raises(ValueError):
        PR.variant_from_trainer_name(name)


def test_architecture_mapping_follows_api():
    """dinounet/api.py:91-110 builds the trainers' network_config from the plans' arch_kwargs with these defaults."""
    got = PR.network_config_from_configuration(CM)
    a = config.DEFAULT_ARCHITECTURE
    assert got["architecture"] == {
        "network_class_name": "dinounet_b200.DinoUNet", "n_stages": a["n_stages"],
        "features_per_stage": a["features_per_stage"], "kernel_sizes": a["kernel_sizes"], "strides": a["strides"],
        "n_conv_per_stage": a["n_conv_per_stage"], "n_conv_per_stage_decoder": a["n_conv_per_stage_decoder"],
        "conv_op": a["conv_op"], "norm_op": a["norm_op"], "nonlin": a["nonlin"], "conv_bias": a["conv_bias"],
        "dropout_op": a["dropout_op"], "norm_op_kwargs": a["norm_op_kwargs"], "nonlin_kwargs": a["nonlin_kwargs"],
        "dropout_op_kwargs": a["dropout_op_kwargs"]}
    assert got["data_config"] == {"batch_size": 12, "patch_size": [512, 512], "spacing": [0.7, 0.7],
                                  "median_image_size_in_voxels": [512, 512]}
    bare = PR.network_config_from_configuration(SimpleNamespace(network_arch_class_name=None, network_arch_init_kwargs={}))
    assert bare["architecture"]["n_stages"] == 0 and bare["architecture"]["conv_bias"] is True
    assert bare["architecture"]["conv_op"] == "" and bare["architecture"]["dropout_op"] is None


def test_build_network_needs_no_pretrained_file(monkeypatch):
    monkeypatch.delenv("DINOUNET_B200_ALLOW_RANDOM_BACKBONE", raising=False)
    net = PR.build_network("DinoUNetTrainer_s", CM, 1, 4)
    assert net.dinov3_model_name == "dinounet_s" and net.num_classes == 4
    assert not net.decoder.deep_supervision
    assert list(net.encoder.target_channels) == list(config.DEFAULT_ARCHITECTURE["features_per_stage"])
    with pytest.raises(ValueError):
        PR.build_network("SomeOtherTrainer", CM, 1, 4)


def _cases(folder, names, channels=2, ending=".nii.gz"):
    os.makedirs(folder, exist_ok=True)
    for n in names:
        for c in range(channels):
            open(os.path.join(folder, f"{n}_{c:04d}{ending}"), "w").close()
    open(os.path.join(folder, "notes.txt"), "w").close()


def test_case_lists_parts_and_output_names(tmp_path):
    src, out = str(tmp_path / "in"), str(tmp_path / "out")
    names = ["c3", "c1", "c2", "c5", "c4"]
    _cases(src, names)
    lists = PR.create_lists_from_splitted_dataset_folder(src, ".nii.gz")
    assert [os.path.basename(l[0]) for l in lists] == [f"c{i}_0000.nii.gz" for i in range(1, 6)]
    assert all(len(l) == 2 and l[1].endswith("_0001.nii.gz") for l in lists)
    seen = []
    for part in range(2):
        lst, outs = PR.manage_input_and_output_lists(src, out, ".nii.gz", True, part, 2)
        assert outs == [os.path.join(out, os.path.basename(l[0])[:-12]) for l in lst]
        seen += [os.path.basename(o) for o in outs]
    assert seen == ["c1", "c3", "c5", "c2", "c4"]
    # overwrite=False drops the finished cases; with probabilities the .npz must exist too
    os.makedirs(out)
    open(os.path.join(out, "c1.nii.gz"), "w").close()
    open(os.path.join(out, "c2.nii.gz"), "w").close()
    open(os.path.join(out, "c2.npz"), "w").close()
    _, outs = PR.manage_input_and_output_lists(src, out, ".nii.gz", False, 0, 1)
    assert [os.path.basename(o) for o in outs] == ["c3", "c4", "c5"]
    _, outs = PR.manage_input_and_output_lists(src, out, ".nii.gz", False, 0, 1, save_probabilities=True)
    assert [os.path.basename(o) for o in outs] == ["c1", "c3", "c4", "c5"]
    # explicit truncated names are kept as given
    lst, outs = PR.manage_input_and_output_lists(lists[:2], ["/x/a", "/x/b"], ".nii.gz")
    assert outs == ["/x/a", "/x/b"] and lst == lists[:2]


def _predictor_stub(previous_stage=None):
    cm = SimpleNamespace(previous_stage_name=previous_stage)
    return SimpleNamespace(dataset_json={"file_ending": ".nii.gz", "labels": {"b": 0}, "name": "z"},
                           plans_manager=SimpleNamespace(plans={"b": 1, "a": [1, 2]}), configuration_manager=cm)


def test_predict_from_files_writes_the_three_json_files(tmp_path):
    src, out = str(tmp_path / "in"), str(tmp_path / "out")
    _cases(src, ["c1", "c2"])
    os.makedirs(out)
    for n in ("c1", "c2"):
        open(os.path.join(out, n + ".nii.gz"), "w").close()
    p = _predictor_stub()
    # every case is finished, so nothing is predicted
    assert PR.predict_from_files(p, src, out, overwrite=False, num_parts=1, part_id=0) is None
    with open(os.path.join(out, "predict_from_raw_data_args.json")) as f:
        args = json.load(f)
    assert args == {"list_of_lists_or_source_folder": src, "output_folder_or_list_of_truncated_output_files": out,
                    "save_probabilities": False, "overwrite": False, "num_processes_preprocessing": 3,
                    "num_processes_segmentation_export": 3, "folder_with_segs_from_prev_stage": None, "num_parts": 1,
                    "part_id": 0}
    with open(os.path.join(out, "dataset.json")) as f:
        assert json.load(f) == p.dataset_json
    with open(os.path.join(out, "plans.json")) as f:
        text = f.read()
    assert json.loads(text) == p.plans_manager.plans and text.index('"b"') < text.index('"a"')   # key order kept


def test_cascade_raises_before_anything_runs(tmp_path):
    out = str(tmp_path / "out")
    with pytest.raises(NotImplementedError):
        PR.predict_from_files(_predictor_stub(), str(tmp_path), out, folder_with_segs_from_prev_stage=str(tmp_path))
    with pytest.raises(NotImplementedError):
        PR.predict_from_files(_predictor_stub("3d_lowres"), str(tmp_path), out)
    assert not os.path.exists(out)
    with pytest.raises(NotImplementedError):
        PR.predict_from_list_of_npy_arrays(_predictor_stub(), [None], np.zeros((1, 2, 2, 2)), [{}], None)
    with pytest.raises(NotImplementedError):
        PR.predict_from_list_of_npy_arrays(_predictor_stub(), [None, None], [None, np.zeros((1, 2, 2, 2))], [{}, {}], None)
    # a list of Nones means no previous stage, as in the reference
    PR.check_no_previous_stage(_predictor_stub(), [None, None])
    PR.check_no_previous_stage(_predictor_stub(), None)
    with pytest.raises(NotImplementedError):
        PR.check_no_previous_stage(_predictor_stub("3d_lowres"), [None])


def test_backbone_check():
    from oracle import dinounet_oracle as O
    a, b = O.make_state_dict("dinounet_s", 2, seed=0), O.make_state_dict("dinounet_s", 2, seed=1)
    assert not backbones_identical([a, b])
    for k in b:
        if ".dinov3_adapter.backbone." in k:
            b[k] = a[k].clone()
    assert backbones_identical([a, b]) and backbones_identical([a, b, dict(b)])
    assert not backbones_identical([a]) and not backbones_identical(None) and not backbones_identical([])
    k = next(k for k in b if k.startswith("decoder.encoder.dinov3_adapter.backbone.blocks.0.attn.qkv.weight"))
    c = dict(b)
    c[k] = b[k].clone()
    c[k].view(-1)[0] = torch.nextafter(c[k].view(-1)[0], torch.tensor(1e9))   # one ulp in a duplicate entry
    assert not backbones_identical([a, c])
    assert backbones_identical([a, {n: t for n, t in b.items() if n != "decoder.seg_layers.2.bias"}])
    assert not backbones_identical([a, {n: t for n, t in b.items() if n != k}])


def test_capture_guard_excludes_writer_device_work():
    """A graph capture waits for the writers inside `device_work()` and keeps new ones out until it ends."""
    import threading
    import time
    from dinounet_b200.engine import _CaptureGuard
    guard = _CaptureGuard()
    log, inside = [], threading.Event()
    release = threading.Event()

    def writer(name, hold):
        with guard.device_work():
            log.append(f"{name} in")
            inside.set()
            if hold:
                release.wait(5)
            log.append(f"{name} out")

    w1 = threading.Thread(target=writer, args=("w1", True))
    w1.start()
    inside.wait(5)

    def capture():
        with guard.capture():
            log.append("capture in")
            time.sleep(0.05)
            log.append("capture out")

    c = threading.Thread(target=capture)
    c.start()
    time.sleep(0.05)
    w2 = threading.Thread(target=writer, args=("w2", False))
    w2.start()
    time.sleep(0.05)
    assert log == ["w1 in"]            # the capture waits for w1; w2 waits behind the capture
    release.set()
    for t in (w1, c, w2):
        t.join(5)
    assert log == ["w1 in", "w1 out", "capture in", "capture out", "w2 in", "w2 out"]
