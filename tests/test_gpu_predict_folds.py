"""Fold ensembles on one backbone and the model-folder prediction entry points, on the device.

The folds of one training run hold the same frozen DINOv3 backbone, so `SlidingWindowPredictor` runs the ViT once per
tile batch and each fold's SPM .. seg head on the shared taps.  Its fp16 logits must have the bits of the route that
reloads the network for every fold; `predict_from_files` over a model folder must write what `predict_single_npy_array`
computes per case.
"""
import os
import pickle
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
MODEL = "dinounet_s"


def _folds(n, ncls, shared=True):
    """n state dicts from different seeds; with `shared`, every fold gets seed 0's backbone tensors (the frozen
    backbone of one training run)."""
    from oracle import dinounet_oracle as O
    folds = [O.make_state_dict(MODEL, ncls, seed=s) for s in range(n)]
    if shared:
        for sd in folds[1:]:
            for k in sd:
                if ".dinov3_adapter.backbone." in k:
                    sd[k] = folds[0][k].clone()
    return folds


def _net(ncls):
    import dinounet_b200
    from dinounet_b200 import config
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, ncls, None, MODEL)
    return net.to(DEV).eval()


def _predictor(net, folds, mirror, tile_batch=4, patch=128, chunk=None):
    from dinounet_b200.sliding_window import SlidingWindowPredictor
    p = SlidingWindowPredictor(tile_step_size=0.5, use_gaussian=True, use_mirroring=mirror, device=DEV,
                               tile_batch=tile_batch)
    p.manual_initialization(net, None, SimpleNamespace(patch_size=[patch, patch]), folds, {}, "DinoUNetTrainer_s",
                            (0, 1))
    p.fold_chunk_slices = chunk
    return p


def _bits(t):
    return t.contiguous().view(torch.int16).cpu()


@pytest.mark.parametrize("nf,mirror,chunk,shape", [
    (2, True, 2, (5, 200, 150)),      # 3 x 2 overlapping tiles per slice, chunks of 2, 2, 1 slices
    (3, False, 2, (5, 200, 150)),
    (3, True, None, (3, 130, 260)),   # 2 x 4 tiles per slice: the default chunk is 2 slices (chunks of 2 and 1)
    (2, True, None, (2, 130, 260)),   # the default chunk covers the whole case
    (2, False, 1, (4, 100, 128)),     # smaller than one tile in H: padded and cropped back
])
def test_shared_backbone_bits_equal_per_fold_route(nf, mirror, chunk, shape):
    ncls = 3
    folds = _folds(nf, ncls)
    net = _net(ncls)
    data = torch.from_numpy((np.random.default_rng(nf + 10 * len(shape)).standard_normal((2, *shape)) * 2)
                            .astype(np.float32)).to(DEV)
    p = _predictor(net, folds, mirror, chunk=chunk)
    got = p.predict_logits_from_preprocessed_data(data)
    assert p.ensemble_route == "shared_backbone"
    assert got.shape == (ncls, *shape) and got.dtype == torch.float16
    last = folds[-1]["decoder.seg_layers.2.weight"]
    assert torch.equal(net.state_dict()["decoder.seg_layers.2.weight"].cpu(), last)   # the module holds the last fold
    # a second case on the same predictor reuses the packed folds and gives the same bits
    again = p.predict_logits_from_preprocessed_data(data)
    assert torch.equal(_bits(got), _bits(again))
    # today's route: a list assigned after initialisation reloads the network for every fold
    p.list_of_parameters = list(folds)
    want = p.predict_logits_from_preprocessed_data(data)
    assert p.ensemble_route == "per_fold"
    assert torch.equal(_bits(got), _bits(want))


def test_different_backbones_take_per_fold_route():
    ncls = 2
    folds = _folds(2, ncls, shared=False)
    net = _net(ncls)
    p = _predictor(net, folds, mirror=False)
    data = torch.from_numpy(np.random.default_rng(1).standard_normal((1, 2, 128, 128)).astype(np.float32)).to(DEV)
    out = p.predict_logits_from_preprocessed_data(data)
    assert p.ensemble_route == "per_fold"
    assert out.shape == (ncls, 2, 128, 128)


def test_accumulate_without_npred_adds_the_same_logits():
    from dinounet_b200 import lib as L
    from dinounet_b200.sliding_window import compute_gaussian
    lib = L.load()
    C, D, H, W, th = 3, 2, 160, 200, 128
    g = torch.Generator(device="cpu").manual_seed(3)
    logits = (torch.randn((4, C, th, th), generator=g) * 5).to(DEV)
    desc = torch.tensor([[1, 20, 50, 0], [1, 20, 50, 1], [1, 20, 50, 2], [1, 20, 50, 3]], dtype=torch.int32, device=DEV)
    gauss = compute_gaussian((th, th), 1. / 8, 10, device=DEV)
    acc0 = (torch.randn((C, D, H, W), generator=g)).half().to(DEV)
    npred0 = torch.rand((D, H, W), generator=g).half().to(DEV)
    a1, n1 = acc0.clone(), npred0.clone()
    a2, n2 = acc0.clone(), npred0.clone()
    stream = torch.cuda.current_stream(DEV).cuda_stream
    L.check(lib.b2u_sw_accumulate(logits.data_ptr(), desc.data_ptr(), 0, 4, gauss.data_ptr(), a1.data_ptr(),
                                  n1.data_ptr(), C, D, H, W, th, th, stream), "sw_accumulate")
    L.check(lib.b2u_sw_accumulate(logits.data_ptr(), desc.data_ptr(), 0, 4, gauss.data_ptr(), a2.data_ptr(), None,
                                  C, D, H, W, th, th, stream), "sw_accumulate")
    torch.cuda.synchronize()
    assert torch.equal(_bits(a1), _bits(a2))
    assert not torch.equal(_bits(a1), _bits(acc0))
    assert torch.equal(_bits(n2), _bits(npred0))
    assert not torch.equal(_bits(n1), _bits(npred0))


# ------------------------------------------------------------------------------------------ model folder end to end
class NpyIO:
    """A reader-writer of `.npy` images ([X, Y, Z] per channel file) and segmentations."""
    spacing = [3.0, 1.0, 1.0]

    def read_images(self, files):
        return np.stack([np.load(f) for f in files]).astype(np.float32), {"spacing": list(self.spacing)}

    def write_seg(self, seg, path, properties):
        np.save(path, seg)


def _managers(regions):
    from dinounet_b200 import config
    from dinounet_b200 import export as EX
    from dinounet_b200 import preprocess as PP
    from oracle import make_golden_preprocess as MG
    conf = {"preprocessor_name": "DefaultPreprocessor", "resampling_fn_data": PP.DEFAULT_RESAMPLING_FN,
            "resampling_fn_data_kwargs": dict(PP.DEFAULT_RESAMPLING_KWARGS),
            "resampling_fn_probabilities": EX.DEFAULT_RESAMPLING_FN,
            "resampling_fn_probabilities_kwargs": dict(EX.DEFAULT_RESAMPLING_KWARGS)}
    cm = SimpleNamespace(spacing=[0.8, 0.8], patch_size=[128, 128], normalization_schemes=["ZScoreNormalization"] * 2,
                         use_mask_for_norm=[False] * 2, configuration=conf, previous_stage_name=None,
                         network_arch_class_name="dinounet_b200.DinoUNet", batch_size=2,
                         median_image_size_in_voxels=[100, 100],
                         network_arch_init_kwargs=dict(config.DEFAULT_ARCHITECTURE))
    if regions:
        lm = SimpleNamespace(has_regions=True, regions_class_order=[1, 2, 3], foreground_labels=[1, 2, 3],
                             foreground_regions=[[1, 2, 3], [2, 3], [3]], num_segmentation_heads=3)
    else:
        lm = SimpleNamespace(has_regions=False, regions_class_order=None, foreground_labels=[1, 2],
                             num_segmentation_heads=3)
    intensity = {str(i): MG.INTENSITY[str(i)] for i in range(2)}
    pm = SimpleNamespace(transpose_forward=[0, 1, 2], transpose_backward=[0, 1, 2], get_label_manager=lambda dj: lm,
                         foreground_intensity_properties_per_channel=intensity, image_reader_writer_class=NpyIO,
                         plans={"plans_name": "test", "configurations": {"2d": {}}},
                         get_configuration=lambda name: cm)
    return pm, cm, lm


def _model_folder(root, folds):
    os.makedirs(root)
    with open(os.path.join(root, "dataset.json"), "w") as f:
        f.write('{"channel_names": {"0": "CT", "1": "CT"}, "labels": {"background": 0}, "file_ending": ".npy"}')
    with open(os.path.join(root, "plans.json"), "w") as f:
        f.write('{"plans_name": "test"}')
    for k, sd in enumerate(folds):
        os.makedirs(os.path.join(root, f"fold_{k}"))
        torch.save({"network_weights": {"module." + n: t for n, t in sd.items()}, "trainer_name": "DinoUNetTrainer_s",
                    "init_args": {"configuration": "2d"}, "inference_allowed_mirroring_axes": (0, 1)},
                   os.path.join(root, f"fold_{k}", "checkpoint_final.pth"))


CASES = (("case_a", (3, 90, 150)), ("case_b", (2, 140, 110)), ("case_c", (4, 100, 100)), ("case_d", (2, 130, 130)))


def _folder_and_cases(tmp_path, monkeypatch, regions, folds):
    from dinounet_b200 import predict as PR
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    pm, cm, lm = _managers(regions)
    monkeypatch.setattr(PR, "_plans_manager", lambda plans: pm)
    model = str(tmp_path / "model")
    _model_folder(model, folds)
    src, out = tmp_path / "in", tmp_path / "out"
    os.makedirs(src)
    rng = np.random.default_rng(7)
    images = {}
    for case, shape in CASES:
        img = (rng.standard_normal((2, *shape)) * 30 + 40).astype(np.float32)
        images[case] = img
        for c in range(2):
            np.save(src / f"{case}_{c:04d}.npy", img[c])
    return model, src, out, images


def _check_outputs(p, out, images):
    for case, img in images.items():
        seg, probs = p.predict_single_npy_array(img, {"spacing": list(NpyIO.spacing)}, None, None, True)
        got = np.load(out / f"{case}.npy")
        assert got.shape == img.shape[1:] and np.array_equal(got, seg)
        got_p = np.load(out / f"{case}.npz")["probabilities"]
        assert np.array_equal(got_p.view(np.int32), probs.view(np.int32))
        with open(out / f"{case}.pkl", "rb") as f:
            assert pickle.load(f)["spacing"] == list(NpyIO.spacing)


@pytest.mark.parametrize("regions", [False, True])
def test_predict_from_files_matches_predict_single_npy_array(tmp_path, monkeypatch, regions):
    from dinounet_b200.sliding_window import SlidingWindowPredictor
    model, src, out, images = _folder_and_cases(tmp_path, monkeypatch, regions, _folds(2, 3))
    p = SlidingWindowPredictor(tile_step_size=0.5, device=DEV, tile_batch=4)
    p.initialize_from_trained_model_folder(model, None)
    assert p.trainer_name == "DinoUNetTrainer_s" and tuple(p.allowed_mirroring_axes) == (0, 1)
    assert len(p.list_of_parameters) == 2
    p.predict_from_files(str(src), str(out), save_probabilities=True, overwrite=True, num_processes_preprocessing=2,
                         num_processes_segmentation_export=2)
    assert p.ensemble_route == "shared_backbone"
    for name in ("predict_from_raw_data_args.json", "dataset.json", "plans.json"):
        assert (out / name).is_file()
    _check_outputs(p, out, images)

    # overwrite=False predicts only the cases whose outputs are missing
    os.remove(out / "case_b.npy")
    calls = []
    run = p.predict_logits_from_preprocessed_data
    monkeypatch.setattr(p, "predict_logits_from_preprocessed_data", lambda d: calls.append(d.shape) or run(d))
    p.predict_from_files(str(src), str(out), save_probabilities=True, overwrite=False)
    assert len(calls) == 1 and (out / "case_b.npy").is_file()

    # predict_from_list_of_npy_arrays without output names returns the segmentations
    res = p.predict_from_list_of_npy_arrays([images["case_a"]], None, [{"spacing": list(NpyIO.spacing)}], None,
                                            save_probabilities=False)
    assert len(res) == 1 and np.array_equal(res[0], np.load(out / "case_a.npy"))


@pytest.mark.parametrize("kind", ["one_fold", "different_backbones"])
def test_predict_from_files_per_fold_route(tmp_path, monkeypatch, kind):
    """One fold, or folds whose backbones differ: the per-fold route repacks the network for every case, and its new
    CUDA graphs are captured while three writer threads export the earlier cases."""
    from dinounet_b200.sliding_window import SlidingWindowPredictor
    folds = _folds(2, 3, shared=False)
    model, src, out, images = _folder_and_cases(tmp_path, monkeypatch, False, folds)
    p = SlidingWindowPredictor(tile_step_size=0.5, device=DEV, tile_batch=4)
    p.initialize_from_trained_model_folder(model, (0,) if kind == "one_fold" else None)
    assert len(p.list_of_parameters) == (1 if kind == "one_fold" else 2)
    p.predict_from_files(str(src), str(out), save_probabilities=True, overwrite=True, num_processes_preprocessing=2,
                         num_processes_segmentation_export=3)
    assert p.ensemble_route == "per_fold"
    _check_outputs(p, out, images)
