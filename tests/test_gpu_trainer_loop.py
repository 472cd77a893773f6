"""-m gpu: the training loop's optimizer state and final validation on the device.

* Resume: 3 native train steps on dinounet_s at 128^2, network and FusedSGD state through torch.save / torch.load into a
  fresh network and optimizer, then one step on a fixed set of gradients (the backward kernels use atomics, so their
  gradients are not reproducible bit for bit): parameters and momentum buffers are bitwise equal.
* Against torch: from one state dict, 3 steps of FusedSGD and of torch.optim.SGD(momentum 0.99, nesterov) after
  clip_grad_norm_(12) on the same gradients agree within RTOL / ATOL (fp32: the clip coefficient is summed in float64
  here and in fp32 by torch, and the update's multiply-adds are ordered differently).
* Lazy buffers: torch's first-step rule for a parameter whose first gradient comes at step 2; no buffer for a frozen one.
* Final validation: `perform_actual_validation` of a stand-in trainer on three preprocessed cases (label maps; regions
  with an ignore label) writes, per case, the label volume of the oracle route (the reference's sliding-window loop
  without mirroring, oracle/sliding_window_oracle.py, then the export oracle), up to near-ties of the top two
  probabilities for label maps as in tests/test_gpu_export.py; `summary.json` is the device evaluation of those files;
  with `save_probabilities` the `.npz` / `.pkl` files are what the export writes.
"""
import copy
import os
import pickle
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import dinounet_b200
from dinounet_b200 import config, evaluation, export as EX, lib as L
from dinounet_b200 import training as TR
from dinounet_b200.loss import DC_and_CE_loss, validation_statistics
from dinounet_b200.preprocess import _save_case
from dinounet_b200.train_path import FusedSGD, train_step
from oracle import dinounet_oracle as O
from oracle import export_oracle as EO
from oracle import sliding_window_oracle as SWO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
RTOL, ATOL = 1e-5, 1e-6
PROB_ULP = 8   # tests/test_gpu_export.py


def _net(ncls=2, in_ch=3):
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, in_ch, ncls, None,
                                             "dinounet_s")
    net.load_state_dict(O.make_state_dict("dinounet_s", ncls, seed=0), strict=True)
    return net.to(DEV)


def _fixed_grads(opt, seed, scale):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [None if p not in opt.state else torch.randn(p.shape, generator=g, device=DEV) * scale for p in opt.params]


def _set_grads(params, grads):
    for p, g in zip(params, grads):
        p.grad = None if g is None else g.clone()


def _trained(tmp_path):
    net = _net().train()
    crit = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, weight_ce=1, weight_dice=1)
    opt = FusedSGD(net.parameters(), lr=1e-2, weight_decay=3e-5, momentum=0.99, max_norm=12.0)
    x = O.make_input(2, 128, 5).to(DEV)
    target = torch.randint(0, 2, (2, 1, 128, 128), generator=torch.Generator().manual_seed(3)).float().to(DEV)
    n0 = L.launch_count()
    for _ in range(3):
        train_step(net, crit, opt, x, target)
    torch.cuda.synchronize()
    assert L.launch_count() - n0 > 500, "native kernels did not run"
    path = str(tmp_path / "checkpoint.pth")
    torch.save({"network_weights": net.state_dict(), "optimizer_state": opt.state_dict()}, path)
    return net, opt, path


def test_resume_from_a_checkpoint_is_bitwise_identical(tmp_path):
    net, opt, path = _trained(tmp_path)
    trainable = [p for p in net.parameters() if p.requires_grad]
    # every parameter is in the group; buffers exist for the ones that received a gradient (the frozen backbone never
    # does, nor do the unused deep-supervision heads)
    assert len(opt.params) == len(list(net.parameters())) and 200 < len(opt.state) <= len(trainable)
    assert all(p.requires_grad for p in opt.state)

    ck = torch.load(path, map_location=DEV, weights_only=False)
    net2 = _net().train()
    net2.load_state_dict(ck["network_weights"])
    opt2 = FusedSGD(net2.parameters(), lr=0.5, weight_decay=0.0, momentum=0.9, max_norm=12.0)
    opt2.load_state_dict(ck["optimizer_state"])
    assert opt2.param_groups[0]["lr"] == 1e-2 and len(opt2.state) == len(opt.state)

    grads = _fixed_grads(opt, 7, 1e-4)   # total norm far below 12: the clip coefficient is exactly 1 on both sides
    _set_grads(opt.params, grads)
    _set_grads(opt2.params, grads)
    opt.step()
    opt2.step()
    torch.cuda.synchronize()
    for (n, a), b in zip(net.named_parameters(), net2.parameters()):
        assert torch.equal(a, b), n
        if a in opt.state:
            assert torch.equal(opt.state[a]["momentum_buffer"], opt2.state[b]["momentum_buffer"]), n


def test_three_steps_agree_with_torch_sgd(tmp_path):
    net, opt, _ = _trained(tmp_path)
    ps = opt.params
    ref = [p.detach().clone().requires_grad_(p.requires_grad) for p in ps]
    topt = torch.optim.SGD(ref, lr=1.0, momentum=0.99, nesterov=True)
    topt.load_state_dict(copy.deepcopy(opt.state_dict()))   # load_state_dict keeps the given buffers
    assert topt.param_groups[0]["weight_decay"] == 3e-5
    for step in range(3):
        grads = _fixed_grads(opt, 20 + step, 1.0 if step == 1 else 1e-3)   # step 1 exceeds the clip threshold
        _set_grads(ps, grads)
        _set_grads(ref, grads)
        torch.nn.utils.clip_grad_norm_(ref, 12)
        topt.step()
        opt.step()
        worst = 0.0
        for p, r in zip(ps, ref):
            assert torch.allclose(p, r, rtol=RTOL, atol=ATOL), step
            worst = max(worst, float((p.detach() - r.detach()).abs().max()))
        for p, r in zip(ps, ref):
            if p in opt.state:
                b, rb = opt.state[p]["momentum_buffer"], topt.state[r]["momentum_buffer"]
                assert torch.allclose(b, rb, rtol=RTOL, atol=ATOL * max(1.0, float(rb.abs().max()))), step
        print(f"step {step}: grad norm {opt.grad_norm():.3f}, max |param - torch| {worst:.2e}")


def test_lazy_buffers_follow_torch_first_step():
    g = torch.Generator(device=DEV).manual_seed(0)
    ps = [torch.randn(300, generator=g, device=DEV).requires_grad_(), torch.randn(40, generator=g, device=DEV),
          torch.randn(17, 5, generator=g, device=DEV).requires_grad_()]
    ref = [p.detach().clone().requires_grad_(p.requires_grad) for p in ps]
    opt = FusedSGD(ps, lr=1e-2, weight_decay=3e-5, momentum=0.99)
    topt = torch.optim.SGD(ref, lr=1e-2, weight_decay=3e-5, momentum=0.99, nesterov=True)
    for step in range(3):
        grads = [torch.randn(p.shape, generator=g, device=DEV) * 0.1 if (i == 0 or (i == 2 and step >= 1)) else None
                 for i, p in enumerate(ps)]
        _set_grads(ps, grads)
        _set_grads(ref, grads)
        before = ps[2].detach().clone()
        torch.nn.utils.clip_grad_norm_(ref, 12)   # norms of about 2: no clipping
        topt.step()
        opt.step()
        assert (ps[2] in opt.state) == (step >= 1) and ps[1] not in opt.state
        for p, r in zip(ps, ref):
            assert torch.allclose(p, r, rtol=RTOL, atol=ATOL), step
        if step == 1:   # first step of parameter 2: buffer = gradient + weight decay * parameter, no momentum term
            buf = opt.state[ps[2]]["momentum_buffer"]
            assert torch.allclose(buf, grads[2] + 3e-5 * before, rtol=RTOL, atol=ATOL)
            assert torch.allclose(buf, topt.state[ref[2]]["momentum_buffer"], rtol=RTOL, atol=ATOL)
    assert torch.equal(ps[1], ref[1])


# ------------------------------------------------------------------------------------------------- final validation
class _NpyRW:
    """Reader-writer on .npy files, as the reference's writers: write_seg(seg) stores [1, *seg.shape]."""
    spacing = (3.0, 0.8, 0.9)

    def write_seg(self, seg, path, props):
        np.save(path, seg[None])

    def read_seg(self, path):
        return np.load(path), {"spacing": self.spacing}


class _Dataset:
    """nnUNetDataset's `keys()` / `load_case(key)` over `<key>.npz` (data, seg) and `<key>.pkl`."""

    def __init__(self, folder, keys, folder_with_segs_from_previous_stage=None):
        assert folder_with_segs_from_previous_stage is None
        self.folder, self._keys = folder, list(keys)

    def keys(self):
        return list(self._keys)

    def load_case(self, k):
        f = np.load(os.path.join(self.folder, k + ".npz"))
        with open(os.path.join(self.folder, k + ".pkl"), "rb") as fh:
            return f["data"], f["seg"], pickle.load(fh)


PATCH = [128, 128]
TRANSPOSE_BACKWARD = [0, 2, 1]
CASES = [  # preprocessed [Z, h, w], shape after cropping [Z, H, W], shape before cropping, bbox
    ((2, 140, 150), (2, 120, 170), (3, 130, 180), [[1, 3], [5, 125], [4, 174]]),
    ((1, 128, 200), (1, 128, 200), (1, 140, 210), [[0, 1], [6, 134], [3, 203]]),
    ((3, 100, 131), (3, 150, 97), (4, 152, 100), [[0, 3], [1, 151], [2, 99]]),
]


def _label_manager(regions):
    if regions:
        return SimpleNamespace(has_regions=True, regions_class_order=[1, 2, 3], foreground_labels=[1, 2, 3],
                               foreground_regions=[(1, 2, 3), (2, 3), (3,)], num_segmentation_heads=3, ignore_label=4)
    return SimpleNamespace(has_regions=False, regions_class_order=None, foreground_labels=[1, 2],
                           foreground_regions=None, num_segmentation_heads=3, ignore_label=None)


def _smooth_labels(shape, n, seed):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(1, n, shape[0], shape[1] // 8 + 2, shape[2] // 8 + 2, generator=g)
    z = torch.nn.functional.interpolate(z, size=tuple(shape), mode="trilinear", align_corners=False)
    return z[0].argmax(0).numpy().astype(np.uint8)


def _stand_in(tmp_path, net, regions):
    """A trainer with the attributes perform_actual_validation reads, its preprocessed cases on disk as
    DevicePreprocessor.run_case_save writes them, and gt_segmentations/ in the original geometry."""
    base = tmp_path / ("regions" if regions else "labels")
    pre, gt = base / "preprocessed", base / "preprocessed" / "gt_segmentations"
    folder = pre / "DinoUNetPlans_2d"
    for d in (folder, gt):
        d.mkdir(parents=True)
    lm = _label_manager(regions)
    keys = []
    for i, (shape, after, before, bbox) in enumerate(CASES):
        k = f"case_{i:03d}"
        keys.append(k)
        g = torch.Generator().manual_seed(40 + i)
        data = (torch.randn(1, *shape, generator=g) * 0.8).numpy().astype(np.float32)
        props = {"spacing": [3.0, 0.8, 0.9], "shape_before_cropping": list(before), "bbox_used_for_cropping": bbox,
                 "shape_after_cropping_and_before_resampling": list(after)}
        _save_case(str(folder / k), data, np.zeros((1, *shape), dtype=np.int8), props)
        ref = _smooth_labels(before, 5 if regions else 3, 60 + i).transpose(TRANSPOSE_BACKWARD)
        np.save(str(gt / (k + ".npy")), ref[None])
    conf = {"resampling_fn_probabilities": EX.DEFAULT_RESAMPLING_FN,
            "resampling_fn_probabilities_kwargs": dict(EX.DEFAULT_RESAMPLING_KWARGS)}
    tr = TR.DinoUNetTrainer_s.__new__(TR.DinoUNetTrainer_s)
    tr.logged = []
    tr.print_to_log_file = lambda *a, **kw: tr.logged.append(" ".join(str(x) for x in a))
    tr.network, tr.device, tr.is_ddp, tr.local_rank, tr.is_cascaded = net, DEV, False, 0, False
    tr.configuration_manager = SimpleNamespace(patch_size=PATCH, next_stage_names=None, spacing=[0.7, 0.75],
                                               configuration=conf)
    tr.plans_manager = SimpleNamespace(transpose_backward=TRANSPOSE_BACKWARD, get_label_manager=lambda dj: lm,
                                       image_reader_writer_class=_NpyRW)
    tr.label_manager, tr.dataset_json = lm, {"file_ending": ".npy"}
    tr.output_folder = str(base / "fold_0")
    tr.preprocessed_dataset_folder, tr.preprocessed_dataset_folder_base = str(folder), str(pre)
    tr.folder_with_segs_from_previous_stage = None
    tr.inference_allowed_mirroring_axes = (0, 1)
    tr.do_split = lambda: (["train_case"], list(keys))
    return tr, keys


def _oracle_labels(net, data, props, lm):
    def network(t):                      # the reference's forward: autocast fp16 output
        with torch.no_grad():
            return net(t).half()
    logits = SWO.predict_sliding_window_return_logits(network, torch.from_numpy(data).to(DEV), PATCH, 3, 0.5, True,
                                                      None, results_device=DEV)
    _, seg, probs = EO.convert(logits.cpu(), props, TRANSPOSE_BACKWARD, len(lm.foreground_labels), lm.has_regions,
                               lm.regions_class_order, True)
    return seg, probs


def _fresh(state_dict, ncls=3, in_ch=1):
    """A network with an engine of its own, packed from `state_dict`: the expected side never shares the engine that the
    network under test cached."""
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, in_ch, ncls, None,
                                             "dinounet_s")
    net.load_state_dict(state_dict, strict=True)
    return net.to(DEV).eval()


def _crit():
    return DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, weight_ce=1, weight_dice=1)


def _train_in_place(net):
    """What a run does to the network before its final validation: native train steps (the first one builds and caches
    the engine), then an in-place change of the seg head that moves most labels."""
    net.train()
    opt = FusedSGD(net.parameters(), lr=1e-2)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(2, 1, 128, 128, generator=g).to(DEV)
    target = torch.randint(0, 3, (2, 1, 128, 128), generator=g).float().to(DEV)
    for _ in range(2):
        train_step(net, _crit(), opt, x, target)
    with torch.no_grad():
        dict(net.named_parameters())["decoder.seg_layers.2.weight"].neg_()
    net.eval()


@pytest.mark.parametrize("regions", [False, True], ids=["label_maps", "regions_ignore"])
def test_final_validation_against_the_oracle_route(tmp_path, monkeypatch, regions):
    """After training the network in place: validation/ holds the labels of its current weights."""
    monkeypatch.setattr(TR, "_validation_dataset", _Dataset)
    net = _net(ncls=3, in_ch=1)
    initial = _fresh(copy.deepcopy(net.state_dict()))
    _train_in_place(net)
    current = _fresh(net.state_dict())
    tr, keys = _stand_in(tmp_path, net, regions)
    lm = tr.label_manager
    n0 = L.launch_count()
    tr.perform_actual_validation(save_probabilities=regions)
    torch.cuda.synchronize()
    assert L.launch_count() - n0 > 100, "native kernels did not run"
    val = os.path.join(tr.output_folder, "validation")
    for k in keys:
        assert f"predicting {k}" in tr.logged
        assert any(line.startswith(f"{k}, shape torch.Size([1, ") for line in tr.logged)
    assert any(line.startswith("Mean Validation Dice:") for line in tr.logged)

    data_dir = tr.preprocessed_dataset_folder
    for k in keys:
        data, _, props = _Dataset(data_dir, [k]).load_case(k)
        seg = np.load(os.path.join(val, k + ".npy"))[0]
        want, want_p = _oracle_labels(current, data, props, lm)
        assert seg.dtype == want.dtype and seg.shape == want.shape
        stale, _ = _oracle_labels(initial, data, props, lm)
        print(f"{k}: {float((stale != want).mean()):.1%} of the labels differ between the initial and the trained weights")
        assert (stale != want).mean() > 0.05, k     # a validation on the weights packed before training would fail
        if regions:
            assert np.array_equal(seg, want), k
        else:
            top2 = np.sort(want_p, axis=0)[-2:]
            near_tie = np.abs(top2[1].view(np.int32).astype(np.int64) - top2[0].view(np.int32)) <= PROB_ULP
            diff = seg != want
            print(f"{k}: {int(diff.sum())} of {seg.size} labels differ from the oracle route, all at near-ties")
            assert not (diff & ~near_tie).any(), k
        assert os.path.isfile(os.path.join(val, k + ".npz")) == regions
        assert os.path.isfile(os.path.join(val, k + ".pkl")) == regions

    again = str(tmp_path / f"summary_{int(regions)}.json")
    evaluation.compute_metrics_on_folder(os.path.join(tr.preprocessed_dataset_folder_base, "gt_segmentations"), val, again,
                                         _NpyRW(), ".npy", lm.foreground_regions if regions else lm.foreground_labels,
                                         lm.ignore_label, chill=True)
    with open(os.path.join(val, "summary.json")) as a, open(again) as b:
        assert a.read() == b.read()
    summary = evaluation.load_summary_json(os.path.join(val, "summary.json"))
    assert len(summary["metric_per_case"]) == len(keys)

    if regions:   # the probabilities the export writes for the predictor's logits
        from dinounet_b200.sliding_window import SlidingWindowPredictor
        p = SlidingWindowPredictor(tile_step_size=0.5, use_gaussian=True, use_mirroring=False, device=DEV)
        p.manual_initialization(current, tr.plans_manager, tr.configuration_manager, None, tr.dataset_json, "t", None)
        for k in keys:
            data, _, props = _Dataset(data_dir, [k]).load_case(k)
            out = str(tmp_path / f"direct_{k}")
            EX.export_prediction_from_logits(p.predict_sliding_window_return_logits(torch.from_numpy(data)), props,
                                             tr.configuration_manager, tr.plans_manager, tr.dataset_json, out, True)
            got, want = np.load(os.path.join(val, k + ".npz"))["probabilities"], np.load(out + ".npz")["probabilities"]
            assert got.dtype == np.float32 and np.array_equal(got, want), k
            with open(os.path.join(val, k + ".pkl"), "rb") as fa, open(out + ".pkl", "rb") as fb:
                assert pickle.load(fa) == pickle.load(fb) == props


def test_validation_step_after_train_steps_sees_the_new_weights():
    """The trainer's online validation after its train steps: the statistics of the current weights (a fresh network's),
    not of the weights the engine packed at the first step."""
    net = _net(ncls=2, in_ch=3)
    crit = _crit()
    tr = TR.DinoUNetTrainer_s.__new__(TR.DinoUNetTrainer_s)
    tr.network, tr.loss, tr.device, tr.is_ddp = net.train(), crit, DEV, False
    tr.optimizer = FusedSGD(net.parameters(), lr=1e-2)
    g = torch.Generator().manual_seed(9)
    batch = {"data": torch.randn(2, 3, 128, 128, generator=g),
             "target": torch.randint(0, 2, (2, 1, 128, 128), generator=g).float()}
    x, t = batch["data"].to(DEV), batch["target"].to(DEV)
    with torch.no_grad():
        before = validation_statistics(crit, _fresh(net.state_dict(), 2, 3)(x), t)
    for _ in range(2):
        tr.train_step(batch)
    net.eval()
    got = tr.validation_step(batch)
    with torch.no_grad():
        want = validation_statistics(crit, _fresh(net.state_dict(), 2, 3)(x), t)
    print(f"validation loss: initial weights {float(before['loss']):.6f}, after 2 steps {float(got['loss']):.6f}")
    assert abs(float(got["loss"]) - float(before["loss"])) > 1e-5 * abs(float(before["loss"]))   # the steps moved it
    assert float(got["loss"]) == pytest.approx(float(want["loss"]), rel=1e-6)
    for key in ("tp_hard", "fp_hard", "fn_hard"):
        assert np.array_equal(np.asarray(got[key]), np.asarray(want[key])), key


def test_cascade_and_next_stage_raise_before_any_launch(tmp_path, monkeypatch):
    monkeypatch.setattr(TR, "_validation_dataset", _Dataset)
    tr, _ = _stand_in(tmp_path, _net(ncls=3, in_ch=1).eval(), False)
    torch.cuda.synchronize()
    n0 = L.launch_count()
    tr.is_cascaded = True
    with pytest.raises(NotImplementedError):
        tr.perform_actual_validation()
    tr.is_cascaded = False
    tr.configuration_manager.next_stage_names = ["3d_lowres"]
    with pytest.raises(NotImplementedError):
        tr.perform_actual_validation()
    assert L.launch_count() == n0 and not os.path.exists(os.path.join(tr.output_folder, "validation"))
