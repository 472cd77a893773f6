"""CPU: deep supervision without a GPU.

* The oracle restatement (oracle/deep_supervision_oracle.py: the three decoder heads, the weighted loss and its
  gradients through the oracle forward) against tests/golden/deep_supervision_cases.npz, the REAL reference's
  DinoUNet(deep_supervision=True) + DeepSupervisionWrapper (oracle/make_golden_deep_supervision.py), for a label map and
  for regions with an ignore channel.
* The target restatement (skimage's resize, order 0, mode edge) against hand-checked picks and scipy's zoom.
* The scales and weights the trainer derives from the plan, with and without DDP.
* The trainer's plumbing through recording stand-ins: the wrapped loss, lists passed to the train step and the loss,
  device-made targets handed to the target kernel, the counts from output[0] / target[0], and the toggle that never
  switches deep supervision on for a trainer without it.
"""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dinounet_b200 import deep_supervision as DS
from dinounet_b200 import lib as L
from dinounet_b200 import training as TR
from dinounet_b200.loss import DC_and_BCE_loss, DC_and_CE_loss, DeepSupervisionWrapper, validation_statistics
from oracle import deep_supervision_oracle as DSO
from oracle import dinounet_oracle as O
from oracle import loss_oracle as LO
from oracle import region_loss_oracle as RO

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "deep_supervision_cases.npz")
PLAN_POOLS = [[1, 1], [2, 2], [2, 2], [2, 2]]
SCALES = [[1.0, 1.0], [0.5, 0.5], [0.25, 0.25]]


@pytest.fixture(autouse=True)
def _no_kernels(monkeypatch):
    def refuse():
        raise AssertionError("a CPU deep-supervision test loaded the native library")
    monkeypatch.setattr(L, "load", refuse)


# ------------------------------------------------------------------------------------------------ oracle vs golden
def _golden_case(prefix):
    from oracle import make_golden_deep_supervision as MG
    t = MG.label_map() if prefix == "lm" else MG.region_target()
    targets = [torch.from_numpy(a) for a in DSO.downsample_seg_for_ds(t.numpy(), MG.SCALES)]
    if prefix == "lm":
        fn = lambda o, tt: LO.dc_and_ce_loss(o, tt, batch_dice=True)[0]
    else:
        fn = lambda o, tt: RO.dc_and_bce_loss(o, tt, batch_dice=True, use_ignore=True)[0]
    sd = O.make_state_dict(MG.MODEL, MG.NCLS, seed=MG.WSEED)
    x = O.make_input(MG.B, MG.S, MG.WSEED)
    return sd, x, targets, fn, MG


@pytest.mark.parametrize("prefix", ["lm", "rg"], ids=["label_map", "regions_ignore"])
def test_oracle_matches_the_reference_golden(prefix):
    g = np.load(GOLDEN)
    sd, x, targets, fn, MG = _golden_case(prefix)
    outs, loss, grads = DSO.loss_and_grads(sd, MG.MODEL, x, targets, fn, g["weights"])
    for i, o in enumerate(outs):
        want = g[f"logits{i}"]
        assert o.shape == want.shape
        assert np.abs(o.numpy() - want).max() <= 1e-5 * np.abs(want).max(), i
    assert abs(float(loss) - float(g[f"{prefix}_loss"])) <= 1e-5 * abs(float(g[f"{prefix}_loss"]))
    names = [str(n) for n in g[f"{prefix}_names"]]
    assert set(names) == set(grads)
    for i, k in enumerate(names):
        gr = grads[k]
        assert (gr is not None) == bool(g[f"{prefix}_has_grad"][i]), k
        if gr is None:
            continue
        want = float(g[f"{prefix}_norms"][i])
        assert abs(gr.double().norm().item() - want) <= 1e-4 * want + 1e-9, k
        f = gr.reshape(-1)
        samp = f[:: max(1, f.numel() // 16)][:16].numpy()
        ws = g[f"{prefix}_s{i}"]
        assert np.abs(samp - ws).max() <= 1e-4 * np.abs(ws).max() + 1e-9, k
    assert grads["decoder.seg_layers.0.weight"] is None and grads["decoder.seg_layers.1.weight"] is not None


# ------------------------------------------------------------------------------------------------ targets
def test_target_restatement_picks_by_hand():
    assert DSO.axis_picks(8, 4).tolist() == [1, 3, 5, 7]          # factor 2: (o + 0.5) * 2 - 0.5 = 2o + 0.5 -> 2o + 1
    assert DSO.axis_picks(8, 2).tolist() == [2, 6]                # factor 4: 4o + 1.5 -> 4o + 2
    assert DSO.axis_picks(5, 5).tolist() == [0, 1, 2, 3, 4]
    seg = np.arange(64, dtype=np.int16).reshape(1, 1, 8, 8)
    full, half, quarter = DSO.downsample_seg_for_ds(seg, SCALES)
    assert full is seg
    assert half.dtype == np.int16 and half[0, 0].tolist() == [[8 * y + x for x in (1, 3, 5, 7)] for y in (1, 3, 5, 7)]
    assert quarter[0, 0].tolist() == [[18, 22], [50, 54]]
    for n, m in ((512, 256), (512, 128), (128, 32), (9, 4), (7, 3)):
        assert np.array_equal(DSO.axis_picks(n, m), DSO.zoom_picks(n, m)), (n, m)


def test_scales_and_weights_follow_the_plan():
    assert DS.deep_supervision_scales(PLAN_POOLS) == SCALES
    for bad in ([[1, 1], [2, 2], [2, 2]], [[1, 1], [2, 2], [2, 2], [2, 2], [2, 2]], [[1, 1], [2, 2], [3, 3], [2, 2]],
                [[2, 2], [2, 2], [2, 2], [2, 2]]):
        with pytest.raises(NotImplementedError):
            DS.deep_supervision_scales(bad)
    assert np.allclose(DS.deep_supervision_weights(3, False), [2 / 3, 1 / 3, 0], rtol=0, atol=1e-15)
    assert DS.deep_supervision_weights(3, False)[-1] == 0
    ddp = DS.deep_supervision_weights(3, True)
    assert np.allclose(ddp, np.array([1, 0.5, 1e-6]) / 1.500001, rtol=1e-15) and ddp.sum() == pytest.approx(1)
    for d in (False, True):
        assert np.array_equal(DS.deep_supervision_weights(3, d), DSO.ds_weights(3, d))


def test_target_kernel_wrapper_refuses_host_tensors():
    t = torch.zeros(2, 1, 16, 16, dtype=torch.int16)
    with pytest.raises(L.NativeLibraryError):
        DS.downsample_targets(t, SCALES)       # host tensors never reach the kernel


# ------------------------------------------------------------------------------------------------ trainer plumbing
class _Decoder:
    deep_supervision = False


class _Net:
    """Records calls; returns the three heads (or one) of a 2-class network at the input's resolution."""

    def __init__(self):
        self.decoder = _Decoder()

    def __call__(self, x):
        if self.decoder.deep_supervision:
            return [torch.zeros(x.shape[0], 2, x.shape[2] >> i, x.shape[3] >> i) for i in range(3)]
        return torch.zeros(x.shape[0], 2, *x.shape[2:])


def _trainer(ds, ddp=False, regions=False):
    tr = TR.DinoUNetTrainer_s.__new__(TR.DinoUNetTrainer_s)
    if ds is not None:
        tr.enable_deep_supervision = ds
    tr.is_ddp, tr.device = ddp, torch.device("cpu")
    tr.network = _Net()
    tr.configuration_manager = SimpleNamespace(batch_dice=True, pool_op_kernel_sizes=PLAN_POOLS)
    tr.label_manager = SimpleNamespace(has_regions=regions, ignore_label=None)
    tr.optimizer = tr.loss = None
    return tr


@pytest.mark.parametrize("ddp", [False, True])
def test_build_loss_wraps_with_the_reference_weights(ddp):
    loss = _trainer(True, ddp)._build_loss()
    assert isinstance(loss, DeepSupervisionWrapper) and isinstance(loss.loss, DC_and_CE_loss)
    assert np.array_equal(loss.weight_factors, DSO.ds_weights(3, ddp))
    assert (loss.weight_factors[-1] == 0) != ddp
    assert isinstance(_trainer(True, ddp, regions=True)._build_loss().loss, DC_and_BCE_loss)
    for ds in (None, False):
        assert isinstance(_trainer(ds, ddp)._build_loss(), DC_and_CE_loss)


def test_build_loss_rejects_a_plan_with_other_scales():
    tr = _trainer(True)
    tr.configuration_manager.pool_op_kernel_sizes = [[1, 1], [2, 2], [2, 2], [2, 2], [2, 2]]
    with pytest.raises(NotImplementedError):
        tr._build_loss()
    tr.enable_deep_supervision = False
    assert isinstance(tr._build_loss(), DC_and_CE_loss)     # without deep supervision the scales are not read


def test_train_step_passes_lists(monkeypatch):
    import dinounet_b200.train_path as TP
    seen = []
    monkeypatch.setattr(TP, "train_step", lambda net, loss, opt, data, target: seen.append(target) or torch.tensor(0.5))
    tr = _trainer(True)
    host = [torch.zeros(2, 1, 16 >> i, 16 >> i) for i in range(3)]
    assert tr.train_step({"data": torch.zeros(2, 3, 16, 16), "target": host})["loss"] == np.float32(0.5)
    assert isinstance(seen[-1], list) and [t.shape for t in seen[-1]] == [t.shape for t in host]
    # a target made on the device (device augmentation / loading) goes through the target kernel at the plan's scales
    calls = []
    monkeypatch.setattr(TR.DS, "downsample_targets", lambda t, scales: calls.append(scales) or ["ds", t])
    tr.train_step({"data": torch.zeros(2, 3, 16, 16), "target": torch.zeros(2, 1, 16, 16)})
    assert calls == [SCALES] and seen[-1][0] == "ds"
    # without deep supervision: the full-resolution target only, as before
    tr = _trainer(False)
    tr.train_step({"data": torch.zeros(2, 3, 16, 16), "target": host})
    assert seen[-1] is host[0]
    assert len(calls) == 1


def test_validation_step_counts_from_the_first_output(monkeypatch):
    seen = []

    class _Inner(DC_and_CE_loss):
        def _run(self, o, t):
            seen.append((tuple(o.shape), tuple(t.shape)))
            k = o.shape[-1]
            return torch.tensor(float(k)), None, torch.full((3, 2), k, dtype=torch.int64), None

    tr = _trainer(True)
    tr.network.decoder.deep_supervision = True
    tr.loss = DeepSupervisionWrapper(_Inner({"batch_dice": True, "do_bg": False}, {}), DS.deep_supervision_weights(3, False))
    host = [torch.zeros(2, 1, 16 >> i, 16 >> i) for i in range(3)]
    out = tr.validation_step({"data": torch.zeros(2, 3, 16, 16), "target": host})
    # the weight-0 scale is not evaluated; the loss is the weighted sum; the counts are scale 0's (background dropped)
    assert seen == [((2, 2, 16, 16), (2, 1, 16, 16)), ((2, 2, 8, 8), (2, 1, 8, 8))]
    assert float(out["loss"]) == pytest.approx(2 / 3 * 16 + 1 / 3 * 8)
    assert out["tp_hard"].tolist() == [16.0] and out["fn_hard"].tolist() == [16.0]
    # the same through validation_statistics directly
    seen.clear()
    st = validation_statistics(tr.loss, tr.network(torch.zeros(2, 3, 16, 16)), host)
    assert st["fp_hard"].tolist() == [16.0] and len(seen) == 2


def test_toggle_never_enables_deep_supervision_without_it():
    for ds in (None, False):
        tr = _trainer(ds)
        tr.set_deep_supervision_enabled(True)
        assert tr.network.decoder.deep_supervision is False
    tr = _trainer(True)
    tr.set_deep_supervision_enabled(False)
    assert tr.network.decoder.deep_supervision is False
    tr.set_deep_supervision_enabled(True)
    assert tr.network.decoder.deep_supervision is True
    tr = _trainer(True, ddp=True)
    inner = tr.network
    tr.network = SimpleNamespace(module=inner)
    tr.set_deep_supervision_enabled(True)
    assert inner.decoder.deep_supervision is True
