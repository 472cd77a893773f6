"""CPU: train-mode semantics ("reference") of the training step.

  * the torch restatement (oracle/train_mode_oracle.py), fed the draws recorded in tests/golden/train_mode_cases.npz,
    reproduces what the REAL reference computed in .train(): loss, gradients and the updated BatchNorm running statistics
    (so the recorded draws are the ones the reference used);
  * with a recording stand-in for the native library, `trainable_forward` issues today's calls without a TrainMode and
    the stats -> finalize -> apply sequence with one; DinoUNet rejects what "reference" does not cover before any launch.
"""
import contextlib
import os

import numpy as np
import pytest
import torch

from dinounet_b200 import lib as L
from dinounet_b200 import train_path as TP
from oracle import dinounet_oracle as O
from oracle import train_mode_oracle as T

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "train_mode_cases.npz")
MODEL, B, S, NCLS, WSEED = "dinounet_s", 2, 128, 2, 0


def test_restatement_reproduces_the_reference_train_mode_golden():
    g = np.load(GOLDEN)
    sd = O.make_state_dict(MODEL, NCLS, seed=WSEED)
    x = O.make_input(B, S, WSEED)
    target = torch.randint(0, NCLS, (B, 1, S, S), generator=torch.Generator().manual_seed(WSEED + 7)).float()
    loss, grads, bufs = T.loss_and_grads(sd, MODEL, x, target, torch.from_numpy(g["rope_scales"]), torch.from_numpy(g["drop_keep"]))
    assert abs(loss.item() - float(g["loss"])) <= 1e-6 * max(1.0, abs(float(g["loss"]))), (loss.item(), float(g["loss"]))
    names = [str(n) for n in g["names"]]
    assert sorted(grads) == names
    for i, k in enumerate(names):
        norm, want = grads[k].double().norm().item(), float(g["norms"][i])
        assert abs(norm - want) <= 1e-4 * want + 1e-9, (k, norm, want)
    for j, p in enumerate(T.BN_LAYERS):
        for key, name in ((f"rm{j}", ".running_mean"), (f"rv{j}", ".running_var")):
            got, want = bufs[p + name].numpy(), g[key]
            assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max(), (p + name, np.abs(got - want).max())
        assert int(bufs[p + ".num_batches_tracked"]) == int(g[f"nbt{j}"]) == 1


def test_recorded_draws_are_well_formed():
    g = np.load(GOLDEN)
    assert g["rope_scales"].shape == (O.VARIANTS[MODEL].depth,) and g["drop_keep"].shape == (6, B)
    assert ((g["rope_scales"] >= 0.5) & (g["rope_scales"] <= 2.0)).all()
    assert set(np.unique(g["drop_keep"]).tolist()) == {0.0, 1.0}


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
    r = _Recorder()
    monkeypatch.setattr(L, "load", lambda: r)
    monkeypatch.setattr(TP, "_s", lambda t: 0)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda dev=None: type("S", (), {"cuda_stream": 0})())
    return r


def _inputs(Sz=64):
    P = {k: t.clone() for k, t in O.make_state_dict(MODEL, NCLS, seed=0).items()}
    for k, t in P.items():
        if t.is_floating_point() and not k.endswith(("running_mean", "running_var")):
            t.requires_grad_(True)
    x = torch.zeros(B, 3, Sz, Sz)
    taps = [torch.zeros(B, (Sz // 16) ** 2, O.VARIANTS[MODEL].dim) for _ in range(4)]
    return P, x, taps


def _train_mode():
    return TP.TrainMode(bn={p: (0.1, 1e-5) for p in T.BN_LAYERS}, drop_scale=torch.ones(6, B) / 0.7)


def _names(r, prefix=""):
    return [n for n, _ in r.calls if n.startswith(prefix)]


def test_oracle_semantics_issues_todays_calls(rec):
    P, x, taps = _inputs()
    TP.trainable_forward(P, MODEL, x, taps, NCLS, "fp32")
    bn = [a for n, a in rec.calls if n == "b2u_f32_bn_act"]
    assert len(bn) == 10
    rms = {P[p + ".running_mean"].data_ptr() for p in T.BN_LAYERS}
    rvs = {P[p + ".running_var"].data_ptr() for p in T.BN_LAYERS}
    assert {a[4] for a in bn} == rms and {a[5] for a in bn} == rvs          # normalised with the running statistics
    new = {"b2u_f32_bn_stats", "b2u_f32_bn_finalize", "b2u_f32_droppath_add", "b2u_rope_tables", "b2u_f32_bn_work_doubles"}
    assert not new & set(_names(rec))


def test_reference_semantics_issues_stats_finalize_apply(rec):
    P, x, taps = _inputs()
    logits = TP.trainable_forward(P, MODEL, x, taps, NCLS, "fp32", _train_mode())
    seq = [(n, a) for n, a in rec.calls if n in ("b2u_f32_bn_stats", "b2u_f32_bn_finalize", "b2u_f32_bn_act")]
    assert [n for n, _ in seq] == ["b2u_f32_bn_stats", "b2u_f32_bn_finalize", "b2u_f32_bn_act"] * 10
    for j, p in enumerate(T.BN_LAYERS):
        stats, fin, act = (a for _, a in seq[3 * j:3 * j + 3])
        assert fin[0] == stats[4]                                            # finalize reads the sums the stats pass wrote
        assert (fin[4], fin[5], fin[6]) == (P[p + ".running_mean"].data_ptr(), P[p + ".running_var"].data_ptr(),
                                            P[p + ".num_batches_tracked"].data_ptr())
        assert (act[4], act[5]) == (fin[2], fin[3])                          # normalised with the batch mean / variance
    assert len(_names(rec, "b2u_f32_droppath_add")) == 6
    rec.calls.clear()
    logits.sum().backward()
    bwd = [n for n, _ in rec.calls if n.startswith("b2u_f32_bn_train_bwd")]
    assert bwd == ["b2u_f32_bn_train_bwd_reduce", "b2u_f32_bn_train_bwd_apply"] * 10
    dp = [a for n, a in rec.calls if n == "b2u_f32_droppath_add"]
    assert len(dp) == 6 and all(a[0] is None for a in dp)                   # the branch's backward: s * dy
    assert "b2u_f32_bn_act_bwd" not in _names(rec)


def _net():
    import dinounet_b200
    from dinounet_b200 import config
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    return dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, 2, None, MODEL).train()


def test_dinounet_rejects_what_reference_semantics_does_not_cover(rec):
    net = _net()
    x = torch.zeros(1, 3, 64, 64)
    assert net.train_semantics == "oracle"
    net.train_semantics = "train"
    with pytest.raises(ValueError):
        net(x)
    net.train_semantics = "reference"
    net.dinov3_model_name = "dinounet_7b"
    with pytest.raises(NotImplementedError, match="dinounet_7b"):
        net(x)
    net.dinov3_model_name = MODEL
    net.encoder.dinov3_adapter.spm.stem[1].momentum = None
    with pytest.raises(NotImplementedError, match="momentum"):
        net(x)
    net.encoder.dinov3_adapter.spm.stem[1].momentum = 0.1
    net.encoder.dinov3_adapter.norm2.track_running_stats = False
    with pytest.raises(NotImplementedError, match="track_running_stats"):
        net(x)
    assert rec.calls == []


def test_trainer_sets_train_semantics():
    from dinounet_b200 import config
    from dinounet_b200.training import DinoUNetTrainer, DinoUNetTrainer_s
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    try:
        DinoUNetTrainer_s.set_network_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, train_semantics="reference")
        net = DinoUNetTrainer.build_network_architecture("DinoUNet", {}, [], 3, 2, False)
        assert net.train_semantics == "reference"
        DinoUNetTrainer_s.set_network_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)})
        net = DinoUNetTrainer.build_network_architecture("DinoUNet", {}, [], 3, 2, False)
        assert net.train_semantics == "oracle"
    finally:
        DinoUNetTrainer_s.set_network_config(None)
