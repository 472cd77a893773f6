"""CPU: the recomputed extractor segments of the training step (`DinoUNet.train_recompute`, train_path.py).

  * the switch: default off, set through the trainer's `set_network_config`, not part of the state dict, bools only;
  * with a recording stand-in for the native library: the forward issues the same calls with and without recompute, and
    the backward replays exactly the six extractors' forward calls - on the step's matrix-product tier, after the module
    global has gone back to its default - and never the SPM's or the adapter tail's BatchNorm statistics.
"""
import contextlib
import os

import pytest
import torch

from dinounet_b200 import config
from dinounet_b200 import lib as L
from dinounet_b200 import train_path as TP
from oracle import dinounet_oracle as O
from oracle import train_mode_oracle as T

MODEL, B, NCLS = "dinounet_s", 2, 2
#: what one extractor's forward launches (the GEMMs aside): two LayerNorms, the deformable-sampling prologue and kernel,
#: the FFN LayerNorm, the depthwise conv and GELU
EXTRACTOR_CALLS = ["b2u_f32_layernorm", "b2u_f32_layernorm", "b2u_f32_msda_prep", "b2u_msda_forward_f32",
                   "b2u_f32_layernorm", "b2u_f32_dwconv3x3", "b2u_f32_act"]


def _net():
    import dinounet_b200
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    return dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, NCLS, None, MODEL)


def test_switch_defaults_off_and_stays_out_of_the_state_dict():
    net = _net()
    assert net.train_recompute is False
    keys = list(net.state_dict())
    net.train_recompute = True
    assert list(net.state_dict()) == keys
    assert set(keys) == set(O.make_state_dict(MODEL, NCLS))


def test_non_bool_is_rejected_before_anything_runs():
    net = _net().train()
    for bad in (1, "yes", None):
        net.train_recompute = bad
        with pytest.raises(ValueError, match="train_recompute"):
            net(torch.zeros(1, 3, 64, 64))
    from dinounet_b200.training import DinoUNetTrainer_s
    with pytest.raises(ValueError, match="train_recompute"):
        DinoUNetTrainer_s.set_network_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, train_recompute=1)


def test_trainer_sets_train_recompute():
    from dinounet_b200.training import DinoUNetTrainer, DinoUNetTrainer_s
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    arch = {"architecture": dict(config.DEFAULT_ARCHITECTURE)}
    try:
        DinoUNetTrainer_s.set_network_config(arch, train_recompute=True)
        net = DinoUNetTrainer.build_network_architecture("DinoUNet", {}, [], 3, 2, False)
        assert net.train_recompute is True
        DinoUNetTrainer_s.set_network_config(arch, None, None, "default", "reference", False)   # the earlier signature
        net = DinoUNetTrainer.build_network_architecture("DinoUNet", {}, [], 3, 2, False)
        assert net.train_recompute is False and net.train_semantics == "reference"
    finally:
        DinoUNetTrainer_s.set_network_config(None)


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


def _calls(rec, gemm, train_mode, recompute):
    P, x, taps = _inputs()
    rec.calls.clear()
    logits = TP.trainable_forward(P, MODEL, x, taps, NCLS, gemm, train_mode, recompute)
    fwd = [n for n, _ in rec.calls]
    rec.calls.clear()
    logits.sum().backward()
    bwd = [n for n, _ in rec.calls]
    grads = {k for k, t in P.items() if isinstance(t, torch.Tensor) and t.grad is not None}
    return fwd, bwd, grads


def _without(calls, names):
    out = list(calls)
    for n in names:
        out.remove(n)
    return out


@pytest.mark.parametrize("gemm", ["fp32", "tf32"])
@pytest.mark.parametrize("semantics", ["oracle", "reference"])
def test_backward_replays_the_extractors_on_the_step_tier(rec, gemm, semantics):
    mode = None if semantics == "oracle" else TP.TrainMode(bn={p: (0.1, 1e-5) for p in T.BN_LAYERS},
                                                          drop_scale=torch.ones(6, B) / 0.7)
    fwd0, bwd0, grads0 = _calls(rec, gemm, mode, False)
    fwd1, bwd1, grads1 = _calls(rec, gemm, mode, True)
    assert fwd1 == fwd0
    assert grads1 == grads0
    other = "b2u_tf32_gemm" if gemm == "fp32" else "b2u_f32_gemm"
    assert other not in fwd1 + bwd1                          # the replay ran on the step's tier, not the default
    mine = "b2u_tf32_gemm" if gemm == "tf32" else "b2u_f32_gemm"
    # per extractor: value, offsets / weights, output projection, fc1, fc2 (+ the DropPath add under train mode)
    replay = (EXTRACTOR_CALLS + [mine] * 5 + (["b2u_f32_droppath_add"] if mode else [])) * 6
    assert sorted(_without(bwd1, replay)) == sorted(bwd0)
    assert TP._GEMM_TIER == "tf32"
    if mode is not None:                                     # statistics and running-statistic updates happen once
        for n in ("b2u_f32_bn_stats", "b2u_f32_bn_finalize"):
            assert fwd1.count(n) == 10 and n not in bwd1
