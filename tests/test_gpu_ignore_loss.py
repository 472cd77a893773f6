"""-m gpu: fused Dice+CE with an ignore label (csrc/loss.cu through dinounet_b200.loss.DC_and_CE_loss(ignore_label=...))
against the reference's own numbers (tests/golden/ignore_loss_cases.npz) and the ignore-label oracle (bit-identical to the
reference classes, tests/test_ignore_loss_cpu.py) in fp64.  Tolerances as tests/test_gpu_loss.py: loss within 2e-6
relative, gradient within 1e-5 of max|grad|; counts exact.  The gradient at ignored pixels must be exactly 0.0, and the
logits there must not reach the loss or the gradient elsewhere at all (bitwise)."""
import os

import numpy as np
import pytest
import torch

from dinounet_b200.loss import DC_and_CE_loss, validation_statistics
from oracle import ignore_loss_oracle as IO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
REF = np.load(os.path.join(os.path.dirname(__file__), "golden", "ignore_loss_cases.npz"))
DTYPES = (torch.float32, torch.uint8, torch.int32, torch.int64)


def _mod(batch_dice, ignore_label, **kw):
    return DC_and_CE_loss({"batch_dice": batch_dice, "smooth": 1e-5, "do_bg": False, "ddp": False}, {},
                          ignore_label=ignore_label, **kw)


def _check_golden(key, z, t, C, batch_dice):
    mod = _mod(batch_dice, C)
    want, gref = float(REF[key + "_loss"]), REF[key + "_grad"]
    for dt in DTYPES:
        z1 = z.to(DEV).requires_grad_(True)
        tt = t.to(DEV).to(dt)
        got = mod(z1, tt)
        assert abs(float(got.detach()) - want) <= 2e-6 * max(1.0, abs(want)), (dt, float(got.detach()), want)
        got.backward()
        g = IO.strided(z1.grad).cpu().numpy()
        scale = max(float(np.abs(gref).max()), 1e-30)
        assert float(np.abs(g - gref).max()) <= 1e-5 * scale, (dt, float(np.abs(g - gref).max()), scale)
        ign = (tt == C).expand_as(z1)
        assert not z1.grad[ign].any(), dt
        out = validation_statistics(mod, z.to(DEV), tt)
        for name in ("tp", "fp", "fn"):
            assert np.array_equal(out[name + "_hard"], REF[f"{key}_{name}"][1:]), (dt, name)
    return z1.grad, mod._run(z.to(DEV), t.to(DEV))[1]


@pytest.mark.parametrize("seed,case", list(enumerate(IO.IGN_CASES)))
def test_matches_reference_golden(seed, case):
    bd, C = case
    B, H, W = IO.IGN_SHAPE
    z, t = IO.ignore_case(B, C, H, W, seed)
    _check_golden(f"ign_{int(bd)}_{C}", z, t, C, bd)


def test_one_sample_ignored_matches_golden():
    B, H, W = IO.IGN_SHAPE
    z, t = IO.ignore_case(B, IO.EDGE_C, H, W, 98, ignored_samples=(1,))
    grad, _ = _check_golden("onesample", z, t, IO.EDGE_C, False)
    assert not grad[1].any() and grad[0].any()


def test_all_ignored_matches_golden():
    B, H, W = IO.IGN_SHAPE
    z, t = IO.ignore_case(B, IO.EDGE_C, H, W, 99, ignored_samples=range(B))
    grad, out3 = _check_golden("allign", z, t, IO.EDGE_C, True)
    assert float(out3[1]) == 0.0 and float(out3[2]) == -1.0 and float(out3[0]) == -1.0
    assert not grad.any()


@pytest.mark.parametrize("B,C,H,W", [(2, 2, 512, 512), (3, 4, 96, 200), (1, 3, 33, 17), (4, 16, 64, 64), (2, 5, 127, 129),
                                     (2, 7, 63, 97), (1, 21, 129, 127), (2, 32, 65, 63)])
@pytest.mark.parametrize("batch_dice", [True, False])
def test_class_counts_match_fp64_oracle(B, C, H, W, batch_dice):
    z, t = IO.ignore_case(B, C, H, W, B * 100 + C)
    z, t = z.to(DEV), t.to(DEV)
    z1 = z.clone().requires_grad_(True)
    got = _mod(batch_dice, C)(z1, t)
    z2 = z.double().requires_grad_(True)
    want, _, _ = IO.dc_and_ce_loss(z2, t, C, batch_dice=batch_dice)
    g, w = float(got.detach()), float(want.detach())
    assert abs(g - w) <= 2e-6 * max(1.0, abs(w)), (g, w)
    (got * 3.0).backward()
    (want * 3.0).backward()
    err = float((z1.grad.double() - z2.grad).abs().max() / z2.grad.abs().max())
    assert err < 1e-5, err


@pytest.mark.parametrize("ignore_label", [3, 255, 0])
def test_ignored_pixels_do_not_reach_the_loss(ignore_label):
    """Gradient exactly 0.0 at ignored pixels; other logits there change no bit of the loss or of the gradient
    elsewhere; two launches give identical bits.  Also an ignore label inside [0, C) and one far outside it."""
    C = 3
    z, t = IO.ignore_case(2, C, 100, 100, 7, ignore_label=ignore_label)
    z, t = z.to(DEV), t.to(DEV)
    ign = (t == ignore_label).expand_as(z)
    mod = _mod(True, ignore_label, weight_ce=0.5, weight_dice=2)
    want, _, _ = IO.dc_and_ce_loss(z.double(), t, ignore_label, batch_dice=True, weight_ce=0.5, weight_dice=2)
    grads, losses = [], []
    for zz in (z, z, torch.where(ign, torch.randn_like(z) * 50, z)):
        z1 = zz.clone().requires_grad_(True)
        loss = mod(z1, t)
        loss.backward()
        losses.append(loss.detach())
        grads.append(z1.grad)
    assert abs(float(losses[0]) - float(want)) < 2e-6 * max(1.0, abs(float(want)))
    assert (grads[0][ign] == 0).all() and not torch.signbit(grads[0][ign]).any()
    assert torch.equal(losses[0], losses[1]) and torch.equal(grads[0], grads[1])
    assert torch.equal(losses[0], losses[2]) and torch.equal(grads[0], grads[2])


def test_labels_are_checked_except_the_ignore_label():
    C = 3
    z, t = IO.ignore_case(2, C, 64, 64, 11)
    z, t = z.to(DEV), t.to(DEV)
    mod = _mod(True, C)
    mod.check_labels = True
    mod(z, t)                                      # label C is the ignore label: accepted
    for stray in (C + 1, -1):
        bad = t.clone()
        bad[1, 0, 5, 7] = stray
        with pytest.raises(RuntimeError):
            mod(z, bad)
        with pytest.raises(RuntimeError):
            validation_statistics(_mod(True, C), z, bad)


def _trainer(net, ignore_label):
    from types import SimpleNamespace
    import dinounet_b200
    tr = dinounet_b200.DinoUNetTrainer_s.__new__(dinounet_b200.DinoUNetTrainer_s)
    tr.device, tr.network, tr.is_ddp = DEV, net, False
    tr.label_manager = SimpleNamespace(has_regions=False, ignore_label=ignore_label, has_ignore_label=True)
    tr.configuration_manager = SimpleNamespace(batch_dice=True)
    tr.loss = tr._build_loss()
    return tr


def _net(train=False):
    import dinounet_b200
    from dinounet_b200 import config
    from oracle import dinounet_oracle as O
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, 2, None, "dinounet_s")
    net.load_state_dict(O.make_state_dict("dinounet_s", 2, seed=0), strict=True)
    if train:
        net.precision = "fp32"
        net.train_gemm = "fp32"
        return net.to(DEV).train()
    return net.to(DEV).eval()


def test_trainer_validation_step_with_ignore_label():
    """`DinoUNetTrainer.validation_step` on the native dinounet_s forward, C = 2, ignore label 2."""
    from oracle import dinounet_oracle as O
    net = _net()
    tr = _trainer(net, 2)
    _, t = IO.ignore_case(2, 2, 256, 256, 5)
    batch = {"data": O.make_input(2, 256, 5), "target": t}
    out = tr.validation_step(batch)
    with torch.no_grad():
        logits = net(batch["data"].to(DEV)).float()
    tt = t.to(DEV)
    want, _, _ = IO.dc_and_ce_loss(logits.double(), tt, 2, batch_dice=True)
    tp, fp, fn = IO.validation_counts(logits, tt, 2)
    assert abs(float(out["loss"]) - float(want)) < 2e-6 * max(1.0, abs(float(want)))
    for k, v in (("tp_hard", tp), ("fp_hard", fp), ("fn_hard", fn)):
        assert np.array_equal(out[k], v.cpu().numpy()[1:]), (k, out[k], v)


def test_trainer_train_step_with_ignore_label():
    """One native `train_step` (train_gemm "fp32") with the trainer's fused ignore-label loss == the same step with the
    oracle loss in torch autograd on the native network: max|d_fused - d_oracle| <= 1e-4 * max|d_oracle| (the training
    backward accumulates with atomics, so the bits differ)."""
    from dinounet_b200.train_path import FusedSGD, train_step
    from oracle import dinounet_oracle as O
    x = O.make_input(2, 128, 9)
    _, t = IO.ignore_case(2, 2, 128, 128, 10)

    def delta(loss_fn):
        net = _net(train=True)
        before = {n: p.detach().clone() for n, p in net.named_parameters() if p.requires_grad}
        train_step(net, loss_fn, FusedSGD(net.parameters(), lr=1e-2), x.to(DEV), t.to(DEV))
        return torch.cat([(p.detach() - before[n]).reshape(-1) for n, p in net.named_parameters() if n in before])

    fused = delta(_trainer(None, 2).loss)
    ref = delta(lambda logits, target: IO.dc_and_ce_loss(logits.float(), target, 2, batch_dice=True)[0])
    err = float((fused - ref).abs().max() / ref.abs().max())
    print("fused ignore-label loss vs oracle loss, one train_step: max|d_f - d_o| / max|d_o| =", err)
    assert err <= 1e-4, err
