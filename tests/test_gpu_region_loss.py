"""-m gpu: fused region Dice+BCE and its validation counts (csrc/loss.cu through dinounet_b200.loss.DC_and_BCE_loss)
against the region-loss oracle (bit-identical to the reference classes, tests/test_region_loss_cpu.py), in fp64.
Tolerances as tests/test_gpu_loss.py: loss within 2e-6 relative, gradient within 1e-5 of max|grad|; counts exact."""
import numpy as np
import pytest
import torch

from dinounet_b200.loss import DC_and_BCE_loss, validation_statistics
from oracle import region_loss_oracle as RO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _mod(batch_dice, ign, **kw):
    return DC_and_BCE_loss({}, {"batch_dice": batch_dice, "do_bg": True, "smooth": 1e-5, "ddp": False},
                           use_ignore_label=ign, **kw)


def _case(B, R, H, W, ign, seed):
    z, t = RO.region_case(B, R, H, W, seed, use_ignore=ign)
    return z.to(DEV), t.to(DEV)


@pytest.mark.parametrize("B,R,H,W", [(2, 1, 512, 512), (3, 2, 33, 17), (2, 3, 512, 512), (1, 5, 33, 17), (2, 8, 64, 96),
                                     (2, 32, 33, 17), (1, 32, 128, 128)])
@pytest.mark.parametrize("ign", [False, True])
@pytest.mark.parametrize("batch_dice", [True, False])
def test_region_loss_and_gradient_match_oracle(B, R, H, W, ign, batch_dice):
    z, t = _case(B, R, H, W, ign, B * 100 + R)
    mod = _mod(batch_dice, ign)
    want = None
    for tt in (t, t.to(torch.uint8), t.long()):
        z1 = z.clone().requires_grad_(True)
        got = mod(z1, tt)
        if want is None:
            z2 = z.double().requires_grad_(True)
            want, _, _ = RO.dc_and_bce_loss(z2, t.double(), batch_dice=batch_dice, use_ignore=ign)
        assert abs(float(got) - float(want)) <= 2e-6 * max(1.0, abs(float(want))), (tt.dtype, float(got), float(want))
        (got * 3.0).backward()
        if z2.grad is None:
            (want * 3.0).backward()
        err = float((z1.grad.double() - z2.grad).abs().max() / z2.grad.abs().max())
        assert err < 1e-5, (tt.dtype, err)


def test_weights_and_determinism():
    z, t = _case(2, 3, 100, 100, True, 7)
    mod = _mod(True, True, weight_ce=0.5, weight_dice=2)
    want, _, _ = RO.dc_and_bce_loss(z.double(), t.double(), batch_dice=True, use_ignore=True, weight_ce=0.5, weight_dice=2)
    z1, z2 = z.clone().requires_grad_(True), z.clone().requires_grad_(True)
    a, b = mod(z1, t), mod(z2, t)
    assert abs(float(a) - float(want)) < 2e-6 * max(1.0, abs(float(want))) and torch.equal(a, b)
    a.backward()
    b.backward()
    assert torch.equal(z1.grad, z2.grad)


def test_all_ignored():
    z, t = RO.region_case(2, 3, 65, 33, 99, use_ignore=True, ignore_all=True)
    z = z.to(DEV).requires_grad_(True)
    loss, out3, counts, _ = _mod(True, True)._run(z, t.to(DEV))
    assert float(out3[1]) == 0.0 and float(out3[2]) == -1.0 and float(loss) == -1.0
    loss.backward()
    assert not z.grad.any()
    assert not counts.any()


@pytest.mark.parametrize("ign", [False, True])
def test_region_validation_counts_match_torch(ign):
    """sigmoid(z) > 0.5 per region, weighted by 1 - t_ign, with logits planted exactly at 0 and at +-1e-7."""
    z, t = _case(4, 3, 128, 96, ign, 11)
    z[0, :, :8, :8] = 0.0
    z[1, :, :8, :8] = 1e-7
    z[2, :, :8, :8] = -1e-7
    mod = _mod(True, ign)
    out = validation_statistics(mod, z, t)
    tp, fp, fn = RO.region_validation_counts(z, t, use_ignore=ign)
    for k, v in (("tp_hard", tp), ("fp_hard", fp), ("fn_hard", fn)):
        assert out[k].dtype == np.float32 and out[k].shape == (3,)
        assert np.array_equal(out[k], v.cpu().numpy()), (k, out[k], v)
    want, _, _ = RO.dc_and_bce_loss(z.double(), t.double(), batch_dice=True, use_ignore=ign)
    assert abs(float(out["loss"]) - float(want)) < 2e-6 * max(1.0, abs(float(want)))


def test_trainer_validation_step_with_regions():
    """`DinoUNetTrainer.validation_step` on the native dinounet_s forward with 3 sigmoid heads, ignore channel on."""
    import os
    from types import SimpleNamespace
    import dinounet_b200
    from dinounet_b200 import config
    from oracle import dinounet_oracle as O
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, 3, None, "dinounet_s")
    net.load_state_dict(O.make_state_dict("dinounet_s", 3, seed=0), strict=True)
    net = net.to(DEV).eval()
    tr = dinounet_b200.DinoUNetTrainer_s.__new__(dinounet_b200.DinoUNetTrainer_s)
    tr.device, tr.network, tr.is_ddp = DEV, net, False
    tr.label_manager = SimpleNamespace(has_regions=True, ignore_label=3, has_ignore_label=True)
    tr.configuration_manager = SimpleNamespace(batch_dice=True)
    tr.loss = tr._build_loss()
    _, t = RO.region_case(2, 3, 256, 256, 5, use_ignore=True)
    batch = {"data": O.make_input(2, 256, 5), "target": t}
    out = tr.validation_step(batch)
    with torch.no_grad():
        logits = net(batch["data"].to(DEV)).float()
    tt = t.to(DEV)
    want, _, _ = RO.dc_and_bce_loss(logits.double(), tt.double(), batch_dice=True, use_ignore=True)
    tp, fp, fn = RO.region_validation_counts(logits, tt, use_ignore=True)
    assert abs(float(out["loss"]) - float(want)) < 2e-6 * max(1.0, abs(float(want)))
    assert np.array_equal(out["tp_hard"], tp.cpu().numpy()) and np.array_equal(out["fp_hard"], fp.cpu().numpy())
    assert np.array_equal(out["fn_hard"], fn.cpu().numpy())
