"""Region-loss and data-parallel batch-Dice oracle (oracle/region_loss_oracle.py) pinned bit for bit against what the REAL
reference classes computed (tests/golden/region_loss_cases.npz, oracle/make_golden_region_loss.py), including both ranks
of a 2-process gloo run; the product-side argument contract and the trainer's loss construction, without a GPU."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import region_loss_oracle as RO

REF = np.load(os.path.join(os.path.dirname(__file__), "golden", "region_loss_cases.npz"))


@pytest.mark.parametrize("seed,case", list(enumerate(RO.REGION_CASES)))
def test_region_oracle_equals_reference_classes(seed, case):
    """DC_and_BCE_loss (nnUNetTrainer.py:356-361) and validation_step's region counts, bit for bit."""
    bd, ign, R = case
    B, H, W = RO.REGION_SHAPE
    z, t = RO.region_case(B, R, H, W, seed, use_ignore=ign)
    key = f"bce_{int(bd)}_{int(ign)}_{R}"
    z1 = z.clone().requires_grad_(True)
    got, _, _ = RO.dc_and_bce_loss(z1, t, batch_dice=bd, use_ignore=ign)
    assert np.array_equal(got.detach().numpy(), REF[key + "_loss"])
    got.backward()
    assert np.array_equal(RO.strided(z1.grad).numpy(), REF[key + "_grad"])
    tp, fp, fn = RO.region_validation_counts(z, t, use_ignore=ign)
    for name, v in (("tp", tp), ("fp", fp), ("fn", fn)):
        assert v.dtype == torch.float32 and np.array_equal(v.numpy(), REF[f"{key}_{name}"]), name


def test_region_oracle_all_ignored():
    B, H, W = RO.REGION_SHAPE
    z, t = RO.region_case(B, 3, H, W, 99, use_ignore=True, ignore_all=True)
    z1 = z.clone().requires_grad_(True)
    loss, bce, dc = RO.dc_and_bce_loss(z1, t, batch_dice=True, use_ignore=True)
    assert np.array_equal(loss.detach().numpy(), REF["allign_loss"])
    assert float(bce.detach()) == 0.0 and float(dc.detach()) == -1.0
    loss.backward()
    assert np.array_equal(RO.strided(z1.grad).numpy(), REF["allign_grad"]) and not z1.grad.any()


@pytest.mark.parametrize("kind", ["bce", "ce"])
def test_ddp_oracle_equals_gloo_reference(kind):
    """W ranks simulated in one process == the reference's AllGatherGrad run on 2 gloo processes, both ranks."""
    shards = [RO.ddp_shard(kind, r) for r in range(RO.DDP_WORLD)]
    zs = [z.clone().requires_grad_(True) for z, _ in shards]
    losses = RO.ddp_losses(kind, zs, [t for _, t in shards], use_ignore=kind == "bce")
    sum(s * l for s, l in zip(RO.DDP_SCALES, losses)).backward()
    for r in range(RO.DDP_WORLD):
        assert np.array_equal(losses[r].detach().numpy(), REF[f"ddp_{kind}_{r}_loss"]), r
        assert np.array_equal(RO.strided(zs[r].grad).numpy(), REF[f"ddp_{kind}_{r}_grad"]), r


def test_ddp_oracle_one_rank_is_the_plain_loss():
    z, t = RO.region_case(2, 3, 16, 16, 4, use_ignore=True)
    (a,) = RO.ddp_losses("bce", [z], [t], use_ignore=True)
    assert torch.equal(a, RO.dc_and_bce_loss(z, t, batch_dice=True, use_ignore=True)[0])


def test_region_loss_argument_contract():
    from dinounet_b200.lib import NativeLibraryError
    from dinounet_b200.loss import DC_and_BCE_loss, DC_and_CE_loss
    with pytest.raises(NotImplementedError):
        DC_and_BCE_loss({"pos_weight": torch.ones(1)}, {"batch_dice": True})
    with pytest.raises(NotImplementedError):
        DC_and_BCE_loss({}, {"batch_dice": True, "square": True})
    with pytest.raises(NotImplementedError):
        DC_and_BCE_loss({}, {"batch_dice": True, "do_bg": False})
    with pytest.raises(NotImplementedError):
        DC_and_CE_loss({"batch_dice": True}, {}, ignore_label=3)
    m = DC_and_BCE_loss({}, {"batch_dice": True, "do_bg": True, "smooth": 1e-5, "ddp": False}, use_ignore_label=True)
    assert m.batch_dice and m.do_bg and m.smooth == 1e-5 and m.use_ignore_label and not m.ddp
    with pytest.raises(NativeLibraryError):
        m(torch.zeros(1, 2, 4, 4), torch.zeros(1, 3, 4, 4))      # CPU tensors: no fallback


@pytest.mark.parametrize("ignore_label", [None, 4])
@pytest.mark.parametrize("is_ddp", [False, True])
@pytest.mark.parametrize("batch_dice", [False, True])
def test_trainer_builds_reference_region_loss(ignore_label, is_ddp, batch_dice):
    """`_build_loss` with regions: DC_and_BCE_loss({}, {batch_dice, do_bg True, smooth 1e-5, ddp}, use_ignore_label)
    (nnUNetTrainer.py:356-361); label maps keep DC_and_CE_loss with the trainer's ddp flag."""
    import dinounet_b200
    from dinounet_b200.loss import DC_and_BCE_loss, DC_and_CE_loss
    tr = dinounet_b200.DinoUNetTrainer_s.__new__(dinounet_b200.DinoUNetTrainer_s)
    tr.is_ddp = is_ddp
    tr.configuration_manager = SimpleNamespace(batch_dice=batch_dice)
    tr.label_manager = SimpleNamespace(has_regions=True, ignore_label=ignore_label,
                                       has_ignore_label=ignore_label is not None)
    m = tr._build_loss()
    assert isinstance(m, DC_and_BCE_loss)
    assert (m.batch_dice, m.do_bg, m.smooth, m.ddp) == (batch_dice, True, 1e-5, is_ddp)
    assert (m.weight_ce, m.weight_dice, m.use_ignore_label) == (1, 1, ignore_label is not None)
    tr.label_manager = SimpleNamespace(has_regions=False, ignore_label=None, has_ignore_label=False)
    m = tr._build_loss()
    assert isinstance(m, DC_and_CE_loss) and (m.batch_dice, m.do_bg, m.ddp) == (batch_dice, False, is_ddp)
