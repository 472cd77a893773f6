"""Loss oracle (oracle/loss_oracle.py) pinned against what the REAL reference loss classes compute (stored in
tests/golden/reference_cases.npz by oracle/make_golden_reference_cases.py) and against committed known answers;
product-side argument handling that needs no GPU."""
import os

import numpy as np
import pytest
import torch

from oracle import loss_oracle as LO

REF = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_cases.npz"))


def _case(B, C, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, C, H, W, generator=g) * 3, torch.randint(0, C, (B, 1, H, W), generator=g).float()


@pytest.mark.parametrize("batch_dice", [True, False])
def test_loss_oracle_equals_reference_classes(batch_dice):
    """DC_and_CE_loss with MemDice (nnUNetTrainer.py:363-365) and get_tp_fp_fn_tn, bit for bit."""
    for seed, (B, C) in enumerate([(2, 2), (3, 4), (1, 3)]):
        key = f"loss_{int(batch_dice)}_{seed}"
        z, t = _case(B, C, 24, 20, seed)
        z2 = z.clone().requires_grad_(True)
        got, _, _ = LO.dc_and_ce_loss(z2, t, batch_dice=batch_dice)
        assert np.array_equal(got.detach().numpy(), REF[key + "_loss"])
        got.backward()
        g = z2.grad.reshape(-1).numpy()
        assert np.array_equal(g[:: max(1, g.size // 256)][:256], REF[key + "_grad"])
        otp, ofp, ofn = LO.validation_hard_counts(z, t)
        assert np.array_equal(otp.numpy(), REF[key + "_tp"]) and np.array_equal(ofp.numpy(), REF[key + "_fp"])
        assert np.array_equal(ofn.numpy(), REF[key + "_fn"])


def test_loss_oracle_known_answers():
    """Hand-checkable cases: a perfect confident prediction -> CE ~ 0, dice term ~ -1; uniform logits -> CE = ln C."""
    t = torch.zeros(1, 1, 4, 4)
    t[..., 2:] = 1
    z = torch.zeros(1, 2, 4, 4)
    z[:, 0] = torch.where(t[:, 0] == 0, 30.0, -30.0)
    z[:, 1] = -z[:, 0]
    loss, ce, dc = LO.dc_and_ce_loss(z, t)
    assert abs(float(ce)) < 1e-6 and abs(float(dc) + 1) < 1e-6 and abs(float(loss) + 1) < 1e-6
    loss, ce, dc = LO.dc_and_ce_loss(torch.zeros(2, 4, 8, 8), torch.zeros(2, 1, 8, 8))
    assert abs(float(ce) - np.log(4)) < 1e-6
    # no foreground at all: every fg class has I=0, G=0, P=N/4 -> dc_c = s / (P + s)
    assert abs(float(dc) + 1e-5 / (2 * 64 / 4 + 1e-5)) < 1e-9
    tp, fp, fn = LO.validation_hard_counts(z, t)
    assert tp.tolist() == [8, 8] and fp.tolist() == [0, 0] and fn.tolist() == [0, 0]


def test_product_loss_argument_contract():
    from dinounet_b200.loss import DC_and_CE_loss
    from dinounet_b200.lib import NativeLibraryError
    with pytest.raises(NotImplementedError):
        DC_and_CE_loss({"batch_dice": True}, {}, ignore_label=3)
    m = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, weight_ce=1, weight_dice=1)
    assert m.batch_dice and not m.do_bg and m.smooth == 1e-5
    with pytest.raises(NativeLibraryError):
        m(torch.zeros(1, 2, 4, 4), torch.zeros(1, 1, 4, 4))      # CPU tensors: no fallback
