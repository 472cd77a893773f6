"""TEST INFRASTRUCTURE — writes tests/golden/deep_supervision_cases.npz: one deep-supervision training objective of the
REAL reference (DinoUNet with deep_supervision=True, dinounet_s, B=2, 128x128, 2 output channels, CPU, fp32, eval-mode
modules as the gradient goldens) for tests/test_deep_supervision_cpu.py and tests/test_gpu_deep_supervision.py.
Run where the reference is importable (oracle/ref_loader.py):  python oracle/make_golden_deep_supervision.py

The network is built by ref_loader.build_reference_model and its decoder's `deep_supervision` flag is set, which is what
DinoUNet.from_config does with architecture["deep_supervision"] = True (dinounet_training.py:560-629).  The targets are
downsampled by the restatement in oracle/deep_supervision_oracle.py at the plan's scales [1, 1/2, 1/4], and the loss is
the reference's DeepSupervisionWrapper (training/loss/deep_supervision.py) with the weights [2/3, 1/3, 0].
Cases (prefix): "lm" = DC_and_CE_loss (batch Dice, no background) on a label map; "rg" = DC_and_BCE_loss with an ignore
channel on two regions (labels {1, 2} and {2}) + ignore channel (label 3) of a label map in 0..3.
Contents: logits0..2 (the forward's three outputs, highest resolution first), weights; per case <p>_loss, <p>_names,
<p>_norms, <p>_has_grad and <p>_s<i> (the grads_*.npz format: per trainable tensor its gradient norm and 16 strided
samples; a tensor without a gradient, seg_layers.0, has has_grad False, norm 0).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import deep_supervision_oracle as DSO  # noqa: E402
from oracle import dinounet_oracle as O  # noqa: E402
from oracle import grad_oracle as G  # noqa: E402
from oracle import region_loss_oracle as RO  # noqa: E402
from oracle.ref_loader import build_reference_model, load_reference_module  # noqa: E402

MODEL, B, S, NCLS, WSEED = "dinounet_s", 2, 128, 2, 0
SCALES = [[1.0, 1.0], [0.5, 0.5], [0.25, 0.25]]


def label_map():
    return torch.randint(0, NCLS, (B, 1, S, S), generator=torch.Generator().manual_seed(WSEED + 7)).float()


def region_target():
    """[B, 3, S, S] float: regions {1, 2} and {2} of a label map in 0..3, then the ignore channel (label 3)."""
    lab = torch.randint(0, 4, (B, 1, S, S), generator=torch.Generator().manual_seed(WSEED + 11))
    return torch.cat([((lab == 1) | (lab == 2)), lab == 2, lab == 3], 1).float()


def targets(t: torch.Tensor):
    return [torch.from_numpy(a) for a in DSO.downsample_seg_for_ds(t.numpy(), SCALES)]


def _load_ds_wrapper():
    load_reference_module()
    RO.load_reference_region_loss()                 # puts the reference's training/ on the package path
    from dinounet.training.loss.deep_supervision import DeepSupervisionWrapper
    return DeepSupervisionWrapper


def main():
    sd = O.make_state_dict(MODEL, NCLS, seed=WSEED)
    x = O.make_input(B, S, WSEED)
    load_reference_module()
    msda_mod = sys.modules["dinounet.dinov3.eval.segmentation.models.utils.ms_deform_attn"]
    DC_and_BCE_loss, DC_and_CE_loss, MemDice, _ = RO.load_reference_region_loss()
    DeepSupervisionWrapper = _load_ds_wrapper()
    weights = DSO.ds_weights(len(SCALES), ddp=False)

    class _Differentiable:                                 # the extension-backed backward cannot run on CPU
        @staticmethod
        def apply(value, shapes, lsi, loc, aw, step):
            return msda_mod.ms_deform_attn_core_pytorch(value, shapes, loc, aw)

    cases = {
        "lm": (DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, weight_ce=1,
                              weight_dice=1, ignore_label=None, dice_class=MemDice), label_map()),
        "rg": (DC_and_BCE_loss({}, {"batch_dice": True, "do_bg": True, "smooth": 1e-5, "ddp": False},
                               use_ignore_label=True, dice_class=MemDice), region_target()),
    }
    out = {"weights": weights}
    names = sorted(G.trainable_keys(MODEL, NCLS))
    orig = msda_mod.MSDeformAttnFunction
    msda_mod.MSDeformAttnFunction = _Differentiable
    try:
        for prefix, (crit, target) in cases.items():
            net = build_reference_model(MODEL, NCLS, sd)      # eval-mode modules
            net.decoder.deep_supervision = True
            outputs = net(x)
            assert isinstance(outputs, list) and [tuple(o.shape[2:]) for o in outputs] == [(S, S), (S // 2, S // 2), (S // 4, S // 4)]
            for i, o in enumerate(outputs):
                out[f"logits{i}"] = o.detach().numpy()
            loss = DeepSupervisionWrapper(crit, weights)(outputs, targets(target))
            loss.backward()
            sdv = net.state_dict(keep_vars=True)
            has = [sdv[k].grad is not None for k in names]
            grads = [sdv[k].grad if sdv[k].grad is not None else torch.zeros_like(sdv[k]) for k in names]
            assert not has[names.index("decoder.seg_layers.0.weight")]
            out[f"{prefix}_loss"] = np.float64(loss.item())
            out[f"{prefix}_names"] = np.array(names)
            out[f"{prefix}_has_grad"] = np.array(has)
            out[f"{prefix}_norms"] = np.array([g.double().norm().item() for g in grads])
            for i, g in enumerate(grads):
                f = g.reshape(-1)
                out[f"{prefix}_s{i}"] = f[:: max(1, f.numel() // 16)][:16].detach().numpy().astype(np.float32)
            print(prefix, "loss", float(loss))
    finally:
        msda_mod.MSDeformAttnFunction = orig
    path = os.path.join(ROOT, "tests", "golden", "deep_supervision_cases.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
