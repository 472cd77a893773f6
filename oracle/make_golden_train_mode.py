"""TEST INFRASTRUCTURE — writes tests/golden/train_mode_cases.npz: one TRAIN-MODE training step of the REAL reference
(dinounet_s, B=2, 128x128, 2 classes, CPU, fp32) that tests/test_train_mode_cpu.py and tests/test_gpu_train_mode.py
compare the train-mode restatement (oracle/train_mode_oracle.py) and the native path against.
Run where the reference is importable (oracle/ref_loader.py):  python oracle/make_golden_train_mode.py

The CPU generator is seeded, then the reference's draw order is replayed to record what it will draw: one 1-element
uniform per ViT block (rope_position_encoding.py:93-97, vision_transformer.py:271-272), then one (B, 1, 1) Bernoulli(0.7)
per extractor (dinov3_adapter.py:18-27).  The generator is re-seeded and the reference runs in .train().
Contents: rope_scales [depth], drop_keep [6, B]; loss, names, norms, s<i> (the grads_*.npz format: per trainable tensor its
gradient norm and 16 strided samples); for each of the 10 BatchNorm layers (order: train_mode_oracle.BN_LAYERS) the
updated running statistics rm<j>, rv<j> and num_batches_tracked nbt<j>.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import dinounet_oracle as O  # noqa: E402
from oracle import grad_oracle as G  # noqa: E402
from oracle import loss_oracle as LO  # noqa: E402
from oracle import train_mode_oracle as T  # noqa: E402
from oracle.ref_loader import build_reference_model, load_reference_module  # noqa: E402

MODEL, B, S, NCLS, WSEED, DRAW_SEED = "dinounet_s", 2, 128, 2, 0, 5


def replay_draws(seed: int):
    """What the reference draws in a train-mode forward after torch.manual_seed(seed), in its order."""
    torch.manual_seed(seed)
    depth = O.VARIANTS[MODEL].depth
    scales = torch.cat([torch.empty(1, dtype=torch.float32).uniform_(-np.log(2), np.log(2)).exp() for _ in range(depth)])
    keep = torch.stack([torch.empty((B, 1, 1), dtype=torch.float32).bernoulli_(T.DROP_KEEP).reshape(B) for _ in range(6)])
    return scales, keep


def main():
    sd = O.make_state_dict(MODEL, NCLS, seed=WSEED)
    x = O.make_input(B, S, WSEED)
    target = torch.randint(0, NCLS, (B, 1, S, S), generator=torch.Generator().manual_seed(WSEED + 7)).float()
    scales, keep = replay_draws(DRAW_SEED)
    assert (keep == 0).any() and (keep == 1).any(), keep

    net = build_reference_model(MODEL, NCLS, sd).train()
    load_reference_module()
    msda_mod = sys.modules["dinounet.dinov3.eval.segmentation.models.utils.ms_deform_attn"]
    DC_and_CE_loss, MemDice, _ = LO.load_reference_loss()

    class _Differentiable:                                 # the extension-backed backward cannot run on CPU
        @staticmethod
        def apply(value, shapes, lsi, loc, aw, step):
            return msda_mod.ms_deform_attn_core_pytorch(value, shapes, loc, aw)

    orig = msda_mod.MSDeformAttnFunction
    msda_mod.MSDeformAttnFunction = _Differentiable
    try:
        crit = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, weight_ce=1,
                              weight_dice=1, ignore_label=None, dice_class=MemDice)
        torch.manual_seed(DRAW_SEED)
        loss = crit(net(x), target)
        after_fwd = torch.get_rng_state()
        loss.backward()
    finally:
        msda_mod.MSDeformAttnFunction = orig
    # the forward consumed exactly the replayed draws
    replay_draws(DRAW_SEED)
    assert torch.equal(after_fwd, torch.get_rng_state()), "the reference drew more or less than the replayed sequence"

    sdv = net.state_dict(keep_vars=True)
    names = sorted(G.trainable_keys(MODEL, NCLS))
    out = {"rope_scales": scales.numpy(), "drop_keep": keep.numpy(), "loss": np.float64(loss.item()), "names": np.array(names)}
    grads = [sdv[k].grad if sdv[k].grad is not None else torch.zeros_like(sdv[k]) for k in names]
    out["norms"] = np.array([g.double().norm().item() for g in grads])
    for i, g in enumerate(grads):
        f = g.reshape(-1)
        out[f"s{i}"] = f[:: max(1, f.numel() // 16)][:16].detach().numpy().astype(np.float32)
    for j, p in enumerate(T.BN_LAYERS):
        out[f"rm{j}"] = sdv[p + ".running_mean"].detach().numpy().copy()
        out[f"rv{j}"] = sdv[p + ".running_var"].detach().numpy().copy()
        out[f"nbt{j}"] = np.int64(sdv[p + ".num_batches_tracked"].item())
    path = os.path.join(ROOT, "tests", "golden", "train_mode_cases.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes; loss", float(loss), "scales", scales.numpy().round(3), "keep", keep.numpy())


if __name__ == "__main__":
    main()
