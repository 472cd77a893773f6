"""TEST INFRASTRUCTURE — writes tests/golden/reference_cases.npz: what the REAL reference computes for the cases that
tests/test_oracle_vs_reference.py, tests/test_loss_cpu.py, tests/test_grad_oracle_cpu.py and
tests/test_sliding_window_cpu.py compare the oracle against, so that those comparisons run without the reference.
Run where the reference is importable (oracle/ref_loader.py):  python oracle/make_golden_reference_cases.py
Contents (values exactly as the reference returned them; large tensors as SAMPLES = strided samples of the flattened tensor):
  fwd_<model>, spec_<model>      forward logits of the parity cases (SAMPLES values + the packed argmax map, 2 classes) and
                                 the SHA-256 of the reference state-dict's sorted (key, shape) list as JSON (spec_json);
                                 fwd_single_channel: the 1-channel input path
  loss_<bd>_<i>_{loss,grad,tp,fp,fn}   DC_and_CE_loss value, d loss / d logits (SAMPLES values), hard validation counts
  grad_loss, grad_names, grad_none, grad_max, grad_samp   reference autograd of dinounet_s: loss, SHA-256 of the sorted
                                 trainable parameter names as JSON, per parameter: gradient is None, max |g| and
                                 16 strided samples per trainable parameter
  sw_<i>                         the reference sliding-window predictor around the toy network (SAMPLES values)
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import dinounet_oracle as O  # noqa: E402
from oracle import loss_oracle as LO  # noqa: E402
from oracle.ref_loader import build_reference_model, load_reference_module  # noqa: E402

FWD_CASES = [("dinounet_s", 128), ("dinounet_b", 64), ("dinounet_7b_tiny", 64)]
LOSS_SHAPES = [(2, 2), (3, 4), (1, 3)]
SW_CASES = [((3, 2, 70, 45), (32, 32), 0.5, True, (0, 1)), ((1, 1, 100, 100), (64, 64), 0.3, True, (0,))]
GRAD_SAMPLES = 16
SAMPLES = 1024


def loss_case(B, C, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, C, H, W, generator=g) * 3, torch.randint(0, C, (B, 1, H, W), generator=g).float()


def grad_case(model, B, S, ncls, seed):
    sd = O.make_state_dict(model, ncls, seed=seed)
    x = O.make_input(B, S, seed)
    target = torch.randint(0, ncls, (B, 1, S, S), generator=torch.Generator().manual_seed(seed + 7)).float()
    return sd, x, target


def strided(t, n):
    f = t.detach().reshape(-1)
    return f[:: max(1, f.numel() // n)][:n]


def spec_json(obj):
    return json.dumps(obj).encode()


def sha(obj):
    return np.frombuffer(hashlib.sha256(spec_json(obj)).digest(), dtype=np.uint8)


def main():
    out = {}
    with torch.no_grad():
        for model, size in FWD_CASES:
            sd = O.make_state_dict(model, 2, seed=3)
            net = build_reference_model(model, 2)
            out[f"spec_{model}"] = sha(sorted([k, list(t.shape)] for k, t in net.state_dict().items()))
            net.load_state_dict(sd, strict=True)
            y = net(O.make_input(2, size, 5))
            out[f"fwd_{model}"], out[f"fwd_{model}_argmax"] = strided(y, SAMPLES).numpy(), np.packbits(y.argmax(1).numpy())
        sd = O.make_state_dict("dinounet_s", 2, seed=3)
        net = build_reference_model("dinounet_s", 2, sd)
        y = net(O.make_input(1, 64, 7, channels=1))
        out["fwd_single_channel"], out["fwd_single_channel_argmax"] = strided(y, SAMPLES).numpy(), np.packbits(y.argmax(1).numpy())

    DC_and_CE_loss, MemDice, get_tp_fp_fn_tn = LO.load_reference_loss()
    for bd in (True, False):
        ref = DC_and_CE_loss({"batch_dice": bd, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, weight_ce=1,
                             weight_dice=1, ignore_label=None, dice_class=MemDice)
        for seed, (B, C) in enumerate(LOSS_SHAPES):
            z, t = loss_case(B, C, 24, 20, seed)
            z1 = z.clone().requires_grad_(True)
            want = ref(z1, t)
            want.backward()
            pred = torch.zeros_like(z).scatter_(1, z.argmax(1)[:, None], 1)
            tp, fp, fn, _ = get_tp_fp_fn_tn(pred, t, axes=[0, 2, 3], mask=None)
            key = f"loss_{int(bd)}_{seed}"
            out[key + "_loss"], out[key + "_grad"] = want.detach().numpy(), strided(z1.grad, SAMPLES // 4).numpy()
            out[key + "_tp"], out[key + "_fp"], out[key + "_fn"] = tp.numpy(), fp.numpy(), fn.numpy()

    model, ncls = "dinounet_s", 2
    sd, x, target = grad_case(model, 1, 128, ncls, 3)
    net = build_reference_model(model, ncls, sd)          # eval mode: BN running stats, DropPath off
    load_reference_module()
    msda_mod = sys.modules["dinounet.dinov3.eval.segmentation.models.utils.ms_deform_attn"]

    class _Differentiable:                                 # the extension-backed backward cannot run on CPU
        @staticmethod
        def apply(value, shapes, lsi, loc, aw, step):
            return msda_mod.ms_deform_attn_core_pytorch(value, shapes, loc, aw)

    orig = msda_mod.MSDeformAttnFunction
    msda_mod.MSDeformAttnFunction = _Differentiable
    try:
        crit = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, weight_ce=1,
                              weight_dice=1, ignore_label=None, dice_class=MemDice)
        loss_ref = crit(net(x), target)
        loss_ref.backward()
    finally:
        msda_mod.MSDeformAttnFunction = orig
    ref = sorted((n, p.grad) for n, p in net.named_parameters() if p.requires_grad)
    out["grad_loss"] = loss_ref.detach().numpy()
    out["grad_names"] = sha([n for n, _ in ref])
    out["grad_none"] = np.array([g is None for _, g in ref], dtype=np.uint8)
    out["grad_max"] = np.array([0.0 if g is None else float(g.abs().max()) for _, g in ref], dtype=np.float32)
    out["grad_samp"] = np.stack([np.zeros(GRAD_SAMPLES, np.float32) if g is None else
                                 np.pad(strided(g, GRAD_SAMPLES).numpy(), (0, max(0, GRAD_SAMPLES - g.numel())))
                                 for _, g in ref])

    from oracle.make_golden_sliding_window import reference_loop
    for seed, (shape, patch, step, ug, ma) in enumerate(SW_CASES):
        _, want = reference_loop(shape, patch, step, ug, ma, heads=3, seed=seed + 5)
        out[f"sw_{seed}"] = strided(want, SAMPLES).numpy()

    path = os.path.join(ROOT, "tests", "golden", "reference_cases.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
