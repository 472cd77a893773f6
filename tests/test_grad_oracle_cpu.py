"""Gradient oracle (oracle/grad_oracle.py = autograd through the oracle forward + loss oracle), the backward target:
pinned against autograd through the REAL reference module + REAL reference loss (stored in
tests/golden/reference_cases.npz by oracle/make_golden_reference_cases.py), and against committed golden gradient
norms / samples."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import dinounet_oracle as O
from oracle import grad_oracle as G
from oracle.make_golden_reference_cases import sha

REF = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_cases.npz"))


def _case(model, B, S, ncls, seed):
    sd = O.make_state_dict(model, ncls, seed=seed)
    x = O.make_input(B, S, seed)
    target = torch.randint(0, ncls, (B, 1, S, S), generator=torch.Generator().manual_seed(seed + 7)).float()
    return sd, x, target


def test_grad_oracle_matches_golden():
    files = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "grads_*.npz")))
    assert files
    for f in files:
        model, b, s, c, w = os.path.basename(f)[len("grads_"):-4].rsplit("_", 4)
        g = np.load(f)
        sd, x, target = _case(model, int(b[1:]), int(s[1:]), int(c[1:]), int(w[1:]))
        loss, grads = G.loss_and_grads(sd, model, x, target)
        assert abs(loss.item() - float(g["loss"])) < 1e-6
        names = [str(n) for n in g["names"]]
        assert names == sorted(grads)
        norms = np.array([grads[k].double().norm().item() for k in names])
        assert np.allclose(norms, g["norms"], rtol=1e-4, atol=1e-9)
        for i, k in enumerate(names):
            fl = grads[k].reshape(-1)
            samp = fl[:: max(1, fl.numel() // 16)][:16].numpy()
            assert np.allclose(samp, g[f"s{i}"], rtol=1e-3, atol=1e-7), k


def test_grad_oracle_equals_reference_autograd():
    """Reference autograd (eval mode, its pure-PyTorch deformable-attention core) of dinounet_s: loss, the trainable
    parameter set, max |g| per parameter and 16 strided gradient samples per parameter."""
    model, ncls = "dinounet_s", 2
    sd, x, target = _case(model, 1, 128, ncls, 3)
    loss, grads = G.loss_and_grads(sd, model, x, target)
    assert abs(loss.item() - float(REF["grad_loss"])) < 1e-6
    # the reference's named_parameters() lists each shared Parameter once; every trainable oracle key must be among them
    names = sorted(grads)
    assert np.array_equal(sha(names), REF["grad_names"])
    worst = 0.0
    n_s = REF["grad_samp"].shape[1]
    for i, k in enumerate(names):
        go = grads[k]
        if REF["grad_none"][i]:
            assert float(go.abs().max()) == 0.0, k
            continue
        denom = float(REF["grad_max"][i]) + 1e-12
        worst = max(worst, abs(float(go.abs().max()) - float(REF["grad_max"][i])) / denom)
        f = go.reshape(-1)
        samp = f[:: max(1, f.numel() // n_s)][:n_s].numpy()
        worst = max(worst, float(np.abs(samp - REF["grad_samp"][i][:samp.size]).max()) / denom)
    assert worst < 1e-4, worst
