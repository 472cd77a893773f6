"""-m gpu: the training path (dinounet_b200/train_path.py: autograd Functions over hand-written forward / backward
kernels; matrix products on the fp32 SIMT tier here unless a test says tf32) against the gradient oracle's goldens (tests/golden/grads_*.npz = autograd through the oracle forward + loss
oracle, itself pinned to autograd through the REAL reference, tests/test_grad_oracle_cpu.py).  BASELINE.json config 3.

Tolerance: fp32 with different summation orders (split-K atomics): loss 1e-5 rel; per-tensor gradient norm 2e-3 rel
(+1e-7 abs); 16 strided samples per tensor within 2e-3 of the tensor's largest sample + 1e-7.
"""
import glob
import os

import numpy as np
import pytest
import torch

import dinounet_b200
from dinounet_b200 import config, lib
from dinounet_b200.loss import DC_and_CE_loss
from dinounet_b200.train_path import FusedSGD
from oracle import dinounet_oracle as O
from oracle import grad_oracle as G

pytestmark = pytest.mark.gpu


def _net(model, sd, ncls, gemm="fp32"):
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, ncls, None, model)
    net.load_state_dict(sd, strict=True)
    net.precision = "fp32"          # frozen ViT on the fp32 tier: the goldens are fp32 end to end
    net.train_gemm = gemm           # "fp32": SIMT matrix products (the 2e-3 bar); "tf32": the tensor-core tier
    return net.to("cuda").train()


def test_gradients_match_the_reference_autograd_goldens():
    files = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "grads_*.npz")))
    assert files
    for f in files:
        model, b, s, c, w = os.path.basename(f)[len("grads_"):-4].rsplit("_", 4)
        B, S, ncls, seed = int(b[1:]), int(s[1:]), int(c[1:]), int(w[1:])
        g = np.load(f)
        sd = O.make_state_dict(model, ncls, seed=seed)
        x = O.make_input(B, S, seed)
        target = torch.randint(0, ncls, (B, 1, S, S), generator=torch.Generator().manual_seed(seed + 7)).float()
        net = _net(model, sd, ncls)
        crit = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, weight_ce=1, weight_dice=1)
        n0 = lib.launch_count()
        logits = net(x.cuda())
        loss = crit(logits, target.cuda())
        loss.backward()
        torch.cuda.synchronize()
        assert lib.launch_count() - n0 > 500, "native kernels did not run"
        assert abs(loss.item() - float(g["loss"])) <= 1e-5 * max(1.0, abs(float(g["loss"]))), (loss.item(), float(g["loss"]))
        names = [str(n) for n in g["names"]]
        params = dict(net.named_parameters())
        assert set(names) == set(G.trainable_keys(model, ncls))
        bad, worst = [], 0.0
        for i, k in enumerate(names):
            p = params[k] if k in params else net.state_dict(keep_vars=True)[k]
            if p.grad is None:      # parameters the forward never touches (unused deep-supervision heads): oracle grad == 0
                assert float(g["norms"][i]) == 0.0, k
                continue
            gr = p.grad.detach().float().cpu()
            norm, want = gr.double().norm().item(), float(g["norms"][i])
            rel = abs(norm - want) / max(want, 1e-12)
            fl = gr.reshape(-1)
            samp = fl[:: max(1, fl.numel() // 16)][:16].numpy()
            ws = g[f"s{i}"]
            serr = np.abs(samp - ws).max() / max(np.abs(ws).max(), 1e-12)
            worst = max(worst, rel if want > 1e-4 else 0.0)
            if not (abs(norm - want) <= 2e-3 * want + 1e-7) or not (np.abs(samp - ws).max() <= 2e-3 * np.abs(ws).max() + 1e-7):
                bad.append((k, norm, want, float(serr)))
        print(f"{os.path.basename(f)}: loss {loss.item():.6f} (golden {float(g['loss']):.6f}), {len(names)} tensors, worst norm rel err {worst:.2e}")
        assert not bad, bad[:8]
        # no gradient reaches the frozen backbone
        assert all(p.grad is None for n, p in net.named_parameters() if n.startswith("encoder.dinov3_adapter.backbone."))


def test_tensor_core_tier_gradients_stay_within_tf32_of_the_goldens():
    """The same goldens through the TF32 tensor-core matrix products (train_gemm = "tf32", the default of the train step).
    Operands carry 10 mantissa bits - the fp16 autocast the reference trains under has the same - and single gradient elements
    of this random-init network are ill-conditioned (tools/grad_tier_report.py compares the tiers on full tensors; the
    reference's own fp16 autocast regime overflows to NaN on these synthetic weights, as it does in the forward).  Bars:
    loss 2e-3, per-tensor norm 5e-2, and over ALL sampled elements, each tensor scaled to unit RMS, a relative L2 error of
    0.15 and a cosine of 0.98 (an addressing / tier mix-up is an O(1) error in these numbers)."""
    files = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "grads_*.npz")))
    assert files
    for f in files:
        model, b, s, c, w = os.path.basename(f)[len("grads_"):-4].rsplit("_", 4)
        B, S, ncls, seed = int(b[1:]), int(s[1:]), int(c[1:]), int(w[1:])
        g = np.load(f)
        sd = O.make_state_dict(model, ncls, seed=seed)
        x = O.make_input(B, S, seed)
        target = torch.randint(0, ncls, (B, 1, S, S), generator=torch.Generator().manual_seed(seed + 7)).float()
        net = _net(model, sd, ncls, gemm="tf32")
        crit = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, weight_ce=1, weight_dice=1)
        n0 = lib.launch_count()
        loss = crit(net(x.cuda()), target.cuda())
        loss.backward()
        torch.cuda.synchronize()
        assert lib.launch_count() - n0 > 500, "native kernels did not run"
        assert abs(loss.item() - float(g["loss"])) <= 2e-3 * max(1.0, abs(float(g["loss"]))), (loss.item(), float(g["loss"]))
        names = [str(n) for n in g["names"]]
        params = dict(net.named_parameters())
        top = float(np.max(g["norms"]))
        bad, worst_n, errs, refs = [], 0.0, [], []
        for i, k in enumerate(names):
            p = params[k] if k in params else net.state_dict(keep_vars=True)[k]
            want = float(g["norms"][i])
            if p.grad is None or want <= 1e-4 * top:
                continue
            gr = p.grad.detach().float().cpu()
            assert torch.isfinite(gr).all(), k
            rel = abs(gr.double().norm().item() - want) / want
            fl = gr.reshape(-1)
            samp = fl[:: max(1, fl.numel() // 16)][:16].numpy().astype(np.float64)
            rms = want / np.sqrt(fl.numel())
            errs.append((samp - g[f"s{i}"]) / rms)
            refs.append(g[f"s{i}"] / rms)
            worst_n = max(worst_n, rel)
            if rel > 5e-2:
                bad.append((k, rel))
        E, R = np.concatenate(errs), np.concatenate(refs)
        rel_l2 = float(np.linalg.norm(E) / np.linalg.norm(R))
        cos = float(np.dot(R + E, R) / (np.linalg.norm(R + E) * np.linalg.norm(R)))
        print(f"{os.path.basename(f)} [tf32 tier]: loss {loss.item():.6f} (golden {float(g['loss']):.6f}), worst norm rel err {worst_n:.2e}, "
              f"sampled elements ({E.size}): rel L2 {rel_l2:.3e}, cosine {cos:.5f}")
        assert not bad, bad[:8]
        assert rel_l2 <= 0.15 and cos >= 0.98, (rel_l2, cos)


def test_fused_sgd_step_matches_torch_sgd():
    """clip_grad_norm_(12) + SGD(momentum 0.99, nesterov, weight decay 3e-5) (nnUNetTrainer.py:486-489, 922-923)."""
    torch.manual_seed(0)
    ps = [torch.randn(1000, device="cuda").requires_grad_(), torch.randn(33, 7, device="cuda").requires_grad_()]
    ref = [p.detach().clone().requires_grad_() for p in ps]
    opt = FusedSGD(ps, lr=1e-2, weight_decay=3e-5, momentum=0.99, max_norm=12.0)
    topt = torch.optim.SGD(ref, lr=1e-2, weight_decay=3e-5, momentum=0.99, nesterov=True)
    for step in range(3):
        gs = [torch.randn_like(p) * (50.0 if step == 1 else 0.1) for p in ps]     # step 1 exceeds the clip threshold
        for p, r, gg in zip(ps, ref, gs):
            p.grad, r.grad = gg.clone(), gg.clone()
        torch.nn.utils.clip_grad_norm_(ref, 12)
        topt.step()
        opt.step()
        for p, r in zip(ps, ref):
            assert torch.allclose(p, r, rtol=1e-5, atol=1e-6), step


def test_training_steps_reduce_the_loss():
    """A few optimizer steps on one batch: loss goes down, the backbone stays untouched, eval forward sees the new weights."""
    model, ncls = "dinounet_s", 2
    sd = O.make_state_dict(model, ncls, seed=0)
    net = _net(model, sd, ncls)
    net.precision = "16"
    net.repack()
    x = O.make_input(2, 128, 5).cuda()
    target = torch.randint(0, ncls, (2, 1, 128, 128), generator=torch.Generator().manual_seed(3)).float().cuda()
    crit = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, weight_ce=1, weight_dice=1)
    opt = FusedSGD(net.parameters(), lr=1e-3)
    bb = {n: p.detach().clone() for n, p in net.named_parameters() if n.startswith("encoder.dinov3_adapter.backbone.blocks.0.")}
    losses = []
    for _ in range(4):
        opt.zero_grad()
        loss = crit(net(x), target)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    print("losses", losses, "grad norm", opt.grad_norm())
    assert losses[-1] < losses[0]
    assert all(torch.equal(p, bb[n]) for n, p in net.named_parameters() if n in bb)
    net.eval()
    net.repack()
    with torch.no_grad():
        y = net(x)
    assert torch.isfinite(y).all()
