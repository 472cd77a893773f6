"""-m gpu: train_semantics="reference" (the reference's train mode) on the native training step.

  * one step with the recorded draws against tests/golden/train_mode_cases.npz (the REAL reference in .train(), CPU
    fp32), plus the updated running statistics (1e-4 of each tensor's largest value + 1e-7) and num_batches_tracked.
    This step is far worse conditioned than the eval-mode one of test_gpu_train.py: batch-statistics BatchNorm over as
    few as 32 rows per channel (B=2, the 4x4 level) amplifies rounding.  The golden itself, an fp32 computation, differs
    from an fp64 run of the restatement by up to 1.2e-3 in a gradient norm and 2.5e-2 of a tensor's largest sample (243
    tensors beyond 2e-3).  So the fp32 tier keeps the loss (1e-5) and norm (2e-3 rel) bars of test_gpu_train.py, with an
    absolute part of 2e-5 of the largest gradient norm (for tensors whose gradient is nearly zero, e.g. conv biases ahead
    of an InstanceNorm), and holds the samples to 5e-2 of the tensor's largest sample.  Measured on an H100: every norm
    within 1.3e-4 of the largest norm, every tensor above 1e-3 of it within 1.9e-3 rel, samples within 2.5e-2.  The TF32
    tier keeps that file's loss and sampled-element bars; its per-tensor norm bar (5e-2) gets an absolute part of 1e-3
    of the largest norm for the same reason;
  * the new kernels against torch: batch-statistics BatchNorm (+ReLU) forward / backward / running-statistic update,
    bit-identical across launches; per-block RoPE tables and ViT taps with injected scales against the oracle;
  * the draws, "oracle" leaving the BatchNorm buffers alone, and the eval forward seeing what training changed.
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dinounet_b200
from dinounet_b200 import config, lib
from dinounet_b200.loss import DC_and_CE_loss
from dinounet_b200.train_path import BNTrainF, FusedSGD
from oracle import dinounet_oracle as O
from oracle import train_mode_oracle as T

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "train_mode_cases.npz")
MODEL, B, S, NCLS, WSEED = "dinounet_s", 2, 128, 2, 0


def _net(gemm="fp32", precision="fp32", semantics="reference", seed=WSEED):
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, NCLS, None, MODEL)
    net.load_state_dict(O.make_state_dict(MODEL, NCLS, seed=seed), strict=True)
    net.precision = precision
    net.train_gemm = gemm
    net.train_semantics = semantics
    return net.to("cuda").train()


def _crit():
    return DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, weight_ce=1, weight_dice=1)


def _golden_step(gemm):
    g = np.load(GOLDEN)
    net = _net(gemm)
    x = O.make_input(B, S, WSEED).cuda()
    target = torch.randint(0, NCLS, (B, 1, S, S), generator=torch.Generator().manual_seed(WSEED + 7)).float().cuda()
    n0 = lib.launch_count()
    logits = net.train_forward(x, rope_scales=torch.from_numpy(g["rope_scales"]).cuda(),
                               drop_keep=torch.from_numpy(g["drop_keep"]).cuda())
    loss = _crit()(logits, target)
    loss.backward()
    torch.cuda.synchronize()
    assert lib.launch_count() - n0 > 500, "native kernels did not run"
    return g, net, loss.item()


def _check_buffers(g, net):
    sd = net.state_dict()
    for j, p in enumerate(T.BN_LAYERS):
        for key, name in ((f"rm{j}", ".running_mean"), (f"rv{j}", ".running_var")):
            got, want = sd[p + name].cpu().numpy(), g[key]
            err = np.abs(got - want).max()
            assert err <= 1e-4 * np.abs(want).max() + 1e-7, (p + name, err)
        assert int(sd[p + ".num_batches_tracked"]) == int(g[f"nbt{j}"])


def test_fp32_tier_matches_the_reference_train_mode_golden():
    g, net, loss = _golden_step("fp32")
    assert abs(loss - float(g["loss"])) <= 1e-5 * max(1.0, abs(float(g["loss"]))), (loss, float(g["loss"]))
    sdv = net.state_dict(keep_vars=True)
    top = float(np.max(g["norms"]))
    bad, worst, errs = [], 0.0, []
    for i, k in enumerate(str(n) for n in g["names"]):
        p = sdv[k]
        want = float(g["norms"][i])
        if p.grad is None:
            assert want <= 1e-7, k
            continue
        gr = p.grad.detach().float().cpu()
        norm = gr.double().norm().item()
        fl = gr.reshape(-1)
        samp = fl[:: max(1, fl.numel() // 16)][:16].numpy()
        ws = g[f"s{i}"]
        worst = max(worst, abs(norm - want) / want if want > 1e-4 else 0.0)
        serr = float(np.abs(samp - ws).max() / max(np.abs(ws).max(), 1e-12))
        if not (abs(norm - want) <= 2e-3 * want + 2e-5 * top) or not (np.abs(samp - ws).max() <= 5e-2 * np.abs(ws).max() + 2e-5 * top):
            bad.append((k, norm, want, serr))
        errs.append(serr if want > 1e-6 else 0.0)
    print(f"train mode, fp32 tier: loss {loss:.6f} (golden {float(g['loss']):.6f}), worst norm rel err {worst:.2e}, "
          f"worst sample err {max(errs):.2e}, tensors beyond 2e-3: {sum(e > 2e-3 for e in errs)}")
    assert not bad, bad[:8]
    _check_buffers(g, net)


def test_tf32_tier_stays_within_tf32_of_the_train_mode_golden():
    g, net, loss = _golden_step("tf32")
    assert abs(loss - float(g["loss"])) <= 2e-3 * max(1.0, abs(float(g["loss"]))), (loss, float(g["loss"]))
    sdv = net.state_dict(keep_vars=True)
    top = float(np.max(g["norms"]))
    bad, errs, refs = [], [], []
    for i, k in enumerate(str(n) for n in g["names"]):
        p = sdv[k]
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
        if abs(gr.double().norm().item() - want) > 5e-2 * want + 1e-3 * top:
            bad.append((k, rel))
    E, R = np.concatenate(errs), np.concatenate(refs)
    rel_l2 = float(np.linalg.norm(E) / np.linalg.norm(R))
    cos = float(np.dot(R + E, R) / (np.linalg.norm(R + E) * np.linalg.norm(R)))
    print(f"train mode, tf32 tier: loss {loss:.6f}, sampled rel L2 {rel_l2:.3e}, cosine {cos:.5f}")
    assert not bad, bad[:8]
    assert rel_l2 <= 0.15 and cos >= 0.98, (rel_l2, cos)


@pytest.mark.parametrize("act", [lib.ACT_NONE, lib.ACT_RELU])
def test_bn_train_kernels_match_torch_batch_norm(act):
    torch.manual_seed(1)
    rows, Cc = 3001, 80                                    # C not a multiple of 32
    x = (torch.randn(rows, Cc, device="cuda") * 1.7 + 0.4).requires_grad_(True)
    gamma = (torch.rand(Cc, device="cuda") + 0.5).requires_grad_(True)
    beta = (torch.randn(Cc, device="cuda") * 0.2).requires_grad_(True)
    rm0, rv0 = torch.randn(Cc, device="cuda") * 0.1, torch.rand(Cc, device="cuda") + 0.5
    dy = torch.randn(rows, Cc, device="cuda")
    outs = []
    for _ in range(2):
        rm, rv, nbt = rm0.clone(), rv0.clone(), torch.zeros((), dtype=torch.int64, device="cuda")
        y = BNTrainF.apply(x, gamma, beta, rm, rv, nbt, act, 0.1, 1e-5, False)
        dx, dg, db = torch.autograd.grad(y, (x, gamma, beta), dy)
        outs.append((y, dx, dg, db, rm, rv, nbt))
    for a, b in zip(*outs):
        assert torch.equal(a, b)                          # no atomics: identical bits
    y, dx, dg, db, rm, rv, nbt = outs[0]
    trm, trv = rm0.clone(), rv0.clone()
    ty = F.batch_norm(x, trm, trv, gamma, beta, True, 0.1, 1e-5)
    if act == lib.ACT_RELU:
        ty = F.relu(ty)
    tdx, tdg, tdb = torch.autograd.grad(ty, (x, gamma, beta), dy)
    for name, a, b in (("y", y, ty), ("dx", dx, tdx), ("dgamma", dg, tdg), ("dbeta", db, tdb), ("running_mean", rm, trm),
                       ("running_var", rv, trv)):
        err = float((a.detach() - b.detach()).abs().max() / b.detach().abs().max())
        assert err <= 1e-5, (name, err)
    assert int(nbt) == 1


@pytest.mark.parametrize("scale", [0.5, 1.0, 2.0])
def test_rope_tables_match_the_oracle(scale):
    from dinounet_b200.train_path import _call
    periods = O.make_state_dict(MODEL, NCLS)["encoder.dinov3_adapter.backbone.rope_embed.periods"]
    h, hd, depth = 8, 64, 3
    scales = torch.tensor([scale, 1.0, scale], device="cuda")
    sin = torch.empty(depth, h * h, hd, device="cuda")
    cos = torch.empty_like(sin)
    _call("b2u_rope_tables", periods.cuda(), scales, sin, cos, depth, h, h, hd)
    for i in range(depth):
        ws, wc = T.rope_sincos_scaled(periods, h, h, scales[i].cpu())
        assert float((sin[i].cpu() - ws).abs().max()) <= 1e-5 and float((cos[i].cpu() - wc).abs().max()) <= 1e-5


@pytest.mark.parametrize("precision,tol", [("fp32", 1e-5), ("16", 1.2e-2)])
def test_vit_taps_with_injected_scales_match_the_oracle(precision, tol):
    net = _net(precision=precision)
    x = O.make_input(1, 256, 3)
    scales = torch.exp(torch.linspace(-0.69, 0.69, O.VARIANTS[MODEL].depth))
    taps = net._get_engine(torch.device("cuda")).extract_vit_features(x.cuda(), rope_scales=scales.cuda())
    P = O.make_state_dict(MODEL, NCLS, seed=WSEED)
    with torch.no_grad():
        want, _ = T.vit_taps(P, O.VARIANTS[MODEL], x, scales)
    for k in range(4):
        err = float((taps[k].cpu() - want[k][0]).abs().max() / want[k][0].abs().max())
        assert err <= tol, (k, err)
    plain = net._get_engine(torch.device("cuda")).extract_vit_features(x.cuda())
    assert not torch.equal(plain[0], taps[0])             # the eval launch list keeps its own (unscaled) tables


def test_draws():
    net = _net()
    torch.manual_seed(123)
    s1, k1 = net._draw_train_randomness(2000, torch.device("cuda"))
    torch.manual_seed(123)
    s2, k2 = net._draw_train_randomness(2000, torch.device("cuda"))
    assert torch.equal(s1, s2) and torch.equal(k1, k2)
    assert k1.numel() >= 10 ** 4 and set(k1.unique().tolist()) <= {0.0, 1.0}
    assert abs(float(k1.mean()) - 0.7) <= 0.02
    many = torch.cat([net._draw_train_randomness(1, torch.device("cuda"))[0] for _ in range(200)])
    assert float(many.min()) >= 0.5 and float(many.max()) <= 2.0


def _steps(net, n, seed=4):
    x = O.make_input(B, S, seed).cuda()
    target = torch.randint(0, NCLS, (B, 1, S, S), generator=torch.Generator().manual_seed(seed)).float().cuda()
    opt = FusedSGD(net.parameters(), lr=1e-2)
    crit = _crit()
    for _ in range(n):
        opt.zero_grad()
        crit(net(x), target).backward()
        opt.step()
    torch.cuda.synchronize()


def test_oracle_semantics_leaves_the_batchnorm_buffers_alone():
    net = _net(semantics="oracle")
    before = {k: t.clone() for k, t in net.state_dict().items() if k.split(".")[-1] in ("running_mean", "running_var", "num_batches_tracked")}
    _steps(net, 2)
    after = net.state_dict()
    assert all(torch.equal(after[k], t) for k, t in before.items())


def test_eval_forward_sees_the_trained_state_without_repack():
    torch.manual_seed(0)
    net = _net()
    x = O.make_input(1, 128, 6)
    with torch.no_grad():
        net.eval()
        net(x.cuda())                                     # an engine packed before training
        net.train()
    _steps(net, 3)
    assert all(int(net.state_dict()[p + ".num_batches_tracked"]) == 3 for p in T.BN_LAYERS)
    net.eval()
    with torch.no_grad():
        y = net(x.cuda()).cpu()
    sd = {k: t.detach().cpu() for k, t in net.state_dict().items()}
    ref = O.forward(sd, MODEL, x)
    err = float((y - ref).abs().max() / ref.abs().max())
    assert err <= 1e-5, err
