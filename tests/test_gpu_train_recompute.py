"""-m gpu: the training step with the adapter's extractors recomputed in the backward (`DinoUNet.train_recompute`).

  * the forward is the same: training-mode logits bitwise equal with and without recompute, under both semantics;
  * the gradients are the same.  Backward passes without recompute are compared first: where they are bitwise equal,
    recompute must be too.  Where they are not (the LayerNorm weight gradients and the deformable-attention value
    gradient are summed with fp32 atomics), the gap to recompute must stay within RUN_TO_RUN times the largest gap
    between three runs without it, per tensor relative to its largest element.  The order of those atomics follows where
    the tensors sit: runs with the same allocations often agree bit for bit, and recompute allocates differently.  So the
    three runs without recompute start behind pad allocations of different sizes.  Both matrix-product tiers: a replay on
    the default TF32 tier in an fp32 step would show TF32-sized gaps, orders of magnitude above the fp32 run-to-run one;
  * the gradient goldens of test_gpu_train.py / test_gpu_train_mode.py, run unchanged with recompute on;
  * the BatchNorm running statistics are updated once;
  * the memory is freed: the peak of a dinounet_s step at 512^2 drops by at least half of what the extractors would
    otherwise keep;
  * three FusedSGD steps end on the same parameters, by the gradients' rule;
  * dinounet_7b's width (D = 4096, deformable-attention heads of 128 channels) through the trainable part against float64
    autograd of the gradient oracle, and the kernels whose shapes are new at that width at the per-kernel bars of
    test_gpu_train_functions.py.
"""
import os

import pytest
import torch

import dinounet_b200
from dinounet_b200 import config, lib
from dinounet_b200 import train_path as TP
from dinounet_b200.loss import DC_and_CE_loss
from dinounet_b200.train_path import FusedSGD, train_step
from oracle import dinounet_oracle as O
from oracle import grad_oracle as G
from oracle import loss_oracle as LO
from oracle import train_mode_oracle as T
from tests import test_gpu_train as golden
from tests import test_gpu_train_functions as fn
from tests import test_gpu_train_mode as golden_mode

pytestmark = pytest.mark.gpu
NCLS = 2
#: the recompute run is one more draw of the atomics' run-to-run variation; 4x the largest gap seen between three runs
#: without it leaves room for that draw's tail
RUN_TO_RUN = 4.0


def _net(model="dinounet_s", gemm="tf32", semantics="oracle", recompute=False, seed=0):
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, NCLS, None, model)
    net.load_state_dict(O.make_state_dict(model, NCLS, seed=seed), strict=True)
    net.train_gemm, net.train_semantics, net.train_recompute = gemm, semantics, recompute
    return net.to("cuda").train()


def _crit():
    return DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, weight_ce=1, weight_dice=1)


def _batch(B, S, seed=3):
    x = O.make_input(B, S, seed).cuda()
    t = torch.randint(0, NCLS, (B, 1, S, S), generator=torch.Generator().manual_seed(seed)).float().cuda()
    return x, t


def _draws(B):
    g = torch.Generator().manual_seed(11)
    scales = torch.exp(torch.empty(O.VARIANTS["dinounet_s"].depth).uniform_(-0.69, 0.69, generator=g))
    keep = torch.bernoulli(torch.full((6, B), 0.7), generator=g)
    return scales.cuda(), keep.cuda()


def _counting_checkpoint(monkeypatch):
    n = []
    real = TP.checkpoint

    def counted(*a, **k):
        n.append(1)
        return real(*a, **k)
    monkeypatch.setattr(TP, "checkpoint", counted)
    return n


@pytest.mark.parametrize("semantics", ["oracle", "reference"])
def test_same_forward(semantics):
    x, _ = _batch(2, 128)
    scales, keep = _draws(2)
    out = []
    for recompute in (False, True):
        net = _net(semantics=semantics, recompute=recompute)
        out.append(net.train_forward(x, rope_scales=scales, drop_keep=keep).detach())
    assert torch.equal(out[0], out[1])


#: sizes of the allocation a run starts behind (bytes): the runs without recompute see their tensors at other addresses
PADS = (0, 5 << 20, 11 << 20)


def _grads(gemm, recompute, semantics="oracle", pad=0):
    held = torch.empty(pad, dtype=torch.uint8, device="cuda")  # noqa: F841 (kept until the run ends)
    net = _net(gemm=gemm, semantics=semantics, recompute=recompute)
    x, t = _batch(2, 128)
    scales, keep = _draws(2)
    _crit()(net.train_forward(x, rope_scales=scales, drop_keep=keep), t).backward()
    return {n: p.grad.detach().clone() for n, p in net.named_parameters() if p.grad is not None}


def _rel_gaps(a, b):
    """{name: max |a - b| / max |a|} over the tensors of a."""
    return {k: float((a[k] - b[k]).abs().max() / a[k].abs().max().clamp_min(1e-30)) for k in a}


def _same_by_run_to_run(runs, rec, what):
    """runs: three results without recompute, rec: one with.  Bitwise equal if the runs are; else within RUN_TO_RUN x the
    largest run-to-run gap."""
    a = runs[0]
    assert set(rec) == set(a)
    spread = max(max(_rel_gaps(a, r).values()) for r in runs[1:])
    gaps = _rel_gaps(a, rec)
    print(f"{what}: run-to-run spread {spread:.3e}, recompute gap {max(gaps.values()):.3e}, "
          f"{sum(g > 0 for g in gaps.values())} of {len(gaps)} tensors differ")
    if spread == 0.0:
        assert all(torch.equal(a[k], rec[k]) for k in a), [k for k in a if not torch.equal(a[k], rec[k])][:8]
    else:
        bad = {k: g for k, g in gaps.items() if g > RUN_TO_RUN * spread}
        assert not bad, (spread, sorted(bad.items(), key=lambda kv: -kv[1])[:8])


@pytest.mark.parametrize("gemm", ["fp32", "tf32"])
@pytest.mark.parametrize("semantics", ["oracle", "reference"])
def test_same_gradients(gemm, semantics):
    runs = [_grads(gemm, False, semantics, pad) for pad in PADS]
    _same_by_run_to_run(runs, _grads(gemm, True, semantics), f"gradients, {gemm} tier, {semantics}")


def test_gradient_goldens_hold_with_recompute(monkeypatch):
    n = _counting_checkpoint(monkeypatch)
    monkeypatch.setattr(dinounet_b200.DinoUNet, "train_recompute", True)
    golden.test_gradients_match_the_reference_autograd_goldens()
    assert n, "no extractor was recomputed"
    n.clear()
    golden.test_tensor_core_tier_gradients_stay_within_tf32_of_the_goldens()
    assert n


def test_train_mode_goldens_hold_with_recompute(monkeypatch):
    n = _counting_checkpoint(monkeypatch)
    monkeypatch.setattr(dinounet_b200.DinoUNet, "train_recompute", True)
    golden_mode.test_fp32_tier_matches_the_reference_train_mode_golden()
    golden_mode.test_tf32_tier_stays_within_tf32_of_the_train_mode_golden()
    assert len(n) == 12


def test_batchnorm_statistics_are_updated_once():
    x, t = _batch(2, 128)
    scales, keep = _draws(2)
    bufs = []
    for recompute in (False, True):
        net = _net(semantics="reference", recompute=recompute)
        _crit()(net.train_forward(x, rope_scales=scales, drop_keep=keep), t).backward()
        sd = net.state_dict()
        bufs.append({p + s: sd[p + s].clone() for p in T.BN_LAYERS for s in (".running_mean", ".running_var", ".num_batches_tracked")})
    assert all(int(bufs[1][p + ".num_batches_tracked"]) == 1 for p in T.BN_LAYERS)
    assert all(torch.equal(bufs[0][k], bufs[1][k]) for k in bufs[0])


def test_recompute_frees_the_extractor_activations():
    """dinounet_s, B = 2, 512^2.  Per sample and extractor, without recompute the step keeps in fp32: the normalised
    feature map (P*D) and value (P*D/2), locations and weights (Lq*192), the normalised query (Lq*D), the sampled
    values (Lq*D/2), the query after attention (Lq*D), its FFN norm (Lq*D), fc1 / dwconv / GELU (3*Lq*D/4) and the output
    (Lq*D); recompute keeps the input query only: (4.25*Lq*D + 1.5*P*D) * 4 bytes less per extractor, Lq*192 aside."""
    B, S = 2, 512
    D = config.VARIANTS["dinounet_s"].embed_dim
    P, Lq = (S // 16) ** 2, 21 * (S // 32) ** 2
    analytic = 6 * B * (4.25 * Lq * D + 1.5 * P * D) * 4
    x, t = _batch(B, S)
    peaks = {}
    for recompute in (False, True):
        net = _net(recompute=recompute)
        for _ in range(2):                   # the first step packs the engine and builds its plan
            net.zero_grad(set_to_none=True)
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            _crit()(net(x), t).backward()
            torch.cuda.synchronize()
            peaks[recompute] = torch.cuda.max_memory_allocated() - base
        del net
        torch.cuda.empty_cache()
    saved = peaks[False] - peaks[True]
    print(f"dinounet_s B {B} {S}^2: peak above the resident state {peaks[False] / 2**30:.3f} GiB without recompute, "
          f"{peaks[True] / 2**30:.3f} GiB with; saved {saved / 2**20:.0f} MiB, analytic {analytic / 2**20:.0f} MiB")
    assert saved >= 0.5 * analytic


def _params_after_steps(gemm, recompute, steps=3, pad=0):
    held = torch.empty(pad, dtype=torch.uint8, device="cuda")  # noqa: F841 (kept until the run ends)
    net = _net(gemm=gemm, recompute=recompute)
    opt = FusedSGD(net.parameters(), lr=1e-2)
    x, t = _batch(2, 128)
    for _ in range(steps):
        train_step(net, _crit(), opt, x, t)
    torch.cuda.synchronize()
    return {n: p.detach().clone() for n, p in net.named_parameters() if not n.startswith("encoder.dinov3_adapter.backbone.")}


def test_fused_sgd_steps_end_on_the_same_parameters():
    """Parameters move by lr * update, so the run-to-run gap is measured on the change from the start, not the values."""
    start = {n: p.detach().cuda() for n, p in _net().named_parameters() if not n.startswith("encoder.dinov3_adapter.backbone.")}
    delta = lambda ps: {k: ps[k] - start[k] for k in ps}
    runs = [delta(_params_after_steps("tf32", False, pad=pad)) for pad in PADS]
    moved = {k for k in runs[0] if runs[0][k].abs().max() > 0}
    keep = lambda d: {k: d[k] for k in moved}
    _same_by_run_to_run([keep(r) for r in runs], keep(delta(_params_after_steps("tf32", True))), "FusedSGD x3, tf32 tier")


# ------------------------------------------------------------------------------------------------ dinounet_7b's width
def _trainable_7b(B, S, seed=5):
    """dinounet_7b's trainable parameters and BatchNorm buffers (reference keys) generated on the device, and four random
    taps [B, (S/16)^2, 4096]: the trainable part needs nothing from the 6.7 B-parameter backbone but its taps."""
    from bench import SyntheticParams
    gen = SyntheticParams("dinounet_7b", NCLS, torch.device("cuda"))
    P = {k: gen[k] for k, _, _ in O.param_spec("dinounet_7b", NCLS) if not k.startswith("encoder.dinov3_adapter.backbone.")}
    g = torch.Generator(device="cuda").manual_seed(seed)
    D = config.VARIANTS["dinounet_7b"].embed_dim
    taps = [torch.randn(B, (S // 16) ** 2, D, generator=g, device="cuda") for _ in range(4)]
    return P, taps


def test_dinounet_7b_width_against_float64_autograd(monkeypatch):
    """B = 2 at 64^2 (a 4 x 4 tap map), fp32 tier, recompute on, against the gradient oracle in float64 on the device fed
    the same taps (its deformable sampling in fp32, as the reference's).  Loss 1e-5 rel.  The per-tensor bars of
    test_gpu_train_mode.py's fp32 tier, with every element in place of 16 samples: norm within 2e-3, elements within 5e-2
    of the tensor's largest element.  Both get an absolute part of 1e-4 of the largest gradient norm, for tensors whose
    gradient is rounding noise around zero (biases ahead of an InstanceNorm): on an H100 such a tensor reached 4.9e-2 of
    its largest element plus 2e-5 of the largest norm.  A mis-addressed kernel is an O(1) error."""
    B, S, model = 2, 64, "dinounet_7b"
    P, taps = _trainable_7b(B, S)
    x, t = _batch(B, S, seed=9)
    keys = G.trainable_keys(model, NCLS)
    for k in keys:
        P[k].requires_grad_(True)
    n0 = lib.launch_count()
    logits = TP.trainable_forward(P, model, x, taps, NCLS, "fp32", recompute=True)
    loss = _crit()(logits, t)
    loss.backward()
    torch.cuda.synchronize()
    assert lib.launch_count() - n0 > 500, "native kernels did not run"

    h = S // 16
    taps64 = [(tp.double(), None) for tp in taps]
    monkeypatch.setattr(O, "vit_taps", lambda P_, v, x_, collect=None: (taps64, (h, h)))
    # the oracle samples in fp32, as the reference's op casts its inputs (ms_deform_attn.py:30); its result goes on in
    # float64
    msda_core = O.msda_core
    monkeypatch.setattr(O, "msda_core", lambda *a: msda_core(*a).double())
    want_loss, want = G.loss_and_grads({k: v.detach().double() if v.is_floating_point() else v for k, v in P.items()},
                                       model, x.double(), t.double())
    assert abs(loss.item() - want_loss.item()) <= 1e-5 * max(1.0, abs(want_loss.item())), (loss.item(), want_loss.item())
    bad, worst = [], 0.0
    top_norm = max(float(want[k].norm()) for k in keys)
    for k in keys:
        ref = want[k]
        got = P[k].grad.double() if P[k].grad is not None else torch.zeros_like(ref)
        top = float(ref.abs().max())
        err = float((got - ref).abs().max())
        nerr = abs(float(got.norm()) - float(ref.norm()))
        worst = max(worst, err / (top + 2e-5 * top_norm))
        if err > 5e-2 * top + 1e-4 * top_norm or nerr > 2e-3 * float(ref.norm()) + 1e-4 * top_norm:
            bad.append((k, err / max(top, 1e-30), nerr))
    print(f"dinounet_7b width, B {B} {S}^2: loss {loss.item():.6f} (float64 {want_loss.item():.6f}), {len(keys)} tensors, "
          f"worst max-element err / (tensor max + 2e-5 largest norm) {worst:.2e}")
    assert not bad, bad[:8]


@pytest.mark.parametrize("rows", [84 * 2, 5376 * 2])
def test_dinounet_7b_layernorm_width(rows):
    """LayerNormF at D = 4096: the query stream at 64^2 and at 512^2, B = 2."""
    fn.test_layernorm(rows, 4096)


def test_dinounet_7b_msda_head_width():
    """MSDAF with 128 channels per head (4096 / 2 / 16), on the 512^2 tap map and a non-square one."""
    fn.test_msda(1, 32, 32, 128)
    fn.test_msda(1, 8, 12, 128)


def test_dinounet_7b_ffn_dwconv_width():
    """The ConvFFN's depthwise conv at 4096 / 4 channels."""
    fn._dwconv_case(2, 8, 8, 1024, 3, [(16, 16), (8, 8), (4, 4)], seed=20)
