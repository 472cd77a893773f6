"""-m gpu: the full CUDA forward (through the module surface -> engine -> C-ABI kernels) against
  (a) the CPU fp32 oracle restatement of the reference on identical seeded weights/inputs,
  (b) the committed golden logits produced by the REAL reference (tests/golden, oracle/make_golden.py),
  (c) the oracle run in the reference's own GPU precision regime (outer fp16 / inner bf16 autocast) with torch eager.

Tolerances (stated, per the contract in BASELINE.json north_star and the noise floors in BASELINE.md section 5):
  * 16-bit tier: max|dlogit| / max|logit| <= 1.2e-2 (bf16 ViT, the reference's inner autocast dtype) and <= 5e-3 (fp16
    ViT) against the fp32 reference goldens = 1.4x the measured band (6.4-8.6e-3 / 3.4e-3).  The north_star figure
    (1e-3) is tighter than the reference's OWN mixed-precision GPU forward achieves against fp32 (1.1e-2 measured in the
    survey, re-measured here in (c)), so the second binding assertion is: our error vs the fp32 truth <= 1.5 x the
    reference-regime error + 2e-3.  The fp32 tier (tests/test_gpu_fp32_tier.py) is the one held to 1e-5.
  * argmax masks: identical wherever the fp32 class margin exceeds 4x the measured max logit error; the flip count on
    all pixels is reported and must not exceed the reference-regime's own flip count by more than 25 %.
"""
import glob
import os

import numpy as np
import pytest
import torch

import dinounet_b200
from dinounet_b200 import config, lib
from oracle import dinounet_oracle as O

pytestmark = pytest.mark.gpu


def _net(model, sd, vit="bf16", rest="fp16", query="fp32"):
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, 2, None, model)
    net.load_state_dict(sd, strict=True)
    net.vit_dtype, net.rest_dtype, net.query_dtype = vit, rest, query
    return net.to("cuda").eval()


TOL_BF16, TOL_FP16 = 1.2e-2, 5e-3


def _compare(y, ref, ref_regime=None, name="", tol=TOL_BF16):
    y, ref = y.float().cpu(), ref.float().cpu()
    scale = ref.abs().max().item()
    err = (y - ref).abs().max().item() / scale
    margin = (ref[:, 0] - ref[:, 1]).abs()
    flips = (y.argmax(1) != ref.argmax(1))
    msg = f"{name}: rel err {err:.3e}, flips {int(flips.sum())}/{flips.numel()}"
    if ref_regime is not None and not torch.isfinite(ref_regime).all():
        # observed for dinounet_l with the synthetic O(1) weights: the reference's OWN fp16/bf16 autocast regime overflows
        # (non-finite logits from torch eager), while the kernel path (fp32 residual/query streams) stays finite.
        print(f"{name}: reference-regime eager forward is NON-FINITE on this case; comparing against fp32 truth only")
        ref_regime = None
    if ref_regime is not None:
        rr = ref_regime.float().cpu()
        err_r = (rr - ref).abs().max().item() / scale
        flips_r = (rr.argmax(1) != ref.argmax(1))
        msg += f" | reference-regime eager: rel err {err_r:.3e}, flips {int(flips_r.sum())}"
        print(msg)
        assert err <= 1.5 * err_r + 2e-3, msg
        assert int(flips.sum()) <= 1.25 * int(flips_r.sum()) + 8, msg
    else:
        print(msg)
    assert err <= tol, msg
    safe = margin > 4 * err * scale
    assert not (flips & safe).any(), msg
    return err


@pytest.mark.parametrize("model,B,S", [("dinounet_s", 2, 256), ("dinounet_b", 1, 256), ("dinounet_l", 1, 256)])
def test_forward_matches_oracle_and_golden(model, B, S, golden_dir):
    sd = O.make_state_dict(model, 2, seed=0)
    x = O.make_input(B, S, 0)
    net = _net(model, sd)
    n0 = lib.launch_count()
    with torch.no_grad():
        y = net(x.cuda())
        labels = net.predict_labels(x.cuda())
    torch.cuda.synchronize()
    assert lib.launch_count() - n0 > 200, "native kernels did not run"
    g = np.load(os.path.join(golden_dir, f"{model}_b{B}_s{S}_w0_x0.npz"))
    golden = torch.from_numpy(g["logits"])
    sd_cuda = {k: v.cuda() for k, v in sd.items()}
    regime = O.forward(sd_cuda, model, x.cuda(), autocast_like_reference=True)
    _compare(y, golden, regime, f"{model} B{B} S{S} vs golden(reference)")
    assert (labels.cpu().long() == y.argmax(1).cpu()).all()


@pytest.mark.parametrize("model,B,S,xseed", [("dinounet_l", 2, 512, 3), ("dinounet_b", 1, 512, 4), ("dinounet_s", 4, 512, 5)])
def test_forward_benchmarked_shapes_match_reference(model, B, S, xseed, golden_dir):
    """The configurations bench.py / BASELINE.json quote (512^2; dinounet_l at B >= 2 so that batch strides, the 9 query
    tiles of N = 1029 tokens and the CTA-pair GEMMs at M = B*1029 are exercised): every pixel against the oracle run
    live on the host cores (bit-identical to the reference), the subsampled logits and the full argmax mask against the
    golden written by the REAL reference (oracle/make_golden.py BENCH_CASES)."""
    sd = O.make_state_dict(model, 2, seed=0)
    x = O.make_input(B, S, xseed)
    net = _net(model, sd)
    with torch.no_grad():
        y = net(x.cuda()).float().cpu()
        y_graph, lab = net._engine.forward(x.cuda(), use_graph=True)
        y_graph, lab = y_graph.float().cpu(), lab.cpu()
    g = np.load(os.path.join(golden_dir, f"{model}_b{B}_s{S}_w0_x{xseed}.npz"))
    sub = int(g["sub"])
    gs = torch.from_numpy(g["logits_sub"])
    scale = float(g["absmax"])
    err_g = (y[:, :, ::sub, ::sub] - gs).abs().max().item() / scale
    ref = O.forward(sd, model, x)
    # the host of the GPU box picks other fp32 CPU kernels than the build container: fp32 rounding noise only
    noise = (ref[:, :, ::sub, ::sub] - gs).abs().max().item() / scale
    assert noise <= 1e-4, f"live oracle deviates from the committed reference golden by {noise:.2e}"
    gmask = torch.from_numpy(np.unpackbits(g["argmax_bits"])[: B * S * S].reshape(B, S, S).astype(np.int64))
    mism = ref.argmax(1) != gmask
    assert not (mism & ((ref[:, 0] - ref[:, 1]).abs() > 1e-3 * scale)).any() and int(mism.sum()) <= 1e-4 * mism.numel()
    y_flips = int((y.argmax(1) != gmask).sum())
    print(f"  live-oracle vs golden noise {noise:.2e}; argmax flips vs the reference golden mask: {y_flips}/{gmask.numel()}")
    err = _compare(y, ref, None, f"{model} B{B} S{S} (bench shape) vs oracle==reference")
    print(f"  golden(reference) subsample 1/{sub}: rel err {err_g:.3e}; full: {err:.3e}")
    assert err_g <= err + 1e-9
    assert torch.equal(y_graph, y), "CUDA-graph replay differs from eager launches at the bench shape"
    assert torch.equal(lab.long(), y.argmax(1))
    for b in range(B):     # batch items are independent: item b alone gives the same logits bit for bit
        if B > 1 and b in (0, B - 1):
            with torch.no_grad():
                yb = net(x[b:b + 1].cuda()).float().cpu()
            assert torch.equal(yb, y[b:b + 1]), f"batch item {b} depends on its neighbours"


@pytest.mark.parametrize("ncls", [5, 14])
def test_forward_multiclass_matches_oracle(ncls):
    """More than two segmentation heads (the plans' label set decides; nnUNetTrainer.py:201-208): logits and argmax
    labels against the fp32 oracle and the reference-regime eager forward."""
    model = "dinounet_s"
    sd = O.make_state_dict(model, ncls, seed=0)
    x = O.make_input(1, 256, 0)
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, ncls, None, model)
    net.load_state_dict(sd, strict=True)
    net = net.to("cuda").eval()
    with torch.no_grad():
        y = net(x.cuda())
        labels = net.predict_labels(x.cuda())
    ref = O.forward(sd, model, x)
    regime = O.forward({k: v.cuda() for k, v in sd.items()}, model, x.cuda(), autocast_like_reference=True).float().cpu()
    scale = ref.abs().max().item()
    err = (y.cpu() - ref).abs().max().item() / scale
    err_r = (regime - ref).abs().max().item() / scale
    flips = int((y.argmax(1).cpu() != ref.argmax(1)).sum())
    flips_r = int((regime.argmax(1) != ref.argmax(1)).sum())
    print(f"{ncls} classes: rel err {err:.3e} (reference regime {err_r:.3e}), flips {flips} (regime {flips_r}) / {ref[:, 0].numel()}")
    assert y.shape == (1, ncls, 256, 256) and torch.isfinite(y).all() and err < TOL_BF16
    if torch.isfinite(regime).all():       # the reference's own fp16 regime overflows on some synthetic weight sets
        assert err <= 1.5 * err_r + 2e-3 and flips <= 1.25 * flips_r + 8
    else:
        margin = ref.topk(2, dim=1).values
        safe = (margin[:, 0] - margin[:, 1]) > 4 * err * scale
        assert not ((y.argmax(1).cpu() != ref.argmax(1)) & safe).any()
    assert (labels.cpu().long() == y.argmax(1).cpu()).all()


def test_query_stream_fp32_vs_16bit(golden_dir):
    """The adapter's query stream in fp32 (default = the reference's dtype) vs the opt-in 16-bit storage: both inside the
    tolerance; prints both errors."""
    model, B, S = "dinounet_l", 1, 256
    sd = O.make_state_dict(model, 2, seed=0)
    x = O.make_input(B, S, 0)
    golden = torch.from_numpy(np.load(os.path.join(golden_dir, f"{model}_b{B}_s{S}_w0_x0.npz"))["logits"])
    errs = {}
    for q in ("16", "fp32"):
        net = _net(model, sd, query=q)
        with torch.no_grad():
            y = net(x.cuda())
        errs[q] = _compare(y, golden, None, f"{model} query stream {q}")
    assert errs["16"] <= errs["fp32"] * 1.5 + 2e-3


def test_forward_512_golden_and_fp16_vit(golden_dir):
    model = "dinounet_s"
    sd = O.make_state_dict(model, 2, seed=0)
    x = O.make_input(1, 512, 1)
    golden = torch.from_numpy(np.load(os.path.join(golden_dir, "dinounet_s_b1_s512_w0_x1.npz"))["logits"])
    with torch.no_grad():
        y = _net(model, sd)(x.cuda())
        y16 = _net(model, sd, vit="fp16")(x.cuda())
    _compare(y, golden, None, "s 512 bf16-vit vs golden")
    _compare(y16, golden, None, "s 512 fp16-vit vs golden", tol=TOL_FP16)


def test_intermediate_stages_match_oracle():
    """Localises errors: ViT taps, adapter outputs, skips and decoder stages against the fp32 oracle."""
    model = "dinounet_s"
    sd = O.make_state_dict(model, 2, seed=0)
    x = O.make_input(1, 256, 0)
    cap = {}
    O.forward(sd, model, x, collect=cap)
    net = _net(model, sd)
    with torch.no_grad():
        net(x.cuda())
    torch.cuda.synchronize()
    eng = net._engine
    _, bufs = eng.get_plan(1, 256)
    D = 384

    def nchw(t, C, r):
        return t.float().view(1, r, r, C).permute(0, 3, 1, 2).cpu()

    checks = []
    for k in range(4):
        checks.append((f"vit_tap{k}", bufs[f"tap{k}"].view(1, 256, D).cpu(), cap[f"vit_tap{k}"]))
    for i, r in enumerate((64, 32, 16, 8)):
        checks.append((f"f{i + 1}", nchw(bufs[f"f{i + 1}"], D, r), cap[f"f{i + 1}"]))
    checks.append(("skip3", nchw(bufs["skip3"], 256, 32), cap["skip3"]))
    checks.append(("skip0", nchw(bufs["cat2"].view(-1, 64)[:, 32:], 32, 256), cap["skip0"]))
    bad = []
    for name, got, ref in checks:
        e = ((got.float() - ref).abs().max() / ref.abs().max()).item()
        print(f"  stage {name}: rel err {e:.3e}")
        if not e < (1.2e-2 if name.startswith("vit_tap") else 2e-2):
            bad.append((name, e))
    assert not bad, bad


def test_batch_items_are_independent_and_deterministic():
    model = "dinounet_s"
    sd = O.make_state_dict(model, 2, seed=0)
    net = _net(model, sd)
    x = O.make_input(3, 128, 2).cuda()
    with torch.no_grad():
        y3 = net(x)
        y1 = net(x[1:2].contiguous())
        y3b = net(x)
    assert torch.equal(y3, y3b)
    assert torch.equal(y3[1:2], y1)   # per-image reductions have a fixed order (no float atomics anywhere)


def test_cuda_graph_replay_matches_eager_launches():
    model = "dinounet_s"
    sd = O.make_state_dict(model, 2, seed=0)
    net = _net(model, sd)
    x = O.make_input(2, 128, 3).cuda()
    with torch.no_grad():
        y = net(x)
        eng = net._engine
        yg, _ = eng.forward(x, use_graph=True)
        yg2, _ = eng.forward(x, use_graph=True)
    torch.cuda.synchronize()
    assert torch.equal(yg, y) and torch.equal(yg2, y)


def test_streamed_predictor_matches_direct_forward():
    from dinounet_b200.inference import StreamedPredictor
    model = "dinounet_s"
    sd = O.make_state_dict(model, 2, seed=0)
    net = _net(model, sd)
    xs = [O.make_input(2, 128, 10 + i).pin_memory() for i in range(5)]
    with torch.no_grad():
        direct = [net(x.cuda()).cpu() for x in xs]
    outs = [y.clone() for y in StreamedPredictor(net).run(xs)]
    assert len(outs) == 5 and all(torch.equal(a, b) for a, b in zip(outs, direct))
    # the documented lifetime: a yielded buffer survives ONE further advance (ADVICE r1: hold result i-1 while fetching i)
    held, prev = [], None
    for y in StreamedPredictor(net).run(xs):
        if prev is not None:
            held.append(prev.clone())       # read the previous result only after the generator advanced once more
        prev = y
    held.append(prev.clone())
    assert all(torch.equal(a, b) for a, b in zip(held, direct))
    labs = [y.clone() for y in StreamedPredictor(net, want_labels=True).run(xs)]
    assert all(torch.equal(l.long(), d.argmax(1)) for l, d in zip(labs, direct))


def test_7b_recipe_forward_matches_reference_golden(golden_dir):
    """SwiGLU FFN + head_dim 128 + no qkv bias (the dinounet_7b recipe, hub/backbones.py:452-494) on a miniature
    (`dinounet_7b_tiny`, registered test-only) against the golden produced by the REAL reference code."""
    import dataclasses
    from dinounet_b200 import config as cfgmod
    name = "dinounet_7b_tiny"
    cfgmod.VARIANTS[name] = cfgmod.VariantConfig(name, 1024, 4, 8, "swiglu64", 2048, False, (0, 1, 2, 3), True, 0.4)
    try:
        sd = O.make_state_dict(name, 2, seed=0)
        x = O.make_input(1, 256, 0)
        net = _net(name, sd)
        with torch.no_grad():
            y = net(x.cuda())
        golden = torch.from_numpy(np.load(os.path.join(golden_dir, f"{name}_b1_s256_w0_x0.npz"))["logits"])
        sd_cuda = {k: v.cuda() for k, v in sd.items()}
        regime = O.forward(sd_cuda, name, x.cuda(), autocast_like_reference=True)
        # SwiGLU hidden 2048 + head_dim 128 in bf16 (the reference's own autocast regime is non-finite on these synthetic
        # weights, so the fp32 golden is the only anchor)
        _compare(y, golden, regime, "7b-recipe tiny B1 S256 vs golden(reference)", tol=1.6e-2)
    finally:
        cfgmod.VARIANTS.pop(name, None)


def test_frozen_vit_feature_caching_is_bit_identical():
    """SURVEY.md 8f rank 3: the tapped ViT outputs depend only on the image (frozen backbone, eval mode): caching them and
    running only SPM + extractors + FAPM + decoder must reproduce the full forward bit for bit."""
    model = "dinounet_s"
    sd = O.make_state_dict(model, 2, seed=0)
    net = _net(model, sd)
    x = O.make_input(2, 256, 21).cuda()
    with torch.no_grad():
        y = net(x)
        feats = net.extract_vit_features(x)
        n0 = lib.launch_count()
        y2 = net.forward_from_vit_features(x, feats)
        n_rest = lib.launch_count() - n0
        other = net(O.make_input(2, 256, 22).cuda())      # overwrite the engine's tap buffers in between
        y3 = net.forward_from_vit_features(x, [f.clone() for f in feats])
    assert len(feats) == 4 and feats[0].shape == (2, 256, 384) and feats[0].dtype == torch.float32
    assert torch.equal(y2, y) and torch.equal(y3, y) and not torch.equal(other, y)
    plan, _ = net._engine.get_plan(2, 256)
    assert n_rest == len(plan.calls) - plan.vit_end and plan.vit_end > 0.3 * len(plan.calls)


@pytest.mark.parametrize("S", [384, 640])
def test_forward_non_power_of_two_sizes(S):
    """Sizes that are multiples of 128 but not powers of two (h = 24 / 40 patch rows, N = 581 / 1605 tokens, 48- / 80-px conv
    rows): against the oracle run live on the host (no golden: the oracle is pinned to the reference by the other cases)."""
    model = "dinounet_s"
    sd = O.make_state_dict(model, 2, seed=0)
    x = O.make_input(1, S, 11)
    net = _net(model, sd)
    with torch.no_grad():
        y = net(x.cuda()).float().cpu()
        yg, lab = net._engine.forward(x.cuda(), use_graph=True)
    ref = O.forward(sd, model, x)
    _compare(y, ref, None, f"{model} {S}x{S} vs oracle")
    assert torch.equal(yg.float().cpu(), y) and torch.equal(lab.long().cpu(), y.argmax(1))
