"""Conditioning report for the training path's gradient tiers (run on the GPU).

For the gradient-golden case (dinounet_s, B=2, 128x128): FULL gradient tensors of
  gold  = the oracle port's autograd in fp32 on the GPU (cuDNN / cuBLAS TF32 off) - checked against the committed goldens,
  fp32  = this repo's training path, matrix products on the fp32 SIMT tier,
  tf32  = this repo's training path, matrix products on the TF32 tensor cores (the default tier),
  ref16 = the oracle port under the reference's regime (fp16 autocast, inner bf16 ViT), loss scaled by 1024,
and per tensor  rel_l2 = |g - gold| / |gold|  and the norm error.  The point: how ill-conditioned single gradient
elements are at random init (fp32-tier error x ~8000 = tf32-tier error), and that the tf32 tier sits at or below the
reference's own regime.  Writes gpurun_out/grad_tier_report.json; tests/test_gpu_train.py's tf32 bars come from it."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
os.environ.setdefault("DINOUNET_B200_ALLOW_RANDOM_BACKBONE", "1")
import dinounet_b200                           # noqa: E402
from dinounet_b200 import config              # noqa: E402
from dinounet_b200.loss import DC_and_CE_loss  # noqa: E402
from oracle import dinounet_oracle as O        # noqa: E402
from oracle import grad_oracle as G            # noqa: E402
from oracle import loss_oracle as LO           # noqa: E402


def repo_grads(model, sd, ncls, x, target, tier):
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, ncls, None, model)
    net.load_state_dict(sd, strict=True)
    net.precision, net.train_gemm = "fp32", tier
    net = net.to("cuda").train()
    crit = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, weight_ce=1, weight_dice=1)
    loss = crit(net(x), target)
    loss.backward()
    torch.cuda.synchronize()
    params = dict(net.named_parameters())
    return loss.item(), {k: params[k].grad.detach().float() for k in G.trainable_keys(model, ncls) if k in params and params[k].grad is not None}


def ref16_grads(model, sd, x, target, scale=1024.0):
    ncls = sd["decoder.seg_layers.2.weight"].shape[0]
    keys = G.trainable_keys(model, ncls)
    P = {k: v.detach().clone() for k, v in sd.items()}
    leaves = {k: P[k].requires_grad_(True) for k in keys}
    for k, v in O.expand_aliases(leaves).items():
        P[k] = v
    with torch.autocast("cuda", dtype=torch.float16):
        logits = O.decoder_forward(P, O.encoder_forward(P, O.VARIANTS[model], x, True, None), None)
        loss, _, _ = LO.dc_and_ce_loss(logits.float(), target, batch_dice=True)
    grads = torch.autograd.grad(loss * scale, [leaves[k] for k in keys], allow_unused=True)
    return loss.item(), {k: g.float() / scale for k, g in zip(keys, grads) if g is not None}


def main():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model, B, S, ncls, seed = "dinounet_s", 2, 128, 2, 0
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", f"grads_{model}_b{B}_s{S}_c{ncls}_w{seed}.npz"))
    sd = O.make_state_dict(model, ncls, seed=seed)
    x = O.make_input(B, S, seed).cuda()
    target = torch.randint(0, ncls, (B, 1, S, S), generator=torch.Generator().manual_seed(seed + 7)).float().cuda()
    sdc = {k: v.cuda() for k, v in sd.items()}
    gl, gold = G.loss_and_grads(sdc, model, x, target)
    names = [str(n) for n in g["names"]]
    gold_vs_npz = max(abs(gold[k].double().norm().item() - float(g["norms"][i])) / max(float(g["norms"][i]), 1e-12)
                      for i, k in enumerate(names) if float(g["norms"][i]) > 1e-6)
    out = {"case": f"{model} B={B} {S}x{S}", "gold_loss": float(gl), "golden_loss": float(g["loss"]), "gold_vs_committed_goldens_worst_norm_rel": gold_vs_npz,
           "tiers": {}}
    top = max(v.double().norm().item() for v in gold.values())
    tiers = {}
    for tier in ("fp32", "tf32"):
        tiers[tier] = repo_grads(model, sd, ncls, x, target, tier)
    try:
        tiers["ref16"] = ref16_grads(model, sdc, x, target)
    except Exception as e:   # noqa: BLE001
        out["ref16_error"] = repr(e)
    for tier, (loss, grads) in tiers.items():
        rows = []
        for k, gg in gold.items():
            gn = gg.double().norm().item()
            if gn <= 1e-4 * top or k not in grads:
                continue
            d = grads[k].double() - gg.double()
            fin = bool(torch.isfinite(grads[k]).all())
            rows.append({"name": k, "numel": gg.numel(), "gold_norm": gn, "rel_l2": (d.norm().item() / gn) if fin else float("inf"),
                         "norm_rel": abs(grads[k].double().norm().item() - gn) / gn if fin else float("inf"),
                         "max_abs_over_rms": (d.abs().max().item() / (gn / gg.numel() ** 0.5)) if fin else float("inf")})
        rl = np.array([r["rel_l2"] for r in rows])
        flat_g = torch.cat([gold[r["name"]].double().reshape(-1) for r in rows])
        flat_t = torch.cat([grads[r["name"]].double().reshape(-1) for r in rows])
        out["tiers"][tier] = {"loss": loss, "loss_rel_err": abs(loss - float(gl)) / abs(float(gl)), "tensors": len(rows),
                              "rel_l2_max": float(rl.max()), "rel_l2_median": float(np.median(rl)), "rel_l2_p90": float(np.percentile(rl, 90)),
                              "norm_rel_max": max(r["norm_rel"] for r in rows), "max_abs_over_rms_max": max(r["max_abs_over_rms"] for r in rows),
                              "global_rel_l2": ((flat_t - flat_g).norm() / flat_g.norm()).item(),
                              "global_cosine": (torch.dot(flat_t, flat_g) / (flat_t.norm() * flat_g.norm())).item(),
                              "worst": sorted(rows, key=lambda r: -r["rel_l2"])[:12]}
        print(tier, {k: v for k, v in out["tiers"][tier].items() if k != "worst"}, flush=True)
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump(out, open("gpurun_out/grad_tier_report.json", "w"), indent=1)


if __name__ == "__main__":
    main()
