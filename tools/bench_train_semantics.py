"""Step time of `train_semantics="reference"` (the reference's train mode: batch-statistics SyncBatchNorm, DropPath,
per-block RoPE rescaling) against the default "oracle" semantics: one `train_step` of dinounet_b at the training
configuration (batch 32, 512x512, TF32 tier), both semantics in one process on the same network, alternated step by step
after a warm-up, timed with CUDA events.  Prints the card's name and power limit and one JSON line.

  python tools/bench_train_semantics.py [--model dinounet_b] [--batch 32] [--size 512] [--steps 10] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="dinounet_b")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    os.environ.setdefault("DINOUNET_B200_ALLOW_RANDOM_BACKBONE", "1")
    import dinounet_b200
    from dinounet_b200 import config
    from dinounet_b200.loss import DC_and_CE_loss
    from dinounet_b200.train_path import FusedSGD, train_step
    from oracle import dinounet_oracle as O

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card)
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, 2, None, a.model)
    net.load_state_dict(O.make_state_dict(a.model, 2, seed=0), strict=True)
    net = net.to("cuda").train()
    net.train_gemm = "tf32"
    g = torch.Generator().manual_seed(1)
    x = torch.randn(a.batch, 3, a.size, a.size, generator=g).cuda()
    t = torch.randint(0, 2, (a.batch, 1, a.size, a.size), generator=g).float().cuda()
    crit = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, weight_ce=1, weight_dice=1)
    opt = FusedSGD(net.parameters(), lr=1e-4)
    times = {"oracle": [], "reference": []}
    for i in range(a.warmup + a.steps):
        for sem in ("oracle", "reference"):
            net.train_semantics = sem
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            train_step(net, crit, opt, x, t)
            e1.record()
            e1.synchronize()
            if i >= a.warmup:
                times[sem].append(e0.elapsed_time(e1))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    print(json.dumps({"model": a.model, "batch": a.batch, "size": a.size, "steps": a.steps, "card": card,
                      "oracle_ms": round(med["oracle"], 2), "reference_ms": round(med["reference"], 2),
                      "overhead_ms": round(med["reference"] - med["oracle"], 2),
                      "overhead_pct": round(100 * (med["reference"] / med["oracle"] - 1), 2),
                      "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 1e9, 1),
                      "all_ms": {k: [round(v, 1) for v in vs] for k, vs in times.items()}}))


if __name__ == "__main__":
    main()
