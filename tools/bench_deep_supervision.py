"""Step time of deep-supervision training against the default (off): one `train_step` of dinounet_b at the training
configuration (batch 32, 512x512, TF32 tier, label maps), deep supervision on (three heads, the weighted Dice+CE over the
two weighted scales, targets downsampled on the device by b2u_ds_targets inside the timed step) and off, alternated
step by step in one process after a warm-up, timed with CUDA events; then `downsample_targets` alone (int16 label maps
[32, 1, 512, 512] -> 256^2 and 128^2: allocation + one b2u_ds_targets launch) per call over many calls with CUDA events.  Prints the card's name and power limit and
one JSON line.

  python tools/bench_deep_supervision.py [--model dinounet_b] [--batch 32] [--size 512] [--steps 10] [--warmup 2]
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
    ap.add_argument("--kernel-iters", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    os.environ.setdefault("DINOUNET_B200_ALLOW_RANDOM_BACKBONE", "1")
    import dinounet_b200
    from dinounet_b200 import config
    from dinounet_b200 import deep_supervision as DS
    from dinounet_b200.loss import DC_and_CE_loss, DeepSupervisionWrapper
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
    scales = DS.deep_supervision_scales([[1, 1], [2, 2], [2, 2], [2, 2]])
    base = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, weight_ce=1, weight_dice=1)
    crit = {False: base, True: DeepSupervisionWrapper(base, DS.deep_supervision_weights(len(scales), False))}
    opt = FusedSGD(net.parameters(), lr=1e-4)
    times = {False: [], True: []}
    for i in range(a.warmup + a.steps):
        for ds in (False, True):
            net.decoder.deep_supervision = ds
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            train_step(net, crit[ds], opt, x, DS.downsample_targets(t, scales) if ds else t)
            e1.record()
            e1.synchronize()
            if i >= a.warmup:
                times[ds].append(e0.elapsed_time(e1))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}

    lab = t.to(torch.int16)
    for _ in range(10):
        DS.downsample_targets(lab, scales)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.kernel_iters):
        DS.downsample_targets(lab, scales)
    e1.record()
    e1.synchronize()
    kernel_us = 1e3 * e0.elapsed_time(e1) / a.kernel_iters
    out_bytes = sum(a.batch * (a.size // f) ** 2 * 2 for f in (2, 4))
    print(json.dumps({"model": a.model, "batch": a.batch, "size": a.size, "steps": a.steps, "card": card,
                      "ds_off_ms": round(med[False], 2), "ds_on_ms": round(med[True], 2),
                      "overhead_ms": round(med[True] - med[False], 2),
                      "overhead_pct": round(100 * (med[True] / med[False] - 1), 2),
                      "downsample_targets_us_per_call_int16": round(kernel_us, 2), "target_out_bytes": out_bytes,
                      "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 1e9, 1),
                      "all_ms": {("on" if k else "off"): [round(v, 1) for v in vs] for k, vs in times.items()}}))


if __name__ == "__main__":
    main()
