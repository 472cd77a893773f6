"""Times the fused losses (forward + backward) with CUDA events and compares them with the torch-eager restatement of the
reference on the same GPU.  Prints one JSON line per configuration and the card's name and power limit.

  python tools/bench_loss.py [--batch 32] [--size 512] [--reps 20]

Traffic is what the algorithm has to move (fp32 logits, the target, the fp32 gradient): forward reads logits + target,
backward reads them again and writes the gradient.  Achieved GB/s = that traffic over the median time; the share of
peak is against the 3.35 TB/s of the H100 SXM data sheet.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dinounet_b200.loss import DC_and_BCE_loss, DC_and_CE_loss  # noqa: E402
from oracle import ignore_loss_oracle as IO  # noqa: E402
from oracle import loss_oracle as LO  # noqa: E402
from oracle import region_loss_oracle as RO  # noqa: E402

PEAK_BYTES = 3.35e12


def _time(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def _fwd_bwd(loss_fn, z, t):
    def run():
        zz = z.detach().requires_grad_(True)
        loss_fn(zz, t).backward()
    return run


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_loss needs a GPU")
    dev = torch.device("cuda", 0)
    B, S = a.batch, a.size
    px = B * S * S
    print(json.dumps({"card": _card(), "batch": B, "size": S}))
    g = torch.Generator().manual_seed(0)
    configs = []
    z = (torch.randn(B, 2, S, S, generator=g) * 3).to(dev)
    t = torch.randint(0, 2, (B, 1, S, S), generator=g).float().to(dev)
    ce = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, 1, 1)
    configs.append(("softmax C=2", z, t, ce, lambda zz, tt: LO.dc_and_ce_loss(zz, tt)[0], 2 * (2 * 4 + 4) + 2 * 4))
    z, t = IO.ignore_case(B, 2, S, S, 2)          # about 20 % of the pixels labelled 2, the ignore label
    z, t = z.to(dev), t.to(dev)
    ce = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, 1, 1, ignore_label=2)
    configs.append(("softmax C=2, ignore label", z, t, ce, lambda zz, tt: IO.dc_and_ce_loss(zz, tt, 2)[0],
                    2 * (2 * 4 + 4) + 2 * 4))
    for ign in (False, True):
        z, t = RO.region_case(B, 3, S, S, 1, use_ignore=ign)
        z, t = z.to(dev), t.to(dev)
        m = DC_and_BCE_loss({}, {"batch_dice": True, "do_bg": True, "smooth": 1e-5, "ddp": False}, use_ignore_label=ign)
        tch = 3 + int(ign)
        configs.append((f"region R=3 ignore={ign}", z, t, m,
                        lambda zz, tt, ign=ign: RO.dc_and_bce_loss(zz, tt, batch_dice=True, use_ignore=ign)[0],
                        2 * (3 * 4 + tch * 4) + 3 * 4))
    for name, z, t, native, eager, bytes_per_px in configs:
        ms = _time(_fwd_bwd(native, z, t), a.reps)
        ms_eager = _time(_fwd_bwd(eager, z, t), a.reps)
        gbs = bytes_per_px * px / (ms * 1e-3) / 1e9
        print(json.dumps({"loss": name, "fused_ms": round(ms, 4), "torch_eager_ms": round(ms_eager, 4),
                          "speedup": round(ms_eager / ms, 2), "traffic_MB": round(bytes_per_px * px / 1e6, 1),
                          "achieved_GBps": round(gbs, 1), "share_of_3.35TBps": round(gbs * 1e9 / PEAK_BYTES, 3)}))


if __name__ == "__main__":
    main()
