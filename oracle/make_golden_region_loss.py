"""TEST INFRASTRUCTURE — writes tests/golden/region_loss_cases.npz: what the REAL reference loss classes compute for the
region loss and for data-parallel batch Dice, so that tests/test_region_loss_cpu.py can pin
oracle/region_loss_oracle.py against them without the reference.
Run where the reference is importable (oracle/ref_loader.py):  python oracle/make_golden_region_loss.py
Contents (float32 values exactly as the reference returned them; gradients as 256 strided samples, region_loss_oracle.strided):
  bce_<bd>_<ign>_<R>_{loss,grad,tp,fp,fn}   DC_and_BCE_loss({}, {batch_dice, do_bg True, smooth 1e-5, ddp False},
                                            use_ignore_label) on REGION_CASES, d loss / d logits, and the validation
                                            counts of (sigmoid > 0.5).long() via get_tp_fp_fn_tn with mask 1 - t_ign
  allign_{loss,grad}                        every pixel ignored (batch_dice, R = 3)
  ddp_<kind>_<rank>_{loss,grad}             2-process gloo run, ddp=True, batch_dice=True, rank r backpropagates
                                            DDP_SCALES[r] * loss: kind 'bce' = DC_and_BCE_loss with an ignore channel,
                                            'ce' = DC_and_CE_loss (do_bg False) with MemoryEfficientSoftDiceLoss
"""
import os
import socket
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import region_loss_oracle as RO  # noqa: E402


def _bce_loss(cls, dice, bd, ign):
    return cls({}, {"batch_dice": bd, "do_bg": True, "smooth": 1e-5, "ddp": False}, use_ignore_label=ign,
               dice_class=dice)


def _ddp_worker(rank, port, q):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=RO.DDP_WORLD)
    try:
        DC_and_BCE_loss, DC_and_CE_loss, MemDice, _ = RO.load_reference_region_loss()
        out = {}
        for kind in ("bce", "ce"):
            if kind == "bce":
                crit = DC_and_BCE_loss({}, {"batch_dice": True, "do_bg": True, "smooth": 1e-5, "ddp": True},
                                       use_ignore_label=True, dice_class=MemDice)
            else:
                crit = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": True}, {},
                                      weight_ce=1, weight_dice=1, ignore_label=None, dice_class=MemDice)
            z, t = RO.ddp_shard(kind, rank)
            z = z.requires_grad_(True)
            loss = crit(z, t)
            (loss * RO.DDP_SCALES[rank]).backward()
            out[f"ddp_{kind}_{rank}_loss"] = loss.detach().numpy()
            out[f"ddp_{kind}_{rank}_grad"] = RO.strided(z.grad).numpy()
        q.put(out)
    finally:
        dist.destroy_process_group()


def main():
    out = {}
    DC_and_BCE_loss, _, MemDice, get_tp_fp_fn_tn = RO.load_reference_region_loss()
    B, H, W = RO.REGION_SHAPE
    for seed, (bd, ign, R) in enumerate(RO.REGION_CASES):
        z, t = RO.region_case(B, R, H, W, seed, use_ignore=ign)
        z1 = z.clone().requires_grad_(True)
        want = _bce_loss(DC_and_BCE_loss, MemDice, bd, ign)(z1, t)
        want.backward()
        pred = (torch.sigmoid(z) > 0.5).long()
        mask, gt = (1 - t[:, -1:], t[:, :-1]) if ign else (None, t)
        tp, fp, fn, _ = get_tp_fp_fn_tn(pred, gt, axes=[0, 2, 3], mask=mask)
        key = f"bce_{int(bd)}_{int(ign)}_{R}"
        out[key + "_loss"], out[key + "_grad"] = want.detach().numpy(), RO.strided(z1.grad).numpy()
        out[key + "_tp"], out[key + "_fp"], out[key + "_fn"] = tp.numpy(), fp.numpy(), fn.numpy()

    z, t = RO.region_case(B, 3, H, W, 99, use_ignore=True, ignore_all=True)
    z1 = z.clone().requires_grad_(True)
    want = _bce_loss(DC_and_BCE_loss, MemDice, True, True)(z1, t)
    want.backward()
    out["allign_loss"], out["allign_grad"] = want.detach().numpy(), RO.strided(z1.grad).numpy()

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = torch.multiprocessing.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_ddp_worker, args=(r, port, q)) for r in range(RO.DDP_WORLD)]
    for p in procs:
        p.start()
    for _ in procs:
        out.update(q.get(timeout=600))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0, p.exitcode

    path = os.path.join(ROOT, "tests", "golden", "region_loss_cases.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
