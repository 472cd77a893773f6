"""TEST INFRASTRUCTURE — writes tests/golden/ignore_loss_cases.npz: what the REAL reference classes compute for the softmax
Dice + CE loss with an ignore label, so that tests/test_ignore_loss_cpu.py can pin oracle/ignore_loss_oracle.py against
them without the reference.
Run where the reference is importable (oracle/ref_loader.py):  python oracle/make_golden_ignore_loss.py
Contents (float32 values exactly as the reference returned them; gradients as 256 strided samples, ignore_loss_oracle.strided):
  ign_<bd>_<C>_{loss,grad,tp,fp,fn}   DC_and_CE_loss({batch_dice, smooth 1e-5, do_bg False, ddp False}, {},
                                      ignore_label=C, dice_class=MemoryEfficientSoftDiceLoss) on IGN_CASES (about 20 %
                                      of the pixels ignored), d loss / d logits, and validation_step's counts: argmax
                                      one-hot vs the target with ignored pixels set to 0, get_tp_fp_fn_tn with mask
                                      (target != ignore) over every class
  onesample_{loss,grad,tp,fp,fn}      sample 1 of 2 fully ignored, per-sample Dice, C = EDGE_C
  allign_{loss,grad,tp,fp,fn}         every pixel ignored, batch Dice, C = EDGE_C
  ddp_<rank>_{loss,grad}              2-process gloo run, ddp=True, batch_dice=True, rank r backpropagates
                                      DDP_SCALES[r] * loss, C = DDP_C
"""
import os
import socket
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ignore_loss_oracle as IO  # noqa: E402
from oracle import region_loss_oracle as RO  # noqa: E402


def _crit(cls, dice, bd, C, ddp=False):
    return cls({"batch_dice": bd, "smooth": 1e-5, "do_bg": False, "ddp": ddp}, {}, weight_ce=1, weight_dice=1,
               ignore_label=C, dice_class=dice)


def _case(out, key, crit, get_tp_fp_fn_tn, z, t, C):
    z1 = z.clone().requires_grad_(True)
    want = crit(z1, t.clone())
    want.backward()
    out[key + "_loss"], out[key + "_grad"] = want.detach().numpy(), IO.strided(z1.grad).numpy()
    # validation_step (nnUNetTrainer.py:977-994), label-map branch with an ignore label
    pred = torch.zeros(z.shape, dtype=torch.float32)
    pred.scatter_(1, z.argmax(1)[:, None], 1)
    target = t.clone()
    mask = (target != C).float()
    target[target == C] = 0
    tp, fp, fn, _ = get_tp_fp_fn_tn(pred, target, axes=[0, 2, 3], mask=mask)
    out[key + "_tp"], out[key + "_fp"], out[key + "_fn"] = tp.numpy(), fp.numpy(), fn.numpy()


def _ddp_worker(rank, port, q):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=IO.DDP_WORLD)
    try:
        _, DC_and_CE_loss, MemDice, _ = RO.load_reference_region_loss()
        crit = _crit(DC_and_CE_loss, MemDice, True, IO.DDP_C, ddp=True)
        z, t = IO.ddp_shard(rank)
        z = z.requires_grad_(True)
        loss = crit(z, t)
        (loss * IO.DDP_SCALES[rank]).backward()
        q.put({f"ddp_{rank}_loss": loss.detach().numpy(), f"ddp_{rank}_grad": IO.strided(z.grad).numpy()})
    finally:
        dist.destroy_process_group()


def main():
    out = {}
    _, DC_and_CE_loss, MemDice, get_tp_fp_fn_tn = RO.load_reference_region_loss()
    B, H, W = IO.IGN_SHAPE
    for seed, (bd, C) in enumerate(IO.IGN_CASES):
        z, t = IO.ignore_case(B, C, H, W, seed)
        _case(out, f"ign_{int(bd)}_{C}", _crit(DC_and_CE_loss, MemDice, bd, C), get_tp_fp_fn_tn, z, t, C)
    C = IO.EDGE_C
    z, t = IO.ignore_case(B, C, H, W, 98, ignored_samples=(1,))
    _case(out, "onesample", _crit(DC_and_CE_loss, MemDice, False, C), get_tp_fp_fn_tn, z, t, C)
    z, t = IO.ignore_case(B, C, H, W, 99, ignored_samples=range(B))
    _case(out, "allign", _crit(DC_and_CE_loss, MemDice, True, C), get_tp_fp_fn_tn, z, t, C)

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = torch.multiprocessing.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_ddp_worker, args=(r, port, q)) for r in range(IO.DDP_WORLD)]
    for p in procs:
        p.start()
    for _ in procs:
        out.update(q.get(timeout=600))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0, p.exitcode

    path = os.path.join(ROOT, "tests", "golden", "ignore_loss_cases.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
