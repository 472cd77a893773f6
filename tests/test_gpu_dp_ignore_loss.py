"""-m gpu, needs >= 2 GPUs (skipped below): data-parallel batch Dice with an ignore label over NCCL, spawned processes as
in test_gpu_dp_loss.py.  Per-rank loss and d loss / d logits of DC_and_CE_loss(ignore_label=C) with ddp=True,
batch_dice=True and per-rank backward scales 1 and 2 against the reference's 2-process gloo run
(tests/golden/ignore_loss_cases.npz), within the tolerances of test_gpu_loss.py.  The masked Dice sums are all-reduced;
the CE and its valid-pixel count stay per rank."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0
needs2 = pytest.mark.skipif(NGPU < 2, reason="needs two GPUs")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ignore_loss_cases.npz")


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        from dinounet_b200.loss import DC_and_CE_loss
        from oracle import ignore_loss_oracle as IO
        ref = np.load(GOLDEN)
        crit = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": True}, {}, 1, 1,
                              ignore_label=IO.DDP_C)
        z, t = IO.ddp_shard(rank)
        z = z.to(dev).requires_grad_(True)
        loss = crit(z, t.to(dev))
        (loss * IO.DDP_SCALES[rank]).backward()
        want, gref = ref[f"ddp_{rank}_loss"], ref[f"ddp_{rank}_grad"]
        q.put((rank, abs(float(loss) - float(want)) / max(1.0, abs(float(want))),
               float(np.abs(IO.strided(z.grad).cpu().numpy() - gref).max() / np.abs(gref).max())))
    finally:
        dist.destroy_process_group()


@needs2
def test_nccl_ignore_label_batch_dice_matches_gloo_reference():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=900) for _ in range(2)], key=lambda r: r[0])
    for p in procs:
        p.join(timeout=120)
    for rank, lerr, gerr in res:
        assert lerr <= 2e-6 and gerr < 1e-5, (rank, lerr, gerr)
