"""-m gpu, needs >= 2 GPUs (skipped below): data-parallel batch Dice over NCCL, spawned processes as in test_gpu_multi.py.

  * per-rank loss and d loss / d logits of DC_and_BCE_loss (ignore channel) and DC_and_CE_loss with ddp=True,
    batch_dice=True and per-rank backward scales 1 and 2 against the reference's 2-process gloo run
    (tests/golden/region_loss_cases.npz), within the tolerances of test_gpu_loss.py;
  * one `train_step` (train_gemm "fp32") on 2 ranks x 2 samples leaves bitwise-identical parameters on both ranks, and
    the same update as one step on one GPU with the 4 samples: max|d_dp - d_1| <= 1e-4 * max|d_1| (fp32 with different
    summation orders in the all-reduced gradients; the loss-level agreement above is ~1e-7).
"""
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
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "region_loss_cases.npz")


def _net(dev):
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    import dinounet_b200
    from dinounet_b200 import config
    from oracle import dinounet_oracle as O
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, 2, None, "dinounet_s")
    net.load_state_dict(O.make_state_dict("dinounet_s", 2, seed=0), strict=True)
    net.precision = "fp32"
    net.train_gemm = "fp32"
    return net.to(dev).train()


def _step_inputs():
    from oracle import dinounet_oracle as O
    x = O.make_input(4, 128, 9)
    t = torch.randint(0, 2, (4, 1, 128, 128), generator=torch.Generator().manual_seed(10)).float()
    return x, t


def _train_delta(dev, x, t):
    from dinounet_b200.loss import DC_and_CE_loss
    from dinounet_b200.train_path import FusedSGD, train_step
    net = _net(dev)
    before = {n: p.detach().clone() for n, p in net.named_parameters() if p.requires_grad}
    crit = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": True}, {}, weight_ce=1, weight_dice=1)
    train_step(net, crit, FusedSGD(net.parameters(), lr=1e-2), x.to(dev), t.to(dev))
    return {n: (p.detach() - before[n]).cpu() for n, p in net.named_parameters() if n in before}


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        from dinounet_b200.loss import DC_and_BCE_loss, DC_and_CE_loss
        from oracle import region_loss_oracle as RO
        ref = np.load(GOLDEN)
        errs = {}
        for kind in ("bce", "ce"):
            if kind == "bce":
                crit = DC_and_BCE_loss({}, {"batch_dice": True, "do_bg": True, "smooth": 1e-5, "ddp": True},
                                       use_ignore_label=True)
            else:
                crit = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": True}, {}, 1, 1)
            z, t = RO.ddp_shard(kind, rank)
            z = z.to(dev).requires_grad_(True)
            loss = crit(z, t.to(dev))
            (loss * RO.DDP_SCALES[rank]).backward()
            want, gref = ref[f"ddp_{kind}_{rank}_loss"], ref[f"ddp_{kind}_{rank}_grad"]
            errs[kind] = (abs(float(loss) - float(want)) / max(1.0, abs(float(want))),
                          float(np.abs(RO.strided(z.grad).cpu().numpy() - gref).max() / np.abs(gref).max()))
        x, t = _step_inputs()
        lo, hi = rank * 2, rank * 2 + 2
        delta = _train_delta(dev, x[lo:hi], t[lo:hi])
        flat = torch.cat([d.reshape(-1) for d in delta.values()]).to(dev)
        other = flat.clone()
        dist.broadcast(other, src=0)
        same = bool(torch.equal(flat, other))
        q.put((rank, errs, same, {n: d for n, d in delta.items()} if rank == 0 else None))
    finally:
        dist.destroy_process_group()


@needs2
def test_nccl_batch_dice_matches_gloo_reference_and_single_gpu_step():
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
    for rank, errs, same, _ in res:
        for kind, (lerr, gerr) in errs.items():
            assert lerr <= 2e-6 and gerr < 1e-5, (rank, kind, lerr, gerr)
        assert same, f"rank {rank}: parameters differ between ranks after the step"
    dp = res[0][3]
    x, t = _step_inputs()
    one = _train_delta(torch.device("cuda", 0), x, t)
    d1 = torch.cat([one[n].reshape(-1) for n in one])
    ddp = torch.cat([dp[n].reshape(-1) for n in one])
    err = float((ddp - d1).abs().max() / d1.abs().max())
    print("data-parallel step vs one GPU: max|d_dp - d_1| / max|d_1| =", err)
    assert err <= 1e-4, err
