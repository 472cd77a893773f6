"""-m gpu, needs >= 2 GPUs (skipped below): train_semantics="reference" under data parallelism, spawned processes as in
test_gpu_dp_loss.py.  One train step (fp32 tiers) on 2 ranks x 2 samples against one GPU with the 4 samples, with the
same injected RoPE scales and each rank given its slice of the DropPath keep flags:

  * the BatchNorm statistics are taken over both ranks (SyncBatchNorm): the running statistics are bit-identical on the
    two ranks and within 1e-5 (relative to each tensor's largest value) of the one-GPU run;
  * the parameter update agrees: max|d_dp - d_1| <= 1e-4 * max|d_1|.
"""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0
needs2 = pytest.mark.skipif(NGPU < 2, reason="needs two GPUs")
BN_SUFFIXES = (".running_mean", ".running_var", ".num_batches_tracked")


def _inputs():
    from oracle import dinounet_oracle as O
    x = O.make_input(4, 128, 9)
    t = torch.randint(0, 2, (4, 1, 128, 128), generator=torch.Generator().manual_seed(10)).float()
    g = torch.Generator().manual_seed(11)
    scales = torch.exp(torch.empty(12).uniform_(-0.69, 0.69, generator=g))
    keep = torch.tensor([[1, 0, 1, 1], [0, 1, 1, 0], [1, 1, 0, 1], [1, 1, 1, 1], [0, 1, 1, 1], [1, 0, 1, 0]], dtype=torch.float32)
    return x, t, scales, keep


def _step(dev, lo, hi):
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    import dinounet_b200
    from dinounet_b200 import config
    from dinounet_b200.loss import DC_and_CE_loss
    from dinounet_b200.train_path import FusedSGD, all_reduce_gradients
    from oracle import dinounet_oracle as O
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, 2, None, "dinounet_s")
    net.load_state_dict(O.make_state_dict("dinounet_s", 2, seed=0), strict=True)
    net.precision, net.train_gemm, net.train_semantics = "fp32", "fp32", "reference"
    net = net.to(dev).train()
    x, t, scales, keep = _inputs()
    before = {n: p.detach().clone() for n, p in net.named_parameters() if p.requires_grad}
    crit = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": True}, {}, weight_ce=1, weight_dice=1)
    opt = FusedSGD(net.parameters(), lr=1e-2)
    opt.zero_grad()
    logits = net.train_forward(x[lo:hi].to(dev), rope_scales=scales.to(dev), drop_keep=keep[:, lo:hi].to(dev))
    crit(logits, t[lo:hi].to(dev)).backward()
    all_reduce_gradients(opt.params)
    opt.step()
    torch.cuda.synchronize(dev)
    delta = {n: (p.detach() - before[n]).cpu() for n, p in net.named_parameters() if n in before}
    bufs = {k: v.detach().cpu().clone() for k, v in net.state_dict().items() if k.endswith(BN_SUFFIXES) and not k.startswith("decoder.")}
    return delta, bufs


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        delta, bufs = _step(dev, 2 * rank, 2 * rank + 2)
        q.put((rank, delta if rank == 0 else None, bufs))
    finally:
        dist.destroy_process_group()


@needs2
def test_sync_batchnorm_step_on_two_ranks_matches_one_gpu():
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
    b0, b1 = res[0][2], res[1][2]
    assert len(b0) == 30
    assert all(torch.equal(b0[k], b1[k]) for k in b0), "running statistics differ between ranks"
    one, b_one = _step(torch.device("cuda", 0), 0, 4)
    for k, v in b_one.items():
        err = float((b0[k].double() - v.double()).abs().max() / max(v.double().abs().max(), 1e-12))
        assert err <= 1e-5, (k, err)
    dp = res[0][1]
    d1 = torch.cat([one[n].reshape(-1) for n in one])
    ddp = torch.cat([dp[n].reshape(-1) for n in one])
    err = float((ddp - d1).abs().max() / d1.abs().max())
    print("reference-semantics data-parallel step vs one GPU: max|d_dp - d_1| / max|d_1| =", err)
    assert err <= 1e-4, err
