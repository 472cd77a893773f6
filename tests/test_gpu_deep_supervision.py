"""-m gpu: deep supervision on the native path.

* Target kernel (b2u_ds_targets) bit-exact against the restatement of skimage's order-0 resize
  (oracle/deep_supervision_oracle.py) at batch 32, 512^2: int16 label maps and fp32 regions + ignore channel; scale 1
  is the input itself; shapes it cannot tile raise before any launch.
* Eval forward with decoder.deep_supervision set: the three heads against the REAL reference's
  (tests/golden/deep_supervision_cases.npz) within 1e-5 on the fp32 tier and 1.2e-2 on the 16-bit tier (relative to the
  largest logit, as smoke()); logits@S bit-identical to the forward without deep supervision.
* Training step: gradients of the weighted objective against the golden on the fp32 GEMM tier (test_gpu_train.py's 2e-3
  bar) and the TF32 tier (its TF32 bars), label maps and regions + ignore channel; seg_layers.0 gets no gradient.
* Two ranks (gloo on one device) with the DDP weights: the 1e-6 head gets a real gradient, the same on both ranks.
* A short trainer run with device augmentation, device loading and deep supervision: train steps, a validation step, a
  checkpoint, and a final validation whose files equal a trainer's without deep supervision on the same weights.
"""
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import dinounet_b200
from dinounet_b200 import config, lib as L
from dinounet_b200 import deep_supervision as DS
from dinounet_b200.loss import DC_and_BCE_loss, DC_and_CE_loss, DeepSupervisionWrapper
from oracle import deep_supervision_oracle as DSO
from oracle import dinounet_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "deep_supervision_cases.npz")
SCALES = [[1.0, 1.0], [0.5, 0.5], [0.25, 0.25]]
MODEL, B, S, NCLS, WSEED = "dinounet_s", 2, 128, 2, 0


def _net(precision="fp32", gemm="fp32"):
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, NCLS, None, MODEL)
    net.load_state_dict(O.make_state_dict(MODEL, NCLS, seed=WSEED), strict=True)
    net.precision, net.train_gemm = precision, gemm
    net.decoder.deep_supervision = True
    return net.to(DEV)


# ------------------------------------------------------------------------------------------------ target kernel
def test_target_kernel_is_bit_exact_at_batch_32_512():
    g = torch.Generator().manual_seed(3)
    lab = torch.randint(-1, 5, (32, 1, 512, 512), generator=g, dtype=torch.int16)
    reg = torch.rand((32, 3, 512, 512), generator=g).round()
    reg[:, 1] *= 0.5                                   # values other than 0 / 1 pass through unchanged too
    for t in (lab, reg):
        td = t.to(DEV)
        n0 = L.launch_count()
        got = DS.downsample_targets(td, SCALES)
        torch.cuda.synchronize()
        assert L.launch_count() - n0 == 1
        want = DSO.downsample_seg_for_ds(t.numpy(), SCALES)
        assert got[0] is td
        for s in (1, 2):
            assert got[s].dtype == t.dtype and tuple(got[s].shape) == want[s].shape
            assert np.array_equal(got[s].cpu().numpy(), want[s]), (t.dtype, s)
        print(f"{t.dtype}: {[tuple(x.shape) for x in got]} bit-exact")


def test_target_kernel_rejects_before_launching():
    t = torch.zeros(2, 1, 510, 512, dtype=torch.int16, device=DEV)
    torch.cuda.synchronize()
    n0 = L.launch_count()
    with pytest.raises(NotImplementedError):
        DS.downsample_targets(t, SCALES)               # 510 / 4 is not an integer
    with pytest.raises(NotImplementedError):
        DS.downsample_targets(t, [[1 / 3, 1 / 3]])     # 512 / 3 is not an integer
    with pytest.raises(ValueError):
        DS.downsample_targets(t.long(), SCALES)
    assert L.launch_count() == n0


# ------------------------------------------------------------------------------------------------ eval forward
@pytest.mark.parametrize("precision,bar", [("fp32", 1e-5), ("16", 1.2e-2)])
def test_eval_forward_heads_match_the_reference(precision, bar):
    g = np.load(GOLDEN)
    net = _net(precision).eval()
    x = O.make_input(B, S, WSEED).to(DEV)
    n0 = L.launch_count()
    with torch.no_grad():
        outs = net(x)
        torch.cuda.synchronize()
        assert L.launch_count() - n0 > 100, "native kernels did not run"
        assert isinstance(outs, list) and len(outs) == 3
        for i, o in enumerate(outs):
            want = g[f"logits{i}"]
            assert tuple(o.shape) == want.shape
            err = np.abs(o.cpu().numpy() - want).max() / np.abs(want).max()
            print(f"[{precision}] logits{i} {tuple(o.shape)}: max rel err {err:.3e}")
            assert err <= bar, (i, err)
        net.decoder.deep_supervision = False
        plain = net(x)
        assert torch.equal(plain, outs[0])              # logits@S: the forward without deep supervision, bit for bit
        assert torch.equal(net.predict_labels(x), plain.argmax(1).to(torch.uint8))


# ------------------------------------------------------------------------------------------------ training step
SAMPLE_BAR = {"lm": 2e-3, "rg": 2e-2}


def _targets(prefix):
    from oracle import make_golden_deep_supervision as MG
    t = MG.label_map() if prefix == "lm" else MG.region_target()
    return DS.downsample_targets(t.to(DEV), SCALES)


def _crit(prefix, ddp=False):
    if prefix == "lm":
        base = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": ddp}, {}, weight_ce=1, weight_dice=1)
    else:
        base = DC_and_BCE_loss({}, {"batch_dice": True, "do_bg": True, "smooth": 1e-5, "ddp": ddp}, use_ignore_label=True)
    return DeepSupervisionWrapper(base, DS.deep_supervision_weights(3, ddp))


def _grads(prefix, gemm):
    net = _net("fp32", gemm).train()
    x = O.make_input(B, S, WSEED).to(DEV)
    n0 = L.launch_count()
    outs = net(x)
    assert isinstance(outs, list) and [tuple(o.shape[2:]) for o in outs] == [(S, S), (S // 2, S // 2), (S // 4, S // 4)]
    loss = _crit(prefix)(outs, _targets(prefix))
    loss.backward()
    torch.cuda.synchronize()
    assert L.launch_count() - n0 > 500, "native kernels did not run"
    sdv = net.state_dict(keep_vars=True)
    assert sdv["decoder.seg_layers.0.weight"].grad is None and sdv["decoder.seg_layers.0.bias"].grad is None
    assert sdv["decoder.seg_layers.1.weight"].grad is not None
    return loss.item(), sdv


@pytest.mark.parametrize("prefix", ["lm", "rg"], ids=["label_map", "regions_ignore"])
def test_fp32_tier_gradients_match_the_golden(prefix):
    """Loss 1e-5; per-tensor norms 2e-3 (+1e-7); 16 strided samples per tensor within SAMPLE_BAR[prefix] of the tensor's
    largest sample (+1e-7): 2e-3 for label maps as test_gpu_train.py, 2e-2 for the region loss, whose BCE + Dice gradient
    cancels to small values in many elements."""
    g = np.load(GOLDEN)
    loss, sdv = _grads(prefix, "fp32")
    want_loss = float(g[f"{prefix}_loss"])
    assert abs(loss - want_loss) <= 1e-5 * max(1.0, abs(want_loss)), (loss, want_loss)
    bad, worst = [], 0.0
    for i, k in enumerate(str(n) for n in g[f"{prefix}_names"]):
        gr = sdv[k].grad
        assert (gr is not None) == bool(g[f"{prefix}_has_grad"][i]), k
        if gr is None:
            continue
        gr = gr.detach().float().cpu()
        want = float(g[f"{prefix}_norms"][i])
        fl = gr.reshape(-1)
        samp = fl[:: max(1, fl.numel() // 16)][:16].numpy()
        ws = g[f"{prefix}_s{i}"]
        serr = float(np.abs(samp - ws).max() / max(np.abs(ws).max(), 1e-12))
        worst = max(worst, serr)
        if not (abs(gr.double().norm().item() - want) <= 2e-3 * want + 1e-7) or \
                not (np.abs(samp - ws).max() <= SAMPLE_BAR[prefix] * np.abs(ws).max() + 1e-7):
            bad.append((k, gr.double().norm().item(), want, serr))
    print(f"[fp32 {prefix}] loss {loss:.6f} (golden {want_loss:.6f}), worst sample err {worst:.2e}, {len(bad)} tensors off")
    assert not bad, bad[:8]


def test_tf32_tier_gradients_stay_within_the_tf32_bars():
    """test_gpu_train.py's TF32 bars: loss 2e-3, per-tensor norm 5e-2 (here for the tensors above 1e-2 of the largest
    norm: the small SE gradients of this objective land just above it), sampled elements rel L2 0.15 and cosine 0.98."""
    g = np.load(GOLDEN)
    loss, sdv = _grads("lm", "tf32")
    assert abs(loss - float(g["lm_loss"])) <= 2e-3 * max(1.0, abs(float(g["lm_loss"])))
    top = float(np.max(g["lm_norms"]))
    bad, errs, refs = [], [], []
    for i, k in enumerate(str(n) for n in g["lm_names"]):
        want = float(g["lm_norms"][i])
        gr = sdv[k].grad
        if gr is None or want <= 1e-4 * top:
            continue
        gr = gr.detach().float().cpu()
        assert torch.isfinite(gr).all(), k
        rel = abs(gr.double().norm().item() - want) / want
        fl = gr.reshape(-1)
        samp = fl[:: max(1, fl.numel() // 16)][:16].numpy().astype(np.float64)
        rms = want / np.sqrt(fl.numel())
        errs.append((samp - g[f"lm_s{i}"]) / rms)
        refs.append(g[f"lm_s{i}"] / rms)
        if rel > 5e-2 and want > 1e-2 * top:
            bad.append((k, rel))
    E, R = np.concatenate(errs), np.concatenate(refs)
    rel_l2 = float(np.linalg.norm(E) / np.linalg.norm(R))
    cos = float(np.dot(R + E, R) / (np.linalg.norm(R + E) * np.linalg.norm(R)))
    print(f"[tf32] loss {loss:.6f}, rel L2 {rel_l2:.3e}, cosine {cos:.5f}")
    assert not bad, bad[:8]
    assert rel_l2 <= 0.15 and cos >= 0.98


# ------------------------------------------------------------------------------------------------ two ranks
def _ddp_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        _ddp_rank(rank, q)
    except BaseException as e:
        q.put((rank, repr(e)))          # the parent fails at once instead of waiting for a result
        raise
    finally:
        dist.destroy_process_group()


def _ddp_rank(rank, q):
    from dinounet_b200.train_path import FusedSGD, train_step
    net = _net("fp32", "fp32").train()
    crit = _crit("lm", ddp=True)
    assert crit.weight_factors[-1] > 0
    x = O.make_input(2, S, 20 + rank).to(DEV)
    t = torch.randint(0, NCLS, (2, 1, S, S), generator=torch.Generator().manual_seed(30 + rank)).float().to(DEV)
    opt = FusedSGD(net.parameters(), lr=1e-2)
    w0 = dict(net.named_parameters())["decoder.seg_layers.0.weight"].detach().clone()
    # the gradient of the 1e-6 head alone, before the exchange
    net.zero_grad()
    outs = net(x)
    (crit.weight_factors[2] * crit.loss(outs[2], DS.downsample_targets(t, SCALES)[2])).backward()
    local = dict(net.named_parameters())["decoder.seg_layers.0.weight"].grad.detach().clone()
    loss = train_step(net, crit, opt, x, DS.downsample_targets(t, SCALES))
    g0 = dict(net.named_parameters())["decoder.seg_layers.0.weight"].grad.detach().cpu()
    w1 = dict(net.named_parameters())["decoder.seg_layers.0.weight"].detach()
    q.put((rank, float(loss), local.cpu().numpy(), g0.numpy(), bool(torch.equal(w0, w1)),
           {n: p.detach().cpu().numpy() for n, p in net.named_parameters() if n.startswith("decoder.")}))


def test_two_ranks_give_the_small_weight_head_a_real_gradient():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    procs = [ctx.Process(target=_ddp_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=300) for _ in procs), key=lambda r: r[0])
    assert all(len(r) > 2 for r in res), res
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    (_, l0, loc0, g0, same0, p0), (_, l1, loc1, g1, same1, p1) = res
    assert np.isfinite(g0).all() and np.abs(g0).max() > 0 and np.array_equal(g0, g1)
    # the exchanged gradient is the mean of the ranks' own 1e-6 terms (the other terms do not reach seg_layers.0)
    assert np.allclose(g0, (loc0 + loc1) / 2, rtol=1e-5, atol=1e-12)
    assert not same0 and not same1                      # the optimizer updated the head
    for k in p0:
        assert np.array_equal(p0[k], p1[k]), k
    print(f"losses {l0:.6f} {l1:.6f}; |grad seg_layers.0| {float(np.linalg.norm(g0)):.3e}")


# ------------------------------------------------------------------------------------------------ trainer run
def test_trainer_run_with_device_pipeline_and_deep_supervision(tmp_path, monkeypatch):
    from dinounet_b200 import training as TR
    from dinounet_b200.dataloading import DeviceDataLoader2D
    from tests import test_gpu_dataloader as TDL
    from tests import test_gpu_trainer_loop as TTL
    monkeypatch.setattr(TR.DinoUNetTrainer, "_device_augmentation", True)
    monkeypatch.setattr(TR.DinoUNetTrainer, "_device_dataloading", True)
    monkeypatch.setattr(TR, "_validation_dataset", TTL._Dataset)
    sd = O.make_state_dict("dinounet_s", 3, seed=0)
    net = TDL._net(sd).train()
    tr, _, _ = TDL._trainer(net, (TDL._cases(3, 10), TDL._cases(2, 20)))
    tr.enable_deep_supervision = True
    tr.configuration_manager.pool_op_kernel_sizes = [[1, 1], [2, 2], [2, 2], [2, 2]]
    tr.configuration_manager.batch_dice = True
    tr.loss = tr._build_loss()
    assert isinstance(tr.loss, DeepSupervisionWrapper)
    tr.set_deep_supervision_enabled(True)
    assert net.decoder.deep_supervision
    dl_tr, dl_val = tr.get_dataloaders()
    assert isinstance(dl_tr, DeviceDataLoader2D)
    try:
        before = {n: p.detach().clone() for n, p in net.named_parameters() if n.startswith("decoder.seg_layers.")}
        losses = [float(tr.train_step(next(dl_tr))["loss"]) for _ in range(3)]
        after = dict(net.named_parameters())
        assert not torch.equal(before["decoder.seg_layers.1.weight"], after["decoder.seg_layers.1.weight"])
        assert torch.equal(before["decoder.seg_layers.0.weight"], after["decoder.seg_layers.0.weight"])
        net.eval()
        st = tr.validation_step(next(dl_val))
        assert np.isfinite(st["loss"]) and st["tp_hard"].shape == (2,)
        print(f"train losses {losses}, validation loss {float(st['loss']):.4f}")
    finally:
        dl_tr.close()
        dl_val.close()
    path = str(tmp_path / "checkpoint_final.pth")
    torch.save({"network_weights": net.state_dict(), "optimizer_state": tr.optimizer.state_dict()}, path)
    ck = torch.load(path, map_location=DEV, weights_only=False)
    # final validation with and without deep supervision on the same weights
    files = []
    for ds in (True, False):
        other = TDL._net(ck["network_weights"]).eval()
        vt, keys = TTL._stand_in(tmp_path / f"ds{int(ds)}", other, False)
        vt.enable_deep_supervision = ds
        other.decoder.deep_supervision = ds
        vt.perform_actual_validation()
        assert other.decoder.deep_supervision == ds        # switched off for the validation, back on after it
        files.append([np.load(os.path.join(vt.output_folder, "validation", k + ".npy")) for k in keys])
    for a, b in zip(*files):
        assert np.array_equal(a, b)
