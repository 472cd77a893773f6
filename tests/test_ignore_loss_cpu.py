"""Ignore-label loss oracle (oracle/ignore_loss_oracle.py) pinned bit for bit against what the REAL reference classes
computed (tests/golden/ignore_loss_cases.npz, oracle/make_golden_ignore_loss.py), including both ranks of a 2-process
gloo run; which C-ABI entry points `DC_and_CE_loss` calls with and without an ignore label (recording stand-in for the
native library); the ignore label's argument contract and the trainer's loss construction, without a GPU."""
import contextlib
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import ignore_loss_oracle as IO

REF = np.load(os.path.join(os.path.dirname(__file__), "golden", "ignore_loss_cases.npz"))


def _check_case(key, z, t, C, batch_dice):
    z1 = z.clone().requires_grad_(True)
    got, ce, dc = IO.dc_and_ce_loss(z1, t, C, batch_dice=batch_dice)
    assert np.array_equal(got.detach().numpy(), REF[key + "_loss"])
    got.backward()
    assert np.array_equal(IO.strided(z1.grad).numpy(), REF[key + "_grad"])
    tp, fp, fn = IO.validation_counts(z, t, C)
    for name, v in (("tp", tp), ("fp", fp), ("fn", fn)):
        assert v.dtype == torch.float32 and np.array_equal(v.numpy(), REF[f"{key}_{name}"]), name
    return z1.grad, ce, dc


@pytest.mark.parametrize("seed,case", list(enumerate(IO.IGN_CASES)))
def test_ignore_oracle_equals_reference_classes(seed, case):
    """DC_and_CE_loss(ignore_label=C) (nnUNetTrainer.py:363-365) and validation_step's masked counts, bit for bit."""
    bd, C = case
    B, H, W = IO.IGN_SHAPE
    z, t = IO.ignore_case(B, C, H, W, seed)
    ign = t == C
    assert 0.1 < float(ign.float().mean()) < 0.3
    grad, _, _ = _check_case(f"ign_{int(bd)}_{C}", z, t, C, bd)
    assert not grad.masked_select(ign.expand_as(grad)).any()


def test_ignore_oracle_one_sample_ignored():
    B, H, W = IO.IGN_SHAPE
    z, t = IO.ignore_case(B, IO.EDGE_C, H, W, 98, ignored_samples=(1,))
    grad, _, _ = _check_case("onesample", z, t, IO.EDGE_C, False)
    assert not grad[1].any() and grad[0].any()


def test_ignore_oracle_all_ignored():
    B, H, W = IO.IGN_SHAPE
    z, t = IO.ignore_case(B, IO.EDGE_C, H, W, 99, ignored_samples=range(B))
    grad, ce, dc = _check_case("allign", z, t, IO.EDGE_C, True)
    assert float(ce.detach()) == 0.0 and float(dc.detach()) == -1.0 and not grad.any()
    assert not REF["allign_tp"].any() and not REF["allign_fp"].any() and not REF["allign_fn"].any()


def test_ddp_ignore_oracle_equals_gloo_reference():
    """W ranks simulated in one process == the reference's AllGatherGrad run on 2 gloo processes, both ranks."""
    shards = [IO.ddp_shard(r) for r in range(IO.DDP_WORLD)]
    zs = [z.clone().requires_grad_(True) for z, _ in shards]
    losses = IO.ddp_losses(zs, [t for _, t in shards], IO.DDP_C)
    sum(s * l for s, l in zip(IO.DDP_SCALES, losses)).backward()
    for r in range(IO.DDP_WORLD):
        assert np.array_equal(losses[r].detach().numpy(), REF[f"ddp_{r}_loss"]), r
        assert np.array_equal(IO.strided(zs[r].grad).numpy(), REF[f"ddp_{r}_grad"]), r


# ---- which native entry points run


class _Recorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*a):
            self.calls.append((name, a))
            return 64 if name.endswith("_work_doubles") else 0
        return fn


@pytest.fixture
def rec(monkeypatch):
    from dinounet_b200 import lib as L
    from dinounet_b200 import loss as LS
    r = _Recorder()
    monkeypatch.setattr(L, "load", lambda: r)
    # CPU tensors stand in for device buffers: the stand-in library never reads them
    prep = lambda z, t, *_: (z.float().contiguous(), t.contiguous(), z.shape[0], z.shape[1], int(np.prod(z.shape[2:])))
    monkeypatch.setattr(LS, "_prep", prep)
    monkeypatch.setattr(LS, "_prep_regions", prep)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda dev=None: type("S", (), {"cuda_stream": 0})())
    return r


def _fwd_bwd(monkeypatch, regions, ignore, batch_dice, all_reduce):
    """One forward + backward of the label-map loss (ignore label 3) or the region loss (ignore channel); with
    `all_reduce`, as under data-parallel batch Dice (the all-reduce itself is the identity here)."""
    from dinounet_b200 import loss as LS
    if all_reduce:
        monkeypatch.setattr(LS, "_ddp_batch_dice", lambda batch_dice, ddp: True)
        monkeypatch.setattr(torch.distributed, "all_reduce", lambda t: None)
    dice_kw = {"batch_dice": batch_dice, "smooth": 1e-5, "do_bg": regions, "ddp": all_reduce}
    if regions:
        mod, t = LS.DC_and_BCE_loss({}, dice_kw, use_ignore_label=ignore), torch.zeros(2, 3 + ignore, 8, 8)
    else:
        mod, t = LS.DC_and_CE_loss(dice_kw, {}, 1, 1, ignore_label=3 if ignore else None), torch.zeros(2, 1, 8, 8)
    z = torch.zeros(2, 3, 8, 8, requires_grad=True)
    mod(z, t).backward()


# argument positions in the (stats, finalize, backward) calls: work, batch_sums, and the has-ignore flag; batch_dice in
# finalize and backward
_POS = {"dice_ce": dict(work=(5, 0, 5), bsum=(6, 1, 6), ign=(3, 7, 3), batch_dice=(10, 13)),
        "dice_bce": dict(work=(4, 0, 4), bsum=(5, 1, 5), ign=(3, 10, 3), batch_dice=(9, 12))}


def _check_calls(rec, fam, ignore, batch_dice, all_reduce):
    """The one call sequence of every configuration: one work buffer shared by the three calls; the batch sums NULL in
    all three for label maps without an all-reduce, else one buffer shared by all three; batch_dice reaching finalize
    and backward.  Returns the (stats, finalize, backward) arguments."""
    assert [n for n, _ in rec.calls] == [f"b2u_{fam}_{s}" for s in ("work_doubles", "stats", "finalize", "backward")]
    calls = [a for _, a in rec.calls[1:]]
    pos = _POS[fam]
    work = {a[i] for a, i in zip(calls, pos["work"])}
    assert len(work) == 1 and None not in work and 0 not in work
    bsum = [a[i] for a, i in zip(calls, pos["bsum"])]
    assert bsum == [bsum[0]] * 3 and (bsum[0] is not None) == (all_reduce or fam == "dice_bce")
    assert [a[i] for a, i in zip(calls, pos["ign"])] == [int(ignore)] * 3
    (fin, bwd), (i_fin, i_bwd) = calls[1:], pos["batch_dice"]
    assert fin[i_fin] == batch_dice and bwd[i_bwd] == batch_dice
    return calls


# batch_dice (the ids the label-map cases had when they took only that), the same under an all-reduce, the region loss
_CASES = [pytest.param(False, False, False, id="False"), pytest.param(True, False, False, id="True"),
          pytest.param(True, True, False, id="all_reduce"), pytest.param(False, False, True, id="regions-False"),
          pytest.param(True, False, True, id="regions-True"), pytest.param(True, True, True, id="regions-all_reduce")]


@pytest.mark.parametrize("batch_dice,all_reduce,regions", _CASES)
def test_no_ignore_label_runs_todays_calls(rec, monkeypatch, batch_dice, all_reduce, regions):
    _fwd_bwd(monkeypatch, regions, False, batch_dice, all_reduce)
    bwd = _check_calls(rec, "dice_bce" if regions else "dice_ce", False, batch_dice, all_reduce)[2]
    if not regions and not all_reduce:   # unit scales in the kernel; the incoming gradient is applied in torch
        assert bwd[16] is None and bwd[17] is None


@pytest.mark.parametrize("batch_dice,all_reduce,regions", _CASES)
def test_ignore_label_runs_the_ignore_family(rec, monkeypatch, batch_dice, all_reduce, regions):
    _fwd_bwd(monkeypatch, regions, True, batch_dice, all_reduce)
    stats, _, bwd = _check_calls(rec, "dice_bce" if regions else "dice_ce", True, batch_dice, all_reduce)
    if not regions:
        assert stats[4] == 3 and bwd[4] == 3                               # the ignore label reaches both passes
    assert bwd[-3] is not None and bwd[-2] is not None                     # the scales come from the device


# ---- argument contract and the trainer


def test_ignore_label_argument_contract():
    """Accepted for the trainer's label-map configuration (do_bg=False); rejected with do_bg=True, for a label that is
    not a 32-bit integer, and for CE options; CPU tensors raise (no fallback)."""
    from dinounet_b200.lib import NativeLibraryError
    from dinounet_b200.loss import DC_and_CE_loss
    kw = {"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}
    m = DC_and_CE_loss(kw, {}, weight_ce=1, weight_dice=1, ignore_label=3)
    assert (m.ignore_label, m.batch_dice, m.do_bg, m.smooth) == (3, True, False, 1e-5)
    assert DC_and_CE_loss(kw, {}, ignore_label=np.int64(4)).ignore_label == 4
    for bad in (2.5, 2 ** 31):
        with pytest.raises(ValueError):
            DC_and_CE_loss(kw, {}, ignore_label=bad)
    for dice_kw in ({"batch_dice": True}, {**kw, "do_bg": True}):
        with pytest.raises(NotImplementedError):
            DC_and_CE_loss(dice_kw, {}, ignore_label=3)
    with pytest.raises(NotImplementedError):
        DC_and_CE_loss(kw, {"label_smoothing": 0.1}, ignore_label=3)
    with pytest.raises(NativeLibraryError):
        m(torch.zeros(1, 2, 4, 4), torch.zeros(1, 1, 4, 4))


@pytest.mark.parametrize("is_ddp", [False, True])
@pytest.mark.parametrize("batch_dice", [False, True])
def test_trainer_builds_ignore_label_loss(is_ddp, batch_dice):
    """`_build_loss` for a label-map dataset with an ignore label: DC_and_CE_loss({batch_dice, smooth 1e-5, do_bg False,
    ddp}, {}, 1, 1, ignore_label) (nnUNetTrainer.py:363-365)."""
    import dinounet_b200
    from dinounet_b200.loss import DC_and_CE_loss
    tr = dinounet_b200.DinoUNetTrainer_s.__new__(dinounet_b200.DinoUNetTrainer_s)
    tr.is_ddp = is_ddp
    tr.configuration_manager = SimpleNamespace(batch_dice=batch_dice)
    tr.label_manager = SimpleNamespace(has_regions=False, ignore_label=4, has_ignore_label=True)
    m = tr._build_loss()
    assert isinstance(m, DC_and_CE_loss)
    assert (m.batch_dice, m.do_bg, m.smooth, m.ddp, m.ignore_label) == (batch_dice, False, 1e-5, is_ddp, 4)
    assert (m.weight_ce, m.weight_dice) == (1, 1)
