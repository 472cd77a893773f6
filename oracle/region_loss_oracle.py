"""TEST INFRASTRUCTURE ONLY — torch restatement of the reference's region loss (Dice + BCE), its online-validation
counts, and data-parallel batch Dice for both losses.

Follows: training/loss/compound_losses.py:59-99 (`DC_and_BCE_loss.forward`, with and without the ignore channel),
dice.py:72-119 (`MemoryEfficientSoftDiceLoss.forward`, sigmoid or softmax, `ddp`), utilities/ddp_allgather.py
(`AllGatherGrad`: all_gather -> stack forward, all_reduce(SUM) of the incoming gradient backward), dice.py:122-178
(`get_tp_fp_fn_tn`), nnUNetTrainer.py:356-365 (construction) and :973-994 (validation_step's region branch).
Pinned against the REAL reference classes through tests/golden/region_loss_cases.npz
(oracle/make_golden_region_loss.py), including a 2-process gloo run of the DDP path.
"""
import os
import sys

import torch
import torch.nn.functional as F


def region_case(B, R, H, W, seed, use_ignore=False, ignore_all=False):
    """Seeded logits [B, R, H, W] (scale 3) and a float region target [B, R(+1), H, W] (about 20% ignored pixels)."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, R, H, W, generator=g) * 3
    t = (torch.rand(B, R, H, W, generator=g) < 0.4).float()
    if use_ignore:
        ign = torch.ones(B, 1, H, W) if ignore_all else (torch.rand(B, 1, H, W, generator=g) < 0.2).float()
        t = torch.cat([t, ign], 1)
    return z, t


def label_case(B, C, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, C, H, W, generator=g) * 3, torch.randint(0, C, (B, 1, H, W), generator=g).float()


# golden cases (oracle/make_golden_region_loss.py, tests/test_region_loss_cpu.py, tests/test_gpu_dp_loss.py)
REGION_CASES = [(bd, ign, R) for bd in (True, False) for ign in (True, False) for R in (1, 3)]
REGION_SHAPE = (2, 23, 19)                         # B, H, W
DDP_WORLD, DDP_SHARD, DDP_SHAPE, DDP_SCALES = 2, 2, (21, 17), (1.0, 2.0)
DDP_CASES = {"bce": dict(R=3, use_ignore=True), "ce": dict(C=3)}


def ddp_shard(kind, rank):
    """Rank `rank`'s shard of the data-parallel golden case."""
    H, W = DDP_SHAPE
    if kind == "bce":
        return region_case(DDP_SHARD, DDP_CASES["bce"]["R"], H, W, 500 + rank, use_ignore=True)
    return label_case(DDP_SHARD, DDP_CASES["ce"]["C"], H, W, 600 + rank)


def strided(t, n=256):
    f = t.detach().reshape(-1)
    return f[:: max(1, f.numel() // n)][:n]


def _dice_sums(x, y, loss_mask=None, do_bg=True):
    """intersect, sum_pred, sum_gt [B, C] of MemoryEfficientSoftDiceLoss after its nonlinearity (dice.py:80-104)."""
    axes = tuple(range(2, x.ndim))
    with torch.no_grad():
        if x.ndim != y.ndim:
            y = y.view((y.shape[0], 1, *y.shape[1:]))
        if x.shape == y.shape:
            y_onehot = y
        else:
            y_onehot = torch.zeros(x.shape, device=x.device, dtype=torch.bool)
            y_onehot.scatter_(1, y.long(), 1)
        if not do_bg:
            y_onehot = y_onehot[:, 1:]
        sum_gt = y_onehot.sum(axes) if loss_mask is None else (y_onehot * loss_mask).sum(axes)
    if not do_bg:
        x = x[:, 1:]
    if loss_mask is None:
        intersect = (x * y_onehot).sum(axes)
        sum_pred = x.sum(axes)
    else:
        intersect = (x * y_onehot * loss_mask).sum(axes)
        sum_pred = (x * loss_mask).sum(axes)
    return intersect, sum_pred, sum_gt


def _dice_from_sums(intersect, sum_pred, sum_gt, batch_dice, smooth):
    if batch_dice:
        intersect, sum_pred, sum_gt = intersect.sum(0), sum_pred.sum(0), sum_gt.sum(0)
    dc = (2 * intersect + smooth) / (torch.clip(sum_gt + sum_pred + smooth, 1e-8))
    return -dc.mean()


def _split_ignore(target, use_ignore):
    if not use_ignore:
        return target, None
    return torch.clone(target[:, :-1]), (1 - target[:, -1:]).bool()


def _bce(logits, target_regions, mask):
    if mask is None:
        return F.binary_cross_entropy_with_logits(logits, target_regions)
    return (F.binary_cross_entropy_with_logits(logits, target_regions, reduction="none") * mask).sum() / \
        torch.clip(mask.sum(), min=1e-8)


def dc_and_bce_loss(logits, target, batch_dice=True, use_ignore=False, smooth=1e-5, weight_ce=1, weight_dice=1):
    """DC_and_BCE_loss as the trainer builds it (do_bg, MemoryEfficientSoftDiceLoss on sigmoid, ddp off).
    target [B, R(+1 ignore channel), ...] float -> (loss, bce, dice term)"""
    target_regions, mask = _split_ignore(target, use_ignore)
    dc = _dice_from_sums(*_dice_sums(torch.sigmoid(logits), target_regions, mask), batch_dice, smooth)
    ce = _bce(logits, target_regions, mask)
    return weight_ce * ce + weight_dice * dc, ce, dc


def region_validation_counts(logits, target, use_ignore=False):
    """nnUNetTrainer.py:973-994 for regions: tp, fp, fn of (sigmoid > 0.5) per region, weighted by 1 - t_ign."""
    axes = [0] + list(range(2, logits.ndim))
    pred = (torch.sigmoid(logits) > 0.5).long()
    mask = None
    if use_ignore:
        mask = 1 - target[:, -1:]
        target = target[:, :-1]
    tp = pred * target
    fp = pred * (1 - target)
    fn = (1 - pred) * target
    if mask is not None:
        mask_here = torch.tile(mask, (1, tp.shape[1], *[1 for _ in range(2, tp.ndim)]))
        tp, fp, fn = tp * mask_here, fp * mask_here, fn * mask_here
    return tp.sum(dim=axes), fp.sum(dim=axes), fn.sum(dim=axes)


def ddp_losses(kind, logits, targets, use_ignore=False, do_bg=None, smooth=1e-5, weight_ce=1, weight_dice=1):
    """Per-rank losses of W data-parallel ranks simulated in one process, batch_dice and ddp on.

    kind 'bce' (DC_and_BCE_loss, do_bg True) or 'ce' (DC_and_CE_loss, do_bg False, no ignore label); logits / targets are
    lists with one shard per rank.  Each rank's Dice sums go through AllGatherGrad -> `stack` -> `sum(0)` -> `sum(0)`
    (dice.py:106-114) from one shared stacked tensor, so that backward of sum_r(scale_r * loss_r) accumulates into that
    tensor the sum over ranks of their incoming gradients -- exactly what AllGatherGrad's all_reduce hands each rank.
    The CE / BCE term stays local."""
    if do_bg is None:
        do_bg = kind == "bce"
    sums, ces = [], []
    for z, t in zip(logits, targets):
        if kind == "bce":
            t_reg, mask = _split_ignore(t, use_ignore)
            sums.append(_dice_sums(torch.sigmoid(z), t_reg, mask, do_bg=True))
            ces.append(_bce(z, t_reg, mask))
        else:
            sums.append(_dice_sums(torch.softmax(z, 1), t, None, do_bg=do_bg))
            ces.append(F.cross_entropy(z, t[:, 0].long()))
    gathered = [torch.stack([s[k] for s in sums], dim=0) for k in range(3)]
    losses = []
    for ce in ces:
        intersect, sum_pred, sum_gt = (g.sum(0) for g in gathered)
        dc = _dice_from_sums(intersect, sum_pred, sum_gt, True, smooth)
        losses.append(weight_ce * ce + weight_dice * dc)
    return losses


def load_reference_region_loss():
    """The REAL `DC_and_BCE_loss`, `DC_and_CE_loss`, `MemoryEfficientSoftDiceLoss`, `get_tp_fp_fn_tn` (where the
    reference is importable; oracle/ref_loader.py shims)."""
    from . import ref_loader
    ref_loader._install_shims()
    tr = sys.modules["dinounet.training"]
    real = os.path.join(ref_loader.REF_ROOT, "dinounet", "training")
    if real not in tr.__path__:
        tr.__path__.append(real)
    from dinounet.training.loss.compound_losses import DC_and_BCE_loss, DC_and_CE_loss
    from dinounet.training.loss.dice import MemoryEfficientSoftDiceLoss, get_tp_fp_fn_tn
    return DC_and_BCE_loss, DC_and_CE_loss, MemoryEfficientSoftDiceLoss, get_tp_fp_fn_tn
