"""TEST INFRASTRUCTURE ONLY — torch restatement of the reference's softmax Dice + CE loss with an ignore label, its
online-validation counts, and data-parallel batch Dice with the ignore label.

Follows: training/loss/compound_losses.py:21-56 (`DC_and_CE_loss` with `ignore_label`: loss_mask = target != ignore,
Dice on where(mask, target, 0), CE with ignore_index, skipped when no pixel is valid), dice.py:72-119
(`MemoryEfficientSoftDiceLoss.forward` with `loss_mask`), robust_ce_loss.py:12-16, nnUNetTrainer.py:977-994
(validation_step's label-map branch with an ignore label) and dice.py:122-178 (`get_tp_fp_fn_tn` with a mask).
Pinned against the REAL reference classes through tests/golden/ignore_loss_cases.npz
(oracle/make_golden_ignore_loss.py), including a 2-process gloo run of the DDP path.
"""
import torch
import torch.nn.functional as F

from .region_loss_oracle import DDP_SCALES, DDP_SHAPE, DDP_SHARD, DDP_WORLD, _dice_from_sums, _dice_sums, strided  # noqa: F401

# golden cases (oracle/make_golden_ignore_loss.py, tests/test_ignore_loss_cpu.py, tests/test_gpu_ignore_loss.py)
IGN_CASES = [(bd, C) for bd in (True, False) for C in (2, 3, 5)]
IGN_SHAPE = (2, 23, 19)                            # B, H, W
IGN_FRACTION = 0.2
EDGE_C = 3                                         # class count of the fully ignored sample / batch cases
DDP_C = 3


def ignore_case(B, C, H, W, seed, ignore_label=None, fraction=IGN_FRACTION, ignored_samples=()):
    """Seeded logits [B, C, H, W] (scale 3) and a float label map [B, 1, H, W] in [0, C) with about `fraction` of the
    pixels, and every pixel of the samples in `ignored_samples`, set to `ignore_label` (default C, as nnU-Net has it)."""
    ign = C if ignore_label is None else ignore_label
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, C, H, W, generator=g) * 3
    t = torch.randint(0, C, (B, 1, H, W), generator=g).float()
    t[torch.rand(B, 1, H, W, generator=g) < fraction] = ign
    for b in ignored_samples:
        t[b] = ign
    return z, t


def ddp_shard(rank):
    """Rank `rank`'s shard of the data-parallel golden case."""
    H, W = DDP_SHAPE
    return ignore_case(DDP_SHARD, DDP_C, H, W, 700 + rank)


def _mask_and_dice_target(target, ignore_label):
    mask = target != ignore_label
    return mask, torch.where(mask, target, 0)


def _ce(logits, target, ignore_label, mask):
    if not mask.sum() > 0:                         # the reference skips the CE (compound_losses.py:52-53)
        return logits.new_zeros(())
    return F.cross_entropy(logits, target[:, 0].long(), ignore_index=ignore_label)


def dc_and_ce_loss(logits, target, ignore_label, batch_dice=True, do_bg=False, smooth=1e-5, weight_ce=1, weight_dice=1):
    """DC_and_CE_loss with ignore_label as the trainer builds it (MemoryEfficientSoftDiceLoss, ddp off).
    target [B, 1, ...] labels (any numeric dtype) -> (loss, ce, dice term)"""
    mask, target_dice = _mask_and_dice_target(target, ignore_label)
    dc = _dice_from_sums(*_dice_sums(torch.softmax(logits, 1), target_dice, mask, do_bg=do_bg), batch_dice, smooth)
    ce = _ce(logits, target, ignore_label, mask)
    return weight_ce * ce + weight_dice * dc, ce, dc


def validation_counts(logits, target, ignore_label):
    """nnUNetTrainer.py:977-994 for label maps with an ignore label: tp, fp, fn of the argmax one-hot per class
    (background included), each pixel weighted by target != ignore_label."""
    axes = [0] + list(range(2, logits.ndim))
    pred = torch.zeros(logits.shape, device=logits.device, dtype=torch.float32)
    pred.scatter_(1, logits.argmax(1)[:, None], 1)
    mask = (target != ignore_label).float()
    target = target.clone()
    target[target == ignore_label] = 0
    onehot = torch.zeros(logits.shape, device=logits.device)
    onehot.scatter_(1, target.long(), 1)
    mask_here = torch.tile(mask, (1, pred.shape[1], *[1 for _ in range(2, pred.ndim)]))
    tp = pred * onehot * mask_here
    fp = pred * (1 - onehot) * mask_here
    fn = (1 - pred) * onehot * mask_here
    return tp.sum(dim=axes), fp.sum(dim=axes), fn.sum(dim=axes)


def ddp_losses(logits, targets, ignore_label, do_bg=False, smooth=1e-5, weight_ce=1, weight_dice=1):
    """Per-rank losses of W data-parallel ranks simulated in one process, batch_dice and ddp on (as
    region_loss_oracle.ddp_losses): the masked Dice sums of every rank go through one shared stacked tensor, so that
    backward of sum_r(scale_r * loss_r) hands each rank the sum of the incoming gradients; the CE and its valid-pixel
    count stay local."""
    sums, ces = [], []
    for z, t in zip(logits, targets):
        mask, target_dice = _mask_and_dice_target(t, ignore_label)
        sums.append(_dice_sums(torch.softmax(z, 1), target_dice, mask, do_bg=do_bg))
        ces.append(_ce(z, t, ignore_label, mask))
    gathered = [torch.stack([s[k] for s in sums], dim=0) for k in range(3)]
    losses = []
    for ce in ces:
        intersect, sum_pred, sum_gt = (g.sum(0) for g in gathered)
        dc = _dice_from_sums(intersect, sum_pred, sum_gt, True, smooth)
        losses.append(weight_ce * ce + weight_dice * dc)
    return losses
