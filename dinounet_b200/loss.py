"""Dice + cross-entropy / Dice + BCE losses and the online-validation statistics on the logits of the native forward path.

Mirror of the reference objects the trainer builds and calls (nnUNetTrainer.py:355-365, :961-1005):
`DC_and_CE_loss(soft_dice_kwargs, ce_kwargs, weight_ce, weight_dice, ignore_label, dice_class)` for label maps and
`DC_and_BCE_loss(bce_kwargs, soft_dice_kwargs, weight_ce, weight_dice, use_ignore_label, dice_class)` for region-based
datasets (sigmoid Dice over every region, optional ignore channel as the last target channel), with the same constructor
arguments and `forward(net_output, target)` (training/loss/compound_losses.py:9-99), and `validation_statistics` = what
`validation_step` derives from one batch ('loss', 'tp_hard', 'fp_hard', 'fn_hard').
One fused pass over the logits (csrc/loss.cu) instead of the reference's dozen full-tensor torch ops; the gradient with
respect to the logits comes from a second fused pass (autograd.Function).

Data-parallel batch Dice (`ddp=True`, `batch_dice=True`, default process group with more than one rank): the per-class
batch sums of intersect / sum_pred / sum_gt are summed across ranks with one all-reduce between the statistics pass and
the finalisation, as the reference's AllGatherGrad + sum does (dice.py:106-110).  Each rank's loss is its local CE/BCE
plus the global Dice term; in backward the Dice part of the gradient is scaled by the sum of the ranks' incoming
gradients (the AllGatherGrad backward, ddp_allgather.py:43-48).  Both happen on the current stream, without a host sync.

Ignore label of the softmax loss (`DC_and_CE_loss(..., ignore_label=N)`, sparsely annotated label maps): pixels labelled N
add nothing to the Dice sums, the CE (mean over the valid pixels of the local batch, 0 when there are none, as the
reference skips it) or the validation counts, and their gradient is exactly 0.  It runs the same entry points with the
kernels' ignore-label variant, with the same data-parallel batch Dice; the CE weight 1 / #valid stays on the device.

Not covered (raise): an ignore label with `do_bg=True`.  The ignore-label loss covers the configuration the reference
trainer builds for label maps (Dice without the background class, nnUNetTrainer.py:363-365), as the region loss covers
only its trainer configuration (do_bg=True).
"""
from typing import Dict

import numpy as np
import torch
from torch import nn
from torch.autograd import Function

from . import lib as L

_KIND = {torch.uint8: 0, torch.int32: 1, torch.int64: 2, torch.float32: 3}


def _prep(logits: torch.Tensor, target: torch.Tensor):
    if not logits.is_cuda:
        raise L.NativeLibraryError("dinounet_b200 losses run on CUDA tensors only (no CPU fallback)")
    if logits.ndim < 3:
        raise ValueError("net_output must be [B, C, spatial...]")
    B, C = logits.shape[:2]
    plane = int(np.prod(logits.shape[2:]))
    if target.ndim == logits.ndim:
        assert target.shape[1] == 1, "target must be b, c, x, y(, z) with c=1"
    if target.numel() != B * plane:
        raise ValueError(f"target has {target.numel()} labels for {B * plane} pixels")
    if target.dtype not in _KIND:
        target = target.float()
    return logits.float().contiguous(), target.contiguous(), B, C, plane


def _ddp_batch_dice(batch_dice: bool, ddp: bool) -> bool:
    """True when the batch Dice sums are summed across ranks (dice.py:106: batch_dice and ddp, under DDP)."""
    dist = torch.distributed
    return bool(batch_dice and ddp and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1)


def _grad_scales(g: torch.Tensor, all_reduce: bool):
    """Device scalars (local incoming gradient, Dice-part gradient scale = the incoming gradients summed over ranks)."""
    local = g.detach().reshape(1).float().clone()
    if not all_reduce:
        return local, local
    total = local.clone()
    torch.distributed.all_reduce(total)
    return local, total


def _prep_regions(logits: torch.Tensor, target: torch.Tensor, has_ignore: bool):
    if not logits.is_cuda:
        raise L.NativeLibraryError("dinounet_b200 losses run on CUDA tensors only (no CPU fallback)")
    if logits.ndim < 3:
        raise ValueError("net_output must be [B, R, spatial...]")
    B, R = logits.shape[:2]
    if not 1 <= R <= 32:
        raise ValueError(f"{R} regions: the fused region loss covers 1 to 32")
    plane = int(np.prod(logits.shape[2:]))
    want = (B, R + int(has_ignore), *logits.shape[2:])
    if tuple(target.shape) != want:
        raise ValueError(f"target shape {tuple(target.shape)} != {want} (regions{' + ignore channel' if has_ignore else ''})")
    if target.dtype not in _KIND:
        target = target.float()
    return logits.float().contiguous(), target.contiguous(), B, R, plane


def _ptr(x):
    return None if x is None else x.data_ptr()   # None: NULL


class _LabelMaps:
    """Softmax Dice + CE on label maps (b2u_dice_ce_*), with or without an ignore label."""
    name, counts_dtype, has_bad_label = "dice_ce", torch.int64, True

    def __init__(self, m: "DC_and_CE_loss"):
        self.all_reduce = _ddp_batch_dice(m.batch_dice, m.ddp)
        self.ign = int(m.ignore_label is not None)
        self.label = m.ignore_label if self.ign else 0
        self.batch_sums = self.all_reduce   # else NULL: finalize and backward sum the per-sample records in work
        self.cfg = (float(m.weight_ce), float(m.weight_dice), int(m.batch_dice), int(m.do_bg), float(m.smooth))
        # without an ignore label or an all-reduce the kernel runs unscaled and the incoming gradient is applied in torch
        self.device_scales = bool(self.ign or self.all_reduce)

    def prep(self, logits, target):
        return _prep(logits, target)

    def work_doubles(self, B, C, plane):
        return L.load().b2u_dice_ce_work_doubles(B, C, plane, self.ign)

    def stats(self, z, t, work, bsum, bad, B, C, plane, s):
        return L.load().b2u_dice_ce_stats(z.data_ptr(), t.data_ptr(), _KIND[t.dtype], self.ign, self.label,
                                          work.data_ptr(), _ptr(bsum), bad.data_ptr(), B, C, plane, s)

    def finalize(self, work, bsum, out3, counts, B, C, plane, s):
        return L.load().b2u_dice_ce_finalize(work.data_ptr(), _ptr(bsum), out3.data_ptr(), counts.data_ptr(), B, C,
                                             plane, self.ign, *self.cfg, s)

    def backward(self, z, t, work, bsum, grad, ce_scale, dice_scale, B, C, plane, s):
        return L.load().b2u_dice_ce_backward(z.data_ptr(), t.data_ptr(), _KIND[t.dtype], self.ign, self.label,
                                             work.data_ptr(), _ptr(bsum), grad.data_ptr(), B, C, plane, *self.cfg,
                                             _ptr(ce_scale), _ptr(dice_scale), s)


class _Regions:
    """Sigmoid Dice + BCE on region targets (b2u_dice_bce_*), with or without an ignore channel."""
    name, counts_dtype, has_bad_label, device_scales = "dice_bce", torch.float32, False, True
    batch_sums = True                       # the region kernels take the batch Dice from the batch sums only

    def __init__(self, m: "DC_and_BCE_loss"):
        self.all_reduce = _ddp_batch_dice(m.batch_dice, m.ddp)
        self.ign = int(m.use_ignore_label)
        self.w = (float(m.weight_ce), float(m.weight_dice), int(m.batch_dice))
        self.smooth = float(m.smooth)

    def prep(self, logits, target):
        return _prep_regions(logits, target, self.ign)

    def work_doubles(self, B, R, plane):
        return L.load().b2u_dice_bce_work_doubles(B, R, plane)

    def stats(self, z, t, work, bsum, bad, B, R, plane, s):
        return L.load().b2u_dice_bce_stats(z.data_ptr(), t.data_ptr(), _KIND[t.dtype], self.ign, work.data_ptr(),
                                           _ptr(bsum), B, R, plane, s)

    def finalize(self, work, bsum, out3, counts, B, R, plane, s):
        return L.load().b2u_dice_bce_finalize(work.data_ptr(), _ptr(bsum), out3.data_ptr(), counts.data_ptr(), B, R,
                                              plane, *self.w, self.ign, self.smooth, s)

    def backward(self, z, t, work, bsum, grad, ce_scale, dice_scale, B, R, plane, s):
        return L.load().b2u_dice_bce_backward(z.data_ptr(), t.data_ptr(), _KIND[t.dtype], self.ign, work.data_ptr(),
                                              _ptr(bsum), grad.data_ptr(), B, R, plane, *self.w, self.smooth,
                                              _ptr(ce_scale), _ptr(dice_scale), s)


class _FusedLoss(Function):
    """Statistics pass, all-reduce of the batch Dice sums across ranks (`fam.all_reduce`), finalisation; the gradient
    pass in backward.  `fam` (_LabelMaps, _Regions) binds its family's entry points to the loss's configuration."""

    @staticmethod
    def forward(ctx, logits, target, fam):
        z, t, B, n, plane = fam.prep(logits, target)
        dev = z.device
        work = torch.empty(int(fam.work_doubles(B, n, plane)), dtype=torch.float64, device=dev)
        bsum = torch.empty((n, 3), dtype=torch.float64, device=dev) if fam.batch_sums else None
        out3 = torch.empty(3, dtype=torch.float32, device=dev)
        counts = torch.empty((3, n), dtype=fam.counts_dtype, device=dev)
        bad = torch.zeros(1, dtype=torch.int32, device=dev) if fam.has_bad_label else None
        with torch.cuda.device(dev):
            s = torch.cuda.current_stream(dev).cuda_stream
            L.check(fam.stats(z, t, work, bsum, bad, B, n, plane, s), fam.name + "_stats")
            if fam.all_reduce:
                torch.distributed.all_reduce(bsum)
            L.check(fam.finalize(work, bsum, out3, counts, B, n, plane, s), fam.name + "_finalize")
        ctx.save_for_backward(z, t, work, bsum)
        ctx.fam, ctx.dims = fam, (B, n, plane)
        ctx.in_dtype, ctx.in_shape = logits.dtype, logits.shape
        ctx.mark_non_differentiable(*(x for x in (out3, counts, bad) if x is not None))
        return out3[0].clone(), out3, counts, bad

    @staticmethod
    def backward(ctx, g, *_unused):
        z, t, work, bsum = ctx.saved_tensors
        fam = ctx.fam
        scales = _grad_scales(g, fam.all_reduce) if fam.device_scales else (None, None)
        grad = torch.empty_like(z)
        with torch.cuda.device(z.device):
            L.check(fam.backward(z, t, work, bsum, grad, *scales, *ctx.dims,
                                 torch.cuda.current_stream(z.device).cuda_stream), fam.name + "_backward")
        if not fam.device_scales:
            grad = grad * g
        return grad.view(ctx.in_shape).to(ctx.in_dtype), None, None


class DC_and_CE_loss(nn.Module):
    def __init__(self, soft_dice_kwargs: dict, ce_kwargs: dict, weight_ce=1, weight_dice=1, ignore_label=None,
                 dice_class=None):
        super().__init__()
        if ignore_label is not None:
            if int(ignore_label) != ignore_label or not -2 ** 31 <= int(ignore_label) < 2 ** 31:
                raise ValueError(f"ignore_label must be a 32-bit integer, got {ignore_label!r}")
            ignore_label = int(ignore_label)
        if ce_kwargs:
            raise NotImplementedError(f"cross-entropy options {sorted(ce_kwargs)} are not covered by the fused native loss")
        kw = dict(soft_dice_kwargs)
        self.batch_dice = bool(kw.pop("batch_dice", False))
        self.do_bg = bool(kw.pop("do_bg", True))
        self.smooth = float(kw.pop("smooth", 1.))
        self.ddp = bool(kw.pop("ddp", True))
        kw.pop("apply_nonlin", None)
        if kw:
            raise NotImplementedError(f"soft dice options {sorted(kw)} are not covered by the fused native loss")
        if ignore_label is not None and self.do_bg:
            raise NotImplementedError("ignore_label with do_bg=True is not covered by the fused native loss (the "
                                      "trainer's label-map loss, do_bg=False, is)")
        self.weight_dice = weight_dice
        self.weight_ce = weight_ce
        self.ignore_label = ignore_label
        # True: synchronise and raise on labels outside [0, C) other than ignore_label (torch device-asserts)
        self.check_labels = False

    def _run(self, net_output, target):
        loss, out3, counts, bad = _FusedLoss.apply(net_output, target, _LabelMaps(self))
        if self.check_labels and int(bad.item()):
            raise RuntimeError("target contains labels outside [0, num_classes)")
        return loss, out3, counts, bad

    def forward(self, net_output: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        return self._run(net_output, target)[0]


class DC_and_BCE_loss(nn.Module):
    """Region-based Dice + BCE (compound_losses.py:59-99): sigmoid Dice over every region (do_bg) plus BCE with logits.
    `target` is [B, R, ...] with real values (the regions' one-hot encoding), plus a last ignore channel when
    `use_ignore_label`: a pixel counts where (1 - t_ign) != 0, and the masked BCE is sum(bce * mask) / #valid pixels."""

    def __init__(self, bce_kwargs: dict, soft_dice_kwargs: dict, weight_ce=1, weight_dice=1,
                 use_ignore_label: bool = False, dice_class=None):
        super().__init__()
        if bce_kwargs:
            raise NotImplementedError(f"BCE options {sorted(bce_kwargs)} are not covered by the fused native loss")
        kw = dict(soft_dice_kwargs)            # MemoryEfficientSoftDiceLoss defaults (dice.py:60-61)
        self.batch_dice = bool(kw.pop("batch_dice", False))
        self.do_bg = bool(kw.pop("do_bg", True))
        self.smooth = float(kw.pop("smooth", 1.))
        self.ddp = bool(kw.pop("ddp", True))
        if not self.do_bg:
            raise NotImplementedError("do_bg=False is not covered by the fused region loss (every region is foreground)")
        if kw:
            raise NotImplementedError(f"soft dice options {sorted(kw)} are not covered by the fused native loss")
        self.weight_dice = weight_dice
        self.weight_ce = weight_ce
        self.use_ignore_label = bool(use_ignore_label)

    def _run(self, net_output, target):
        return _FusedLoss.apply(net_output, target, _Regions(self))

    def forward(self, net_output: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        return self._run(net_output, target)[0]


class DeepSupervisionWrapper(nn.Module):
    """training/loss/deep_supervision.py: `loss` applied to every (output, target) pair of the lists it is given,
    weighted by `weight_factors` (all 1 when None); a pair whose weight is 0 is not evaluated, so the head that produced
    it gets no gradient.  Wraps the fused losses above (one fused pass per scale)."""

    def __init__(self, loss, weight_factors=None):
        super().__init__()
        if weight_factors is not None:
            assert any(x != 0 for x in weight_factors), "At least one weight factor should be != 0.0"
            weight_factors = tuple(float(x) for x in weight_factors)
        self.weight_factors = weight_factors
        self.loss = loss

    def _weights(self, n):
        return (1.0,) * n if self.weight_factors is None else self.weight_factors

    def forward(self, *args):
        assert all(isinstance(i, (tuple, list)) for i in args), \
            f"all args must be either tuple or list, got {[type(i) for i in args]}"
        w = self._weights(len(args[0]))
        return sum(w[i] * self.loss(*inputs) for i, inputs in enumerate(zip(*args)) if w[i] != 0.0)

    def _run(self, net_output, target):
        """(weighted loss over every scale, and scale 0's out3 / counts / bad): what `validation_statistics` reads."""
        w = self._weights(len(net_output))
        loss, first = None, None
        for i, (o, t) in enumerate(zip(net_output, target)):
            if w[i] == 0.0 and i > 0:
                continue
            r = self.loss._run(o, t)
            if i == 0:
                first = r
            if w[i] != 0.0:
                loss = w[i] * r[0] if loss is None else loss + w[i] * r[0]
        return (loss, *first[1:])


def validation_statistics(loss_module, net_output: torch.Tensor, target: torch.Tensor) -> Dict[str, np.ndarray]:
    """What `nnUNetTrainer.validation_step` returns for one batch (nnUNetTrainer.py:961-1005): the loss and the hard
    tp / fp / fn, float32.  Label maps (`DC_and_CE_loss`): argmax(net_output) per foreground class (background dropped),
    over the pixels not labelled with the loss's ignore label.  Regions (`DC_and_BCE_loss`): sigmoid(net_output) > 0.5 per region, each pixel weighted by 1 - t_ign when the target
    carries an ignore channel.  Under data-parallel batch Dice the loss uses the all-reduced sums; the counts stay per
    rank (the trainer gathers them at the end of the epoch).  With a `DeepSupervisionWrapper`, `net_output` and `target`
    are lists: the loss is the weighted sum over the scales, the counts come from scale 0 (nnUNetTrainer.py:964-967)."""
    with torch.no_grad():
        loss, _, counts, bad = loss_module._run(net_output, target)
    counts = counts.cpu().numpy()          # synchronises
    if bad is not None and int(bad.item()):
        raise RuntimeError("target contains labels outside [0, num_classes)")
    f = counts.astype(np.float32)          # the reference sums float products
    base = loss_module.loss if isinstance(loss_module, DeepSupervisionWrapper) else loss_module
    if isinstance(base, DC_and_BCE_loss):
        return {"loss": loss.detach().cpu().numpy(), "tp_hard": f[0], "fp_hard": f[1], "fn_hard": f[2]}
    return {"loss": loss.detach().cpu().numpy(), "tp_hard": f[0, 1:], "fp_hard": f[1, 1:], "fn_hard": f[2, 1:]}
