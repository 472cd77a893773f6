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
reference skips it) or the validation counts, and their gradient is exactly 0.  It runs the split entry points
(b2u_dice_ce_ign_*), with the same data-parallel batch Dice; the CE weight 1 / #valid stays on the device.

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


class _DiceCE(Function):
    @staticmethod
    def forward(ctx, logits, target, weight_ce, weight_dice, batch_dice, do_bg, smooth):
        z, t, B, C, plane = _prep(logits, target)
        lib = L.load()
        dev = z.device
        work = torch.empty(int(lib.b2u_dice_ce_work_doubles(B, C, plane)), dtype=torch.float64, device=dev)
        out3 = torch.empty(3, dtype=torch.float32, device=dev)
        counts = torch.empty((3, C), dtype=torch.int64, device=dev)
        bad = torch.zeros(1, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            L.check(lib.b2u_dice_ce_forward(z.data_ptr(), t.data_ptr(), _KIND[t.dtype], work.data_ptr(), out3.data_ptr(),
                                            counts.data_ptr(), bad.data_ptr(), B, C, plane, float(weight_ce),
                                            float(weight_dice), int(batch_dice), int(do_bg), float(smooth),
                                            torch.cuda.current_stream(dev).cuda_stream), "dice_ce_forward")
        ctx.save_for_backward(z, t, work)
        ctx.cfg = (B, C, plane, float(weight_ce), float(weight_dice), int(batch_dice), int(do_bg), float(smooth))
        ctx.in_dtype, ctx.in_shape = logits.dtype, logits.shape
        ctx.mark_non_differentiable(out3, counts, bad)
        return out3[0].clone(), out3, counts, bad

    @staticmethod
    def backward(ctx, g, *_unused):
        z, t, work = ctx.saved_tensors
        B, C, plane, wce, wdc, bd, bg, smooth = ctx.cfg
        grad = torch.empty_like(z)
        with torch.cuda.device(z.device):
            L.check(L.load().b2u_dice_ce_backward(z.data_ptr(), t.data_ptr(), _KIND[t.dtype], work.data_ptr(),
                                                  grad.data_ptr(), B, C, plane, wce, wdc, bd, bg, smooth, 1.0,
                                                  torch.cuda.current_stream(z.device).cuda_stream), "dice_ce_backward")
        grad = (grad * g).view(ctx.in_shape).to(ctx.in_dtype)
        return grad, None, None, None, None, None, None


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


class _DiceCEAllReduced(Function):
    """Dice + CE whose batch Dice sums are all-reduced across the data-parallel ranks."""

    @staticmethod
    def forward(ctx, logits, target, weight_ce, weight_dice, do_bg, smooth):
        z, t, B, C, plane = _prep(logits, target)
        lib = L.load()
        dev = z.device
        work = torch.empty(int(lib.b2u_dice_ce_work_doubles(B, C, plane)), dtype=torch.float64, device=dev)
        bsum = torch.empty((C, 3), dtype=torch.float64, device=dev)
        out3 = torch.empty(3, dtype=torch.float32, device=dev)
        counts = torch.empty((3, C), dtype=torch.int64, device=dev)
        bad = torch.zeros(1, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            L.check(lib.b2u_dice_ce_stats(z.data_ptr(), t.data_ptr(), _KIND[t.dtype], work.data_ptr(), bsum.data_ptr(),
                                          bad.data_ptr(), B, C, plane, torch.cuda.current_stream(dev).cuda_stream),
                    "dice_ce_stats")
            torch.distributed.all_reduce(bsum)
            L.check(lib.b2u_dice_ce_finalize(work.data_ptr(), bsum.data_ptr(), out3.data_ptr(), counts.data_ptr(), B, C,
                                             plane, float(weight_ce), float(weight_dice), 1, int(do_bg), float(smooth),
                                             torch.cuda.current_stream(dev).cuda_stream), "dice_ce_finalize")
        ctx.save_for_backward(z, t, work, bsum)
        ctx.cfg = (B, C, plane, float(weight_ce), float(weight_dice), int(do_bg), float(smooth))
        ctx.in_dtype, ctx.in_shape = logits.dtype, logits.shape
        ctx.mark_non_differentiable(out3, counts, bad)
        return out3[0].clone(), out3, counts, bad

    @staticmethod
    def backward(ctx, g, *_unused):
        z, t, work, bsum = ctx.saved_tensors
        B, C, plane, wce, wdc, bg, smooth = ctx.cfg
        local, total = _grad_scales(g, all_reduce=True)
        grad = torch.empty_like(z)
        with torch.cuda.device(z.device):
            L.check(L.load().b2u_dice_ce_backward_scaled(z.data_ptr(), t.data_ptr(), _KIND[t.dtype], work.data_ptr(),
                                                         bsum.data_ptr(), grad.data_ptr(), B, C, plane, wce, wdc, 1, bg,
                                                         smooth, local.data_ptr(), total.data_ptr(),
                                                         torch.cuda.current_stream(z.device).cuda_stream),
                    "dice_ce_backward_scaled")
        return grad.view(ctx.in_shape).to(ctx.in_dtype), None, None, None, None, None


class _DiceCEIgnore(Function):
    """Dice + CE over the pixels whose label is not `ignore_label` (compound_losses.py:38-53); the batch Dice sums are
    all-reduced across the data-parallel ranks when `all_reduce`."""

    @staticmethod
    def forward(ctx, logits, target, ignore_label, weight_ce, weight_dice, batch_dice, do_bg, smooth, all_reduce):
        z, t, B, C, plane = _prep(logits, target)
        lib = L.load()
        dev = z.device
        work = torch.empty(int(lib.b2u_dice_ce_ign_work_doubles(B, C, plane)), dtype=torch.float64, device=dev)
        bsum = torch.empty((C, 3), dtype=torch.float64, device=dev)
        out3 = torch.empty(3, dtype=torch.float32, device=dev)
        counts = torch.empty((3, C), dtype=torch.int64, device=dev)
        bad = torch.zeros(1, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            L.check(lib.b2u_dice_ce_ign_stats(z.data_ptr(), t.data_ptr(), _KIND[t.dtype], ignore_label, work.data_ptr(),
                                              bsum.data_ptr(), bad.data_ptr(), B, C, plane,
                                              torch.cuda.current_stream(dev).cuda_stream), "dice_ce_ign_stats")
            if all_reduce:
                torch.distributed.all_reduce(bsum)
            L.check(lib.b2u_dice_ce_ign_finalize(work.data_ptr(), bsum.data_ptr(), out3.data_ptr(), counts.data_ptr(), B,
                                                 C, plane, float(weight_ce), float(weight_dice), int(batch_dice),
                                                 int(do_bg), float(smooth), torch.cuda.current_stream(dev).cuda_stream),
                    "dice_ce_ign_finalize")
        ctx.save_for_backward(z, t, work, bsum)
        ctx.cfg = (ignore_label, B, C, plane, float(weight_ce), float(weight_dice), int(batch_dice), int(do_bg),
                   float(smooth), bool(all_reduce))
        ctx.in_dtype, ctx.in_shape = logits.dtype, logits.shape
        ctx.mark_non_differentiable(out3, counts, bad)
        return out3[0].clone(), out3, counts, bad

    @staticmethod
    def backward(ctx, g, *_unused):
        z, t, work, bsum = ctx.saved_tensors
        ign, B, C, plane, wce, wdc, bd, bg, smooth, all_reduce = ctx.cfg
        local, total = _grad_scales(g, all_reduce)
        grad = torch.empty_like(z)
        with torch.cuda.device(z.device):
            L.check(L.load().b2u_dice_ce_ign_backward(z.data_ptr(), t.data_ptr(), _KIND[t.dtype], ign, work.data_ptr(),
                                                      bsum.data_ptr(), grad.data_ptr(), B, C, plane, wce, wdc, bd, bg,
                                                      smooth, local.data_ptr(), total.data_ptr(),
                                                      torch.cuda.current_stream(z.device).cuda_stream),
                    "dice_ce_ign_backward")
        return grad.view(ctx.in_shape).to(ctx.in_dtype), None, None, None, None, None, None, None, None


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


class _DiceBCE(Function):
    @staticmethod
    def forward(ctx, logits, target, weight_ce, weight_dice, batch_dice, has_ignore, smooth, all_reduce):
        z, t, B, R, plane = _prep_regions(logits, target, has_ignore)
        lib = L.load()
        dev = z.device
        work = torch.empty(int(lib.b2u_dice_bce_work_doubles(B, R, plane)), dtype=torch.float64, device=dev)
        bsum = torch.empty((R, 3), dtype=torch.float64, device=dev)
        out3 = torch.empty(3, dtype=torch.float32, device=dev)
        counts = torch.empty((3, R), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            L.check(lib.b2u_dice_bce_stats(z.data_ptr(), t.data_ptr(), _KIND[t.dtype], int(has_ignore), work.data_ptr(),
                                           bsum.data_ptr(), B, R, plane, torch.cuda.current_stream(dev).cuda_stream),
                    "dice_bce_stats")
            if all_reduce:
                torch.distributed.all_reduce(bsum)
            L.check(lib.b2u_dice_bce_finalize(work.data_ptr(), bsum.data_ptr(), out3.data_ptr(), counts.data_ptr(), B, R,
                                              plane, float(weight_ce), float(weight_dice), int(batch_dice),
                                              int(has_ignore), float(smooth), torch.cuda.current_stream(dev).cuda_stream),
                    "dice_bce_finalize")
        ctx.save_for_backward(z, t, work, bsum)
        ctx.cfg = (B, R, plane, float(weight_ce), float(weight_dice), int(batch_dice), int(has_ignore), float(smooth),
                   bool(all_reduce))
        ctx.in_dtype, ctx.in_shape = logits.dtype, logits.shape
        ctx.mark_non_differentiable(out3, counts)
        return out3[0].clone(), out3, counts

    @staticmethod
    def backward(ctx, g, *_unused):
        z, t, work, bsum = ctx.saved_tensors
        B, R, plane, wce, wdc, bd, ign, smooth, all_reduce = ctx.cfg
        local, total = _grad_scales(g, all_reduce)
        grad = torch.empty_like(z)
        with torch.cuda.device(z.device):
            L.check(L.load().b2u_dice_bce_backward(z.data_ptr(), t.data_ptr(), _KIND[t.dtype], ign, work.data_ptr(),
                                                   bsum.data_ptr(), grad.data_ptr(), B, R, plane, wce, wdc, bd, smooth,
                                                   local.data_ptr(), total.data_ptr(),
                                                   torch.cuda.current_stream(z.device).cuda_stream), "dice_bce_backward")
        return grad.view(ctx.in_shape).to(ctx.in_dtype), None, None, None, None, None, None, None


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
        if self.ignore_label is not None:
            loss, out3, counts, bad = _DiceCEIgnore.apply(net_output, target, self.ignore_label, self.weight_ce,
                                                          self.weight_dice, self.batch_dice, self.do_bg, self.smooth,
                                                          _ddp_batch_dice(self.batch_dice, self.ddp))
        elif _ddp_batch_dice(self.batch_dice, self.ddp):
            loss, out3, counts, bad = _DiceCEAllReduced.apply(net_output, target, self.weight_ce, self.weight_dice,
                                                              self.do_bg, self.smooth)
        else:
            loss, out3, counts, bad = _DiceCE.apply(net_output, target, self.weight_ce, self.weight_dice,
                                                    self.batch_dice, self.do_bg, self.smooth)
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
        loss, out3, counts = _DiceBCE.apply(net_output, target, self.weight_ce, self.weight_dice, self.batch_dice,
                                            self.use_ignore_label, self.smooth,
                                            _ddp_batch_dice(self.batch_dice, self.ddp))
        return loss, out3, counts, None

    def forward(self, net_output: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        return self._run(net_output, target)[0]


def validation_statistics(loss_module, net_output: torch.Tensor, target: torch.Tensor) -> Dict[str, np.ndarray]:
    """What `nnUNetTrainer.validation_step` returns for one batch (nnUNetTrainer.py:961-1005): the loss and the hard
    tp / fp / fn, float32.  Label maps (`DC_and_CE_loss`): argmax(net_output) per foreground class (background dropped),
    over the pixels not labelled with the loss's ignore label.  Regions (`DC_and_BCE_loss`): sigmoid(net_output) > 0.5 per region, each pixel weighted by 1 - t_ign when the target
    carries an ignore channel.  Under data-parallel batch Dice the loss uses the all-reduced sums; the counts stay per
    rank (the trainer gathers them at the end of the epoch)."""
    with torch.no_grad():
        loss, _, counts, bad = loss_module._run(net_output, target)
    counts = counts.cpu().numpy()          # synchronises
    if bad is not None and int(bad.item()):
        raise RuntimeError("target contains labels outside [0, num_classes)")
    f = counts.astype(np.float32)          # the reference sums float products
    if isinstance(loss_module, DC_and_BCE_loss):
        return {"loss": loss.detach().cpu().numpy(), "tp_hard": f[0], "fp_hard": f[1], "fn_hard": f[2]}
    return {"loss": loss.detach().cpu().numpy(), "tp_hard": f[0, 1:], "fp_hard": f[1, 1:], "fn_hard": f[2, 1:]}
