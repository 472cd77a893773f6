"""Dice + cross-entropy loss and the online-validation statistics on the logits of the native forward path.

Mirror of the reference objects the trainer builds and calls (nnUNetTrainer.py:363-365, :961-1005):
`DC_and_CE_loss(soft_dice_kwargs, ce_kwargs, weight_ce, weight_dice, ignore_label, dice_class)` with the same
constructor arguments and `forward(net_output, target)` (training/loss/compound_losses.py:9-56), and
`validation_statistics` = what `validation_step` derives from one batch ('loss', 'tp_hard', 'fp_hard', 'fn_hard').
One fused pass over the logits (csrc/loss.cu) instead of the reference's dozen full-tensor torch ops; the gradient with
respect to the logits comes from a second fused pass (autograd.Function), ready for the round-2 backward.

Not covered (raise): ignore labels, region-based (sigmoid/BCE) training, DDP batch-dice all-gather.
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


class DC_and_CE_loss(nn.Module):
    def __init__(self, soft_dice_kwargs: dict, ce_kwargs: dict, weight_ce=1, weight_dice=1, ignore_label=None,
                 dice_class=None):
        super().__init__()
        if ignore_label is not None:
            raise NotImplementedError("ignore_label is not covered by the fused native loss")
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
        self.weight_dice = weight_dice
        self.weight_ce = weight_ce
        self.ignore_label = None
        self.check_labels = False     # True: synchronise and raise on labels outside [0, C) (torch device-asserts)

    def _run(self, net_output, target):
        if self.batch_dice and self.ddp and torch.distributed.is_available() and torch.distributed.is_initialized() \
                and torch.distributed.get_world_size() > 1:
            raise NotImplementedError("DDP batch-dice (all-gather of the dice sums) is not covered by the fused native loss")
        loss, out3, counts, bad = _DiceCE.apply(net_output, target, self.weight_ce, self.weight_dice, self.batch_dice,
                                                self.do_bg, self.smooth)
        if self.check_labels and int(bad.item()):
            raise RuntimeError("target contains labels outside [0, num_classes)")
        return loss, out3, counts, bad

    def forward(self, net_output: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        return self._run(net_output, target)[0]


def validation_statistics(loss_module: DC_and_CE_loss, net_output: torch.Tensor, target: torch.Tensor) -> Dict[str, np.ndarray]:
    """What `nnUNetTrainer.validation_step` returns for one batch (nnUNetTrainer.py:961-1005, no regions / ignore label):
    the loss and the hard per-foreground-class tp / fp / fn of argmax(net_output) against the target."""
    with torch.no_grad():
        loss, _, counts, bad = loss_module._run(net_output, target)
    counts = counts.cpu().numpy()          # synchronises
    if int(bad.item()):
        raise RuntimeError("target contains labels outside [0, num_classes)")
    f = counts.astype(np.float32)          # the reference sums float one-hot products
    return {"loss": loss.detach().cpu().numpy(), "tp_hard": f[0, 1:], "fp_hard": f[1, 1:], "fn_hard": f[2, 1:]}
