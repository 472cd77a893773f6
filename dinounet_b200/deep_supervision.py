"""Deep supervision on the native path: the scales, the loss weights and the downsampled targets of nnU-Net's default
training regime (nnUNetTrainer.py:300-306 `_get_deep_supervision_scales`, :370-390 `_build_loss`, :770-772 / :799-801
`DownsampleSegForDSTransform2`).

The network side lives in `DinoUNet.forward` (the list of decoder-head logits) and the loss side in
`loss.DeepSupervisionWrapper`; this module holds what the trainer derives from the plans and the device kernel that
downsamples a target batch (b2u_ds_targets, csrc/deep_supervision.cu).
"""
from typing import List, Sequence

import numpy as np
import torch

from . import lib as L

#: the decoder's three heads, highest resolution first: what the native network returns with deep supervision
NUM_OUTPUTS = 3


def deep_supervision_scales(pool_op_kernel_sizes) -> List[List[float]]:
    """`1 / cumprod(pool_op_kernel_sizes)[:-1]` per axis (nnUNetTrainer.py:300-306).  NotImplementedError unless there
    is one scale per decoder head, each an integer division of the patch per axis: what the native network and the
    target kernel produce."""
    scales = [list(map(float, s)) for s in 1 / np.cumprod(np.vstack(pool_op_kernel_sizes), axis=0)][:-1]
    if len(scales) != NUM_OUTPUTS:
        raise NotImplementedError(f"deep supervision on the native path has {NUM_OUTPUTS} outputs; the plan's "
                                  f"pool_op_kernel_sizes {pool_op_kernel_sizes} give {len(scales)} scales")
    for i, s in enumerate(scales):
        want = 1.0 / (2 ** i)
        if any(abs(v - want) > 1e-12 for v in s):
            raise NotImplementedError(f"deep supervision scale {i} is {s}; the native network's head {i} is at "
                                      f"1/{2 ** i} per axis")
    return scales


def deep_supervision_weights(n: int, ddp: bool) -> np.ndarray:
    """nnUNetTrainer.py:376-388: 1/2^i, the last set to 0 (1e-6 under DDP, whose unused-parameter check the reference
    avoids so), normalised to sum 1.  Without DDP and n = 3: [2/3, 1/3, 0]."""
    w = np.array([1 / (2 ** i) for i in range(n)])
    w[-1] = 1e-6 if ddp else 0
    return w / w.sum()


_DTYPES = {torch.int16: L.DS_INT16, torch.float32: L.DS_FP32}


def downsample_targets(target: torch.Tensor, scales: Sequence[Sequence[float]]) -> List[torch.Tensor]:
    """DownsampleSegForDSTransform2(scales, order=0) on a device batch: target [B, C, H, W] (int16 label maps, or
    float32 label maps / region channels + ignore channel) -> one tensor per scale, [B, C, round(H*sy), round(W*sx)] of
    the target's dtype.  Scale 1 is the input itself (no copy); every other scale comes from one b2u_ds_targets
    launch.  Only scales whose inverse is an integer dividing the extent are taken; others raise before any launch."""
    if not target.is_cuda:
        raise L.NativeLibraryError("dinounet_b200 downsamples deep-supervision targets on CUDA tensors only")
    if target.ndim != 4:
        raise ValueError(f"target must be [B, C, H, W], got {tuple(target.shape)}")
    if target.dtype not in _DTYPES:
        raise ValueError(f"target dtype {target.dtype}: the target kernel takes int16 or float32")
    B, Cc, H, W = target.shape
    src = target.contiguous()
    outs: List[torch.Tensor] = []
    p = L.DsTargetsParams()
    p.src, p.dtype, p.B, p.C, p.H, p.W = src.data_ptr(), _DTYPES[src.dtype], B, Cc, H, W
    n = 0
    for s in scales:
        if len(s) != 2:
            raise ValueError(f"scale {s}: two axes expected")
        if all(v == 1 for v in s):
            outs.append(target)
            continue
        fy, fx = (int(round(1 / v)) if v > 0 else 0 for v in s)
        if fy < 1 or fx < 1 or abs(fy * s[0] - 1) > 1e-9 or abs(fx * s[1] - 1) > 1e-9 or H % fy or W % fx:
            raise NotImplementedError(f"scale {list(s)} of a {H}x{W} target: the target kernel takes integer "
                                      "downsampling factors that divide the patch")
        if n == L.DS_MAX_SCALES:
            raise NotImplementedError(f"at most {L.DS_MAX_SCALES} downsampled scales per launch")
        out = torch.empty((B, Cc, H // fy, W // fx), dtype=src.dtype, device=src.device)
        p.fy[n], p.fx[n], p.dst[n] = fy, fx, out.data_ptr()
        n += 1
        outs.append(out)
    if n:
        p.nscales = n
        lib = L.load()
        with torch.cuda.device(src.device):
            L.check(lib.b2u_ds_targets(p, torch.cuda.current_stream(src.device).cuda_stream), "ds_targets")
    return outs
