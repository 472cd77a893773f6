"""TEST INFRASTRUCTURE ONLY — restatement of nnU-Net's deep-supervision targets and loss weights.

Targets: `DownsampleSegForDSTransform2(scales, order=0)` (nnUNetTrainer.py:770-772, :799-801) calls batchgenerators'
`resize_segmentation(seg, new_shape, order=0)` per sample and channel, new_shape = np.round(shape * scale).astype(int);
for order 0 that is `skimage.transform.resize(seg.astype(float), new_shape, 0, mode="edge", clip=True,
anti_aliasing=False).astype(seg.dtype)`.  Restated from scikit-image 0.19-0.24 `skimage/transform/_warps.py::resize`:
a float image is not rescaled (`convert_to_float` keeps float input), `factors = input_shape / output_shape`, and the
resampling is `ndi.zoom(image, 1 / factors, order=0, mode="nearest" (= "edge"), grid_mode=True)`.  With grid_mode, output
index o of an axis of n -> m samples reads input coordinate x = (o + 0.5) * (n / m) - 0.5, and the order-0 spline takes
floor(x + 0.5) clipped to [0, n - 1] (ndimage's ni_interpolation.c for even orders).  At a factor of 2 that is 2o + 1,
at 4 it is 4o + 2.  scikit-image is not a dependency here, so this is the statement the kernel is held to; `zoom_picks`
computes the same with scipy for a cross-check.

Weights: nnUNetTrainer.py:376-388.
"""
import numpy as np
import torch


def axis_picks(n: int, m: int) -> np.ndarray:
    """The input index each of m outputs of an axis of n samples reads (resize order 0, mode edge)."""
    x = (np.arange(m, dtype=np.float64) + 0.5) * (n / m) - 0.5
    return np.clip(np.floor(x + 0.5).astype(np.int64), 0, n - 1)


def resize_segmentation_order0(seg: np.ndarray, new_shape) -> np.ndarray:
    """resize_segmentation(seg, new_shape, order=0) of one 2-D plane."""
    iy = axis_picks(seg.shape[0], int(new_shape[0]))
    ix = axis_picks(seg.shape[1], int(new_shape[1]))
    return seg.astype(np.float64)[iy][:, ix].astype(seg.dtype)


def downsample_seg_for_ds(seg: np.ndarray, scales):
    """DownsampleSegForDSTransform2(scales, order=0) on a [B, C, H, W] batch: one array per scale; scale 1 (every axis)
    passes the input through."""
    out = []
    for s in scales:
        if all(v == 1 for v in s):
            out.append(seg)
            continue
        new_shape = np.round(np.array(seg.shape[2:]) * np.array(s)).astype(int)
        r = np.empty((*seg.shape[:2], *new_shape), dtype=seg.dtype)
        for b in range(seg.shape[0]):
            for c in range(seg.shape[1]):
                r[b, c] = resize_segmentation_order0(seg[b, c], new_shape)
        out.append(r)
    return out


def zoom_picks(n: int, m: int) -> np.ndarray:
    """The same picks from scipy.ndimage.zoom(order=0, mode="nearest", grid_mode=True) on an index ramp."""
    from scipy import ndimage
    return ndimage.zoom(np.arange(n, dtype=np.float64), m / n, order=0, mode="nearest", grid_mode=True).astype(np.int64)


def ds_weights(n: int, ddp: bool) -> np.ndarray:
    """nnUNetTrainer.py:376-388: 1/2^i, the last 0 (1e-6 under DDP without compile), normalised to sum 1."""
    w = np.array([1 / (2 ** i) for i in range(n)])
    w[-1] = 1e-6 if ddp else 0
    return w / w.sum()


def forward(P, model: str, x):
    """DinoUNet.forward with deep_supervision=True (dinounet_training.py:603-629) on the oracle restatement:
    [seg_layers[2](stage 2), seg_layers[1](stage 1), seg_layers[0](stage 0)], highest resolution first."""
    from . import dinounet_oracle as O
    collect = {}
    skips = O.encoder_forward(P, O.VARIANTS[model], x, False, None)
    logits = O.decoder_forward(P, skips, collect)
    return [logits] + [O._conv(collect[f"dec{s}"], P, f"decoder.seg_layers.{s}") for s in (1, 0)]


def loss_and_grads(sd, model: str, x, targets, loss_fn, weights):
    """(outputs, weighted loss, {key: grad or None}) of the deep-supervision objective sum_i w_i loss_fn(out_i, t_i) over
    the pairs with w_i != 0, through the oracle forward; a trainable tensor no term reaches has None."""
    from . import dinounet_oracle as O
    from . import grad_oracle as G
    num_classes = sd["decoder.seg_layers.2.weight"].shape[0]
    keys = G.trainable_keys(model, num_classes)
    P = {k: v.detach().clone() for k, v in sd.items()}
    leaves = {k: P[k].requires_grad_(True) for k in keys}
    P.update(O.expand_aliases(dict(leaves)))
    outs = forward(P, model, x)
    loss = sum(w * loss_fn(o, t) for o, t, w in zip(outs, targets, weights) if w != 0)
    grads = torch.autograd.grad(loss, [leaves[k] for k in keys], allow_unused=True)
    return [o.detach() for o in outs], loss.detach(), dict(zip(keys, grads))
