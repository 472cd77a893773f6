"""TEST INFRASTRUCTURE ONLY — torch restatement of the reference's TRAIN-MODE training step (nnUNetTrainer.py:889-890
`self.network.train()`, then train_step), fp32, with the random draws given instead of drawn:

  * all 10 SyncBatchNorm layers (SPM stem / conv2-4, dinov3_adapter.py:239-277; adapter norm1-4, :479-482) normalise with
    the batch mean and biased variance and update running_mean / running_var (unbiased) / num_batches_tracked;
  * DropPath(0.3) on each extractor's ConvFFN branch (dinov3_adapter.py:18-27, 148) with per-sample keep flags
    `drop_keep` [6, B] (rows: interactions.0..3.extractor, interactions.3.extra_extractors.0..1), kept samples scaled 1/0.7;
  * the frozen ViT's RoPE coordinates of block i multiplied by `rope_scales[i]` (rope_position_encoding.py:93-97, one
    draw per block: vision_transformer.py:271-272); everything else in the ViT is the eval forward, without gradient.

`world=W` restates SyncBatchNorm over W data-parallel ranks in one process (the batch split into W equal slices): the
per-rank sums of x, x^2 and the counts are added before the finalize, as torch's SyncBatchNorm all-reduces them.

Built from the eval oracle's pieces (oracle/dinounet_oracle.py, unchanged); only the functions whose train-mode
behaviour differs are restated here.  Pinned to the REAL reference's train mode by tests/golden/train_mode_cases.npz
(oracle/make_golden_train_mode.py).
"""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import torch
import torch.nn.functional as F

from . import dinounet_oracle as O
from . import grad_oracle as G
from . import loss_oracle as LO

Tensor = torch.Tensor
A = "encoder.dinov3_adapter."
BN_LAYERS = [A + "spm." + n for n in ("stem.1", "stem.4", "stem.7", "conv2.1", "conv3.1", "conv4.1")] + \
    [f"{A}norm{i}" for i in range(1, 5)]
EXTRACTORS = [f"{A}interactions.{i}.extractor." for i in range(4)] + \
    [f"{A}interactions.3.extra_extractors.{j}." for j in range(2)]
DROP_KEEP = 0.7


def rope_sincos_scaled(periods: Tensor, H: int, W: int, scale: Tensor) -> Tuple[Tensor, Tensor]:
    """rope_position_encoding.py:57-106 in train mode ('separate' coordinates, rescale factor `scale`), fp32."""
    dd = dict(device=periods.device, dtype=torch.float32)
    ch = torch.arange(0.5, H, **dd) / H
    cw = torch.arange(0.5, W, **dd) / W
    coords = torch.stack(torch.meshgrid(ch, cw, indexing="ij"), dim=-1).flatten(0, 1)
    coords = 2.0 * coords - 1.0
    coords = coords * scale.reshape(1).to(**dd)
    ang = 2 * math.pi * coords[:, :, None] / periods[None, None, :]
    ang = ang.flatten(1, 2).tile(2)
    return torch.sin(ang), torch.cos(ang)


def vit_taps(P: Dict[str, Tensor], v: O.VariantCfg, x: Tensor, rope_scales: Tensor):
    """O.vit_taps with block i's RoPE tables from coordinates scaled by rope_scales[i]."""
    Bk = A + "backbone."
    B = x.shape[0]
    D, nh = v.dim, v.heads
    t = O._conv(x, P, Bk + "patch_embed.proj", stride=16)
    h, w = t.shape[2], t.shape[3]
    t = t.flatten(2).transpose(1, 2)
    cls = P[Bk + "cls_token"] + 0 * P[Bk + "mask_token"]
    tok = torch.cat([cls.expand(B, -1, -1), P[Bk + "storage_tokens"].expand(B, -1, -1), t], dim=1)
    taps = []
    for i in range(v.depth):
        sin, cos = rope_sincos_scaled(P[Bk + "rope_embed.periods"], h, w, rope_scales[i])
        p = f"{Bk}blocks.{i}."
        y = O._ln(tok, P, p + "norm1", 1e-5)
        bias = P[p + "attn.qkv.bias"] * P[p + "attn.qkv.bias_mask"].to(P[p + "attn.qkv.bias"].dtype) if v.qkv_bias else None
        qkv = F.linear(y, P[p + "attn.qkv.weight"], bias)
        N = qkv.shape[1]
        q, k, val = torch.unbind(qkv.reshape(B, N, 3, nh, D // nh), 2)
        q, k, val = [z.transpose(1, 2) for z in (q, k, val)]
        q, k = O._rope(q, sin, cos), O._rope(k, sin, cos)
        a = F.scaled_dot_product_attention(q, k, val).transpose(1, 2).reshape(B, N, D)
        tok = tok + O._lin(a, P, p + "attn.proj") * P[p + "ls1.gamma"]
        y = O._ln(tok, P, p + "norm2", 1e-5)
        if v.ffn == "mlp":
            m = O._lin(F.gelu(O._lin(y, P, p + "mlp.fc1")), P, p + "mlp.fc2")
        else:
            m = O._lin(F.silu(O._lin(y, P, p + "mlp.w1")) * O._lin(y, P, p + "mlp.w2"), P, p + "mlp.w3")
        tok = tok + m * P[p + "ls2.gamma"]
        if i in v.taps:
            o = O._ln(tok, P, Bk + "norm", 1e-5)
            taps.append((o[:, O.N_PREFIX:], o[:, 0]))
    return taps, (h, w)


def bn_train(x: Tensor, P: Dict[str, Tensor], p: str, world: int = 1, momentum: float = 0.1, eps: float = 1e-5) -> Tensor:
    """SyncBatchNorm.forward in train mode on NCHW x (the global batch; `world` equal rank slices).  Updates P's running
    statistics and num_batches_tracked in place (they must not require grad)."""
    P[p + ".num_batches_tracked"].add_(1)
    if world == 1:              # one process: SyncBatchNorm.forward falls back to F.batch_norm (torch/nn/modules/batchnorm.py)
        return F.batch_norm(x, P[p + ".running_mean"], P[p + ".running_var"], P[p + ".weight"], P[p + ".bias"], True, momentum,
                            eps)
    dims = (0, 2, 3)
    parts = x.chunk(world, 0)
    n = sum(t.numel() // t.shape[1] for t in parts)
    s1 = sum(t.double().sum(dims) for t in parts)
    s2 = sum((t.double() * t.double()).sum(dims) for t in parts)
    mean = (s1 / n).float()
    var = (s2 / n - (s1 / n) ** 2).float()
    with torch.no_grad():
        # torch's running-statistic update: mean and unbiased variance, momentum-weighted (torch/nn/modules/batchnorm.py)
        xd = x.detach().double()
        m64 = xd.mean(dims)
        v64 = xd.var(dims, unbiased=False)
        rm, rv = P[p + ".running_mean"], P[p + ".running_var"]
        rm.copy_((momentum * m64 + (1 - momentum) * rm.double()).float())
        rv.copy_((momentum * v64 * n / (n - 1) + (1 - momentum) * rv.double()).float())
    shape = (1, -1, 1, 1)
    return (x - mean.view(shape)) / torch.sqrt(var.view(shape) + eps) * P[p + ".weight"].view(shape) + P[p + ".bias"].view(shape)


def spm(P, x, world):
    """SpatialPriorModule.forward (dinov3_adapter.py:279-302), train-mode BatchNorm."""
    S = A + "spm."
    bn = lambda t, p: F.relu(bn_train(t, P, S + p, world))
    c1 = bn(O._conv(x, P, S + "stem.0", 2, 1), "stem.1")
    c1 = bn(O._conv(c1, P, S + "stem.3", 1, 1), "stem.4")
    c1 = bn(O._conv(c1, P, S + "stem.6", 1, 1), "stem.7")
    c1 = F.max_pool2d(c1, 3, 2, 1)
    c2 = bn(O._conv(c1, P, S + "conv2.0", 2, 1), "conv2.1")
    c3 = bn(O._conv(c2, P, S + "conv3.0", 2, 1), "conv3.1")
    c4 = bn(O._conv(c3, P, S + "conv4.0", 2, 1), "conv4.1")
    c1, c2, c3, c4 = (O._conv(c, P, S + f"fc{i + 1}") for i, c in enumerate((c1, c2, c3, c4)))
    tm = lambda t: t.flatten(2).transpose(1, 2)
    return c1, tm(c2), tm(c3), tm(c4)


def extractor(P, p, c, ref, feat, hw_tok, H_c, W_c, keep: Tensor) -> Tensor:
    """Extractor.forward (dinov3_adapter.py:140-156) with DropPath on the ConvFFN branch (keep [B] 0/1)."""
    a = O.msda_module(P, p + "attn.", O._ln(c, P, p + "query_norm", 1e-6), ref, O._ln(feat, P, p + "feat_norm", 1e-6), hw_tok)
    c = c + a
    f = O.conv_ffn(P, p + "ffn.", O._ln(c, P, p + "ffn_norm", 1e-6), H_c, W_c)
    return c + f * (keep / DROP_KEEP).view(-1, 1, 1)


def adapter_forward(P, v, x, rope_scales, drop_keep, world) -> List[Tensor]:
    """DINOv3_Adapter.forward (dinov3_adapter.py:408-484) in train mode."""
    bs, _, h, w = x.shape
    ref = O.reference_points([(h // 8, w // 8), (h // 16, w // 16), (h // 32, w // 32)], x.device)
    c1, c2, c3, c4 = spm(P, x, world)
    le = P[A + "level_embed"]
    c2, c3, c4 = c2 + le[0], c3 + le[1], c4 + le[2]
    n2, n3 = c2.shape[1], c3.shape[1]
    c = torch.cat([c2, c3, c4], dim=1)
    H_c, W_c = h // 16, w // 16
    with torch.no_grad():
        taps, (Ht, Wt) = vit_taps(P, v, x, rope_scales)
    outs = []
    e = 0
    for i in range(4):
        xi, _cls = taps[i]
        for p in [f"{A}interactions.{i}.extractor."] + ([f"{A}interactions.3.extra_extractors.{j}." for j in range(2)] if i == 3 else []):
            c = extractor(P, p, c, ref, xi, (Ht, Wt), H_c, W_c, drop_keep[e])
            e += 1
        outs.append(xi.transpose(1, 2).reshape(bs, v.dim, Ht, Wt).contiguous())
    sp = lambda t, hh, ww: t.transpose(1, 2).reshape(bs, v.dim, hh, ww).contiguous()
    c2 = sp(c[:, :n2], H_c * 2, W_c * 2)
    c3 = sp(c[:, n2:n2 + n3], H_c, W_c)
    c4 = sp(c[:, n2 + n3:], H_c // 2, W_c // 2)
    c1 = F.conv_transpose2d(c2, P[A + "up.weight"], P[A + "up.bias"], stride=2) + c1
    sizes = [(4 * H_c, 4 * W_c), (2 * H_c, 2 * W_c), (H_c, W_c), (H_c // 2, W_c // 2)]
    xs = [F.interpolate(o, size=s, mode="bilinear", align_corners=False) for o, s in zip(outs, sizes)]
    cs = [c1 + xs[0], c2 + xs[1], c3 + xs[2], c4 + xs[3]]
    return [bn_train(ci, P, f"{A}norm{i + 1}", world) for i, ci in enumerate(cs)]


def forward(P, model: str, x: Tensor, rope_scales: Tensor, drop_keep: Tensor, world: int = 1) -> Tensor:
    """Train-mode logits of 3-channel x [B, 3, S, S]; updates P's BatchNorm running statistics in place."""
    v = O.VARIANTS[model]
    feats = adapter_forward(P, v, x, rope_scales, drop_keep, world)
    ys = O.fapm_forward(P, feats)
    skips = []
    for i, y in enumerate(ys):
        for _ in range(2):
            y = F.conv_transpose2d(y, P[f"encoder.ups.{i}.up2.weight"], P[f"encoder.ups.{i}.up2.bias"], stride=2)
        skips.append(y)
    return O.decoder_forward(P, skips)


def loss_and_grads(sd: Dict[str, Tensor], model: str, x: Tensor, target: Tensor, rope_scales: Tensor, drop_keep: Tensor,
                   world: int = 1, batch_dice: bool = True):
    """(loss, {trainable key: grad}, {BatchNorm buffer key: updated value}) of one train-mode step on a copy of sd.
    With world > 1 the loss is the mean of the W rank losses on equal batch slices (what DDP's gradient average
    differentiates); batch Dice is then taken per rank."""
    num_classes = sd["decoder.seg_layers.2.weight"].shape[0]
    keys = G.trainable_keys(model, num_classes)
    P = {k: t.detach().clone() for k, t in sd.items()}
    leaves = {k: P[k].requires_grad_(True) for k in keys}
    for k, t in O.expand_aliases(leaves).items():
        P[k] = t
    logits = forward(P, model, x, rope_scales, drop_keep, world)
    losses = [LO.dc_and_ce_loss(z, t, batch_dice=batch_dice)[0] for z, t in zip(logits.chunk(world, 0), target.chunk(world, 0))]
    loss = sum(losses) / world
    grads = torch.autograd.grad(loss, [leaves[k] for k in keys], allow_unused=True)
    bufs = {p + s: P[p + s].detach().clone() for p in BN_LAYERS for s in (".running_mean", ".running_var", ".num_batches_tracked")}
    return loss.detach(), {k: (g if g is not None else torch.zeros_like(leaves[k])) for k, g in zip(keys, grads)}, bufs
