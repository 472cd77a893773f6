"""Training path: forward + backward of the TRAINABLE part of Dino U-Net (SURVEY.md section 8f rank 2, BASELINE.json config 3).

The reference's train step (`nnUNetTrainer.train_step`, nnUNetTrainer.py:899-929) runs the whole model under autograd;
the DINOv3 backbone is frozen and evaluated under `no_grad` (dinov3_adapter.py:326, 422-426), so gradients exist only
for SPM, the six extractors, `up`, the four adapter BatchNorms, FAPM, the learnable upsamplers, the decoder and the seg
head (289 tensors).  Here:

  * the frozen ViT runs on the 16-bit tensor-core engine (`ForwardEngine.extract_vit_features`) or, with
    `vit_precision="fp32"`, on the fp32 tier - no gradient flows into it;
  * every differentiable operator is a `torch.autograd.Function` whose forward AND backward call hand-written
    kernels through the C-ABI (csrc/gemm_tf32.cu, csrc/fp32_tier.cu, csrc/train_bwd.cu, msda.cu, loss.cu).  torch.autograd
    is used as the tape only: what it executes itself is data movement (views, cat, contiguous) and gradient accumulation
    for tensors with several consumers;
  * the matrix products (F.linear / Conv2d / ConvTranspose2d: forward, data gradient, weight gradient) have two tiers
    with ONE parameter block: `gemm="tf32"` (default) = `b2u_tf32_gemm`, wgmma tensor cores with TF32-rounded operands
    and fp32 accumulation (the mantissa of the fp16 autocast the reference trains under); `gemm="fp32"` = `b2u_f32_gemm`,
    the IEEE-fp32 SIMT kernel the gradient goldens are held to at 2e-3.  Everything else is fp32 in both tiers;
  * semantics (`DinoUNet.train_semantics`): "oracle" (default) = the gradient oracle's (oracle/grad_oracle.py, pinned to
    autograd through the REAL reference): eval-mode BatchNorm (running statistics), DropPath off, fp32.  "reference" = the
    reference's train mode (`TrainMode`): batch-statistics SyncBatchNorm with the running-statistic update, DropPath on the
    extractors' ConvFFN branch, and the ViT taps computed with per-block rescaled RoPE coordinates (engine.py).

Layout: activations are 2-D fp32 tensors [rows, C] (tokens, or NHWC pixels), exactly the fp32 tier's.
"""
from __future__ import annotations

import contextlib
import ctypes as C
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
from torch.autograd import Function
from torch.utils.checkpoint import checkpoint

from . import config as cfg
from . import lib as L


def _s(t: torch.Tensor) -> int:
    return torch.cuda.current_stream(t.device).cuda_stream


#: matrix-product tier of the Functions created from now on ("tf32" | "fp32"); `trainable_forward` sets it for the duration
#: of its forward and every Function remembers it for its backward
_GEMM_TIER = "tf32"


def _gemm(A, W, out, M, N, K, *, lda=None, ldw=None, ldc=None, bias=None, residual=None, conv=0, img=(0, 0, 0), cpad=0,
          ps=None, a_trans=0, w_mode=0, w_cpad=0, ksplit=0, col_off=0, tier=None):
    p = L.F32GemmParams()
    p.M, p.N, p.K = int(M), int(N), int(K)
    p.A, p.lda = A.data_ptr(), int(lda if lda is not None else A.shape[-1])
    p.W, p.ldw = W.data_ptr(), int(ldw if ldw is not None else W.shape[-1])
    p.conv = conv
    if conv:
        p.Hin, p.Win, p.C = [int(t) for t in img]
        p.Cpad = int(cpad)
    p.out, p.ldc, p.col_off = out.data_ptr(), int(ldc if ldc is not None else out.shape[-1]), int(col_off)
    if ps is not None:
        p.ps_cout, p.ps_h, p.ps_w = [int(t) for t in ps]
    p.bias = None if bias is None else bias.data_ptr()
    if residual is not None:
        p.residual, p.ldres = residual.data_ptr(), int(residual.shape[-1])
    p.a_trans, p.w_mode, p.w_cpad, p.ksplit = int(a_trans), int(w_mode), int(w_cpad), int(ksplit)
    fn = "b2u_tf32_gemm" if (tier or _GEMM_TIER) == "tf32" else "b2u_f32_gemm"
    with torch.cuda.device(out.device):
        L.check(getattr(L.load(), fn)(C.byref(p), C.c_void_p(_s(out))), fn)


def _ksplit(rows: int) -> int:
    return max(1, min(64, rows // 2048))


def _call(name, *args):
    dev = next(a for a in args if isinstance(a, torch.Tensor)).device
    raw = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    with torch.cuda.device(dev):
        L.check(getattr(L.load(), name)(*raw, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), name)


def _colsum(t: torch.Tensor, Cc: int) -> torch.Tensor:
    out = torch.zeros(Cc, dtype=torch.float32, device=t.device)
    _call("b2u_f32_colsum", t, t.shape[-1], t.numel() // t.shape[-1], Cc, out)
    return out


# ------------------------------------------------------------------------------------------------------------ Functions
class LinearF(Function):
    """y = x W^T + b (+ residual): F.linear / 1x1 conv.  x [M, K], W [N, K]."""

    @staticmethod
    def forward(ctx, x, W, b, residual):
        x, W = x.contiguous(), W.contiguous()
        M, K, N = x.shape[0], x.shape[1], W.shape[0]
        y = torch.empty((M, N), dtype=torch.float32, device=x.device)
        _gemm(x, W, y, M, N, K, bias=b, residual=residual)
        ctx.save_for_backward(x, W)
        ctx.has_b, ctx.has_r, ctx.tier = b is not None, residual is not None, _GEMM_TIER
        return y

    @staticmethod
    def backward(ctx, dy):
        x, W = ctx.saved_tensors
        dy = dy.contiguous()
        M, K, N = x.shape[0], x.shape[1], W.shape[0]
        dx = dW = db = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            _gemm(dy, W, dx, M, K, N, w_mode=1, tier=ctx.tier)        # dx[m,k] = sum_n dy[m,n] W[n,k]
        if ctx.needs_input_grad[1]:
            dW = torch.zeros_like(W)
            _gemm(dy, x, dW, N, K, M, a_trans=1, w_mode=1, ksplit=_ksplit(M), tier=ctx.tier)   # dW[n,k] = sum_m dy[m,n] x[m,k]
        if ctx.has_b and ctx.needs_input_grad[2]:
            db = _colsum(dy, N)
        return dx, dW, db, (dy if ctx.has_r else None)


class Conv3x3F(Function):
    """Conv2d(3x3, pad 1, stride s) + bias on NHWC rows.  x [B*H*W, C], W [N, C, 3, 3]."""

    @staticmethod
    def forward(ctx, x, W, b, B, H, Wd, stride):
        x = x.contiguous()
        N, Cc = W.shape[0], W.shape[1]
        Wp = W.permute(0, 2, 3, 1).reshape(N, 9 * Cc).contiguous()    # k = tap*C + c
        Ho, Wo = H // stride, Wd // stride
        y = torch.empty((B * Ho * Wo, N), dtype=torch.float32, device=x.device)
        _gemm(x, Wp, y, B * Ho * Wo, N, 9 * Cc, bias=b, conv=L.CONV3X3_S2 if stride == 2 else L.CONV3X3_S1, img=(H, Wd, Cc), cpad=Cc)
        ctx.save_for_backward(x, Wp)
        ctx.geo = (B, H, Wd, Cc, N, stride)
        ctx.has_b, ctx.tier = b is not None, _GEMM_TIER
        return y

    @staticmethod
    def backward(ctx, dy):
        x, Wp = ctx.saved_tensors
        B, H, Wd, Cc, N, stride = ctx.geo
        dy = dy.contiguous()
        Ho, Wo = H // stride, Wd // stride
        dx = dW = db = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            if stride == 1:   # correlation of dy with the flipped, transposed weights: the GEMM kernel's conv data-gradient mode
                _gemm(dy, Wp, dx, B * H * Wd, Cc, 9 * N, conv=L.CONV3X3_S1, img=(H, Wd, N), cpad=N, w_mode=2, w_cpad=Cc, ldw=9 * Cc,
                      tier=ctx.tier)
            else:
                _call("b2u_f32_conv3x3_dgrad", dy, Wp, dx, B, H, Wd, Cc, Cc, N, stride)
        if ctx.needs_input_grad[1]:
            # dWp[n, (tap, c)] = sum_pix dy[pix, n] * window(x)[pix, tap, c]: the GEMM with A' = dy^T and the window on the W side
            dWp = torch.zeros_like(Wp)
            npix = B * Ho * Wo
            _gemm(dy, x, dWp, N, 9 * Cc, npix, a_trans=1, lda=N, w_mode=3, conv=L.CONV3X3_S2 if stride == 2 else L.CONV3X3_S1,
                  img=(H, Wd, Cc), cpad=Cc, ksplit=max(1, min(256, npix // 4096)), tier=ctx.tier)
            dW = dWp.view(N, 3, 3, Cc).permute(0, 3, 1, 2).contiguous()
        if ctx.has_b and ctx.needs_input_grad[2]:
            db = _colsum(dy, N)
        return dx, dW, db, None, None, None, None


class ConvT2x2F(Function):
    """ConvTranspose2d(k 2, s 2) + bias: x [B*h*w, Cin], W [Cin, Cout, 2, 2] -> [B*2h*2w, Cout] (a GEMM + pixel shuffle)."""

    @staticmethod
    def forward(ctx, x, W, b, B, h, w):
        x = x.contiguous()
        Cin, Cout = W.shape[0], W.shape[1]
        Wp = W.permute(2, 3, 1, 0).reshape(4 * Cout, Cin).contiguous()
        y = torch.empty((B * 4 * h * w, Cout), dtype=torch.float32, device=x.device)
        _gemm(x, Wp, y, B * h * w, 4 * Cout, Cin, bias=b.repeat(4).contiguous(), ps=(Cout, h, w))
        ctx.save_for_backward(x, Wp)
        ctx.geo = (B, h, w, Cin, Cout)
        ctx.tier = _GEMM_TIER
        return y

    @staticmethod
    def backward(ctx, dy):
        x, Wp = ctx.saved_tensors
        B, h, w, Cin, Cout = ctx.geo
        dy = dy.contiguous()
        M = B * h * w
        dyu = torch.empty((M, 4 * Cout), dtype=torch.float32, device=dy.device)
        _call("b2u_f32_unshuffle", dy, Cout, 0, dyu, B, h, w, Cout)
        dx = dW = db = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            _gemm(dyu, Wp, dx, M, Cin, 4 * Cout, w_mode=1, tier=ctx.tier)
        if ctx.needs_input_grad[1]:
            dWp = torch.zeros_like(Wp)
            _gemm(dyu, x, dWp, 4 * Cout, Cin, M, a_trans=1, w_mode=1, ksplit=_ksplit(M), tier=ctx.tier)
            dW = dWp.view(2, 2, Cout, Cin).permute(3, 2, 0, 1).contiguous()
        if ctx.needs_input_grad[2]:
            db = _colsum(dy, Cout)
        return dx, dW, db, None, None, None


class LayerNormF(Function):
    @staticmethod
    def forward(ctx, x, g, b, eps):
        x = x.contiguous()
        rows, D = x.shape
        y = torch.empty_like(x)
        _call("b2u_f32_layernorm", x, y, g, b, rows, D, float(eps), 0, 0, 0)
        ctx.save_for_backward(x, g)
        ctx.eps = float(eps)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, g = ctx.saved_tensors
        dy = dy.contiguous()
        dx = torch.empty_like(x)
        dg, db = torch.zeros_like(g), torch.zeros_like(g)
        _call("b2u_f32_layernorm_bwd", x, g, dy, dx, dg, db, x.shape[0], x.shape[1], ctx.eps)
        return (dx if ctx.needs_input_grad[0] else None), dg, db, None


class InstNormLReLUF(Function):
    """InstanceNorm2d(affine, eps 1e-5) + LeakyReLU(0.01) on [B*HW, C]."""

    @staticmethod
    def forward(ctx, x, g, b, B, HW):
        x = x.contiguous()
        Cc = x.shape[1]
        y = torch.empty_like(x)
        work = torch.empty(2 * B * Cc, dtype=torch.float64, device=x.device)
        stats = torch.empty(2 * B * Cc, dtype=torch.float32, device=x.device)
        _call("b2u_f32_instnorm", x, Cc, y, Cc, g, b, work, stats, B, HW, Cc, cfg.IN_EPS, 1)
        ctx.save_for_backward(x, g, b, stats)
        ctx.geo = (B, HW, Cc)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, g, b, stats = ctx.saved_tensors
        B, HW, Cc = ctx.geo
        dy = dy.contiguous()
        dx = torch.empty_like(x)
        dg, db = torch.zeros_like(g), torch.zeros_like(b)
        work = torch.empty(2 * B * Cc, dtype=torch.float64, device=x.device)
        _call("b2u_f32_instnorm_bwd", x, Cc, dy, Cc, g, b, stats, work, dx, Cc, dg, db, B, HW, Cc, 1)
        return dx, dg, db, None, None


class BNActF(Function):
    """eval-mode (Sync)BatchNorm + optional ReLU on [rows, C] (running statistics are buffers, gamma / beta train)."""

    @staticmethod
    def forward(ctx, x, gamma, beta, rm, rv, act):
        x = x.contiguous()
        rows, Cc = x.shape
        y = torch.empty_like(x)
        _call("b2u_f32_bn_act", x, y, gamma, beta, rm, rv, cfg.BN_EPS, rows, Cc, act)
        ctx.save_for_backward(x, gamma, beta, rm, rv)
        ctx.act = act
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, beta, rm, rv = ctx.saved_tensors
        dy = dy.contiguous()
        dx = torch.empty_like(x)
        dg, db = torch.zeros_like(gamma), torch.zeros_like(beta)
        _call("b2u_f32_bn_act_bwd", x, dy, gamma, beta, rm, rv, cfg.BN_EPS, dx, dg, db, x.shape[0], x.shape[1], ctx.act)
        return (dx if ctx.needs_input_grad[0] else None), dg, db, None, None, None


def _bn_sync() -> bool:
    """torch SyncBatchNorm's `need_sync`: train mode under an initialised default process group of more than one rank."""
    dist = torch.distributed
    return bool(dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1)


class BNTrainF(Function):
    """train-mode (Sync)BatchNorm + optional ReLU on [rows, C]: normalises with the batch mean and biased variance and
    updates running_mean / running_var / num_batches_tracked in place (torch SyncBatchNorm.forward in train mode).  With
    `sync`, the per-channel sums and the row count are all-reduced on the current stream before the finalize, and the
    backward's sum dy' and sum dy' xhat before dx; dgamma / dbeta stay local (DDP averages them)."""

    @staticmethod
    def forward(ctx, x, gamma, beta, rm, rv, nbt, act, momentum, eps, sync):
        x = x.contiguous()
        rows, Cc = x.shape
        if rows < 2:
            raise ValueError(f"BatchNorm in train mode needs more than 1 value per channel, got {rows} rows")
        dev = x.device
        lib = L.load()
        work = torch.empty(int(lib.b2u_f32_bn_work_doubles(rows, Cc)), dtype=torch.float64, device=dev)
        sums = torch.empty(2 * Cc + 1, dtype=torch.float64, device=dev)
        mean = torch.empty(Cc, dtype=torch.float32, device=dev)
        var = torch.empty(Cc, dtype=torch.float32, device=dev)
        _call("b2u_f32_bn_stats", x, rows, Cc, work, sums)
        if sync:
            torch.distributed.all_reduce(sums)
        _call("b2u_f32_bn_finalize", sums, Cc, mean, var, rm, rv, nbt, float(momentum))
        y = torch.empty_like(x)
        _call("b2u_f32_bn_act", x, y, gamma, beta, mean, var, float(eps), rows, Cc, act)
        ctx.save_for_backward(x, gamma, beta, mean, var)
        ctx.cfg = (act, float(eps), bool(sync))
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, beta, mean, var = ctx.saved_tensors
        act, eps, sync = ctx.cfg
        dy = dy.contiguous()
        rows, Cc = x.shape
        dev = x.device
        work = torch.empty(int(L.load().b2u_f32_bn_work_doubles(rows, Cc)), dtype=torch.float64, device=dev)
        red = torch.empty(2 * Cc + 1, dtype=torch.float64, device=dev)
        dg, db = torch.empty_like(gamma), torch.empty_like(beta)
        _call("b2u_f32_bn_train_bwd_reduce", x, dy, gamma, beta, mean, var, eps, rows, Cc, act, work, red, dg, db)
        if sync:
            torch.distributed.all_reduce(red)
        dx = torch.empty_like(x)
        _call("b2u_f32_bn_train_bwd_apply", x, dy, gamma, beta, mean, var, eps, red, dx, rows, Cc, act)
        return dx, dg, db, None, None, None, None, None, None, None


class DropPathAddF(Function):
    """c + s[sample] * f on [B*rows_per_sample, D] (the extractor's `query + drop_path(ffn(...))`, per-sample scale
    s = keep / (1 - drop_prob)); backward: dc = dy, df = s * dy."""

    @staticmethod
    def forward(ctx, c, f, s, rows_per_sample):
        c, f = c.contiguous(), f.contiguous()
        y = torch.empty_like(c)
        _call("b2u_f32_droppath_add", c, f, s, y, c.shape[0], c.shape[1], rows_per_sample)
        ctx.save_for_backward(s)
        ctx.rps = rows_per_sample
        return y

    @staticmethod
    def backward(ctx, dy):
        (s,) = ctx.saved_tensors
        dy = dy.contiguous()
        df = torch.empty_like(dy)
        _call("b2u_f32_droppath_add", None, dy, s, df, dy.shape[0], dy.shape[1], ctx.rps)
        return dy, df, None, None


class ActF(Function):
    @staticmethod
    def forward(ctx, x, act):
        x = x.contiguous()
        y = torch.empty_like(x)
        _call("b2u_f32_act", x, y, x.numel(), act)
        ctx.save_for_backward(x)
        ctx.act = act
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        dx = torch.empty_like(x)
        _call("b2u_f32_act_bwd", x, dy.contiguous(), dx, x.numel(), ctx.act)
        return dx, None


class DWConvF(Function):
    """depthwise 3x3 + bias on token-major planes (planes 1: one HxW image, 3: the ConvFFN pyramid)."""

    @staticmethod
    def forward(ctx, x, W, b, B, H, Wd, planes):
        x = x.contiguous()
        Cc = x.shape[1]
        w9 = W.reshape(Cc, 9).t().contiguous()
        y = torch.empty_like(x)
        _call("b2u_f32_dwconv3x3", x, y, w9, b, B, H, Wd, Cc, planes, 0)
        ctx.save_for_backward(x, w9)
        ctx.geo = (B, H, Wd, Cc, planes)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w9 = ctx.saved_tensors
        B, H, Wd, Cc, planes = ctx.geo
        dy = dy.contiguous()
        dx = torch.empty_like(x)
        zero_b = torch.zeros(Cc, dtype=torch.float32, device=x.device)
        _call("b2u_f32_dwconv3x3", dy, dx, w9.flip(0).contiguous(), zero_b, B, H, Wd, Cc, planes, 0)
        dw9 = torch.zeros_like(w9)
        db = torch.zeros(Cc, dtype=torch.float32, device=x.device)
        _call("b2u_f32_dwconv_wgrad", x, dy, dw9, db, B, H, Wd, Cc, planes)
        return dx, dw9.t().reshape(Cc, 1, 3, 3).contiguous(), db, None, None, None, None


class MaxPoolF(Function):
    @staticmethod
    def forward(ctx, x, B, H, Wd):
        x = x.contiguous()
        Cc = x.shape[1]
        y = torch.empty((B * (H // 2) * (Wd // 2), Cc), dtype=torch.float32, device=x.device)
        _call("b2u_f32_maxpool3x3s2", x, y, B, H, Wd, Cc)
        ctx.save_for_backward(x)
        ctx.geo = (B, H, Wd, Cc)
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        B, H, Wd, Cc = ctx.geo
        dx = torch.zeros_like(x)
        _call("b2u_f32_maxpool3x3s2_bwd", x, dy.contiguous(), dx, B, H, Wd, Cc)
        return dx, None, None, None


class MSDAF(Function):
    """Deformable sampling (ms_deform_attn.py:158-216 minus its three Linears): value [B*HW, heads*dh], offaw [B*Lq, 192]."""

    @staticmethod
    def forward(ctx, value, offaw, B, h, w):
        value, offaw = value.contiguous(), offaw.contiguous()
        heads = cfg.DEFORM_HEADS
        dh = value.shape[1] // heads
        Lq = h * w * 21 // 4
        dev = value.device
        loc = torch.empty((B, Lq, heads, 1, 4, 2), dtype=torch.float32, device=dev)
        attw = torch.empty((B, Lq, heads, 1, 4), dtype=torch.float32, device=dev)
        _call("b2u_f32_msda_prep", offaw, loc, attw, B, h, w, heads)
        shapes = torch.tensor([[h, w]], dtype=torch.int64, device=dev)
        lsi = torch.zeros(1, dtype=torch.int64, device=dev)
        out = torch.empty((B * Lq, heads * dh), dtype=torch.float32, device=dev)
        _call("b2u_msda_forward_f32", value, shapes, lsi, loc, attw, out, B, h * w, Lq, heads, dh, 1, 4)
        ctx.save_for_backward(value, shapes, lsi, loc, attw)
        ctx.geo = (B, h, w, heads, dh, Lq)
        return out

    @staticmethod
    def backward(ctx, dy):
        value, shapes, lsi, loc, attw = ctx.saved_tensors
        B, h, w, heads, dh, Lq = ctx.geo
        dev = value.device
        gval = torch.empty_like(value)
        gloc, gatt = torch.empty_like(loc), torch.empty_like(attw)
        _call("b2u_msda_backward_f32", value, shapes, lsi, loc, attw, dy.contiguous(), gval, gloc, gatt, B, h * w, Lq, heads, dh, 1, 4)
        doff = torch.empty((B * Lq, heads * 12), dtype=torch.float32, device=dev)
        _call("b2u_f32_msda_prep_bwd", attw, gloc, gatt, doff, B, h, w, heads)
        return (gval if ctx.needs_input_grad[0] else None), doff, None, None, None


class FiLMF(Function):
    """z = gamma * zp + beta with (gamma | beta) = gb [px, 2R] and zz = (zs | zp) [px, 2R] (dinounet_training.py:430-432)."""

    @staticmethod
    def forward(ctx, gb, zz):
        gb, zz = gb.contiguous(), zz.contiguous()
        px, R = gb.shape[0], gb.shape[1] // 2
        z = torch.empty((px, R), dtype=torch.float32, device=gb.device)
        _call("b2u_f32_film", gb, zz, z, px, R)
        ctx.save_for_backward(gb, zz)
        return z

    @staticmethod
    def backward(ctx, dz):
        gb, zz = ctx.saved_tensors
        px, R = gb.shape[0], gb.shape[1] // 2
        dgb = torch.empty_like(gb)
        dzz = torch.zeros_like(zz)
        _call("b2u_f32_film_bwd", gb, zz, dz.contiguous(), dgb, dzz, px, R)
        return dgb, dzz


class SEF(Function):
    """out = t * sigmoid(W2 relu(W1 mean_hw(t) + b1) + b2) + shortcut (dinounet_training.py:222-225, 438-441)."""

    @staticmethod
    def forward(ctx, t, sc, w1, b1, w2, b2, B, HW):
        t, sc = t.contiguous(), sc.contiguous()
        Cc, hid = t.shape[1], w1.shape[0]
        w1, w2 = w1.reshape(hid, Cc).contiguous(), w2.reshape(Cc, hid).contiguous()
        pooled = torch.empty((B, Cc), dtype=torch.float32, device=t.device)
        out = torch.empty_like(t)
        _call("b2u_f32_se", t, sc, Cc, pooled, w1, b1, w2, b2, out, B, HW, Cc, hid)
        ctx.save_for_backward(t, pooled, w1, b1, w2, b2)
        ctx.geo = (B, HW, Cc, hid)
        return out

    @staticmethod
    def backward(ctx, dy):
        t, pooled, w1, b1, w2, b2 = ctx.saved_tensors
        B, HW, Cc, hid = ctx.geo
        dy = dy.contiguous()
        dev = t.device
        work = torch.empty(3 * B * Cc, dtype=torch.float32, device=dev)
        dt = torch.empty_like(t)
        dw1, db1, dw2, db2 = torch.zeros_like(w1), torch.zeros_like(b1), torch.zeros_like(w2), torch.zeros_like(b2)
        _call("b2u_f32_se_bwd", t, dy, pooled, w1, b1, w2, b2, work, dt, dw1, db1, dw2, db2, B, HW, Cc, hid)
        return dt, dy, dw1.view(hid, Cc, 1, 1), db1, dw2.view(Cc, hid, 1, 1), db2, None, None


class TailAddF(Function):
    """u = c + bilinear(tap -> r x r) (dinov3_adapter.py:468-476); the ViT tap is frozen: du/dc = identity."""

    @staticmethod
    def forward(ctx, c, tap, B, r, h):
        c = c.contiguous()
        D = c.shape[1]
        ones = torch.ones(D, dtype=torch.float32, device=c.device)
        zeros = torch.zeros(D, dtype=torch.float32, device=c.device)
        u = torch.empty_like(c)
        _call("b2u_f32_tail", c, r * r, 0, tap.contiguous(), u, ones, zeros, B, r, h, D)
        return u

    @staticmethod
    def backward(ctx, du):
        return du, None, None, None, None


# ------------------------------------------------------------------------------------------------------------ the network
@dataclass
class TrainMode:
    """The reference's train-mode semantics for one forward: `bn` maps each BatchNorm prefix of P to its (momentum, eps),
    `drop_scale` [6, B] holds the extractors' per-sample DropPath factors keep / (1 - drop_prob), and `sync` all-reduces
    the BatchNorm statistics across the default process group."""
    bn: Dict[str, Tuple[float, float]]
    drop_scale: torch.Tensor
    sync: bool = False


@contextlib.contextmanager
def _gemm_tier(tier: str):
    global _GEMM_TIER
    prev, _GEMM_TIER = _GEMM_TIER, tier
    try:
        yield
    finally:
        _GEMM_TIER = prev


def trainable_forward(P: Dict[str, torch.Tensor], variant: str, x: torch.Tensor, taps: List[torch.Tensor], num_classes: int,
                      gemm: str = "tf32", train_mode: Optional[TrainMode] = None, recompute: bool = False,
                      deep_supervision: bool = False):
    """Differentiable forward of everything outside the frozen backbone.  P: reference-keyed parameters / buffers
    (`net.state_dict(keep_vars=True)`), x [B,3,S,S] fp32, taps: 4 x [B, P, D] fp32 (frozen ViT outputs) -> logits [B,C,S,S].
    gemm: matrix-product tier, "tf32" (tensor cores) or "fp32" (SIMT parity tier); the backward uses the same tier.
    train_mode: None = eval-mode modules (BatchNorm on running statistics, DropPath off); a TrainMode = batch-statistics
    BatchNorm that updates the running statistics in P, and DropPath with the given factors.
    recompute: keep only each extractor's input query and recompute its internals in the backward (the reference's
    `with_cp=True` checkpointing, dinov3_adapter.py:140-156); the values computed are the same.
    deep_supervision: return [logits@S, logits@S/2, logits@S/4], seg_layers[2] / [1] / [0] on decoder stages 2 / 1 / 0
    (dinounet_training.py:619-629); a head whose logits no loss term reads gets no gradient."""
    if gemm not in ("tf32", "fp32"):
        raise ValueError(f"gemm tier must be 'tf32' or 'fp32', got {gemm!r}")
    with _gemm_tier(gemm):
        return _trainable_forward(P, variant, x, taps, num_classes, train_mode, recompute, deep_supervision)


def _extractor(P, p, c, feat, B, h, drop_scale):
    """One extractor (dinov3_adapter.py:140-156, ms_deform_attn.py:158-216): c [B*Lq, D] -> c + attn, then + ffn
    (+ drop_path(ffn) when `drop_scale` [B] is given)."""
    Lq = h * h * 21 // 4
    lin = lambda t, q, res=None: LinearF.apply(t, P[q + ".weight"].reshape(P[q + ".weight"].shape[0], -1), P.get(q + ".bias"), res)
    qn = LayerNormF.apply(c, P[p + "query_norm.weight"], P[p + "query_norm.bias"], cfg.LN_EPS_ADAPTER)
    fn = LayerNormF.apply(feat, P[p + "feat_norm.weight"], P[p + "feat_norm.bias"], cfg.LN_EPS_ADAPTER)
    value = lin(fn, p + "attn.value_proj")
    offaw = LinearF.apply(qn, torch.cat([P[p + "attn.sampling_offsets.weight"], P[p + "attn.attention_weights.weight"]], 0),
                          torch.cat([P[p + "attn.sampling_offsets.bias"], P[p + "attn.attention_weights.bias"]], 0), None)
    samp = MSDAF.apply(value, offaw, B, h, h)
    c = lin(samp, p + "attn.output_proj", c)                    # c + attn
    fq = LayerNormF.apply(c, P[p + "ffn_norm.weight"], P[p + "ffn_norm.bias"], cfg.LN_EPS_ADAPTER)
    f1 = lin(fq, p + "ffn.fc1")
    f2 = ActF.apply(DWConvF.apply(f1, P[p + "ffn.dwconv.dwconv.weight"], P[p + "ffn.dwconv.dwconv.bias"], B, h, h, 3), L.ACT_GELU)
    if drop_scale is None:
        return lin(f2, p + "ffn.fc2", c)                        # c + ffn
    return DropPathAddF.apply(c, lin(f2, p + "ffn.fc2"), drop_scale, Lq)   # c + drop_path(ffn)


def _recomputed_extractor(tier, *args):
    """`_extractor` on the matrix-product tier of the step that ran it: the backward's replay runs after
    `trainable_forward` has restored the module-global tier."""
    with _gemm_tier(tier):
        return _extractor(*args)


def _trainable_forward(P, variant, x, taps, num_classes, train_mode=None, recompute=False, deep_supervision=False):
    v = cfg.VARIANTS[variant]
    D = v.embed_dim
    B, _, S, _ = x.shape
    h = S // 16
    S2, S4, S8, S16, S32 = S // 2, S // 4, S // 8, S // 16, S // 32
    n4 = S32 * S32
    n3, n2 = 4 * n4, 16 * n4
    Lq = n2 + n3 + n4
    A = "encoder.dinov3_adapter."
    lin = lambda t, p, res=None: LinearF.apply(t, P[p + ".weight"].reshape(P[p + ".weight"].shape[0], -1), P.get(p + ".bias"), res)
    if train_mode is None:
        bn = lambda t, p, act: BNActF.apply(t, P[p + ".weight"], P[p + ".bias"], P[p + ".running_mean"], P[p + ".running_var"], act)
    else:
        bn = lambda t, p, act: BNTrainF.apply(t, P[p + ".weight"], P[p + ".bias"], P[p + ".running_mean"], P[p + ".running_var"],
                                              P[p + ".num_batches_tracked"], act, *train_mode.bn[p], train_mode.sync)

    # ---- SPM (dinov3_adapter.py:279-302)
    Sp = A + "spm."
    xh = x.permute(0, 2, 3, 1).reshape(B * S * S, 3).contiguous()
    c1 = bn(Conv3x3F.apply(xh, P[Sp + "stem.0.weight"], None, B, S, S, 2), Sp + "stem.1", L.ACT_RELU)
    c1 = bn(Conv3x3F.apply(c1, P[Sp + "stem.3.weight"], None, B, S2, S2, 1), Sp + "stem.4", L.ACT_RELU)
    c1 = bn(Conv3x3F.apply(c1, P[Sp + "stem.6.weight"], None, B, S2, S2, 1), Sp + "stem.7", L.ACT_RELU)
    c1 = MaxPoolF.apply(c1, B, S2, S2)
    c2 = bn(Conv3x3F.apply(c1, P[Sp + "conv2.0.weight"], None, B, S4, S4, 2), Sp + "conv2.1", L.ACT_RELU)
    c3 = bn(Conv3x3F.apply(c2, P[Sp + "conv3.0.weight"], None, B, S8, S8, 2), Sp + "conv3.1", L.ACT_RELU)
    c4 = bn(Conv3x3F.apply(c3, P[Sp + "conv4.0.weight"], None, B, S16, S16, 2), Sp + "conv4.1", L.ACT_RELU)
    c1 = lin(c1, Sp + "fc1")
    le = P[A + "level_embed"]
    cs = []
    for i, (t, n) in enumerate(((c2, n2), (c3, n3), (c4, n4))):
        w = P[Sp + f"fc{i + 2}.weight"]
        y = LinearF.apply(t, w.reshape(w.shape[0], -1), P[Sp + f"fc{i + 2}.bias"] + le[i], None)
        cs.append(y.view(B, n, D))
    c = torch.cat(cs, 1).reshape(B * Lq, D)

    # ---- interaction blocks (dinov3_adapter.py:140-231, ms_deform_attn.py:158-216)
    names = [f"{A}interactions.{i}.extractor." for i in range(4)] + [f"{A}interactions.3.extra_extractors.{j}." for j in range(2)]
    # with `recompute`, each extractor is one checkpointed segment from (c, tap) to the new c.  Nothing inside one draws
    # random numbers (DropPath's factors are precomputed) or touches BatchNorm statistics, so the replay needs no RNG state
    # and updates nothing twice.
    for e, k in enumerate((0, 1, 2, 3, 3, 3)):
        feat = taps[k].reshape(B * h * h, D)
        drop_scale = None if train_mode is None else train_mode.drop_scale[e]
        if recompute:
            c = checkpoint(_recomputed_extractor, _GEMM_TIER, P, names[e], c, feat, B, h, drop_scale, use_reentrant=False,
                           preserve_rng_state=False)
        else:
            c = _extractor(P, names[e], c, feat, B, h, drop_scale)

    # ---- adapter tail (dinov3_adapter.py:460-482)
    c3d = c.view(B, Lq, D)
    lv2 = c3d[:, :n2].reshape(B * n2, D)
    lv3 = c3d[:, n2:n2 + n3].reshape(B * n3, D)
    lv4 = c3d[:, n2 + n3:].reshape(B * n4, D)
    up = ConvT2x2F.apply(lv2, P[A + "up.weight"], P[A + "up.bias"], B, S8, S8)
    # c1 = up(c2) + c1 (dinov3_adapter.py:467)
    f_in = [AddF.apply(up, c1), lv2, lv3, lv4]
    feats = []
    for i, (t, r) in enumerate(zip(f_in, (S4, S8, S16, S32))):
        u = TailAddF.apply(t, taps[i].reshape(B * h * h, D), B, r, h)
        feats.append(bn(u, f"{A}norm{i + 1}", L.ACT_NONE))

    # ---- FAPM + learnable upsampling (dinounet_training.py:419-441, 255-264, 499-510)
    Fp = "encoder.fapm."
    R = cfg.FAPM_RANK
    skips = []
    for i, (f, oc) in enumerate(zip(feats, (32, 64, 128, 256))):
        r = S4 >> i
        px = B * r * r
        w1 = torch.cat([P[Fp + "shared_basis.weight"].reshape(R, D), P[f"{Fp}specific_bases.{i}.weight"].reshape(R, D)], 0)
        b1 = torch.cat([P[Fp + "shared_basis.bias"], P[f"{Fp}specific_bases.{i}.bias"]], 0)
        zz = LinearF.apply(f, w1, b1, None)                          # (zs | zp)
        gb = lin(zz[:, :R], f"{Fp}film_generators.{i}")
        z = FiLMF.apply(gb, zz)
        rb = f"{Fp}refinement_blocks.{i}."
        t = InstNormLReLUF.apply(lin(z, rb + "0"), P[rb + "1.weight"], P[rb + "1.bias"], B, r * r)
        t = DWConvF.apply(t, P[rb + "3.depthwise.weight"], P[rb + "3.depthwise.bias"], B, r, r, 1)
        t = InstNormLReLUF.apply(lin(t, rb + "3.pointwise"), P[rb + "3.bn.weight"], P[rb + "3.bn.bias"], B, r * r)
        t = lin(t, rb + "4")
        sc = lin(z, f"{Fp}shortcut_projections.{i}") if (f"{Fp}shortcut_projections.{i}.weight" in P) else z
        y = SEF.apply(t, sc, P[rb + "5.fc.0.weight"], P[rb + "5.fc.0.bias"], P[rb + "5.fc.2.weight"], P[rb + "5.fc.2.bias"], B, r * r)
        uw, ub = P[f"encoder.ups.{i}.up2.weight"], P[f"encoder.ups.{i}.up2.bias"]
        y = ConvT2x2F.apply(y, uw, ub, B, r, r)
        y = ConvT2x2F.apply(y, uw, ub, B, 2 * r, 2 * r)
        skips.append(y)                                              # [B*(4r)^2, oc]

    # ---- decoder (dinounet_training.py:603-629)
    lres = skips[3]
    outs = []
    for s in range(3):
        skip_c = (128, 64, 32)[s]
        r_lo = S8 << s
        r_hi = 2 * r_lo
        t = ConvT2x2F.apply(lres, P[f"decoder.transpconvs.{s}.weight"], P[f"decoder.transpconvs.{s}.bias"], B, r_lo, r_lo)
        t = torch.cat([t, skips[2 - s]], 1)
        for j in range(2):
            p = f"decoder.stages.{s}.convs.{j}."
            t = Conv3x3F.apply(t, P[p + "conv.weight"], P[p + "conv.bias"], B, r_hi, r_hi, 1)
            t = InstNormLReLUF.apply(t, P[p + "norm.weight"], P[p + "norm.bias"], B, r_hi * r_hi)
        lres = t
        if deep_supervision or s == 2:
            y = lin(t, f"decoder.seg_layers.{s}")
            outs.append(y.view(B, r_hi, r_hi, num_classes).permute(0, 3, 1, 2).contiguous())
    if deep_supervision:
        return outs[::-1]
    return outs[0]


class AddF(Function):
    """a + b (the adapter tail's `up(c2) + c1`, dinov3_adapter.py:467) as one elementwise kernel."""

    @staticmethod
    def forward(ctx, a, b):
        a, b = a.contiguous(), b.contiguous()
        out = torch.empty_like(a)
        _call("b2u_f32_add", a, b, out, a.numel())
        return out

    @staticmethod
    def backward(ctx, d):
        return d, d


# ------------------------------------------------------------------------------------------------------------ optimizer
def all_reduce_gradients(params, group=None, average: bool = True):
    """Data-parallel gradient exchange (what DDP does for the reference, nnUNetTrainer.py:216-218): the gradients of the
    ~13-20 M trainable parameters are packed into ONE flat fp32 buffer and summed with a single all-reduce (NCCL over
    NVLink / NVSwitch on GPUs, gloo in the CPU tests), then unpacked in place.  52-80 MB per step: far below the compute
    time of a step, so one bucket is enough; parameters without a gradient contribute zeros so every rank packs the same
    layout."""
    import torch.distributed as dist
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    ps = [p for p in params if p.requires_grad]
    if not ps:
        return
    flat = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1).float() for p in ps])
    dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    if average:
        flat /= dist.get_world_size(group)
    off = 0
    for p in ps:
        n = p.numel()
        g = flat[off:off + n].view_as(p)
        if p.grad is None:
            p.grad = g.clone()
        else:
            p.grad.copy_(g)
        off += n


class FusedSGD(torch.optim.Optimizer):
    """torch.optim.SGD(lr, weight_decay, momentum 0.99, nesterov=True) + clip_grad_norm_(12) (nnUNetTrainer.py:486-489,
    922-923) on the hand-written kernels: one squared-norm reduction per tensor into a device scalar, then one fused update
    per tensor that reads the clip coefficient from device memory (no host synchronisation).

    A `torch.optim.Optimizer`: the reference's PolyLRScheduler (training/lr_scheduler/polylr.py) and torch's schedulers
    construct on it and write `param_groups[i]["lr"]`.  Every parameter given stays in its group, in order, frozen ones
    included, as `torch.optim.SGD(network.parameters())` keeps them; a parameter without a gradient is skipped, and its
    momentum buffer is created the first time it has one (torch's first-step rule: buffer = gradient).  `state_dict()` /
    `load_state_dict()` use torch.optim.SGD's format, so a checkpoint of either optimizer resumes on the other.  The clip
    threshold `max_norm` is a constructor argument on both sides and not part of the state."""

    def __init__(self, params, lr: float, weight_decay: float = 3e-5, momentum: float = 0.99, max_norm: float = 12.0):
        # torch.optim.SGD's group keys, so that the state dicts of the two optimizers are interchangeable
        defaults = dict(lr=lr, momentum=momentum, dampening=0, weight_decay=weight_decay, nesterov=True, maximize=False,
                        foreach=None, differentiable=False, fused=None)
        super().__init__(params, defaults)
        self.max_norm = max_norm
        self._sq = None

    @property
    def params(self) -> List[torch.Tensor]:
        return [p for group in self.param_groups for p in group["params"]]

    def load_state_dict(self, state_dict: dict) -> None:
        """torch.optim.SGD's state dict (`state`: index -> {"momentum_buffer"}, `param_groups` with the index lists).
        ValueError for another parameter count or a buffer shaped unlike its parameter; NotImplementedError for the
        settings the fused update does not compute (nesterov=False, dampening != 0, maximize)."""
        groups, saved = self.param_groups, state_dict["param_groups"]
        if len(groups) != len(saved) or any(len(g["params"]) != len(s["params"]) for g, s in zip(groups, saved)):
            raise ValueError(f"optimizer state holds {[len(s['params']) for s in saved]} parameters per group, this "
                             f"optimizer {[len(g['params']) for g in groups]}")
        for s in saved:
            if not s.get("nesterov", False) or s.get("dampening", 0) != 0 or s.get("maximize", False):
                raise NotImplementedError("FusedSGD computes SGD with nesterov=True, dampening=0 and maximize=False; the "
                                          f"state has nesterov={s.get('nesterov')}, dampening={s.get('dampening')}, "
                                          f"maximize={s.get('maximize')}")
        index_to_param = {i: p for s, g in zip(saved, groups) for i, p in zip(s["params"], g["params"])}
        for i, st in state_dict["state"].items():
            if i not in index_to_param:
                raise ValueError(f"optimizer state has an entry for parameter {i}, which no parameter group lists")
            buf = st.get("momentum_buffer")
            if buf is not None and tuple(buf.shape) != tuple(index_to_param[i].shape):
                raise ValueError(f"momentum buffer {i} has shape {tuple(buf.shape)}, its parameter "
                                 f"{tuple(index_to_param[i].shape)}")
        super().load_state_dict(state_dict)
        for p in self.params:   # the update kernel reads dense buffers; torch.optim.SGD stores None for no buffer
            st = self.state.get(p)
            if st is not None and st.get("momentum_buffer") is None:
                del self.state[p]
            elif st is not None:
                st["momentum_buffer"] = st["momentum_buffer"].contiguous()

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        ps = [p for p in self.params if p.grad is not None]
        if not ps:
            return loss
        dev = ps[0].device
        if self._sq is None:
            self._sq = torch.zeros(1, dtype=torch.float64, device=dev)
        self._sq.zero_()
        for p in ps:
            _call("b2u_f32_sqsum", p.grad.contiguous(), p.numel(), self._sq)
        lib = L.load()
        with torch.cuda.device(dev):
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            for group in self.param_groups:
                for p in group["params"]:
                    if p.grad is None:
                        continue
                    g = p.grad.contiguous()
                    st = self.state[p]
                    first = "momentum_buffer" not in st
                    if first:   # the kernel writes the buffer without reading it on a first step
                        st["momentum_buffer"] = torch.empty_like(p, memory_format=torch.contiguous_format)
                    L.check(lib.b2u_f32_sgd_nesterov(p.data_ptr(), g.data_ptr(), st["momentum_buffer"].data_ptr(), p.numel(),
                                                     group["lr"], group["momentum"], group["weight_decay"],
                                                     self._sq.data_ptr(), self.max_norm, 1 if first else 0, stream), "sgd")
        return loss

    def grad_norm(self) -> float:
        return float(self._sq.sqrt().item())


def train_step(net, loss_fn, optimizer: FusedSGD, data: torch.Tensor, target: torch.Tensor, group=None) -> torch.Tensor:
    """One optimisation step with the semantics of `nnUNetTrainer.train_step` (nnUNetTrainer.py:899-929): zero grads,
    forward, Dice+CE, backward, (data-parallel: one gradient all-reduce), clip 12, SGD-nesterov.  fp32 end to end outside the
    frozen ViT (no GradScaler: there is no fp16 gradient to scale).  The step changes the weights in place, so the next
    eval-path entry of `net` (a validation forward) repacks its engine.  Returns the detached loss."""
    optimizer.zero_grad()
    loss = loss_fn(net(data), target)
    loss.backward()
    all_reduce_gradients(optimizer.params, group)
    optimizer.step()
    net._repack_before_eval = True
    return loss.detach()
