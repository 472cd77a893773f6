"""-m gpu: the matrix products of the training step (dinounet_b200/train_path.py: every LinearF, Conv3x3F and ConvT2x2F
goes through one b2u_f32_gemm_params block into `b2u_tf32_gemm`, csrc/gemm_tf32.cu + gemm_tf32_addr.h, or `b2u_f32_gemm`,
csrc/fp32_tier.cu) and the three helpers beside them in csrc/train_bwd.cu (`b2u_f32_conv3x3_dgrad`, `b2u_f32_colsum`,
`b2u_f32_unshuffle`), at the shapes one forward + backward of dinounet_s/b/l runs at B=2, S=512, and at a few long-K
shapes of the benchmark's batch of 32.

Every launch goes through the C-ABI; every comparison is per element against a float64 reference computed from the
kernel's own fp32 inputs.  Outputs start as NaN (split-K outputs at zero, as the Functions allocate them), and a guard
region after each output buffer must keep its value.  Two checks per case:
  (a) random data against a worst-case rounding bar derived in the test's docstring (u = 2^-24, the fp32 unit roundoff);
  (b) small-integer data, for which every product and partial sum is exact in fp32 and TF32 in any order: the output must
      equal the float64 reference bit for bit, at any K.  (b) sees a dropped, doubled or misplaced element however long
      the K range; (a) sees what (b) cannot: a missing TF32 rounding, or a scalar path that rounds differently.
Run with -s to print each case's worst error as a fraction of its bar.

`b2u_f32_conv3x3_wgrad` stays untested here: no Python path calls it (the step's conv weight gradient is the GEMM's
w_mode 3).  The last test runs WITHOUT a GPU: it records the launches of `trainable_forward` and its backward through a
recording stand-in for the native library and checks that each one's branch signature is in this file's tables."""
import contextlib
import ctypes as C
import math
import types

import pytest
import torch
import torch.nn.functional as F

from dinounet_b200 import lib as L
from dinounet_b200 import train_path as TP
from tests.test_gpu_tf32_gemm import raw_gemm, tf32

gpu = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24                       # unit roundoff of fp32
TIERS = {"tf32": "b2u_tf32_gemm", "fp32": "b2u_f32_gemm"}
GUARD = 64                           # floats after each output buffer that no launch may touch
GUARD_VALUE = 0.375
_WORST: dict = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if _WORST:
        print("\nworst |got - ref| / bar per family:")
        for k in sorted(_WORST):
            print(f"  {k:28s} {_WORST[k]:.4f}")


def _note(family, worst):
    _WORST[family] = max(_WORST.get(family, 0.0), worst)


# ============================================================================================ the kernels' branch choices
# Python restatements of gemm_tf32_addr.h (pick_bn, pick_modes, make_roles' vector flags, make_epi_row's vec_out): the
# test ids and the coverage signature name the branch of the TF32 kernel each parameter block takes.
def _bn(N):
    return 32 if N <= 32 else (64 if N <= 64 else 128)


def _branches(p, al=(True, True, True)):
    """p: an object with the b2u_f32_gemm_params fields; al: 16-byte alignment of A, W and out."""
    a_al, w_al, o_al = al
    w_blk = bool(p.conv) and w_al and ((p.w_mode == 2 and p.ldw % 4 == 0 and p.w_cpad % 4 == 0 and p.N % 4 == 0)
                                       or (p.w_mode == 3 and p.Cpad % 4 == 0 and p.C % 4 == 0))
    a_blk = w_blk and bool(p.a_trans) and a_al and p.lda % 4 == 0 and p.M % 4 == 0
    window = bool(p.conv) and p.w_mode != 3 and not p.a_trans
    if a_blk:
        a_vec = True
    elif p.a_trans:
        a_vec = False
    elif window:
        a_vec = p.C % 4 == 0 and p.Cpad % 4 == 0 and a_al
    else:
        a_vec = p.lda % 4 == 0 and a_al
    w_vec = w_blk or (p.w_mode == 0 and p.ldw % 4 == 0 and w_al)
    atomic = p.ksplit > 1 or p.accumulate
    o_vec = (not p.ps_cout and not atomic and p.ldc % 4 == 0 and p.col_off % 4 == 0 and o_al
             and (not p.residual or p.ldres % 4 == 0))
    bn = _bn(p.N)
    if p.a_trans and p.w_mode == 1:
        kind = "dW"
    elif p.w_mode == 1:
        kind = "dx"
    elif p.w_mode == 2:
        kind = "dgrad"
    elif p.w_mode == 3:
        kind = f"wgrad{'2' if p.conv == L.CONV3X3_S2 else '1'}"
    elif p.conv:
        kind = f"conv{'2' if p.conv == L.CONV3X3_S2 else '1'}"
    else:
        kind = "ps" if p.ps_cout else "lin"
    kind += ("+b" if p.bias else "") + ("+r" if p.residual else "")
    return dict(kind=kind, bn=bn, stage="AWblk" if a_blk else ("Wblk" if w_blk else "row"),
                paths="A" + "sv"[a_vec] + "W" + "sv"[w_vec] + "O" + "sv"[o_vec], split=p.ksplit > 1,
                tail="quad" if p.N % 4 else ("tile" if p.N % bn else "full"))


def _sig(p, al=(True, True, True)):
    b = _branches(p, al)
    return b["kind"], b["bn"], b["stage"], b["paths"], b["split"], b["tail"]


# ============================================================================================ the case table
_FIELDS = {f: 0 for f, _ in L.F32GemmParams._fields_}


def _ksplit_conv(npix):
    return max(1, min(256, npix // 4096))


def _case(name, M, N, K, A_rows, W_rows, img_A=None, img_W=None, weight=None, **f):
    """One parameter block: A is [A_rows, lda], W is [W_rows, ldw]; img_A / img_W = (B, H, C) of an NHWC image operand;
    `weight` names the operand that holds weights (drawn zero-mean), the others are activations or gradients."""
    p = dict(_FIELDS, M=M, N=N, K=K, ldc=N)
    p.update(f)
    return dict(name=name, p=p, A_rows=A_rows, W_rows=W_rows, img_A=img_A, img_W=img_W, weight=weight,
                bias=bool(f.get("bias")), res=bool(f.get("residual")))


def lin(M, N, K, res=False):
    """LinearF forward: y[M, N] = x[M, K] W[N, K]^T + b (+ residual)."""
    return _case(f"lin{M}x{N}x{K}", M, N, K, M, N, weight="W", lda=K, ldw=K, bias=1, residual=int(res), ldres=N if res else 0)


def dx(M, N, K):
    """LinearF / ConvT2x2F dx: out[M, N] = dy[M, K] W[K, N] (w_mode 1)."""
    return _case(f"dx{M}x{N}x{K}", M, N, K, M, K, weight="W", lda=K, ldw=N, w_mode=1)


def dw(M, N, K):
    """LinearF / ConvT2x2F dW: out[M, N] = dy[K, M]^T x[K, N] (a_trans + w_mode 1, K = rows, split-K)."""
    return _case(f"dW{M}x{N}x{K}", M, N, K, K, K, lda=M, ldw=N, a_trans=1, w_mode=1, ksplit=TP._ksplit(K))


def conv(B, H, C, N, stride, bias):
    """Conv3x3F forward: the 3x3 / pad 1 window of x [B, H, H, C] on the A side, W [N, 9C]."""
    Ho = H // stride
    return _case(f"conv{B}x{H}x{C}to{N}", B * Ho * Ho, N, 9 * C, B * H * H, N, img_A=(B, H, C), weight="W", lda=C, ldw=9 * C,
                 conv=L.CONV3X3_S2 if stride == 2 else L.CONV3X3_S1, Hin=H, Win=H, C=C, Cpad=C, bias=int(bias))


def dgrad(B, H, Cout, Cin):
    """Conv3x3F stride-1 dx (w_mode 2): the window of dy [B, H, H, Cout] against the flipped, transposed W [Cout, 9 Cin]."""
    return _case(f"dgrad{B}x{H}x{Cout}to{Cin}", B * H * H, Cin, 9 * Cout, B * H * H, Cout, img_A=(B, H, Cout), weight="W",
                 lda=Cout, ldw=9 * Cin, conv=L.CONV3X3_S1, Hin=H, Win=H, C=Cout, Cpad=Cout, w_mode=2, w_cpad=Cin)


def wgrad(B, H, C, N, stride):
    """Conv3x3F dW (a_trans + w_mode 3): dy [npix, N]^T against the window of x [B, H, H, C] on the W side, K = npix."""
    Ho = H // stride
    npix = B * Ho * Ho
    return _case(f"wgrad{B}x{H}x{C}to{N}", N, 9 * C, npix, npix, B * H * H, img_W=(B, H, C), lda=N, ldw=C, a_trans=1, w_mode=3,
                 conv=L.CONV3X3_S2 if stride == 2 else L.CONV3X3_S1, Hin=H, Win=H, C=C, Cpad=C, ksplit=_ksplit_conv(npix))


def ps(B, h, Cin, Cout):
    """ConvT2x2F forward: x [B h h, Cin] Wp[4 Cout, Cin]^T + b.repeat(4), stored through the 2x2 pixel shuffle."""
    return _case(f"ps{B}x{h}x{Cin}to{Cout}", B * h * h, 4 * Cout, Cin, B * h * h, 4 * Cout, weight="W", lda=Cin, ldw=Cin,
                 ldc=Cout, bias=1, ps_cout=Cout, ps_h=h, ps_w=h)


def linear_step(M, N, K, res=False):
    """A LinearF's three launches: forward, dx, dW."""
    return [lin(M, N, K, res), dx(M, K, N), dw(N, K, M)]


def conv_step(B, H, C, N, stride, bias):
    """A Conv3x3F's GEMM launches: forward, stride-1 dx, dW (the stride-2 dx is b2u_f32_conv3x3_dgrad)."""
    return [conv(B, H, C, N, stride, bias)] + ([dgrad(B, H, N, C)] if stride == 1 else []) + [wgrad(B, H, C, N, stride)]


def convt_step(B, h, Cin, Cout):
    """A ConvT2x2F's launches: the pixel-shuffle forward and the backward's two plain GEMMs on unshuffled rows."""
    return [ps(B, h, Cin, Cout), dx(B * h * h, Cin, 4 * Cout), dw(4 * Cout, Cin, B * h * h)]


def _unique(cases):
    seen, out = set(), []
    for c in cases:
        if c["name"] not in seen:
            seen.add(c["name"])
            out.append(c)
    return out


# one forward + backward of trainable_forward at B=2, S=512 (dinounet_s / b / l: D = 384 / 768 / 1024; Lq = 5376 queries,
# a 32 x 32 ViT grid, FAPM rank 256, the FAPM scales at 128^2 .. 16^2)
TRAIN_GEMM_TABLE = _unique(
    # the adapter's extractors: value_proj on the ViT grid, sampling offsets + attention weights (192), output_proj + c,
    # ConvFFN fc1 (D / 4), fc2 + c; under DropPath fc2 has no residual
    [c for D in (384, 768, 1024) for c in linear_step(2048, D, D) + linear_step(10752, 192, D) + linear_step(10752, D, D, True)
     + linear_step(10752, D // 4, D) + linear_step(10752, D, D // 4, True) + linear_step(10752, D, D // 4)]
    # SPM fc1..fc4 (dinounet_s), the adapter's `up` ConvTranspose
    + [c for M, K in ((32768, 64), (8192, 128), (2048, 256), (512, 256)) for c in linear_step(M, 384, K)]
    + convt_step(2, 64, 384, 384)
    # FAPM per scale: (zs | zp), FiLM generator, refinement 0 / pointwise / 4, shortcut; the two 2x upsamplers
    + [c for px, oc in ((32768, 32), (8192, 64), (2048, 128), (512, 256))
       for c in linear_step(px, 512, 384) + linear_step(px, 512, 256) + linear_step(px, oc, 256) + linear_step(px, oc, oc)]
    + [c for r, oc in ((128, 32), (64, 64), (32, 128), (16, 256)) for c in convt_step(2, r, oc, oc) + convt_step(2, 2 * r, oc, oc)]
    # SPM: the stride-2 stem from the 3 input channels, two stride-1 stem convs, conv2..conv4 at stride 2
    + conv_step(2, 512, 3, 64, 2, False) + conv_step(2, 256, 64, 64, 1, False) + conv_step(2, 128, 64, 128, 2, False)
    + conv_step(2, 64, 128, 256, 2, False) + conv_step(2, 32, 256, 256, 2, False)
    # decoder: transposed convs, the convs after the concat and the second conv of each stage; the segmentation layer
    + [c for r, ci, co in ((64, 256, 128), (128, 128, 64), (256, 64, 32)) for c in convt_step(2, r, ci, co)]
    + [c for H, ci, co in ((128, 256, 128), (256, 128, 64), (512, 64, 32)) for c in conv_step(2, H, ci, co, 1, True) + conv_step(2, H, co, co, 1, True)]
    + linear_step(2 * 512 * 512, 2, 32)
)


def _id(c):
    b = _branches(types.SimpleNamespace(**c["p"]))
    return f"{c['name']}-{b['kind']}-bn{b['bn']}-{b['stage']}-{b['paths']}-k{c['p']['ksplit'] or 1}-{b['tail']}"


# ============================================================================================ running one case
def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _draw(shape, seed, kind, weight, K):
    """Random: activations / gradients randn + 0.5 (a nonzero mean: the partial sums of every K slice point the same way,
    so a dropped or doubled slice moves an element by about 1/ksplit of it), weights randn.  Integer: activations in
    {0, 1}, weights in {-1, 0, 1, 2} ({-1, 0, 1} where K * 2 could reach 2^24)."""
    g = _gen(seed)
    if kind == "rand":
        return torch.randn(shape, generator=g, device=DEV) + (0.0 if weight else 0.5)
    if not weight:
        return torch.randint(0, 2, shape, generator=g, device=DEV).float()
    hi = 3 if 2 * K + 4 < 2 ** 24 else 2
    return torch.randint(-1, hi, shape, generator=g, device=DEV).float()


def _ref(c, A, W, bias, res):
    """float64 output of the parameter block on float64 operands (the output buffer's layout)."""
    p = c["p"]
    M, N, K = p["M"], p["N"], p["K"]
    kind = _branches(types.SimpleNamespace(**p))["kind"].split("+")[0]
    if kind == "lin":
        y = A @ W.t()
    elif kind == "ps":
        y = A @ W.t()
    elif kind == "dx":
        y = A @ W
    elif kind == "dW":
        y = A.t() @ W
    elif kind.startswith("conv"):
        B, H, Cc = c["img_A"]
        s = 2 if kind == "conv2" else 1
        xi = A.view(B, H, H, Cc).permute(0, 3, 1, 2)
        Wt = W.view(N, 3, 3, Cc).permute(0, 3, 1, 2)
        y = F.conv2d(xi, Wt, stride=s, padding=1).permute(0, 2, 3, 1).reshape(M, N)
    elif kind == "dgrad":
        B, H, Co = c["img_A"]
        Ci = N
        Wt = W.view(Co, 3, 3, Ci).permute(0, 3, 1, 2)
        g = A.view(B, H, H, Co).permute(0, 3, 1, 2)
        y = torch.nn.grad.conv2d_input((B, Ci, H, H), Wt, g, padding=1).permute(0, 2, 3, 1).reshape(M, N)
    else:
        B, H, Cc = c["img_W"]
        s = 2 if kind == "wgrad2" else 1
        Ho = H // s
        xi = W.view(B, H, H, Cc).permute(0, 3, 1, 2)
        g = A.view(B, Ho, Ho, M).permute(0, 3, 1, 2)
        y = torch.nn.grad.conv2d_weight(xi, (M, Cc, 3, 3), g, stride=s, padding=1).permute(0, 2, 3, 1).reshape(M, N)
    if bias is not None:
        y = y + bias
    if kind == "ps":
        B, h, Cout = M // (p["ps_h"] * p["ps_w"]), p["ps_h"], p["ps_cout"]
        y = y.view(B, h, h, 2, 2, Cout).permute(0, 1, 3, 2, 4, 5).reshape(B * 4 * h * h, Cout)
    if res is not None:
        y = y + res
    return y


def _slice_len(tier, K, ksplit):
    """Length of one K slice: whole k-blocks of 32 (TF32 kernel) or 8 (SIMT kernel), as k_slice / f32_gemm_kernel cut them."""
    if ksplit <= 1:
        return K
    kb = 32 if tier == "tf32" else 8
    return min(K, -(-(-(-K // ksplit)) // kb) * kb)


def _coef(tier, K, ksplit):
    """Bar per unit of sum |a||w| of a K-term product.  TF32: the products of two TF32 values are exact in fp32, what is
    left is the accumulation, bounded like the 16-bit wgmma tests' accumulator: (ceil(K_slice / 8) + 2) 2^-23, plus u per
    split-K atomic add.  SIMT fp32: an fma chain of K_slice terms and then the atomics, (K_slice + ksplit + 2) u."""
    ks = max(1, ksplit)
    Ks = _slice_len(tier, K, ks)
    if tier == "tf32":
        return (math.ceil(Ks / 8) + 2) * 2.0 ** -23 + ks * U
    return (Ks + ks + 2) * U


def _run(c, tier, kind, seed):
    """Launch one case on one tier with `kind` data; returns (got, ref, bar), bar None for the integer data."""
    p = dict(c["p"])
    M, N, K = p["M"], p["N"], p["K"]
    A = _draw((c["A_rows"], p["lda"]), seed, kind, c["weight"] == "A", K)
    W = _draw((c["W_rows"], p["ldw"]), seed + 1, kind, c["weight"] == "W", K)
    bias = res = None
    if c["bias"]:
        nb = p["ps_cout"] or N
        bias = (torch.randn(nb, generator=_gen(seed + 2), device=DEV) if kind == "rand"
                else torch.randint(-2, 3, (nb,), generator=_gen(seed + 2), device=DEV).float())
        if p["ps_cout"]:
            bias = bias.repeat(4).contiguous()                       # ConvT2x2F: b.repeat(4)
        p["bias"] = bias
    rows_out = M * 4 if p["ps_cout"] else M
    ncols = p["ps_cout"] or N
    if c["res"]:
        res = (torch.randn((rows_out, ncols), generator=_gen(seed + 3), device=DEV) if kind == "rand"
               else torch.randint(-2, 3, (rows_out, ncols), generator=_gen(seed + 3), device=DEV).float())
        p["residual"] = res
    buf = torch.empty(rows_out * ncols + GUARD, device=DEV)
    out = buf[:rows_out * ncols].view(rows_out, ncols)
    out.fill_(0.0 if p["ksplit"] > 1 else float("nan"))
    buf[rows_out * ncols:] = GUARD_VALUE
    p.update(A=A, W=W, out=out)
    raw_gemm(TIERS[tier], **{k: v for k, v in p.items() if not (isinstance(v, int) and v == 0)})   # unset fields stay 0
    guard = buf[rows_out * ncols:]
    assert (guard == GUARD_VALUE).all(), f"{c['name']} {tier}: the launch wrote past its output"
    rA, rW = (tf32(A), tf32(W)) if tier == "tf32" else (A.double(), W.double())
    bd = None if bias is None else bias.double()
    rd = None if res is None else res.double()
    ref = _ref(c, rA, rW, bd[:N] if (bd is not None and not p["ps_cout"]) else bd, rd)
    if kind == "int":
        return out, ref, None
    absum = _ref(c, rA.abs(), rW.abs(), None, None)
    n_epi = int(bias is not None) + int(res is not None)
    bar = absum * _coef(tier, K, p["ksplit"])
    if n_epi:
        bar = bar + n_epi * U * _ref(c, rA.abs(), rW.abs(), None if bd is None else bd.abs(), None if rd is None else rd.abs())
    return out, ref, bar


def _check(family, what, got, ref, bar):
    """bar None: bitwise equality; else |got - ref| <= bar element by element (an unwritten NaN fails).  Returns the worst
    |got - ref| / bar."""
    got = got.double()
    if bar is None:
        bad = ~(got == ref)
        n = int(bad.sum())
        if n:
            i = int(bad.reshape(-1).nonzero()[0])
            raise AssertionError(f"{what}: {n} of {got.numel()} elements differ from the exact result; first at flat {i}: got "
                                 f"{got.reshape(-1)[i].item():.9g}, exact {ref.reshape(-1)[i].item():.9g}")
        return 0.0
    err = (got - ref).abs()
    assert torch.isfinite(got).all(), f"{what}: {int((~torch.isfinite(got)).sum())} non-finite outputs (unwritten elements?)"
    ratio = torch.where(bar > 0, err / bar.clamp_min(1e-300), torch.where(err > 0, torch.full_like(err, float("inf")), err))
    worst = ratio.max().item()
    _note(family, worst)
    if worst > 1.0:
        i = int(ratio.argmax())
        raise AssertionError(f"{what}: {int((ratio > 1.0).sum())} of {ratio.numel()} elements over the bar; worst: got "
                             f"{got.reshape(-1)[i].item():.9g}, ref {ref.reshape(-1)[i].item():.9g}, bar "
                             f"{bar.reshape(-1)[i].item():.3g} ({worst:.2f}x)")
    return worst


def _gemm_case(c, tier, family):
    cid = _id(c)
    got, ref, bar = _run(c, tier, "rand", 11)
    worst = _check(f"{family} {tier}", f"{cid} {tier} random", got, ref, bar)
    del got, ref, bar
    got, ref, _ = _run(c, tier, "int", 23)
    _check(f"{family} {tier}", f"{cid} {tier} integer", got, ref, None)
    print(f"{cid} {tier}: worst {worst:.4f} of the bar, integer data exact")


@gpu
@pytest.mark.parametrize("tier", ["tf32", "fp32"])
@pytest.mark.parametrize("case", TRAIN_GEMM_TABLE, ids=_id)
def test_train_step_gemm(case, tier):
    """Every matrix-product launch of one training step at B=2, S=512 on both tiers.  Bars (S = sum |a||w|, in float64 on
    the kernel's operands; TF32 tier on TF32-rounded operands, whose products are exact in fp32):
      TF32:  S ((ceil(K_slice / 8) + 2) 2^-23 + ksplit u) + u (S + |b| + |r|) per epilogue add (bias, residual);
      fp32:  S (K_slice + ksplit + 2) u                   + the same epilogue terms.
    Margin to one dropped K slice: with operands randn + 0.5, sum a w over a slice is about (0.25 / 0.80) S / ksplit.  For
    the longest split of this table (the segmentation layer's dW, K = 524288 in 64 slices of 8192) the TF32 bar is
    1.3e-4 S and a slice 4.9e-3 S (39x); the SIMT bar is 4.9e-4 S (10x).  The 512^2 conv weight gradients (K = 524288 in
    128 slices of 4096): TF32 6.9e-5 S against 2.4e-3 S (35x), SIMT 2.5e-4 S (10x).  Integer data must match exactly."""
    _gemm_case(case, tier, _branches(types.SimpleNamespace(**case["p"]))["kind"])


# the benchmark's batch: the segmentation layer's dW over 32 x 512^2 = 8.4 M rows (64 slices of 131072) and the last
# decoder conv's weight gradient over the same pixels (256 slices of 32768)
LONG_K_TABLE = [dw(2, 32, 32 * 512 * 512), wgrad(32, 512, 32, 32, 1)]


@gpu
@pytest.mark.parametrize("tier", ["tf32", "fp32"])
@pytest.mark.parametrize("case", LONG_K_TABLE, ids=_id)
def test_long_k_at_the_benchmark_batch(case, tier):
    """Same bars as above.  Here a worst-case rounding bar comes close to the size of one slice (segmentation dW, K = 8.4 M
    in 64 slices of 131072: the TF32 bar is 2.0e-3 S against a slice of 4.9e-3 S, 2.5x; the SIMT bar 7.8e-3 S exceeds a
    slice; the conv weight gradient, 256 slices of 32768: TF32 5.0e-4 S against 1.2e-3 S), so the random data checks
    the rounding and the integer data (both operands are activations or gradients, drawn from {0, 1}: every partial sum
    is at most 2^23) checks that each of the 8.4 M rows is added exactly once."""
    _gemm_case(case, tier, "longK")
    torch.cuda.empty_cache()


# ============================================================================================ the helper kernels
def _call(fn, *args):
    raw = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    L.check(getattr(L.load(), fn)(*raw, C.c_void_p(torch.cuda.current_stream().cuda_stream)), fn)


# (B, H, Wd, Cc, Cpad, N, stride): the SPM's conv2..conv4 at 512^2 (the same for s, b and l: the SPM is 64 wide)
DGRAD_TABLE = [(2, 128, 128, 64, 64, 128, 2), (2, 64, 64, 128, 128, 256, 2), (2, 32, 32, 256, 256, 256, 2)]


@gpu
@pytest.mark.parametrize("shape", DGRAD_TABLE, ids=lambda s: "x".join(map(str, s)))
def test_conv3x3_dgrad(shape):
    """b2u_f32_conv3x3_dgrad (the stride-2 data gradient): one fma chain over at most 9 N terms per element, so the bar is
    (9 N + 1) u sum |dy||w| against float64 conv2d_input.  A wrong tap or parity test moves an element by O(|dy||w|)."""
    B, H, Wd, Cc, Cpad, N, s = shape
    Ho, Wo = H // s, Wd // s
    for kind, seed in (("rand", 5), ("int", 6)):
        dy = _draw((B * Ho * Wo, N), seed, kind, False, 9 * N)
        Wp = _draw((N, 9 * Cpad), seed + 1, kind, True, 9 * N)
        dxo = torch.full((B * H * Wd, Cc), float("nan"), device=DEV)
        _call("b2u_f32_conv3x3_dgrad", dy, Wp, dxo, B, H, Wd, Cc, Cpad, N, s)

        def ref(g, w):
            Wt = w.view(N, 3, 3, Cpad)[..., :Cc].permute(0, 3, 1, 2)
            gi = g.view(B, Ho, Wo, N).permute(0, 3, 1, 2)
            return torch.nn.grad.conv2d_input((B, Cc, H, Wd), Wt, gi, stride=s, padding=1).permute(0, 2, 3, 1).reshape(B * H * Wd, Cc)
        r = ref(dy.double(), Wp.double())
        bar = None if kind == "int" else (9 * N + 1) * U * ref(dy.double().abs(), Wp.double().abs())
        w = _check("conv3x3_dgrad", f"dgrad {shape} {kind}", dxo, r, bar)
        print(f"dgrad {shape} {kind}: worst {w:.4f} of the bar")


def _colsum_splits(rows):
    return 64 if rows > 65536 else (8 if rows > 2048 else 1)


# (rows, Cc): both sides of the split boundaries (1 / 8 / 64 splits above 2048 / 65536 rows) at the bias widths of a step
# (2: the segmentation layer, 21 and 3 off the 32-column blocks), then the row counts of a step and the benchmark batch
COLSUM_TABLE = sorted(set(
    [(r, cc) for r in (2048, 2049, 65536, 65537) for cc in (2, 3, 21, 32, 64, 384, 1024)]
    + [(524288, cc) for cc in (2, 3, 21, 32, 64)] + [(32 * 512 * 512, 2)]
    # the step's bias gradients (dinounet_s / b / l at B=2, S=512)
    + [(r, cc) for r in (512, 2048, 8192, 32768) for cc in (32, 64, 128, 256, 384, 512, 768, 1024)]
    + [(r, cc) for r in (2048, 10752) for cc in (96, 192, 256, 384, 768, 1024)]
    + [(131072, 32), (131072, 64), (524288, 32), (524288, 2)]))


@gpu
@pytest.mark.parametrize("rows,Cc", COLSUM_TABLE, ids=lambda v: str(v))
def test_colsum(rows, Cc):
    """b2u_f32_colsum (every bias gradient): per split each of 8 row groups sums a chain of ceil(rows / splits / 8) rows, the
    8 partials are added in a chain and the split's total atomically: bar (ceil(rows / splits / 8) + 8 + splits + 1) u
    sum |x| per column.  With x = randn + 0.5 a dropped split moves a column by about (0.5 / 0.9) / splits of sum |x|: at
    8.4 M rows (64 splits, chains of 16384) 8.7e-3 against a bar of 9.8e-4 (9x).  Integer data ({-1, 0, 1, 2}, {0, 1} at
    8.4 M rows) must sum exactly: a dropped or doubled row shows at any length."""
    splits = _colsum_splits(rows)
    for kind, seed in (("rand", 3), ("int", 4)):
        g = _gen(seed)
        if kind == "rand":
            x = torch.randn((rows, Cc), generator=g, device=DEV) + 0.5
        else:
            x = torch.randint(0 if rows * 2 >= 2 ** 24 else -1, 2 if rows * 2 >= 2 ** 24 else 3, (rows, Cc), generator=g, device=DEV).float()
        buf = torch.full((Cc + GUARD,), GUARD_VALUE, device=DEV)
        out = buf[:Cc]
        out.zero_()
        _call("b2u_f32_colsum", x, Cc, rows, Cc, out)
        assert (buf[Cc:] == GUARD_VALUE).all(), "colsum wrote past its output"
        xd = x.double()
        ref = xd.sum(0)
        bar = None if kind == "int" else (math.ceil(rows / splits / 8) + 8 + splits + 1) * U * xd.abs().sum(0)
        w = _check("colsum", f"colsum {rows}x{Cc} {kind}", out, ref, bar)
        if kind == "rand":
            print(f"colsum {rows}x{Cc}: worst {w:.4f} of the bar, integer data exact")


# (B, h, w, Cout): the decoder's and FAPM's ConvTranspose backward at 512^2 (s / b / l: the `up` one is D wide)
UNSHUFFLE_TABLE = sorted(set([(2, r, r, c) for r, c in ((16, 256), (32, 256), (32, 128), (64, 128), (64, 64), (128, 64), (128, 32),
                                                         (256, 32), (64, 384), (64, 768), (64, 1024))]))


@gpu
@pytest.mark.parametrize("shape", UNSHUFFLE_TABLE + [(1, 5, 7, 3)], ids=lambda s: "x".join(map(str, s)))
def test_unshuffle(shape):
    """b2u_f32_unshuffle is a permutation: bitwise equal to the torch permute of the same data, every element written.
    Also read from columns [col_off, col_off + Cout) of a wider image (the kernel's ld / col_off arguments)."""
    B, h, w, Cout = shape
    for ld, col_off in ((Cout, 0), (Cout + 5, 3)):
        dy = torch.randn((B * 4 * h * w, ld), generator=_gen(7), device=DEV)
        out = torch.full((B * h * w, 4 * Cout), float("nan"), device=DEV)
        _call("b2u_f32_unshuffle", dy, ld, col_off, out, B, h, w, Cout)
        want = dy[:, col_off:col_off + Cout].reshape(B, h, 2, w, 2, Cout).permute(0, 1, 3, 2, 4, 5).reshape(B * h * w, 4 * Cout)
        assert torch.equal(out, want), f"unshuffle {shape} ld {ld}: {int((out != want).sum())} elements differ"


# ============================================================================================ the Functions at step shapes
def _function_case(tier, make, fwd, ref_fwd, grads):
    """Forward + backward of one Function on `tier` against float64 autograd.  make(): fp32 leaves; fwd(*leaves) -> y;
    ref_fwd(*float64 leaves) -> y; grads: per output name (y, then one per leaf) the (coefficient, K) of its bar:
    got within coef * S of the float64 value, S from the same autograd on |operands| and |dy|.  On the TF32 tier the
    GEMM outputs are compared with the autograd on TF32-rounded operands; the outputs of fp32 helpers (colsum, the stride-2
    data gradient) with the unrounded one."""
    prev, TP._GEMM_TIER = TP._GEMM_TIER, tier
    try:
        leaves = [t.requires_grad_() for t in make()]
        y = fwd(*leaves)
        g = torch.randn(y.shape, generator=_gen(99), device=DEV) + 0.5
        y.backward(g)
        got = [y.detach()] + [t.grad for t in leaves]
    finally:
        TP._GEMM_TIER = prev

    def run(op, gop):
        ls = [op(i, t.detach()).requires_grad_() for i, t in enumerate(leaves)]
        yr = ref_fwd(*ls)
        yr.backward(gop(g))
        return [yr.detach()] + [t.grad for t in ls]
    plain = run(lambda i, t: t.double(), lambda t: t.double())
    # the GEMMs round x, W and dy to TF32; the bias is added in fp32
    rounded = run(lambda i, t: tf32(t) if i < 2 else t.double(), tf32) if tier == "tf32" else plain
    absum = run(lambda i, t: t.double().abs(), lambda t: t.double().abs())
    for (name, rule), a, r_plain, r_round, s in zip(grads, got, plain, rounded, absum):
        coef, fp32_side = rule(tier)
        ref = r_plain if (fp32_side or tier == "fp32") else r_round
        w = _check(f"Function {tier}", f"{name} {tier}", a, ref, coef * s)
        print(f"{name} {tier}: worst {w:.4f} of the bar")


def _gemm_rule(K, ksplit=1, epi=0):
    return lambda tier: (_coef(tier, K, ksplit) + epi * U, False)


def _colsum_rule(rows):
    return lambda tier: ((math.ceil(rows / _colsum_splits(rows) / 8) + 8 + _colsum_splits(rows) + 1) * U, True)


@gpu
@pytest.mark.parametrize("tier", ["tf32", "fp32"])
def test_linear_function_segmentation_layer(tier):
    """LinearF at the segmentation layer (32 -> 2 over 2 x 512^2 rows): forward + bias, dx (K = 2), dW (K = 524288 in
    64 slices), db (colsum over 524288 rows); the bars are the per-launch bars above."""
    M, K, N = 2 * 512 * 512, 32, 2
    _function_case(tier, lambda: [torch.randn((M, K), generator=_gen(1), device=DEV) + 0.5,
                                  torch.randn((N, K), generator=_gen(2), device=DEV), torch.randn(N, generator=_gen(3), device=DEV)],
                   lambda x, W, b: TP.LinearF.apply(x, W, b, None), lambda x, W, b: F.linear(x, W, b),
                   [("linear y", _gemm_rule(K, 1, 1)), ("linear dx", _gemm_rule(N)), ("linear dW", _gemm_rule(M, TP._ksplit(M))),
                    ("linear db", _colsum_rule(M))])


@gpu
@pytest.mark.parametrize("tier", ["tf32", "fp32"])
@pytest.mark.parametrize("B,H,Cin,Cout,stride", [(2, 512, 64, 32, 1), (2, 128, 64, 128, 2)], ids=["dec512-s1", "spm-conv2-s2"])
def test_conv3x3_function(tier, B, H, Cin, Cout, stride):
    """Conv3x3F at the last decoder stage's first conv (64 -> 32 at 512^2, stride 1: the GEMM's w_mode 2 data gradient)
    and the SPM's conv2 (64 -> 128, stride 2: b2u_f32_conv3x3_dgrad): the weight permute to [N, 9 C] and back, the conv
    weight gradient's split-K and colsum for db."""
    Ho = H // stride
    npix = B * Ho * Ho

    def ref(x, W, b):
        return F.conv2d(x.view(B, H, H, Cin).permute(0, 3, 1, 2), W, b, stride=stride, padding=1).permute(0, 2, 3, 1).reshape(npix, Cout)
    dx_rule = _gemm_rule(9 * Cout) if stride == 1 else (lambda tier: ((9 * Cout + 1) * U, True))
    _function_case(tier, lambda: [torch.randn((B * H * H, Cin), generator=_gen(1), device=DEV) + 0.5,
                                  torch.randn((Cout, Cin, 3, 3), generator=_gen(2), device=DEV),
                                  torch.randn(Cout, generator=_gen(3), device=DEV)],
                   lambda x, W, b: TP.Conv3x3F.apply(x, W, b, B, H, H, stride), ref,
                   [("conv y", _gemm_rule(9 * Cin, 1, 1)), ("conv dx", dx_rule), ("conv dW", _gemm_rule(npix, _ksplit_conv(npix))),
                    ("conv db", _colsum_rule(npix))])


@gpu
@pytest.mark.parametrize("tier", ["tf32", "fp32"])
def test_convt2x2_function_first_fapm_upsampler(tier):
    """ConvT2x2F at the first FAPM upsampler (32 -> 32, 128^2 -> 256^2): b.repeat(4), the pixel shuffle, the unshuffled
    backward's dx and dW (K = 32768 rows in 16 slices), the dW view / permute back to [Cin, Cout, 2, 2], colsum for db."""
    B, h, Cin, Cout = 2, 128, 32, 32
    M = B * h * h

    def ref(x, W, b):
        return F.conv_transpose2d(x.view(B, h, h, Cin).permute(0, 3, 1, 2), W, b, stride=2).permute(0, 2, 3, 1).reshape(4 * M, Cout)
    _function_case(tier, lambda: [torch.randn((M, Cin), generator=_gen(1), device=DEV) + 0.5,
                                  torch.randn((Cin, Cout, 2, 2), generator=_gen(2), device=DEV),
                                  torch.randn(Cout, generator=_gen(3), device=DEV)],
                   lambda x, W, b: TP.ConvT2x2F.apply(x, W, b, B, h, h), ref,
                   [("convT y", _gemm_rule(Cin, 1, 1)), ("convT dx", _gemm_rule(4 * Cout)), ("convT dW", _gemm_rule(M, TP._ksplit(M))),
                    ("convT db", _colsum_rule(4 * M))])


# ============================================================================================ coverage (CPU)
class _Recorder:
    """Stand-in for the native library: records every call, computes nothing."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*a):
            self.calls.append((name, a))
            return 0
        return fn


@pytest.fixture
def rec(monkeypatch):
    r = _Recorder()
    monkeypatch.setattr(L, "load", lambda: r)
    monkeypatch.setattr(TP, "_s", lambda t: 0)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda dev=None: type("S", (), {"cuda_stream": 0})())
    return r


@pytest.mark.parametrize("variant", ["dinounet_s", "dinounet_b", "dinounet_l"])
def test_train_step_launches_are_covered(rec, monkeypatch, variant):
    """Runs trainable_forward and its backward at B=2, S=512 on the CPU against the recording stand-in, once with eval
    semantics and once with a TrainMode, and checks that every matrix-product launch's branch signature (kind, BN,
    staging, vector paths, split-K, N tail) is in TRAIN_GEMM_TABLE and every helper launch's shape in its table, so a
    change of the step names the launch whose tests no longer cover it."""
    from oracle import dinounet_oracle as O
    from oracle import train_mode_oracle as T
    wrapped = {"_gemm": 0, "_call": 0}

    def counting(name, fn):
        def f(*a, **k):
            wrapped[name] += 1
            return fn(*a, **k)
        return f
    monkeypatch.setattr(TP, "_gemm", counting("_gemm", TP._gemm))
    monkeypatch.setattr(TP, "_call", counting("_call", TP._call))
    B, S = 2, 512
    sigs = {_sig(types.SimpleNamespace(**c["p"])) for c in TRAIN_GEMM_TABLE}
    colsum, unshuffle, dgrad_shapes = set(COLSUM_TABLE), set(UNSHUFFLE_TABLE), set(DGRAD_TABLE)
    P = {k: t.clone() for k, t in O.make_state_dict(variant, 2, seed=0).items()}
    for k, t in P.items():
        if t.is_floating_point() and not k.endswith(("running_mean", "running_var")):
            t.requires_grad_(True)
    x = torch.zeros(B, 3, S, S)
    taps = [torch.randn(B, (S // 16) ** 2, O.VARIANTS[variant].dim) for _ in range(4)]
    missing, seen = [], set()
    for mode in (None, TP.TrainMode(bn={p: (0.1, 1e-5) for p in T.BN_LAYERS}, drop_scale=torch.ones(6, B) / 0.7)):
        rec.calls.clear()
        wrapped.update(_gemm=0, _call=0)
        TP.trainable_forward(P, variant, x, taps, 2, "tf32", mode).sum().backward()
        for k in P:
            if isinstance(P[k], torch.Tensor):
                P[k].grad = None
        n = {"gemm": 0, "b2u_f32_colsum": 0, "b2u_f32_unshuffle": 0, "b2u_f32_conv3x3_dgrad": 0}
        for name, a in rec.calls:
            if name.endswith("_gemm"):
                assert name == "b2u_tf32_gemm"
                p = a[0]._obj
                s = _sig(p, tuple(v % 16 == 0 for v in (p.A, p.W, p.out)))
                seen.add(s)
                n["gemm"] += 1
                if s not in sigs:
                    missing.append(f"b2u_tf32_gemm M={p.M} N={p.N} K={p.K}: {s} not in TRAIN_GEMM_TABLE")
            elif name == "b2u_f32_colsum":
                ld, rows, Cc = a[1:4]
                n[name] += 1
                if ld != Cc or (rows, Cc) not in colsum:
                    missing.append(f"colsum ld={ld} rows={rows} Cc={Cc} not in COLSUM_TABLE")
            elif name == "b2u_f32_unshuffle":
                ld, col_off, Bb, h, w, Cout = a[1:3] + a[4:8]
                n[name] += 1
                if ld != Cout or col_off or (Bb, h, w, Cout) not in unshuffle:
                    missing.append(f"unshuffle {(ld, col_off, Bb, h, w, Cout)} not in UNSHUFFLE_TABLE")
            elif name == "b2u_f32_conv3x3_dgrad":
                n[name] += 1
                if tuple(a[3:10]) not in dgrad_shapes:
                    missing.append(f"conv3x3_dgrad {tuple(a[3:10])} not in DGRAD_TABLE")
        # 82 forward products (5 SPM convs, 4 SPM linears, 5 per extractor, the `up` ConvTranspose, 8 per FAPM scale,
        # 3 + 6 in the decoder, the segmentation layer) and 2 in the backward of each, less the stem's dx (the input needs
        # none) and the 3 stride-2 data gradients (b2u_f32_conv3x3_dgrad): 242; 12 ConvTranspose backwards unshuffle
        assert n["gemm"] == wrapped["_gemm"] == 242, n
        assert n["b2u_f32_unshuffle"] == 12 and n["b2u_f32_conv3x3_dgrad"] == 3 and n["b2u_f32_colsum"] > 50, n
        assert sum(n.values()) - n["gemm"] <= wrapped["_call"]
    assert not missing, "\n".join(sorted(set(missing)))
