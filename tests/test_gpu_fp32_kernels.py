"""-m gpu: the fp32 parity tier's kernels (csrc/fp32_tier.cu, the launches of engine_fp32.build_plan_fp32) and the
optimizer kernels behind FusedSGD (csrc/train_bwd.cu) against float64 references, one kernel at a time through the
C-ABI, at the shapes a 512x512 forward of dinounet_s/b/l runs, at the odd half-grids of S = 96 / 160 / 224, and on both
sides of every branch these kernels pick from the shape.

Every comparison is per element: |got - ref| <= bar, with ref computed in float64 from the kernel's own fp32 inputs.
A bar is a worst-case bound derived in each test's docstring from these terms (u = 2^-24, the fp32 unit roundoff):
  * a dot product or sum evaluated as a chain or tree of depth k is within k u sum|terms| of the exact sum;
  * every further fp32 operation adds u times its magnitude (a contracted fma rounds once, so it never adds more);
  * expf and erff are within 2 ulp (CUDA's documented bounds; the build has no fast-math), i.e. 4u relative;
  * an error e in the input of a function with slope at most L is carried as L e (sup |GELU'| = 1.13).
The bars are worst-case bounds: rounding errors of a long chain mostly cancel, so a K-term dot product typically lands
about sqrt(K) below its bar.  A wrong tap, head, row remap or dropped partial is off by the size of the data, orders of
magnitude over these bars.  Outputs start as NaN, so an element the kernel does not write fails; where a launch writes
a sub-block of a buffer (row remap, pixel shuffle, column offset), everything outside it must keep its NaN.  Run with
-s to print each kernel's worst error as a fraction of its bar."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dinounet_b200 import config as cfg
from dinounet_b200 import lib as L
from oracle import dinounet_oracle as O
from tests.gpu_helpers import P, stream

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24                       # unit roundoff of fp32
U64 = 2.0 ** -53                     # unit roundoff of fp64
GELU_SLOPE = 1.13                    # sup |GELU'(x)| = 1.1289 (at x = sqrt(2))
SLOPE = float(np.float32(0.01))      # the kernels' LeakyReLU slope 0.01f
_WORST: dict = {}
_NOTES: list = []


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |got - ref| / bar per kernel:")
    for k in sorted(_WORST):
        print(f"  {k:22s} {_WORST[k]:.3f}")
    for n in _NOTES:
        print("  " + n)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(shape, seed, scale=1.0, shift=0.0):
    return torch.randn(shape, generator=_gen(seed), device=DEV) * scale + shift


def _nan(shape, dt=torch.float32):
    return torch.full((shape,) if isinstance(shape, int) else shape, float("nan"), device=DEV, dtype=dt)


def _check(kernel, what, got, ref, bar):
    """|got - ref| <= bar element by element.  Where ref is NaN (an element the launch must not write), got must be NaN
    too."""
    got, ref = got.double(), ref.double()
    bar = bar.double().expand_as(ref)
    skip = torch.isnan(ref)
    assert torch.equal(torch.isnan(got), skip), \
        f"{what}: {int((torch.isnan(got) & ~skip).sum())} elements not written, {int((~torch.isnan(got) & skip).sum())} written outside the target"
    got, ref, bar = got[~skip], ref[~skip], bar[~skip]
    assert torch.isfinite(got).all(), f"{what}: {int((~torch.isfinite(got)).sum())} non-finite outputs"
    ratio = (got - ref).abs() / bar
    worst = ratio.max().item() if ratio.numel() else 0.0
    _WORST[kernel] = max(_WORST.get(kernel, 0.0), worst)
    if worst > 1.0:
        i = int(ratio.argmax())
        raise AssertionError(f"{what}: {int((ratio > 1.0).sum())} of {ratio.numel()} elements over the bar; worst: got "
                             f"{got[i].item():.9g}, ref {ref[i].item():.9g}, bar {bar[i].item():.3g} ({worst:.1f}x)")
    return worst


def _call(fn, *args):
    L.check(getattr(L.load(), fn)(*args, stream()), fn)


def _id(prefix, case):
    return prefix + "-".join(str(c) for c in case)


def _gelu_prop(v, e):
    """GELU of a value v known within e, as f32_act computes it (0.5f * v * (1 + erff(v * 0.70710678f))): the float64
    GELU and the bar.  The input error is carried through sup|GELU'|; the product v * c rounds (u) with c itself within u
    of 1/sqrt(2), moving erf by erf'(z) 2u |z|; erff adds 4u (its value is at most 1), 1 + erf one rounding of at most 2,
    and the final product one rounding of the result."""
    z = v / math.sqrt(2.0)
    g = 0.5 * v * (1 + torch.erf(z))
    derf = 2 / math.sqrt(math.pi) * torch.exp(-z * z)
    return g, GELU_SLOPE * e + 0.5 * v.abs() * (derf * 2 * U * z.abs() + 6 * U) + U * g.abs()


# ============================================================================================ case tables
# The launches of build_plan_fp32 for dinounet_s/b/l at (B=2, S=512) must all appear here (test_plan_shapes_are_covered),
# beside cases at other sizes and on both sides of the kernels' branches.
VIT = ((384, 6), (768, 12), (1024, 16))     # (D, heads) of dinounet_s / b / l; head_dim 64
B2, NTOK, NPATCH, LQ = 2, 1029, 1024, 5376
FAPM = ((32, 128), (64, 64), (128, 32), (256, 16))                   # (channels, side) of the FAPM scales at 512^2
R = cfg.FAPM_RANK
FEATS = (32, 64, 128, 256)


def _cpad(c):
    return (c + 63) // 64 * 64


def G(name, M, N, K, *, lda=None, ldw=None, ldc=None, bias=True, scale=False, shift=False, act1=0, act2=0, res=False,
      rows=None, a_rows=None, ps=None, col_off=0, conv=None):
    """One b2u_f32_gemm case.  conv = (stride, B, H, C): the 3x3 / pad 1 window of a [B, H, H, C] NHWC image, K = 9 Cpad."""
    if conv is not None:
        K = 9 * _cpad(conv[3])
    return dict(name=name, M=M, N=N, K=K, lda=lda or (conv[3] if conv else K), ldw=ldw or K,
                ldc=ldc or (ps[0] if ps else N), bias=bias, scale=scale, shift=shift, act1=act1, act2=act2, res=res,
                rows=rows, a_rows=a_rows, ps=ps, col_off=col_off, conv=conv)


GELU, RELU = L.ACT_GELU, L.ACT_RELU
GEMM_TABLE = []
for _D, _ in VIT:
    GEMM_TABLE += [
        G(f"patch_embed-D{_D}", B2 * NPATCH, _D, 768, rows=(NPATCH, NTOK, 5)),
        G(f"qkv-D{_D}", B2 * NTOK, 3 * _D, _D),
        G(f"proj-D{_D}", B2 * NTOK, _D, _D, scale=True, res=True),
        G(f"fc1-D{_D}", B2 * NTOK, 4 * _D, _D, act1=GELU),
        G(f"fc2-D{_D}", B2 * NTOK, _D, 4 * _D, scale=True, res=True),
        G(f"spm.fc1-D{_D}", B2 * 128 * 128, _D, 64),
        G(f"spm.fc2-D{_D}", B2 * 4096, _D, 128, shift=True, rows=(4096, LQ, 0)),
        G(f"spm.fc3-D{_D}", B2 * 1024, _D, 256, shift=True, rows=(1024, LQ, 4096)),
        G(f"spm.fc4-D{_D}", B2 * 256, _D, 256, shift=True, rows=(256, LQ, 5120)),
        G(f"offaw-D{_D}", B2 * LQ, 192, _D),
        G(f"outproj-D{_D}", B2 * LQ, _D, _D // 2, res=True),
        G(f"ffn2-D{_D}", B2 * LQ, _D, _D // 4, res=True),
        G(f"up-D{_D}", B2 * 4096, 4 * _D, _D, a_rows=(4096, LQ, 0), ps=(_D, 64, 64), res=True),
        G(f"bases-D{_D}", B2 * 128 * 128, 2 * R, _D),
    ]
GEMM_TABLE += [
    G("stem0", B2 * 256 * 256, 64, 0, bias=False, scale=True, shift=True, act2=RELU, conv=(2, B2, 512, 3)),
    G("stem3", B2 * 256 * 256, 64, 0, bias=False, scale=True, shift=True, act2=RELU, conv=(1, B2, 256, 64)),
    G("conv2", B2 * 64 * 64, 128, 0, bias=False, scale=True, shift=True, act2=RELU, conv=(2, B2, 128, 64)),
    G("conv3", B2 * 32 * 32, 256, 0, bias=False, scale=True, shift=True, act2=RELU, conv=(2, B2, 64, 128)),
    G("conv4", B2 * 16 * 16, 256, 0, bias=False, scale=True, shift=True, act2=RELU, conv=(2, B2, 32, 256)),
    G("film_gen", B2 * 64 * 64, 2 * R, R),
]
for _i, (_oc, _r) in enumerate(FAPM):
    GEMM_TABLE += [G(f"reduce_sc-{_oc}", B2 * _r * _r, 2 * _oc if _oc != R else _oc, R),
                   G(f"ups{_i}.a", B2 * _r * _r, 4 * _oc, _oc, ps=(_oc, _r, _r)),
                   G(f"ups{_i}.b", 4 * B2 * _r * _r, 4 * _oc, _oc, ps=(_oc, 2 * _r, 2 * _r),
                     col_off=_oc if _i < 3 else 0, ldc=2 * _oc if _i < 3 else _oc)]
for _s in range(3):
    _skip, _rlo, _below = FEATS[2 - _s], 64 << _s, FEATS[3 - _s]
    GEMM_TABLE += [G(f"d{_s}.transp", B2 * _rlo * _rlo, 4 * _skip, _below, ps=(_skip, _rlo, _rlo), ldc=2 * _skip),
                   G(f"d{_s}.conv0", B2 * 4 * _rlo * _rlo, _skip, 0, conv=(1, B2, 2 * _rlo, 2 * _skip)),
                   G(f"d{_s}.conv1", B2 * 4 * _rlo * _rlo, _skip, 0, conv=(1, B2, 2 * _rlo, _skip))]
GEMM_TABLE += [
    G("seg-2cls", B2 * 512 * 512, 2, 32),
    # sizes off the 128 x 128 x 8 tile, leading dimensions that are not multiples of 4 (the scalar-load paths)
    G("plain-odd", 257, 129, 31, lda=33, ldw=35, bias=False),
    G("gelu-odd", 130, 200, 77, ldw=79, act1=GELU),
    G("lscale-odd", 300, 70, 45, lda=47, scale=True, res=True),
    G("all-odd", 129, 131, 13, lda=13, ldw=15, scale=True, shift=True, act1=GELU, act2=RELU, res=True),
    G("rows-odd", 3 * 37, 70, 45, lda=45, shift=True, rows=(37, 50, 6)),
    G("up-odd", 2 * 36, 4 * 20, 33, lda=35, a_rows=(36, 53, 9), ps=(20, 6, 6), res=True),
    G("ps-col-odd", 3 * 25, 4 * 20, 20, ps=(20, 5, 5), col_off=20, ldc=40),
    G("conv-odd", 3 * 10 * 10, 33, 0, conv=(1, 3, 10, 20)),
    G("stem0-S96", 48 * 48, 64, 0, bias=False, scale=True, shift=True, act2=RELU, conv=(2, 1, 96, 3)),
    G("conv4-S160", 5 * 5, 256, 0, bias=False, scale=True, shift=True, act2=RELU, conv=(2, 1, 10, 256)),
    G("spm.fc4-S160", 25, 384, 256, shift=True, rows=(25, 525, 500)),
    G("up-S160", 400, 4 * 384, 384, a_rows=(400, 525, 0), ps=(384, 20, 20), res=True),
] + [G(f"seg-{_n}cls", 3 * 1000 + 7, _n, 32) for _n in (3, 5, 117)]


def _sig_case(c):
    """Which epilogue / addressing features a case sets, in the form _sig_params reads from a parameter block."""
    s = [k for k in ("bias", "scale", "shift", "res") if c[k]]
    s += [f"act1={c['act1']}"] if c["act1"] else []
    s += [f"act2={c['act2']}"] if c["act2"] else []
    s += [k for k in ("rows", "a_rows", "ps", "col_off", "conv") if c[k]]
    return tuple(s)


def _sig_params(p):
    s = [k for k, f in (("bias", p.bias), ("scale", p.scale), ("shift", p.shift), ("res", p.residual)) if f]
    s += [f"act1={p.act1}"] if p.act1 else []
    s += [f"act2={p.act2}"] if p.act2 else []
    s += [k for k, f in (("rows", p.rows_in > 0), ("a_rows", p.a_rows_in > 0), ("ps", p.ps_cout > 0),
                         ("col_off", p.col_off), ("conv", p.conv)) if f]
    return tuple(s)


# (D, rows, in rows per image, out rows per image, in row offset)
LN_TABLE = []
for _D, _ in VIT:
    LN_TABLE += [(_D, B2 * NTOK, 0, 0, 0), (_D, B2 * NPATCH, NTOK, NPATCH, 5), (_D, B2 * LQ, 0, 0, 0), (_D, B2 * NPATCH, 0, 0, 0)]
LN_TABLE += [(384, 3 * 100, 105, 100, 5), (80, 3 * 7, 13, 7, 2), (200, 33, 0, 0, 0)]
# (B, N, heads, hd, tables, q scale): tables "eng" = the engine's RoPE tables, "scaled" = per-block rescaled tables,
# "rand" = random-angle tables (the head dims no variant has); N = P + 5 for S = 96, 160, 512, 1248
ATTN_TABLE = [(B2, NTOK, _h, 64, "eng", 1.0) for _, _h in VIT] + [
    (1, 41, 2, 64, "eng", 1.0), (3, 105, 4, 64, "eng", 1.0), (2, 201, 3, 64, "eng", 1.0), (B2, NTOK, 6, 64, "scaled", 1.0),
    (1, 105, 2, 64, "eng", 8.0), (2, NTOK, 2, 128, "rand", 1.0), (3, 105, 3, 80, "rand", 1.0), (1, 54, 1, 48, "rand", 1.0),
    (1, 6089, 2, 64, "eng", 1.0)]
# (B, Hv, dh): Hv = S / 16, dh = D / 32
MSDA_TABLE = [(B2, 32, _D // 32) for _D, _ in VIT] + [(2, 6, 12), (1, 10, 24), (1, 14, 32), (3, 10, 12)]
PATCHIFY_TABLE = [(_b, _s) for _b in (1, 2, 3) for _s in (64, 96, 512)]           # (B, S)
NHWC_TABLE = [(_b, 3, _s * _s) for _b, _s in PATCHIFY_TABLE]                       # (B, C, HW)
MAXPOOL_TABLE = [(B2, 256, 256, 64), (1, 48, 48, 64), (3, 10, 14, 64)]             # (B, H, W, C)
# (B, H, W, C, planes, act): the ConvFFN pyramid (H = S / 16, coarse plane H / 2) and the FAPM refinement convs
DW_TABLE = ([(B2, 32, 32, _D // 4, 3, GELU) for _D, _ in VIT] + [(B2, 6, 6, 96, 3, GELU), (1, 10, 10, 192, 3, GELU),
                                                                   (2, 14, 14, 256, 3, GELU)]
            + [(B2, _r, _r, _c, 1, L.ACT_NONE) for _c, _r in FAPM] + [(1, 5, 5, 64, 1, L.ACT_NONE)])
# (B, base rows per image, base row offset, r, h, D): tail1 on the ConvT output, tail2..4 on the query stream's levels
TAIL_TABLE = []
for _D, _ in VIT:
    TAIL_TABLE += [(B2, 128 * 128, 0, 128, 32, _D), (B2, LQ, 0, 64, 32, _D), (B2, LQ, 4096, 32, 32, _D), (B2, LQ, 5120, 16, 32, _D)]
TAIL_TABLE += [(1, 40 * 40, 0, 40, 10, 384), (1, 525, 0, 20, 10, 384), (3, 525, 400, 10, 10, 96), (1, 525, 500, 5, 10, 384)]
FILM_TABLE = [(B2 * _r * _r, R) for _, _r in FAPM] + [(7, 24)]                    # (rows, R)
# (B, HW, C, ld_in, ld_out): FAPM in1 reads the strided RS buffer (ld_in = 2C), in2 and the decoder a dense one; HW picks
# 1 / 8 / 32 row splits (< 4096, < 65536, more)
IN_TABLE = ([(B2, _r * _r, _c, 2 * _c if _c != R else _c, _c) for _c, _r in FAPM] + [(B2, _r * _r, _c, _c, _c) for _c, _r in FAPM]
            + [(B2, 128 * 128, 128, 128, 128), (B2, 256 * 256, 64, 64, 64), (B2, 512 * 512, 32, 32, 32)]
            + [(3, 4095, 48, 96, 48), (1, 65535, 40, 80, 40), (2, 100, 256, 256, 256)])
SE_TABLE = [(B2, _r * _r, _c, max(1, _c // 16), 2 * _c if _c != R else R) for _c, _r in FAPM] + [(3, 100, 80, 5, 160)]
SEG_OUT_TABLE = [(B2, 512 * 512, 2)] + [(2, 4099, _n) for _n in (1, 2, 3, 5, 20, 117, 128, 255, 256)]   # (B, HW, ncls)


# ============================================================================================ 1. GEMM epilogues
def _gemm_out_rows(c):
    M = c["M"]
    if c["rows"]:
        rin, rout, _ = c["rows"]
        return M // rin * rout
    if c["ps"]:
        return 4 * M
    return M


def _gemm_targets(c):
    """Output row [M, N] and column [N] of every product element, as the kernel's epilogue places it."""
    M, N = c["M"], c["N"]
    m = torch.arange(M, device=DEV)
    n = torch.arange(N, device=DEV)
    oc = n.clone()
    qoff = torch.zeros_like(n)
    if c["ps"]:
        cout, h, w = c["ps"]
        pb, rem = m // (h * w), m % (h * w)
        orow = (pb * 2 * h + 2 * (rem // w)) * (2 * w) + 2 * (rem % w)
        q = n // cout
        oc, qoff = n % cout, (q >> 1) * (2 * w) + (q & 1)
    elif c["rows"]:
        rin, rout, off = c["rows"]
        orow = (m // rin) * rout + off + m % rin
    else:
        orow = m
    return orow[:, None] + qoff[None, :], oc + c["col_off"]


@pytest.mark.parametrize("c", GEMM_TABLE, ids=lambda c: f"{c['name']}-{c['M']}x{c['N']}x{c['K']}")
def test_gemm_epilogue(c):
    """b2u_f32_gemm: acc = A W^T, then bias, act1, scale, shift, act2, residual, placed by the row remap, the 2x2 pixel
    shuffle and the column offset.  A is read through the a_rows remap or the 3x3 window of an NHWC image (the window's
    padded channels c >= C multiply finite junk weights, which must count as 0).  Columns of A and W past K, rows of A the
    remap skips and the skipped input rows hold NaN: a kernel that reads them fails.

    Bar: each output is one fmaf chain over k (depth K), within (K + 1) u sum_k |a w|; the bias add rounds once (u |v|);
    GELU as in _gelu_prop; the scale multiplies the error by |scale| and rounds once; shift and residual adds round once
    each; ReLU is 1-Lipschitz."""
    M, N, K = c["M"], c["N"], c["K"]
    seed = M + 7 * N + K
    W = _randn((N, c["ldw"]), seed + 1, K ** -0.5)
    W[:, K:] = float("nan")
    if c["conv"]:
        stride, B, H, Cc = c["conv"]
        cpad = K // 9
        W.view(N, 9, cpad)[:, :, Cc:] = 3.0                       # padded channels: finite junk the window must zero
        A = _randn((B * H * H, Cc), seed, 1.0, 0.2)
    else:
        if c["a_rows"]:
            ain, aout, aoff = c["a_rows"]
            A = _randn((M // ain, aout, c["lda"]), seed, 1.0, 0.2)
            A[:, :aoff] = float("nan")
            A[:, aoff + ain:] = float("nan")
            A = A.view(-1, c["lda"])
        else:
            A = _randn((M, c["lda"]), seed, 1.0, 0.2)
        A[:, K:] = float("nan")
    out_rows = _gemm_out_rows(c)
    out = _nan((out_rows, c["ldc"]))
    vec = lambda s, sc=1.0, sh=0.0: _randn(N, seed + s, sc, sh)
    bias = vec(2, 0.5) if c["bias"] else None
    scale = vec(3, 0.5, 1.0) if c["scale"] else None
    shift = vec(4, 0.5) if c["shift"] else None
    res = _randn((out_rows, c["ldc"]), seed + 5) if c["res"] else None
    p = L.F32GemmParams()
    p.M, p.N, p.K, p.A, p.lda, p.W, p.ldw = M, N, K, P(A), c["lda"], P(W), c["ldw"]
    p.out, p.ldc, p.col_off = P(out), c["ldc"], c["col_off"]
    p.bias, p.scale, p.shift, p.act1, p.act2 = P(bias), P(scale), P(shift), c["act1"], c["act2"]
    if res is not None:
        p.residual, p.ldres = P(res), c["ldc"]
    if c["rows"]:
        p.rows_in, p.rows_out, p.row_off = c["rows"]
    if c["a_rows"]:
        p.a_rows_in, p.a_rows_out, p.a_row_off = c["a_rows"]
    if c["ps"]:
        p.ps_cout, p.ps_h, p.ps_w = c["ps"]
    if c["conv"]:
        p.conv = L.CONV3X3_S2 if stride == 2 else L.CONV3X3_S1
        p.Hin, p.Win, p.C, p.Cpad = H, H, Cc, cpad
    L.check(L.load().b2u_f32_gemm(C.byref(p), stream()), "b2u_f32_gemm")
    torch.cuda.synchronize()

    Wd = W[:, :K].double()
    if c["conv"]:
        xi = A.double().view(B, H, H, Cc).permute(0, 3, 1, 2)
        w4 = Wd.view(N, 3, 3, cpad)[..., :Cc].permute(0, 3, 1, 2)
        acc = F.conv2d(xi, w4, stride=stride, padding=1).permute(0, 2, 3, 1).reshape(M, N)
        mag = F.conv2d(xi.abs(), w4.abs(), stride=stride, padding=1).permute(0, 2, 3, 1).reshape(M, N)
    else:
        if c["a_rows"]:
            Ar = A.view(M // ain, aout, -1)[:, aoff:aoff + ain].reshape(M, -1)[:, :K].double()
        else:
            Ar = A[:, :K].double()
        acc, mag = Ar @ Wd.t(), Ar.abs() @ Wd.abs().t()
    v, e = acc, (K + 1) * U * mag
    if bias is not None:
        v = v + bias.double()
        e = e + U * v.abs()
    if c["act1"] == GELU:
        v, e = _gelu_prop(v, e)
    if scale is not None:
        e = scale.double().abs() * e
        v = v * scale.double()
        e = e + U * v.abs()
    if shift is not None:
        v = v + shift.double()
        e = e + U * v.abs()
    if c["act2"] == RELU:
        v = F.relu(v)
    rr, cc = _gemm_targets(c)
    cc = cc[None, :].expand(M, N)
    if res is not None:
        v = v + res.double()[rr, cc]
        e = e + U * v.abs()
    ref, bar = _nan((out_rows, c["ldc"]), torch.float64), torch.ones((out_rows, c["ldc"]), dtype=torch.float64, device=DEV)
    ref[rr, cc], bar[rr, cc] = v, e
    _check("f32_gemm", f"gemm {c['name']}", out, ref, bar)


# ============================================================================================ 2. attention
@pytest.fixture(scope="module")
def eng_s():
    from dinounet_b200.engine import ForwardEngine
    eng = ForwardEngine("dinounet_s", O.make_state_dict("dinounet_s", 2, seed=0), 2, torch.device(DEV), precision="fp32")
    yield eng
    del eng
    torch.cuda.empty_cache()


def _attn_tables(kind, h, hd, eng, keep):
    """(sin, cos) [P, hd] fp32 tables and the pointers the launch gets."""
    if kind == "eng":
        sin, cos = eng._rope_tables(h, h)
        return sin, cos, P(sin), P(cos)
    if kind == "scaled":
        # per-block tables filled by b2u_rope_tables from rescaled coordinates; block 1's slice, as scaled_vit_plan hands it
        # to _patch_attention_rope
        periods = eng.w["periods"].to(DEV).float().contiguous()
        scales = torch.tensor([0.75, 1.3], device=DEV)
        sin = torch.empty((2, h * h, hd), device=DEV)
        cos = torch.empty_like(sin)
        _call("b2u_rope_tables", P(periods), P(scales), P(sin), P(cos), 2, h, h, hd)
        keep += [periods, scales, sin, cos]
        return sin[1], cos[1], P(sin[1]), P(cos[1])
    ang = (torch.rand((h * h, hd // 2), generator=_gen(hd), device=DEV) * 2 - 1) * math.pi
    ang = ang.tile(2)
    sin, cos = torch.sin(ang), torch.cos(ang)
    return sin, cos, P(sin), P(cos)


@pytest.mark.parametrize("case", ATTN_TABLE, ids=lambda c: _id("B-N-heads-hd-tables-qscale=", c))
def test_attention(case, eng_s):
    """b2u_f32_attention: RoPE on q and k while loading them (x cos + rotate_half(x) sin on tokens >= 5, the prefix
    tokens unrotated), softmax(q k^T scale) v per head, blocks of 8 query rows (N = P + 5 leaves the last block partial).
    The reference rotates in float64 from the same fp32 tables, then runs float64 attention.  N = 6089 (S = 1248) is the
    largest token count a plan can have whose score rows fit the 200 KB of shared memory.

    Bar: a rotated element is within e_x = 2u (|x cos| + |rot(x) sin|).  A score is a chain of hd / 32 fmas per lane and
    five shuffle adds (depth k = ceil(hd/32) + 5), so a logit L is within E = scale (k u sum|q k| + sum e_q |k| + |q| e_k)
    + u |L|.  The shifted exponent of key j is then within E_j + max E + u |L_j - max L|, expf adds 4u: relative error eps_j
    of p_j.  The row sum l (N/32 serial adds per lane, five shuffles) is within sum_j P_j eps_j + (N/32 + 5) u relative,
    and sum_j p_j v_j is an N-deep fma chain; so |out - ref| <= sum_j P_j |v_j| (eps_j + eps_l + N u) + u |out|."""
    B, N, heads, hd, kind, qscale = case
    npre = cfg.N_PREFIX
    Pn = N - npre
    h = int(round(math.sqrt(Pn)))
    assert h * h == Pn
    keep = []
    sin, cos, psin, pcos = _attn_tables(kind, h, hd, eng_s, keep)
    D = heads * hd
    qkv = _randn((B * N, 3 * D), N + hd + heads)
    qkv[:, :D] *= qscale
    out = _nan((B * N, D))
    scale = hd ** -0.5
    args = (P(qkv), psin, pcos, P(out), B, N, heads, hd, npre, scale)
    if kind == "scaled":
        from dinounet_b200.engine_fp32 import _patch_attention_rope
        args = _patch_attention_rope((P(qkv), 0, 0) + args[3:], psin, pcos, keep)
    _call("b2u_f32_attention", *args)
    torch.cuda.synchronize()

    t = qkv.double().view(B, N, 3, heads, hd).permute(2, 0, 3, 1, 4)       # [3, B, heads, N, hd]
    s64, c64 = sin.double(), cos.double()

    def rope(x):
        rh = torch.cat([-x[..., hd // 2:], x[..., :hd // 2]], -1)
        xr, ex = x.clone(), torch.zeros_like(x)
        xr[..., npre:, :] = x[..., npre:, :] * c64 + rh[..., npre:, :] * s64
        ex[..., npre:, :] = 2 * U * ((x[..., npre:, :] * c64).abs() + (rh[..., npre:, :] * s64).abs())
        return xr, ex

    (q, eq), (k, ek), v = rope(t[0]), rope(t[1]), t[2]
    sc = float(np.float32(scale))
    depth = -(-hd // 32) + 5
    Lg = q @ k.transpose(-1, -2) * sc
    E = sc * (depth * U * (q.abs() @ k.abs().transpose(-1, -2)) + eq @ k.abs().transpose(-1, -2)
              + q.abs() @ ek.transpose(-1, -2)) + U * Lg.abs()
    mx = Lg.amax(-1, keepdim=True)
    Pm = torch.softmax(Lg, -1)
    eps = E + E.amax(-1, keepdim=True) + U * (Lg - mx).abs() + 4 * U
    del E, Lg
    eps_l = (Pm * eps).sum(-1, keepdim=True) + (-(-N // 32) + 5) * U
    ref = Pm @ v
    bar = (Pm * (eps + eps_l + N * U)) @ v.abs() + U * ref.abs()
    del Pm, eps
    got = out.view(B, N, heads, hd).permute(0, 2, 1, 3)
    _check("f32_attention", f"attention{case}", got, ref, bar)
    if qscale > 1:
        _NOTES.append(f"attention q x{qscale:g}: logits span {float((q @ k.transpose(-1, -2) * sc).std()):.1f} (std)")


def test_attention_rejects_rows_over_shared_memory():
    """One step above the largest plan size (S = 1280, N = 6405): the score rows need more than 200 KB of shared memory,
    so the entry point returns an error without launching, and the output stays unwritten."""
    B, N, heads, hd = 1, 6405, 1, 64
    qkv = _randn((B * N, 3 * heads * hd), 3)
    tab = torch.zeros((N - 5, hd), device=DEV)
    out = _nan((B * N, heads * hd))
    lib = L.load()
    n0 = L.launch_count()
    rc = lib.b2u_f32_attention(P(qkv), P(tab), P(tab), P(out), B, N, heads, hd, 5, hd ** -0.5, stream())
    torch.cuda.synchronize()
    assert rc != 0, "N = 6405 was accepted"
    assert L.launch_count() == n0, "a kernel was launched"
    assert torch.isnan(out).all()


# ============================================================================================ 3. MSDA
def _msda_ref_points(Hv):
    pts = []
    for g in (2 * Hv, Hv, Hv // 2):
        c = (torch.arange(g, dtype=torch.float64, device=DEV) + 0.5) / g
        yy, xx = torch.meshgrid(c, c, indexing="ij")
        pts.append(torch.stack([xx.reshape(-1), yy.reshape(-1)], -1))
    return torch.cat(pts, 0)


@pytest.mark.parametrize("case", MSDA_TABLE, ids=lambda c: _id("B-Hv-dh=", c))
def test_msda(case):
    """b2u_f32_msda (16 heads x 4 points over the 2Hv, Hv and Hv/2 query grids; Hv = 6 / 10 / 14 make the coarse grid
    odd) against float64 O.msda_core on the float64 locations (reference point + fp32 offset / Hv) and the float64 softmax
    of the fp32 logits.  Head 0 samples exactly at pixel -1 and Hv (the zero-padding edges), head 1 exactly on integer
    pixels, point 2 of head 2 and point 3 of head 3 lie 1000 pixels outside the map, the rest are N(0, 3) pixels away.
    Logits are uniform in +-30, so the softmax needs its max subtraction.

    Bar: a location is within 4u (4 Hv + 2|offset|) pixels (the same steps as the 16-bit kernel), moving a sample by at
    most 2 max|v| per pixel.  The weight of point j: a_j - max rounds (u |a_j - max|), expf adds 4u, so e_j is within
    eps_j = (4 + |a_j - max|) u relative; the sum of four is within max eps + 3u and the division adds u.  The bilinear
    corner weights and the four-term sum take 8u, the weighted accumulation 8u more:
    sum_j w_j (eps_j + max eps + 20u) sum_c w_c |v_c| plus the location term."""
    B, Hv, dh = case
    heads = cfg.DEFORM_HEADS
    HW = Hv * Hv
    Lq = 21 * HW // 4
    value = _randn((B, HW, heads, dh), Hv + dh)
    off = _randn((B, Lq, heads, 4, 2), Hv + dh + 1, 3.0)
    logits = (torch.rand((B, Lq, heads, 4), generator=_gen(Hv + dh + 2), device=DEV) * 2 - 1) * 30
    ref_pts = _msda_ref_points(Hv)
    rx, ry = ref_pts[:, 0], ref_pts[:, 1]
    # pixel = ref * Hv + off - 0.5: -1 and Hv on both axes (points 0 / 1 of head 0)
    off[:, :, 0, 0, 0], off[:, :, 0, 0, 1] = (-0.5 - rx * Hv).float(), (-0.5 - ry * Hv).float()
    off[:, :, 0, 1, 0], off[:, :, 0, 1, 1] = (Hv + 0.5 - rx * Hv).float(), (Hv + 0.5 - ry * Hv).float()
    ix = torch.randint(-1, Hv + 1, (B, Lq, 4, 2), generator=_gen(Hv + dh + 3), device=DEV).double()
    off[:, :, 1, :, 0] = (ix[..., 0] + 0.5 - rx[None, :, None] * Hv).float()
    off[:, :, 1, :, 1] = (ix[..., 1] + 0.5 - ry[None, :, None] * Hv).float()
    off[:, :, 2, 2] = 1000.0
    off[:, :, 3, 3] = -1000.0
    offaw = torch.cat([off.reshape(B * Lq, heads * 8), logits.reshape(B * Lq, heads * 4)], 1).contiguous()
    out = _nan((B * Lq, heads * dh))
    _call("b2u_f32_msda", P(value), P(offaw), P(out), B, Hv, Hv, heads, dh)
    torch.cuda.synchronize()
    offd = off.double()
    loc = ref_pts[None, :, None, None, None, :] + offd.view(B, Lq, heads, 1, 4, 2) / Hv
    lg = logits.double()
    aw = F.softmax(lg, -1)
    eps = (4 + (lg - lg.amax(-1, keepdim=True)).abs()) * U
    wb = aw * (eps + eps.amax(-1, keepdim=True) + 20 * U)
    v64 = value.double()
    ref = O.msda_core(v64, [(Hv, Hv)], loc, aw.view(B, Lq, heads, 1, 4))
    sabs = O.msda_core(v64.abs(), [(Hv, Hv)], loc, wb.view(B, Lq, heads, 1, 4))
    loc_px = 4 * U * (4 * Hv + 2 * offd.abs().sum(-1))
    loc_term = (aw * loc_px).sum(-1) * 2 * v64.abs().max()
    bar = sabs + loc_term.repeat_interleave(dh, -1)
    _check("f32_msda", f"msda{case}", out.view(B, Lq, heads * dh), ref, bar)


# ============================================================================================ 4. input reshapes
@pytest.mark.parametrize("case", PATCHIFY_TABLE, ids=lambda c: _id("B-S=", c))
def test_patchify_and_nhwc(case):
    """b2u_f32_patchify == F.unfold(x, 16, stride=16) and b2u_f32_nchw_to_nhwc == permute, bit for bit."""
    B, S = case
    x = _randn((B, 3, S, S), S + B, 2.0)
    out = _nan((B * (S // 16) ** 2, 768))
    _call("b2u_f32_patchify", P(x), P(out), B, S)
    xh = _nan((B * S * S, 3))
    _call("b2u_f32_nchw_to_nhwc", P(x), P(xh), B, 3, S * S)
    torch.cuda.synchronize()
    assert torch.equal(out, F.unfold(x, 16, stride=16).transpose(1, 2).reshape(-1, 768))
    assert torch.equal(xh, x.permute(0, 2, 3, 1).reshape(-1, 3))


@pytest.mark.parametrize("case", MAXPOOL_TABLE, ids=lambda c: _id("B-H-W-C=", c))
def test_maxpool(case):
    """b2u_f32_maxpool3x3s2 == F.max_pool2d(3, 2, 1) bit for bit, with all-negative windows at the padding."""
    B, H, W, Cc = case
    x = _randn((B, H, W, Cc), H + Cc)
    x[:, :5, :5] = -x[:, :5, :5].abs() - 0.01
    out = _nan((B, H // 2, W // 2, Cc))
    _call("b2u_f32_maxpool3x3s2", P(x), P(out), B, H, W, Cc)
    torch.cuda.synchronize()
    assert torch.equal(out, F.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1))


# ============================================================================================ 5. seg output
@pytest.mark.parametrize("case", SEG_OUT_TABLE, ids=lambda c: _id("B-HW-ncls=", c))
def test_seg_out(case):
    """b2u_f32_seg_out: lin [B*HW, ncls] -> logits NCHW bit for bit, labels = the first maximum.  Logits are multiples of
    0.5 in [-2, 2], so ties are everywhere; every 7th pixel has all classes equal (label 0) and the pixels 3 after those
    have their maximum at the last two classes (label ncls - 2)."""
    B, HW, ncls = case
    g = _gen(ncls + HW)
    lin = torch.randint(-4, 5, (B * HW, ncls), generator=g, device=DEV).float() * 0.5
    lin[::7] = 1.0
    if ncls >= 2:
        lin[3::7, -2:] = 3.0
    logits = _nan((B, ncls, HW))
    labels = torch.full((B * HW,), 77, dtype=torch.uint8, device=DEV)
    _call("b2u_f32_seg_out", P(lin), P(logits), P(labels), B, HW, ncls)
    torch.cuda.synchronize()
    assert torch.equal(logits, lin.view(B, HW, ncls).permute(0, 2, 1))
    first = (lin == lin.amax(1, keepdim=True)).int().argmax(1)              # index of the first maximum
    assert torch.equal(labels.long(), first)
    assert (labels[::7] == 0).all()
    if ncls >= 2:
        assert (labels[3::7] == ncls - 2).all()


@pytest.mark.parametrize("ncls", [0, 257, 1000])
def test_seg_out_rejects_class_counts_labels_cannot_hold(ncls):
    """uint8 labels hold classes 0..255: ncls outside 1..256 returns an error, launches nothing and writes nothing."""
    lin = _randn((16, max(ncls, 1)), 1)
    labels = torch.full((16,), 77, dtype=torch.uint8, device=DEV)
    logits = _nan((1, max(ncls, 1), 16))
    n0 = L.launch_count()
    rc = L.load().b2u_f32_seg_out(P(lin), P(logits), P(labels), 1, 16, ncls, stream())
    torch.cuda.synchronize()
    assert rc != 0 and L.launch_count() == n0
    assert (labels == 77).all() and torch.isnan(logits).all()


# ============================================================================================ 6. plan-only modes
@pytest.mark.parametrize("case", LN_TABLE, ids=lambda c: _id("D-rows-rin-rout-off=", c))
def test_layernorm(case):
    """b2u_f32_layernorm, optionally with the tap remap (output row r reads row (r / rout) rin + off + r % rout: the patch
    rows of each image).  Rows have |mean| up to ~30x their std; rows the remap skips hold NaN.

    Bar: each lane sums D/32 elements serially, then five shuffles: depth k = D/32 + 5, so the mean is within
    e_m = (k + 1) u mean|x|.  The centred square sum is within (k + 3) u of itself plus D e_m^2; sqrtf, the division and
    1/x give rstd a relative error eps_r = (k + 3) u / 2 + 4u + e_m^2 / (2 (var + eps)).  Then
    |y - ref| <= |g| rstd (e_m + |x - mean| eps_r) + 4u (|g x_hat| + |b|)."""
    D, rows, rin, rout, off = case
    nimg = rows // rout if rout else 1
    n_in = nimg * rin if rout else rows
    g0 = _gen(D + rows)
    mu = torch.randn(n_in, 1, generator=g0, device=DEV) * 10
    sd = torch.exp(torch.randn(n_in, 1, generator=g0, device=DEV) * 0.7)
    x = mu + sd * torch.randn(n_in, D, generator=g0, device=DEV)
    if rout:
        xv = x.view(nimg, rin, D)
        xv[:, :off] = float("nan")
        xv[:, off + rout:] = float("nan")
        xs = xv[:, off:off + rout].reshape(rows, D)
    else:
        xs = x
    w, b = _randn(D, 1, 0.3, 1.0), _randn(D, 2, 0.5)
    eps = cfg.LN_EPS_VIT
    out = _nan((rows + 3, D))
    _call("b2u_f32_layernorm", P(x), P(out), P(w), P(b), rows, D, eps, rin, rout, off)
    torch.cuda.synchronize()
    xd = xs.double()
    mean = xd.mean(-1, keepdim=True)
    xc = xd - mean
    var = (xc * xc).mean(-1, keepdim=True)
    rstd = (var + float(np.float32(eps))).rsqrt()
    ref = xc * rstd * w.double() + b.double()
    k = -(-D // 32) + 5
    e_m = (k + 1) * U * xd.abs().mean(-1, keepdim=True)
    eps_r = (k + 3) * U / 2 + 4 * U + e_m ** 2 / (2 * (var + eps))
    bar = w.double().abs() * rstd * (e_m + xc.abs() * eps_r) + 4 * U * ((xc * rstd * w.double()).abs() + b.double().abs())
    ref = torch.cat([ref, _nan((3, D), torch.float64)])
    bar = torch.cat([bar, torch.ones((3, D), dtype=torch.float64, device=DEV)])
    _check("f32_layernorm", f"layernorm{case}", out, ref, bar)


@pytest.mark.parametrize("case", IN_TABLE, ids=lambda c: _id("B-HW-C-ldin-ldout=", c))
def test_instnorm(case):
    """b2u_f32_instnorm + LeakyReLU(0.01f) reading C of every ld_in columns (the other columns hold |values| ~ 30 the
    statistics must not see), HW rows split over 1 / 8 / 32 blocks.  Channel means up to 8x their std.

    Bar: mean and centred square sum are float64 sums (relative error below HW 2^-53), rounded to fp32 (u); rstd takes
    four more roundings (var, + eps, sqrtf, 1/x): 4u relative.  y = (x - mean) rstd g + b rounds four times:
    |y - ref| <= |g| rstd (e_mean + 4u |x - mean|) + 4u (|g x_hat| + |b|), times 0.01 on the negative side plus one
    rounding of the slope product.  The stats output (mean, rstd) is checked against u |mean| and 4u rstd: the mean is
    a single rounding of a float64 value, so its ratio may come close to 1 without any slack being lost."""
    B, HW, Cc, ldi, ldo = case
    g0 = _gen(HW + Cc + ldi)
    mu = torch.linspace(-4, 4, Cc, device=DEV)
    sd = torch.exp(torch.linspace(-1, 1, Cc, device=DEV))[torch.randperm(Cc, generator=g0, device=DEV)]
    xb = torch.randn(B, HW, ldi, generator=g0, device=DEV) * 30
    xb[..., :Cc] = mu + sd * torch.randn(B, HW, Cc, generator=g0, device=DEV)
    w, b = _randn(Cc, Cc + 5, 0.5, 1.0), _randn(Cc, Cc + 6, 0.5)
    out = _nan((B * HW, ldo))
    work = torch.zeros(2 * B * Cc, dtype=torch.float64, device=DEV)
    stats = _nan((B, Cc, 2))
    _call("b2u_f32_instnorm", P(xb), ldi, P(out), ldo, P(w), P(b), P(work), P(stats), B, HW, Cc, cfg.IN_EPS, 1)
    torch.cuda.synchronize()
    xd = xb[..., :Cc].double()
    mean = xd.mean(1, keepdim=True)
    xc = xd - mean
    var = (xc * xc).mean(1, keepdim=True)
    rstd = (var + float(np.float32(cfg.IN_EPS))).rsqrt()
    gd, bd = w.double(), b.double()
    pre = xc * rstd * gd + bd
    e_mean = U * mean.abs() + HW * U64 * xd.abs().mean(1, keepdim=True)
    e = gd.abs() * rstd * (e_mean + 4 * U * xc.abs()) + 4 * U * ((xc * rstd * gd).abs() + bd.abs())
    ref = torch.where(pre > 0, pre, SLOPE * pre)
    neg = (pre < 0) & (pre.abs() > e)
    bar = torch.where(neg, SLOPE * e, e) + U * ref.abs()
    got = out.view(B, HW, ldo)
    ref_buf = torch.cat([ref, _nan((B, HW, ldo - Cc), torch.float64)], -1)
    bar_buf = torch.cat([bar, torch.ones((B, HW, ldo - Cc), dtype=torch.float64, device=DEV)], -1)
    _check("f32_instnorm", f"instnorm{case}", got, ref_buf, bar_buf)
    _check("f32_instnorm(stats)", f"instnorm{case} mean", stats[..., 0], mean[:, 0], e_mean[:, 0])
    _check("f32_instnorm(stats)", f"instnorm{case} rstd", stats[..., 1], rstd[:, 0], 4 * U * rstd[:, 0])


@pytest.mark.parametrize("case", TAIL_TABLE, ids=lambda c: _id("B-crows-coff-r-h-D=", c))
def test_tail(case):
    """b2u_f32_tail: (c + bilinear(tap h x h -> r x r, align_corners=False)) * sc + sh, with c a slice of r^2 rows at
    c_off inside a buffer of c_rows_per_b rows per image (the query stream Cst for tail2..4); rows outside the slice hold
    NaN.  The bilinear weights are exact in fp32 at these power-of-two ratios, so c + four weighted taps is within
    5u (|c| + sum w |tap|); the affine scales that by |sc| and adds 2u of its terms."""
    B, crows, coff, r, h, D = case
    tap = _randn((B * h * h, D), r + D)
    cs = _randn((B, crows, D), r + D + 1)
    cs[:, :coff] = float("nan")
    cs[:, coff + r * r:] = float("nan")
    sc, sh = _randn(D, 3, 0.5, 1.0), _randn(D, 4, 0.5)
    out = _nan((B * r * r, D))
    _call("b2u_f32_tail", P(cs), crows, coff, P(tap), P(out), P(sc), P(sh), B, r, h, D)
    torch.cuda.synchronize()
    t = tap.double().view(B, h, h, D).permute(0, 3, 1, 2)
    up = F.interpolate(t, size=(r, r), mode="bilinear", align_corners=False)
    up_abs = F.interpolate(t.abs(), size=(r, r), mode="bilinear", align_corners=False)
    cd = cs[:, coff:coff + r * r].double().view(B, r, r, D).permute(0, 3, 1, 2)
    scd, shd = sc.double()[None, :, None, None], sh.double()[None, :, None, None]
    pre = cd + up
    ref = pre * scd + shd
    bar = scd.abs() * 5 * U * (cd.abs() + up_abs) + 2 * U * ((pre * scd).abs() + shd.abs())
    _check("f32_tail", f"tail{case}", out.view(B, r, r, D).permute(0, 3, 1, 2), ref, bar)


@pytest.mark.parametrize("case", FILM_TABLE, ids=lambda c: _id("rows-R=", c))
def test_film(case):
    """b2u_f32_film: z = gamma * zp + beta from gb = (gamma | beta), zz = (zs | zp); 2u (|gamma zp| + |beta|)."""
    rows, Rr = case
    gb, zz = _randn((rows, 2 * Rr), rows + 1), _randn((rows, 2 * Rr), rows + 2)
    zz[:, :Rr] = float("nan")                                   # zs is not read
    z = _nan((rows, Rr))
    _call("b2u_f32_film", P(gb), P(zz), P(z), rows, Rr)
    torch.cuda.synchronize()
    g, be, zp = gb[:, :Rr].double(), gb[:, Rr:].double(), zz[:, Rr:].double()
    _check("f32_film", f"film{case}", z, g * zp + be, 2 * U * ((g * zp).abs() + be.abs()))


@pytest.mark.parametrize("case", SE_TABLE, ids=lambda c: _id("B-HW-C-hid-ldsc=", c))
def test_se(case):
    """b2u_f32_se: out = t * sigmoid(W2 relu(W1 mean_hw(t) + b1) + b2) + sc, with the shortcut read from the second half
    of a [rows, 2C] row (ldsc = 2C, the FAPM RS buffer) or from a [rows, 256] FiLM output.  Hidden unit 0 is dead.

    Bar: the float64 mean rounds to fp32 (e_p = u |p|); the hidden pre-activation is a (C + 1)-deep chain:
    e_h = (C + 1) u (|W1| |p| + |b1|) + |W1| e_p, ReLU 1-Lipschitz; the gate input a likewise
    e_a = (hid + 1) u (|W2| h + |b2|) + |W2| e_h; the gate g = 1 / (1 + expf(-a)) is within 0.25 e_a + 4u g (1 - g) + 2u g;
    out = t g + sc within |t| e_g + 2u (|t g| + |sc|)."""
    B, HW, Cc, hid, ldsc = case
    t = _randn((B * HW, Cc), HW + Cc, 1.0, 0.3)
    scb = _randn((B * HW, ldsc), HW + Cc + 1)
    if ldsc == 2 * Cc:
        scb[:, :Cc] = float("nan")                               # the reduce half is not read
        sc_ptr, sc = scb.data_ptr() + Cc * 4, scb[:, Cc:]
    else:
        sc_ptr, sc = P(scb), scb
    w1, b1 = _randn((hid, Cc), Cc + 2, 0.3), _randn(hid, Cc + 3, 0.1, 0.2)
    w2, b2 = _randn((Cc, hid), Cc + 4, 0.5), _randn(Cc, Cc + 5, 0.5)
    b1[0] = -50.0
    pooled = _nan((B, Cc))
    out = _nan((B * HW, Cc))
    _call("b2u_f32_se", P(t), sc_ptr, ldsc, P(pooled), P(w1), P(b1), P(w2), P(b2), P(out), B, HW, Cc, hid)
    torch.cuda.synchronize()
    td = t.double().view(B, HW, Cc)
    p = td.mean(1)
    W1, B1, W2, B2_ = w1.double(), b1.double(), w2.double(), b2.double()
    hdn = F.relu(p @ W1.t() + B1)
    a = hdn @ W2.t() + B2_
    gte = torch.sigmoid(a)
    e_p = U * p.abs()
    e_h = (Cc + 1) * U * (p.abs() @ W1.abs().t() + B1.abs()) + e_p @ W1.abs().t()
    e_a = (hid + 1) * U * (hdn @ W2.abs().t() + B2_.abs()) + e_h @ W2.abs().t()
    e_g = 0.25 * e_a + 4 * U * gte * (1 - gte) + 2 * U * gte
    scd = sc.double().reshape(B, HW, Cc)
    ref = td * gte[:, None] + scd
    bar = td.abs() * e_g[:, None] + 2 * U * ((td * gte[:, None]).abs() + scd.abs())
    _check("f32_se", f"se{case}", out.view(B, HW, Cc), ref, bar)


def _planes(H, W, planes):
    if planes == 1:
        return [(0, H, W)]
    return [(0, 2 * H, 2 * W), (4 * H * W, H, W), (5 * H * W, H // 2, W // 2)]


@pytest.mark.parametrize("case", DW_TABLE, ids=lambda c: _id("B-H-W-C-planes-act=", c))
def test_dwconv(case):
    """b2u_f32_dwconv3x3 per plane against a float64 depthwise conv with zero padding at each plane's own border (the
    ConvFFN pyramid 2H x 2W | H x W | H/2 x W/2 with GELU, at H = 6 / 10 / 14 an odd coarse plane, and the FAPM convs).
    Bar: nine fmas and the bias add: d = 10u (sum|w x| + |bias|); GELU as in _gelu_prop."""
    B, H, W, Cc, planes, act = case
    pl = _planes(H, W, planes)
    rows = sum(ph * pw for _, ph, pw in pl)
    x = _randn((B, rows, Cc), H + Cc + planes)
    w = _randn((Cc, 1, 3, 3), Cc + 1, 1 / 3)
    bias = _randn(Cc, Cc + 2, 0.3)
    w9 = w.reshape(Cc, 9).t().contiguous()
    out = _nan((B, rows, Cc))
    _call("b2u_f32_dwconv3x3", P(x), P(out), P(w9), P(bias), B, H, W, Cc, planes, act)
    torch.cuda.synchronize()
    for k, (r0, ph, pw) in enumerate(pl):
        t = x[:, r0:r0 + ph * pw].double().transpose(1, 2).reshape(B, Cc, ph, pw)
        conv = F.conv2d(t, w.double(), bias.double(), padding=1, groups=Cc)
        d = 10 * U * F.conv2d(t.abs(), w.double().abs(), bias.double().abs(), padding=1, groups=Cc)
        ref, bar = _gelu_prop(conv, d) if act == GELU else (conv, d)
        got = out[:, r0:r0 + ph * pw].transpose(1, 2).reshape(B, Cc, ph, pw)
        _check("f32_dwconv3x3", f"dwconv{case} plane {k} ({ph}x{pw})", got, ref, bar)


# ============================================================================================ 7. coverage guard
def _key(fname, a):
    """The shape arguments of one fp32-plan launch, as this file's tables list them."""
    if fname == "b2u_f32_layernorm":
        return "LN_TABLE", (a[5], a[4], a[7], a[8], a[9])
    if fname == "b2u_f32_attention":
        return "ATTN_TABLE", (a[4], a[5], a[6], a[7])
    if fname == "b2u_f32_msda":
        return "MSDA_TABLE", (a[3], a[4], a[7])
    if fname == "b2u_f32_patchify":
        return "PATCHIFY_TABLE", (a[2], a[3])
    if fname == "b2u_f32_nchw_to_nhwc":
        return "NHWC_TABLE", (a[2], a[3], a[4])
    if fname == "b2u_f32_maxpool3x3s2":
        return "MAXPOOL_TABLE", (a[2], a[3], a[4], a[5])
    if fname == "b2u_f32_dwconv3x3":
        return "DW_TABLE", (a[4], a[5], a[6], a[7], a[8], a[9])
    if fname == "b2u_f32_tail":
        return "TAIL_TABLE", (a[7], a[1], a[2], a[8], a[9], a[10])
    if fname == "b2u_f32_film":
        return "FILM_TABLE", (a[3], a[4])
    if fname == "b2u_f32_instnorm":
        return "IN_TABLE", (a[8], a[9], a[10], a[1], a[3])
    if fname == "b2u_f32_se":
        return "SE_TABLE", (a[9], a[10], a[11], a[12], a[2])
    if fname == "b2u_f32_seg_out":
        return "SEG_OUT_TABLE", (a[3], a[4], a[5])
    if fname == "b2u_write_prefix":                 # the 16-bit forward's kernel (test_gpu_forward_kernels.py)
        return "PREFIX_TABLE", (a[2], a[3], a[4], a[5])
    return None


def _covered():
    from tests.test_gpu_forward_kernels import PREFIX_TABLE
    return {"LN_TABLE": set(LN_TABLE), "ATTN_TABLE": {c[:4] for c in ATTN_TABLE}, "MSDA_TABLE": set(MSDA_TABLE),
            "PATCHIFY_TABLE": set(PATCHIFY_TABLE), "NHWC_TABLE": set(NHWC_TABLE), "MAXPOOL_TABLE": set(MAXPOOL_TABLE),
            "DW_TABLE": set(DW_TABLE), "TAIL_TABLE": set(TAIL_TABLE), "FILM_TABLE": set(FILM_TABLE),
            "IN_TABLE": set(IN_TABLE), "SE_TABLE": set(SE_TABLE), "SEG_OUT_TABLE": set(SEG_OUT_TABLE),
            "PREFIX_TABLE": set(PREFIX_TABLE)}


@pytest.mark.parametrize("variant", ["dinounet_s", "dinounet_b", "dinounet_l"])
def test_plan_shapes_are_covered(variant):
    """Builds build_plan_fp32 at (B=2, S=512) and checks that every non-GEMM launch has its shape arguments in this
    file's case tables, and every b2u_f32_gemm launch's epilogue signature (which of bias / scale / shift / act1 / act2 /
    residual / rows / a_rows / ps / col_off / conv it sets) in GEMM_TABLE, so a change of the plan names the kernel whose
    tests no longer cover it."""
    from dinounet_b200.engine import ForwardEngine
    from dinounet_b200.engine_fp32 import build_plan_fp32
    eng = ForwardEngine(variant, O.make_state_dict(variant, 2, seed=0), 2, torch.device(DEV), precision="fp32")
    plan, _ = build_plan_fp32(eng, B2, 512)
    tables = _covered()
    sigs = {_sig_case(c) for c in GEMM_TABLE}
    missing, n_gemm, n_other = [], 0, 0
    for name, fn, args in plan.calls:
        fname = fn.__name__
        if fname == "b2u_f32_gemm":
            n_gemm += 1
            s = _sig_params(args[0]._obj)
            if s not in sigs:
                missing.append(f"{name} (b2u_f32_gemm): epilogue {s} not in GEMM_TABLE")
            continue
        k = _key(fname, args)
        assert k is not None, f"{name}: {fname} has no case table in this file"
        n_other += 1
        if k[1] not in tables[k[0]]:
            missing.append(f"{name} ({fname}): {k[1]} not in {k[0]}")
    del plan, eng
    torch.cuda.empty_cache()
    assert n_gemm > 50 and n_other > 50
    assert not missing, "\n".join(missing)


# ============================================================================================ 8. end to end at S = 160
def test_forward_s160_odd_half_grids():
    """The whole fp32-tier forward of dinounet_s at 160 x 160 (B = 1): the MSDA coarse grid, the ConvFFN's coarse plane
    and the SPM's last level are 5 x 5, the 1/32 tail 5 x 5.  Against the oracle's fp32 forward under the tier's gate
    (1e-5 of max |logit|)."""
    from tests.test_gpu_fp32_tier import _check as check_logits, _net
    model = "dinounet_s"
    sd = O.make_state_dict(model, 2, seed=0)
    x = O.make_input(1, 160, 3)
    net = _net(model, sd)
    with torch.no_grad():
        y = net(x.cuda())
    check_logits(y, O.forward(sd, model, x), "fp32 tier dinounet_s B1 160 vs oracle")


# ============================================================================================ 9. optimizer
def _grid_sqsum(n):
    return max(1, min(512, n // 4096))


def _exact_sqsum(*ts):
    """Sum of squares of fp32 tensors in extended precision (each square is exact there), and its own error bound."""
    s = np.longdouble(0)
    n = 0
    for t in ts:
        a = t.detach().reshape(-1).cpu().numpy().astype(np.longdouble)
        s += np.sum(a * a)
        n += a.size
    return s, float(s) * (math.log2(max(n, 2)) + len(ts) + 1) * float(np.finfo(np.longdouble).eps)


def _sqsum_depth(n):
    """Depth of b2u_f32_sqsum's float64 sum: a serial chain per thread over its grid-stride elements, an 8-level tree
    per block, then one atomic add per block."""
    grid = _grid_sqsum(n)
    return -(-n // (grid * 256)) + 8 + grid


@pytest.mark.parametrize("n", [1, 7, 4095, 4096, 8191, 8192, 589_824, 2 ** 21 - 1, 2 ** 21, 2 ** 21 + 12_293, 10 ** 7])
def test_sqsum(n):
    """b2u_f32_sqsum adds sum g^2 (float64) to *out: one block below 8192 elements, n / 4096 blocks with a grid-stride
    loop up to the 512-block cap (n >= 2^21), the blocks meeting in float64 atomics.  A second call must add to the first.

    Bar: every square of an fp32 value is exact in float64 and all terms are positive, so a sum of depth k is within
    k 2^-53 of the exact sum relatively: k = the per-thread chain + 8 tree levels + one atomic per block, plus one for the
    value already in out; the extended-precision reference adds its own (much smaller) bound.  Few terms (n = 1, 7) are
    usually summed exactly, so their ratio is 0."""
    g = _randn(n, n % 1000 + 1, 1.5, 0.3)
    out = torch.zeros(1, dtype=torch.float64, device=DEV)
    _call("b2u_f32_sqsum", P(g), n, P(out))
    torch.cuda.synchronize()
    once = out.item()
    _call("b2u_f32_sqsum", P(g), n, P(out))
    torch.cuda.synchronize()
    twice = out.item()
    S, ref_err = _exact_sqsum(g)
    k = _sqsum_depth(n)
    for what, got, ref, depth in (("one call", once, S, k + 1), ("second call", twice, 2 * S, 2 * k + 2)):
        err = float(abs(np.longdouble(got) - ref))
        bar = depth * U64 * float(ref) + 2 * ref_err
        _WORST["f32_sqsum"] = max(_WORST.get("f32_sqsum", 0.0), err / bar)
        assert err <= bar, f"sqsum n={n} {what}: got {got!r}, exact {float(ref)!r}, err {err:.3g} > bar {bar:.3g}"


def _sgd_ref(p, g, buf, S, lr, mom, wd, max_norm, first, rel_s=0.0):
    """Float64 restatement of clip_grad_norm_(max_norm) + torch.optim.SGD(momentum, nesterov=True, weight_decay) on one
    tensor, from the kernel's fp32 inputs (lr, mom, wd, max_norm and the 1e-6f of the clip lifted from fp32), with bars.

    The clip coefficient is within e_c = (4u + rel_s) coef (the norm's conversion to fp32, + 1e-6f, the division; rel_s =
    the relative error of the squared norm); g coef + wd p within E_g = |g| e_c + 3u (|g coef| + |wd p|); the buffer
    mom buf + gg within E_b = E_g + 2u (|mom buf| + |gg|) (E_g on a first step); the step t = gg + mom b within
    E_t = E_g + mom E_b + 2u (|gg| + |mom b|), and p - lr t within lr E_t + 2u (|p| + |lr t|)."""
    lr, mom, wd, max_norm = (float(np.float32(v)) for v in (lr, mom, wd, max_norm))
    eps = float(np.float32(1e-6))
    norm = math.sqrt(float(S))
    coef = min(1.0, max_norm / (norm + eps))
    e_c = (4 * U + rel_s) * coef
    p, g = p.double(), g.double()
    gg = g * coef + wd * p
    E_g = g.abs() * e_c + 3 * U * ((g * coef).abs() + (wd * p).abs())
    if first:
        b, E_b = gg, E_g
    else:
        buf = buf.double()
        b = mom * buf + gg
        E_b = E_g + 2 * U * ((mom * buf).abs() + gg.abs())
    t = gg + mom * b
    E_t = E_g + mom * E_b + 2 * U * (gg.abs() + (mom * b).abs())
    pn = p - lr * t
    E_p = lr * E_t + 2 * U * (p.abs() + (lr * t).abs())
    return pn, E_p, b, E_b


# (name, n, grad scale, first step, lr, weight decay): the clip is active when sqrt(n) * scale > 12
SGD_CASES = [("clip-inactive", 1000, 0.1, 0, 1e-2, 3e-5), ("clip-active", 1000, 5.0, 0, 1e-2, 3e-5),
             ("norm-equals-max", 144, 1.0, 0, 1e-2, 3e-5), ("zero-grad", 1000, 0.0, 0, 1e-2, 3e-5),
             ("first-step", 256 * 37 + 3, 0.3, 1, 1e-2, 3e-5), ("first-step-clipped", 4099, 2.0, 1, 1e-2, 3e-5),
             ("lr0", 1000, 5.0, 0, 0.0, 3e-5), ("wd0", 589_824, 0.05, 0, 1e-2, 0.0), ("large-wd", 777, 0.2, 0, 0.1, 0.5)]


@pytest.mark.parametrize("case", SGD_CASES, ids=lambda c: c[0])
def test_sgd_nesterov(case):
    """b2u_f32_sgd_nesterov against _sgd_ref per element, parameters and momentum buffer.  The squared norm is handed in
    exactly (the sqsum has its own test); "norm-equals-max" has 144 gradients of +-1, a norm of exactly 12.  On a first
    step the buffer holds NaN (it must not be read); with lr = 0 the parameters must not change at all."""
    name, n, gs, first, lr, wd = case
    p = _randn(n, n + 1, 0.5)
    if name == "norm-equals-max":
        g = torch.where(torch.rand(n, generator=_gen(3), device=DEV) < 0.5, -1.0, 1.0)
    else:
        g = _randn(n, n + 2, gs)
    buf = _nan(n) if first else _randn(n, n + 3, 0.05)
    S, _ = _exact_sqsum(g)
    if name == "norm-equals-max":
        assert float(S) == 144.0
    sq = torch.tensor([float(S)], dtype=torch.float64, device=DEV)
    p0, buf0 = p.clone(), buf.clone()
    _call("b2u_f32_sgd_nesterov", P(p), P(g), P(buf), n, lr, 0.99, wd, P(sq), 12.0, first)
    torch.cuda.synchronize()
    pn, E_p, b, E_b = _sgd_ref(p0, g, buf0, S, lr, 0.99, wd, 12.0, first)
    _check("f32_sgd_nesterov", f"sgd {name} params", p, pn, E_p)
    _check("f32_sgd_nesterov", f"sgd {name} buffer", buf, b, E_b)
    if lr == 0.0:
        assert torch.equal(p, p0)


def test_fused_sgd_real_parameter_list():
    """FusedSGD (lr 1e-2, weight decay 3e-5, momentum 0.99, clip 12) over dinounet_s's 289 trainable tensors at their
    real sizes, three steps: clip inactive, active, just inactive.  Before each step the kernel's own fp32 parameters and
    buffers are lifted to float64, so each comparison is one step deep (_sgd_ref's bars, with the squared norm's bound
    from the sqsum depths of all 289 tensors: a dropped or doubled block changes the clip coefficient by far more).
    grad_norm() must equal the float64 norm within that bound."""
    import os
    import dinounet_b200
    from dinounet_b200.train_path import FusedSGD
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(cfg.DEFAULT_ARCHITECTURE)}, 3, 2, None, "dinounet_s")
    net.load_state_dict(O.make_state_dict("dinounet_s", 2, seed=0), strict=True)
    ps = [p.detach().to(DEV).clone().requires_grad_() for p in net.parameters() if p.requires_grad]
    del net
    assert len(ps) == 289
    ntot = sum(p.numel() for p in ps)
    depth = max(-(-p.numel() // (_grid_sqsum(p.numel()) * 256)) for p in ps) + 8 + sum(_grid_sqsum(p.numel()) for p in ps) + 1
    opt = FusedSGD(ps, lr=1e-2, weight_decay=3e-5, momentum=0.99, max_norm=12.0)
    for step, norm_target in enumerate((6.0, 100.0, 11.9)):
        gs = [_randn(p.shape, 100 * step + i, norm_target / math.sqrt(ntot)) for i, p in enumerate(ps)]
        for p, g in zip(ps, gs):
            p.grad = g
        before = [(p.detach().clone(), opt.state[p]["momentum_buffer"].clone() if p in opt.state else None) for p in ps]
        opt.step()
        torch.cuda.synchronize()
        S, ref_err = _exact_sqsum(*gs)
        rel_s = depth * U64 + ref_err / float(S)
        norm = math.sqrt(float(S))
        got = opt.grad_norm()
        assert abs(got - norm) <= norm * (rel_s / 2 + 2 * U64), f"step {step}: grad_norm {got!r} vs float64 {norm!r}"
        _NOTES.append(f"FusedSGD step {step}: norm {norm:.4f}, clip {'active' if norm > 12 else 'inactive'}, "
                      f"grad_norm rel err {abs(got - norm) / norm:.1e}")
        for i, (p, g, (p0, b0)) in enumerate(zip(ps, gs, before)):
            pn, E_p, b, E_b = _sgd_ref(p0, g, b0, S, 1e-2, 0.99, 3e-5, 12.0, b0 is None, rel_s)
            _check("fused_sgd", f"step {step} tensor {i} {tuple(p.shape)} params", p.detach(), pn, E_p)
            _check("fused_sgd", f"step {step} tensor {i} buffer", opt.state[p]["momentum_buffer"], b, E_b)
