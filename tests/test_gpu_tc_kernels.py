"""-m gpu: the 16-bit forward's tensor-core kernels against float64 references - the persistent wgmma GEMM with every
epilogue the engine uses (b2u_gemm, csrc/gemm_tc2.cu + gemm_api.cu), its implicit-GEMM 3x3 convolutions, the QKV
projection with its RoPE / head-split / V^T epilogue (b2u_qkv_rope) and the flash attention (b2u_attention_tc,
b2u_attention_tc_hd, csrc/attention_tc3.cu; b2u_attention_rows, csrc/attention_tc.cu).  Every kernel is called through
the C-ABI, at the shapes a 512x512 forward of dinounet_s/b/l runs (both query_dtype settings), at the ViT-7B widths, and on
both sides of every branch the code picks from the shape; the test id names the branch.

Every comparison is per element: |got - ref| <= bar, ref computed in float64 from the kernel's own 16-bit / fp32 inputs.
A bar has four parts, derived in each test's docstring:
  * accumulation: the wgmma adds fp32 products of 16-bit inputs (exact) in an order and with a rounding that are not
    documented, so a K-term sum is held to (ceil(K/16) + 2) 2^-23 sum_k |a_k w_k|;
  * fp32 epilogue operations: u = 2^-24 times the magnitude of each add / FMA (bias, affine, residual, add16);
  * a 16-bit rounding the kernel reproduces from the reference (round16 before the activation, the QKV output before
    RoPE, SwiGLU's silu(x1), attention's P): the two may land on neighbouring 16-bit values, so one ulp of the
    intermediate is carried through the gain of what follows (GELU <= 1.13, SiLU <= 1.1, |scale|, the RoPE rotation);
  * output rounding: one ulp of the 16-bit output at |ref| + the propagated error (bar16), u |ref| for fp32 outputs.
A dropped partial K block, a wrong tap, a mis-indexed head or pixel-shuffle quadrant is off by the size of the data, far
over these bars.  Outputs start as NaN (or hold known values for in-place epilogues), and everything outside the written
region must keep them.  Run with -s to print each kernel's worst error as a fraction of its bar."""
import ctypes as C
import math
from typing import NamedTuple, Tuple

import pytest
import torch
import torch.nn.functional as F

from dinounet_b200 import config as cfg
from dinounet_b200 import lib as L
from oracle import dinounet_oracle as O
from tests.gpu_helpers import TD, U, P, bar16, check, gemm, stream, ulp16

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [L.BF16, L.F16]
DNAME = {L.BF16: "bf16", L.F16: "f16"}
UR = {L.BF16: 2.0 ** -8, L.F16: 2.0 ** -11}          # unit roundoff of the 16-bit types
GELU_SLOPE, SILU_SLOPE = 1.13, 1.1                     # sup |GELU'| = 1.1289, sup |SiLU'| = 1.0998
EX2_REL = 2.0 ** -21                                   # ex2.approx.ftz.f32 relative error (documented 2^-22), with margin
TC_ENTRY_POINTS = {"b2u_gemm", "b2u_qkv_rope", "b2u_attention_tc", "b2u_attention_tc_hd", "b2u_attention_rows"}
_WORST: dict = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |got - ref| / bar per kernel:")
    for k in sorted(_WORST):
        print(f"  {k:28s} {_WORST[k]:.3f}")


def _check(kernel, what, got, ref, bar):
    return check(_WORST, kernel, what, got, ref, bar)


def _r16(x, dtype):
    return x.to(TD[dtype]).double()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(shape, seed, scale=1.0, dt=torch.float32):
    return (torch.randn(shape, generator=_gen(seed), device=DEV) * scale).to(dt)


def _nan(shape, dt):
    return torch.full(shape, float("nan"), device=DEV, dtype=dt)


def _acc_bar(K, sabs):
    """Bar of a K-term fp32 wgmma sum whose sum of |products| is sabs."""
    return (math.ceil(K / 16) + 2) * 2.0 ** -23 * sabs


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


# ============================================================================================ case tables
class G(NamedTuple):
    """One b2u_gemm launch: its shape and epilogue signature (res / add: 0 none, 1 the output buffer itself (in place),
    2 a separate tensor)."""
    M: int
    N: int
    K: int
    lda: int
    ldc: int
    col_off: int
    rows: Tuple[int, int, int]      # (rows_in, rows_out, row_off); zeros: no remap
    ps: Tuple[int, int, int]        # pixel shuffle (cout, h, w); zeros: none
    o32: int
    bias: int
    scale: int
    shift: int
    res: int
    add: int
    act1: int
    act2: int
    r16: int
    conv: int
    img: Tuple[int, int, int, int]  # (B, Hin, Win, C) of a convolution


def g(M, N, K, *, lda=None, ldc=None, col_off=0, rows=(0, 0, 0), ps=(0, 0, 0), o32=0, bias=1, scale=0, shift=0, res=0,
      add=0, act1=0, act2=0, r16=1):
    if ldc is None:
        ldc = N // 2 if act1 == L.ACT_SWIGLU else (ps[0] if ps[0] else N)
    return G(M, N, K, K if lda is None else lda, ldc, col_off, rows, ps, o32, bias, scale, shift, res, add, act1, act2,
             r16, 0, (0, 0, 0, 0))


def conv(B, H, W, Cin, Cout, stride, bn_relu):
    """An implicit-GEMM 3x3 convolution as the engine launches it: M = 0, K = 9 Cin, lda = Cin; epilogue folded BN +
    ReLU (no bias) or bias only."""
    return G(0, Cout, 9 * Cin, Cin, Cout, 0, (0, 0, 0), (0, 0, 0), 0, 0 if bn_relu else 1, int(bn_relu), int(bn_relu),
             0, 0, 0, L.ACT_RELU if bn_relu else 0, 1, L.CONV3X3_S2 if stride == 2 else L.CONV3X3_S1, (B, H, W, Cin))


B2, S512 = 2, 512
VIT = {"s": (384, 6, "mlp", 1536, True), "b": (768, 12, "mlp", 3072, True), "l": (1024, 16, "mlp", 4096, True),
       "7b_tiny": (1024, 8, "swiglu64", 2048, False)}          # (D, heads, ffn, hidden, qkv bias); 7b_tiny: test_gpu_parity
FEATS, FAPM_R = (32, 64, 128, 256), cfg.FAPM_RANK


def _vit_gemms(tag, B, S, D, ffn, Hd):
    h = S // 16
    Pn, T = h * h, B * (h * h + cfg.N_PREFIX)
    out = [(f"{tag}.patch_embed", g(B * Pn, D, 768, rows=(Pn, Pn + cfg.N_PREFIX, cfg.N_PREFIX), o32=1)),
           (f"{tag}.proj", g(T, D, D, o32=1, scale=1, res=1)),
           (f"{tag}.fc2", g(T, D, Hd, o32=1, scale=1, res=1))]
    if ffn == "mlp":
        out.append((f"{tag}.fc1", g(T, Hd, D, act1=L.ACT_GELU)))
    else:
        out.append((f"{tag}.fc1.swiglu", g(T, 2 * Hd, D, act1=L.ACT_SWIGLU)))
    return out


def _plan_gemms(tag, D, ffn, Hd, B=B2, S=S512):
    """Every b2u_gemm of ForwardEngine.build_plan(B, S) for an embedding width D, both query_dtype settings."""
    S4, S8 = S // 4, S // 8
    n4 = (S // 32) ** 2
    n3, n2 = 4 * n4, 16 * n4
    Lq, Pn = n2 + n3 + n4, (S // 16) ** 2
    out = _vit_gemms(tag, B, S, D, ffn, Hd)
    out.append((f"{tag}.spm.fc1", g(B * S4 * S4, D, 64)))
    for i, (kk, nl, off) in enumerate(((128, n2, 0), (256, n3, n2), (256, n4, n2 + n3))):
        for o32 in (1, 0):
            out.append((f"{tag}.spm.fc{i + 2}.{'c32' if o32 else 'c16'}", g(B * nl, D, kk, rows=(nl, Lq, off), o32=o32,
                                                                             shift=1)))
    out += [(f"{tag}.value", g(B * Pn, D // 2, D)), (f"{tag}.offaw", g(B * Lq, 192, D, o32=1)),
            (f"{tag}.outproj.c32", g(B * Lq, D, D // 2, o32=1, res=1)), (f"{tag}.outproj.c16", g(B * Lq, D, D // 2, add=1)),
            (f"{tag}.ffn1", g(B * Lq, D // 4, D)),
            (f"{tag}.ffn2.c32", g(B * Lq, D, D // 4, o32=1, res=1)), (f"{tag}.ffn2.c16", g(B * Lq, D, D // 4, add=1)),
            (f"{tag}.up", g(B * n2, 4 * D, D, ldc=D, ps=(D, S8, S8), add=2))]
    for i, oc in enumerate(FEATS):
        out.append((f"{tag}.f{i}.bases", g(B * (S4 >> i) ** 2, 2 * FAPM_R, D)))
    return out


def _shared_gemms(B=B2, S=S512):
    """The plan's D-independent GEMMs: FAPM, the learnable upsampling and the decoder's transposed convolutions."""
    S4, S8 = S // 4, S // 8
    out = []
    for i, oc in enumerate(FEATS):
        r = S4 >> i
        px = B * r * r
        out += [(f"f{i}.film_gen", g(px, 2 * FAPM_R, FAPM_R, lda=2 * FAPM_R)),
                (f"f{i}.reduce_sc", g(px, 2 * oc if oc != FAPM_R else oc, FAPM_R)),
                (f"f{i}.pw_refine", g(px, oc, oc)),
                (f"ups{i}.a", g(px, 4 * oc, oc, ps=(oc, r, r))),
                (f"ups{i}.b", g(4 * px, 4 * oc, oc, ldc=2 * oc if i < 3 else oc, col_off=oc if i < 3 else 0,
                                ps=(oc, 2 * r, 2 * r)))]
    below = FEATS[3]
    for s in range(3):
        skip, r_lo = FEATS[2 - s], S8 << s
        out.append((f"d{s}.transp", g(B * r_lo * r_lo, 4 * skip, below, ldc=2 * skip, ps=(skip, r_lo, r_lo))))
        below = skip
    return out


def _plan_convs(B=B2, S=S512):
    S2, S4 = S // 2, S // 4
    out = [("stem3_6", conv(B, S2, S2, 64, 64, 1, True)), ("conv2", conv(B, S4, S4, 64, 128, 2, True)),
           ("conv3", conv(B, S4 // 2, S4 // 2, 128, 256, 2, True)), ("conv4", conv(B, S4 // 4, S4 // 4, 256, 256, 2, True))]
    for s in range(3):
        skip, r_hi = FEATS[2 - s], (S // 4) << s
        out += [(f"d{s}.conv0", conv(B, r_hi, r_hi, 2 * skip, skip, 1, False)),
                (f"d{s}.conv1", conv(B, r_hi, r_hi, skip, skip, 1, False))]
    return out


_V7B = cfg.VARIANTS["dinounet_7b"]
GEMM_BOUNDARY = [
    ("bn32-Moff-K40-lda48", g(1000, 32, 40, lda=48)),
    ("bn32-o32-shift-norows", g(300, 32, 64, o32=1, bias=0, shift=1)),
    ("bn64-K200-lda256-res-prefetch", g(777, 64, 200, lda=256, o32=1, scale=1, res=1)),
    ("bn64-M1", g(1, 64, 64)),
    ("bn128-M130-K64", g(130, 128, 64)),
    ("bn128-N160-K96-lda104", g(1000, 160, 96, lda=104)),
    ("bn128-N96-single-tile-K72", g(515, 96, 72, o32=1)),
    ("res-kb8-prefetch-on", g(1029, 384, 512, o32=1, scale=1, res=1)),
    ("res-kb9-prefetch-off", g(1029, 384, 576, o32=1, scale=1, res=1)),
    ("round16-off-o32", g(2058, 384, 384, o32=1, r16=0)),
    ("round16-off-o32-K8192", g(1029, 256, 8192, o32=1, r16=0)),
    ("round16-off-16bit-gelu", g(700, 256, 128, r16=0, act1=L.ACT_GELU)),
    ("relu-after-affine", g(1000, 128, 96, bias=1, scale=1, shift=1, act2=L.ACT_RELU)),
    ("lrelu-after-affine", g(1000, 64, 64, bias=0, scale=1, shift=1, act2=L.ACT_LRELU)),
    ("ps-half-quadrants", g(512, 64, 64, ldc=32, ps=(32, 16, 16))),
    ("ps-add16-sep-coloff", g(2048, 256, 64, ldc=128, col_off=64, ps=(64, 32, 32), add=2)),
    ("swiglu-N128-Moff", g(300, 128, 64, act1=L.ACT_SWIGLU)),
    ("swiglu-N192-half-tile", g(515, 192, 96, act1=L.ACT_SWIGLU)),
    ("add16-inplace-K40", g(600, 96, 40, add=1)),
    ("rows-16bit-bias-scale", g(3 * 64, 128, 64, rows=(64, 69, 5), scale=1)),
] + _vit_gemms("7b", 1, S512, _V7B.embed_dim, _V7B.ffn_layer, _V7B.ffn_hidden)

CONV_BOUNDARY = [
    ("s2-Wo12-TW4-Ho-partial-B3", conv(3, 24, 24, 256, 256, 2, False)),
    ("s2-Wo24-TW8-Ho-partial", conv(1, 48, 48, 128, 256, 2, True)),
    ("s2-Wo40-TW8-TH16-partial", conv(2, 80, 80, 128, 256, 2, False)),
    ("s2-Wo80-TW16-exact", conv(1, 160, 160, 64, 128, 2, True)),
    ("s2-nonsquare-20x12-TW4", conv(2, 40, 24, 64, 128, 2, False)),
    ("s1-C32-half-kblock-TW32", conv(1, 96, 96, 32, 32, 1, True)),
    ("s1-C96-TW8", conv(2, 12, 8, 96, 64, 1, False)),
    ("s1-nonsquare-20x28-TW4", conv(3, 20, 28, 64, 64, 1, True)),
    ("s1-40x192-TW64", conv(1, 40, 192, 64, 64, 1, False)),
    ("s1-36x384-TW128", conv(1, 36, 384, 32, 32, 1, True)),
    ("s1-4x4-TW4", conv(2, 4, 4, 64, 64, 1, False)),
] + [(f"S640.{n}", c) for n, c in _plan_convs(1, 640) if c.img[1] <= 320] + \
    [(f"S384.{n}", c) for n, c in _plan_convs(1, 384) if c.img[1] <= 192]


def _dedupe(rows):
    seen, out = set(), []
    for name, c in rows:
        if c not in seen:
            seen.add(c)
            out.append((name, c))
    return out


_PLAN_GEMMS = []
for _t, (_D, _H, _ffn, _Hd, _qb) in VIT.items():
    _PLAN_GEMMS += _plan_gemms(_t, _D, _ffn, _Hd)
GEMM_TABLE = _dedupe(_PLAN_GEMMS + _shared_gemms() + GEMM_BOUNDARY)
CONV_TABLE = _dedupe(_plan_convs() + CONV_BOUNDARY)


def _bn(c):
    if c.act1 == L.ACT_SWIGLU:
        return 128
    return 32 if c.N <= 32 else (64 if c.N <= 64 else 128)


def _gemm_id(nc):
    name, c = nc
    s = f"{name}-M{c.M}N{c.N}K{c.K}-bn{_bn(c)}"
    if c.lda != c.K:
        s += f"-lda{c.lda}"
    if c.res:
        s += "-pf" if (c.K + 63) // 64 <= 8 and _bn(c) >= 64 else "-nopf"
    return s


def _conv_id(nc):
    name, c = nc
    B, H, W, Cc = c.img
    st = 2 if c.conv == L.CONV3X3_S2 else 1
    Wo = W // st
    tw = 128
    while Wo % tw:
        tw //= 2
    return f"{name}-B{B}-{H}x{W}x{Cc}-{c.N}-s{st}-TW{tw}TH{128 // tw}-{'bnrelu' if c.scale else 'bias'}"


# ============================================================================================ GEMM epilogue reference
def _epilogue_ref(acc, e, c, dtype, bias, scale, shift, res0, addv):
    """Float64 value of the generic epilogue on the accumulator `acc` (within `e` of the kernel's), and its bar.

    out = add16 + residual + act2(act1(r16(acc + bias)) * scale + shift): the bias add and every later fp32 operation add
    u |result|; the reproduced rounding carries ulp16(|acc + bias| + e) + e; GELU scales that by 1.13 and adds its own
    8u |x| (erf by Abramowitz-Stegun 7.1.26, 2.5u absolute, on rcp / ex2.approx) + u |GELU|; the affine (one FMA) scales
    it by |scale|; ReLU / LeakyReLU are 1-Lipschitz."""
    a = acc + bias if bias is not None else acc
    ea = e + (U * a.abs() if bias is not None else 0)
    if c.r16:
        r = _r16(a, dtype)
        er = ulp16(a.abs() + ea, dtype) + ea
    else:
        r, er = a, ea
    if c.act1 == L.ACT_GELU:
        y = F.gelu(r)
        ey = GELU_SLOPE * er + 8 * U * r.abs() + U * y.abs()
    else:
        y, ey = r, er
    if scale is not None or shift is not None:
        sc = scale if scale is not None else torch.ones_like(y[:1])
        z = y * sc + (shift if shift is not None else 0)
        ez = sc.abs() * ey + U * z.abs()
    else:
        z, ez = y, ey
    if c.act2 == L.ACT_RELU:
        z = F.relu(z)
    elif c.act2 == L.ACT_LRELU:
        z = torch.where(z > 0, z, 0.01 * z)
        ez = ez + U * z.abs()
    for t in (res0, addv):
        if t is not None:
            z = z + t
            ez = ez + U * z.abs()
    return z, (ez + U * z.abs() if c.o32 else bar16(z, ez, dtype))


def _swiglu_ref(acc, e, bias, dtype):
    """SwiGLU epilogue: the accumulator columns come in 64-column groups [x1 (32) | x2 (32)]; out = r16(silu(r16(x1 + b1)))
    * r16(x2 + b2).  Each reproduced rounding carries one ulp of its input's bar; silu (ex2.approx + rcp.approx, a product
    and an add) is within (12 + |x|) u relative, and its gain is <= 1.1; the product adds the cross terms and u |h|."""
    M, N = acc.shape
    sp = lambda t: (t.view(M, N // 64, 2, 32)[:, :, 0].reshape(M, N // 2), t.view(M, N // 64, 2, 32)[:, :, 1].reshape(M, N // 2))
    bb = bias.double()[None].expand(M, N) if bias is not None else torch.zeros_like(acc)
    (x1, x2), (e1, e2), (b1, b2) = sp(acc), sp(e), sp(bb)
    a1, a2 = x1 + b1, x2 + b2
    e1, e2 = e1 + U * a1.abs(), e2 + U * a2.abs()
    r1, r2 = _r16(a1, dtype), _r16(a2, dtype)
    er1, er2 = ulp16(a1.abs() + e1, dtype) + e1, ulp16(a2.abs() + e2, dtype) + e2
    s = F.silu(r1)
    es = SILU_SLOPE * er1 + (12 + r1.abs()) * U * s.abs()
    rs = _r16(s, dtype)
    ers = ulp16(s.abs() + es, dtype) + es
    h = rs * r2
    eh = r2.abs() * ers + rs.abs() * er2 + ers * er2 + U * h.abs()
    return h, bar16(h, eh, dtype)


def _dest(c, M, Nout, dev=DEV):
    """Output row / column of every (logical row, output column): the row remap, the pixel shuffle, col_off."""
    m = torch.arange(M, device=dev)
    n = torch.arange(Nout, device=dev)
    if c.ps[0]:
        cout, h, w = c.ps
        pb, rem = m // (h * w), m % (h * w)
        rbase = (pb * 2 * h + 2 * (rem // w)) * (2 * w) + 2 * (rem % w)
        qd = n // cout
        R = rbase[:, None] + ((qd >> 1) * (2 * w) + (qd & 1))[None, :]
        Cc = (n % cout) + c.col_off
        return R, Cc[None, :].expand(M, Nout), B_rows(c, M)
    if c.rows[0]:
        rin, rout, roff = c.rows
        R = (m // rin) * rout + roff + m % rin
    else:
        R = m
    return R[:, None].expand(M, Nout), (n + c.col_off)[None, :].expand(M, Nout), B_rows(c, M)


def B_rows(c, M):
    """Rows of the output buffer the launch addresses."""
    if c.ps[0]:
        return (M // (c.ps[1] * c.ps[2])) * 4 * c.ps[1] * c.ps[2]
    if c.rows[0]:
        return (M // c.rows[0]) * c.rows[1]
    return M


def _run_gemm_case(kernel, what, c, dtype, A, W, acc, sabs, Keff, x_shape=None):
    """Launch b2u_gemm for case c on A / W (the convolution's image when c.conv), check every written element against
    the float64 epilogue of `acc` (bar from `sabs`), and every other element of the output buffer for its sentinel."""
    td = TD[dtype]
    M, N = acc.shape
    swiglu = c.act1 == L.ACT_SWIGLU
    Nout = N // 2 if swiglu else N
    seed = M + N + c.K
    bias = _randn(N, seed + 1, 0.5) if c.bias else None
    scale = _randn(N, seed + 2) if c.scale else None
    shift = (_randn(N, seed + 3) - 0.5) if c.shift else None
    R, Cc, nrows = _dest(c, M, Nout)
    odt = torch.float32 if c.o32 else td
    if c.res == 1 or c.add == 1:
        out = _randn((nrows + 8, c.ldc), seed + 4, 2.0, odt)
    else:
        out = _nan((nrows + 8, c.ldc), odt)
    orig = out.clone()
    addt = _randn((nrows, c.ldc), seed + 5, 1.0, td) if c.add == 2 else None
    kw = dict(M=c.M, K=c.K, lda=c.lda, ldc=c.ldc, out_fp32=bool(c.o32), col_off=c.col_off,
              rows=c.rows if c.rows[0] else None, ps=c.ps if c.ps[0] else None, bias=bias, scale=scale, shift=shift,
              act1=c.act1, act2=c.act2, round16=c.r16, conv=c.conv, img=c.img)
    if c.res == 1:
        kw.update(residual=out, ldres=c.ldc)
    if c.add:
        kw.update(add16=out if c.add == 1 else addt, ldadd=c.ldc)
    gemm(A, W, out, dtype, **kw)
    torch.cuda.synchronize()
    e = _acc_bar(Keff, sabs)
    if swiglu:
        ref, bar = _swiglu_ref(acc, e, bias, dtype)
    else:
        res0 = orig[R, Cc].double() if c.res == 1 else None
        addv = (orig if c.add == 1 else addt)[R, Cc].double() if c.add else None
        ref, bar = _epilogue_ref(acc, e, c, dtype, None if bias is None else bias.double(),
                                 None if scale is None else scale.double(), None if shift is None else shift.double(),
                                 res0, addv)
    _check(kernel, what, out[R, Cc], ref, bar)
    written = torch.zeros(out.shape, dtype=torch.bool, device=DEV)
    written[R, Cc] = True
    assert written.sum() == M * Nout, "two outputs share a destination"
    moved = (_bits(out) != _bits(orig)) & ~written
    assert not moved.any(), f"{what}: {int(moved.sum())} elements outside the written region changed, first at " \
                            f"{tuple(int(t) for t in moved.nonzero()[0])}"


# ============================================================================================ b2u_gemm
@pytest.mark.parametrize("dtype", DTYPES, ids=DNAME.get)
@pytest.mark.parametrize("case", GEMM_TABLE, ids=_gemm_id)
def test_gemm(case, dtype):
    """b2u_gemm on plain operands: A [M, K] (row stride lda; columns K..lda hold NaN, which must never be read) times
    W [N, K]^T, then the epilogue of the case (see _epilogue_ref / _swiglu_ref for the bar).  The accumulation bar is
    (ceil(K/16) + 2) 2^-23 |A| |W|^T.  Rows past the output, columns outside [col_off, col_off + N), the pixel-shuffle
    quadrants not written and the rows a remap skips keep their NaN (or their original bits, in place)."""
    name, c = case
    td = TD[dtype]
    Abuf = _nan((c.M, c.lda), td)
    Abuf[:, :c.K] = _randn((c.M, c.K), c.M + c.K, 1.0, td)
    A = Abuf[:, :c.K]
    W = _randn((c.N, c.K), c.N + 7 * c.K, c.K ** -0.5, td)
    Ad, Wd = A.double(), W.double()
    acc = Ad @ Wd.t()
    sabs = Ad.abs() @ Wd.abs().t()
    del Ad, Wd
    if c.act1 == L.ACT_SWIGLU:
        kernel = "gemm.swiglu"
    elif c.o32 and not c.r16 and not (c.scale or c.shift or c.res or c.add):
        kernel = "gemm.o32.accumulate"       # acc + bias in fp32: the accumulation bar measured on its own
    else:
        kernel = "gemm.o32" if c.o32 else "gemm.16"
    _run_gemm_case(kernel, f"gemm {name}", c, dtype, A, W, acc, sabs, c.K)


# ============================================================================================ implicit-GEMM 3x3 conv
@pytest.mark.parametrize("dtype", DTYPES, ids=DNAME.get)
@pytest.mark.parametrize("case", CONV_TABLE, ids=_conv_id)
def test_conv3x3(case, dtype):
    """b2u_gemm with conv = 3x3 stride 1 / 2, padding 1, on an NHWC image; W packed [Cout, 9 x ceil(C/64) x 64] in
    (dy, dx, channel) order with zero channel padding, as the engine packs it.  The reference is nine shifted float64
    GEMMs over the zero-padded image, so every border pixel sees its padding taps; the accumulation bar counts the
    9 ceil(C/64) 64-wide k-blocks the kernel runs.  Output rows past B Ho Wo keep their NaN."""
    name, c = case
    td = TD[dtype]
    B, H, W, Cc = c.img
    st = 2 if c.conv == L.CONV3X3_S2 else 1
    Ho, Wo = H // st, W // st
    cb = (Cc + 63) // 64
    x = _randn((B, H, W, Cc), H + W + Cc, 1.0, td)
    wp = torch.zeros(c.N, 9, cb * 64, device=DEV, dtype=td)
    wp[:, :, :Cc] = _randn((c.N, 9, Cc), c.N + Cc, (9 * Cc) ** -0.5, td)
    Wbuf = wp.reshape(c.N, 9 * cb * 64)
    xp = torch.zeros(B, H + 2, W + 2, Cc, device=DEV, dtype=torch.float64)
    xp[:, 1:-1, 1:-1] = x.double()
    acc = torch.zeros(B, Ho, Wo, c.N, device=DEV, dtype=torch.float64)
    sabs = torch.zeros_like(acc)
    for tap in range(9):
        dy, dx = divmod(tap, 3)
        xs = xp[:, dy:dy + st * (Ho - 1) + 1:st, dx:dx + st * (Wo - 1) + 1:st]
        wt = wp[:, tap, :Cc].double()
        acc += xs @ wt.t()
        sabs += xs.abs() @ wt.abs().t()
    del xp
    _run_gemm_case("conv3x3.s%d" % st, f"conv {name}", c, dtype, x.view(-1, Cc), Wbuf, acc.view(-1, c.N),
                   sabs.view(-1, c.N), 9 * cb * 64)


# ============================================================================================ b2u_qkv_rope
class Q(NamedTuple):
    B: int
    gh: int       # RoPE grid (ntok = gh * gw + 5)
    gw: int
    D: int
    heads: int
    bias: int
    sep: int      # 1: separable shared-memory tables (rope_w = gw), 0: the global tables
    vt: int       # 1: V written transposed [B, heads, hd, npad]
    scale: float  # RoPE coordinate scale of the tables (1: eval; else the train-mode rescaling, scaled_vit_plan)


QKV_TABLE = [(f"{t}.qkv", Q(B2, 32, 32, D, H, int(qb), 1, 1, 1.0)) for t, (D, H, _f, _h, qb) in VIT.items()] + [
    ("7b.qkv", Q(1, 32, 32, _V7B.embed_dim, _V7B.num_heads, 0, 1, 1, 1.0)),
    ("hd64-global-tables-scaled", Q(B2, 32, 32, 384, 6, 1, 0, 1, 1.37)),
    ("hd64-smem-tables-scaled", Q(B2, 32, 32, 768, 12, 1, 1, 1, 0.61)),
    ("hd128-smem-tables-scaled-nobias", Q(B2, 32, 32, 1024, 8, 0, 1, 1, 1.37)),
    ("hd64-nonsquare-24x40-smem", Q(3, 24, 40, 384, 6, 1, 1, 1, 1.0)),
    ("hd64-nonsquare-24x40-global-V", Q(1, 24, 40, 384, 6, 0, 0, 0, 1.0)),
    ("hd128-nonsquare-40x16-smem-V", Q(2, 40, 16, 512, 4, 1, 1, 0, 1.21)),
    ("hd64-largest-smem-grid-114x113", Q(1, 114, 113, 384, 6, 1, 1, 1, 1.0)),
    ("hd128-largest-smem-grid-60x60", Q(1, 60, 60, 512, 4, 0, 1, 1, 1.0)),
]


def _rope_tables(gh, gw, hd, scale):
    """sin / cos [gh gw, hd] from b2u_rope_tables (the per-block tables of scaled_vit_plan) with coordinate scale."""
    periods = (cfg.ROPE_BASE ** (2 * torch.arange(hd // 4, dtype=torch.float32) / (hd // 2))).to(DEV)
    scales = torch.full((1,), scale, device=DEV)
    sin = _nan((gh * gw, hd), torch.float32)
    cos = _nan((gh * gw, hd), torch.float32)
    lib = L.load()
    L.check(lib.b2u_rope_tables(P(periods), P(scales), P(sin), P(cos), 1, gh, gw, hd, stream()), "rope_tables")
    return sin, cos


def _qkv_params(c, Y, Wq, bias, sin, cos, q, k, v, dtype):
    ntok = c.gh * c.gw + cfg.N_PREFIX
    p = L.QkvParams()
    p.B, p.ntok, p.D, p.heads, p.prefix = c.B, ntok, c.D, c.heads, cfg.N_PREFIX
    p.A, p.lda, p.Wp, p.ldw, p.bias = P(Y), c.D, P(Wq), c.D, P(bias)
    p.rope_sin, p.rope_cos, p.q, p.k, p.v, p.dtype = P(sin), P(cos), P(q), P(k), P(v), dtype
    p.v_transposed, p.npad, p.rope_w = c.vt, ((ntok + 7) // 8 * 8) if c.vt else 0, c.gw if c.sep else 0
    return p


@pytest.mark.parametrize("dtype", DTYPES, ids=DNAME.get)
@pytest.mark.parametrize("case", QKV_TABLE, ids=lambda nc: f"{nc[0]}-B{nc[1].B}-D{nc[1].D}-hd{nc[1].D // nc[1].heads}")
def test_qkv_rope(case, dtype):
    """b2u_qkv_rope: qkv = Y Wqkv^T + b rounded to 16 bits (reproduced), split into q / k / v [B, heads, ntok, hd];
    q and k rotated (lo' = lo cos - hi sin, hi' = hi cos + lo sin, angle j of the token's table row) on the patch rows
    t >= 5, the five prefix rows unrotated; V optionally stored as V^T [B, heads, hd, npad].

    Bar: the accumulation bar e plus u |qkv| for the bias; unrotated outputs are the 16-bit rounding of that value
    (bar16(qkv, e)); rotated ones carry the reproduced rounding er = ulp16(|qkv| + e) + e of both inputs through
    |cos| er_lo + |sin| er_hi, plus 2u (|lo cos| + |hi sin|) for the fp32 rotation, plus the output rounding.  The V^T
    padding columns [ntok, npad) keep their NaN."""
    name, c = case
    td = TD[dtype]
    hd = c.D // c.heads
    ntok = c.gh * c.gw + cfg.N_PREFIX
    npad = (ntok + 7) // 8 * 8
    Y = _randn((c.B * ntok, c.D), c.D + ntok, 1.0, td)
    Wq = _randn((3 * c.D, c.D), c.D + 1, c.D ** -0.5, td)
    bias = _randn(3 * c.D, c.D + 2, 0.3) if c.bias else None
    sin, cos = _rope_tables(c.gh, c.gw, hd, c.scale)
    q, k = (_nan((c.B, c.heads, ntok, hd), td) for _ in range(2))
    v = _nan((c.B, c.heads, hd, npad) if c.vt else (c.B, c.heads, ntok, hd), td)
    p = _qkv_params(c, Y, Wq, bias, sin, cos, q, k, v, dtype)
    L.check(L.load().b2u_qkv_rope(C.byref(p), stream()), "b2u_qkv_rope")
    torch.cuda.synchronize()
    Yd, Wd = Y.double(), Wq.double()
    acc = Yd @ Wd.t()
    e = _acc_bar(c.D, Yd.abs() @ Wd.abs().t())
    del Yd, Wd
    if bias is not None:
        acc = acc + bias.double()
        e = e + U * acc.abs()
    split = lambda t: t.view(c.B, ntok, 3, c.heads, hd).permute(2, 0, 3, 1, 4)      # [3, B, heads, ntok, hd]
    acc, e = split(acc), split(e)
    r = _r16(acc, dtype)
    er = ulp16(acc.abs() + e, dtype) + e
    sn, cs = sin.double(), cos.double()
    h2 = hd // 2
    npre = cfg.N_PREFIX
    for which, got in ((0, q), (1, k)):
        a, ea, rr, ee = acc[which], e[which], r[which], er[which]
        _check("qkv_rope.prefix", f"{name} {'qk'[which]} prefix rows", got[:, :, :npre], a[:, :, :npre],
               bar16(a[:, :, :npre], ea[:, :, :npre], dtype))
        lo, hi = rr[:, :, npre:, :h2], rr[:, :, npre:, h2:]
        elo, ehi = ee[:, :, npre:, :h2], ee[:, :, npre:, h2:]
        c_lo, s_lo, c_hi, s_hi = cs[:, :h2], sn[:, :h2], cs[:, h2:], sn[:, h2:]
        ref = torch.cat([lo * c_lo - hi * s_lo, hi * c_hi + lo * s_hi], -1)
        prop = torch.cat([c_lo.abs() * elo + s_lo.abs() * ehi + 2 * U * ((lo * c_lo).abs() + (hi * s_lo).abs()),
                          c_hi.abs() * ehi + s_hi.abs() * elo + 2 * U * ((hi * c_hi).abs() + (lo * s_hi).abs())], -1)
        _check("qkv_rope.rotated", f"{name} {'qk'[which]} rotated rows", got[:, :, npre:], ref, bar16(ref, prop, dtype))
    vgot = v[..., :ntok].transpose(2, 3) if c.vt else v
    _check("qkv_rope.v", f"{name} v", vgot, acc[2], bar16(acc[2], e[2], dtype))
    if c.vt:
        assert torch.isnan(v[..., ntok:].float()).all(), "V^T padding columns were written"


def test_qkv_rope_grid_limit():
    """The separable tables are staged in 32 KB of shared memory: (h + w)(2 hd + 16) bytes.  The largest admitted grids
    run in test_qkv_rope (114 + 113 at hd 64, 60 + 60 at hd 128); one row more must be refused without a launch (the
    outputs keep their NaN and the launch counter does not move), and so must a grid that does not match ntok."""
    lib = L.load()
    dtype, td = L.BF16, torch.bfloat16
    for c in (Q(1, 61, 60, 512, 4, 0, 1, 1, 1.0), Q(1, 115, 113, 384, 6, 0, 1, 1, 1.0)):
        hd = c.D // c.heads
        ntok = c.gh * c.gw + cfg.N_PREFIX
        Y = _randn((ntok, c.D), 1, 1.0, td)
        Wq = _randn((3 * c.D, c.D), 2, c.D ** -0.5, td)
        sin, cos = _rope_tables(c.gh, c.gw, hd, 1.0)
        q, k = (_nan((1, c.heads, ntok, hd), td) for _ in range(2))
        vt = _nan((1, c.heads, hd, (ntok + 7) // 8 * 8), td)
        torch.cuda.synchronize()
        too_large = _qkv_params(c, Y, Wq, None, sin, cos, q, k, vt, dtype)
        mismatched = _qkv_params(c, Y, Wq, None, sin, cos, q, k, vt, dtype)
        mismatched.rope_w = c.gw - 1                   # (ntok - 5) is not a multiple of it
        for p in (too_large, mismatched):
            n0 = L.launch_count()
            assert lib.b2u_qkv_rope(C.byref(p), stream()) != 0, f"rope grid for rope_w {p.rope_w} at hd {hd} was accepted"
            assert L.launch_count() == n0, "a refused call launched"
        torch.cuda.synchronize()
        assert all(torch.isnan(t.float()).all() for t in (q, k, vt))


# ============================================================================================ attention
class A(NamedTuple):
    B: int
    heads: int
    ntok: int
    hd: int
    q_begin: int
    pattern: str   # random | rising | lastmax | dominant | equal | q8


ATTN_TABLE = [(f"{t}.attn", A(B2, H, 1029, D // H, 0, "random")) for t, (D, H, _f, _h, _qb) in VIT.items()]
ATTN_TABLE += [("7b.attn", A(1, _V7B.num_heads, 1029, _V7B.embed_dim // _V7B.num_heads, 0, "random"))]
for _hd in (64, 128):
    ATTN_TABLE += [(f"keytail{_r}", A(1, 2, 1024 + _r, _hd, 0, "random")) for _r in (1, 16, 17, 32, 33, 48, 64, 65, 127, 0)]
    ATTN_TABLE += [("single-chunk", A(1, 2, _n, _hd, 0, "random")) for _n in (1, 100, 128)]
    ATTN_TABLE += [(f"pattern-{_p}", A(1, 2, 1029, _hd, 0, _p)) for _p in ("rising", "lastmax", "dominant", "equal", "q8")]
ATTN_TABLE += [("querytail-hd64-2-empty-consumers", A(2, 3, 970, 64, 0, "random")),
               ("querytail-hd128-1-empty-consumer", A(2, 3, 1034, 128, 0, "random"))]
ATTN_TABLE += [(f"qbegin{_q}+rows", A(2, 3, 1029, 64, _q, "random")) for _q in (1, 5, 8)]
ATTN_TABLE += [("qbegin8+rows-rising", A(1, 2, 1029, 64, 8, "rising")), ("qbegin3+rows-tail1", A(1, 2, 1025, 64, 3, "q8"))]


def _tail_branch(a):
    J = (a.ntok + 127) // 128
    tail = a.ntok - (J - 1) * 128
    if J == 1:
        return "J1-n128"
    return f"J{J}-n{16 if tail <= 16 else 32 if tail <= 32 else 64 if tail <= 64 else 128}"


def _attn_id(nc):
    name, a = nc
    return f"{name}-B{a.B}H{a.heads}N{a.ntok}-hd{a.hd}-{_tail_branch(a)}"


def _attn_inputs(a, dtype):
    """q, k, v [B, H, ntok, hd] in the 16-bit type, shaped by the logit pattern: `rising` adds 24 per 128 keys to
    k[..., 0] against q[..., 0] = 4 (the running maximum moves by > 8 in log2 units on every chunk, so the lazy rescale
    fires each time); `lastmax` puts k[..., 0] = 20 on the keys of the last chunk only; `dominant` one key (517) with
    k[..., 0] = 30; `equal` every key the same (each query's answer is the exact mean of V); `q8` scales q by 8 (P near
    2^8 in the kernel's lazily scaled units)."""
    B, H, N, hd = a.B, a.heads, a.ntok, a.hd
    seed = B * 7 + H * 13 + N + hd
    q = _randn((B, H, N, hd), seed)
    k = _randn((B, H, N, hd), seed + 1)
    v = _randn((B, H, N, hd), seed + 2)
    j = torch.arange(N, device=DEV, dtype=torch.float32)
    if a.pattern in ("rising", "lastmax", "dominant"):
        q[..., 0] = 4.0
    if a.pattern == "rising":
        k[..., 0] = 24.0 * torch.floor(j / 128) + 0.2 * (j % 128) / 128
    elif a.pattern == "lastmax":
        k[..., 0] = torch.where(j >= (N - 1) // 128 * 128, 20.0, 0.0)
    elif a.pattern == "dominant":
        k[..., 517 % N, 0] = 30.0
    elif a.pattern == "equal":
        k = k[:, :, :1].expand(B, H, N, hd).contiguous()
    elif a.pattern == "q8":
        q = q * 8
    td = TD[dtype]
    return q.to(td), k.to(td), v.to(td)


def _attn_ref(q, k, v, scale, dtype):
    """Float64 softmax(q k^T scale) v and its bar, in reference units p_j = 2^(x_j - max x), x = s scale log2(e), l = sum p.

    The kernel's p_j carries a relative error d_j: the logit's accumulation bar times scale, the fp32 scale log2(e)
    (2u) and the exponent's FMA (u |x - m|, |m| <= A = max |x|), ex2.approx (2^-21), and, for each of the <= J rescales
    of the running maximum after its chunk, the rescale factor's ex2 and subtraction (2^-21 + 2u A ln 2).  That moves O
    by sum_j d_j p_j |v_j - O| / l <= (sum_j d_j p_j |v_j| + |O| sum_j d_j p_j) / l.  Rounding P to 16 bits for the PV
    MMA while l sums the unrounded values adds u16 sum_j p_j |v_j| / l (u16: the type's unit roundoff), and for f16
    probabilities below 2^-14 (subnormal) ntok 2^-25 max|v| / l.  The PV sum is an fp32 wgmma accumulation over 8 J
    K = 16 steps with up to J rescales of O: (8J + 2) 2^-23 + J u relative to sum p |v| / l (times 1 + u16 for the
    rounded P); l is a sum of depth <= 2J + 20 (< (2J + 20) u |O|); the reciprocal and product add 3u |O|."""
    N, hd = q.shape[-2], q.shape[-1]
    J = (N + 127) // 128
    qd, kd, vd = q.double(), k.double(), v.double()
    sl2 = float(torch.tensor(scale, dtype=torch.float32)) * math.log2(math.e)
    s = qd @ kd.transpose(-1, -2)
    x = s * sl2
    del s
    mx = x.amax(-1, keepdim=True)
    amax = x.abs().amax(-1, keepdim=True)
    p = torch.exp2(x - mx)
    l = p.sum(-1, keepdim=True)
    d = math.log(2) * (_acc_bar(hd, qd.abs() @ kd.abs().transpose(-1, -2)) * sl2 + 2 * U * x.abs() + U * (x - mx).abs()
                       + U * amax) + (J + 1) * (EX2_REL + 2 * math.log(2) * U * amax)
    del x
    va = vd.abs()
    O = (p @ vd) / l
    pv = (p @ va) / l
    dp = d * p
    del d
    prop = (dp @ va) / l + O.abs() * dp.sum(-1, keepdim=True) / l
    prop = prop + UR[dtype] * pv + ((8 * J + 2) * 2.0 ** -23 + J * U) * (1 + UR[dtype]) * pv
    if dtype == L.F16:
        prop = prop + N * 2.0 ** -25 * va.amax((-1, -2), keepdim=True) / l
    prop = prop + (2 * J + 23) * U * O.abs()
    return O, bar16(O, prop, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=DNAME.get)
@pytest.mark.parametrize("case", ATTN_TABLE, ids=_attn_id)
def test_attention(case, dtype):
    """b2u_attention_tc (head_dim 64) / b2u_attention_tc_hd (64, 128) over query rows [q_begin, ntok), V read as V^T
    [B, H, hd, npad] with zero padding columns, output [B, ntok, H hd]; for q_begin > 0 the rows [0, q_begin) come from
    b2u_attention_rows (head_dim 64), launched after the wgmma kernel has been checked to leave them NaN.  The test id
    names the MMA width of the last key chunk (J chunks of 128 keys).  Bar: _attn_ref."""
    name, a = case
    td = TD[dtype]
    lib = L.load()
    q, k, v = _attn_inputs(a, dtype)
    B, H, N, hd = a.B, a.heads, a.ntok, a.hd
    npad = (N + 7) // 8 * 8
    vt = torch.zeros(B, H, hd, npad, device=DEV, dtype=td)
    vt[..., :N] = v.transpose(2, 3)
    out = _nan((B, N, H * hd), td)
    scale = hd ** -0.5
    if hd == 64:
        rc = lib.b2u_attention_tc(P(q), P(k), P(vt), P(out), B, H, N, npad, a.q_begin, scale, dtype, stream())
    else:
        assert a.q_begin == 0
        rc = lib.b2u_attention_tc_hd(P(q), P(k), P(vt), P(out), B, H, N, npad, hd, scale, dtype, stream())
    L.check(rc, "attention")
    torch.cuda.synchronize()
    O, bar = _attn_ref(q, k, v, scale, dtype)
    O, bar = O.transpose(1, 2).reshape(B, N, H * hd), bar.transpose(1, 2).reshape(B, N, H * hd)
    if a.q_begin:
        assert torch.isnan(out[:, :a.q_begin].float()).all(), "rows before q_begin were written"
        L.check(lib.b2u_attention_rows(P(q), P(k), P(vt), P(out), B, H, N, npad, 0, a.q_begin, scale, dtype, stream()),
                "attention_rows")
        torch.cuda.synchronize()
        _check("attention_rows", f"{name} rows [0, {a.q_begin})", out[:, :a.q_begin], O[:, :a.q_begin],
               bar[:, :a.q_begin])
    _check(f"attention_tc.hd{hd}", f"{name} rows [{a.q_begin}, {N})", out[:, a.q_begin:], O[:, a.q_begin:],
           bar[:, a.q_begin:])


@pytest.mark.parametrize("dtype", DTYPES, ids=DNAME.get)
@pytest.mark.parametrize("nrows", [1, 2, 7, 8])
@pytest.mark.parametrize("ntok", [69, 1029])
def test_attention_rows(ntok, nrows, dtype):
    """b2u_attention_rows alone over rows [row_begin, row_begin + nrows) (exact row maximum, fp32 softmax sums, P rounded
    to 16 bits for the PV sum): the bar of _attn_ref (J = 1 there covers its shorter sums), and every other row keeps its
    NaN."""
    td = TD[dtype]
    lib = L.load()
    a = A(2, 3, ntok, 64, 0, "random")
    q, k, v = _attn_inputs(a, dtype)
    npad = (ntok + 7) // 8 * 8
    vt = torch.zeros(2, 3, 64, npad, device=DEV, dtype=td)
    vt[..., :ntok] = v.transpose(2, 3)
    out = _nan((2, ntok, 3 * 64), td)
    r0 = 3 if nrows < 8 else 0
    L.check(lib.b2u_attention_rows(P(q), P(k), P(vt), P(out), 2, 3, ntok, npad, r0, nrows, 0.125, dtype, stream()), "rows")
    torch.cuda.synchronize()
    O, bar = _attn_ref(q, k, v, 0.125, dtype)
    O, bar = O.transpose(1, 2).reshape(2, ntok, 192), bar.transpose(1, 2).reshape(2, ntok, 192)
    _check("attention_rows", f"rows [{r0}, {r0 + nrows})", out[:, r0:r0 + nrows], O[:, r0:r0 + nrows],
           bar[:, r0:r0 + nrows])
    rest = torch.ones(ntok, dtype=torch.bool, device=DEV)
    rest[r0:r0 + nrows] = False
    assert torch.isnan(out[:, rest].float()).all(), "rows outside the range were written"


# ============================================================================================ shape-drift guard
def _gemm_key(p):
    e = p.epi
    own = lambda ptr, ld: 0 if not ptr else ((1 if ptr == e.out else 2) if ld == e.ldc else -1)
    return G(p.M, p.N, p.K, p.lda, e.ldc, e.col_off, (e.rows_in, e.rows_out, e.row_off), (e.ps_cout, e.ps_h, e.ps_w),
             e.out_fp32, int(bool(e.bias)), int(bool(e.scale)), int(bool(e.shift)), own(e.residual, e.ldres),
             own(e.add16, e.ldadd), e.act1, e.act2, e.round16, p.conv, (p.B, p.Hin, p.Win, p.C))


def _key(fname, args):
    """(table, shape key) of one plan launch of the five entry points."""
    if fname == "b2u_gemm":
        c = _gemm_key(args[0]._obj)
        return ("CONV_TABLE" if c.conv else "GEMM_TABLE"), c
    if fname == "b2u_qkv_rope":
        p = args[0]._obj
        return "QKV_TABLE", (p.B, p.ntok, p.D, p.heads, p.prefix, int(bool(p.bias)), p.rope_w, p.v_transposed, p.npad)
    if fname == "b2u_attention_tc":
        return "ATTN_TABLE", (args[4], args[5], args[6], args[7], args[8], 64)
    if fname == "b2u_attention_tc_hd":
        return "ATTN_TABLE", (args[4], args[5], args[6], args[7], 0, args[8])
    return "ROWS", (args[4], args[5], args[6], args[7], args[8], args[9])


def _covered():
    def qkey(c):
        ntok = c.gh * c.gw + cfg.N_PREFIX
        return (c.B, ntok, c.D, c.heads, cfg.N_PREFIX, c.bias, c.gw if c.sep else 0, c.vt, (ntok + 7) // 8 * 8 if c.vt else 0)
    return {"GEMM_TABLE": {c for _, c in GEMM_TABLE}, "CONV_TABLE": {c for _, c in CONV_TABLE},
            "QKV_TABLE": {qkey(c) for _, c in QKV_TABLE},
            "ATTN_TABLE": {(a.B, a.heads, a.ntok, (a.ntok + 7) // 8 * 8, a.q_begin, a.hd) for _, a in ATTN_TABLE},
            "ROWS": set()}


@pytest.mark.parametrize("query_dtype", ["fp32", "16"])
@pytest.mark.parametrize("variant", ["dinounet_s", "dinounet_b", "dinounet_l", "dinounet_7b_tiny"])
def test_plan_shapes_are_covered(variant, query_dtype):
    """Builds the engine's launch plan at (B=2, S=512) and checks that every b2u_gemm (shape and epilogue signature: which
    of bias / scale / shift / residual / add16 are set and whether in place, act1 / act2, round16, row remap, pixel
    shuffle, col_off, conv and image), b2u_qkv_rope and attention launch appears in this file's tables, naming the
    launches that do not.  dinounet_7b_tiny (SwiGLU, head_dim 128, no qkv bias) is registered as test_gpu_parity.py
    does."""
    from dinounet_b200.engine import ForwardEngine
    if variant == "dinounet_7b_tiny":
        cfg.VARIANTS[variant] = cfg.VariantConfig(variant, 1024, 4, 8, "swiglu64", 2048, False, (0, 1, 2, 3), True, 0.4)
    try:
        eng = ForwardEngine(variant, O.make_state_dict(variant, 2, seed=0), 2, torch.device(DEV), query_dtype=query_dtype)
        plan, _ = eng.build_plan(B2, S512)
        tables = _covered()
        missing, n = [], 0
        for name, fn, args in plan.calls:
            fname = fn.__name__
            if fname not in TC_ENTRY_POINTS:
                continue
            n += 1
            t, key = _key(fname, args)
            if key not in tables[t]:
                missing.append(f"{name} ({fname}): {key} not in {t}")
        del plan, eng
        torch.cuda.empty_cache()
    finally:
        if variant == "dinounet_7b_tiny":
            cfg.VARIANTS.pop(variant, None)
    assert n > 40
    assert not missing, "\n".join(missing)
