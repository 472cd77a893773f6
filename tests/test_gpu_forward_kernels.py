"""-m gpu: the forward pass's normalisation, elementwise and deformable-attention kernels (csrc/elementwise.cu,
csrc/msda.cu) against float64 references, at the shapes a 512x512 forward of dinounet_s/b/l runs and on both sides of
every branch these kernels pick from the shape.  Every kernel is called through the C-ABI.

Every comparison is per element: |got - ref| <= bar, with ref computed in float64 from the kernel's own 16-bit or fp32
inputs.  A bar is a worst-case bound built from three terms, derived in each test's docstring:
  * output rounding: one unit in the last place of the 16-bit output type, taken at |ref| plus the propagated error
    (`_bar16`), which also covers a result that rounds across a power of two;
  * fp32 arithmetic: a sum evaluated as a tree of depth k is within k * u * sum|terms| of the exact sum (u = 2^-24), and
    each further fp32 operation adds u times its magnitude;
  * a 16-bit rounding the kernel reproduces from the reference (the stem conv output, the depthwise conv's GELU input,
    the seg head's normalised activation): the kernel and the reference may round a value to neighbouring 16-bit numbers,
    so one ulp of that intermediate is carried through the gain of what follows.
Nothing else is rounded in the references.  A wrong tap, a dropped partial or a mis-indexed head is off by the size of
the data, orders of magnitude over these bars.  Run with -s to print each kernel's worst error as a fraction of its bar.

The maxpool uses fmaxf, which drops a NaN where torch propagates it; no test depends on that."""
import pytest
import torch
import torch.nn.functional as F

from dinounet_b200 import config as cfg
from dinounet_b200 import lib as L
from oracle import dinounet_oracle as O
from tests.gpu_helpers import TD, U, P, check, stream, ulp16
from tests.gpu_helpers import bar16 as _bar16

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [L.BF16, L.F16]
DNAME = {L.BF16: "bf16", L.F16: "f16"}
GELU_SLOPE = 1.13                    # sup |GELU'(x)| = 1.1289 (at x = sqrt(2))
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


def _r16(x, dtype):
    return x.to(TD[dtype]).double()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(shape, seed, scale=1.0, dt=torch.float32):
    return (torch.randn(shape, generator=_gen(seed), device=DEV) * scale).to(dt)


def _nan(shape, dt):
    return torch.full(shape, float("nan"), device=DEV, dtype=dt)


def _check(kernel, what, got, ref, bar):
    return check(_WORST, kernel, what, got, ref, bar)


def _call(fn, *args):
    lib = L.load()
    L.check(getattr(lib, fn)(*args, stream()), fn)


def _id(prefix, case):
    return prefix + "-".join(str(int(c)) for c in case)


# ============================================================================================ case tables
# Each table lists the shape arguments of one kernel.  The engine's own launches for dinounet_s/b/l at (B=2, S=512) must
# all appear here (test_engine_shapes_are_covered), beside the boundary cases on each side of the kernel's branches.
VIT_D = (384, 768, 1024)           # dinounet_s / b / l
B2, NTOK, NPATCH, LQ = 2, 1029, 1024, 5376

# (in16, D, rows, rows_in, rows_out, row_off, out_fp32)
LN_TABLE = []
for _D in VIT_D:
    LN_TABLE += [(0, _D, B2 * NTOK, 0, 0, 0, 0),             # ViT ln1 / ln2 over B * ntok rows (last 8-row block partial)
                 (0, _D, B2 * NPATCH, NTOK, NPATCH, 5, 1),    # ViT taps: the patch rows of each image, fp32 out
                 (0, _D, B2 * LQ, 0, 0, 0, 0),                # adapter query / FFN norm over the fp32 query stream
                 (0, _D, B2 * NPATCH, 0, 0, 0, 0),            # adapter feat_norm on a tap
                 (1, _D, B2 * LQ, 0, 0, 0, 0)]                # query / FFN norm over the 16-bit query stream
for _in16 in (0, 1):
    for _o32 in (0, 1):
        LN_TABLE += [(_in16, 4096, B2 * NTOK, 0, 0, 0, _o32),  # ViT-7B width: the generic kernel
                     (_in16, 260, 13, 0, 0, 0, _o32),          # generic kernel, D % 128 != 0, one partial block
                     (_in16, 384, 1031, 0, 0, 0, _o32)]        # register kernel, partial last block
LN_TABLE += [(0, 4096, B2 * NPATCH, NTOK, NPATCH, 5, 1), (0, 260, 3 * 12, 13, 12, 1, 0)]

# (rows, D, rows_in, rows_out, row_off)
CAST_TABLE = [(B2 * 4096, _D, LQ, 4096, 0) for _D in VIT_D] + [(B2 * NPATCH, 384, NTOK, NPATCH, 5), (3 * 12, 1024, 13, 12, 1)]
PATCHIFY_TABLE = [(2, 512), (3, 128)]                               # (B, S)
PREFIX_TABLE = [(B2, NTOK, 5, _D) for _D in VIT_D + (4096,)] + [(3, 69, 5, 128)]   # (B, ntok, n_prefix, D)
STEM_TABLE = [(2, 512), (3, 128)]                                   # (B, S)
MAXPOOL_TABLE = [(2, 256, 256, 64), (3, 64, 64, 64)]                # (B, H, W, C)
# (B, H, W, C, planes, act)
DW_TABLE = ([(B2, 32, 32, _C, 3, L.ACT_GELU) for _C in (96, 192, 256, 1024)] + [(B2, 8, 8, 96, 3, L.ACT_GELU)]
            + [(B2, _r, _r, _C, 1, L.ACT_NONE) for _r in (128, 64, 32, 16) for _C in (32, 64, 128, 256)])
# (B, H, Ht, D, base_fp32, base rows per image, base row offset)
TAIL_TABLE = []
for _D in VIT_D:
    TAIL_TABLE += [(B2, 128, 32, _D, 0, 128 * 128, 0),       # x4 up-kernel, 16-bit base (the ConvT output UP)
                   (B2, 64, 32, _D, 1, LQ, 0),               # x2 up-kernel, base = level-2 rows of the fp32 query stream
                   (B2, 32, 32, _D, 1, LQ, 4096),            # identity: generic kernel
                   (B2, 16, 32, _D, 1, LQ, 5120)]            # down-sampling: generic kernel
TAIL_TABLE += [(B2, 128, 32, 384, 1, 128 * 128, 0), (B2, 64, 32, 384, 0, LQ, 0), (B2, 32, 32, 384, 0, LQ, 4096),
               (B2, 16, 32, 384, 0, LQ, 5120)]               # the other base type (16-bit query stream, fp32 UP)
# (B, Hv, dh): Hv = S / 16 at 512^2 (dh = D / 32 for s/b/l, 128 for ViT-7B); 56 / 58 / 64 straddle the 200 KB slab limit
MSDA_TABLE = [(B2, 32, _dh) for _dh in (12, 24, 32, 128)] + [(1, _hv, _dh) for _hv in (56, 58, 64) for _dh in (12, 24, 32)]
# (B, rows, C, ldx): chunk 64 below 1024 rows, 256 below 8192, 2048 from there; ldx = 2C is the FAPM shortcut layout
IN_TABLE = [(B2, _rows, _C, _ld) for _rows in (256, 1023, 1024, 4096, 8191, 8192, 16384, 65536, 262144)
            for _C in (32, 64, 128, 256) if _rows * _C <= 1 << 23 for _ld in (_C, 2 * _C)]
FAPM = ((32, 128), (64, 64), (128, 32), (256, 16))                  # (channels, side) of the four FAPM scales at 512^2
SE_GATE_TABLE = [(B2, _C, _C // 16, _r * _r) for _C, _r in FAPM]   # (B, C, Cr, rows)
SE_APPLY_TABLE = [(B2, _r * _r, _C, 2 * _C if _C != 256 else 256) for _C, _r in FAPM]   # (B, rows, C, ldsc)
FILM_TABLE = [(B2 * _r * _r, 256) for _, _r in FAPM]                # (rows, R)
SEG_TABLE = [(B2, 512 * 512, _n) for _n in (2, 8, 9, 128)]          # (B, rows, ncls)


def _msda_path(Hv, dh, option):
    """The layout b2u_msda_forward picks (msda.cu: the first (dh, heads per CTA, pitch) whose slab fits 200 KB, in the
    order listed there; option 1 == 1 forces the warp-per-query kernel, option 1 == 2 skips the padded one-head layouts)."""
    if option != 1:
        layouts = ([(32, 1, 32), (24, 1, 32), (12, 1, 16)] if option != 2 else []) + \
                  [(12, 8, 96), (24, 4, 96), (32, 2, 64), (12, 2, 24), (24, 1, 24), (32, 1, 32)]
        for d, hpc, pitch in layouts:
            if d == dh and Hv * Hv * pitch * 2 <= 200 * 1024:
                return f"smem{d}x{hpc}p{pitch}"
    return "warp"


# ============================================================================================ LayerNorm
def _ln_rows(n, D, seed):
    """Rows whose |mean| is up to ~30x their std (the ViT residual stream), std spread over two decades."""
    g = _gen(seed)
    mu = torch.randn(n, 1, generator=g, device=DEV) * 10
    mu[::3] = 0
    sd = torch.exp(torch.randn(n, 1, generator=g, device=DEV) * 0.7)
    return mu + sd * torch.randn(n, D, generator=g, device=DEV)


@pytest.mark.parametrize("dtype", DTYPES, ids=DNAME.get)
@pytest.mark.parametrize("case", LN_TABLE, ids=lambda c: _id("in16o32-D-rows-rin-rout-off=", c))
def test_layernorm(case, dtype):
    """b2u_layernorm (fp32 in) / b2u_layernorm16 (16-bit in), 16-bit or fp32 out, optional row remap.

    Bar: the kernel sums a row as a tree of depth k = D/128 + 7 (D/128 vectors per lane, two levels inside a vector,
    five shuffles), so the mean is within e_m = (k + 1) u mean|x|.  The centred square sum is within (k + 3) u of
    itself plus the second-order D e_m^2 from the mean's error; rsqrtf adds 2 ulp, so rstd has relative error
    eps_r = (k + 3) u / 2 + 4u + e_m^2 / (2 (var + eps)).  Then |y - ref| <= |g| rstd (e_m + |x - mean| eps_r)
    + 4u (|g x_hat| + |b|), plus the 16-bit output rounding.  Rows of the output buffer past `rows` and the input rows the
    remap skips hold NaN: a kernel that reads a skipped row or writes past the end shows up."""
    in16, D, rows, rows_in, rows_out, off, out32 = case
    td = TD[dtype]
    nimg = rows // rows_out if rows_out else 1
    n_in = nimg * rows_in if rows_out else rows
    x = _ln_rows(n_in, D, seed=D + rows)
    if in16:
        x = x.to(td)
    if rows_out:
        xv = x.view(nimg, rows_in, D)
        xv[:, :off] = float("nan")
        xv[:, off + rows_out:] = float("nan")
        xs = xv[:, off:off + rows_out].reshape(rows, D)
    else:
        xs = x
    g, b = _randn(D, 1), _randn(D, 2, 0.5)
    eps = cfg.LN_EPS_VIT if D != 260 else cfg.LN_EPS_ADAPTER
    out = _nan((rows + 8, D), torch.float32 if out32 else td)
    _call("b2u_layernorm16" if in16 else "b2u_layernorm", P(x), P(out), P(g), P(b), rows, D, eps, rows_in, rows_out, off,
          out32, dtype)
    torch.cuda.synchronize()
    assert torch.isnan(out[rows:].float()).all(), "rows past the end were written"
    xd = xs.double()
    mean = xd.mean(-1, keepdim=True)
    xc = xd - mean
    var = (xc * xc).mean(-1, keepdim=True)
    rstd = (var + eps).rsqrt()
    ref = xc * rstd * g.double() + b.double()
    k = D // 128 + 7
    e_m = (k + 1) * U * xd.abs().mean(-1, keepdim=True)
    eps_r = (k + 3) * U / 2 + 4 * U + e_m ** 2 / (2 * (var + eps))
    prop = g.double().abs() * rstd * (e_m + xc.abs() * eps_r) + 4 * U * ((xc * rstd * g.double()).abs() + b.double().abs())
    bar = prop if out32 else _bar16(ref, prop, dtype)
    _check("layernorm" + ("16" if in16 else ""), f"layernorm{case}", out[:rows], ref, bar)


# ============================================================================================ row gathers (bit-exact)
@pytest.mark.parametrize("dtype", DTYPES, ids=DNAME.get)
@pytest.mark.parametrize("case", CAST_TABLE, ids=lambda c: _id("rows-D-rin-rout-off=", c))
def test_cast_and_copy_rows(case, dtype):
    """b2u_cast_rows (fp32 -> 16-bit, round to nearest even) and b2u_copy_rows16 (16-bit gather) against torch's own
    conversion and slicing, bit for bit.  Skipped source rows hold NaN; output rows past the end keep NaN."""
    rows, D, rows_in, rows_out, off = case
    td = TD[dtype]
    nimg = rows // rows_out
    src = _randn((nimg, rows_in, D), rows + D, 3.0)
    src[:, :off] = float("nan")
    src[:, off + rows_out:] = float("nan")
    want = src[:, off:off + rows_out].reshape(rows, D).to(td)
    out = _nan((rows + 8, D), td)
    _call("b2u_cast_rows", P(src), P(out), rows, D, rows_in, rows_out, off, dtype)
    src16 = src.to(td)
    out16 = _nan((rows + 8, D), td)
    _call("b2u_copy_rows16", P(src16), P(out16), rows, D, rows_in, rows_out, off)
    torch.cuda.synchronize()
    assert torch.equal(out[:rows], want), "cast_rows differs from torch's rounding"
    assert torch.equal(out16[:rows], want), "copy_rows16 differs from the slice"
    assert torch.isnan(out[rows:].float()).all() and torch.isnan(out16[rows:].float()).all(), "rows past the end written"


@pytest.mark.parametrize("dtype", DTYPES, ids=DNAME.get)
@pytest.mark.parametrize("case", PATCHIFY_TABLE, ids=lambda c: _id("B-S=", c))
def test_patchify(case, dtype):
    """b2u_patchify == F.unfold(x, 16, stride=16) rounded to the ViT type, bit for bit."""
    B, S = case
    x = _randn((B, 3, S, S), S + B, 2.0)
    out = _nan((B * (S // 16) ** 2, 768), TD[dtype])
    _call("b2u_patchify", P(x), P(out), B, S, dtype)
    torch.cuda.synchronize()
    assert torch.equal(out, F.unfold(x, 16, stride=16).transpose(1, 2).reshape(-1, 768).to(TD[dtype]))


@pytest.mark.parametrize("case", PREFIX_TABLE, ids=lambda c: _id("B-ntok-npre-D=", c))
def test_write_prefix(case):
    """b2u_write_prefix writes the cls + storage tokens into rows [0, n_prefix) of every image and nothing else: every
    other row keeps its sentinel value, bit for bit."""
    B, ntok, npre, D = case
    X = _randn((B * ntok, D), D + 7, 1.0)
    X0 = X.clone()
    prefix = _randn((npre, D), D + 8, 1.0)
    _call("b2u_write_prefix", P(X), P(prefix), B, ntok, npre, D)
    torch.cuda.synchronize()
    want = X0.view(B, ntok, D).clone()
    want[:, :npre] = prefix
    assert torch.equal(X, want.view(B * ntok, D))


# ============================================================================================ SPM stem + maxpool
@pytest.mark.parametrize("dtype", DTYPES, ids=DNAME.get)
@pytest.mark.parametrize("case", STEM_TABLE, ids=lambda c: _id("B-S=", c))
def test_stem_conv0(case, dtype):
    """b2u_stem_conv0: Conv2d(3, 64, 3, s2, p1) in fp32, the conv output rounded to 16 bits (reproduced), folded BN,
    ReLU.  The 27-term fp32 sum is within d = 27 u sum|w x| of the float64 conv; the two roundings of that value may land
    one ulp apart, so r16 is off by at most ulp16(|conv| + d) + d, scaled by |scale|; the affine adds 2u of its terms
    and ReLU is 1-Lipschitz.  Borders (padding on the top / left) are part of the checked output."""
    B, S = case
    x = _randn((B, 3, S, S), S + 11, 1.5)
    w = _randn((64, 3, 3, 3), 12, 27 ** -0.5)
    sc, sh = _randn(64, 13).abs() + 0.5, _randn(64, 14, 0.5)
    out = _nan((B, S // 2, S // 2, 64), TD[dtype])
    _call("b2u_stem_conv0", P(x), P(w), P(sc), P(sh), P(out), B, S, dtype)
    torch.cuda.synchronize()
    conv = F.conv2d(x.double(), w.double(), stride=2, padding=1)
    d = 27 * U * F.conv2d(x.double().abs(), w.double().abs(), stride=2, padding=1)
    r = _r16(conv, dtype)
    scd, shd = sc.double()[None, :, None, None], sh.double()[None, :, None, None]
    ref = F.relu(r * scd + shd)
    prop = scd * (ulp16(conv.abs() + d, dtype) + d) + 2 * U * ((r * scd).abs() + shd.abs())
    _check("stem_conv0", f"stem{case}", out.permute(0, 3, 1, 2), ref, _bar16(ref, prop, dtype))


@pytest.mark.parametrize("dtype", DTYPES, ids=DNAME.get)
@pytest.mark.parametrize("case", MAXPOOL_TABLE, ids=lambda c: _id("B-H-W-C=", c))
def test_maxpool(case, dtype):
    """b2u_maxpool3x3s2 == F.max_pool2d(3, 2, 1), bit for bit, including windows whose values are all negative at the
    top / left padding and inside the image (padding must act as -inf, not 0)."""
    B, H, W, Cc = case
    x = _randn((B, H, W, Cc), H + Cc, 1.0)
    x[:, :9, :9] = -x[:, :9, :9].abs() - 0.01
    x[:, 20:29, 30:41] = -x[:, 20:29, 30:41].abs() - 0.01
    x = x.to(TD[dtype])
    out = _nan((B, H // 2, W // 2, Cc), TD[dtype])
    _call("b2u_maxpool3x3s2", P(x), P(out), B, H, W, Cc, dtype)
    torch.cuda.synchronize()
    want = F.max_pool2d(x.permute(0, 3, 1, 2).double(), 3, 2, 1).to(TD[dtype]).permute(0, 2, 3, 1)
    assert (out[:, :4, :4].float() < 0).all()
    assert torch.equal(out, want)


# ============================================================================================ depthwise conv
def _planes(H, W, planes):
    """(first row, height, width) of each plane of one image."""
    if planes == 1:
        return [(0, H, W)]
    return [(0, 2 * H, 2 * W), (4 * H * W, H, W), (5 * H * W, H // 2, W // 2)]


@pytest.mark.parametrize("dtype", DTYPES, ids=DNAME.get)
@pytest.mark.parametrize("case", DW_TABLE, ids=lambda c: _id("B-H-W-C-planes-act=", c))
def test_dwconv3x3(case, dtype):
    """b2u_dwconv3x3 per plane against a float64 depthwise conv (zero padding at every plane's own border).

    The fp32 sum (bias + 9 taps) is within d = 10 u (sum|w x| + |bias|).  Without activation the bar is that plus the
    16-bit output rounding.  With GELU the conv output is rounded to 16 bits before the GELU (reproduced): the two
    roundings may differ by ulp16(|conv| + d) + d, carried through sup|GELU'| = 1.13, and the fp32 erf-based GELU adds
    8u |x|.  Border rows / columns of each plane and its interior are checked separately."""
    B, H, W, Cc, planes, act = case
    td = TD[dtype]
    pl = _planes(H, W, planes)
    rows = sum(ph * pw for _, ph, pw in pl)
    x = _randn((B, rows, Cc), H + Cc + planes, 1.0, td)
    w = _randn((Cc, 1, 3, 3), Cc + 1, 1 / 3)
    bias = _randn(Cc, Cc + 2, 0.3)
    w9 = w.reshape(Cc, 9).t().contiguous()
    out = _nan((B, rows, Cc), td)
    _call("b2u_dwconv3x3", P(x), P(out), P(w9), P(bias), B, H, W, Cc, planes, act, dtype)
    torch.cuda.synchronize()
    for k, (r0, ph, pw) in enumerate(pl):
        t = x[:, r0:r0 + ph * pw].double().transpose(1, 2).reshape(B, Cc, ph, pw)
        conv = F.conv2d(t, w.double(), bias.double(), padding=1, groups=Cc)
        d = 10 * U * (F.conv2d(t.abs(), w.double().abs(), bias.double().abs(), padding=1, groups=Cc))
        if act == L.ACT_GELU:
            r = _r16(conv, dtype)
            ref = F.gelu(r)
            prop = GELU_SLOPE * (ulp16(conv.abs() + d, dtype) + d) + 8 * U * r.abs()
        else:
            ref, prop = conv, d
        bar = _bar16(ref, prop, dtype)
        got = out[:, r0:r0 + ph * pw].transpose(1, 2).reshape(B, Cc, ph, pw)
        border = torch.zeros(ph, pw, dtype=torch.bool, device=DEV)
        border[0], border[-1], border[:, 0], border[:, -1] = True, True, True, True
        for name, m in (("border", border), ("interior", ~border)):
            _check("dwconv3x3", f"dwconv{case} plane {k} ({ph}x{pw}) {name}", got[..., m], ref[..., m], bar[..., m])


# ============================================================================================ adapter tail
@pytest.mark.parametrize("dtype", DTYPES, ids=DNAME.get)
@pytest.mark.parametrize("case", TAIL_TABLE, ids=lambda c: _id("B-H-Ht-D-base32-brows-boff=", c))
def test_tail_fuse(case, dtype):
    """b2u_tail_fuse: (base + bilinear(tap)) * scale + shift, the tap resized from Ht x Ht to H x H as
    F.interpolate(mode="bilinear", align_corners=False).  The base is a row slice at an offset inside a buffer with
    `base rows per image` rows per image (the engine's query stream Cst, stride Lq * D); rows outside the slice hold NaN.

    The bilinear weights are exact in fp32 at these integer ratios, so base + four weighted taps is within
    5u (|base| + sum w |tap|); the affine scales that by |scale| and adds 2u of its terms; then the 16-bit rounding."""
    B, H, Ht, D, base32, brows, boff = case
    td = TD[dtype]
    tap = _randn((B * Ht * Ht, D), H + D, 1.0)
    base_buf = _randn((B, brows, D), H + D + 1, 1.0, torch.float32 if base32 else td)
    base_buf[:, :boff] = float("nan")
    base_buf[:, boff + H * H:] = float("nan")
    sc, sh = _randn(D, 3).abs() + 0.5, _randn(D, 4, 0.5)
    out = _nan((B * H * H, D), td)
    _call("b2u_tail_fuse", base_buf.data_ptr() + boff * D * base_buf.element_size(), base32, brows * D, P(tap), P(out),
          P(sc), P(sh), B, H, H, Ht, Ht, D, dtype)
    torch.cuda.synchronize()
    t = tap.double().view(B, Ht, Ht, D).permute(0, 3, 1, 2)
    up = F.interpolate(t, size=(H, H), mode="bilinear", align_corners=False)
    up_abs = F.interpolate(t.abs(), size=(H, H), mode="bilinear", align_corners=False)
    bd = base_buf[:, boff:boff + H * H].double().view(B, H, H, D).permute(0, 3, 1, 2)
    scd, shd = sc.double()[None, :, None, None], sh.double()[None, :, None, None]
    pre = bd + up
    ref = pre * scd + shd
    prop = scd * 5 * U * (bd.abs() + up_abs) + 2 * U * ((pre * scd).abs() + shd.abs())
    got = out.view(B, H, H, D).permute(0, 3, 1, 2)
    _check("tail_fuse", f"tail_fuse{case}", got, ref, _bar16(ref, prop, dtype))


# ============================================================================================ deformable attention
def _msda_ref_points(Hv):
    """Float64 reference point (x, y) of every query: cell centres of the 2Hv, Hv and Hv/2 levels."""
    pts = []
    for g in (2 * Hv, Hv, Hv // 2):
        c = (torch.arange(g, dtype=torch.float64, device=DEV) + 0.5) / g
        yy, xx = torch.meshgrid(c, c, indexing="ij")
        pts.append(torch.stack([xx.reshape(-1), yy.reshape(-1)], -1))
    return torch.cat(pts, 0)


_MSDA_IDS = [f"B{b}-Hv{hv}-dh{dh}-opt{o}-{_msda_path(hv, dh, o)}" for b, hv, dh in MSDA_TABLE for o in (0, 1, 2)]


@pytest.mark.parametrize("dtype", DTYPES, ids=DNAME.get)
@pytest.mark.parametrize("case", [(b, hv, dh, o) for b, hv, dh in MSDA_TABLE for o in (0, 1, 2)], ids=_MSDA_IDS)
def test_msda_forward(case, dtype):
    """b2u_msda_forward (16 heads x 4 points, one Hv x Hv level) against float64 O.msda_core on the same float64
    locations (reference point + fp32 offset / Hv) and softmaxed weights.  The test id names the kernel layout that
    msda.cu's selection rule picks for (Hv, dh, option 1).

    Offsets: head 0 samples exactly at pixel -0.5 (point 0) and Hv - 0.5 (point 1) on both axes, head 1 on one axis
    each, point 2 of head 2 and point 3 of head 3 lie 1000 pixels outside the map; the rest are N(0, 3) pixels.
    Bar: the kernel's location is within 4u (4 Hv + 2|offset|) pixels of the float64 one, moving a sample by at most
    2 max|v| per pixel; __expf and the softmax normalisation leave the weights within 40u relative; 16 fmas add 16u;
    together 64u sum_p aw_p sum_c w_c |v_c| plus the location term, plus the 16-bit output rounding."""
    B, Hv, dh, option = case
    td, heads = TD[dtype], 16
    HW = Hv * Hv
    Lq = 21 * HW // 4
    value = _randn((B, HW, heads, dh), Hv + dh, 1.0, td)
    off = _randn((B, Lq, heads, 4, 2), Hv + dh + 1, 3.0)
    logits = _randn((B, Lq, heads, 4), Hv + dh + 2, 2.0)
    ref_pts = _msda_ref_points(Hv)                     # [Lq, 2]
    rx, ry = ref_pts[:, 0], ref_pts[:, 1]
    off[:, :, 0, 0, 0], off[:, :, 0, 0, 1] = (-rx * Hv).float(), (-ry * Hv).float()
    off[:, :, 0, 1, 0], off[:, :, 0, 1, 1] = ((1 - rx) * Hv).float(), ((1 - ry) * Hv).float()
    off[:, :, 1, 0, 0], off[:, :, 1, 1, 1] = (-rx * Hv).float(), ((1 - ry) * Hv).float()
    off[:, :, 2, 2] = 1000.0
    off[:, :, 3, 3] = -1000.0
    offaw = torch.cat([off.reshape(B * Lq, heads * 8), logits.reshape(B * Lq, heads * 4)], 1).contiguous()
    out = _nan((B * Lq, heads * dh), td)
    lib = L.load()
    lib.b2u_set_option(1, option)
    try:
        L.check(lib.b2u_msda_forward(P(value), P(offaw), P(out), B, Hv, Hv, heads, dh, 4, dtype, stream()), "msda")
        torch.cuda.synchronize()
    finally:
        lib.b2u_set_option(1, 0)
    offd = off.double()
    loc = ref_pts[None, :, None, None, None, :] + offd.view(B, Lq, heads, 1, 4, 2) / Hv
    aw = F.softmax(logits.double(), -1).view(B, Lq, heads, 1, 4)
    v64 = value.double()
    ref = O.msda_core(v64, [(Hv, Hv)], loc, aw)
    sabs = O.msda_core(v64.abs(), [(Hv, Hv)], loc, aw)
    loc_px = 4 * U * (4 * Hv + 2 * offd.abs().sum(-1))                            # [B, Lq, heads, 4]
    loc_term = (aw.view(B, Lq, heads, 4) * loc_px).sum(-1) * 2 * v64.abs().max()   # [B, Lq, heads]
    prop = 64 * U * sabs + loc_term.repeat_interleave(dh, -1)
    _check("msda_forward", f"msda{case}", out.view(B, Lq, heads * dh), ref, _bar16(ref, prop, dtype))


# ============================================================================================ InstanceNorm
def _in_chunk(rows):
    return 2048 if rows >= 8192 else (256 if rows >= 1024 else 64)


def _in_stats_ref(xd, Cc):
    """Float64 sum and centred square sum of xd [B, rows, C], and their bars for b2u_in_stats.

    The kernel sums x - x0 (x0 = the image's first pixel) per chunk: a per-thread serial sum over chunk / rows_par rows,
    a serial sum over the rows_par row lanes, then a serial sum over the chunks, so a sum is a tree of depth
    k = chunk / rows_par + rows_par + nchunks.  sum x = rows x0 + that, within k u sum|x - x0| + u (rows |x0| + |sum|).
    The square sum is taken about each chunk's own mean m_c and merged with n_c (m_c - mean)^2 (Chan et al.): within
    (k + 4) u sum (x - m_c)^2 for the sums of squares, 2u sum |x - x0| |x - m_c| for the rounding of x - x0, and
    n_c e_c (2 |m_c - mean| + e_c) per chunk for the merge, e_c = (k + 2) u sum_c |x - x0| / n_c."""
    B, rows, _ = xd.shape
    chunk = _in_chunk(rows)
    rows_par = 256 // (Cc // 8)
    nch = (rows + chunk - 1) // chunk
    k = -(-chunk // rows_par) + rows_par + nch
    s = xd.sum(1)
    mean = s / rows
    m2 = ((xd - mean[:, None]) ** 2).sum(1)
    d = xd - xd[:, :1]
    bar_s = k * U * d.abs().sum(1) + U * (rows * xd[:, 0].abs() + s.abs())
    bar_q = torch.zeros_like(s)
    for c0 in range(0, rows, chunk):
        xc, dc = xd[:, c0:c0 + chunk], d[:, c0:c0 + chunk]
        n_c = xc.shape[1]
        m_c = xc.mean(1, keepdim=True)
        e_c = (k + 2) * U * dc.abs().sum(1) / n_c
        bar_q = bar_q + (k + 4) * U * ((xc - m_c) ** 2).sum(1) + 2 * U * (dc.abs() * (xc - m_c).abs()).sum(1) \
            + n_c * e_c * (2 * (m_c[:, 0] - mean).abs() + e_c)
    return s, m2, bar_s, bar_q


def _in_apply_ref(xd, s, m2, bar_s, bar_q, g, be, eps, dtype):
    """Float64 InstanceNorm + LeakyReLU(0.01) from the exact statistics, and the bar for b2u_in_apply run on the kernel's
    statistics: their error (bar_s / rows in the mean, bar_q / (2 rows (var + eps)) relative in rstd), rsqrtf's 2 ulp,
    2u for the divisions by rows, then 4u of the affine's terms and the 16-bit output rounding."""
    rows = xd.shape[1]
    mean, var = (s / rows)[:, None], (m2 / rows)[:, None]
    rstd = (var + eps).rsqrt()
    gd, bd = g.double(), be.double()
    xc = xd - mean
    t = xc * rstd * gd + bd
    ref = torch.where(t > 0, t, 0.01 * t)
    e_mean = (bar_s / rows)[:, None] + 2 * U * mean.abs()
    eps_r = ((bar_q / rows)[:, None] + 2 * U * var) / (2 * (var + eps)) + 4 * U
    prop = gd.abs() * rstd * (e_mean + xc.abs() * (eps_r + U)) + 4 * U * ((xc * rstd * gd).abs() + bd.abs())
    return ref, _bar16(ref, prop, dtype)


def _in_input(B, rows, Cc, ldx, seed, td):
    """Channel means up to 8x the channel std (the stats are shifted sums for that reason); columns past C of an
    ldx = 2C row are the shortcut half the statistics must not read."""
    g = _gen(seed)
    mu = torch.linspace(-4, 4, Cc, device=DEV)
    sd = torch.exp(torch.linspace(-1, 1, Cc, device=DEV))[torch.randperm(Cc, generator=g, device=DEV)]
    buf = torch.randn(B, rows, ldx, generator=g, device=DEV) * 30
    buf[..., :Cc] = mu + sd * torch.randn(B, rows, Cc, generator=g, device=DEV)
    return buf.to(td)


def _run_in(xbuf, B, rows, Cc, ldx, work, dtype):
    sums = _nan((B, Cc, 2), torch.float32)
    _call("b2u_in_stats", P(xbuf), ldx, P(sums), P(work), B, rows, Cc, dtype)
    return sums


def _check_in(xbuf, sums, B, rows, Cc, ldx, dtype, what, apply=True):
    xd = xbuf.view(B, rows, ldx)[..., :Cc].double()
    s, m2, bar_s, bar_q = _in_stats_ref(xd, Cc)
    _check("in_stats(sum)", f"{what} sum", sums[..., 0], s, bar_s)
    _check("in_stats(M2)", f"{what} centred square sum", sums[..., 1], m2, bar_q)
    if not apply:
        return m2
    td = TD[dtype]
    g, be = _randn(Cc, Cc + 5), _randn(Cc, Cc + 6, 0.5)
    y = _nan((B * rows, Cc), td)
    _call("b2u_in_apply", P(xbuf), ldx, P(y), Cc, P(sums), P(g), P(be), B, rows, Cc, cfg.IN_EPS, dtype)
    torch.cuda.synchronize()
    ref, bar = _in_apply_ref(xd, s, m2, bar_s, bar_q, g, be, cfg.IN_EPS, dtype)
    _check("in_apply", f"{what} apply", y.view(B, rows, Cc), ref, bar)
    return m2


@pytest.mark.parametrize("dtype", DTYPES, ids=DNAME.get)
@pytest.mark.parametrize("case", IN_TABLE, ids=lambda c: _id("B-rows-C-ldx=", c))
def test_in_stats_apply(case, dtype):
    """b2u_in_stats (per-image, per-channel sum and centred square sum) and b2u_in_apply (InstanceNorm + LeakyReLU)
    against float64, bars as derived in _in_stats_ref / _in_apply_ref.  A second launch gives the same bits."""
    B, rows, Cc, ldx = case
    lib = L.load()
    xbuf = _in_input(B, rows, Cc, ldx, rows + Cc + ldx, TD[dtype])
    work = torch.zeros(int(lib.b2u_in_stats_work_floats(B, rows, Cc)), device=DEV)
    sums = _run_in(xbuf, B, rows, Cc, ldx, work, dtype)
    again = _run_in(xbuf, B, rows, Cc, ldx, work, dtype)
    torch.cuda.synchronize()
    assert torch.equal(sums, again), "a repeated launch gives different bits"
    _check_in(xbuf, sums, B, rows, Cc, ldx, dtype, f"in{case}")


@pytest.mark.parametrize("dtype", DTYPES, ids=DNAME.get)
@pytest.mark.parametrize("k_sigma", [5, 20, 200])
def test_in_stats_outlier_first_pixel(k_sigma, dtype):
    """The statistics shift every sum by the image's first pixel.  Here that pixel sits k_sigma standard deviations from
    the channel mean (a hot pixel at (0, 0), a padded border), at the largest InstanceNorm of a 512^2 forward
    (262144 rows x 32 channels).  Squares taken about that shift would leave the variance as the difference of two
    sums k_sigma^2 times larger than it; the bars are those of test_in_stats_apply, and the normalised output is held
    to its 16-bit ulp."""
    B, rows, Cc = 2, 262144, 32
    lib = L.load()
    x = _randn((B, rows, Cc), 77, 1.0) + 0.3
    sign = torch.where(torch.arange(Cc, device=DEV) % 2 == 0, 1.0, -1.0)
    x[:, 0] = 0.3 + k_sigma * sign
    x = x.to(TD[dtype])
    work = torch.zeros(int(lib.b2u_in_stats_work_floats(B, rows, Cc)), device=DEV)
    sums = _run_in(x, B, rows, Cc, Cc, work, dtype)
    torch.cuda.synchronize()
    xd = x.double()
    m2 = ((xd - xd.mean(1, keepdim=True)) ** 2).sum(1)
    rel = ((sums[..., 1].double() - m2).abs() / m2).max().item()
    _NOTES.append(f"in_stats first pixel {k_sigma:>3d} sigma off ({DNAME[dtype]}): variance relative error {rel:.2e}")
    _check_in(x, sums, B, rows, Cc, Cc, dtype, f"outlier {k_sigma} sigma")


def test_in_stats_shared_workspace_sequence():
    """One workspace serves every InstanceNorm of a 512^2 forward, of different (rows, C), as the engine's `in_work`
    does, followed by calls with other batch sizes: the self-resetting tickets must leave each call correct (one call's
    partials must not land on another call's tickets), a replay of the whole sequence must give the same bits, and two
    identical images in one call must get identical statistics."""
    lib = L.load()
    dtype, td = L.F16, torch.float16
    seq = []
    for Cc, r in FAPM:
        ld = 2 * Cc if Cc != 256 else Cc
        seq += [(B2, r * r, Cc, ld), (B2, r * r, Cc, Cc), (B2, r * r, Cc, Cc)]
    seq += [(B2, 128 * 128, 128, 128), (B2, 256 * 256, 64, 64), (B2, 512 * 512, 32, 32)]
    seq += [(3, 1023, 64, 128), (1, 8191, 256, 256)]
    wfl = max(int(lib.b2u_in_stats_work_floats(*c[:3])) for c in seq)
    work = torch.zeros(wfl, device=DEV)
    inputs = [_in_input(*c, seed=i, td=td) for i, c in enumerate(seq)]
    twin = inputs[-3].clone()
    twin[1] = twin[0]
    seq.append(seq[-3])
    inputs.append(twin)
    first = [_run_in(xb, *c, work, dtype) for xb, c in zip(inputs, seq)]
    second = [_run_in(xb, *c, work, dtype) for xb, c in zip(inputs, seq)]
    torch.cuda.synchronize()
    for i, (a, b_, xb, c) in enumerate(zip(first, second, inputs, seq)):
        assert torch.equal(a, b_), f"call {i} {c}: replay differs"
        _check_in(xb, a, *c, dtype, f"call {i} {c}", apply=False)
    assert torch.equal(first[-1][0], first[-1][1]), "identical images got different statistics"


# ============================================================================================ FiLM, SE, seg head
@pytest.mark.parametrize("dtype", DTYPES, ids=DNAME.get)
@pytest.mark.parametrize("case", FILM_TABLE, ids=lambda c: _id("rows-R=", c))
def test_film(case, dtype):
    """b2u_film: z = gamma * z_in + beta, gamma|beta rows [rows, 2R], z_in the second half of a [rows, 2R] row.
    Bar: 2u (|gamma z| + |beta|) for the product and sum, plus the 16-bit output rounding."""
    rows, R = case
    td = TD[dtype]
    gb, zz = _randn((rows, 2 * R), rows + 1, 1.0, td), _randn((rows, 2 * R), rows + 2, 1.0, td)
    z = _nan((rows, R), td)
    _call("b2u_film", P(gb), P(zz), 2 * R, R, P(z), rows, R, dtype)
    torch.cuda.synchronize()
    g, b, zi = gb[:, :R].double(), gb[:, R:].double(), zz[:, R:].double()
    ref = g * zi + b
    _check("film", f"film{case}", z, ref, _bar16(ref, 2 * U * ((g * zi).abs() + b.abs()), dtype))


@pytest.mark.parametrize("case", SE_GATE_TABLE, ids=lambda c: _id("B-C-Cr-rows=", c))
def test_se_gate(case):
    """b2u_se_gate: sigmoid(W2 relu(W1 mean + b1) + b2) from the statistics' channel sums.  Hidden unit 0 has a zero
    weight row and zero bias (exactly 0 before and after the ReLU); unit 1, where there is one, is far below 0.
    Bar: mean within u; hidden within (C + 1) u (|W1| |mean| + |b1|) + |W1| e_mean; pre-activation a within
    (Cr + 1) u (|W2| h + |b2|) + |W2| e_h; sigmoid' <= 1/4, and __expf's (2 + 1.2|a|) ulp adds
    g (1 - g)(4 + 2|a|) u, the division 4u g."""
    B, Cc, Cr, rows = case
    sums = torch.zeros(B, Cc, 2, device=DEV)
    sums[..., 0] = _randn((B, Cc), Cc, 0.7 * rows)
    sums[..., 1] = float("nan")                        # the gate reads only the sums
    w1, b1 = _randn((Cr, Cc), Cc + 1, Cc ** -0.5), _randn(Cr, Cc + 2, 0.1)
    w2, b2 = _randn((Cc, Cr), Cc + 3, Cr ** -0.5), _randn(Cc, Cc + 4, 0.1)
    w1[0], b1[0] = 0.0, 0.0
    if Cr > 1:
        b1[1] = -100.0
    gate = _nan((B, Cc), torch.float32)
    _call("b2u_se_gate", P(sums), P(w1), P(b1), P(w2), P(b2), P(gate), B, Cc, Cr, rows)
    torch.cuda.synchronize()
    p = sums[..., 0].double() / rows
    W1, B1, W2, B2_ = w1.double(), b1.double(), w2.double(), b2.double()
    pre = p @ W1.t() + B1
    h = F.relu(pre)
    a = h @ W2.t() + B2_
    ref = torch.sigmoid(a)
    assert (h[:, 0] == 0).all() and (pre[:, 0] == 0).all()
    e_p = U * p.abs()
    e_h = (Cc + 1) * U * (p.abs() @ W1.abs().t() + B1.abs()) + e_p @ W1.abs().t()
    e_a = (Cr + 1) * U * (h @ W2.abs().t() + B2_.abs()) + e_h @ W2.abs().t()
    bar = 0.25 * e_a + ref * (1 - ref) * (4 + 2 * a.abs()) * U + 4 * U * ref
    _check("se_gate", f"se_gate{case}", gate, ref, bar)


@pytest.mark.parametrize("dtype", DTYPES, ids=DNAME.get)
@pytest.mark.parametrize("case", SE_APPLY_TABLE, ids=lambda c: _id("B-rows-C-ldsc=", c))
def test_se_apply(case, dtype):
    """b2u_se_apply: out = t * gate[b, c] + shortcut.  For C < 256 the shortcut is the second half of a [rows, 2C] row
    (ldsc = 2C, the shortcut projection's columns); for C = 256 it is the FiLM output (ldsc = R), produced here by
    b2u_film.  Bar: 2u (|t gate| + |shortcut|) plus the 16-bit output rounding."""
    B, rows, Cc, ldsc = case
    td = TD[dtype]
    t = _randn((B * rows, Cc), rows + Cc, 1.0, td)
    if ldsc == 2 * Cc:
        rs = _randn((B * rows, 2 * Cc), rows + Cc + 1, 1.0, td)
        sc_ptr, sc = rs.data_ptr() + Cc * rs.element_size(), rs[:, Cc:]
    else:
        R = ldsc
        gb, zz = _randn((B * rows, 2 * R), 5, 1.0, td), _randn((B * rows, 2 * R), 6, 1.0, td)
        z = _nan((B * rows, R), td)
        _call("b2u_film", P(gb), P(zz), 2 * R, R, P(z), B * rows, R, dtype)
        sc_ptr, sc = z.data_ptr(), z
    gate = torch.rand(B, Cc, generator=_gen(Cc), device=DEV)
    out = _nan((B * rows, Cc), td)
    _call("b2u_se_apply", P(t), sc_ptr, ldsc, P(gate), P(out), B, rows, Cc, dtype)
    torch.cuda.synchronize()
    tg = t.double().view(B, rows, Cc) * gate.double()[:, None]
    scd = sc.double().reshape(B, rows, Cc)
    ref = tg + scd
    _check("se_apply", f"se_apply{case}", out.view(B, rows, Cc), ref, _bar16(ref, 2 * U * (tg.abs() + scd.abs()), dtype))


@pytest.mark.parametrize("dtype", DTYPES, ids=DNAME.get)
@pytest.mark.parametrize("case", SEG_TABLE, ids=lambda c: _id("B-rows-ncls=", c))
def test_seg_head(case, dtype):
    """b2u_seg_head: InstanceNorm (from the kernel's own statistics) + LeakyReLU, the activation rounded to 16 bits
    (reproduced), 1x1 conv to ncls fp32 logits, first-maximum argmax labels.  ncls <= 8 runs kernel8.

    Bar: the per-channel affine a = rsqrt(var + eps) gamma, b = beta - mean a is within 8u |a| and
    u |beta| + 10u |mean a| + u |b|, so the activation u is within e_u = 8u |x a| + 10u |mean a| + u |beta| + u |b|
    + 2u |u|; its two 16-bit roundings may differ by e_t = ulp16(|u| + e_u) + e_u; the logit is within
    sum_c |w| e_t + (C + 1) u (sum_c |w t| + |bias|).  Labels must equal the first argmax of the kernel's own logits,
    and the float64 argmax wherever the top two reference logits are further apart than their bars."""
    B, rows, ncls = case
    Cc, td = 32, TD[dtype]
    lib = L.load()
    x = (_randn((B * rows, Cc), ncls, 2.0) + 0.5).to(td)
    work = torch.zeros(int(lib.b2u_in_stats_work_floats(B, rows, Cc)), device=DEV)
    sums = _run_in(x, B, rows, Cc, Cc, work, dtype)
    g, be = _randn(Cc, 1), _randn(Cc, 2, 0.5)
    w, wb = _randn((ncls, Cc), ncls + 3, Cc ** -0.5), _randn(ncls, ncls + 4, 0.5)
    logits = _nan((B, ncls, rows), torch.float32)
    labels = torch.full((B, rows), 255, device=DEV, dtype=torch.uint8)
    _call("b2u_seg_head", P(x), P(sums), P(g), P(be), cfg.IN_EPS, P(w), P(wb), P(logits), P(labels), B, rows, Cc, ncls,
          dtype)
    torch.cuda.synchronize()
    s = sums.double()
    mean, var = s[..., 0] / rows, s[..., 1] / rows
    a = (var + cfg.IN_EPS).rsqrt() * g.double()
    bb = be.double() - mean * a
    xd = x.double().view(B, rows, Cc)
    u = xd * a[:, None] + bb[:, None]
    lu = torch.where(u > 0, u, 0.01 * u)
    t = _r16(lu, dtype)
    W, Wb = w.double(), wb.double()
    ref = (t @ W.t() + Wb).transpose(1, 2)                                       # [B, ncls, rows]
    e_u = 8 * U * (xd * a[:, None]).abs() + (10 * U * (mean * a).abs() + U * be.double().abs() + U * bb.abs())[:, None] \
        + 2 * U * u.abs()
    e_t = ulp16(lu.abs() + e_u, dtype) + e_u
    bar = (e_t @ W.abs().t() + (Cc + 1) * U * (t.abs() @ W.abs().t() + Wb.abs())).transpose(1, 2)
    _check("seg_head", f"seg_head{case}", logits, ref, bar)
    assert torch.equal(labels.long(), logits.argmax(1)), "labels are not the first argmax of the logits"
    if ncls > 1:
        top2, idx2 = ref.topk(2, dim=1)
        bar_top = bar.gather(1, idx2)
        clear = (top2[:, 0] - top2[:, 1]) > bar_top.sum(1)
        assert torch.equal(labels.long()[clear], idx2[:, 0][clear]), "labels disagree with the float64 argmax"


# ============================================================================================ shape-drift guard
def _key(fname, args):
    """The shape arguments of one engine launch, as listed in this file's tables (None: not a kernel tested here)."""
    a = list(args)
    if fname in ("b2u_layernorm", "b2u_layernorm16"):
        return "LN_TABLE", (int(fname == "b2u_layernorm16"), a[5], a[4], a[7], a[8], a[9], a[10])
    if fname in ("b2u_cast_rows", "b2u_copy_rows16"):
        return "CAST_TABLE", (a[2], a[3], a[4], a[5], a[6])
    if fname == "b2u_patchify":
        return "PATCHIFY_TABLE", (a[2], a[3])
    if fname == "b2u_write_prefix":
        return "PREFIX_TABLE", (a[2], a[3], a[4], a[5])
    if fname == "b2u_stem_conv0":
        return "STEM_TABLE", (a[5], a[6])
    if fname == "b2u_maxpool3x3s2":
        return "MAXPOOL_TABLE", (a[2], a[3], a[4], a[5])
    if fname == "b2u_dwconv3x3":
        return "DW_TABLE", (a[4], a[5], a[6], a[7], a[8], a[9])
    if fname == "b2u_tail_fuse":
        return "TAIL_TABLE", (a[7], a[8], a[10], a[12], a[1], a[2] // a[12])
    if fname == "b2u_msda_forward":
        return "MSDA_TABLE", (a[4], a[7])
    if fname == "b2u_in_stats":
        return "IN_TABLE", (a[4], a[5], a[6], a[1])
    if fname == "b2u_in_apply":
        return "IN_TABLE", (a[7], a[8], a[9], a[1])
    if fname == "b2u_film":
        return "FILM_TABLE", (a[5], a[6], a[2], a[3])
    if fname == "b2u_se_gate":
        return "SE_GATE_TABLE", (a[6], a[7], a[8], a[9])
    if fname == "b2u_se_apply":
        return "SE_APPLY_TABLE", (a[5], a[6], a[7], a[2])
    if fname == "b2u_seg_head":
        return "SEG_TABLE", (a[9], a[10], a[12], a[11])
    return None


def _covered():
    """Table name -> the keys _key produces for each listed case."""
    return {
        "LN_TABLE": set(LN_TABLE), "CAST_TABLE": set(CAST_TABLE), "PATCHIFY_TABLE": set(PATCHIFY_TABLE),
        "PREFIX_TABLE": set(PREFIX_TABLE), "STEM_TABLE": set(STEM_TABLE), "MAXPOOL_TABLE": set(MAXPOOL_TABLE),
        "DW_TABLE": set(DW_TABLE), "TAIL_TABLE": {c[:6] for c in TAIL_TABLE}, "MSDA_TABLE": {c[1:] for c in MSDA_TABLE},
        "IN_TABLE": set(IN_TABLE), "FILM_TABLE": {(r, R, 2 * R, R) for r, R in FILM_TABLE},
        "SE_GATE_TABLE": set(SE_GATE_TABLE), "SE_APPLY_TABLE": set(SE_APPLY_TABLE),
        "SEG_TABLE": {(b, r, n, 32) for b, r, n in SEG_TABLE},
    }


@pytest.mark.parametrize("variant", ["dinounet_s", "dinounet_b", "dinounet_l"])
def test_engine_shapes_are_covered(variant):
    """Builds the engine's real launch plan at (B=2, S=512) and checks that every non-GEMM, non-attention launch has its
    shape arguments in this file's case tables, so a change of the plan's shapes names the kernel whose tests no longer
    cover it.  The tensor-core GEMM, QKV and attention launches are guarded the same way, with their epilogue signatures,
    by test_gpu_tc_kernels.py::test_plan_shapes_are_covered."""
    from dinounet_b200.engine import ForwardEngine
    from tests.test_gpu_tc_kernels import TC_ENTRY_POINTS
    eng = ForwardEngine(variant, O.make_state_dict(variant, 2, seed=0), 2, torch.device(DEV))
    plan, _ = eng.build_plan(B2, 512)
    tables = _covered()
    missing, n = [], 0
    for name, fn, args in plan.calls:
        fname = fn.__name__
        if fname in TC_ENTRY_POINTS:
            continue
        k = _key(fname, args)
        assert k is not None, f"{name}: {fname} has no case table in this file"
        n += 1
        if k[1] not in tables[k[0]]:
            missing.append(f"{name} ({fname}): {k[1]} not in {k[0]}")
    del plan, eng
    torch.cuda.empty_cache()
    assert n > 50
    assert not missing, "\n".join(missing)
