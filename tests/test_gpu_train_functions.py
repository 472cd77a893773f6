"""-m gpu: the training path's autograd Functions outside the matrix products (dinounet_b200/train_path.py; kernels in
csrc/fp32_tier.cu, csrc/train_bwd.cu and msda.cu), one Function at a time, against torch float64 autograd on the GPU started
from the same fp32 values.  The shapes are the ones a dinounet_b training step at 512^2 runs, plus the row counts on either
side of every reduction-split boundary of the backward kernels (1 / 8 / 64 splits at 2048 / 65536 rows, 1 / 8 / 32 at HW
4096 / 65536, the LayerNorm backward's one-row-per-warp limit of 9472 rows), and edge inputs: activation kinks hit exactly,
max-pool ties, samples outside the deformable-attention map, a dead SE hidden unit.

Bars (estimates: a few fp32 roundings per element, fp32 partial sums of at most ~4096 terms per thread):
  outputs and per-element gradients  max |got - ref| <= 2e-5 * max |ref|
  parameter gradients (row sums)     max |got - ref| <= 5e-5 * max |ref|
  exact where the op is exact        max-pool forward, TailAddF backward, zero-by-construction gradients
The upstream gradient is randn + 0.5: with a nonzero mean every reduction split adds coherently, so a dropped or doubled
split moves a parameter gradient by at least 1/64 of it, far above the bars.

Activation kinks: a pre-activation computed in fp32 can land on the other side of 0 from the fp64 one when it is within
rounding of 0.  dx of BN+ReLU and IN+LReLU is compared where the fp64 pre-activation is exactly 0 or farther than 1e-5
from 0, and at most 1e-5 of the elements may be left out; the inputs that make pre-activations exactly 0 pin the kink rule.
"""
import pytest
import torch
import torch.nn.functional as F

from dinounet_b200 import config as cfg
from dinounet_b200 import lib as L
from dinounet_b200 import train_path as TP
from oracle import dinounet_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
OUT_TOL = 2e-5          # outputs and per-element gradients
PARAM_TOL = 5e-5        # parameter gradients (sums over rows)
KINK = 1e-5             # pre-activations this close to 0 (but not 0) are left out of the dx comparison


def rnd(*shape, seed, scale=1.0, shift=0.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * scale + shift).float()


def upstream(shape, seed):
    return rnd(*shape, seed=seed, shift=0.5)


def lift(*ts):
    """fp64 leaves holding the same values as the fp32 tensors."""
    return [t.detach().double().requires_grad_() for t in ts]


def leaves(*ts):
    return [t.detach().clone().requires_grad_() for t in ts]


def check(got, ref, tol, what, mask=None):
    """max |got - ref| <= tol * max |ref| (over `mask` if given); returns the relative error."""
    got, ref = got.detach().double(), ref.detach().double()
    assert got.shape == ref.shape, f"{what}: shape {tuple(got.shape)} vs {tuple(ref.shape)}"
    if mask is not None:
        got, ref = got[mask], ref[mask]
    err = (got - ref).abs().max().item()                       # NaN (an unwritten element) fails the comparison below
    ref_max = max(ref.abs().max().item(), 1e-30)
    assert err <= tol * ref_max, f"{what}: max err {err:.3e} vs max |ref| {ref_max:.3e} (rel {err / ref_max:.3e}, bar {tol:.0e})"
    return err / ref_max


def report(case, errs):
    worst = max(errs.values())
    print(f"{case}: worst rel err {worst:.2e} (" + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()) + ")")


def kink_mask(pre):
    """Elements whose fp64 pre-activation is exactly 0 or farther than KINK from 0; asserts few are left out."""
    keep = (pre == 0) | (pre.abs() > KINK)
    dropped = int((~keep).sum())
    assert dropped <= KINK * pre.numel(), f"{dropped} of {pre.numel()} pre-activations within {KINK} of 0"
    return keep, dropped


# ------------------------------------------------------------------------------------------------ LayerNormF
@pytest.mark.parametrize("rows,D", [(7, 384), (9472, 768), (9473, 768), (10752, 768), (2048, 1024), (300, 200)])
def test_layernorm(rows, D):
    """f32_layernorm + f32_layernorm_bwd: one row per warp up to 9472 rows, grid-stride beyond (10752 = dinounet_b's query
    stream at B=2, 512^2)."""
    x, w, b = leaves(rnd(rows, D, seed=1, scale=2.0, shift=3.0), rnd(D, seed=2, scale=0.2, shift=1.0), rnd(D, seed=3, scale=0.2))
    y = TP.LayerNormF.apply(x, w, b, cfg.LN_EPS_ADAPTER)
    g = upstream(y.shape, 4)
    y.backward(g)
    xd, wd, bd = lift(x, w, b)
    yd = F.layer_norm(xd, (D,), wd, bd, cfg.LN_EPS_ADAPTER)
    yd.backward(g.double())
    report(f"LayerNormF rows {rows} D {D}", {
        "y": check(y, yd, OUT_TOL, "y"), "dx": check(x.grad, xd.grad, OUT_TOL, "dx"),
        "dw": check(w.grad, wd.grad, PARAM_TOL, "dw"), "db": check(b.grad, bd.grad, PARAM_TOL, "db")})


# ------------------------------------------------------------------------------------------------ InstNormLReLUF
@pytest.mark.parametrize("B,HW,C", [(2, 4095, 32), (2, 4096, 32), (1, 65535, 32), (1, 65536, 32), (2, 262144, 32), (3, 1024, 80)])
def test_instnorm_lrelu(B, HW, C):
    """f32_instnorm + f32_instnorm_bwd (1 / 8 / 32 row splits at HW < 4096 / < 65536 / more).  Channel 0 has gamma = beta = 0,
    so every pre-activation is exactly 0 and its parameter gradients take the LeakyReLU slope branch; channel 1 has mean 10
    and std 0.1 (the forward's fp32 mean costs mean/std * 2^-24 in xhat)."""
    x = rnd(B * HW, C, seed=5)
    x[:, 1] = rnd(B * HW, seed=6, scale=0.1, shift=10.0)
    w, b = rnd(C, seed=7, scale=0.5, shift=2.0), rnd(C, seed=8, scale=0.5)
    w[0], b[0] = 0.0, 0.0
    w[1] = 1.0          # keeps that channel's fp32-mean error in the pre-activation (<= ~5e-6) inside the kink window
    x, w, b = leaves(x, w, b)
    y = TP.InstNormLReLUF.apply(x, w, b, B, HW)
    g = upstream(y.shape, 9)
    y.backward(g)
    xd, wd, bd = lift(x, w, b)
    pre = F.instance_norm(xd.view(B, HW, C).permute(0, 2, 1), weight=wd, bias=bd, eps=cfg.IN_EPS)
    yd = F.leaky_relu(pre, 0.01).permute(0, 2, 1).reshape(B * HW, C)
    yd.backward(g.double())
    keep, dropped = kink_mask(pre.detach().permute(0, 2, 1).reshape(B * HW, C))
    assert (pre.detach()[:, 0] == 0).all()
    report(f"InstNormLReLUF B {B} HW {HW} C {C} (dx: {dropped} near-kink elements left out)", {
        "y": check(y, yd, OUT_TOL, "y"), "dx": check(x.grad, xd.grad, OUT_TOL, "dx", keep),
        "dw": check(w.grad, wd.grad, PARAM_TOL, "dw"), "db": check(b.grad, bd.grad, PARAM_TOL, "db"),
        "dw[0]": check(w.grad[0], wd.grad[0], PARAM_TOL, "dw of the gamma = beta = 0 channel"),
        "db[0]": check(b.grad[0], bd.grad[0], PARAM_TOL, "db of the gamma = beta = 0 channel")})


# ------------------------------------------------------------------------------------------------ BNActF
@pytest.mark.parametrize("act", [L.ACT_NONE, L.ACT_RELU], ids=["none", "relu"])
@pytest.mark.parametrize("rows,C", [(2048, 64), (2049, 80), (65536, 768), (65537, 64), (131072, 80), (131072, 768)])
def test_bn_act(rows, C, act):
    """Eval-mode BatchNorm (+ ReLU): f32_bn_act + f32_bn_act_bwd (1 / 8 / 64 row splits at <= 2048 / <= 65536 / more).  Every
    7th row equals the running mean and every 4th channel has beta = 0: those pre-activations are exactly 0."""
    x = rnd(rows, C, seed=10)
    rm, rv = rnd(C, seed=11, scale=0.5), torch.rand(C, generator=torch.Generator(device=DEV).manual_seed(12), device=DEV) + 0.5
    x[::7] = rm
    gamma, beta = rnd(C, seed=13, scale=0.3, shift=2.0), rnd(C, seed=14, scale=0.5)
    beta[::4] = 0.0
    x, gamma, beta = leaves(x, gamma, beta)
    y = TP.BNActF.apply(x, gamma, beta, rm, rv, act)
    g = upstream(y.shape, 15)
    y.backward(g)
    xd, gd, bd = lift(x, gamma, beta)
    pre = (xd - rm.double()) / torch.sqrt(rv.double() + cfg.BN_EPS) * gd + bd      # F.batch_norm(training=False), written out
    yd = F.relu(pre) if act == L.ACT_RELU else pre
    yd.backward(g.double())
    keep, dropped = kink_mask(pre.detach()) if act == L.ACT_RELU else (None, 0)
    assert (pre.detach()[::7, ::4] == 0).all()
    report(f"BNActF rows {rows} C {C} act {act} (dx: {dropped} near-kink elements left out)", {
        "y": check(y, yd, OUT_TOL, "y"), "dx": check(x.grad, xd.grad, OUT_TOL, "dx", keep),
        "dgamma": check(gamma.grad, gd.grad, PARAM_TOL, "dgamma"), "dbeta": check(beta.grad, bd.grad, PARAM_TOL, "dbeta")})


# ------------------------------------------------------------------------------------------------ ActF
@pytest.mark.parametrize("act", [L.ACT_GELU, L.ACT_RELU, L.ACT_LRELU], ids=["gelu", "relu", "lrelu"])
def test_act(act):
    """f32_act + f32_act_bwd on n = 1 000 003 (a partial last block), with exact zeros and +-8."""
    n = 1_000_003
    x = rnd(n, seed=16, scale=3.0)
    x[::97] = 0.0
    x[1::101], x[2::103] = 8.0, -8.0
    (x,) = leaves(x)
    y = TP.ActF.apply(x, act)
    g = upstream(y.shape, 17)
    y.backward(g)
    (xd,) = lift(x)
    yd = {L.ACT_GELU: F.gelu, L.ACT_RELU: F.relu, L.ACT_LRELU: lambda t: F.leaky_relu(t, 0.01)}[act](xd)
    yd.backward(g.double())
    report(f"ActF act {act} n {n}", {"y": check(y, yd, OUT_TOL, "y"), "dx": check(x.grad, xd.grad, OUT_TOL, "dx")})


# ------------------------------------------------------------------------------------------------ DWConvF
def _dwconv_ref(xd, wd, bd, B, planes_hw):
    """Depthwise 3x3 / pad 1 + bias on token-major planes [B, sum(ph*pw), C], one F.conv2d per plane."""
    C = xd.shape[1]
    xs = xd.view(B, -1, C)
    outs, off = [], 0
    for ph, pw in planes_hw:
        p = xs[:, off:off + ph * pw].reshape(B, ph, pw, C).permute(0, 3, 1, 2)
        outs.append(F.conv2d(p, wd, bd, padding=1, groups=C).permute(0, 2, 3, 1).reshape(B, ph * pw, C))
        off += ph * pw
    assert off == xs.shape[1]
    return torch.cat(outs, 1).reshape(-1, C)


def _dwconv_case(B, H, Wd, C, planes, planes_hw, seed):
    x, W, b = leaves(rnd(B * sum(h * w for h, w in planes_hw), C, seed=seed), rnd(C, 1, 3, 3, seed=seed + 1, scale=0.3),
                     rnd(C, seed=seed + 2, scale=0.3))
    y = TP.DWConvF.apply(x, W, b, B, H, Wd, planes)
    g = upstream(y.shape, seed + 3)
    y.backward(g)
    xd, Wdd, bd = lift(x, W, b)
    yd = _dwconv_ref(xd, Wdd, bd, B, planes_hw)
    yd.backward(g.double())
    report(f"DWConvF planes {planes} B {B} H {H} W {Wd} C {C} ({x.shape[0]} rows)", {
        "y": check(y, yd, OUT_TOL, "y"), "dx": check(x.grad, xd.grad, OUT_TOL, "dx"),
        "dw": check(W.grad, Wdd.grad, PARAM_TOL, "dw"), "db": check(b.grad, bd.grad, PARAM_TOL, "db")})


@pytest.mark.parametrize("B,H,C", [(2, 8, 96), (2, 32, 192), (13, 32, 192)])
def test_dwconv_planes3(B, H, C):
    """The ConvFFN pyramid [16n | 4n | n] = planes 2Hx2W, HxW, H/2xW/2 (32 = dinounet_b at 512^2); f32_dwconv_wgrad takes 1,
    8 and 64 splits of the B * 21/4 H^2 rows."""
    _dwconv_case(B, H, H, C, 3, [(2 * H, 2 * H), (H, H), (H // 2, H // 2)], seed=20)


@pytest.mark.parametrize("B,H,W,C", [(2, 128, 128, 32), (5, 128, 128, 32), (2, 16, 16, 256), (1, 24, 40, 64)])
def test_dwconv_planes1(B, H, W, C):
    """One H x W image per batch item (FAPM refinement blocks); (5, 128, 128) takes 64 splits, (24, 40) is not square."""
    _dwconv_case(B, H, W, C, 1, [(H, W)], seed=30)


# ------------------------------------------------------------------------------------------------ MaxPoolF
@pytest.mark.parametrize("B,H,W,C", [(2, 256, 256, 64), (1, 10, 14, 64)])
def test_maxpool(B, H, W, C):
    """MaxPool2d(3, 2, 1) (the SPM stem at 512^2).  relu(randn) rounded to multiples of 0.25 ties windows among zeros and
    among positives: the gradient goes to the first maximum in row-major window order (ATen's rule)."""
    x0 = torch.round(torch.relu(rnd(B * H * W, C, seed=40)) * 4) / 4
    (x,) = leaves(x0)
    y = TP.MaxPoolF.apply(x, B, H, W)
    g = upstream(y.shape, 41)
    y.backward(g)
    (xd,) = lift(x)
    yd = F.max_pool2d(xd.view(B, H, W, C).permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1).reshape(y.shape)
    yd.backward(g.double())
    assert torch.equal(y.detach().double(), yd.detach()), "max-pool forward is not exact"
    report(f"MaxPoolF B {B} H {H} W {W} C {C}", {"y": 0.0, "dx": check(x.grad, xd.grad, OUT_TOL, "dx")})


# ------------------------------------------------------------------------------------------------ MSDAF
def _query_grid(h, w):
    """(gh, gw) of every query of the [16n | 4n | n] layout: planes 2h x 2w, h x w, h/2 x w/2 (row-major)."""
    rows = []
    for gh, gw in ((2 * h, 2 * w), (h, w), (h // 2, w // 2)):
        ry, rx = torch.meshgrid(torch.arange(gh, device=DEV), torch.arange(gw, device=DEV), indexing="ij")
        rows.append(torch.stack([rx.reshape(-1), ry.reshape(-1), torch.full_like(rx.reshape(-1), gw), torch.full_like(rx.reshape(-1), gh)], 1))
    return torch.cat(rows, 0)                                   # [Lq, 4] = (rx, ry, gw, gh)


@pytest.mark.parametrize("B,h,w,dh", [(2, 32, 32, 48), (1, 8, 8, 24), (1, 8, 12, 64)])
def test_msda(B, h, w, dh):
    """f32_msda_prep (locations bit for bit, attention weights vs softmax), b2u_msda_forward_f32 / backward_f32 and
    f32_msda_prep_bwd against grid_sample (O.msda_core) in fp64, built from the prologue's own fp32 locations and weights.
    Sampling positions have fractional pixel parts in [0.01, 0.99] (bilinear's derivative jumps at cell boundaries) and
    integer parts from -2 to the map size, so some samples fall outside the map and some straddle its border.  The
    non-square map pins the x / y axis order."""
    heads = cfg.DEFORM_HEADS
    Lq = h * w * 21 // 4
    gen = torch.Generator(device=DEV).manual_seed(50)
    q = _query_grid(h, w).double()                              # [Lq, 4]
    refx, refy = (q[:, 0] + 0.5) / q[:, 2], (q[:, 1] + 0.5) / q[:, 3]
    frac = lambda: 0.01 + 0.98 * torch.rand(B, Lq, heads, 4, generator=gen, device=DEV, dtype=torch.float64)
    px = torch.randint(-2, w + 1, (B, Lq, heads, 4), generator=gen, device=DEV).double() + frac()
    py = torch.randint(-2, h + 1, (B, Lq, heads, 4), generator=gen, device=DEV).double() + frac()
    offx = (px + 0.5) - refx[None, :, None, None] * w           # loc = ref + off / W  ->  pixel = loc * W - 0.5
    offy = (py + 0.5) - refy[None, :, None, None] * h
    off = torch.stack([offx, offy], -1).reshape(B * Lq, heads * 8)
    logits = torch.randn(B * Lq, heads * 4, generator=gen, device=DEV, dtype=torch.float64)
    offaw = torch.cat([off, logits], 1).float()
    value = rnd(B * h * w, heads * dh, seed=51)

    # the prologue on its own
    loc = torch.empty((B, Lq, heads, 1, 4, 2), dtype=torch.float32, device=DEV)
    attw = torch.empty((B, Lq, heads, 1, 4), dtype=torch.float32, device=DEV)
    TP._call("b2u_f32_msda_prep", offaw, loc, attw, B, h, w, heads)
    qf = _query_grid(h, w).float()
    o32 = offaw[:, :heads * 8].reshape(B, Lq, heads, 4, 2)
    # divide by a device tensor: torch turns `tensor / python scalar` into a multiply by the reciprocal, which is not
    # the correctly rounded quotient the kernel computes when W or H is not a power of 2
    Wt, Ht = torch.full_like(o32[..., 0], w), torch.full_like(o32[..., 1], h)
    want_x = ((qf[:, 0] + 0.5) / qf[:, 2])[None, :, None, None] + o32[..., 0] / Wt
    want_y = ((qf[:, 1] + 0.5) / qf[:, 3])[None, :, None, None] + o32[..., 1] / Ht
    assert torch.equal(loc.view(B, Lq, heads, 4, 2), torch.stack([want_x, want_y], -1)), "f32_msda_prep locations"
    a_err = check(attw.view(B, Lq, heads, 4), torch.softmax(offaw[:, heads * 8:].reshape(B, Lq, heads, 4), -1), 1e-6, "attention weights")
    outside = ((px <= -1) | (px >= w) | (py <= -1) | (py >= h)).double().mean().item()
    assert 0 < outside < 0.5

    # the Function
    value, offaw = leaves(value, offaw)
    y = TP.MSDAF.apply(value, offaw, B, h, w)
    g = upstream(y.shape, 52)
    y.backward(g)

    vd, locd, ad = lift(value, loc, attw)
    yd = O.msda_core(vd.view(B, h * w, heads, dh), [(h, w)], locd, ad)
    yd.backward(g.double().view(yd.shape))
    dloc = locd.grad.view(B * Lq, heads, 4, 2)
    da, a = ad.grad.view(B * Lq, heads, 4), attw.double().view(B * Lq, heads, 4)
    doff_ref = torch.stack([dloc[..., 0] / w, dloc[..., 1] / h], -1).reshape(B * Lq, heads * 8)
    dlogit_ref = (a * (da - (a * da).sum(-1, keepdim=True))).reshape(B * Lq, heads * 4)
    got = offaw.grad
    report(f"MSDAF B {B} h {h} w {w} dh {dh} ({outside:.1%} of samples outside the map)", {
        "attw": a_err, "y": check(y, yd.view(y.shape), OUT_TOL, "y"),
        "dvalue": check(value.grad, vd.grad.view(value.shape), OUT_TOL, "dvalue"),
        "doffsets": check(got[:, :heads * 8], doff_ref, OUT_TOL, "d sampling offsets"),
        "dlogits": check(got[:, heads * 8:], dlogit_ref, OUT_TOL, "d attention logits")})


# ------------------------------------------------------------------------------------------------ FiLMF
@pytest.mark.parametrize("px", [2 * 128 * 128, 7])
def test_film(px):
    """z = gamma * zp + beta (gb = (gamma | beta), zz = (zs | zp)); the zs half of dzz is exactly 0."""
    R = cfg.FAPM_RANK
    gb, zz = leaves(rnd(px, 2 * R, seed=60), rnd(px, 2 * R, seed=61))
    z = TP.FiLMF.apply(gb, zz)
    g = upstream(z.shape, 62)
    z.backward(g)
    gbd, zzd = lift(gb, zz)
    zd = gbd[:, :R] * zzd[:, R:] + gbd[:, R:]
    zd.backward(g.double())
    assert torch.equal(zz.grad[:, :R], torch.zeros_like(zz.grad[:, :R]))
    report(f"FiLMF px {px} R {R}", {"z": check(z, zd, OUT_TOL, "z"), "dgb": check(gb.grad, gbd.grad, OUT_TOL, "dgb"),
                                    "dzz": check(zz.grad, zzd.grad, OUT_TOL, "dzz")})


# ------------------------------------------------------------------------------------------------ SEF
@pytest.mark.parametrize("B,HW,C,hid", [(2, 16384, 32, 2), (2, 4096, 64, 4), (2, 1024, 128, 8), (2, 256, 256, 16), (3, 100, 80, 5)])
def test_squeeze_excitation(B, HW, C, hid):
    """out = t * sigmoid(W2 relu(W1 mean_hw(t) + b1) + b2) + sc (the FAPM SE blocks at 512^2).  Hidden unit 0 is dead
    (b1 = -50): its W1 row, its b1 and its W2 column get exactly 0."""
    t, sc = rnd(B * HW, C, seed=70, shift=0.3), rnd(B * HW, C, seed=71)
    w1, b1 = rnd(hid, C, 1, 1, seed=72, scale=0.1), rnd(hid, seed=73, scale=0.1, shift=2.0)
    w2, b2 = rnd(C, hid, 1, 1, seed=74, scale=0.5), rnd(C, seed=75, scale=0.5)
    b1[0] = -50.0
    t, sc, w1, b1, w2, b2 = leaves(t, sc, w1, b1, w2, b2)
    y = TP.SEF.apply(t, sc, w1, b1, w2, b2, B, HW)
    g = upstream(y.shape, 76)
    y.backward(g)
    td, scd, w1d, b1d, w2d, b2d = lift(t, sc, w1, b1, w2, b2)
    pooled = td.view(B, HW, C).mean(1)
    hdn = F.relu(pooled @ w1d.view(hid, C).t() + b1d)
    gate = torch.sigmoid(hdn @ w2d.view(C, hid).t() + b2d)
    yd = (td.view(B, HW, C) * gate[:, None, :] + scd.view(B, HW, C)).reshape(B * HW, C)
    yd.backward(g.double())
    assert (b1d.grad[1:] != 0).all(), "every other hidden unit is live"
    for what, got in (("dw1 of the dead unit", w1.grad[0]), ("db1 of the dead unit", b1.grad[0]), ("dw2 of the dead unit", w2.grad[:, 0])):
        assert torch.equal(got, torch.zeros_like(got)), what
    report(f"SEF B {B} HW {HW} C {C} hid {hid}", {
        "y": check(y, yd, OUT_TOL, "y"), "dt": check(t.grad, td.grad, OUT_TOL, "dt"), "dsc": check(sc.grad, scd.grad, OUT_TOL, "dsc"),
        "dw1": check(w1.grad, w1d.grad, PARAM_TOL, "dw1"), "db1": check(b1.grad, b1d.grad, PARAM_TOL, "db1"),
        "dw2": check(w2.grad, w2d.grad, PARAM_TOL, "dw2"), "db2": check(b2.grad, b2d.grad, PARAM_TOL, "db2")})


# ------------------------------------------------------------------------------------------------ TailAddF
@pytest.mark.parametrize("r", [128, 64, 32, 16])
def test_tail_add(r):
    """u = c + bilinear(tap h x h -> r x r, align_corners=False): x4, x2, same size and /2 from dinounet_b's 32 x 32 tap;
    the tap is frozen and du/dc is the identity, so dc == du bit for bit."""
    B, h, D = 2, 32, 768
    (c,) = leaves(rnd(B * r * r, D, seed=80))
    tap = rnd(B * h * h, D, seed=81)
    u = TP.TailAddF.apply(c, tap, B, r, h)
    g = upstream(u.shape, 82)
    u.backward(g)
    (cd,) = lift(c)
    up = F.interpolate(tap.double().view(B, h, h, D).permute(0, 3, 1, 2), size=(r, r), mode="bilinear", align_corners=False)
    ud = cd + up.permute(0, 2, 3, 1).reshape(B * r * r, D)
    assert torch.equal(c.grad, g), "TailAddF backward must pass du through unchanged"
    report(f"TailAddF B {B} h {h} r {r} D {D}", {"u": check(u, ud, OUT_TOL, "u"), "dc": 0.0})
