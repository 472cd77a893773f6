"""-m gpu: the TF32 tensor-core GEMM of the training path (csrc/gemm_tf32.cu, `b2u_tf32_gemm`) in every addressing mode
of its parameter block, against fp64 torch references computed on TF32-ROUNDED operands (round-to-nearest-away to 10
mantissa bits = cvt.rna.tf32.f32, emulated bit-exactly below): what remains is fp32 accumulation order, so the
tolerance is 2e-4 of the largest output (a misplaced chunk / swizzle / descriptor is an O(1) error).  Then the three
autograd Functions that use it (Linear, Conv3x3, ConvT2x2: forward, data gradient, weight gradient, bias gradient)
against fp64 autograd on the UNROUNDED operands at TF32's own precision (3e-3), and the same Functions on the fp32 SIMT
tier (`b2u_f32_gemm`) at 2e-5.

The reference formulas of this file are themselves checked WITHOUT a GPU by tests/test_tf32_gemm_refs_cpu.py, which runs
the same test bodies against a slow torch emulation of the parameter block's addressing (`DEV`, `raw_gemm` are the seams)."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from dinounet_b200 import lib as L

pytestmark = pytest.mark.gpu
TOL = 2e-4
DEV = "cuda"
TENSOR_FIELDS = ("A", "W", "out", "bias", "scale", "shift", "residual")


def raw_gemm(fn: str = "b2u_tf32_gemm", **f):
    """Fill a b2u_f32_gemm_params block from keyword fields (tensors for the pointer fields) and call the C-ABI."""
    p = L.F32GemmParams()
    for k, v in f.items():
        setattr(p, k, v.data_ptr() if isinstance(v, torch.Tensor) else int(v))
    dev = f["out"].device
    with torch.cuda.device(dev):
        L.check(getattr(L.load(), fn)(C.byref(p), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), fn)


def gemm(A, W, out, M, N, K, **f):
    f.setdefault("lda", A.shape[-1])
    f.setdefault("ldw", W.shape[-1])
    f.setdefault("ldc", out.shape[-1])
    if f.get("residual") is not None:
        f.setdefault("ldres", f["residual"].shape[-1])
    f = {k: v for k, v in f.items() if v is not None}
    raw_gemm(A=A, W=W, out=out, M=M, N=N, K=K, **f)


def tf32(t: torch.Tensor) -> torch.Tensor:
    """cvt.rna.tf32.f32: add half an ulp of the 10-bit mantissa to the magnitude, clear the low 13 bits."""
    i = t.detach().float().contiguous().view(torch.int32)
    sign = i & -0x80000000
    mag = ((i & 0x7FFFFFFF) + 0x1000) & 0x7FFFE000
    return (sign | mag).view(torch.float32).double()


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * scale).float()


def check(out, ref, tol=None, what=""):
    tol = TOL if tol is None else tol
    assert torch.isfinite(out).all(), f"{what}: non-finite output (unwritten elements?)"
    err = (out.double() - ref).abs().max().item()
    ref_max = ref.abs().max().item()
    assert err <= tol * max(ref_max, 1e-6), f"{what}: max err {err:.3e} vs max |ref| {ref_max:.3e}"
    return err / max(ref_max, 1e-6)


@pytest.mark.parametrize("M,N,K", [(128, 32, 32), (300, 70, 100), (1000, 200, 77), (5, 3, 9), (257, 129, 31), (4096, 256, 1024), (130, 33, 260)])
def test_plain_rows_bias_activation_residual(M, N, K):
    A, W, b, res = rnd(M, K, seed=1), rnd(N, K, seed=2, scale=0.2), rnd(N, seed=3), rnd(M, N, seed=4)
    out = torch.full((M, N), float("nan"), device=DEV)
    gemm(A, W, out, M, N, K, bias=b, residual=res)
    acc = tf32(A) @ tf32(W).t()
    check(out, acc + b.double() + res.double(), what=f"plain {M}x{N}x{K}")
    sc, sh = rnd(N, seed=5), rnd(N, seed=6)            # every epilogue stage: act1 -> scale/shift -> act2
    for act1, act2 in ((L.ACT_GELU, L.ACT_NONE), (L.ACT_RELU, L.ACT_LRELU)):
        out.fill_(float("nan"))
        gemm(A, W, out, M, N, K, bias=b, scale=sc, shift=sh, act1=act1, act2=act2)
        v = acc + b.double()
        v = F.gelu(v) if act1 == L.ACT_GELU else F.relu(v)
        v = v * sc.double() + sh.double()
        if act2 == L.ACT_LRELU:
            v = F.leaky_relu(v, 0.01)
        check(out, v, what=f"epilogue {act1}/{act2}")


def test_unaligned_leading_dimensions_take_the_scalar_paths():
    M, N, K = 200, 50, 45                                          # lda, ldw, ldc not multiples of 4
    A, W = rnd(M, K, seed=1), rnd(N, K, seed=2)
    big = torch.zeros((M, N + 3), device=DEV)
    gemm(A, W, big, M, N, K, ldc=N + 3, col_off=3)
    check(big[:, 3:], tf32(A) @ tf32(W).t(), what="ldc/col_off")
    assert (big[:, :3] == 0).all()
    acc = torch.ones((M, N), device=DEV)                            # accumulate: out += product
    gemm(A, W, acc, M, N, K, accumulate=1)
    check(acc, tf32(A) @ tf32(W).t() + 1.0, what="accumulate")


@pytest.mark.parametrize("M,N,K,ksplit", [(700, 96, 130, 1), (5000, 192, 64, 4), (70000, 27, 32, 16), (4100, 300, 384, 7), (100, 40, 48, 64)])
def test_transposed_operands_and_split_k(M, N, K, ksplit):
    """LinearF.backward: dx = dy W (w_mode 1); dW = dy^T x (a_trans + w_mode 1, K = rows, split-K atomics; the last case has
    more K slices than k-blocks: empty slices must add nothing)."""
    dy, W, x = rnd(M, N, seed=1), rnd(N, K, seed=2), rnd(M, K, seed=3)
    dx = torch.full((M, K), float("nan"), device=DEV)
    gemm(dy, W, dx, M, K, N, w_mode=1)
    check(dx, tf32(dy) @ tf32(W), what="dx")
    dW = torch.zeros((N, K), device=DEV)
    gemm(dy, x, dW, N, K, M, a_trans=1, w_mode=1, ksplit=ksplit)
    check(dW, tf32(dy).t() @ tf32(x), what=f"dW ksplit {ksplit}")


@pytest.mark.parametrize("B,H,Wd,Cin,Cout,stride", [(2, 16, 16, 32, 32, 1), (1, 32, 24, 64, 32, 1), (2, 16, 16, 3, 32, 2), (1, 24, 40, 20, 7, 1),
                                                    (2, 32, 32, 128, 64, 2), (1, 64, 64, 64, 32, 1)])
def test_conv3x3_forward_data_gradient_weight_gradient(B, H, Wd, Cin, Cout, stride):
    """Conv3x3F's three GEMMs: window on the A side (forward; data gradient with the flipped weights, stride 1) and on the W
    side (weight gradient, K = output pixels, split-K) against fp64 conv2d / its autograd on the TF32-rounded operands."""
    x = rnd(B * H * Wd, Cin, seed=1)
    Wt = rnd(Cout, Cin, 3, 3, seed=2, scale=0.2)
    b = rnd(Cout, seed=3)
    Wp = Wt.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()
    Ho, Wo = H // stride, Wd // stride
    y = torch.full((B * Ho * Wo, Cout), float("nan"), device=DEV)
    conv = L.CONV3X3_S2 if stride == 2 else L.CONV3X3_S1
    gemm(x, Wp, y, B * Ho * Wo, Cout, 9 * Cin, bias=b, conv=conv, Hin=H, Win=Wd, C=Cin, Cpad=Cin)
    xi = tf32(x).view(B, H, Wd, Cin).permute(0, 3, 1, 2)
    ref = F.conv2d(xi, tf32(Wt), b.double(), stride=stride, padding=1).permute(0, 2, 3, 1).reshape(B * Ho * Wo, Cout)
    check(y, ref, what="conv forward")
    dy = rnd(B * Ho * Wo, Cout, seed=4)
    dyi = tf32(dy).view(B, Ho, Wo, Cout).permute(0, 3, 1, 2)
    if stride == 1:
        dx = torch.full((B * H * Wd, Cin), float("nan"), device=DEV)
        gemm(dy, Wp, dx, B * H * Wd, Cin, 9 * Cout, conv=L.CONV3X3_S1, Hin=H, Win=Wd, C=Cout, Cpad=Cout, w_mode=2, w_cpad=Cin, ldw=9 * Cin)
        rdx = torch.nn.grad.conv2d_input((B, Cin, H, Wd), tf32(Wt), dyi, stride=1, padding=1).permute(0, 2, 3, 1).reshape(B * H * Wd, Cin)
        check(dx, rdx, what="conv data gradient")
    npix = B * Ho * Wo
    for ksplit in (1, 5):
        dWp = torch.zeros((Cout, 9 * Cin), device=DEV)
        gemm(dy, x, dWp, Cout, 9 * Cin, npix, a_trans=1, lda=Cout, w_mode=3, conv=conv, Hin=H, Win=Wd, C=Cin, Cpad=Cin, ksplit=ksplit)
        rdW = torch.nn.grad.conv2d_weight(xi, (Cout, Cin, 3, 3), dyi, stride=stride, padding=1).permute(0, 2, 3, 1).reshape(Cout, 9 * Cin)
        check(dWp, rdW, what=f"conv weight gradient ksplit {ksplit}")


def test_conv3x3_channel_padding_rows_are_zero():
    """Cpad > C (k = tap * Cpad + c with padded weight columns): forward ignores the padding, the weight gradient writes 0 there."""
    B, H, Wd, Cin, Cpad, Cout = 2, 16, 24, 20, 24, 12
    x, Wt, dy = rnd(B * H * Wd, Cin, seed=1), rnd(Cout, Cin, 3, 3, seed=2, scale=0.2), rnd(B * H * Wd, Cout, seed=3)
    Wp = torch.zeros((Cout, 9, Cpad), device=DEV)
    Wp[:, :, :Cin] = Wt.permute(0, 2, 3, 1).reshape(Cout, 9, Cin)
    Wp = Wp.reshape(Cout, 9 * Cpad).contiguous()
    y = torch.full((B * H * Wd, Cout), float("nan"), device=DEV)
    gemm(x, Wp, y, B * H * Wd, Cout, 9 * Cpad, conv=L.CONV3X3_S1, Hin=H, Win=Wd, C=Cin, Cpad=Cpad)
    xi = tf32(x).view(B, H, Wd, Cin).permute(0, 3, 1, 2)
    check(y, F.conv2d(xi, tf32(Wt), None, padding=1).permute(0, 2, 3, 1).reshape(B * H * Wd, Cout), what="padded forward")
    dWp = torch.zeros((Cout, 9 * Cpad), device=DEV)
    gemm(dy, x, dWp, Cout, 9 * Cpad, B * H * Wd, a_trans=1, lda=Cout, w_mode=3, conv=L.CONV3X3_S1, Hin=H, Win=Wd, C=Cin, Cpad=Cpad, ksplit=3)
    dyi = tf32(dy).view(B, H, Wd, Cout).permute(0, 3, 1, 2)
    rdW = torch.nn.grad.conv2d_weight(xi, (Cout, Cin, 3, 3), dyi, padding=1).permute(0, 2, 3, 1).reshape(Cout, 9, Cin)
    got = dWp.view(Cout, 9, Cpad)
    check(got[:, :, :Cin], rdW, what="padded weight gradient")
    assert (got[:, :, Cin:] == 0).all()


def test_pixel_shuffle_and_row_remap_epilogues():
    """ConvTranspose2d(k2, s2) = GEMM + 2x2 pixel shuffle (ps_*); row remaps on both sides (a_rows_*, rows_*)."""
    B, h, w, Cin, Cout = 2, 12, 20, 48, 24
    x, Wt, b = rnd(B * h * w, Cin, seed=1), rnd(Cin, Cout, 2, 2, seed=2, scale=0.3), rnd(Cout, seed=3)
    Wp = Wt.permute(2, 3, 1, 0).reshape(4 * Cout, Cin).contiguous()
    y = torch.full((B * 4 * h * w, Cout), float("nan"), device=DEV)
    gemm(x, Wp, y, B * h * w, 4 * Cout, Cin, bias=b.repeat(4).contiguous(), ps_cout=Cout, ps_h=h, ps_w=w)
    ref = F.conv_transpose2d(tf32(x).view(B, h, w, Cin).permute(0, 3, 1, 2), tf32(Wt), b.double(), stride=2)
    check(y, ref.permute(0, 2, 3, 1).reshape(B * 4 * h * w, Cout), what="pixel shuffle")
    # rows: read rows [5, 5+40) of every 64-row block of A, write them to rows [3, 3+40) of every 50-row block of out
    nb, N, K = 7, 36, 64
    A, W = rnd(nb * 64, K, seed=4), rnd(N, K, seed=5)
    out = torch.zeros((nb * 50, N), device=DEV)
    gemm(A, W, out, nb * 40, N, K, a_rows_in=40, a_rows_out=64, a_row_off=5, rows_in=40, rows_out=50, row_off=3)
    ref = torch.zeros((nb, 50, N), dtype=torch.float64, device=DEV)
    ref[:, 3:43] = tf32(A).view(nb, 64, K)[:, 5:45] @ tf32(W).t()
    check(out, ref.view(nb * 50, N), what="row remap")


def test_tensor_core_tier_matches_the_fp32_tier_and_counts_as_native():
    """Same call through both tiers: TF32's own error (about 1e-3 of the largest output), never more."""
    M, N, K = 3000, 384, 1536
    A, W = rnd(M, K, seed=1), rnd(N, K, seed=2, scale=0.05)
    a, b = torch.empty((M, N), device=DEV), torch.empty((M, N), device=DEV)
    n0 = L.launch_count()
    raw_gemm("b2u_tf32_gemm", A=A, W=W, out=a, M=M, N=N, K=K, lda=K, ldw=K, ldc=N)
    raw_gemm("b2u_f32_gemm", A=A, W=W, out=b, M=M, N=N, K=K, lda=K, ldw=K, ldc=N)
    assert L.launch_count() - n0 == 2
    err = (a - b).abs().max().item() / b.abs().max().item()
    print(f"tf32 vs fp32 tier, K={K}: {err:.2e}")
    assert 0 < err <= 3e-3


def test_autograd_functions_against_fp64_autograd():
    """LinearF / Conv3x3F / ConvT2x2F forward + backward on the tensor-core tier vs torch fp64 autograd (unrounded operands)
    at TF32's own precision."""
    _autograd_functions_against_fp64_autograd("tf32", 3e-3)


def test_fp32_tier_autograd_functions_against_fp64_autograd():
    """The same Functions and shapes on the fp32 SIMT tier (b2u_f32_gemm, the gradient goldens' tier) at fp32 accumulation's
    precision (2e-5, an estimate)."""
    _autograd_functions_against_fp64_autograd("fp32", 2e-5)


def _autograd_functions_against_fp64_autograd(tier, tol):
    """The stride-2 convolutions include the SPM's shapes at 512^2, whose data gradient is b2u_f32_conv3x3_dgrad on both
    tiers; the last transposed conv is the decoder's at 512^2, whose bias gradient sums 524288 rows (f32_colsum's 64-split
    branch)."""
    from dinounet_b200 import train_path as TP
    prev, TP._GEMM_TIER = TP._GEMM_TIER, tier
    try:
        def cmp(got, want, what):
            err = check(got.detach(), want.detach().double(), tol=tol, what=f"{tier} {what}")
            print(f"{tier} {what}: rel err {err:.2e}")

        M, K, N = 5000, 192, 96                                       # Linear with bias and residual
        x, W, b, r = [t.requires_grad_() for t in (rnd(M, K, seed=1), rnd(N, K, seed=2, scale=0.1), rnd(N, seed=3), rnd(M, N, seed=4))]
        y = TP.LinearF.apply(x, W, b, r)
        g = rnd(M, N, seed=5)
        y.backward(g)
        xd, Wd_, bd, rd = [t.detach().double().requires_grad_() for t in (x, W, b, r)]
        yd = F.linear(xd, Wd_, bd) + rd
        yd.backward(g.double())
        for got, want, what in ((y, yd, "y"), (x.grad, xd.grad, "dx"), (W.grad, Wd_.grad, "dW"), (b.grad, bd.grad, "db"), (r.grad, rd.grad, "dres")):
            cmp(got, want, "linear " + what)
        # Conv3x3: (B, H, Cin, Cout, stride); the stride-2 rows after the first two are the SPM's conv2..conv4 at 512^2
        for B, H, Cin, Cout, stride in ((2, 32, 64, 32, 1), (2, 32, 64, 32, 2), (2, 128, 64, 128, 2), (2, 64, 128, 256, 2),
                                        (2, 32, 256, 256, 2), (1, 24, 20, 7, 2)):
            Wd = H
            x, Wt, b = [t.requires_grad_() for t in (rnd(B * H * Wd, Cin, seed=6), rnd(Cout, Cin, 3, 3, seed=7, scale=0.1), rnd(Cout, seed=8))]
            y = TP.Conv3x3F.apply(x, Wt, b, B, H, Wd, stride)
            g = rnd(*y.shape, seed=9)
            y.backward(g)
            xd, Wtd, bd = [t.detach().double().requires_grad_() for t in (x, Wt, b)]
            yd = F.conv2d(xd.view(B, H, Wd, Cin).permute(0, 3, 1, 2), Wtd, bd, stride=stride, padding=1).permute(0, 2, 3, 1).reshape(y.shape)
            yd.backward(g.double())
            for got, want, what in ((y, yd, "y"), (x.grad, xd.grad, "dx"), (Wt.grad, Wtd.grad, "dW"), (b.grad, bd.grad, "db")):
                cmp(got, want, f"conv s{stride} {B}x{H}x{H}x{Cin}->{Cout} " + what)
        for B, h, w, Cin, Cout in ((2, 16, 16, 64, 32), (2, 256, 256, 64, 32)):          # ConvTranspose 2x2
            x, Wt, b = [t.requires_grad_() for t in (rnd(B * h * w, Cin, seed=10), rnd(Cin, Cout, 2, 2, seed=11, scale=0.1), rnd(Cout, seed=12))]
            y = TP.ConvT2x2F.apply(x, Wt, b, B, h, w)
            g = rnd(*y.shape, seed=13)
            y.backward(g)
            xd, Wtd, bd = [t.detach().double().requires_grad_() for t in (x, Wt, b)]
            yd = F.conv_transpose2d(xd.view(B, h, w, Cin).permute(0, 3, 1, 2), Wtd, bd, stride=2).permute(0, 2, 3, 1).reshape(y.shape)
            yd.backward(g.double())
            for got, want, what in ((y, yd, "y"), (x.grad, xd.grad, "dx"), (Wt.grad, Wtd.grad, "dW"), (b.grad, bd.grad, "db")):
                cmp(got, want, f"convT {B}x{h}x{w}x{Cin}->{Cout} " + what)
    finally:
        TP._GEMM_TIER = prev
