"""The persistent wgmma GEMM runs the epilogue of one tile while the MMA warps compute the next one, both through the single
fp32 accumulator tile in shared memory.  These shapes give every CTA at least 8 tiles and the shortest K the kernel allows
(one 64-wide k-block; 9 taps x 64 channels for the 3x3 convolution), so the main loop is as short as it gets next to the
epilogue: an accumulator tile overwritten before its epilogue has read it shows up as wrong elements.  Each instantiated
epilogue is checked element-wise against an fp32 torch reference, and a second launch must give identical bits."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from dinounet_b200 import lib as L
from oracle import dinounet_oracle as O
from tests.gpu_helpers import TD, P, gemm, stream

pytestmark = pytest.mark.gpu
DEV = "cuda"
M_BIG = 20000          # 157 row tiles: x 8 column tiles of 128 = 1256 tiles, about 9.5 per CTA on 132 SMs
# Every element within TOL x max|ref|.  The reference rounds to 16 bits in its own order, and a one-ulp difference of an
# intermediate (the rounded Linear output) is scaled by the affine factor or mixed by the RoPE rotation; an accumulator
# tile overwritten too early is off by the order of max|ref| itself.
TOL = {L.BF16: 2 ** -5, L.F16: 2 ** -8}
ULP = {L.BF16: 2 ** -7, L.F16: 2 ** -10}   # relative spacing of the 16-bit types


def _rand(*shape, dt=torch.float32, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(DEV).to(dt)


def _assert_close(got, ref, dtype):
    got, ref = got.float(), ref.float()
    assert torch.isfinite(got).all()
    err = (got - ref).abs()
    bad = err > TOL[dtype] * ref.abs().max()
    assert not bad.any(), f"{int(bad.sum())} elements off, max error {err.max().item():.3g} (max |ref| {ref.abs().max().item():.3g})"


def _twice(run, out):
    """Runs the launch twice and checks both give the same bits; returns the first result."""
    out.fill_(float("nan"))
    run()
    torch.cuda.synchronize()
    first = out.clone()
    out.fill_(float("nan"))
    run()
    torch.cuda.synchronize()
    assert torch.equal(first.view(torch.uint8), out.view(torch.uint8)), "two launches differ"
    return first


@pytest.mark.parametrize("dtype,act", [(L.BF16, 0), (L.F16, 0), (L.BF16, L.ACT_GELU), (L.F16, L.ACT_GELU)])
def test_overlap_plain_and_gelu(dtype, act):
    td = TD[dtype]
    M, N, K = M_BIG, 1024, 64
    A, W = _rand(M, K, dt=td), _rand(N, K, dt=td, scale=K ** -0.5, seed=1)
    bias = _rand(N, seed=2)
    out = torch.empty(M, N, device=DEV, dtype=td)
    got = _twice(lambda: gemm(A, W, out, dtype, bias=bias, act1=act), out)
    lin = A.float() @ W.float().t() + bias
    ref = F.gelu(lin.to(td).float()) if act == L.ACT_GELU else lin
    _assert_close(got, ref.to(td), dtype)


@pytest.mark.parametrize("act2", [L.ACT_RELU, L.ACT_LRELU])
@pytest.mark.parametrize("N", [1024, 64, 32])   # BLOCK_N 128, 64, 32
def test_overlap_affine_relu(act2, N):
    dtype, td = L.F16, torch.float16
    M = M_BIG if N == 1024 else M_BIG * (1024 // N)
    K = 64
    A, W = _rand(M, K, dt=td), _rand(N, K, dt=td, scale=K ** -0.5, seed=1)
    sc, sh = _rand(N, seed=3).abs() + 0.5, _rand(N, seed=4)
    out = torch.empty(M, N, device=DEV, dtype=td)
    got = _twice(lambda: gemm(A, W, out, dtype, scale=sc, shift=sh, act2=act2), out)
    y = (A.float() @ W.float().t()).to(td).float() * sc + sh
    ref = F.relu(y) if act2 == L.ACT_RELU else F.leaky_relu(y, 0.01)
    _assert_close(got, ref.to(td), dtype)


@pytest.mark.parametrize("dtype", [L.BF16, L.F16])
def test_overlap_fp32_residual(dtype):
    """LayerScale + fp32 residual stream (ViT proj / fc2 epilogue)."""
    td = TD[dtype]
    M, N, K = M_BIG, 1024, 64
    A, W = _rand(M, K, dt=td), _rand(N, K, dt=td, scale=K ** -0.5, seed=1)
    bias, gamma = _rand(N, seed=2), _rand(N, seed=3)
    R = _rand(M, N, seed=4)
    X = torch.empty(M, N, device=DEV)
    got = _twice(lambda: gemm(A, W, X, dtype, out_fp32=True, bias=bias, scale=gamma, residual=R, ldres=N), X)
    y = (A.float() @ W.float().t() + bias).to(td).float() * gamma
    # one unit in the last place of the 16-bit Linear output, scaled by gamma, plus fp32 rounding of the sum
    bound = 2 * ULP[dtype] * y.abs() + 1e-5 * (1 + R.abs())
    err = (got - (R + y)).abs()
    assert torch.isfinite(got).all()
    assert (err <= bound).all(), f"max error {err.max().item():.3g}"


@pytest.mark.parametrize("dtype", [L.BF16, L.F16])
def test_overlap_swiglu(dtype):
    td = TD[dtype]
    M, D, Hd = M_BIG, 64, 512           # N = 2 Hd = 1024 accumulator columns
    x = _rand(M, D, dt=td)
    w1, w2 = _rand(Hd, D, dt=td, scale=D ** -0.5, seed=1), _rand(Hd, D, dt=td, scale=D ** -0.5, seed=2)
    b1, b2 = _rand(Hd, seed=3, scale=0.2), _rand(Hd, seed=4, scale=0.2)
    Wp = torch.stack([w1.view(Hd // 32, 32, D), w2.view(Hd // 32, 32, D)], 1).reshape(2 * Hd, D).contiguous()
    bp = torch.stack([b1.view(Hd // 32, 32), b2.view(Hd // 32, 32)], 1).reshape(2 * Hd).contiguous()
    out = torch.empty(M, Hd, device=DEV, dtype=td)
    got = _twice(lambda: gemm(x, Wp, out, dtype, bias=bp, act1=L.ACT_SWIGLU, ldc=Hd), out)
    x1 = (x.float() @ w1.float().t() + b1).to(td)
    x2 = (x.float() @ w2.float().t() + b2).to(td)
    ref = F.silu(x1.float()).to(td).float() * x2.float()
    _assert_close(got, ref.to(td), dtype)


@pytest.mark.parametrize("dtype", [L.BF16, L.F16])
def test_overlap_qkv_rope(dtype):
    """QKV with RoPE and the head split, D = 64 (one head, one k-block): 3 x 64 columns = two column tiles, the second
    half empty."""
    td = TD[dtype]
    B, h, D, Hh = 300, 16, 64, 1
    hd, N = D // Hh, h * h + 5          # 78300 token rows: 612 row tiles x 2 column tiles
    lib = L.load()
    Y = _rand(B * N, D, dt=td)
    Wq = _rand(3 * D, D, dt=td, scale=D ** -0.5, seed=1)
    bias = _rand(3 * D, seed=2, scale=0.1)
    periods = 100.0 ** (2 * torch.arange(hd // 4, dtype=torch.float32) / (hd // 2))
    sin, cos = O.rope_sincos(periods, h, h)
    sin, cos = sin.to(DEV).contiguous(), cos.to(DEV).contiguous()
    qkv_out = torch.empty(3, B, Hh, N, hd, device=DEV, dtype=td)
    p = L.QkvParams()
    p.B, p.ntok, p.D, p.heads, p.prefix = B, N, D, Hh, 5
    p.A, p.lda, p.Wp, p.ldw, p.bias = P(Y), D, P(Wq), D, P(bias)
    p.rope_sin, p.rope_cos, p.dtype, p.rope_w = P(sin), P(cos), dtype, h
    p.q, p.k, p.v = P(qkv_out[0]), P(qkv_out[1]), P(qkv_out[2])
    got = _twice(lambda: L.check(lib.b2u_qkv_rope(C.byref(p), stream()), "qkv"), qkv_out)
    qkv = (Y.float() @ Wq.float().t() + bias).to(td)
    qr, kr, vr = [t.transpose(1, 2) for t in torch.unbind(qkv.reshape(B, N, 3, Hh, hd), 2)]
    qr, kr = O._rope(qr, sin, cos), O._rope(kr, sin, cos)
    for g, r in zip(got, (qr, kr, vr)):
        _assert_close(g, r.to(td), dtype)


@pytest.mark.parametrize("cout", [32, 128])
def test_overlap_conv3x3(cout):
    dtype, td = L.F16, torch.float16
    B, hw, cin = 4, 256, 64             # 2048 row tiles of 128 pixels
    x = _rand(B, hw, hw, cin, dt=td)
    w = _rand(cout, cin, 3, 3, scale=(9 * cin) ** -0.5, seed=1)
    bias = _rand(cout, seed=2)
    wp = w.permute(0, 2, 3, 1).reshape(cout, 9 * cin).to(td).contiguous()
    out = torch.empty(B * hw * hw, cout, device=DEV, dtype=td)
    got = _twice(lambda: gemm(x.view(-1, cin), wp, out, dtype, M=0, K=9 * cin, lda=cin, bias=bias, conv=L.CONV3X3_S1,
                              img=(B, hw, hw, cin)), out)
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.to(td).float(), bias, padding=1)
    _assert_close(got.view(B, hw, hw, cout).permute(0, 3, 1, 2), ref.to(td), dtype)
