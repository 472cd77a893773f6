"""-m gpu: every hand-written kernel against a plain PyTorch fp32 reference of the same op, through the C-ABI.
Tolerances are those of the 16-bit storage type (bf16 eps 2^-8, fp16 eps 2^-11) on O(1) data, stated per test."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from dinounet_b200 import lib as L
from oracle import dinounet_oracle as O
from tests.gpu_helpers import TD, P, gemm, rel_err, stream

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(params=["v2"])
def gemm_impl(request):
    """The GEMM-family tests ran on two kernel generations in round 1; only the persistent wgmma kernel remains."""
    yield request.param


def _rand(*shape, dt=torch.float32, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(DEV).to(dt)


@pytest.mark.parametrize("dtype", [L.BF16, L.F16])
@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (1029, 384, 384), (300, 192, 96), (4096, 32, 32), (777, 64, 256),
                                   (2058, 1536, 384), (1500, 1024, 512), (20000, 4096, 256)])
def test_gemm_plain(gemm_impl, dtype, M, N, K):
    td = TD[dtype]
    A, W = _rand(M, K, dt=td), _rand(N, K, dt=td, scale=K ** -0.5, seed=1)
    bias = _rand(N, seed=2)
    out = torch.full((M, N), float("nan"), device=DEV, dtype=td)
    gemm(A, W, out, dtype, bias=bias)
    torch.cuda.synchronize()
    ref = A.float() @ W.float().t() + bias
    tol = 2 ** -7 if dtype == L.BF16 else 2 ** -10
    assert torch.isfinite(out.float()).all()
    assert rel_err(out, ref) < tol, rel_err(out, ref)


def test_gemm_epilogue_residual_scale_gelu_fp32out(gemm_impl):
    M, N, K = 1029 * 2, 384, 1536
    dtype, td = L.BF16, torch.bfloat16
    A, W = _rand(M, K, dt=td), _rand(N, K, dt=td, scale=K ** -0.5, seed=1)
    bias, gamma = _rand(N, seed=2), _rand(N, seed=3)
    X = _rand(M, N, seed=4)
    X0 = X.clone()
    gemm(A, W, X, dtype, out_fp32=True, bias=bias, scale=gamma, residual=X, ldres=N)
    torch.cuda.synchronize()
    lin = (A.float() @ W.float().t() + bias).to(td).float()
    ref = X0 + lin * gamma
    assert (X - ref).abs().max().item() < 2e-2 * ref.abs().max().item() / 4
    # GELU(erf) after rounding, 16-bit store
    out = torch.empty(M, N, device=DEV, dtype=td)
    gemm(A, W, out, dtype, bias=bias, act1=L.ACT_GELU)
    torch.cuda.synchronize()
    ref = F.gelu(lin).to(td)
    assert rel_err(out, ref) < 2 ** -6


@pytest.mark.parametrize("dtype", [L.BF16, L.F16])
@pytest.mark.parametrize("M,D,Hd", [(1029, 256, 512), (300, 128, 64), (2058, 512, 1024 + 64)])
def test_gemm_swiglu_epilogue(dtype, M, D, Hd):
    """SwiGLUFFN first half fused (ffn_layers.py:73-77): hidden = silu(x w1^T + b1) * (x w2^T + b2), with autocast roundings."""
    td = TD[dtype]
    x = _rand(M, D, dt=td)
    w1, w2 = _rand(Hd, D, dt=td, scale=D ** -0.5, seed=1), _rand(Hd, D, dt=td, scale=D ** -0.5, seed=2)
    b1, b2 = _rand(Hd, seed=3, scale=0.2), _rand(Hd, seed=4, scale=0.2)
    # pack 32-row blocks [w1 block | w2 block]
    Wp = torch.stack([w1.view(Hd // 32, 32, D), w2.view(Hd // 32, 32, D)], 1).reshape(2 * Hd, D).contiguous()
    bp = torch.stack([b1.view(Hd // 32, 32), b2.view(Hd // 32, 32)], 1).reshape(2 * Hd).contiguous()
    out = torch.full((M, Hd), float("nan"), device=DEV, dtype=td)
    gemm(x, Wp, out, dtype, bias=bp, act1=L.ACT_SWIGLU, ldc=Hd)
    torch.cuda.synchronize()
    x1 = (x.float() @ w1.float().t() + b1).to(td)
    x2 = (x.float() @ w2.float().t() + b2).to(td)
    ref = (F.silu(x1.float()).to(td).float() * x2.float())
    assert torch.isfinite(out.float()).all()
    assert rel_err(out, ref) < (2 ** -6 if dtype == L.BF16 else 2 ** -9), rel_err(out, ref)


def test_gemm_row_remap_and_coloffset(gemm_impl):
    B, Pn, Nn, D, K = 3, 64, 69, 128, 64
    dtype, td = L.F16, torch.float16
    A, W = _rand(B * Pn, K, dt=td), _rand(D, K, dt=td, scale=K ** -0.5, seed=1)
    X = torch.zeros(B * Nn, 2 * D, device=DEV)
    gemm(A, W, X, dtype, out_fp32=True, rows=(Pn, Nn, 5), col_off=D, ldc=2 * D)
    torch.cuda.synchronize()
    ref = (A.float() @ W.float().t()).to(td).float().view(B, Pn, D)
    got = X.view(B, Nn, 2 * D)
    assert rel_err(got[:, 5:, D:], ref) < 1e-3
    assert got[:, :5].abs().max() == 0 and got[:, :, :D].abs().max() == 0


@pytest.mark.parametrize("cin,cout,hw", [(64, 32, 16), (256, 128, 8), (384, 384, 16)])
def test_gemm_convtranspose_pixelshuffle(gemm_impl, cin, cout, hw):
    B = 2
    dtype, td = L.F16, torch.float16
    x = _rand(B, hw, hw, cin, dt=td)
    w = _rand(cin, cout, 2, 2, scale=cin ** -0.5, seed=1)
    bias = _rand(cout, seed=2)
    add = _rand(B, 2 * hw, 2 * hw, cout, dt=td, seed=3)
    Wp = w.permute(2, 3, 1, 0).reshape(4 * cout, cin).to(td).contiguous()
    out = torch.empty(B * 4 * hw * hw, cout, device=DEV, dtype=td)
    gemm(x.view(-1, cin), Wp, out, dtype, ps=(cout, hw, hw), bias=bias.repeat(4).contiguous(), add16=add, ldadd=cout)
    torch.cuda.synchronize()
    ref = F.conv_transpose2d(x.float().permute(0, 3, 1, 2), w.to(td).float(), bias, stride=2)
    ref = ref.to(td).float() + add.float().permute(0, 3, 1, 2)
    got = out.view(B, 2 * hw, 2 * hw, cout).permute(0, 3, 1, 2).float()
    assert rel_err(got, ref) < 2e-3


def _pack_conv(w, td):
    N, Cc = w.shape[:2]
    cpad = (Cc + 63) // 64 * 64
    p = torch.zeros(N, 9, cpad, device=w.device)
    p[:, :, :Cc] = w.permute(0, 2, 3, 1).reshape(N, 9, Cc)
    return p.reshape(N, 9 * cpad).to(td).contiguous()


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("cin,cout,hw,B", [(64, 64, 32, 2), (32, 32, 64, 1), (256, 128, 16, 2), (128, 256, 8, 3),
                                           (64, 32, 256, 1)])
def test_conv3x3_implicit_gemm(gemm_impl, stride, cin, cout, hw, B):
    dtype, td = L.F16, torch.float16
    x = _rand(B, hw, hw, cin, dt=td)
    w = _rand(cout, cin, 3, 3, scale=(9 * cin) ** -0.5, seed=1)
    bias = _rand(cout, seed=2)
    ho = hw // stride
    out = torch.full((B * ho * ho, cout), float("nan"), device=DEV, dtype=td)
    gemm(x.view(-1, cin), _pack_conv(w, td), out, dtype, M=0, K=9 * cin, lda=cin, bias=bias,
         conv=L.CONV3X3_S2 if stride == 2 else L.CONV3X3_S1, img=(B, hw, hw, cin))
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.to(td).float(), bias, stride=stride, padding=1)
    got = out.view(B, ho, ho, cout).permute(0, 3, 1, 2).float()
    assert torch.isfinite(got).all()
    assert rel_err(got, ref) < 2e-3, rel_err(got, ref)
    # folded-BN + ReLU epilogue (SPM: dinov3_adapter.py:241-273)
    sc, sh = _rand(cout, seed=5).abs() + 0.5, _rand(cout, seed=6)
    gemm(x.view(-1, cin), _pack_conv(w, td), out, dtype, M=0, K=9 * cin, lda=cin, scale=sc, shift=sh, act2=L.ACT_RELU,
         conv=L.CONV3X3_S2 if stride == 2 else L.CONV3X3_S1, img=(B, hw, hw, cin))
    torch.cuda.synchronize()
    ref2 = F.relu((ref - bias[None, :, None, None]).half().float() * sc[None, :, None, None] + sh[None, :, None, None])
    got = out.view(B, ho, ho, cout).permute(0, 3, 1, 2).float()
    assert rel_err(got, ref2) < 3e-3, rel_err(got, ref2)


@pytest.mark.parametrize("cin,cout,hh,ww,B", [(64, 32, 256, 256, 1), (64, 64, 128, 128, 2), (32, 32, 256, 256, 1),
                                              (64, 64, 256, 256, 1), (64, 64, 24, 32, 3), (32, 64, 40, 16, 1)])
def test_conv3x3_implicit_gemm_large_and_partial_tiles(cin, cout, hh, ww, B):
    """Per-tap implicit GEMM on 256^2 images and on images that end in partial tiles (24 and 40 rows)."""
    dtype, td = L.F16, torch.float16
    x = _rand(B, hh, ww, cin, dt=td)
    w = _rand(cout, cin, 3, 3, scale=(9 * cin) ** -0.5, seed=1)
    bias = _rand(cout, seed=2)
    out = torch.full((B * hh * ww, cout), float("nan"), device=DEV, dtype=td)
    gemm(x.view(-1, cin), _pack_conv(w, td), out, dtype, M=0, K=9 * cin, lda=cin, bias=bias, conv=L.CONV3X3_S1,
         img=(B, hh, ww, cin))
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.to(td).float(), bias, stride=1, padding=1)
    got = out.view(B, hh, ww, cout).permute(0, 3, 1, 2).float()
    assert torch.isfinite(got).all()
    assert rel_err(got, ref) < 2e-3, rel_err(got, ref)


@pytest.mark.parametrize("dtype", [L.BF16, L.F16])
@pytest.mark.parametrize("B,h,D,Hh", [(2, 16, 384, 6),    # CTA pairs, 16-warp epilogue, half-empty last n-tile (N = 1152)
                                      (1, 8, 768, 12),    # M = 69 < 256: one CTA per tile (no pairing), 256-wide tiles
                                      (2, 8, 512, 4),     # head_dim 128 (ViT-7B): two 64-column units per head
                                      (3, 16, 128, 2)])   # N = 384 -> 128-wide tiles: the 8-warp epilogue
def test_qkv_rope_and_attention(gemm_impl, dtype, B, h, D, Hh):
    td = TD[dtype]
    hd = D // Hh
    Pn = h * h
    N = Pn + 5
    lib = L.load()
    Y = _rand(B * N, D, dt=td)
    Wq = _rand(3 * D, D, dt=td, scale=D ** -0.5, seed=1)
    bias = _rand(3 * D, seed=2, scale=0.1)
    periods = 100.0 ** (2 * torch.arange(hd // 4, dtype=torch.float32) / (hd // 2))
    sin, cos = O.rope_sincos(periods, h, h)
    sin, cos = sin.to(DEV).contiguous(), cos.to(DEV).contiguous()
    q, k, v = (torch.full((B, Hh, N, hd), float("nan"), device=DEV, dtype=td) for _ in range(3))
    p = L.QkvParams()
    p.B, p.ntok, p.D, p.heads, p.prefix = B, N, D, Hh, 5
    p.A, p.lda, p.Wp, p.ldw, p.bias = P(Y), D, P(Wq), D, P(bias)
    p.rope_sin, p.rope_cos, p.q, p.k, p.v, p.dtype = P(sin), P(cos), P(q), P(k), P(v), dtype
    L.check(lib.b2u_qkv_rope(C.byref(p), stream()), "qkv")
    torch.cuda.synchronize()
    if gemm_impl == "v2":   # separable in-smem rope tables must give bit-identical q/k
        q2, k2, v2_ = (torch.full((B, Hh, N, hd), float("nan"), device=DEV, dtype=td) for _ in range(3))
        p.q, p.k, p.v, p.rope_w = P(q2), P(k2), P(v2_), h
        L.check(lib.b2u_qkv_rope(C.byref(p), stream()), "qkv(smem rope)")
        torch.cuda.synchronize()
        assert torch.equal(q, q2) and torch.equal(k, k2) and torch.equal(v, v2_)
    qkv = (Y.float() @ Wq.float().t() + bias).to(td)
    qr, kr, vr = [t.transpose(1, 2) for t in torch.unbind(qkv.reshape(B, N, 3, Hh, hd), 2)]
    qr, kr = O._rope(qr, sin, cos), O._rope(kr, sin, cos)
    tol = 2 ** -6 if dtype == L.BF16 else 2 ** -9
    assert rel_err(q, qr) < tol and rel_err(k, kr) < tol and rel_err(v, vr) < tol
    # the QKV epilogue's transposed V store feeds the wgmma attention kernel: whole path against SDPA
    npad = (N + 7) // 8 * 8
    vt = torch.zeros(B, Hh, hd, npad, device=DEV, dtype=td)
    p.q, p.k, p.v, p.v_transposed, p.npad, p.rope_w = P(q), P(k), P(vt), 1, npad, h
    L.check(lib.b2u_qkv_rope(C.byref(p), stream()), "qkv(V^T)")
    out = torch.full((B, N, D), float("nan"), device=DEV, dtype=td)
    L.check(lib.b2u_attention_tc_hd(P(q), P(k), P(vt), P(out), B, Hh, N, npad, hd, hd ** -0.5, dtype, stream()), "attention")
    torch.cuda.synchronize()
    assert torch.equal(vt[..., :N], v.transpose(2, 3))
    ref = F.scaled_dot_product_attention(q.float(), k.float(), v.float()).transpose(1, 2).reshape(B, N, D)
    assert torch.isfinite(out.float()).all()
    assert rel_err(out, ref) < (2 ** -6 if dtype == L.BF16 else 2 ** -8), rel_err(out, ref)


@pytest.mark.parametrize("dtype", [L.BF16, L.F16])
@pytest.mark.parametrize("B,Hh,N", [(1, 3, 1029), (2, 6, 261), (3, 2, 128), (1, 1, 700)])
def test_attention_tcgen05(dtype, B, Hh, N):
    """wgmma flash attention (V consumed as zero-padded V^T) == SDPA; QKV epilogue's V^T store == transpose."""
    td = TD[dtype]
    lib = L.load()
    q, k, v = (_rand(B, Hh, N, 64, dt=td, seed=s) for s in range(3))
    npad = (N + 7) // 8 * 8
    vt = torch.zeros(B, Hh, 64, npad, device=DEV, dtype=td)
    vt[..., :N] = v.transpose(2, 3)
    out = torch.full((B, N, Hh * 64), float("nan"), device=DEV, dtype=td)
    L.check(lib.b2u_attention_tc(P(q), P(k), P(vt), P(out), B, Hh, N, npad, 0, 0.125, dtype, stream()), "attention_tc")
    torch.cuda.synchronize()
    ref = F.scaled_dot_product_attention(q.float(), k.float(), v.float()).transpose(1, 2).reshape(B, N, Hh * 64)
    assert torch.isfinite(out.float()).all()
    assert rel_err(out, ref) < (2 ** -6 if dtype == L.BF16 else 2 ** -8), rel_err(out, ref)
    # split launch: rows [5, N) on the wgmma kernel + rows [0, 5) on the few-row kernel == the whole thing
    if N > 5:
        outs = torch.full_like(out, float("nan"))
        L.check(lib.b2u_attention_tc(P(q), P(k), P(vt), P(outs), B, Hh, N, npad, 5, 0.125, dtype, stream()), "attention_tc")
        L.check(lib.b2u_attention_rows(P(q), P(k), P(vt), P(outs), B, Hh, N, npad, 0, 5, 0.125, dtype, stream()), "rows")
        torch.cuda.synchronize()
        assert torch.isfinite(outs.float()).all()
        assert rel_err(outs, ref) < (2 ** -6 if dtype == L.BF16 else 2 ** -8), rel_err(outs, ref)
    # second launch on the same buffers (persistent-loop barrier phases must be clean at exit)
    out2 = torch.empty_like(out)
    L.check(lib.b2u_attention_tc(P(q), P(k), P(vt), P(out2), B, Hh, N, npad, 0, 0.125, dtype, stream()), "attention_tc")
    torch.cuda.synchronize()
    assert torch.equal(out, out2)


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("N", [1029, 300, 144, 129])
def test_attention_tcgen05_lazy_rescale_and_narrow_tail(hd, N):
    """Scores that keep growing along the key axis (|k| ramps up 5x) move the running maximum by large steps several
    times -> the O rescale path; N = 1029 / 300 / 144 / 129 give last key chunks of 5 / 44 / 16 / 1 valid keys (PV
    widths 16 / 48 / 16 / 16) and query tiles whose rows lie partly or wholly beyond ntok."""
    lib = L.load()
    dtype, td = L.BF16, torch.bfloat16
    B, Hh = 2, 2
    q, k, v = (_rand(B, Hh, N, hd, dt=torch.float32, seed=10 + s) for s in range(3))
    k = k * (1.0 + 4.0 * torch.arange(N, device=DEV, dtype=torch.float32) / N)[None, None, :, None]
    q, k, v = q.to(td), k.to(td), v.to(td)
    npad = (N + 7) // 8 * 8
    vt = torch.zeros(B, Hh, hd, npad, device=DEV, dtype=td)
    vt[..., :N] = v.transpose(2, 3)
    out = torch.full((B, N, Hh * hd), float("nan"), device=DEV, dtype=td)
    if hd == 64:
        L.check(lib.b2u_attention_tc(P(q), P(k), P(vt), P(out), B, Hh, N, npad, 0, hd ** -0.5, dtype, stream()), "attn")
    else:
        L.check(lib.b2u_attention_tc_hd(P(q), P(k), P(vt), P(out), B, Hh, N, npad, hd, hd ** -0.5, dtype, stream()), "attn")
    torch.cuda.synchronize()
    ref = F.scaled_dot_product_attention(q.float(), k.float(), v.float()).transpose(1, 2).reshape(B, N, Hh * hd)
    assert torch.isfinite(out.float()).all()
    assert rel_err(out, ref) < 2 ** -6, rel_err(out, ref)


@pytest.mark.parametrize("dtype", [L.BF16, L.F16])
@pytest.mark.parametrize("B,Hh,N", [(1, 2, 1029), (2, 3, 261), (1, 1, 128)])
def test_attention_tcgen05_head_dim_128(dtype, B, Hh, N):
    td = TD[dtype]
    lib = L.load()
    q, k, v = (_rand(B, Hh, N, 128, dt=td, seed=s) for s in range(3))
    npad = (N + 7) // 8 * 8
    vt = torch.zeros(B, Hh, 128, npad, device=DEV, dtype=td)
    vt[..., :N] = v.transpose(2, 3)
    out = torch.full((B, N, Hh * 128), float("nan"), device=DEV, dtype=td)
    L.check(lib.b2u_attention_tc_hd(P(q), P(k), P(vt), P(out), B, Hh, N, npad, 128, 128 ** -0.5, dtype, stream()), "attn128")
    torch.cuda.synchronize()
    ref = F.scaled_dot_product_attention(q.float(), k.float(), v.float()).transpose(1, 2).reshape(B, N, Hh * 128)
    assert torch.isfinite(out.float()).all()
    assert rel_err(out, ref) < (2 ** -6 if dtype == L.BF16 else 2 ** -8), rel_err(out, ref)


def test_qkv_rope_head_dim_128():
    """QKV epilogue for the 7B head size: rope pairs (j, j+64), 32 angles per axis, V^T with 128 rows per head."""
    dtype, td = L.BF16, torch.bfloat16
    B, h, D, Hh = 2, 8, 512, 4
    N = h * h + 5
    npad = (N + 7) // 8 * 8
    lib = L.load()
    Y = _rand(B * N, D, dt=td)
    Wq = _rand(3 * D, D, dt=td, scale=D ** -0.5, seed=1)
    periods = 100.0 ** (2 * torch.arange(32, dtype=torch.float32) / 64)
    sin, cos = [t.to(DEV).contiguous() for t in O.rope_sincos(periods, h, h)]
    qkv = (Y.float() @ Wq.float().t()).to(td)
    qr, kr, vr = [t.transpose(1, 2) for t in torch.unbind(qkv.reshape(B, N, 3, Hh, 128), 2)]
    qr, kr = O._rope(qr, sin, cos), O._rope(kr, sin, cos)
    for rope_w in (0, h):
        q, k = (torch.full((B, Hh, N, 128), float("nan"), device=DEV, dtype=td) for _ in range(2))
        vt = torch.zeros(B, Hh, 128, npad, device=DEV, dtype=td)
        p = L.QkvParams()
        p.B, p.ntok, p.D, p.heads, p.prefix = B, N, D, Hh, 5
        p.A, p.lda, p.Wp, p.ldw, p.bias = P(Y), D, P(Wq), D, None
        p.rope_sin, p.rope_cos, p.q, p.k, p.v, p.dtype = P(sin), P(cos), P(q), P(k), P(vt), dtype
        p.v_transposed, p.npad, p.rope_w = 1, npad, rope_w
        L.check(lib.b2u_qkv_rope(C.byref(p), stream()), "qkv128")
        torch.cuda.synchronize()
        assert rel_err(q, qr) < 2 ** -6 and rel_err(k, kr) < 2 ** -6, (rope_w, rel_err(q, qr), rel_err(k, kr))
        assert rel_err(vt[..., :N].transpose(2, 3), vr) < 2 ** -6 and vt[..., N:].abs().max() == 0


def test_qkv_vt_store_matches_transpose():
    dtype, td = L.BF16, torch.bfloat16
    B, h, D, Hh = 2, 8, 384, 6
    N = h * h + 5
    npad = (N + 7) // 8 * 8
    lib = L.load()
    Y = _rand(B * N, D, dt=td)
    Wq = _rand(3 * D, D, dt=td, scale=D ** -0.5, seed=1)
    periods = 100.0 ** (2 * torch.arange(16, dtype=torch.float32) / 32)
    sin, cos = [t.to(DEV).contiguous() for t in O.rope_sincos(periods, h, h)]
    outs = []
    for vt_mode in (0, 1):
        q, k = (torch.empty(B, Hh, N, 64, device=DEV, dtype=td) for _ in range(2))
        v = torch.zeros((B, Hh, 64, npad) if vt_mode else (B, Hh, N, 64), device=DEV, dtype=td)
        p = L.QkvParams()
        p.B, p.ntok, p.D, p.heads, p.prefix = B, N, D, Hh, 5
        p.A, p.lda, p.Wp, p.ldw, p.bias = P(Y), D, P(Wq), D, None
        p.rope_sin, p.rope_cos, p.q, p.k, p.v, p.dtype = P(sin), P(cos), P(q), P(k), P(v), dtype
        p.v_transposed, p.npad = vt_mode, npad
        L.check(lib.b2u_qkv_rope(C.byref(p), stream()), "qkv")
        torch.cuda.synchronize()
        outs.append((q, k, v))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert torch.equal(outs[1][2][..., :N], outs[0][2].transpose(2, 3))
    assert outs[1][2][..., N:].abs().max() == 0


def test_layernorm_and_cast():
    lib = L.load()
    B, Nn, Pn, D = 2, 69, 64, 384
    X = _rand(B * Nn, D) * 3 + 1
    g, b = _rand(D, seed=1), _rand(D, seed=2)
    out = torch.empty(B * Pn, D, device=DEV)
    L.check(lib.b2u_layernorm(P(X), P(out), P(g), P(b), B * Pn, D, 1e-5, Nn, Pn, 5, 1, L.BF16, stream()), "ln")
    torch.cuda.synchronize()
    ref = F.layer_norm(X.view(B, Nn, D)[:, 5:], (D,), g, b, 1e-5).reshape(B * Pn, D)
    assert (out - ref).abs().max() < 2e-5
    o16 = torch.empty(B * Nn, D, device=DEV, dtype=torch.float16)
    L.check(lib.b2u_layernorm(P(X), P(o16), P(g), P(b), B * Nn, D, 1e-6, 0, 0, 0, 0, L.F16, stream()), "ln16")
    c16 = torch.empty(B * Pn, D, device=DEV, dtype=torch.float16)
    L.check(lib.b2u_cast_rows(P(X), P(c16), B * Pn, D, Nn, Pn, 5, L.F16, stream()), "cast")
    torch.cuda.synchronize()
    assert rel_err(o16, F.layer_norm(X, (D,), g, b, 1e-6)) < 2e-3
    assert torch.equal(c16, X.view(B, Nn, D)[:, 5:].reshape(B * Pn, D).half())


def test_patchify_prefix_stem_maxpool():
    lib = L.load()
    B, S = 2, 64
    x = _rand(B, 3, S, S)
    out = torch.empty(B * 16, 768, device=DEV, dtype=torch.bfloat16)
    L.check(lib.b2u_patchify(P(x), P(out), B, S, L.BF16, stream()), "patchify")
    ref = F.unfold(x, 16, stride=16).transpose(1, 2).reshape(B * 16, 768).bfloat16()
    torch.cuda.synchronize()
    assert torch.equal(out, ref)
    w = _rand(64, 3, 3, 3, scale=27 ** -0.5, seed=1)
    sc, sh = _rand(64, seed=2).abs() + 0.5, _rand(64, seed=3)
    so = torch.empty(B, S // 2, S // 2, 64, device=DEV, dtype=torch.float16)
    L.check(lib.b2u_stem_conv0(P(x), P(w), P(sc), P(sh), P(so), B, S, L.F16, stream()), "stem")
    ref = F.relu(F.conv2d(x, w, stride=2, padding=1).half().float() * sc[None, :, None, None] + sh[None, :, None, None])
    torch.cuda.synchronize()
    assert rel_err(so.permute(0, 3, 1, 2), ref) < 2e-3
    mp = torch.empty(B, S // 4, S // 4, 64, device=DEV, dtype=torch.float16)
    L.check(lib.b2u_maxpool3x3s2(P(so), P(mp), B, S // 2, S // 2, 64, L.F16, stream()), "maxpool")
    torch.cuda.synchronize()
    assert torch.equal(mp.permute(0, 3, 1, 2), F.max_pool2d(so.permute(0, 3, 1, 2).float(), 3, 2, 1).half())


def test_dwconv_three_planes_gelu():
    lib = L.load()
    B, Hc, Cc = 2, 8, 96
    n = (Hc // 2) ** 2
    x = _rand(B, 21 * n, Cc, dt=torch.float16)
    w, bias = _rand(Cc, 1, 3, 3, scale=1 / 3, seed=1), _rand(Cc, seed=2)
    out = torch.empty_like(x)
    w9 = w.reshape(Cc, 9).t().contiguous()
    L.check(lib.b2u_dwconv3x3(P(x), P(out), P(w9), P(bias), B, Hc, Hc, Cc, 3, L.ACT_GELU, L.F16, stream()), "dw")
    torch.cuda.synchronize()
    parts = []
    for sl, hh in ((slice(0, 16 * n), 2 * Hc), (slice(16 * n, 20 * n), Hc), (slice(20 * n, 21 * n), Hc // 2)):
        t = x[:, sl].float().transpose(1, 2).reshape(B, Cc, hh, hh)
        parts.append(F.conv2d(t, w, bias, padding=1, groups=Cc).flatten(2).transpose(1, 2))
    ref = F.gelu(torch.cat(parts, 1).half().float())
    assert rel_err(out, ref) < 2e-3


@pytest.mark.parametrize("impl", [0, 1, 2])
@pytest.mark.parametrize("dh", [12, 24, 32, 128])
def test_msda_forward_matches_reference_sampling(dh, impl):
    """the op the reference itself pins in ops/test.py: CUDA sampling == grid_sample formulation."""
    lib = L.load()
    B, Hv, heads, pts = 2, 16, 16, 4
    HW = Hv * Hv
    Lq = 21 * HW // 4
    value = _rand(B, HW, heads, dh, dt=torch.float16)
    offaw = torch.cat([_rand(B * Lq, 128, scale=3.0, seed=1), _rand(B * Lq, 64, seed=2)], 1).contiguous()
    out = torch.full((B * Lq, heads * dh), float("nan"), device=DEV, dtype=torch.float16)
    lib.b2u_set_option(1, impl)     # 0 = shared-memory slab kernel (dh 32: one swizzled head per CTA), 1 = warp-per-query kernel, 2 = slab kernel without the one-head layout
    try:
        L.check(lib.b2u_msda_forward(P(value), P(offaw), P(out), B, Hv, Hv, heads, dh, pts, L.F16, stream()), "msda")
        torch.cuda.synchronize()
    finally:
        lib.b2u_set_option(1, 0)
    ref_pts = O.reference_points([(2 * Hv, 2 * Hv), (Hv, Hv), (Hv // 2, Hv // 2)], DEV)
    off = offaw[:, :128].view(B, Lq, heads, 1, pts, 2)
    aw = F.softmax(offaw[:, 128:].view(B, Lq, heads, pts), -1).view(B, Lq, heads, 1, pts)
    loc = ref_pts[:, :, None, :, None, :] + off / torch.tensor([Hv, Hv], device=DEV)
    ref = O.msda_core(value.float(), [(Hv, Hv)], loc, aw)
    assert rel_err(out.view(B, Lq, -1), ref) < 2e-3, rel_err(out.view(B, Lq, -1), ref)


def test_msda_f32_dropin_reference_fixture():
    """ops/test.py:24-64 fixture: N,M,D=1,2,2; Lq,L,P=2,2,2; shapes [(6,4),(3,2)]; seed 3."""
    lib = L.load()
    N_, M_, D_, Lq_, L_, P_ = 1, 2, 2, 2, 2, 2
    shapes = torch.as_tensor([(6, 4), (3, 2)], dtype=torch.long, device=DEV)
    lsi = torch.cat((shapes.new_zeros((1,)), shapes.prod(1).cumsum(0)[:-1]))
    S_ = int(shapes.prod(1).sum())
    torch.manual_seed(3)
    value = (torch.rand(N_, S_, M_, D_) * 0.01).to(DEV)
    loc = torch.rand(N_, Lq_, M_, L_, P_, 2).to(DEV)
    aw = torch.rand(N_, Lq_, M_, L_, P_).to(DEV) + 1e-5
    aw = (aw / aw.sum(-1, keepdim=True).sum(-2, keepdim=True)).contiguous()
    out = torch.empty(N_, Lq_, M_ * D_, device=DEV)
    L.check(lib.b2u_msda_forward_f32(P(value), P(shapes), P(lsi), P(loc), P(aw), P(out), N_, S_, Lq_, M_, D_, L_, P_,
                                     stream()), "msda_f32")
    torch.cuda.synchronize()
    ref = O.msda_core(value, [(6, 4), (3, 2)], loc, aw)
    assert torch.allclose(out, ref, rtol=1e-2, atol=1e-3)   # the reference's own fp32 tolerance (ops/test.py:81)
    assert (out - ref).abs().max() < 1e-6


@pytest.mark.parametrize("ncls", [1, 3, 8, 9, 20, 117, 128])
def test_seg_head_many_classes(ncls):
    """1x1 seg conv + argmax for any class count up to 128 (multi-organ label sets), first-maximum argmax."""
    lib = L.load()
    B, rows, Cc = 2, 4096, 32
    x = (_rand(B * rows, Cc, dt=torch.float16, seed=ncls) * 2 + 0.5)
    sums = torch.empty((B, Cc, 2), device=DEV)
    work = torch.zeros(int(lib.b2u_in_stats_work_floats(B, rows, Cc)), device=DEV)
    L.check(lib.b2u_in_stats(P(x), Cc, P(sums), P(work), B, rows, Cc, L.F16, stream()), "stats")
    g, b = _rand(Cc, seed=1), _rand(Cc, seed=2)
    w, wb = _rand(ncls, Cc, seed=3), _rand(ncls, seed=4)
    logits = torch.full((B, ncls, rows), float("nan"), device=DEV)
    labels = torch.empty(B, rows, device=DEV, dtype=torch.uint8)
    L.check(lib.b2u_seg_head(P(x), P(sums), P(g), P(b), 1e-5, P(w), P(wb), P(logits), P(labels), B, rows, Cc, ncls, L.F16,
                             stream()), "seg")
    torch.cuda.synchronize()
    xin = x.float().view(B, rows, Cc).transpose(1, 2).reshape(B, Cc, 64, 64)
    act = F.leaky_relu(F.instance_norm(xin, None, None, g, b, True, 0.1, 1e-5), 0.01).half().float()
    ref = F.conv2d(act, w.view(ncls, Cc, 1, 1), wb).flatten(2)
    assert rel_err(logits, ref) < 3e-3
    assert (labels.long() == logits.argmax(1)).all()
    assert lib.b2u_seg_head(P(x), P(sums), P(g), P(b), 1e-5, P(w), P(wb), P(logits), P(labels), B, rows, Cc, 129, L.F16,
                            stream()) != 0


def _msda_case(N_, M_, D_, Lq_, shapes_list, P_, seed):
    shapes = torch.as_tensor(shapes_list, dtype=torch.long, device=DEV)
    lsi = torch.cat((shapes.new_zeros((1,)), shapes.prod(1).cumsum(0)[:-1]))
    S_ = int(shapes.prod(1).sum())
    L_ = len(shapes_list)
    g = torch.Generator().manual_seed(seed)
    value = (torch.rand(N_, S_, M_, D_, generator=g) * 0.01).to(DEV)
    loc = (torch.rand(N_, Lq_, M_, L_, P_, 2, generator=g) * 1.3 - 0.15).to(DEV)   # some samples leave the map
    aw = torch.rand(N_, Lq_, M_, L_, P_, generator=g).to(DEV) + 1e-5
    aw = (aw / aw.sum(-1, keepdim=True).sum(-2, keepdim=True)).contiguous()
    gout = torch.randn(N_, Lq_, M_ * D_, generator=g).to(DEV)
    return value, shapes, lsi, loc, aw, gout


@pytest.mark.parametrize("channels", [30, 32, 64, 71])
def test_msda_backward_dropin_reference_fixture(channels):
    """ops/test.py:89-121 (`check_gradient_numerical`, its first four channel counts) restated: the op's gradients
    against autograd through the grid_sample formulation, evaluated in fp64 on the CPU."""
    from dinounet_b200 import ops
    value, shapes, lsi, loc, aw, gout = _msda_case(1, 2, channels, 2, [(6, 4), (3, 2)], 2, 3)
    gv, gl, ga = ops.ms_deform_attn_backward(value, shapes, lsi, loc, aw, gout, 2)
    v64, l64, a64 = (t.double().cpu().requires_grad_(True) for t in (value, loc, aw))
    O.msda_core(v64, [(6, 4), (3, 2)], l64, a64).backward(gout.double().cpu())
    for got, want in ((gv, v64.grad), (gl, l64.grad), (ga, a64.grad)):
        assert got.shape == want.shape
        assert rel_err(got.cpu().double(), want) < 1e-5, rel_err(got.cpu().double(), want)


def test_msda_backward_engine_shape_and_autograd_function():
    """dinounet_l's extractor shape (16 heads x 32, one 32x32 level, 4 points, Lq=5376) through the autograd face."""
    from dinounet_b200 import ops
    value, shapes, lsi, loc, aw, gout = _msda_case(2, 16, 32, 5376, [(32, 32)], 4, 11)
    v, l, a = (t.clone().requires_grad_(True) for t in (value, loc, aw))
    out = ops.MSDeformAttnFunction.apply(v, shapes, lsi, l, a, 64)
    out.backward(gout)
    v2, l2, a2 = (t.clone().requires_grad_(True) for t in (value, loc, aw))
    ref = O.msda_core(v2, [(32, 32)], l2, a2)
    ref.backward(gout)
    assert rel_err(out, ref) < 1e-5
    for got, want in ((v.grad, v2.grad), (l.grad, l2.grad), (a.grad, a2.grad)):
        assert rel_err(got, want) < 2e-5, rel_err(got, want)
    with pytest.raises(RuntimeError):
        ops.ms_deform_attn_backward(value.cpu(), shapes, lsi, loc, aw, gout, 64)
    with pytest.raises(RuntimeError):
        ops.ms_deform_attn_forward(value.transpose(1, 2), shapes, lsi, loc, aw, 64)


def test_instancenorm_large_mean_small_std():
    """|mean| >> std: E[x^2] - mean^2 in fp32 loses the variance (x^2 ~ 1e4, var ~ 0.07); the statistics kernel accumulates
    shifted sums instead, so the normalised output still matches torch's (Welford) instance_norm."""
    lib = L.load()
    B, rows, Cc = 2, 16384, 32
    off = torch.linspace(-150.0, 150.0, Cc, device=DEV)
    x = (_rand(B * rows, Cc, seed=5) * 0.25 + off).to(torch.float16)
    sums = torch.full((B, Cc, 2), float("nan"), device=DEV)
    work = torch.zeros(int(lib.b2u_in_stats_work_floats(B, rows, Cc)), device=DEV)
    L.check(lib.b2u_in_stats(P(x), Cc, P(sums), P(work), B, rows, Cc, L.F16, stream()), "stats")
    g, b = _rand(Cc, seed=1), _rand(Cc, seed=2)
    y = torch.empty(B * rows, Cc, device=DEV, dtype=torch.float16)
    L.check(lib.b2u_in_apply(P(x), Cc, P(y), Cc, P(sums), P(g), P(b), B, rows, Cc, 1e-5, L.F16, stream()), "apply")
    torch.cuda.synchronize()
    xd = x.double().view(B, rows, Cc)
    assert rel_err(sums[..., 0], xd.sum(1).float()) < 1e-6
    var = xd.var(1, unbiased=False)
    assert ((sums[..., 1].double() / rows - var).abs() / var).max().item() < 1e-4
    xin = x.float().view(B, rows, Cc).transpose(1, 2).reshape(B, Cc, 128, 128)
    ref = F.leaky_relu(F.instance_norm(xin, None, None, g, b, True, 0.1, 1e-5), 0.01)
    assert rel_err(y.view(B, rows, Cc).transpose(1, 2).reshape(B, Cc, 128, 128), ref) < 3e-3


def test_instancenorm_film_se_seg():
    lib = L.load()
    B, rows, Cc = 2, 4096, 32
    x = (_rand(B * rows, 2 * Cc, dt=torch.float16) * 2 + 0.5)
    sums = torch.full((B, Cc, 2), float("nan"), device=DEV)
    work = torch.zeros(int(lib.b2u_in_stats_work_floats(B, rows, Cc)), device=DEV)
    L.check(lib.b2u_in_stats(P(x), 2 * Cc, P(sums), P(work), B, rows, Cc, L.F16, stream()), "stats")
    s1 = sums.clone()
    L.check(lib.b2u_in_stats(P(x), 2 * Cc, P(sums), P(work), B, rows, Cc, L.F16, stream()), "stats")   # tickets self-reset
    torch.cuda.synchronize()
    assert torch.equal(s1, sums)
    assert rel_err(sums[..., 0], x[:, :Cc].float().view(B, rows, Cc).sum(1)) < 1e-5
    g, b = _rand(Cc, seed=1), _rand(Cc, seed=2)
    y = torch.empty(B * rows, Cc, device=DEV, dtype=torch.float16)
    L.check(lib.b2u_in_apply(P(x), 2 * Cc, P(y), Cc, P(sums), P(g), P(b), B, rows, Cc, 1e-5, L.F16, stream()), "apply")
    torch.cuda.synchronize()
    xin = x[:, :Cc].float().view(B, rows, Cc).transpose(1, 2).reshape(B, Cc, 64, 64)
    ref = F.leaky_relu(F.instance_norm(xin, None, None, g, b, True, 0.1, 1e-5), 0.01)
    assert rel_err(y.view(B, rows, Cc).transpose(1, 2).reshape(B, Cc, 64, 64), ref) < 3e-3
    # seg head on the same statistics
    w, wb = _rand(2, Cc, seed=3), _rand(2, seed=4)
    xc = x[:, :Cc].contiguous()
    logits = torch.empty(B, 2, rows, device=DEV)
    labels = torch.empty(B, rows, device=DEV, dtype=torch.uint8)
    L.check(lib.b2u_seg_head(P(xc), P(sums), P(g), P(b), 1e-5, P(w), P(wb), P(logits), P(labels), B, rows, Cc, 2, L.F16,
                             stream()), "seg")
    torch.cuda.synchronize()
    refl = F.conv2d(ref.half().float(), w.view(2, Cc, 1, 1), wb).flatten(2)
    assert rel_err(logits, refl) < 3e-3
    assert (labels.long() == logits.argmax(1)).all()
    # FiLM
    R = 256
    gb, zz = _rand(1000, 2 * R, dt=torch.float16, seed=5), _rand(1000, 2 * R, dt=torch.float16, seed=6)
    z = torch.empty(1000, R, device=DEV, dtype=torch.float16)
    L.check(lib.b2u_film(P(gb), P(zz), 2 * R, R, P(z), 1000, R, L.F16, stream()), "film")
    torch.cuda.synchronize()
    assert rel_err(z, gb[:, :R].float() * zz[:, R:].float() + gb[:, R:].float()) < 2e-3
    # SE gate + apply
    w1, b1, w2, b2 = _rand(2, Cc, seed=7), _rand(2, seed=8), _rand(Cc, 2, seed=9), _rand(Cc, seed=10)
    gate = torch.empty(B, Cc, device=DEV)
    L.check(lib.b2u_se_gate(P(sums), P(w1), P(b1), P(w2), P(b2), P(gate), B, Cc, 2, rows, stream()), "gate")
    outse = torch.empty(B * rows, Cc, device=DEV, dtype=torch.float16)
    L.check(lib.b2u_se_apply(P(xc), x.data_ptr() + Cc * 2, 2 * Cc, P(gate), P(outse), B, rows, Cc, L.F16, stream()), "se")
    torch.cuda.synchronize()
    pooled = x[:, :Cc].float().view(B, rows, Cc).mean(1)
    gref = torch.sigmoid(F.relu(pooled @ w1.t() + b1) @ w2.t() + b2)
    assert (gate - gref).abs().max() < 1e-4
    ref = x[:, :Cc].float().view(B, rows, Cc) * gref[:, None] + x[:, Cc:].float().view(B, rows, Cc)
    assert rel_err(outse.view(B, rows, Cc), ref) < 2e-3


def test_tail_fuse_bilinear_bn():
    lib = L.load()
    B, D, Ht = 2, 384, 8
    for H in (32, 16, 8, 4):
        tap = _rand(B, Ht * Ht, D, seed=H)
        base = _rand(B, H * H, D, seed=H + 1)
        sc, sh = _rand(D, seed=2).abs() + 0.5, _rand(D, seed=3)
        out = torch.empty(B, H * H, D, device=DEV, dtype=torch.float16)
        L.check(lib.b2u_tail_fuse(P(base), 1, H * H * D, P(tap), P(out), P(sc), P(sh), B, H, H, Ht, Ht, D, L.F16,
                                  stream()), "tail")
        torch.cuda.synchronize()
        t = tap.transpose(1, 2).reshape(B, D, Ht, Ht)
        up = F.interpolate(t, size=(H, H), mode="bilinear", align_corners=False)
        ref = (base.transpose(1, 2).reshape(B, D, H, H) + up) * sc[None, :, None, None] + sh[None, :, None, None]
        got = out.float().transpose(1, 2).reshape(B, D, H, H)
        assert rel_err(got, ref) < 2e-3, (H, rel_err(got, ref))
