"""Helpers for the -m gpu tests: call the C-ABI with torch-owned device memory."""
import ctypes as C

import torch

from dinounet_b200 import lib as L

TD = {L.F16: torch.float16, L.BF16: torch.bfloat16}
U = 2.0 ** -24                       # unit roundoff of fp32
MANT = {L.BF16: 7, L.F16: 10}        # stored mantissa bits
EMIN = {L.BF16: -126, L.F16: -14}    # smallest normal exponent (below it the spacing stays 2^(EMIN - MANT))


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def P(t):
    return None if t is None else t.data_ptr()


def gemm(A, W, out, dtype, *, M=None, K=None, lda=None, N=None, ldc=None, out_fp32=False, col_off=0, rows=None, ps=None,
         bias=None, scale=None, shift=None, act1=0, act2=0, round16=1, residual=None, ldres=0, add16=None, ldadd=0,
         conv=0, img=(0, 0, 0, 0)):
    lib = L.load()
    p = L.GemmParams()
    p.M = A.shape[0] if M is None else M
    p.K = A.shape[-1] if K is None else K
    p.N = W.shape[0] if N is None else N
    p.A, p.lda = P(A), (A.stride(0) if lda is None else lda)
    p.Wp, p.ldw = P(W), W.stride(0)
    p.dtype, p.conv = dtype, conv
    p.B, p.Hin, p.Win, p.C = img
    e = p.epi
    e.out, e.out_fp32, e.ldc, e.col_off = P(out), int(out_fp32), (out.stride(0) if ldc is None else ldc), col_off
    if rows:
        e.rows_in, e.rows_out, e.row_off = rows
    if ps:
        e.ps_cout, e.ps_h, e.ps_w = ps
    e.bias, e.scale, e.shift = P(bias), P(scale), P(shift)
    e.act1, e.act2, e.round16 = act1, act2, round16
    e.residual, e.ldres, e.add16, e.ldadd = P(residual), ldres, P(add16), ldadd
    L.check(lib.b2u_gemm(C.byref(p), stream()), "b2u_gemm")


def rel_err(a, b):
    a, b = a.float(), b.float()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-12)).item()


# ---- per-element comparison against a float64 reference (test_gpu_forward_kernels.py, test_gpu_tc_kernels.py)
def ulp16(x, dtype):
    """Spacing of the 16-bit type at |x| (float64)."""
    a = x.double().abs()
    e = torch.frexp(a)[1].double() - 1          # a = m * 2^e, 1 <= m < 2
    e = torch.where(a > 0, e, torch.full_like(e, EMIN[dtype])).clamp_min(EMIN[dtype])
    return torch.exp2(e - MANT[dtype])


def bar16(ref, prop, dtype):
    """Bar for a 16-bit output whose fp32 value is within `prop` of ref: the rounding (half an ulp, but up to a whole ulp
    at |ref| when the value rounds across a power of two) plus prop."""
    return ulp16(ref.abs() + prop, dtype) + prop


def check(worst, kernel, what, got, ref, bar):
    """|got - ref| <= bar for every element (all finite); records the worst ratio of `kernel` in the dict `worst`."""
    got, ref = got.double(), ref.double()
    bar = bar.double().expand_as(ref)
    assert torch.isfinite(got).all(), f"{what}: {int((~torch.isfinite(got)).sum())} non-finite outputs"
    ratio = (got - ref).abs() / bar
    w = ratio.max().item() if ratio.numel() else 0.0
    worst[kernel] = max(worst.get(kernel, 0.0), w)
    if w > 1.0:
        i = int(ratio.flatten().argmax())
        idx = tuple(int(t) for t in torch.unravel_index(torch.tensor(i), ratio.shape))
        nbad = int((ratio > 1.0).sum())
        raise AssertionError(f"{what}: {nbad} of {ratio.numel()} elements over the bar; worst at {idx}: got "
                             f"{got.flatten()[i].item():.9g}, ref {ref.flatten()[i].item():.9g}, bar "
                             f"{bar.flatten()[i].item():.3g} ({w:.1f}x)")
    return w
