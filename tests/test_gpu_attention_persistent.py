"""-m gpu: the persistent, warp-specialised flash attention (csrc/attention_tc3.cu) on the hazards of its design: many
query tiles per CTA with query and key tails of every kind, barrier phases reused across tiles, lazy rescaling with large
fp16 logits, and launches of a single key chunk (nothing to prefetch)."""
import pytest
import torch
import torch.nn.functional as F

from dinounet_b200 import lib as L
from tests.gpu_helpers import TD, P, rel_err, stream

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _inputs(B, Hh, N, hd, td, seed=0, q_scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed + N + hd)
    q, k, v = (torch.randn(B, Hh, N, hd, generator=g).to(DEV) for _ in range(3))
    q, k, v = (q * q_scale).to(td), k.to(td), v.to(td)
    npad = (N + 7) // 8 * 8
    vt = torch.zeros(B, Hh, hd, npad, device=DEV, dtype=td)
    vt[..., :N] = v.transpose(2, 3)
    return q, k, v, vt, npad


def _attend(lib, q, k, vt, out, B, Hh, N, npad, hd, dtype):
    """NaN-filled out: a row the kernel never writes fails the finiteness check."""
    out.fill_(float("nan"))
    L.check(lib.b2u_attention_tc_hd(P(q), P(k), P(vt), P(out), B, Hh, N, npad, hd, hd ** -0.5, dtype, stream()), "attn")
    torch.cuda.synchronize()


def _ref(q, k, v, B, N, Hh, hd):
    return F.scaled_dot_product_attention(q.float(), k.float(), v.float()).transpose(1, 2).reshape(B, N, Hh * hd)


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("N", [1029, 1040, 1041, 1088, 1089, 1151, 1153])
def test_many_tiles_per_cta_mixed_tails(hd, N):
    """B*H*qtiles >= 128 * 6 tiles >> #SMs.  Key tails of 5, 16, 17, 64, 65, 127 and 1 keys (MMA widths n16 / n16 / n32 /
    n64 / n128 / n128 / n16); the last query tile (192 rows at head_dim 64, 128 at 128) holds between 1 and 191 valid rows,
    so consumer warpgroups with no valid rows, partly valid rows and full rows all occur."""
    lib = L.load()
    dtype, td = L.BF16, torch.bfloat16
    B, Hh = 8, 16
    q, k, v, vt, npad = _inputs(B, Hh, N, hd, td)
    out = torch.empty(B, N, Hh * hd, device=DEV, dtype=td)
    _attend(lib, q, k, vt, out, B, Hh, N, npad, hd, dtype)
    assert torch.isfinite(out.float()).all()
    err = rel_err(out, _ref(q, k, v, B, N, Hh, hd))
    assert err < 2 ** -6, err


@pytest.mark.parametrize("hd", [64, 128])
def test_phase_reuse_across_tiles_is_deterministic(hd):
    """Every CTA runs >= 8 tiles (16 * 16 * 6 = 1536 tiles of 192 rows at head_dim 64, 2304 of 128 rows at 128, on one
    CTA per SM), so every mbarrier and named barrier turns over many phases; two launches must give identical bits."""
    lib = L.load()
    dtype, td = L.BF16, torch.bfloat16
    B, Hh, N = 16, 16, 1029
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows = 192 if hd == 64 else 128
    assert B * Hh * ((N + rows - 1) // rows) >= 8 * sms
    q, k, v, vt, npad = _inputs(B, Hh, N, hd, td, seed=3)
    out = torch.empty(B, N, Hh * hd, device=DEV, dtype=td)
    out2 = torch.empty_like(out)
    _attend(lib, q, k, vt, out, B, Hh, N, npad, hd, dtype)
    _attend(lib, q, k, vt, out2, B, Hh, N, npad, hd, dtype)
    assert torch.isfinite(out.float()).all()
    assert torch.equal(out, out2)


@pytest.mark.parametrize("hd", [64, 128])
def test_fp16_large_logits_lazy_rescale(hd):
    """Q scaled by 8: logits of std ~8, so the running maximum jumps by far more than 8 (log2) and the lazily kept
    maximum leaves probabilities near 2^8 between rescales; fp16 P and O must stay finite and accurate."""
    lib = L.load()
    dtype, td = L.F16, torch.float16
    B, Hh, N = 2, 4, 1029
    q, k, v, vt, npad = _inputs(B, Hh, N, hd, td, seed=7, q_scale=8.0)
    out = torch.empty(B, N, Hh * hd, device=DEV, dtype=td)
    _attend(lib, q, k, vt, out, B, Hh, N, npad, hd, dtype)
    assert torch.isfinite(out.float()).all()
    err = rel_err(out, _ref(q, k, v, B, N, Hh, hd))
    assert err < 2 ** -8, err


@pytest.mark.parametrize("dtype", [L.BF16, L.F16])
@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("N", [77, 128])
def test_single_key_chunk(dtype, hd, N):
    """ntok <= 128: one (masked) key chunk that is both the first and the last, with no next chunk to prefetch."""
    lib = L.load()
    td = TD[dtype]
    B, Hh = 3, 5
    q, k, v, vt, npad = _inputs(B, Hh, N, hd, td, seed=11)
    out = torch.empty(B, N, Hh * hd, device=DEV, dtype=td)
    _attend(lib, q, k, vt, out, B, Hh, N, npad, hd, dtype)
    assert torch.isfinite(out.float()).all()
    err = rel_err(out, _ref(q, k, v, B, N, Hh, hd))
    assert err < (2 ** -6 if dtype == L.BF16 else 2 ** -8), err
