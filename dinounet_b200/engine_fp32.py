"""fp32 parity tier: the launch plan of the whole forward on the plain-SIMT fp32 kernels of csrc/fp32_tier.cu.

`DinoUNet.precision = "fp32"` routes here.  Purpose: BASELINE.json north_star's "1e-5 in fp32" against the reference's
fp32 forward (its CPU regime: the inner autocast self-disables off-GPU, dinov3_adapter.py:422) - which a 16-bit
tensor-core pipeline cannot meet by construction.  Same data layouts, same weight packing (ForwardEngine.pack with
dtype float32) and the same operator order as `ForwardEngine.build_plan`; no fusion beyond the GEMM epilogue, no
tensor cores, not the benchmarked path.  Reference call sites: see the per-section comments (same as engine.py).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Tuple

import torch

from . import config as cfg
from . import lib as L


def _ptr(t):
    return None if t is None else t.data_ptr()


def _patch_attention_rope(args, sin: int, cos: int, keep: list):
    """b2u_f32_attention's arguments (qkv, sin, cos, out, ...) with other RoPE tables."""
    return (args[0], sin, cos) + tuple(args[3:])


def build_plan_fp32(eng, B: int, S: int):
    from .engine import Plan
    if S % 32 or S < 64:
        raise ValueError("fp32 tier: input size must be a multiple of 32 (>= 64)")
    v, w, lib = eng.v, eng.w, eng.lib
    if v.ffn_layer != "mlp":
        raise NotImplementedError("fp32 parity tier implements the Mlp FFN variants (dinounet_s/b/l); SwiGLU (7B) runs on the "
                                  "16-bit tensor-core path only")
    D, Hh, hd = v.embed_dim, v.num_heads, eng.hd
    h = S // 16
    P = h * h
    N = P + cfg.N_PREFIX
    T = B * N
    n4 = (S // 32) ** 2
    n3, n2 = 4 * n4, 16 * n4
    Lq = n2 + n3 + n4
    dev = eng.device
    f32 = torch.float32
    bufs: Dict[str, torch.Tensor] = {}

    def buf(name, shape, dtype=f32):
        t = torch.empty(shape, dtype=dtype, device=dev)
        bufs[name] = t
        return t

    plan = Plan()

    def gemm(name, A, M, K, lda, W, Nn, out, ldc, *, bias=None, scale=None, shift=None, act1=0, act2=0, residual=None,
             ldres=0, col_off=0, rows=None, a_rows=None, ps=None, conv=0, img=(0, 0, 0)):
        p = L.F32GemmParams()
        p.M, p.N, p.K = int(M), int(Nn), int(K)
        p.A, p.lda, p.W, p.ldw = _ptr(A), int(lda), _ptr(W), int(W.shape[1])
        if a_rows is not None:
            p.a_rows_in, p.a_rows_out, p.a_row_off = [int(t) for t in a_rows]
        p.conv = conv
        if conv:
            p.Hin, p.Win, p.C = [int(t) for t in img]
            p.Cpad = int(K) // 9
        p.out, p.ldc, p.col_off = _ptr(out), int(ldc), int(col_off)
        if rows is not None:
            p.rows_in, p.rows_out, p.row_off = [int(t) for t in rows]
        if ps is not None:
            p.ps_cout, p.ps_h, p.ps_w = [int(t) for t in ps]
        p.bias, p.scale, p.shift = _ptr(bias), _ptr(scale), _ptr(shift)
        p.act1, p.act2 = act1, act2
        p.residual, p.ldres = _ptr(residual), int(ldres)
        plan.keep.append(p)
        plan.add(name, lib.b2u_f32_gemm, C.byref(p))

    def ln(name, src, dst, wk, bk, rows, eps, remap=(0, 0, 0)):
        plan.add(name, lib.b2u_f32_layernorm, _ptr(src), _ptr(dst), _ptr(w[wk]), _ptr(w[bk]), rows, D, eps, *remap)

    x = buf("x", (B, 3, S, S))

    # ================= ViT (vision_transformer.py:265-318) =================
    Ape = buf("Ape", (B * P, 768))
    X = buf("X", (T, D))
    Y = buf("Y", (T, D))
    QKV = buf("QKV", (T, 3 * D))
    O = buf("O", (T, D))
    Hid = buf("Hid", (T, v.ffn_hidden))
    taps = [buf(f"tap{k}", (B * P, D)) for k in range(4)]
    sin, cos = eng._rope_tables(h, h)
    bufs["rope_sin"], bufs["rope_cos"] = sin, cos
    plan.add("patchify", lib.b2u_f32_patchify, _ptr(x), _ptr(Ape), B, S)
    gemm("patch_embed", Ape, B * P, 768, 768, w["pe.w"], D, X, D, bias=w["pe.b"], rows=(P, N, cfg.N_PREFIX))
    plan.add("prefix", lib.b2u_write_prefix, _ptr(X), _ptr(w["prefix"]), B, N, cfg.N_PREFIX, D)
    tap_k = 0
    for i in range(v.depth):
        ln(f"b{i}.ln1", X, Y, f"b{i}.n1w", f"b{i}.n1b", T, cfg.LN_EPS_VIT)
        gemm(f"b{i}.qkv", Y, T, D, D, w[f"b{i}.qkv"], 3 * D, QKV, 3 * D, bias=w.get(f"b{i}.qkvb"))
        plan.rope_sites.append((len(plan.calls), i, _patch_attention_rope))
        plan.add(f"b{i}.attn", lib.b2u_f32_attention, _ptr(QKV), _ptr(sin), _ptr(cos), _ptr(O), B, N, Hh, hd, cfg.N_PREFIX,
                 hd ** -0.5)
        gemm(f"b{i}.proj", O, T, D, D, w[f"b{i}.proj"], D, X, D, bias=w[f"b{i}.projb"], scale=w[f"b{i}.ls1"], residual=X, ldres=D)
        ln(f"b{i}.ln2", X, Y, f"b{i}.n2w", f"b{i}.n2b", T, cfg.LN_EPS_VIT)
        gemm(f"b{i}.fc1", Y, T, D, D, w[f"b{i}.fc1"], v.ffn_hidden, Hid, v.ffn_hidden, bias=w[f"b{i}.fc1b"], act1=L.ACT_GELU)
        gemm(f"b{i}.fc2", Hid, T, v.ffn_hidden, v.ffn_hidden, w[f"b{i}.fc2"], D, X, D, bias=w[f"b{i}.fc2b"], scale=w[f"b{i}.ls2"],
             residual=X, ldres=D)
        if i in v.interaction_indexes:
            ln(f"tap{tap_k}", X, taps[tap_k], "norm.w", "norm.b", B * P, cfg.LN_EPS_VIT, (N, P, cfg.N_PREFIX))
            tap_k += 1

    plan.vit_end = len(plan.calls)

    # ================= SPM (dinov3_adapter.py:279-302) =================
    S2, S4, S8, S16, S32 = S // 2, S // 4, S // 8, S // 16, S // 32
    xh = buf("x_nhwc", (B * S * S, 3))
    sA = buf("spmA", (B * S2 * S2, 64))
    sB = buf("spmB", (B * S2 * S2, 64))
    pool = buf("pool", (B * S4 * S4, 64))
    c2s = buf("c2s", (B * S8 * S8, 128))
    c3s = buf("c3s", (B * S16 * S16, 256))
    c4s = buf("c4s", (B * S32 * S32, 256))
    c1 = buf("c1", (B * S4 * S4, D))
    Cst = buf("Cst", (B * Lq, D))
    plan.add("nhwc", lib.b2u_f32_nchw_to_nhwc, _ptr(x), _ptr(xh), B, 3, S * S)

    def conv_bn_relu(name, src, dst, cin, cout, hin, stride, wkey=None):
        W = w[wkey or (name + ".w")]
        gemm(name, src, B * (hin // stride) ** 2, W.shape[1], cin, W, cout, dst, cout, scale=w[name + ".sc"], shift=w[name + ".sh"],
             act2=L.ACT_RELU, conv=L.CONV3X3_S2 if stride == 2 else L.CONV3X3_S1, img=(hin, hin, cin))

    conv_bn_relu("stem0", xh, sA, 3, 64, S, 2, wkey="stem0.w3")
    conv_bn_relu("stem3", sA, sB, 64, 64, S2, 1)
    conv_bn_relu("stem6", sB, sA, 64, 64, S2, 1)
    plan.add("maxpool", lib.b2u_f32_maxpool3x3s2, _ptr(sA), _ptr(pool), B, S2, S2, 64)
    conv_bn_relu("conv2", pool, c2s, 64, 128, S4, 2)
    conv_bn_relu("conv3", c2s, c3s, 128, 256, S8, 2)
    conv_bn_relu("conv4", c3s, c4s, 256, 256, S16, 2)
    gemm("spm.fc1", pool, B * S4 * S4, 64, 64, w["spmfc1.w"], D, c1, D, bias=w["spmfc1.b"])
    le = w["level_embed"]
    for i, (src, kk, nl, off) in enumerate(((c2s, 128, n2, 0), (c3s, 256, n3, n2), (c4s, 256, n4, n2 + n3))):
        gemm(f"spm.fc{i + 2}", src, B * nl, kk, kk, w[f"spmfc{i + 2}.w"], D, Cst, D, bias=w[f"spmfc{i + 2}.b"], shift=le[i],
             rows=(nl, Lq, off))

    # ================= interaction blocks (dinov3_adapter.py:140-231) =================
    QN = buf("QN", (B * Lq, D))
    FN = buf("FN", (B * P, D))
    VAL = buf("VAL", (B * P, D // 2))
    OFFAW = buf("OFFAW", (B * Lq, 192))
    SAMP = buf("SAMP", (B * Lq, D // 2))
    F1 = buf("F1", (B * Lq, D // 4))
    F2 = buf("F2", (B * Lq, D // 4))
    dh = (D // 2) // cfg.DEFORM_HEADS
    for e, k in enumerate((0, 1, 2, 3, 3, 3)):
        pre = f"e{e}."
        ln(pre + "qnorm", Cst, QN, pre + "query_norm.w", pre + "query_norm.b", B * Lq, cfg.LN_EPS_ADAPTER)
        ln(pre + "fnorm", taps[k], FN, pre + "feat_norm.w", pre + "feat_norm.b", B * P, cfg.LN_EPS_ADAPTER)
        gemm(pre + "value", FN, B * P, D, D, w[pre + "val"], D // 2, VAL, D // 2, bias=w[pre + "valb"])
        gemm(pre + "offaw", QN, B * Lq, D, D, w[pre + "offaw"], 192, OFFAW, 192, bias=w[pre + "offawb"])
        plan.add(pre + "msda", lib.b2u_f32_msda, _ptr(VAL), _ptr(OFFAW), _ptr(SAMP), B, h, h, cfg.DEFORM_HEADS, dh)
        gemm(pre + "outproj", SAMP, B * Lq, D // 2, D // 2, w[pre + "out"], D, Cst, D, bias=w[pre + "outb"], residual=Cst, ldres=D)
        ln(pre + "ffnnorm", Cst, QN, pre + "ffn_norm.w", pre + "ffn_norm.b", B * Lq, cfg.LN_EPS_ADAPTER)
        gemm(pre + "ffn1", QN, B * Lq, D, D, w[pre + "f1"], D // 4, F1, D // 4, bias=w[pre + "f1b"])
        plan.add(pre + "dwconv", lib.b2u_f32_dwconv3x3, _ptr(F1), _ptr(F2), _ptr(w[pre + "dw"]), _ptr(w[pre + "dwb"]), B, S16, S16,
                 D // 4, 3, L.ACT_GELU)
        gemm(pre + "ffn2", F2, B * Lq, D // 4, D // 4, w[pre + "f2"], D, Cst, D, bias=w[pre + "f2b"], residual=Cst, ldres=D)

    # ================= adapter tail (dinov3_adapter.py:460-482) =================
    UP = buf("UP", (B * S4 * S4, D))
    fs = [buf("f1", (B * S4 * S4, D)), buf("f2", (B * n2, D)), buf("f3", (B * n3, D)), buf("f4", (B * n4, D))]
    gemm("up", Cst, B * n2, D, D, w["up.w"], 4 * D, UP, D, bias=w["up.b"], a_rows=(n2, Lq, 0), ps=(D, S8, S8), residual=c1, ldres=D)
    plan.add("tail1", lib.b2u_f32_tail, _ptr(UP), S4 * S4, 0, _ptr(taps[0]), _ptr(fs[0]), _ptr(w["bn1.sc"]), _ptr(w["bn1.sh"]),
             B, S4, h, D)
    for i, (off, res) in enumerate(((0, S8), (n2, S16), (n2 + n3, S32))):
        plan.add(f"tail{i + 2}", lib.b2u_f32_tail, _ptr(Cst), Lq, off, _ptr(taps[i + 1]), _ptr(fs[i + 1]), _ptr(w[f"bn{i + 2}.sc"]),
                 _ptr(w[f"bn{i + 2}.sh"]), B, res, h, D)

    # ================= FAPM + ups (dinounet_training.py:419-441, 255-264, 499-510) =================
    R = cfg.FAPM_RANK
    px0 = B * S4 * S4
    ZZ = buf("ZZ", (px0, 2 * R))
    GB = buf("GB", (px0, 2 * R))
    Z = buf("Z", (px0, R))
    RS = buf("RS", (px0 * 64,))
    T1 = buf("T1", (px0 * 32,))
    T2 = buf("T2", (px0 * 32,))
    Yf = buf("Yf", (px0 * 32,))
    U1 = buf("U1", (px0 * 4 * 32,))
    pooled = buf("pooled", (B, 256))
    in_work = buf("in_work", (2 * B * 256,), torch.float64)
    in_stats = buf("in_stats", (B * 256 * 2,))
    feats = eng.features
    cat = [buf("cat0", (B * S4 * S4, 2 * feats[2])), buf("cat1", (B * S2 * S2, 2 * feats[1])), buf("cat2", (B * S * S, 2 * feats[0]))]
    skip3 = buf("skip3", (B * S8 * S8, feats[3]))
    for i, oc in enumerate(feats):
        r = S4 >> i
        px = B * r * r
        pre = f"f{i}."
        has_sc = oc != R
        n3_ = 2 * oc if has_sc else oc
        gemm(pre + "bases", fs[i], px, D, D, w[pre + "w1"], 2 * R, ZZ, 2 * R, bias=w[pre + "b1"])
        gemm(pre + "film_gen", ZZ, px, R, 2 * R, w[pre + "film"], 2 * R, GB, 2 * R, bias=w[pre + "filmb"])
        plan.add(pre + "film", lib.b2u_f32_film, _ptr(GB), _ptr(ZZ), _ptr(Z), px, R)
        gemm(pre + "reduce_sc", Z, px, R, R, w[pre + "w3"], n3_, RS, n3_, bias=w[pre + "b3"])
        plan.add(pre + "in1", lib.b2u_f32_instnorm, _ptr(RS), n3_, _ptr(T1), oc, _ptr(w[pre + "in1w"]), _ptr(w[pre + "in1b"]), _ptr(in_work),
                 _ptr(in_stats), B, r * r, oc, cfg.IN_EPS, 1)
        plan.add(pre + "dw", lib.b2u_f32_dwconv3x3, _ptr(T1), _ptr(T2), _ptr(w[pre + "dw"]), _ptr(w[pre + "dwb"]), B, r, r, oc, 1,
                 L.ACT_NONE)
        gemm(pre + "pw", T2, px, oc, oc, w[pre + "pw"], oc, T1, oc, bias=w[pre + "pwb"])
        plan.add(pre + "in2", lib.b2u_f32_instnorm, _ptr(T1), oc, _ptr(T2), oc, _ptr(w[pre + "in2w"]), _ptr(w[pre + "in2b"]), _ptr(in_work),
                 _ptr(in_stats), B, r * r, oc, cfg.IN_EPS, 1)
        gemm(pre + "refine", T2, px, oc, oc, w[pre + "ref"], oc, T1, oc, bias=w[pre + "refb"])
        if has_sc:
            sc_ptr, ldsc = RS.data_ptr() + oc * 4, n3_
        else:
            sc_ptr, ldsc = Z.data_ptr(), R
        plan.add(pre + "se", lib.b2u_f32_se, _ptr(T1), sc_ptr, ldsc, _ptr(pooled), _ptr(w[pre + "se1"]), _ptr(w[pre + "se1b"]),
                 _ptr(w[pre + "se2"]), _ptr(w[pre + "se2b"]), _ptr(Yf), B, r * r, oc, max(1, oc // 16))
        gemm(f"ups{i}.a", Yf, px, oc, oc, w[f"ups{i}.w"], 4 * oc, U1, oc, bias=w[f"ups{i}.b"], ps=(oc, r, r))
        if i < 3:
            dst, ldc, coff = cat[2 - i], 2 * oc, oc
        else:
            dst, ldc, coff = skip3, oc, 0
        gemm(f"ups{i}.b", U1, 4 * px, oc, oc, w[f"ups{i}.w"], 4 * oc, dst, ldc, bias=w[f"ups{i}.b"], ps=(oc, 2 * r, 2 * r), col_off=coff)

    # ================= decoder (dinounet_training.py:603-629) =================
    CO = buf("CO", (B * S * S * 32,))
    CA = buf("CA", (B * S * S * 32,))
    lin = buf("lin", (B * S * S, eng.ncls))
    logits = buf("logits", (B, eng.ncls, S, S))
    labels = buf("labels", (B, S, S), torch.uint8)
    lres, below = skip3, feats[3]
    for s in range(3):
        skip = feats[2 - s]
        r_lo = S8 << s
        r_hi = 2 * r_lo
        gemm(f"d{s}.transp", lres, B * r_lo * r_lo, below, below, w[f"d{s}.t"], 4 * skip, cat[s], 2 * skip, bias=w[f"d{s}.tb"],
             ps=(skip, r_lo, r_lo))
        src, cin = cat[s], 2 * skip
        for j in range(2):
            W = w[f"d{s}.c{j}"]
            gemm(f"d{s}.conv{j}", src, B * r_hi * r_hi, W.shape[1], cin, W, skip, CO, skip, bias=w[f"d{s}.c{j}b"],
                 conv=L.CONV3X3_S1, img=(r_hi, r_hi, cin))
            plan.add(f"d{s}.in{j}", lib.b2u_f32_instnorm, _ptr(CO), skip, _ptr(CA), skip, _ptr(w[f"d{s}.n{j}w"]),
                     _ptr(w[f"d{s}.n{j}b"]), _ptr(in_work), _ptr(in_stats), B, r_hi * r_hi, skip, cfg.IN_EPS, 1)
            src, cin = CA, skip
        lres, below = CA, skip
    gemm("seg", CA, B * S * S, feats[0], feats[0], w["seg.w"], eng.ncls, lin, eng.ncls, bias=w["seg.b"])
    plan.add("seg_out", lib.b2u_f32_seg_out, _ptr(lin), _ptr(logits), _ptr(labels), B, S * S, eng.ncls)
    return plan, bufs
