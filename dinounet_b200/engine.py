"""Forward engine: packs a Dino U-Net state dict into kernel-native layouts and runs the forward as a fixed launch
plan of hand-written sm_90a kernels (through the C-ABI in include/dinounet_b200.h).

Data layout in HBM (everything channels-last / token-major, C contiguous):
  * ViT residual stream X  [B*ntok, D] fp32; GEMM operands (LN outputs, q/k/v [B,H,ntok,64], attention out, MLP hidden)
    in the ViT 16-bit type (bf16 by default = the reference's inner autocast, dinov3_adapter.py:422).
  * adapter query stream C [B*Lq, D] fp32 (the reference keeps it fp32: fp16 + fp32 level_embed promotes);
    ViT taps [B*P, D] fp32 (LayerNorm output under autocast is fp32).
  * SPM / FAPM / decoder activations NHWC in the "rest" 16-bit type (fp16 by default = the outer autocast,
    predict_from_raw_data.py:695); concat buffers are written in place by the producing GEMM epilogues.
  * weights: [N, K] K-major 16-bit (conv: [N, 9*Cpad], ConvT: [(a,b,co), ci]); biases / norm params fp32.

The plan is a list of (C function, ctypes args) built once per (batch, size); `run` just replays it on a stream, so it
can be captured into a CUDA graph.  There is no PyTorch fallback: torch only owns the device memory.
"""
from __future__ import annotations

import ctypes as C
import math
import threading
from collections import OrderedDict
from contextlib import contextmanager
from typing import Dict, Iterable, List, Optional, Tuple

import torch

from . import config as cfg
from . import lib as L

_TORCH16 = {L.F16: torch.float16, L.BF16: torch.bfloat16}
_CODE = {"fp16": L.F16, "f16": L.F16, "half": L.F16, "bf16": L.BF16, "bfloat16": L.BF16}


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _patch_qkv_rope(args, sin: int, cos: int, keep: list):
    """b2u_qkv_rope's arguments with other RoPE tables (a copy of its parameter block)."""
    qp = L.QkvParams.from_buffer_copy(args[0]._obj)
    qp.rope_sin, qp.rope_cos = sin, cos
    keep.append(qp)
    return (C.byref(qp),)


class _CaptureGuard:
    """Keeps other threads' device work out of CUDA graph captures.  A capture in CUDA's default (global) mode fails,
    together with the caller, when another thread makes a call that is not allowed during a capture (an allocation, a
    synchronisation).  Threads that run device work beside the engine (the prediction's export writers) do it inside
    `device_work()`; a capture waits until none of them is inside and keeps new ones out until it ends."""

    def __init__(self):
        self._cv = threading.Condition()
        self._workers = 0
        self._capturing = False

    @contextmanager
    def capture(self):
        with self._cv:
            self._cv.wait_for(lambda: not self._capturing)
            self._capturing = True
            self._cv.wait_for(lambda: self._workers == 0)
        try:
            yield
        finally:
            with self._cv:
                self._capturing = False
                self._cv.notify_all()

    @contextmanager
    def device_work(self):
        with self._cv:
            self._cv.wait_for(lambda: not self._capturing)
            self._workers += 1
        try:
            yield
        finally:
            with self._cv:
                self._workers -= 1
                self._cv.notify_all()


#: the process's guard around every graph capture of the engines (see `_CaptureGuard`)
GRAPH_CAPTURE = _CaptureGuard()


class Plan:
    """A recorded sequence of C-ABI calls with their (kept-alive) arguments."""

    def __init__(self):
        self.calls: List[Tuple[str, object, tuple]] = []
        self.keep: list = []
        self.vit_end = 0        # calls[:vit_end] = the frozen ViT (patch embed .. taps); calls[vit_end:] = adapter/FAPM/decoder
        # (call index, ViT block, patch(args, sin_ptr, cos_ptr, keep) -> args) for every call that reads the RoPE tables
        self.rope_sites: list = []
        self.scaled_vit = None  # (Plan, scales buffer): the ViT section on per-block rescaled RoPE tables, built on first use
        self.ds = None          # (Plan, [logits@S, @S/2, @S/4]): the deep-supervision forward on these buffers (`ds_plan`)

    def add(self, name: str, fn, *args):
        self.calls.append((name, fn, args))

    def run(self, stream: int, start: int = 0, end: Optional[int] = None):
        s = C.c_void_p(stream)
        for name, fn, args in self.calls[start:end]:
            rc = fn(*args, s)
            if rc != 0:
                raise L.NativeLibraryError(f"{name} failed (rc={rc}): {L.last_error()}")

    def __len__(self):
        return len(self.calls)


class ForwardEngine:
    def __init__(self, variant: str, params: Dict[str, torch.Tensor], num_classes: int, device: torch.device,
                 vit_dtype: str = "bf16", rest_dtype: str = "fp16", features=(32, 64, 128, 256),
                 attn_impl: str = "tc", query_dtype: str = "fp32", precision: str = "16"):
        if variant not in cfg.VARIANTS:
            raise ValueError(f"Unknown model: {variant}")
        self.v = cfg.VARIANTS[variant]
        self.hd = self.v.embed_dim // self.v.num_heads
        if self.hd not in (64, 128) or self.v.ffn_layer not in ("mlp", "swiglu64"):
            raise NotImplementedError(f"{variant}: kernels exist for head_dim 64/128 and mlp / swiglu64 FFNs")
        if attn_impl != "tc":
            raise NotImplementedError("the only attention kernel is the wgmma one (attn_impl='tc'); the first-generation "
                                      "mma.sync kernel was removed in round 2")
        if tuple(features) != (32, 64, 128, 256):
            raise NotImplementedError("kernels are built for the planner's features_per_stage=(32,64,128,256)")
        self.lib = L.load()
        self.device = device
        self.ncls = int(num_classes)
        # precision "16" (default): bf16/fp16 tensor-core path.  "fp32": the parity tier of engine_fp32.py / csrc/fp32_tier.cu
        # (plain fp32 SIMT kernels, same layouts and packing with dtype float32; held to 1e-5 against the reference's fp32
        # forward, not benchmarked).
        if precision not in ("16", "fp32"):
            raise ValueError("precision must be '16' or 'fp32'")
        self.precision = precision
        self.vt, self.rt = _CODE[vit_dtype], _CODE[rest_dtype]
        if precision == "fp32":
            self.tv = self.tr = torch.float32
        else:
            self.tv, self.tr = _TORCH16[self.vt], _TORCH16[self.rt]
        self.features = tuple(features)
        self.attn_impl = attn_impl   # "tc" = wgmma flash-attention kernel
        # The adapter's query stream c [B, 5376, D] (dinov3_adapter.py:210-231).  "fp32" (default) = the reference's dtype
        # under autocast: the 16-bit SPM outputs are promoted to fp32 by `c + level_embed` (fp32 parameter) and stay fp32
        # through `query + attn`.  "16" = opt-in: stored in rest_dtype, every residual update rounded to 16 bits (half the
        # HBM traffic of the 12 stream passes per step; measured +4.4 % throughput, rel err 7.8e-3 -> 8.0e-3).
        if query_dtype not in ("16", "fp32"):
            raise ValueError("query_dtype must be '16' or 'fp32'")
        self.c16 = query_dtype == "16"
        self.w: Dict[str, torch.Tensor] = {}
        # (B, S) -> (plan, buffers) in LRU order; every entry owns a full activation buffer set (GBs at B=32, 512^2) and
        # possibly a CUDA graph, so ragged last batches / varying tile batches must not accumulate without bound
        self._plans: "OrderedDict[Tuple[int, int], Tuple[Plan, dict]]" = OrderedDict()
        self._graphs: Dict[Tuple[int, int], object] = {}
        self.max_plans = 4
        # fold weight sets (`pack_folds`): the packed weights after the taps of each fold of a run whose folds share this
        # engine's backbone, and per (B, S) one "rest" launch list per fold on that plan's buffers
        self._folds: List[Dict[str, torch.Tensor]] = []
        self._fold_plans: Dict[Tuple[int, int], List[Plan]] = {}
        if self.device.type != "cuda":
            raise L.NativeLibraryError("dinounet_b200 runs on CUDA devices only (no CPU fallback)")
        with torch.cuda.device(self.device):
            self.pack(params)

    # ------------------------------------------------------------------ weight packing
    def _dev(self, t: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
        return t.detach().to(device=self.device, dtype=dtype).contiguous()

    def _lin(self, w: torch.Tensor, dt) -> torch.Tensor:
        """[N, K] (or 1x1 conv [N, K, 1, 1]) -> K-major 16-bit."""
        return self._dev(w.reshape(w.shape[0], -1), dt)

    def _conv3(self, w: torch.Tensor, dt) -> torch.Tensor:
        """[N, C, 3, 3] -> [N, 9*Cpad], k = (ky*3+kx)*Cpad + c."""
        N, Cc = w.shape[0], w.shape[1]
        cpad = (Cc + 63) // 64 * 64
        p = torch.zeros(N, 9, cpad, dtype=torch.float32)
        p[:, :, :Cc] = w.detach().float().cpu().permute(0, 2, 3, 1).reshape(N, 9, Cc)
        return self._dev(p.reshape(N, 9 * cpad), dt)

    def _convT(self, w: torch.Tensor, dt) -> torch.Tensor:
        """ConvTranspose2d [Cin, Cout, 2, 2] -> [(a*2+b)*Cout + co, ci]."""
        ci, co = w.shape[0], w.shape[1]
        return self._dev(w.detach().float().permute(2, 3, 1, 0).reshape(4 * co, ci), dt)

    def _bn_fold(self, P, p) -> Tuple[torch.Tensor, torch.Tensor]:
        sc = P[p + ".weight"].float() / torch.sqrt(P[p + ".running_var"].float() + cfg.BN_EPS)
        sh = P[p + ".bias"].float() - P[p + ".running_mean"].float() * sc
        return self._dev(sc), self._dev(sh)

    def pack(self, P: Dict[str, torch.Tensor]):
        """(Re)build the kernel-native weight copies from a reference-keyed state dict."""
        w = self._pack_vit(P)
        w.update(self._pack_rest(P))
        self.w = w
        self._plans.clear()
        self._graphs.clear()
        self._folds = []
        self._fold_plans.clear()

    def _pack_vit(self, P: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        """The frozen backbone's packed weights (patch embed .. final norm): what the plan's ViT section reads."""
        v, w = self.v, {}
        D = v.embed_dim
        A = "encoder.dinov3_adapter."
        Bk = A + "backbone."
        tv = self.tv
        f32 = self._dev
        # ---- ViT
        w["pe.w"] = self._lin(P[Bk + "patch_embed.proj.weight"], tv)
        w["pe.b"] = f32(P[Bk + "patch_embed.proj.bias"])
        cls = P[Bk + "cls_token"].float() + 0 * P[Bk + "mask_token"].float()
        w["prefix"] = f32(torch.cat([cls.reshape(1, D), P[Bk + "storage_tokens"].float().reshape(-1, D)], 0))
        w["periods"] = P[Bk + "rope_embed.periods"].detach().float().cpu()
        for i in range(v.depth):
            p = f"{Bk}blocks.{i}."
            w[f"b{i}.n1w"], w[f"b{i}.n1b"] = f32(P[p + "norm1.weight"]), f32(P[p + "norm1.bias"])
            w[f"b{i}.qkv"] = self._lin(P[p + "attn.qkv.weight"], tv)
            if v.qkv_bias:
                w[f"b{i}.qkvb"] = f32(P[p + "attn.qkv.bias"].float() * P[p + "attn.qkv.bias_mask"].float())
            w[f"b{i}.proj"], w[f"b{i}.projb"] = self._lin(P[p + "attn.proj.weight"], tv), f32(P[p + "attn.proj.bias"])
            w[f"b{i}.ls1"], w[f"b{i}.ls2"] = f32(P[p + "ls1.gamma"]), f32(P[p + "ls2.gamma"])
            w[f"b{i}.n2w"], w[f"b{i}.n2b"] = f32(P[p + "norm2.weight"]), f32(P[p + "norm2.bias"])
            if v.ffn_layer == "mlp":
                w[f"b{i}.fc1"], w[f"b{i}.fc1b"] = self._lin(P[p + "mlp.fc1.weight"], tv), f32(P[p + "mlp.fc1.bias"])
                w[f"b{i}.fc2"], w[f"b{i}.fc2b"] = self._lin(P[p + "mlp.fc2.weight"], tv), f32(P[p + "mlp.fc2.bias"])
            else:   # SwiGLU (ffn_layers.py:73-77): w1|w2 interleaved in 32-row blocks for the fused silu(x1)*x2 epilogue
                hid = v.ffn_hidden
                w1, w2 = P[p + "mlp.w1.weight"].float(), P[p + "mlp.w2.weight"].float()
                w[f"b{i}.fc1"] = self._dev(torch.stack([w1.view(hid // 32, 32, D), w2.view(hid // 32, 32, D)], 1).reshape(2 * hid, D), tv)
                w[f"b{i}.fc1b"] = f32(torch.stack([P[p + "mlp.w1.bias"].float().view(hid // 32, 32),
                                                   P[p + "mlp.w2.bias"].float().view(hid // 32, 32)], 1).reshape(2 * hid))
                w[f"b{i}.fc2"], w[f"b{i}.fc2b"] = self._lin(P[p + "mlp.w3.weight"], tv), f32(P[p + "mlp.w3.bias"])
        w["norm.w"], w["norm.b"] = f32(P[Bk + "norm.weight"]), f32(P[Bk + "norm.bias"])
        return w

    def _pack_rest(self, P: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        """The packed weights after the taps (SPM, extractors, adapter tail, FAPM, ups, decoder, seg head): the part that
        differs between the folds of one training run."""
        w = {}
        A = "encoder.dinov3_adapter."
        tr = self.tr
        f32 = self._dev
        # ---- SPM
        S = A + "spm."
        w["stem0.w"] = f32(P[S + "stem.0.weight"])
        w["stem0.sc"], w["stem0.sh"] = self._bn_fold(P, S + "stem.1")
        if self.precision == "fp32":
            w["stem0.w3"] = self._conv3(P[S + "stem.0.weight"], torch.float32)
        for name, conv, bn in (("stem3", "stem.3", "stem.4"), ("stem6", "stem.6", "stem.7"), ("conv2", "conv2.0", "conv2.1"),
                               ("conv3", "conv3.0", "conv3.1"), ("conv4", "conv4.0", "conv4.1")):
            w[name + ".w"] = self._conv3(P[S + conv + ".weight"], tr)
            w[name + ".sc"], w[name + ".sh"] = self._bn_fold(P, S + bn)
        for i in range(1, 5):
            w[f"spmfc{i}.w"] = self._lin(P[S + f"fc{i}.weight"], tr)
            w[f"spmfc{i}.b"] = f32(P[S + f"fc{i}.bias"])
        w["level_embed"] = f32(P[A + "level_embed"])
        # ---- extractors
        names = [f"{A}interactions.{i}.extractor." for i in range(4)]
        names += [f"{A}interactions.3.extra_extractors.{j}." for j in range(2)]
        for e, p in enumerate(names):
            for nm in ("query_norm", "feat_norm", "ffn_norm"):
                w[f"e{e}.{nm}.w"], w[f"e{e}.{nm}.b"] = f32(P[p + nm + ".weight"]), f32(P[p + nm + ".bias"])
            w[f"e{e}.val"], w[f"e{e}.valb"] = self._lin(P[p + "attn.value_proj.weight"], tr), f32(P[p + "attn.value_proj.bias"])
            w[f"e{e}.offaw"] = self._lin(torch.cat([P[p + "attn.sampling_offsets.weight"].float(),
                                                    P[p + "attn.attention_weights.weight"].float()], 0), tr)
            w[f"e{e}.offawb"] = f32(torch.cat([P[p + "attn.sampling_offsets.bias"].float(),
                                               P[p + "attn.attention_weights.bias"].float()], 0))
            w[f"e{e}.out"], w[f"e{e}.outb"] = self._lin(P[p + "attn.output_proj.weight"], tr), f32(P[p + "attn.output_proj.bias"])
            w[f"e{e}.f1"], w[f"e{e}.f1b"] = self._lin(P[p + "ffn.fc1.weight"], tr), f32(P[p + "ffn.fc1.bias"])
            dw = P[p + "ffn.dwconv.dwconv.weight"].float()
            w[f"e{e}.dw"] = f32(dw.reshape(dw.shape[0], 9).t())
            w[f"e{e}.dwb"] = f32(P[p + "ffn.dwconv.dwconv.bias"])
            w[f"e{e}.f2"], w[f"e{e}.f2b"] = self._lin(P[p + "ffn.fc2.weight"], tr), f32(P[p + "ffn.fc2.bias"])
        w["up.w"] = self._convT(P[A + "up.weight"], tr)
        w["up.b"] = f32(P[A + "up.bias"].float().repeat(4))
        for i in range(1, 5):
            w[f"bn{i}.sc"], w[f"bn{i}.sh"] = self._bn_fold(P, f"{A}norm{i}")
        # ---- FAPM / ups
        Fp = "encoder.fapm."
        for i, oc in enumerate(self.features):
            w[f"f{i}.w1"] = self._lin(torch.cat([P[Fp + "shared_basis.weight"].float(),
                                                 P[f"{Fp}specific_bases.{i}.weight"].float()], 0), tr)
            w[f"f{i}.b1"] = f32(torch.cat([P[Fp + "shared_basis.bias"].float(), P[f"{Fp}specific_bases.{i}.bias"].float()]))
            w[f"f{i}.film"] = self._lin(P[f"{Fp}film_generators.{i}.weight"], tr)
            w[f"f{i}.filmb"] = f32(P[f"{Fp}film_generators.{i}.bias"])
            r = f"{Fp}refinement_blocks.{i}."
            if f"{Fp}shortcut_projections.{i}.weight" in P:
                w[f"f{i}.w3"] = self._lin(torch.cat([P[r + "0.weight"].float(),
                                                     P[f"{Fp}shortcut_projections.{i}.weight"].float()], 0), tr)
                w[f"f{i}.b3"] = f32(torch.cat([P[r + "0.bias"].float(), P[f"{Fp}shortcut_projections.{i}.bias"].float()]))
            else:
                w[f"f{i}.w3"], w[f"f{i}.b3"] = self._lin(P[r + "0.weight"], tr), f32(P[r + "0.bias"])
            w[f"f{i}.in1w"], w[f"f{i}.in1b"] = f32(P[r + "1.weight"]), f32(P[r + "1.bias"])
            dw = P[r + "3.depthwise.weight"].float()
            w[f"f{i}.dw"], w[f"f{i}.dwb"] = f32(dw.reshape(oc, 9).t()), f32(P[r + "3.depthwise.bias"])
            w[f"f{i}.pw"], w[f"f{i}.pwb"] = self._lin(P[r + "3.pointwise.weight"], tr), f32(P[r + "3.pointwise.bias"])
            w[f"f{i}.in2w"], w[f"f{i}.in2b"] = f32(P[r + "3.bn.weight"]), f32(P[r + "3.bn.bias"])
            w[f"f{i}.ref"], w[f"f{i}.refb"] = self._lin(P[r + "4.weight"], tr), f32(P[r + "4.bias"])
            w[f"f{i}.se1"], w[f"f{i}.se1b"] = f32(P[r + "5.fc.0.weight"].reshape(-1, oc)), f32(P[r + "5.fc.0.bias"])
            w[f"f{i}.se2"], w[f"f{i}.se2b"] = f32(P[r + "5.fc.2.weight"].reshape(oc, -1)), f32(P[r + "5.fc.2.bias"])
            w[f"ups{i}.w"] = self._convT(P[f"encoder.ups.{i}.up2.weight"], tr)
            w[f"ups{i}.b"] = f32(P[f"encoder.ups.{i}.up2.bias"].float().repeat(4))
        # ---- decoder
        for s in range(3):
            w[f"d{s}.t"] = self._convT(P[f"decoder.transpconvs.{s}.weight"], tr)
            w[f"d{s}.tb"] = f32(P[f"decoder.transpconvs.{s}.bias"].float().repeat(4))
            for j in range(2):
                p = f"decoder.stages.{s}.convs.{j}."
                w[f"d{s}.c{j}"], w[f"d{s}.c{j}b"] = self._conv3(P[p + "conv.weight"], tr), f32(P[p + "conv.bias"])
                w[f"d{s}.n{j}w"], w[f"d{s}.n{j}b"] = f32(P[p + "norm.weight"]), f32(P[p + "norm.bias"])
        w["seg.w"] = f32(P["decoder.seg_layers.2.weight"].reshape(self.ncls, -1))
        w["seg.b"] = f32(P["decoder.seg_layers.2.bias"])
        for s in range(2):      # the deep-supervision heads on decoder stages 0 and 1 (read by `ds_plan` only)
            if f"decoder.seg_layers.{s}.weight" in P:
                w[f"ds{s}.w"] = f32(P[f"decoder.seg_layers.{s}.weight"].reshape(self.ncls, -1))
                w[f"ds{s}.b"] = f32(P[f"decoder.seg_layers.{s}.bias"])
        return w

    # ------------------------------------------------------------------ plan helpers
    def _rope_tables(self, h: int, wd: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """rope_position_encoding.py:57-106 (eval, 'separate' normalisation, fp32) -> sin, cos [h*w, head_dim]."""
        periods = self.w["periods"]
        ch = torch.arange(0.5, h, dtype=torch.float32) / h
        cw = torch.arange(0.5, wd, dtype=torch.float32) / wd
        coords = torch.stack(torch.meshgrid(ch, cw, indexing="ij"), dim=-1).flatten(0, 1)
        coords = 2.0 * coords - 1.0
        ang = 2 * math.pi * coords[:, :, None] / periods[None, None, :]
        ang = ang.flatten(1, 2).tile(2)
        return self._dev(torch.sin(ang)), self._dev(torch.cos(ang))

    def _gemm(self, plan: Plan, name, A, M, K, lda, W, N, out, ldc, dtype, *, out_fp32=False, col_off=0, rows=None,
              ps=None, bias=None, scale=None, shift=None, act1=0, act2=0, round16=1, residual=None, ldres=0,
              add16=None, ldadd=0, conv=0, img=(0, 0, 0, 0)):
        p = L.GemmParams()
        p.M, p.N, p.K = int(M), int(N), int(K)
        p.A, p.lda = _ptr(A), int(lda)
        p.Wp, p.ldw = _ptr(W), int(W.shape[1])
        p.dtype, p.conv = dtype, conv
        p.B, p.Hin, p.Win, p.C = [int(t) for t in img]
        e = p.epi
        e.out, e.out_fp32, e.ldc, e.col_off = _ptr(out), int(out_fp32), int(ldc), int(col_off)
        if rows is not None:
            e.rows_in, e.rows_out, e.row_off = [int(t) for t in rows]
        if ps is not None:
            e.ps_cout, e.ps_h, e.ps_w = [int(t) for t in ps]
        e.bias, e.scale, e.shift = _ptr(bias), _ptr(scale), _ptr(shift)
        e.act1, e.act2, e.round16 = act1, act2, round16
        e.residual, e.ldres, e.add16, e.ldadd = _ptr(residual), int(ldres), _ptr(add16), int(ldadd)
        plan.keep.append(p)
        plan.add(name, self.lib.b2u_gemm, C.byref(p))

    # ------------------------------------------------------------------ plan
    def build_plan(self, B: int, S: int, w: Optional[Dict[str, torch.Tensor]] = None,
                   share: Optional[Dict[str, torch.Tensor]] = None, ds: bool = False) -> Tuple[Plan, dict]:
        """The (B, S) launch list on the weights `w` (default: the engine's own).  With `share` (the buffers of an
        existing (B, S) plan) every activation buffer is taken from it instead of allocated.  `ds`: also the
        deep-supervision heads seg_layers[1] / [0] on decoder stages 1 / 0, into fp32 NCHW buffers "logits_ds1"
        [B, ncls, S/2, S/2] and "logits_ds2" [B, ncls, S/4, S/4] that are always allocated here."""
        if S < 128 or S % 128:
            # every pyramid level (S/2 ... S/32) must tile: conv row widths multiples of 4, the halo-mode convs multiples of 8,
            # the three-plane depthwise conv S/16 % 8 == 0 -> multiples of 128 (128, 256, 384, 512, 640, ...); the reference's
            # plans force 512
            raise ValueError("input size must be a multiple of 128 (the reference's plan forces 512x512); the fp32 tier takes "
                             "multiples of 32")
        v, lib = self.v, self.lib
        w = self.w if w is None else w
        vt, rt, tv, tr = self.vt, self.rt, self.tv, self.tr
        D, Hh = v.embed_dim, v.num_heads
        h = S // 16
        P = h * h
        N = P + cfg.N_PREFIX
        T = B * N
        n4 = (S // 32) ** 2
        n3, n2 = 4 * n4, 16 * n4
        Lq = n2 + n3 + n4
        dev = self.device
        bufs: Dict[str, torch.Tensor] = {}

        def buf(name, shape, dtype, zero=False):
            if share is not None:
                t = share[name]
            else:
                t = (torch.zeros if zero else torch.empty)(shape, dtype=dtype, device=dev)
            bufs[name] = t
            return t

        plan = Plan()
        x = buf("x", (B, 3, S, S), torch.float32)

        # ================= ViT (vision_transformer.py:265-318) =================
        Ape = buf("Ape", (B * P, 768), tv)
        X = buf("X", (T, D), torch.float32)
        Y = buf("Y", (T, D), tv)
        npad = (N + 7) // 8 * 8
        hd = self.hd
        Q, K_ = buf("Q", (B, Hh, N, hd), tv), buf("K", (B, Hh, N, hd), tv)
        # V^T with zeroed padding columns (never written by the QKV epilogue)
        V = buf("V", (B, Hh, hd, npad), tv, zero=True)
        O = buf("O", (T, D), tv)
        Hid = buf("Hid", (T, v.ffn_hidden), tv)
        taps = [buf(f"tap{k}", (B * P, D), torch.float32) for k in range(4)]
        sin, cos = (share["rope_sin"], share["rope_cos"]) if share is not None else self._rope_tables(h, h)
        bufs["rope_sin"], bufs["rope_cos"] = sin, cos

        plan.add("patchify", lib.b2u_patchify, _ptr(x), _ptr(Ape), B, S, vt)
        self._gemm(plan, "patch_embed", Ape, B * P, 768, 768, w["pe.w"], D, X, D, vt, out_fp32=True,
                   rows=(P, N, cfg.N_PREFIX), bias=w["pe.b"])
        plan.add("prefix", lib.b2u_write_prefix, _ptr(X), _ptr(w["prefix"]), B, N, cfg.N_PREFIX, D)
        tap_k = 0
        for i in range(v.depth):
            plan.add(f"b{i}.ln1", lib.b2u_layernorm, _ptr(X), _ptr(Y), _ptr(w[f"b{i}.n1w"]), _ptr(w[f"b{i}.n1b"]), T, D,
                     cfg.LN_EPS_VIT, 0, 0, 0, 0, vt)
            qp = L.QkvParams()
            qp.B, qp.ntok, qp.D, qp.heads, qp.prefix = B, N, D, Hh, cfg.N_PREFIX
            qp.A, qp.lda, qp.Wp, qp.ldw = _ptr(Y), D, _ptr(w[f"b{i}.qkv"]), D
            qp.bias = _ptr(w.get(f"b{i}.qkvb"))
            qp.rope_sin, qp.rope_cos = _ptr(sin), _ptr(cos)
            qp.q, qp.k, qp.v, qp.dtype = _ptr(Q), _ptr(K_), _ptr(V), vt
            qp.v_transposed, qp.npad = 1, npad
            qp.rope_w = h
            plan.keep.append(qp)
            plan.rope_sites.append((len(plan.calls), i, _patch_qkv_rope))
            plan.add(f"b{i}.qkv", lib.b2u_qkv_rope, C.byref(qp))
            # one launch over all ntok query rows (the 5 cls/storage rows fall in the last query tile, whose consumer
            # warpgroups with no valid rows only keep the barrier protocol; b2u_attention_rows remains available for a
            # split launch)
            if hd == 64:
                plan.add(f"b{i}.attn", lib.b2u_attention_tc, _ptr(Q), _ptr(K_), _ptr(V), _ptr(O), B, Hh, N, npad, 0,
                         hd ** -0.5, vt)
            else:
                plan.add(f"b{i}.attn", lib.b2u_attention_tc_hd, _ptr(Q), _ptr(K_), _ptr(V), _ptr(O), B, Hh, N, npad, hd,
                         hd ** -0.5, vt)
            self._gemm(plan, f"b{i}.proj", O, T, D, D, w[f"b{i}.proj"], D, X, D, vt, out_fp32=True, bias=w[f"b{i}.projb"],
                       scale=w[f"b{i}.ls1"], residual=X, ldres=D)
            plan.add(f"b{i}.ln2", lib.b2u_layernorm, _ptr(X), _ptr(Y), _ptr(w[f"b{i}.n2w"]), _ptr(w[f"b{i}.n2b"]), T, D,
                     cfg.LN_EPS_VIT, 0, 0, 0, 0, vt)
            if v.ffn_layer == "mlp":
                self._gemm(plan, f"b{i}.fc1", Y, T, D, D, w[f"b{i}.fc1"], v.ffn_hidden, Hid, v.ffn_hidden, vt,
                           bias=w[f"b{i}.fc1b"], act1=L.ACT_GELU)
            else:
                self._gemm(plan, f"b{i}.fc1", Y, T, D, D, w[f"b{i}.fc1"], 2 * v.ffn_hidden, Hid, v.ffn_hidden, vt,
                           bias=w[f"b{i}.fc1b"], act1=L.ACT_SWIGLU)
            self._gemm(plan, f"b{i}.fc2", Hid, T, v.ffn_hidden, v.ffn_hidden, w[f"b{i}.fc2"], D, X, D, vt, out_fp32=True,
                       bias=w[f"b{i}.fc2b"], scale=w[f"b{i}.ls2"], residual=X, ldres=D)
            if i in v.interaction_indexes:
                plan.add(f"tap{tap_k}", lib.b2u_layernorm, _ptr(X), _ptr(taps[tap_k]), _ptr(w["norm.w"]), _ptr(w["norm.b"]),
                         B * P, D, cfg.LN_EPS_VIT, N, P, cfg.N_PREFIX, 1, vt)
                tap_k += 1

        plan.vit_end = len(plan.calls)     # everything above depends only on the input image and the FROZEN backbone

        # ================= SPM (dinov3_adapter.py:279-302) =================
        S2, S4, S8, S16, S32 = S // 2, S // 4, S // 8, S // 16, S // 32
        sA = buf("spmA", (B * S2 * S2, 64), tr)
        sB = buf("spmB", (B * S2 * S2, 64), tr)
        pool = buf("pool", (B * S4 * S4, 64), tr)
        c2s = buf("c2s", (B * S8 * S8, 128), tr)
        c3s = buf("c3s", (B * S16 * S16, 256), tr)
        c4s = buf("c4s", (B * S32 * S32, 256), tr)
        c1 = buf("c1", (B * S4 * S4, D), tr)
        c16 = self.c16
        Cst = buf("Cst", (B * Lq, D), tr if c16 else torch.float32)
        ln_c = lib.b2u_layernorm16 if c16 else lib.b2u_layernorm
        plan.add("stem0", lib.b2u_stem_conv0, _ptr(x), _ptr(w["stem0.w"]), _ptr(w["stem0.sc"]), _ptr(w["stem0.sh"]),
                 _ptr(sA), B, S, rt)

        def conv_bn_relu(name, src, dst, cin, cout, hin, stride):
            self._gemm(plan, name, src, 0, 9 * cin, cin, w[name + ".w"], cout, dst, cout, rt, scale=w[name + ".sc"],
                       shift=w[name + ".sh"], act2=L.ACT_RELU, conv=L.CONV3X3_S2 if stride == 2 else L.CONV3X3_S1,
                       img=(B, hin, hin, cin))

        conv_bn_relu("stem3", sA, sB, 64, 64, S2, 1)
        conv_bn_relu("stem6", sB, sA, 64, 64, S2, 1)
        plan.add("maxpool", lib.b2u_maxpool3x3s2, _ptr(sA), _ptr(pool), B, S2, S2, 64, rt)
        conv_bn_relu("conv2", pool, c2s, 64, 128, S4, 2)
        conv_bn_relu("conv3", c2s, c3s, 128, 256, S8, 2)
        conv_bn_relu("conv4", c3s, c4s, 256, 256, S16, 2)
        self._gemm(plan, "spm.fc1", pool, B * S4 * S4, 64, 64, w["spmfc1.w"], D, c1, D, rt, bias=w["spmfc1.b"])
        le = w["level_embed"]
        for i, (src, kk, nl, off) in enumerate(((c2s, 128, n2, 0), (c3s, 256, n3, n2), (c4s, 256, n4, n2 + n3))):
            self._gemm(plan, f"spm.fc{i + 2}", src, B * nl, kk, kk, w[f"spmfc{i + 2}.w"], D, Cst, D, rt, out_fp32=not c16,
                       rows=(nl, Lq, off), bias=w[f"spmfc{i + 2}.b"], shift=le[i])

        # ================= interaction blocks (dinov3_adapter.py:140-231) =================
        QN = buf("QN", (B * Lq, D), tr)
        FN = buf("FN", (B * P, D), tr)
        VAL = buf("VAL", (B * P, D // 2), tr)
        OFFAW = buf("OFFAW", (B * Lq, 192), torch.float32)
        SAMP = buf("SAMP", (B * Lq, D // 2), tr)
        F1 = buf("F1", (B * Lq, D // 4), tr)
        F2 = buf("F2", (B * Lq, D // 4), tr)
        dh = (D // 2) // cfg.DEFORM_HEADS
        for e, k in enumerate((0, 1, 2, 3, 3, 3)):
            pre = f"e{e}."
            plan.add(pre + "qnorm", ln_c, _ptr(Cst), _ptr(QN), _ptr(w[pre + "query_norm.w"]),
                     _ptr(w[pre + "query_norm.b"]), B * Lq, D, cfg.LN_EPS_ADAPTER, 0, 0, 0, 0, rt)
            plan.add(pre + "fnorm", lib.b2u_layernorm, _ptr(taps[k]), _ptr(FN), _ptr(w[pre + "feat_norm.w"]),
                     _ptr(w[pre + "feat_norm.b"]), B * P, D, cfg.LN_EPS_ADAPTER, 0, 0, 0, 0, rt)
            self._gemm(plan, pre + "value", FN, B * P, D, D, w[pre + "val"], D // 2, VAL, D // 2, rt, bias=w[pre + "valb"])
            self._gemm(plan, pre + "offaw", QN, B * Lq, D, D, w[pre + "offaw"], 192, OFFAW, 192, rt, out_fp32=True,
                       bias=w[pre + "offawb"])
            plan.add(pre + "msda", lib.b2u_msda_forward, _ptr(VAL), _ptr(OFFAW), _ptr(SAMP), B, h, h, cfg.DEFORM_HEADS, dh,
                     cfg.DEFORM_POINTS, rt)
            if c16:
                self._gemm(plan, pre + "outproj", SAMP, B * Lq, D // 2, D // 2, w[pre + "out"], D, Cst, D, rt,
                           bias=w[pre + "outb"], add16=Cst, ldadd=D)
            else:
                self._gemm(plan, pre + "outproj", SAMP, B * Lq, D // 2, D // 2, w[pre + "out"], D, Cst, D, rt, out_fp32=True,
                           bias=w[pre + "outb"], residual=Cst, ldres=D)
            plan.add(pre + "ffnnorm", ln_c, _ptr(Cst), _ptr(QN), _ptr(w[pre + "ffn_norm.w"]),
                     _ptr(w[pre + "ffn_norm.b"]), B * Lq, D, cfg.LN_EPS_ADAPTER, 0, 0, 0, 0, rt)
            self._gemm(plan, pre + "ffn1", QN, B * Lq, D, D, w[pre + "f1"], D // 4, F1, D // 4, rt, bias=w[pre + "f1b"])
            plan.add(pre + "dwconv", lib.b2u_dwconv3x3, _ptr(F1), _ptr(F2), _ptr(w[pre + "dw"]), _ptr(w[pre + "dwb"]), B,
                     S16, S16, D // 4, 3, L.ACT_GELU, rt)
            if c16:
                self._gemm(plan, pre + "ffn2", F2, B * Lq, D // 4, D // 4, w[pre + "f2"], D, Cst, D, rt,
                           bias=w[pre + "f2b"], add16=Cst, ldadd=D)
            else:
                self._gemm(plan, pre + "ffn2", F2, B * Lq, D // 4, D // 4, w[pre + "f2"], D, Cst, D, rt, out_fp32=True,
                           bias=w[pre + "f2b"], residual=Cst, ldres=D)

        # ================= adapter tail (dinov3_adapter.py:460-482) =================
        C16 = buf("C16", (B * n2, D), tr)
        UP = buf("UP", (B * S4 * S4, D), tr)
        fs = [buf("f1", (B * S4 * S4, D), tr), buf("f2", (B * n2, D), tr), buf("f3", (B * n3, D), tr),
              buf("f4", (B * n4, D), tr)]
        if c16:
            plan.add("cast_c2", lib.b2u_copy_rows16, _ptr(Cst), _ptr(C16), B * n2, D, Lq, n2, 0)
        else:
            plan.add("cast_c2", lib.b2u_cast_rows, _ptr(Cst), _ptr(C16), B * n2, D, Lq, n2, 0, rt)
        self._gemm(plan, "up", C16, B * n2, D, D, w["up.w"], 4 * D, UP, D, rt, ps=(D, S8, S8), bias=w["up.b"], add16=c1,
                   ldadd=D)
        plan.add("tail1", lib.b2u_tail_fuse, _ptr(UP), 0, S4 * S4 * D, _ptr(taps[0]), _ptr(fs[0]), _ptr(w["bn1.sc"]),
                 _ptr(w["bn1.sh"]), B, S4, S4, h, h, D, rt)
        for i, (off, res) in enumerate(((0, S8), (n2, S16), (n2 + n3, S32))):
            plan.add(f"tail{i + 2}", lib.b2u_tail_fuse, Cst.data_ptr() + off * D * (2 if c16 else 4), 0 if c16 else 1, Lq * D,
                     _ptr(taps[i + 1]),
                     _ptr(fs[i + 1]), _ptr(w[f"bn{i + 2}.sc"]), _ptr(w[f"bn{i + 2}.sh"]), B, res, res, h, h, D, rt)

        # ================= FAPM + ups (dinounet_training.py:419-441, 255-264, 499-510) =================
        R = cfg.FAPM_RANK
        px0 = B * S4 * S4
        ZZ = buf("ZZ", (px0, 2 * R), tr)
        GB = buf("GB", (px0, 2 * R), tr)
        Z = buf("Z", (px0, R), tr)
        RS = buf("RS", (px0 * 64,), tr)   # [px, 2*oc]: px*2*oc is the same (<= px0*64) at every scale
        T1 = buf("T1", (px0 * 32,), tr)
        T2 = buf("T2", (px0 * 32,), tr)
        Yf = buf("Yf", (px0 * 32,), tr)
        U1 = buf("U1", (px0 * 4 * 32,), tr)
        n_stats = 3 * 4 + 6
        stats = buf("stats", (n_stats, B, 256, 2), torch.float32)
        gate = buf("gate", (B, 256), torch.float32)
        wfl = max(int(lib.b2u_in_stats_work_floats(B, (S4 >> i) ** 2, oc)) for i, oc in enumerate(self.features))
        wfl = max([wfl] + [int(lib.b2u_in_stats_work_floats(B, (S4 << s) ** 2, self.features[2 - s])) for s in range(3)])
        in_work = buf("in_work", (wfl,), torch.float32, zero=True)   # ticket counters start at zero
        feats = self.features
        cat = [buf("cat0", (B * S4 * S4, 2 * feats[2]), tr), buf("cat1", (B * S2 * S2, 2 * feats[1]), tr),
               buf("cat2", (B * S * S, 2 * feats[0]), tr)]
        skip3 = buf("skip3", (B * S8 * S8, feats[3]), tr)
        slot = 0

        def sums_slot():
            nonlocal slot
            t = stats[slot]
            slot += 1
            return t

        for i, oc in enumerate(feats):
            r = S4 >> i
            px = B * r * r
            pre = f"f{i}."
            has_sc = oc != R
            n3_ = 2 * oc if has_sc else oc
            self._gemm(plan, pre + "bases", fs[i], px, D, D, w[pre + "w1"], 2 * R, ZZ, 2 * R, rt, bias=w[pre + "b1"])
            self._gemm(plan, pre + "film_gen", ZZ, px, R, 2 * R, w[pre + "film"], 2 * R, GB, 2 * R, rt, bias=w[pre + "filmb"])
            plan.add(pre + "film", lib.b2u_film, _ptr(GB), _ptr(ZZ), 2 * R, R, _ptr(Z), px, R, rt)
            self._gemm(plan, pre + "reduce_sc", Z, px, R, R, w[pre + "w3"], n3_, RS, n3_, rt, bias=w[pre + "b3"])
            s_a, s_b, s_c = sums_slot(), sums_slot(), sums_slot()
            plan.add(pre + "in1.stats", lib.b2u_in_stats, _ptr(RS), n3_, _ptr(s_a), _ptr(in_work), B, r * r, oc, rt)
            plan.add(pre + "in1.apply", lib.b2u_in_apply, _ptr(RS), n3_, _ptr(T1), oc, _ptr(s_a), _ptr(w[pre + "in1w"]),
                     _ptr(w[pre + "in1b"]), B, r * r, oc, cfg.IN_EPS, rt)
            plan.add(pre + "dw", lib.b2u_dwconv3x3, _ptr(T1), _ptr(T2), _ptr(w[pre + "dw"]), _ptr(w[pre + "dwb"]), B, r, r, oc,
                     1, L.ACT_NONE, rt)
            self._gemm(plan, pre + "pw", T2, px, oc, oc, w[pre + "pw"], oc, T1, oc, rt, bias=w[pre + "pwb"])
            plan.add(pre + "in2.stats", lib.b2u_in_stats, _ptr(T1), oc, _ptr(s_b), _ptr(in_work), B, r * r, oc, rt)
            plan.add(pre + "in2.apply", lib.b2u_in_apply, _ptr(T1), oc, _ptr(T2), oc, _ptr(s_b), _ptr(w[pre + "in2w"]),
                     _ptr(w[pre + "in2b"]), B, r * r, oc, cfg.IN_EPS, rt)
            self._gemm(plan, pre + "refine", T2, px, oc, oc, w[pre + "ref"], oc, T1, oc, rt, bias=w[pre + "refb"])
            plan.add(pre + "se.pool", lib.b2u_in_stats, _ptr(T1), oc, _ptr(s_c), _ptr(in_work), B, r * r, oc, rt)
            plan.add(pre + "se.gate", lib.b2u_se_gate, _ptr(s_c), _ptr(w[pre + "se1"]), _ptr(w[pre + "se1b"]), _ptr(w[pre + "se2"]),
                     _ptr(w[pre + "se2b"]), _ptr(gate), B, oc, max(1, oc // 16), r * r)
            if has_sc:
                sc_ptr, ldsc = RS.data_ptr() + oc * 2, n3_
            else:
                sc_ptr, ldsc = Z.data_ptr(), R
            plan.add(pre + "se.apply", lib.b2u_se_apply, _ptr(T1), sc_ptr, ldsc, _ptr(gate), _ptr(Yf), B, r * r, oc, rt)
            # LearnableUpsampleBlock: the same ConvT twice (x4); the second writes straight into the decoder concat buffer
            self._gemm(plan, f"ups{i}.a", Yf, px, oc, oc, w[f"ups{i}.w"], 4 * oc, U1, oc, rt, ps=(oc, r, r), bias=w[f"ups{i}.b"])
            if i < 3:
                dst, ldc, coff = cat[2 - i], 2 * oc, oc
            else:
                dst, ldc, coff = skip3, oc, 0
            self._gemm(plan, f"ups{i}.b", U1, 4 * px, oc, oc, w[f"ups{i}.w"], 4 * oc, dst, ldc, rt, col_off=coff,
                       ps=(oc, 2 * r, 2 * r), bias=w[f"ups{i}.b"])

        # ================= decoder (dinounet_training.py:603-629) =================
        CO = buf("CO", (B * S * S * 32,), tr)
        CA = buf("CA", (B * S * S * 32,), tr)
        lres, below = skip3, feats[3]
        logits = buf("logits", (B, self.ncls, S, S), torch.float32)
        labels = buf("labels", (B, S, S), torch.uint8)
        for s in range(3):
            skip = feats[2 - s]
            r_lo = S8 << s
            r_hi = 2 * r_lo
            self._gemm(plan, f"d{s}.transp", lres, B * r_lo * r_lo, below, below, w[f"d{s}.t"], 4 * skip, cat[s], 2 * skip, rt,
                       ps=(skip, r_lo, r_lo), bias=w[f"d{s}.tb"])
            src, cin = cat[s], 2 * skip
            for j in range(2):
                self._gemm(plan, f"d{s}.conv{j}", src, 0, 9 * cin, cin, w[f"d{s}.c{j}"], skip, CO, skip, rt,
                           bias=w[f"d{s}.c{j}b"], conv=L.CONV3X3_S1, img=(B, r_hi, r_hi, cin))
                ss = sums_slot()
                plan.add(f"d{s}.in{j}.stats", lib.b2u_in_stats, _ptr(CO), skip, _ptr(ss), _ptr(in_work), B, r_hi * r_hi, skip, rt)
                if ds and s < 2 and j == 1:
                    # dinounet_training.py:619-626: seg_layers[s] on the stage output = the seg head on the pre-norm
                    # conv output and its statistics (16-bit activation, fp32 logits), no argmax
                    out = bufs[f"logits_ds{2 - s}"] = torch.empty((B, self.ncls, r_hi, r_hi), dtype=torch.float32, device=dev)
                    plan.add(f"d{s}.ds_head", lib.b2u_seg_head, _ptr(CO), _ptr(ss), _ptr(w[f"d{s}.n{j}w"]),
                             _ptr(w[f"d{s}.n{j}b"]), cfg.IN_EPS, _ptr(w[f"ds{s}.w"]), _ptr(w[f"ds{s}.b"]), _ptr(out), None,
                             B, r_hi * r_hi, skip, self.ncls, rt)
                if s == 2 and j == 1:
                    plan.add("seg_head", lib.b2u_seg_head, _ptr(CO), _ptr(ss), _ptr(w[f"d{s}.n{j}w"]), _ptr(w[f"d{s}.n{j}b"]),
                             cfg.IN_EPS, _ptr(w["seg.w"]), _ptr(w["seg.b"]), _ptr(logits), _ptr(labels), B, r_hi * r_hi, skip,
                             self.ncls, rt)
                else:
                    plan.add(f"d{s}.in{j}.apply", lib.b2u_in_apply, _ptr(CO), skip, _ptr(CA), skip, _ptr(ss),
                             _ptr(w[f"d{s}.n{j}w"]), _ptr(w[f"d{s}.n{j}b"]), B, r_hi * r_hi, skip, cfg.IN_EPS, rt)
                src, cin = CA, skip
            lres, below = CA, skip
        assert slot == n_stats
        return plan, bufs

    # ------------------------------------------------------------------ execution
    def get_plan(self, B: int, S: int) -> Tuple[Plan, dict]:
        key = (B, S)
        if key in self._plans:
            self._plans.move_to_end(key)
            return self._plans[key]
        while len(self._plans) >= max(1, self.max_plans):      # evict the least recently used buffer set + graph
            old, _ = self._plans.popitem(last=False)
            self._fold_plans.pop(old, None)
            for gk in [k for k in self._graphs if k[:2] == old]:
                self._graphs.pop(gk)
        with torch.cuda.device(self.device):                   # kernels, TMA maps and num_sms() use the current device
            if self.precision == "fp32":
                from .engine_fp32 import build_plan_fp32
                self._plans[key] = build_plan_fp32(self, B, S)
            else:
                self._plans[key] = self.build_plan(B, S)
        return self._plans[key]

    def ds_plan(self, B: int, S: int) -> Tuple[Plan, List[torch.Tensor]]:
        """The deep-supervision variant of the (B, S) plan (`build_plan(ds=True)` or the fp32 tier's), on the activation
        buffers of the (B, S) plan, built on first use and dropped with it: (plan, [logits@S, logits@S/2, logits@S/4]).
        The eval plan, its CUDA graphs and its launch list are untouched."""
        plan, bufs = self.get_plan(B, S)
        if plan.ds is None:
            if "ds0.w" not in self.w:
                raise KeyError("deep supervision needs decoder.seg_layers.0 / .1 in the packed state dict")
            with torch.cuda.device(self.device):
                if self.precision == "fp32":
                    from .engine_fp32 import build_plan_fp32
                    dp, dbufs = build_plan_fp32(self, B, S, share=bufs, ds=True)
                else:
                    dp, dbufs = self.build_plan(B, S, share=bufs, ds=True)
            plan.ds = (dp, [bufs["logits"], dbufs["logits_ds1"], dbufs["logits_ds2"]])
        return plan.ds

    def forward_ds(self, x: torch.Tensor) -> List[torch.Tensor]:
        """x: fp32 [B, 3, S, S] -> [logits@S, logits@S/2, logits@S/4] (fp32 NCHW, highest resolution first, as the
        reference's decoder returns them with deep supervision, dinounet_training.py:627-629).  logits@S is what `forward`
        computes.  The returned tensors are the engine's own buffers (overwritten by the next call)."""
        if x.device.type != "cuda":
            raise L.NativeLibraryError("dinounet_b200 runs on CUDA devices only (no CPU fallback)")
        B, Cc, S, S_ = x.shape
        if Cc != 3 or S != S_:
            raise ValueError("expected [B, 3, S, S]")
        if x.device != self.device:
            raise ValueError(f"input on {x.device}, engine on {self.device}")
        _, bufs = self.get_plan(B, S)
        dp, outs = self.ds_plan(B, S)
        bufs["x"].copy_(x, non_blocking=True)
        with torch.cuda.device(self.device):
            dp.run(torch.cuda.current_stream(self.device).cuda_stream)
        return outs

    def clear_plans(self):
        """Frees every cached (batch, size) buffer set and CUDA graph."""
        self._plans.clear()
        self._graphs.clear()
        self._fold_plans.clear()

    # ------------------------------------------------------------------ fold ensembles on one backbone
    def pack_folds(self, fold_params: Iterable[Dict[str, torch.Tensor]]):
        """Packs the weights after the taps of every fold (reference-keyed state dicts whose backbone is the one this
        engine was packed with: the backbone is frozen in training, so every fold of a run has it bit for bit).  The
        ViT section stays packed once; each fold adds only its trainable weights, and its "rest" launch list runs on the
        activation, tap and input buffers of the shared (B, S) plan."""
        with torch.cuda.device(self.device):
            folds = [self._pack_rest(P) for P in fold_params]
        self._folds = folds
        self._fold_plans.clear()
        for gk in [k for k in self._graphs if len(k) == 4 and k[2] == "fold"]:
            self._graphs.pop(gk)

    @property
    def num_folds(self) -> int:
        return len(self._folds)

    def fold_bytes(self) -> List[int]:
        """Device bytes of each fold's packed weights."""
        return [sum(t.numel() * t.element_size() for t in f.values() if t.is_cuda) for f in self._folds]

    def _fold_plan(self, B: int, S: int, f: int) -> Plan:
        _, bufs = self.get_plan(B, S)
        plans = self._fold_plans.setdefault((B, S), [None] * len(self._folds))
        if plans[f] is None:
            w = dict(self.w)
            w.update(self._folds[f])
            with torch.cuda.device(self.device):
                if self.precision == "fp32":
                    from .engine_fp32 import build_plan_fp32
                    plans[f], _ = build_plan_fp32(self, B, S, w=w, share=bufs)
                else:
                    plans[f], _ = self.build_plan(B, S, w=w, share=bufs)
        return plans[f]

    def run_fold_rest(self, B: int, S: int, f: int, use_graph: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
        """`run_resident(B, S, part="rest")` on fold f's weights (`pack_folds`): SPM .. seg head on whatever the shared
        plan's input and tap buffers hold, into its logits / labels buffers (overwritten by the next fold)."""
        if not 0 <= f < len(self._folds):
            raise IndexError(f"fold {f} of {len(self._folds)} packed fold weight sets")
        plan = self._fold_plan(B, S, f)
        _, bufs = self.get_plan(B, S)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device).cuda_stream
            if use_graph:
                key = (B, S, "fold", f)
                g = self._graphs.get(key)
                if g is None:
                    g = self._graphs[key] = self._capture(plan, stream, plan.vit_end, None)
                g.replay()
            else:
                plan.run(stream, plan.vit_end)
        return bufs["logits"], bufs["labels"]

    def forward(self, x: torch.Tensor, use_graph: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
        """x: fp32 [B, 3, S, S] on the engine's device -> (logits fp32 [B, ncls, S, S], labels uint8 [B, S, S]).
        The returned tensors are the engine's own output buffers (overwritten by the next call)."""
        if x.device.type != "cuda":
            raise L.NativeLibraryError("dinounet_b200 runs on CUDA devices only (no CPU fallback)")
        B, Cc, S, S_ = x.shape
        if Cc != 3 or S != S_:
            raise ValueError("expected [B, 3, S, S]")
        if x.device != self.device:
            raise ValueError(f"input on {x.device}, engine on {self.device}")
        plan, bufs = self.get_plan(B, S)
        bufs["x"].copy_(x, non_blocking=True)
        return self.run_resident(B, S, use_graph)

    def _capture(self, plan: Plan, stream: int, lo: int, hi: Optional[int]):
        """calls[lo:hi] of `plan` as a CUDA graph, with no other thread's device work in flight (`GRAPH_CAPTURE`)."""
        with GRAPH_CAPTURE.capture():
            plan.run(stream, lo, hi)  # warm-up (cudaFuncSetAttribute etc. must happen outside capture)
            torch.cuda.synchronize(self.device)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                plan.run(torch.cuda.current_stream(self.device).cuda_stream, lo, hi)
        return g

    def run_resident(self, B: int, S: int, use_graph: bool = False, part: str = "all") -> Tuple[torch.Tensor, torch.Tensor]:
        """Runs the (B, S) plan on whatever `get_plan(B, S)[1]["x"]` holds (a producer kernel, e.g. the sliding-window
        tile gather, wrote the batch there on the current stream).  part: "all", "vit" (patch embed .. ViT taps only) or
        "rest" (everything after the taps: SPM, extractors, FAPM, decoder - on whatever the tap buffers hold)."""
        plan, bufs = self.get_plan(B, S)
        lo, hi = {"all": (0, None), "vit": (0, plan.vit_end), "rest": (plan.vit_end, None)}[part]
        with torch.cuda.device(self.device):     # the model may live on a device that is not the process's current one
            stream = torch.cuda.current_stream(self.device).cuda_stream
            if use_graph:
                key = (B, S, part)
                g = self._graphs.get(key)
                if g is None:
                    g = self._graphs[key] = self._capture(plan, stream, lo, hi)
                g.replay()
            else:
                plan.run(stream, lo, hi)
        return bufs["logits"], bufs["labels"]

    # ------------------------------------------------------------------ frozen-ViT feature caching (SURVEY.md 8f rank 3)
    def scaled_vit_plan(self, B: int, S: int) -> Tuple[Plan, torch.Tensor]:
        """The ViT section of the (B, S) plan on per-block RoPE tables (the reference's train-mode coordinate rescaling,
        rope_position_encoding.py:93-97, drawn once per block, vision_transformer.py:271-272): one b2u_rope_tables launch
        fills [depth, P, head_dim] sin / cos from the returned `scales` buffer [depth], then the plan's own ViT calls run with
        each block's RoPE pointers moved to its slice.  Shares every activation buffer of the (B, S) plan; the eval launch
        list and its CUDA graphs are untouched."""
        plan, _ = self.get_plan(B, S)
        if plan.scaled_vit is None:
            h, depth, hd = S // 16, self.v.depth, self.hd
            dev = self.device
            scales = torch.ones(depth, dtype=torch.float32, device=dev)
            periods = self._dev(self.w["periods"])
            sin = torch.empty((depth, h * h, hd), dtype=torch.float32, device=dev)
            cos = torch.empty_like(sin)
            sp = Plan()
            sp.keep += [scales, periods, sin, cos]
            sp.add("rope_tables", self.lib.b2u_rope_tables, _ptr(periods), _ptr(scales), _ptr(sin), _ptr(cos), depth, h, h, hd)
            sites = {idx: (blk, patch) for idx, blk, patch in plan.rope_sites}
            for idx, (name, fn, args) in enumerate(plan.calls[:plan.vit_end]):
                if idx in sites:
                    blk, patch = sites[idx]
                    args = patch(args, sin[blk].data_ptr(), cos[blk].data_ptr(), sp.keep)
                sp.calls.append((name, fn, args))
            assert len(sites) == depth
            plan.scaled_vit = (sp, scales)
        return plan.scaled_vit

    def extract_vit_features(self, x: torch.Tensor, use_graph: bool = False,
                             rope_scales: Optional[torch.Tensor] = None) -> List[torch.Tensor]:
        """The four tapped, final-LayerNorm'ed ViT outputs [B, P, D] (fp32) of the FROZEN backbone
        (dinov3_adapter.py:422-426: `with torch.no_grad()` around get_intermediate_layers).  In eval mode they depend only
        on the image, so a caller that sees a sample repeatedly (every training epoch, every mirrored / overlapping
        sliding-window pass over the same tile) may cache them and skip 57-88 % of the forward FLOPs with
        `forward_from_vit_features`.  rope_scales [depth] (fp32): block i's RoPE coordinates are multiplied by
        rope_scales[i] (the reference's train mode; runs `scaled_vit_plan`, without a CUDA graph).  Returns fresh tensors
        (not the engine's buffers)."""
        B, _, S, _ = x.shape
        plan, bufs = self.get_plan(B, S)
        bufs["x"].copy_(x, non_blocking=True)
        if rope_scales is None:
            self.run_resident(B, S, use_graph, part="vit")
        else:
            if tuple(rope_scales.shape) != (self.v.depth,):
                raise ValueError(f"rope_scales must have shape [{self.v.depth}], got {tuple(rope_scales.shape)}")
            sp, scales = self.scaled_vit_plan(B, S)
            scales.copy_(rope_scales, non_blocking=True)
            with torch.cuda.device(self.device):
                sp.run(torch.cuda.current_stream(self.device).cuda_stream)
        P = (S // 16) ** 2
        return [bufs[f"tap{k}"].view(B, P, -1).clone() for k in range(4)]

    def forward_from_vit_features(self, x: torch.Tensor, feats: List[torch.Tensor], use_graph: bool = False):
        """Everything after the backbone (SPM needs the image, the extractors need the cached taps)."""
        B, _, S, _ = x.shape
        plan, bufs = self.get_plan(B, S)
        bufs["x"].copy_(x, non_blocking=True)
        for k in range(4):
            bufs[f"tap{k}"].view(feats[k].shape).copy_(feats[k], non_blocking=True)
        return self.run_resident(B, S, use_graph, part="rest")
