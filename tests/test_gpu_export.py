"""-m gpu: the export kernels against the oracle restatement of the reference's export chain (oracle/export_oracle.py,
pinned to scipy and to the reference's LabelManager in tests/test_export_cpu.py).

* b2u_export_resample_f16 is bit-identical to the golden data and to the torch-float64 restatement of scipy's zoom.
* b2u_export_segment: probabilities within PROB_ULP ulp of torch's CPU softmax / sigmoid, and labels identical except
  where the oracle's top-two probabilities are that close (counted and bounded); region labels identical, the threshold
  exhaustively over all 65,536 fp16 values.
* SlidingWindowPredictor -> export_prediction_from_logits writes the oracle route's label volume."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dinounet_b200 import export as EX
from dinounet_b200 import lib as L
from oracle import export_oracle as EO
from tests.gpu_helpers import stream

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
REF = np.load(os.path.join(os.path.dirname(__file__), "golden", "export_cases.npz"))
# torch's CPU softmax (vectorised expf, then the sum and the division) is itself up to 4 ulp from an fp32 restatement
# with correctly rounded exp at 8-32 channels, and the kernel uses CUDA's expf: 8 ulp covers both.
PROB_ULP = 8


def _bits(t):
    return t.detach().cpu().contiguous().view(torch.int16)


def _resample(x, H, W):
    C, Z, h, w = x.shape
    out = torch.empty((C, Z, H, W), dtype=torch.half, device=DEV)
    L.check(L.load().b2u_export_resample_f16(x.data_ptr(), out.data_ptr(), C, Z, h, w, H, W, stream()), "resample")
    return out


def _segment(x, mode, region_labels=None, label_bytes=1, want_probs=True):
    C = x.shape[0]
    vox = x[0].numel()
    labels = torch.empty(vox, dtype=torch.uint8 if label_bytes == 1 else torch.int16, device=DEV)
    probs = torch.empty((C, vox), dtype=torch.float32, device=DEV) if want_probs else None
    rl = None if region_labels is None else torch.tensor(region_labels, dtype=torch.int32, device=DEV)
    L.check(L.load().b2u_export_segment(x.data_ptr(), C, vox, mode, None if rl is None else rl.data_ptr(),
                                        labels.data_ptr(), label_bytes, None if probs is None else probs.data_ptr(),
                                        stream()), "segment")
    torch.cuda.synchronize()
    lab = labels.cpu()
    if label_bytes == 2:
        lab = torch.from_numpy(lab.numpy().view(np.uint16).astype(np.int32))
    return lab.long(), (probs.cpu() if probs is not None else None)


@pytest.mark.parametrize("case", EO.GOLDEN_CASES, ids=[c[0] for c in EO.GOLDEN_CASES])
def test_resample_bit_identical_to_golden(case):
    name, target = case[0], case[5]
    x = torch.from_numpy(REF[f"{name}_logits"]).to(DEV)
    got = _resample(x, target[1], target[2])
    want = torch.from_numpy(REF[f"{name}_resampled"])
    assert torch.equal(_bits(got), _bits(want))
    assert torch.equal(_bits(got), _bits(EO.resample_f16(x.cpu(), target[1], target[2])))


SWEEP = [  # C, Z, h, w, H, W: odd sizes, factors < 1 and > 1 per axis, 1 to 32 channels
    (1, 1, 7, 13, 29, 5), (2, 3, 1, 9, 5, 1), (3, 4, 512, 512, 300, 700), (5, 2, 101, 257, 384, 200),
    (17, 1, 64, 64, 63, 65), (32, 2, 33, 31, 97, 17), (4, 2, 512, 512, 768, 768), (9, 1, 300, 700, 512, 512),
]


@pytest.mark.parametrize("C,Z,h,w,H,W", SWEEP)
def test_resample_sweep_bit_identical_to_restatement(C, Z, h, w, H, W):
    g = torch.Generator().manual_seed(C * 7 + h)
    x = (torch.randn(C, Z, h, w, generator=g) * 6).half()
    got = _resample(x.to(DEV), H, W)
    assert torch.equal(_bits(got), _bits(EO.resample_f16(x, H, W)))


def test_identity_shape_returns_input():
    x = (torch.randn(3, 2, 17, 23, generator=torch.Generator().manual_seed(5)) * 5).half()
    x[0, 0, 0, :4] = torch.tensor([-0.0, 0.0, float("nan"), float("-inf")]).half()
    xd = x.to(DEV)
    assert torch.equal(_bits(_resample(xd, 17, 23)), _bits(x))
    L.check(L.load().b2u_export_resample_f16(xd.data_ptr(), xd.data_ptr(), 3, 2, 17, 23, 17, 23, stream()))
    assert torch.equal(_bits(xd), _bits(x))


def _ulp_dist(a, b):
    return (a.contiguous().view(torch.int32).long() - b.contiguous().view(torch.int32).long()).abs()


@pytest.mark.parametrize("C", [1, 2, 3, 4, 8, 17, 32])
def test_segment_label_maps_against_oracle(C):
    g = torch.Generator().manual_seed(100 + C)
    x = (torch.randn(C, 3, 67, 131, generator=g) * 4).half()
    x[:, 0, 0, :8] = x[0, 0, 0, :8].clone()  # exact ties: the first maximum wins
    lab, probs = _segment(x.to(DEV), 0)
    want_p, want_s = EO.nonlin_and_segment(x, False)
    want_p, want_s = want_p.reshape(C, -1), want_s.reshape(-1)
    assert int(_ulp_dist(probs, want_p).max()) <= PROB_ULP
    if C > 1:
        top2 = want_p.topk(2, dim=0).values
        near_tie = _ulp_dist(top2[0], top2[1]) <= PROB_ULP
    else:
        near_tie = torch.zeros_like(want_s, dtype=torch.bool)
    diff = lab != want_s
    n = int(diff.sum())
    print(f"C={C}: {n} of {lab.numel()} labels differ, all at near-ties ({int(near_tie.sum())} near-ties)")
    assert not (diff & ~near_tie).any() and n <= max(8, lab.numel() // 10000)
    assert (lab[:8] == 0).all()
    lab2, none = _segment(x.to(DEV), 0, want_probs=False)
    assert none is None and torch.equal(lab2, lab)


@pytest.mark.parametrize("C", [1, 3, 7, 32])
def test_segment_regions_against_oracle(C):
    g = torch.Generator().manual_seed(200 + C)
    x = (torch.randn(C, 2, 45, 77, generator=g) * 3).half()
    order = [int(v) for v in torch.randperm(C, generator=g) + 1]
    lab, probs = _segment(x.to(DEV), 1, order)
    want_p, want_s = EO.nonlin_and_segment(x, True, order)
    assert torch.equal(lab, want_s.reshape(-1).long())
    assert int(_ulp_dist(probs, want_p.reshape(C, -1)).max()) <= PROB_ULP
    # uint16 labels (>= 255 foreground labels): the reference's int16 painting read back as uint16
    big = [300 + v for v in order]
    lab16, _ = _segment(x.to(DEV), 1, big, label_bytes=2, want_probs=False)
    _, want16 = EO.nonlin_and_segment(x, True, big)
    assert torch.equal(lab16, want16.reshape(-1).long())


def test_region_threshold_exhaustive_over_fp16():
    """Every fp16 bit pattern: kernel foreground == torch.sigmoid(x.float()) > 0.5 on the CPU (tiny positive logits
    such as 2^-24 are NOT foreground in fp32)."""
    x = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.float16).reshape(1, -1)
    lab, probs = _segment(x.to(DEV), 1, [1])
    want = (torch.sigmoid(x.float()) > 0.5).reshape(-1)
    assert torch.equal(lab.bool(), want)
    tiny = torch.tensor([2.0 ** -24], dtype=torch.half).view(torch.int16)
    assert not bool(lab[int(tiny) + 32768])
    finite = torch.isfinite(x.float().reshape(-1))
    assert int(_ulp_dist(probs[0][finite], torch.sigmoid(x.float()).reshape(-1)[finite]).max()) <= PROB_ULP


def test_repeat_launches_identical():
    x = (torch.randn(4, 3, 200, 180, generator=torch.Generator().manual_seed(9)) * 5).half().to(DEV)
    r1, r2 = _resample(x, 317, 263), _resample(x, 317, 263)
    assert torch.equal(_bits(r1), _bits(r2))
    (l1, p1), (l2, p2) = _segment(r1, 0), _segment(r1, 0)
    assert torch.equal(l1, l2) and torch.equal(p1.view(torch.int32), p2.view(torch.int32))
    (l1, p1), (l2, p2) = _segment(r1, 1, [3, 1, 2, 4]), _segment(r1, 1, [3, 1, 2, 4])
    assert torch.equal(l1, l2) and torch.equal(p1.view(torch.int32), p2.view(torch.int32))


class _RecordingWriter:
    written = []

    def write_seg(self, seg, fname, props):
        _RecordingWriter.written.append((seg.copy(), fname, props))


def test_predictor_to_export_end_to_end(tmp_path):
    """SlidingWindowPredictor's fp16 logits (a strided view after un-padding) -> export_prediction_from_logits, for a
    label-map and a region dataset: the written label volume equals the oracle route's."""
    import dinounet_b200
    from dinounet_b200 import config
    from dinounet_b200.sliding_window import SlidingWindowPredictor
    from oracle import dinounet_oracle as O
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, 3, None,
                                             "dinounet_s")
    net.load_state_dict(O.make_state_dict("dinounet_s", 3, seed=0), strict=True)
    net = net.to(DEV).eval()
    p = SlidingWindowPredictor(tile_step_size=0.5, use_gaussian=True, use_mirroring=True, device=DEV, tile_batch=4)
    p.manual_initialization(net, None, SimpleNamespace(patch_size=[128, 128]), None, {}, "DinoUNetTrainer_s", (0, 1))
    x = torch.randn(3, 2, 100, 170, generator=torch.Generator().manual_seed(11))
    logits = p.predict_sliding_window_return_logits(x)
    assert logits.shape == (3, 2, 100, 170) and not logits.is_contiguous()
    props = {"shape_after_cropping_and_before_resampling": [2, 131, 97], "shape_before_cropping": [3, 140, 110],
             "bbox_used_for_cropping": [[1, 3], [4, 135], [6, 103]], "spacing": [3.0, 0.7, 0.9]}
    conf = {"resampling_fn_probabilities": EX.DEFAULT_RESAMPLING_FN,
            "resampling_fn_probabilities_kwargs": dict(EX.DEFAULT_RESAMPLING_KWARGS)}
    cm = SimpleNamespace(spacing=[0.53, 0.53], configuration=conf)
    for regions, order in ((False, None), (True, [2, 1, 3])):
        lm = SimpleNamespace(has_regions=regions, regions_class_order=order, foreground_labels=[1, 2, 3] if regions else [1, 2],
                             num_segmentation_heads=3)
        pm = SimpleNamespace(transpose_backward=[0, 2, 1], get_label_manager=lambda dj: lm,
                             image_reader_writer_class=_RecordingWriter)
        out = str(tmp_path / f"case_{int(regions)}")
        EX.export_prediction_from_logits(logits, props, cm, pm, {"file_ending": ".nii.gz"}, out, save_probabilities=True)
        seg, fname, _ = _RecordingWriter.written[-1]
        _, want, want_p = EO.convert(logits.cpu(), props, [0, 2, 1], len(lm.foreground_labels), regions, order, True)
        assert fname == out + ".nii.gz" and seg.dtype == want.dtype and seg.shape == (3, 110, 140)
        if regions:
            assert np.array_equal(seg, want)
        else:
            top2 = np.sort(want_p, axis=0)[-2:]
            near_tie = np.abs(top2[1].view(np.int32).astype(np.int64) - top2[0].view(np.int32)) <= PROB_ULP
            diff = seg != want
            print(f"label maps end to end: {int(diff.sum())} of {seg.size} labels differ at near-ties")
            assert not (diff & ~near_tie).any()
        got_p = np.load(out + ".npz")["probabilities"]
        assert got_p.shape == want_p.shape
        assert np.abs(got_p.view(np.int32).astype(np.int64) - want_p.view(np.int32)).max() <= PROB_ULP
