"""Device export without a GPU: the torch-float64 restatement of the reference's resampling against scipy and the golden
data (tests/golden/export_cases.npz, oracle/make_golden_export.py), the label and probability steps against the
reference's own `LabelManager`, the host paste / transpose / probability crop-revert, the rejections (before any
launch) and which C-ABI calls the export makes with which arguments (recording stand-in for the native library)."""
import contextlib
import os
import pickle
import sys
import types
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dinounet_b200 import export as EX
from oracle import export_oracle as EO

REF = np.load(os.path.join(os.path.dirname(__file__), "golden", "export_cases.npz"))
CASES = {c[0]: c for c in EO.GOLDEN_CASES}


def _bits(a):
    return np.asarray(a).view(np.uint16)


@pytest.mark.parametrize("name", list(CASES))
def test_restatement_reproduces_golden(name):
    _, C, regions, order, shape, target, _, _, tb, save = CASES[name]
    logits = torch.from_numpy(REF[f"{name}_logits"])
    r, seg, probs = EO.convert(logits, EO.golden_properties(CASES[name]), tb, 3 if regions else C - 1, regions, order, save)
    assert np.array_equal(_bits(r.numpy()), _bits(REF[f"{name}_resampled"]))
    assert seg.dtype == REF[f"{name}_seg"].dtype and np.array_equal(seg, REF[f"{name}_seg"])
    if save:
        assert probs.dtype == np.float32 and np.array_equal(probs, REF[f"{name}_probs"])
    else:
        assert probs is None and f"{name}_probs" not in REF.files


@pytest.mark.parametrize("h,w,H,W", [(37, 53, 300, 700), (512, 512, 300, 700), (512, 512, 384, 384), (1, 5, 3, 9),
                                     (2, 3, 7, 1), (300, 700, 512, 512), (13, 1, 4, 1), (64, 80, 64, 41), (9, 9, 9, 10)])
def test_torch_restatement_equals_scipy_in_float64(h, w, H, W):
    """scipy's order-1 zoom (NI_ZoomShift) bit for bit in float64, per-volume (Z unchanged) as the reference calls it."""
    import scipy.ndimage as ndi
    x = (torch.randn(2, 3, h, w, generator=torch.Generator().manual_seed(h * 1000 + W)) * 4).half()
    data = x.numpy().astype(float)
    want = np.stack([ndi.zoom(data[c], (1, H / h, W / w), order=1, mode="nearest", grid_mode=True) for c in range(2)])
    got = EO.resample_torch64(x, H, W).numpy()
    assert want.shape == got.shape and np.array_equal(want, got)
    # ... and per slice (separate-z with the low-resolution axis 0) gives the same bits
    per_slice = np.stack([np.stack([ndi.zoom(data[c, z], (H / h, W / w), order=1, mode="nearest", grid_mode=True)
                                    for z in range(3)]) for c in range(2)])
    assert np.array_equal(per_slice, want)
    assert np.array_equal(_bits(EO.to_f16(torch.from_numpy(want)).numpy()), _bits(want.astype(np.float16)))


# ---- the reference's LabelManager


def _reference_label_manager_class():
    from oracle import ref_loader
    if not ref_loader.reference_available():
        pytest.skip("reference sources not present")
    ref_loader.load_reference_module()
    # label_handling.py imports two third-party helpers that are not installed here; stand-ins with their semantics
    if "acvl_utils" not in sys.modules:
        for name in ("acvl_utils", "acvl_utils.cropping_and_padding"):
            sys.modules[name] = types.ModuleType(name)
        bb = types.ModuleType("acvl_utils.cropping_and_padding.bounding_boxes")
        bb.bounding_box_to_slice = lambda bbox: tuple(slice(*i) for i in bbox)
        sys.modules[bb.__name__] = bb
    if "batchgenerators" not in sys.modules:
        for name in ("batchgenerators", "batchgenerators.utilities"):
            sys.modules[name] = types.ModuleType(name)
        fo = types.ModuleType("batchgenerators.utilities.file_and_folder_operations")
        fo.join = os.path.join
        sys.modules[fo.__name__] = fo
    import importlib
    return importlib.import_module("dinounet.utilities.label_handling.label_handling").LabelManager


def _label_dict(C, regions):
    if regions:   # overlapping regions, as in BraTS-style datasets
        return {"background": 0, "whole": [1, 2, 3], "core": [2, 3], "enh": [3]}
    return {"background": 0, **{f"c{i}": i for i in range(1, C)}}


@pytest.mark.parametrize("name", list(CASES))
def test_segment_and_revert_equal_reference_label_manager(name):
    LabelManager = _reference_label_manager_class()
    _, C, regions, order, _, _, _, _, tb, _ = CASES[name]
    lm = LabelManager(_label_dict(C, regions), list(order) if regions else None)
    assert lm.num_segmentation_heads == C and lm.has_regions == regions
    r = torch.from_numpy(REF[f"{name}_resampled"])
    probs, seg = EO.nonlin_and_segment(r, regions, order)
    want_p = lm.apply_inference_nonlin(r)
    want_s = lm.convert_probabilities_to_segmentation(want_p)
    assert torch.equal(probs, want_p) and torch.equal(seg, want_s) and seg.dtype == want_s.dtype
    props = EO.golden_properties(CASES[name])
    want_rev = lm.revert_cropping_on_probabilities(want_p, props["bbox_used_for_cropping"], props["shape_before_cropping"])
    want_rev = want_rev.numpy().transpose([0] + [i + 1 for i in tb])
    assert np.array_equal(EX.probabilities_to_original_geometry(probs.numpy(), props, tb, regions), want_rev)
    n_fg = len(lm.foreground_labels)
    _, oracle_p = EO.revert_geometry(seg.numpy(), probs.numpy(), props, tb, n_fg, regions)
    assert np.array_equal(oracle_p, want_rev)


def test_host_paste_and_transpose():
    """export_prediction.py:43-52: uint8 below 255 foreground labels, uint16 from 255, zeros outside the box."""
    props = EO.golden_properties(CASES["reg3_mixed"])
    seg = np.random.default_rng(0).integers(0, 4, size=(2, 39, 71)).astype(np.uint8)
    out = EX.labels_to_original_geometry(seg, props, (2, 1, 0), 3)
    want, _ = EO.revert_geometry(seg, None, props, (2, 1, 0), 3, True)
    assert out.dtype == np.uint8 and out.shape == (80, 39, 5) and np.array_equal(out, want)
    assert EX.labels_to_original_geometry(seg.astype(np.uint16) + 300, props, (2, 1, 0), 300).dtype == np.uint16
    p = np.random.default_rng(1).random((3, 2, 39, 71), dtype=np.float32)
    for regions in (False, True):
        got = EX.probabilities_to_original_geometry(p, props, (2, 1, 0), regions)
        assert got.shape == (3, 80, 39, 5)
        assert np.array_equal(got, EO.revert_geometry(seg, p, props, (2, 1, 0), 3, regions)[1])
        outside = np.ones(props["shape_before_cropping"], bool)
        outside[1:3, 0:39, 4:75] = False
        assert (got[0][outside.transpose(2, 1, 0)] == (0.0 if regions else 1.0)).all()


# ---- argument contract and call sequence (recording stand-in for the native library)


class _Recorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*a):
            self.calls.append((name, a))
            return 0
        return fn


@pytest.fixture
def rec(monkeypatch):
    from dinounet_b200 import lib as L
    r = _Recorder()
    monkeypatch.setattr(L, "load", lambda: r)
    # CPU tensors stand in for device buffers: the stand-in library never reads them
    monkeypatch.setattr(EX, "_to_device", lambda t: t.contiguous())
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda dev=None: SimpleNamespace(cuda_stream=0))
    return r


def _managers(C=3, regions=False, order=(1, 2, 3), n_fg=None, spacing=(1.0, 1.0), fn=EX.DEFAULT_RESAMPLING_FN,
              kwargs=None, tb=(0, 1, 2)):
    conf = {"resampling_fn_probabilities": fn,
            "resampling_fn_probabilities_kwargs": dict(EX.DEFAULT_RESAMPLING_KWARGS if kwargs is None else kwargs)}
    cm = SimpleNamespace(spacing=list(spacing), configuration=conf)
    n_fg = (C if regions else C - 1) if n_fg is None else n_fg
    lm = SimpleNamespace(has_regions=regions, regions_class_order=list(order) if regions else None,
                         foreground_labels=list(range(1, n_fg + 1)), num_segmentation_heads=C)
    pm = SimpleNamespace(transpose_backward=list(tb), get_label_manager=lambda dj: lm)
    return pm, cm, lm


def _props(target, before=None, bbox=None, spacing=(1.0, 1.0, 1.0)):
    before = list(target) if before is None else list(before)
    bbox = [[0, s] for s in target] if bbox is None else bbox
    return {"shape_after_cropping_and_before_resampling": list(target), "shape_before_cropping": before,
            "bbox_used_for_cropping": bbox, "spacing": list(spacing)}


def _convert(logits, props, managers, probs=False):
    pm, cm, lm = managers
    return EX.convert_predicted_logits_to_segmentation_with_correct_shape(logits, pm, cm, lm, props, probs)


def test_call_sequence_label_maps(rec):
    """Resample (fp16 [C, Z, h, w] -> [C, Z, H, W]) then segment in mode 0 with uint8 labels; the logits may be a strided
    view; probabilities only when asked."""
    logits = torch.zeros(3, 2, 40, 50, dtype=torch.half)[:, :, 5:35, 3:48]
    seg = _convert(logits, _props((2, 20, 64)), _managers(3))
    assert seg.dtype == np.uint8 and seg.shape == (2, 20, 64)
    (n1, a1), (n2, a2) = rec.calls
    assert n1 == "b2u_export_resample_f16" and a1[2:8] == (3, 2, 30, 45, 20, 64) and a1[1] == a2[0]
    assert n2 == "b2u_export_segment" and a2[1:4] == (3, 2 * 20 * 64, 0) and a2[4] is None and a2[6] == 1
    assert a2[7] is None
    rec.calls.clear()
    seg, p = _convert(logits, _props((2, 20, 64)), _managers(3), probs=True)
    assert p.dtype == np.float32 and p.shape == (3, 2, 20, 64) and rec.calls[1][1][7] is not None


def test_call_sequence_identity_and_regions(rec):
    """Equal shapes skip the resampling (the reference returns the array unchanged); regions run mode 1 with the
    regions_class_order; >= 255 foreground labels give uint16."""
    logits = np.zeros((2, 3, 16, 16), dtype=np.float16)
    seg = _convert(logits, _props((3, 16, 16), before=(4, 20, 16), bbox=[[1, 4], [2, 18], [0, 16]], spacing=(5, 1, 1)),
                   _managers(2, regions=True, order=(7, 3), tb=(2, 0, 1)))
    assert [n for n, _ in rec.calls] == ["b2u_export_segment"]
    a = rec.calls[0][1]
    assert a[1:4] == (2, 3 * 16 * 16, 1) and a[4] is not None and a[6] == 1
    assert seg.shape == (16, 4, 20) and seg.dtype == np.uint8
    rec.calls.clear()
    seg = _convert(logits, _props((3, 16, 16)), _managers(2, regions=True, order=(300, 301), n_fg=300))
    assert rec.calls[0][1][6] == 2 and seg.dtype == np.uint16


def test_rejections_before_any_launch(rec):
    logits = torch.zeros(3, 2, 30, 40, dtype=torch.half)
    cases = [
        (_props((2, 20, 20)), _managers(fn="resample_data_or_seg_to_spacing"), NotImplementedError),
        (_props((2, 20, 20)), _managers(kwargs={**EX.DEFAULT_RESAMPLING_KWARGS, "order": 3}), NotImplementedError),
        (_props((2, 20, 20)), _managers(kwargs={**EX.DEFAULT_RESAMPLING_KWARGS, "force_separate_z": True}),
         NotImplementedError),
        (_props((3, 20, 20)), _managers(), NotImplementedError),                                    # Z changes
        # low-resolution axis 1 (in-plane, spacing 4 vs 1) whose size changes: order 0 along it in the reference
        (_props((2, 20, 40), spacing=(1.0, 1.0, 1.0)), _managers(spacing=(4.0, 1.0)), NotImplementedError),
        (_props((2, 30, 20), spacing=(1.0, 1.0, 4.0)), _managers(spacing=(1.0, 1.0)), NotImplementedError),
        (_props((2, 20, 20)), _managers(C=4), AssertionError),                                      # heads != channels
    ]
    for props, mgr, exc in cases:
        with pytest.raises(exc):
            _convert(logits, props, mgr)
    with pytest.raises(NotImplementedError):
        _convert(logits.float(), _props((2, 20, 20)), _managers())
    with pytest.raises(NotImplementedError):
        _convert(torch.zeros(33, 1, 4, 4, dtype=torch.half), _props((1, 4, 4)), _managers(33))
    assert rec.calls == []
    # the same in-plane low-resolution axis is fine while its size stays; z as the low-resolution axis is fine too
    _convert(logits, _props((2, 30, 20)), _managers(spacing=(4.0, 1.0)))
    _convert(logits, _props((2, 20, 20), spacing=(5.0, 1.0, 1.0)), _managers(spacing=(1.0, 1.0)))
    assert [n for n, _ in rec.calls] == ["b2u_export_resample_f16", "b2u_export_segment"] * 2


def test_export_prediction_from_logits_writes_reference_files(rec, tmp_path):
    """export_prediction.py:70-104: the writer gets the segmentation; .npz (key `probabilities`) and .pkl only with
    save_probabilities; a dataset.json path is read."""
    written = []

    class RW:
        def write_seg(self, seg, fname, props):
            written.append((seg, fname, props))

    pm, cm, lm = _managers(2)
    pm.image_reader_writer_class = RW
    props = _props((1, 8, 8))
    logits = torch.zeros(2, 1, 8, 8, dtype=torch.half)
    out = str(tmp_path / "case_0")
    EX.export_prediction_from_logits(logits, props, cm, pm, {"file_ending": ".nii.gz"}, out, False)
    assert written[-1][1] == out + ".nii.gz" and written[-1][2] is props and written[-1][0].shape == (1, 8, 8)
    assert not os.path.exists(out + ".npz") and not os.path.exists(out + ".pkl")
    dj = tmp_path / "dataset.json"
    dj.write_text('{"file_ending": ".png"}')
    EX.export_prediction_from_logits(logits, props, cm, pm, str(dj), out, True)
    assert written[-1][1] == out + ".png"
    assert np.load(out + ".npz")["probabilities"].shape == (2, 1, 8, 8)
    with open(out + ".pkl", "rb") as f:
        assert pickle.load(f) == props
