"""Device preprocessing without a GPU: the restatements of oracle/preprocess_oracle.py against scipy's order-3 zoom and
numpy's float32 reductions over shape and layout sweeps, the whole restated case against the reference's own
`run_case_npy` (tests/golden/preprocess_cases.npz, oracle/make_golden_preprocess.py), the `properties` keys, the
rejections (before any launch) and the C-ABI call sequence (recording stand-in for the native library)."""
import contextlib
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dinounet_b200 import preprocess as PP
from oracle import make_golden_preprocess as MG
from oracle import preprocess_oracle as PO

REF = np.load(os.path.join(os.path.dirname(__file__), "golden", "preprocess_cases.npz"))


@pytest.mark.parametrize("h,w,H,W", [(7, 9, 13, 5), (30, 40, 61, 17), (256, 256, 512, 512), (1, 5, 3, 9),
                                     (2, 3, 5, 2), (333, 417, 512, 512), (1, 1, 4, 3)])
def test_zoom_restatement_equals_scipy_2d(h, w, H, W):
    import scipy.ndimage as ndi
    x = np.random.default_rng(h * 31 + W).standard_normal((h, w)) * 50
    want = ndi.zoom(x, (H / h, W / w), order=3, mode="nearest", grid_mode=True)
    got = PO.zoom_order3_torch64(torch.from_numpy(x), (H, W)).numpy()
    assert want.shape == got.shape and np.array_equal(want, got)


@pytest.mark.parametrize("z,h,w,H,W", [(3, 17, 23, 40, 11), (1, 9, 8, 12, 12), (5, 2, 3, 7, 1), (2, 64, 48, 33, 97)])
def test_zoom_restatement_equals_scipy_3d_z_unchanged(z, h, w, H, W):
    import scipy.ndimage as ndi
    x = np.random.default_rng(z * 7 + h).standard_normal((z, h, w)) * 20
    want = ndi.zoom(x, (1.0, H / h, W / w), order=3, mode="nearest", grid_mode=True)
    got = PO.zoom_order3_torch64(torch.from_numpy(x), (z, H, W)).numpy()
    assert want.shape == got.shape and np.array_equal(want, got)


def test_spline_filter_equals_scipy_on_padded_lengths():
    import scipy.ndimage as ndi
    rng = np.random.default_rng(3)
    for n in (25, 26, 37, 100, 281, 548):
        x = rng.standard_normal((4, n)) * 10
        want = ndi.spline_filter1d(x, 3, axis=1, output=np.float64, mode="nearest")
        assert np.array_equal(PO.spline_filter_axis(torch.from_numpy(x), 1).numpy(), want), n


@pytest.mark.parametrize("n", [1, 5, 8, 9, 127, 128, 129, 255, 1000, 8191, 8193, 40000, (1 << 20) + 37])
def test_pairwise_sum_and_mean_std_equal_numpy(n):
    a = (np.random.default_rng(n).standard_normal(n) * 100 + 3).astype(np.float32)
    assert PO.pairwise_sum_f32(a) == a.sum(dtype=np.float32)
    m, s = PO.mean_std_f32(a)
    assert m == a.mean() and s == a.std()


@pytest.mark.parametrize("shape,perm", [((3, 70, 90), (0, 2, 1)), ((40, 33, 17), (1, 0, 2)), ((5, 300, 800), (2, 1, 0))])
def test_reduction_order_of_views(shape, perm):
    """Without a mask numpy reduces a transposed view in memory order; with the mask it gathers in the view's order."""
    a = (np.random.default_rng(len(shape) + shape[1]).standard_normal(shape) * 7 + 1).astype(np.float32)
    v = a.transpose(perm)
    assert PO.mean_std_f32(PO.memory_order(v)) == (v.mean(), v.std())
    mask = np.ones(v.shape, bool)
    assert PO.mean_std_f32(v.ravel()) == (v[mask].mean(), v[mask].std())


@pytest.mark.parametrize("case", MG.CASES, ids=[c[0] for c in MG.CASES])
def test_restatement_reproduces_golden(case):
    name, _, _, spacing, tf, cfg_spacing, schemes, use_mask = case
    data = REF[f"{name}_input"]
    out, props = PO.preprocess_case(data, spacing, tf, cfg_spacing, schemes, use_mask, MG.INTENSITY)
    want = REF[f"{name}_output"]
    assert out.dtype == np.float32 and out.shape == want.shape
    assert np.array_equal(out.view(np.int32), want.view(np.int32))
    assert list(props["shape_before_cropping"]) == REF[f"{name}_shape_before_cropping"].tolist()
    assert props["bbox_used_for_cropping"] == REF[f"{name}_bbox"].tolist()
    assert list(props["shape_after_cropping_and_before_resampling"]) == REF[f"{name}_shape_after"].tolist()


# ---- argument contract and call sequence (recording stand-in for the native library)


class _Recorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*a):
            self.calls.append((name, a))
            return 64 if name.endswith("_work_doubles") else 0
        return fn


@pytest.fixture
def rec(monkeypatch):
    from dinounet_b200 import lib as L
    r = _Recorder()
    monkeypatch.setattr(L, "load", lambda: r)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda dev=None: SimpleNamespace(cuda_stream=0))
    return r


def _managers(schemes=("ZScoreNormalization",), use_mask=None, spacing=(0.5, 0.5), tf=(0, 1, 2), conf=None):
    c = {"preprocessor_name": "DefaultPreprocessor", "resampling_fn_data": PP.DEFAULT_RESAMPLING_FN,
         "resampling_fn_data_kwargs": dict(PP.DEFAULT_RESAMPLING_KWARGS)}
    c.update(conf or {})
    cm = SimpleNamespace(spacing=list(spacing), normalization_schemes=list(schemes), configuration=c,
                         use_mask_for_norm=list(use_mask if use_mask is not None else [False] * len(schemes)))
    pm = SimpleNamespace(transpose_forward=list(tf), foreground_intensity_properties_per_channel=MG.INTENSITY)
    return pm, cm


def _run(data, spacing, managers, seg=None):
    pm, cm = managers
    props = {"spacing": list(spacing)}
    return PP.DevicePreprocessor(device=torch.device("cpu")).run_case_npy(data, seg, props, pm, cm, {}), props


def test_call_sequence_slices_and_properties(rec):
    data = np.ones((2, 3, 20, 16), np.float32)
    (out, seg), props = _run(data, [5.0, 1.0, 1.0], _managers(("ZScoreNormalization", "CTNormalization"), [True, False],
                                                               tf=(0, 2, 1)))
    assert props["shape_before_cropping"] == (3, 16, 20) == props["shape_after_cropping_and_before_resampling"]
    assert props["bbox_used_for_cropping"] == [[0, 3], [0, 16], [0, 20]]
    assert out.shape == (2, 3, 32, 40) and out.dtype == torch.float32
    assert seg.shape == (1, 3, 32, 40) and seg.dtype == np.int8 and not seg.any()
    names = [n for n, _ in rec.calls]
    assert names == ["b2u_pre_minmax_f32"] * 2 + ["b2u_pre_zscore", "b2u_pre_normalize", "b2u_pre_resample3_work_doubles"] + \
        ["b2u_pre_resample3"] * 2
    z = rec.calls[2][1]
    assert z[1:8] == (960, 3, 16, 20, 320, 1, 16)        # use_mask: the transposed view's order
    ct = rec.calls[3][1]
    assert ct[1:3] == (960, 1) and ct[4:8] == (-1.0, 1.0, 0.0, 1.0)   # channel 1's properties
    r = rec.calls[5][1]
    assert r[1:11] == (3, 16, 20, 320, 1, 16, 32, 40, 0, r[10]) and r[9] == 0   # per slice


def test_call_sequence_3d_memory_order_and_identity(rec):
    data = np.ones((1, 4, 10, 12), np.float32)
    (out, _), _ = _run(data, [1.0, 1.0, 1.0], _managers(spacing=(0.5, 1.2)))
    z = [a for n, a in rec.calls if n == "b2u_pre_zscore"][0]
    assert z[2:8] == (1, 1, 480, 0, 0, 1)                # memory order without the mask
    r = [a for n, a in rec.calls if n == "b2u_pre_resample3"][0]
    assert r[7:10] == (20, 10, 1) and out.shape == (1, 4, 20, 10)   # 3-D path
    rec.calls.clear()
    (out, seg), _ = _run(data, [4.0, 1.0, 1.0], _managers(("RGBTo01Normalization",), spacing=(1.0, 1.0)))
    assert "b2u_pre_resample3" not in [n for n, _ in rec.calls] and out.shape == (1, 4, 10, 12)


def test_rejections_before_any_launch(rec):
    data = np.ones((1, 3, 20, 16), np.float32)
    sp = [5.0, 1.0, 1.0]
    cases = [
        (sp, _managers(conf={"preprocessor_name": "OtherPreprocessor"}), None),
        (sp, _managers(conf={"resampling_fn_data": "resample_data_or_seg_to_spacing"}), None),
        (sp, _managers(conf={"resampling_fn_data_kwargs": {**PP.DEFAULT_RESAMPLING_KWARGS, "order": 1}}), None),
        (sp, _managers(spacing=(5.0, 0.5, 0.5)), None),                         # 3-D configuration
        (sp, _managers(("ZScoreNormalization", "GammaNormalization")), None),
        (sp, _managers(conf={"preprocessor_name": None}), None),                # no preprocessor named
        (sp, _managers(), np.zeros((1, 3, 20, 16), np.int8)),                    # training / cascade seg
    ]
    for spacing, mgr, seg in cases:
        with pytest.raises(NotImplementedError):
            _run(np.ones((2, 3, 20, 16), np.float32) if "Gamma" in str(mgr) else data, spacing, mgr, seg)
    # the target changes Z (3-D target spacing would), and separate z with an in-plane low-resolution axis
    with pytest.raises(NotImplementedError):
        PP.resampling_path((3, 20, 16), (4, 20, 16), [1, 1, 1], [0.75, 1, 1])
    with pytest.raises(NotImplementedError):
        _run(data, [1.0, 5.0, 1.0], _managers(spacing=(5.0, 2.0)))
    assert rec.calls == []


def test_predict_single_npy_array_rejects_cascade_before_any_launch(rec):
    from dinounet_b200.sliding_window import SlidingWindowPredictor
    p = SlidingWindowPredictor(device=torch.device("cuda", 0))
    pm, cm = _managers()
    p.plans_manager, p.configuration_manager, p.dataset_json = pm, cm, {}
    with pytest.raises(NotImplementedError):
        p.predict_single_npy_array(np.ones((1, 3, 20, 16), np.float32), {"spacing": [5.0, 1.0, 1.0]},
                                   segmentation_previous_stage=np.zeros((3, 20, 16), np.int8))
    p.plans_manager = None
    with pytest.raises(ValueError):
        p.predict_single_npy_array(np.ones((1, 3, 20, 16), np.float32), {"spacing": [5.0, 1.0, 1.0]})
    assert rec.calls == []


# ZScore without the mask (channel 0, sums in memory order) and with it (channel 1, the transposed view's order)
LAYOUT_CASE = ("layout", (2, 5, 130, 70), "float32", [4.0, 1.0, 1.0], [0, 2, 1], [0.8, 1.1],
               ["ZScoreNormalization", "ZScoreNormalization"], [False, True])


def layout_input():
    return (np.random.default_rng(1).standard_normal(LAYOUT_CASE[1]) * 9 + 2).astype(np.float32)


LAYOUTS = {
    "C": lambda a: a,
    "F": np.asfortranarray,
    "transposed": lambda a: np.ascontiguousarray(a.transpose(0, 3, 1, 2)).transpose(0, 2, 3, 1),
    "flipped": lambda a: np.ascontiguousarray(a[:, :, ::-1])[:, :, ::-1],
}


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_memory_axes_follow_numpy_copy(layout):
    """The device copy's channel order is the memory order of the reference's np.copy (order 'K'), so ZScore without
    the mask sums what numpy sums."""
    a = LAYOUTS[layout](layout_input())
    ref_copy = np.copy(a)
    axes = PP.memory_axes(a)
    dev_layout = np.ascontiguousarray(a.transpose(0, *[i + 1 for i in axes]))
    for c in range(2):
        assert np.array_equal(dev_layout[c].ravel(), PO.memory_order(ref_copy[c]))
        assert PO.mean_std_f32(dev_layout[c].ravel()) == (ref_copy[c].mean(), ref_copy[c].std())
    assert PP.memory_axes(torch.from_numpy(np.ascontiguousarray(a))) == [0, 1, 2]


@pytest.mark.parametrize("layout", ["F", "transposed"])
def test_oracle_equals_reference_on_other_layouts(layout, tmp_path):
    """The reference's run_case_npy on a Fortran-ordered and a transposed input (ZScore with and without the mask) equals
    the restatement, which the GPU tests hold the device to.  The reference runs in a subprocess, so its module
    stand-ins stay out of this process."""
    import subprocess
    import sys
    from oracle import ref_loader
    if not ref_loader.reference_available():
        pytest.skip("reference sources not present")
    case = LAYOUT_CASE
    data = LAYOUTS[layout](layout_input())
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    # the input is rebuilt there with the same layout (an .npy file keeps C or Fortran order only)
    code = ("import sys, numpy as np; sys.path.insert(0, '.'); from oracle import make_golden_preprocess as MG; "
            "from tests.test_preprocess_cpu import LAYOUTS, LAYOUT_CASE, layout_input; "
            "out, _, _ = MG.run_reference(LAYOUT_CASE, LAYOUTS[sys.argv[1]](layout_input())); np.save(sys.argv[2], out)")
    subprocess.run([sys.executable, "-c", code, layout, str(tmp_path / "out.npy")], cwd=root, check=True,
                   capture_output=True)
    want = np.load(tmp_path / "out.npy")
    _, _, _, spacing, tf, cfg_spacing, schemes, use_mask = case
    got, _ = PO.preprocess_case(data, spacing, tf, cfg_spacing, schemes, use_mask, MG.INTENSITY)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    # the layout matters: the unmasked channel's bits differ from those of the C-ordered input
    c_order, _ = PO.preprocess_case(layout_input(), spacing, tf, cfg_spacing, schemes, use_mask, MG.INTENSITY)
    assert not np.array_equal(got[0], c_order[0]) and np.array_equal(got[1], c_order[1])


def test_predict_logits_ensemble_order():
    """Folds: the first copied, the others added, then one division by the number of folds."""
    calls = []
    runs = [torch.ones(2, 3, dtype=torch.half) * k for k in (1, 2, 3)]
    acc = PP.ensemble_logits(iter(runs), 3, lambda a, x, d: calls.append((x is None, d)))
    assert calls == [(False, 0), (False, 0), (True, 3)] and torch.equal(acc, runs[0])
    calls.clear()
    PP.ensemble_logits(iter(runs[:1]), 1, lambda a, x, d: calls.append(d))
    assert calls == []


def test_fp16_ensemble_rule_matches_torch_cpu():
    """The kernel's rule fp16(fp32(a) + fp32(b)), fp16(fp32(a) / n) is what torch's CPU fp16 `+=` and `/=` compute."""
    g = torch.Generator().manual_seed(0)
    a = (torch.randn(100000, generator=g) * 30).half()
    b = (torch.randn(100000, generator=g) * 30).half()
    c = (torch.randn(100000, generator=g) * 30).half()
    want = a.clone()
    want += b
    want += c
    want /= 3
    got = (a.float() + b.float()).half()
    got = (got.float() + c.float()).half()
    got = (got.float() / 3.0).half()
    assert torch.equal(want.view(torch.int16), got.view(torch.int16))
