"""-m gpu: device preprocessing against the reference's run_case_npy (tests/golden/preprocess_cases.npz) and against the
restatements of oracle/preprocess_oracle.py (pinned to scipy and numpy in tests/test_preprocess_cpu.py), bit for bit;
and predict_single_npy_array end to end against the oracle's preprocessing -> sliding window -> device export."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dinounet_b200 import lib as L
from dinounet_b200 import preprocess as PP
from oracle import make_golden_preprocess as MG
from oracle import preprocess_oracle as PO
from tests.gpu_helpers import stream

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
REF = np.load(os.path.join(os.path.dirname(__file__), "golden", "preprocess_cases.npz"))


def _managers(schemes, use_mask, cfg_spacing, tf):
    conf = {"preprocessor_name": "DefaultPreprocessor", "resampling_fn_data": PP.DEFAULT_RESAMPLING_FN,
            "resampling_fn_data_kwargs": dict(PP.DEFAULT_RESAMPLING_KWARGS)}
    cm = SimpleNamespace(spacing=list(cfg_spacing), normalization_schemes=list(schemes),
                         use_mask_for_norm=list(use_mask), configuration=conf)
    pm = SimpleNamespace(transpose_forward=list(tf), foreground_intensity_properties_per_channel=MG.INTENSITY)
    return pm, cm


def _preprocess(data, spacing, schemes, use_mask, cfg_spacing, tf):
    pm, cm = _managers(schemes, use_mask, cfg_spacing, tf)
    props = {"spacing": list(spacing)}
    out, seg = PP.DevicePreprocessor(device=DEV).run_case_npy(data, None, props, pm, cm, {})
    torch.cuda.synchronize()
    return out, seg, props


def _bits(a):
    return np.ascontiguousarray(a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a).view(np.int32)


@pytest.mark.parametrize("case", MG.CASES, ids=[c[0] for c in MG.CASES])
def test_golden_cases_bit_identical(case):
    name, _, _, spacing, tf, cfg_spacing, schemes, use_mask = case
    out, seg, props = _preprocess(REF[f"{name}_input"], spacing, schemes, use_mask, cfg_spacing, tf)
    assert out.is_cuda and out.dtype == torch.float32
    assert np.array_equal(_bits(out), _bits(REF[f"{name}_output"]))
    assert seg.dtype == np.int8 and list(seg.shape) == REF[f"{name}_seg_shape"].tolist() and not seg.any()
    assert props["bbox_used_for_cropping"] == REF[f"{name}_bbox"].tolist()
    assert list(props["shape_before_cropping"]) == REF[f"{name}_shape_before_cropping"].tolist()


def _resample(x, H, W, three_d):
    Z, h, w = x.shape
    consts = PP.filter_consts(Z + 24) + PP.filter_consts(h + 24) + PP.filter_consts(w + 24)
    import ctypes
    arr = (ctypes.c_double * 15)(*consts)
    lib = L.load()
    work = torch.empty(int(lib.b2u_pre_resample3_work_doubles(Z, h, w, int(three_d))), dtype=torch.float64, device=DEV)
    out = torch.empty((Z, H, W), dtype=torch.float32, device=DEV)
    L.check(lib.b2u_pre_resample3(x.data_ptr(), Z, h, w, h * w, w, 1, H, W, int(three_d), ctypes.addressof(arr),
                                  work.data_ptr(), out.data_ptr(), stream()), "resample3")
    torch.cuda.synchronize()
    return out


SWEEP = [  # Z, h, w, H, W, three_d: odd sizes, factors above and below 1, both paths
    (3, 37, 53, 64, 29, False), (1, 1, 9, 5, 17, False), (2, 101, 77, 512, 512, False), (5, 256, 256, 97, 131, False),
    (3, 17, 23, 40, 11, True), (1, 9, 8, 12, 12, True), (4, 65, 33, 30, 70, True), (2, 2, 3, 7, 1, True),
]


@pytest.mark.parametrize("Z,h,w,H,W,three_d", SWEEP)
def test_resample_sweep_bit_identical_to_restatement(Z, h, w, H, W, three_d):
    x = (torch.randn(Z, h, w, generator=torch.Generator().manual_seed(Z * 100 + h)) * 3).float()
    got = _resample(x.to(DEV), H, W, three_d)
    want = PO.resample_channel(x.numpy(), H, W, three_d)
    assert torch.equal(got.cpu().view(torch.int32), want.view(torch.int32))


@pytest.mark.parametrize("shape,perm,mask", [((4, 70, 90), (0, 2, 1), False), ((4, 70, 90), (0, 2, 1), True),
                                             ((60, 33, 417), (1, 0, 2), True), ((60, 333, 417), (0, 1, 2), False)])
def test_zscore_bit_identical_to_numpy(shape, perm, mask):
    a = (np.random.default_rng(shape[1]).standard_normal(shape) * 40 + 7).astype(np.float32)
    v = a.transpose(perm)
    if mask:
        m = np.ones(v.shape, bool)
        mean, std = v[m].mean(), v[m].std()
        o = [v.shape[0], v.shape[1], v.shape[2], *(s // 4 for s in v.strides)]
    else:
        mean, std = v.mean(), v.std()
        o = [1, 1, a.size, 0, 0, 1]
    want = (v - mean) / max(std, 1e-8)
    x = torch.from_numpy(a).to(DEV)
    work = torch.empty((a.size + 7) // 8, dtype=torch.float32, device=DEV)
    stats = torch.empty(2, dtype=torch.float32, device=DEV)
    L.check(L.load().b2u_pre_zscore(x.data_ptr(), a.size, *o, work.data_ptr(), stats.data_ptr(), stream()), "zscore")
    torch.cuda.synchronize()
    s = stats.cpu().numpy()
    assert s[0] == mean and s[1] == max(std, np.float32(1e-8))
    assert np.array_equal(x.cpu().numpy().transpose(perm).view(np.int32), np.ascontiguousarray(want).view(np.int32))


def test_realistic_case_and_repeat_launches():
    """3 x 60 x 333 x 417 -> 60 x 512 x 512 per slice (0.9 mm in-plane, 4 mm slices), ZScore with and without the mask."""
    data = (np.random.default_rng(1).standard_normal((3, 60, 333, 417)) * 100 + 40).astype(np.float32)
    args = ([4.0, 0.9, 0.9], ["ZScoreNormalization", "ZScoreNormalization", "CTNormalization"],
            [False, True, False], [0.9 * 333 / 512, 0.9 * 417 / 512], [0, 1, 2])
    out1, _, props = _preprocess(data, *args)
    out2, _, _ = _preprocess(data, *args)
    assert out1.shape == (3, 60, 512, 512)
    assert torch.equal(out1.view(torch.int32), out2.view(torch.int32))
    want, _ = PO.preprocess_case(data, args[0], args[4], args[3], args[1], args[2], MG.INTENSITY)
    assert np.array_equal(_bits(out1), want.view(np.int32))


def test_nonfinite_and_rgb_range_raise():
    data = np.ones((1, 1, 8, 8), np.float32)
    data[0, 0, 3, 3] = np.nan
    with pytest.raises(ValueError):
        _preprocess(data, [1, 1, 1], ["ZScoreNormalization"], [False], [1, 1], [0, 1, 2])
    with pytest.raises(AssertionError):
        _preprocess(np.full((1, 1, 8, 8), 300, np.float32), [1, 1, 1], ["RGBTo01Normalization"], [False], [1, 1],
                    [0, 1, 2])


def test_predict_single_npy_array_end_to_end():
    """predict_single_npy_array (device preprocessing -> fold ensemble -> device export) gives the labels of the oracle's
    preprocessing uploaded -> predict_sliding_window_return_logits -> the fp16 CPU ensemble -> the device export."""
    import dinounet_b200
    from dinounet_b200 import config, export as EX
    from dinounet_b200.sliding_window import SlidingWindowPredictor
    from oracle import dinounet_oracle as O
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, 3, None,
                                             "dinounet_s")
    folds = [O.make_state_dict("dinounet_s", 3, seed=s) for s in (0, 1)]
    net.load_state_dict(folds[0], strict=True)
    net = net.to(DEV).eval()
    conf = {"preprocessor_name": "DefaultPreprocessor", "resampling_fn_data": PP.DEFAULT_RESAMPLING_FN,
            "resampling_fn_data_kwargs": dict(PP.DEFAULT_RESAMPLING_KWARGS),
            "resampling_fn_probabilities": EX.DEFAULT_RESAMPLING_FN,
            "resampling_fn_probabilities_kwargs": dict(EX.DEFAULT_RESAMPLING_KWARGS)}
    cm = SimpleNamespace(spacing=[0.8, 0.8], patch_size=[128, 128], normalization_schemes=["ZScoreNormalization"] * 3,
                         use_mask_for_norm=[False] * 3, configuration=conf)
    lm = SimpleNamespace(has_regions=False, regions_class_order=None, foreground_labels=[1, 2], num_segmentation_heads=3)
    pm = SimpleNamespace(transpose_forward=[0, 1, 2], transpose_backward=[0, 1, 2], get_label_manager=lambda dj: lm,
                         foreground_intensity_properties_per_channel=MG.INTENSITY)
    image = (np.random.default_rng(5).standard_normal((3, 2, 90, 150)) * 20).astype(np.float32)
    for params in (None, folds):
        p = SlidingWindowPredictor(tile_step_size=0.5, use_gaussian=True, use_mirroring=True, device=DEV, tile_batch=4)
        p.manual_initialization(net, pm, cm, params, {}, "DinoUNetTrainer_s", (0, 1))
        props = {"spacing": [3.0, 1.0, 1.0]}
        seg, probs = p.predict_single_npy_array(image, props, None, None, True)
        # oracle route
        data, oprops = PO.preprocess_case(image, [3.0, 1.0, 1.0], [0, 1, 2], [0.8, 0.8], ["ZScoreNormalization"] * 3,
                                          [False] * 3, MG.INTENSITY)
        assert {k: props[k] for k in oprops} == oprops
        acc = None
        for sd in (params or [None]):
            if sd is not None:
                net.load_state_dict(sd)
                net.repack()
            lg = p.predict_sliding_window_return_logits(torch.from_numpy(data).to(DEV)).cpu()
            if acc is None:
                acc = lg.clone()
            else:
                acc += lg
        if params:
            acc /= len(params)
        got_logits = p.predict_logits_from_preprocessed_data(torch.from_numpy(data).to(DEV))
        assert torch.equal(got_logits.cpu().view(torch.int16), acc.view(torch.int16))
        want_seg, want_p = EX.convert_predicted_logits_to_segmentation_with_correct_shape(acc, pm, cm, lm, props, True)
        assert seg.shape == (2, 90, 150) and np.array_equal(seg, want_seg)
        assert np.array_equal(probs.view(np.int32), want_p.view(np.int32))


def test_caller_input_is_never_written():
    """A contiguous fp32 device tensor (what a caller chaining device stages passes) is copied, not normalized in
    place, and gives the same bits as host input; so does a second call on the same tensor."""
    case = next(c for c in MG.CASES if c[0] == "volume_mixed_ct_rescale")
    name, _, _, spacing, tf, cfg_spacing, schemes, use_mask = case
    x = torch.from_numpy(REF[f"{name}_input"]).to(DEV)
    before = x.clone()
    for _ in range(2):
        out, _, _ = _preprocess(x, spacing, schemes, use_mask, cfg_spacing, tf)
        assert torch.equal(x.view(torch.int32), before.view(torch.int32))
        assert np.array_equal(_bits(out), _bits(REF[f"{name}_output"]))
    host = REF[f"{name}_input"].copy()
    _preprocess(host, spacing, schemes, use_mask, cfg_spacing, tf)
    assert np.array_equal(host, REF[f"{name}_input"])


@pytest.mark.parametrize("layout", ["C", "F", "transposed", "flipped", "device_strided"])
def test_input_layouts_bit_identical_to_restatement(layout):
    """ZScore without the mask sums in the memory order of the reference's np.copy (order 'K'): Fortran-ordered,
    transposed and flipped inputs each give the restatement's bits (pinned to the reference in the CPU suite)."""
    from tests.test_preprocess_cpu import LAYOUT_CASE, LAYOUTS, layout_input
    _, _, _, spacing, tf, cfg_spacing, schemes, use_mask = LAYOUT_CASE
    host = LAYOUTS["transposed" if layout == "device_strided" else layout](layout_input())
    want, _ = PO.preprocess_case(host, spacing, tf, cfg_spacing, schemes, use_mask, MG.INTENSITY)
    data = host
    if layout == "device_strided":   # the same layout as a strided device tensor
        data = torch.from_numpy(np.ascontiguousarray(host.transpose(0, 3, 1, 2))).to(DEV).permute(0, 2, 3, 1)
    out, _, _ = _preprocess(data, spacing, schemes, use_mask, cfg_spacing, tf)
    assert np.array_equal(_bits(out), want.view(np.int32))
