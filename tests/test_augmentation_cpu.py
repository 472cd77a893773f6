"""CPU: the restatement of the training augmentation (oracle/augmentation_oracle.py) pinned to scipy, the host side of
dinounet_b200/augmentation.py (initial patch size, draw order, record) and the trainer's opt-in switch."""
import importlib.util
import os
import sys
import types

import numpy as np
import pytest
import torch
from scipy import ndimage as ndi

import dinounet_b200.training as TR
from dinounet_b200 import augmentation as A
from oracle import augmentation_oracle as AO
from oracle.ref_loader import REF_ROOT

REF_PATCH = os.path.join(REF_ROOT, "dinounet", "training", "data_augmentation", "compute_initial_patch_size.py")


def _coords(in_shape, out_shape, angle, scale):
    H, W = out_shape
    c0, c1 = np.meshgrid(np.arange(H) - (H - 1) / 2.0, np.arange(W) - (W - 1) / 2.0, indexing="ij")
    c0, c1 = c0 * np.cos(angle) + c1 * np.sin(angle), c1 * np.cos(angle) - c0 * np.sin(angle)
    return c0 * scale + in_shape[0] / 2.0 - 0.5, c1 * scale + in_shape[1] / 2.0 - 0.5


@pytest.mark.parametrize("order", [1, 3])
@pytest.mark.parametrize("shape,out", [((37, 29), (30, 24)), ((5, 4), (7, 6)), ((2, 3), (4, 4)), ((64, 71), (50, 60))])
@pytest.mark.parametrize("angle,scale", [(0.0, 1.0), (0.3, 1.1), (2.5, 0.8), (-3.0, 1.39)])
def test_map_coordinates_equals_scipy(order, shape, out, angle, scale):
    x = np.random.RandomState(sum(shape)).randn(*shape).astype(np.float32).astype(float)
    c0, c1 = _coords(shape, out, angle, scale)
    for cval in (0.0, -1.0):
        want = ndi.map_coordinates(x, [c0, c1], order=order, mode="constant", cval=cval)
        got = AO.map_coordinates_torch64(x, c0, c1, order, cval).numpy()
        assert np.array_equal(want, got)


@pytest.mark.parametrize("labels", [2, 5, 255])
def test_seg_rule_equals_per_label_scipy(labels):
    """interpolate_img(is_seg=True, order 1, cval -1): one scipy map per label, ascending, later labels win ties."""
    rng = np.random.RandomState(labels)
    seg = rng.randint(-1, labels, (33, 41)).astype(np.int16)
    seg[:8, :8] = 3 % labels                               # blocks so that half-way ties occur on edges
    for angle, scale in ((0.0, 1.0), (np.pi / 2, 1.0), (0.4, 0.9), (1.0, 1.3)):
        c0, c1 = _coords(seg.shape, (30, 36), angle, scale)
        c0, c1 = np.round(c0 * 2) / 2, np.round(c1 * 2) / 2  # half-integer coordinates: sums of exactly 0.5
        want = np.zeros(c0.shape, seg.dtype)
        for c in np.unique(seg):
            m = ndi.map_coordinates((seg == c).astype(float), [c0, c1], order=1, mode="constant", cval=-1)
            want[m >= 0.5] = c
        assert np.array_equal(AO.interpolate_seg(seg, c0, c1), want)


@pytest.mark.parametrize("sigma", [0.5, 0.61, 0.77, 0.99, 1.0])
@pytest.mark.parametrize("shape", [(37, 29), (3, 5), (64, 64)])
def test_gaussian_filter_equals_scipy(sigma, shape):
    x = (np.random.RandomState(3).randn(*shape) * 100).astype(np.float32)
    assert np.array_equal(AO.gaussian_filter_2d(x, sigma), ndi.gaussian_filter(x, sigma))
    for axis in (0, 1):
        assert np.array_equal(AO.gaussian_filter1d_torch64(x, sigma, axis), ndi.gaussian_filter1d(x, sigma, axis))


@pytest.mark.parametrize("target", [(17, 29), (24, 20), (32, 40), (16, 20)])
def test_lowres_equals_scipy_zoom_with_clip(target):
    """skimage resize(order 0 down, order 3 up, mode 'edge') = scipy zoom(grid_mode, mode 'nearest') + the clip."""
    x = np.random.RandomState(1).randn(32, 40).astype(np.float32)
    down = ndi.zoom(x.astype(float), np.divide(target, x.shape), order=0, mode="nearest", grid_mode=True)
    assert down.shape == target
    up = ndi.zoom(down, np.divide(x.shape, target), order=3, mode="nearest", grid_mode=True)
    want = np.clip(up, down.min(), down.max()).astype(np.float32)
    assert np.array_equal(AO.lowres_channel(x, target), want)


def _reference_get_patch_size():
    """The reference's get_patch_size with batchgenerators' rotate_coords_2d restated in a stub module."""
    def rotate_coords_2d(coords, angle):
        rot_matrix = np.array([[np.cos(angle), -np.sin(angle)], [np.sin(angle), np.cos(angle)]])
        return np.dot(coords.reshape(len(coords), -1).transpose(), rot_matrix).transpose().reshape(coords.shape)

    stub = types.ModuleType("batchgenerators.augmentations.utils")
    stub.rotate_coords_2d = rotate_coords_2d
    stub.rotate_coords_3d = None
    mods = {"batchgenerators": types.ModuleType("batchgenerators"),
            "batchgenerators.augmentations": types.ModuleType("batchgenerators.augmentations"),
            "batchgenerators.augmentations.utils": stub}
    spec = importlib.util.spec_from_file_location("_ref_initial_patch", REF_PATCH)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.get_patch_size, mods


@pytest.mark.skipif(not os.path.exists(REF_PATCH), reason="reference sources not present")
@pytest.mark.parametrize("patch", [(512, 512), (40, 56), (56, 40), (320, 256), (64, 200), (128, 128), (17, 33)])
def test_initial_patch_size_equals_reference(patch, monkeypatch):
    get_patch_size, mods = _reference_get_patch_size()
    for k, v in mods.items():
        monkeypatch.setitem(sys.modules, k, v)
    rot = A.rotation_for_da_2d(patch)
    want = get_patch_size(patch, *rot.values(), (0.85, 1.25))
    assert np.array_equal(A.initial_patch_size_2d(patch), want)
    assert tuple(A.initial_patch_size_2d((512, 512))) == (602, 602)


def _decisions(p):
    out = []
    B, C = p.noise.shape
    for b in range(B):
        if p.rotate[b]:
            out.append(("rot", b, -1, p.angle[b]))
        if p.scale_on[b]:
            out.append(("scale", b, -1, p.scale[b]))
    for b in range(B):
        if p.noise[b].any():
            out.append(("noise_std", b, -1, p.noise_std[b]))
            out += [("noise", b, c, 1) for c in range(C) if p.noise[b, c]]
    out += [("blur", b, c, p.blur_sigma[b, c]) for b in range(B) for c in range(C) if p.blur_sigma[b, c] > 0]
    out += [("brightness", b, c, p.brightness[b, c]) for b in range(B) if p.brightness_on[b] for c in range(C)]
    out += [("contrast", b, c, p.contrast[b, c]) for b in range(B) for c in range(C) if p.contrast_on[b, c]]
    out += [("lowres", b, c, tuple(p.lowres_shape[b, c])) for b in range(B) for c in range(C) if p.lowres_shape[b, c, 0]]
    out += [("gamma_inv", b, c, p.gamma_inv[b, c]) for b in range(B) if p.gamma_inv_on[b] for c in range(C)]
    out += [("gamma", b, c, p.gamma[b, c]) for b in range(B) if p.gamma_on[b] for c in range(C)]
    out += [("flip", b, ax, 1) for b in range(B) for ax in (0, 1) if p.flip[b, ax]]
    return out


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("B,C,patch", [(8, 1, (512, 512)), (5, 3, (40, 56)), (2, 2, (64, 200))])
def test_sampler_follows_batchgenerators_draw_order(seed, B, C, patch):
    rot = A.rotation_for_da_2d(patch)["x"]
    rng_a, rng_b = np.random.RandomState(seed), np.random.RandomState(seed)
    for _ in range(3):  # consecutive batches share the stream
        p = A.sample_augmentation_params(B, C, patch, rng_a)
        want = AO.draw_decisions(B, C, patch, rng_b, rot)
        got = _decisions(p)
        assert [g[:3] for g in got] == [w[:3] for w in want]
        for g, w in zip(got, want):
            assert np.array_equal(np.asarray(g[3]), np.asarray(w[3]))
    assert rng_a.uniform() == rng_b.uniform()


def test_firing_rates_are_close_to_the_probabilities():
    rng = np.random.RandomState(0)
    B, C, n = 64, 2, 40
    ps = [A.sample_augmentation_params(B, C, (128, 128), rng) for _ in range(n)]
    rate = lambda f: float(np.mean([f(p) for p in ps]))  # noqa: E731
    assert abs(rate(lambda p: p.rotate.mean()) - 0.2) < 0.02
    assert abs(rate(lambda p: p.scale_on.mean()) - 0.2) < 0.02
    assert abs(rate(lambda p: p.noise[:, 0].mean()) - 0.1) < 0.02
    assert abs(rate(lambda p: (p.blur_sigma > 0).mean()) - 0.1) < 0.02
    assert abs(rate(lambda p: p.brightness_on.mean()) - 0.15) < 0.02
    assert abs(rate(lambda p: p.contrast_on[:, 0].mean()) - 0.15) < 0.02
    assert abs(rate(lambda p: (p.lowres_shape[..., 0] > 0).mean()) - 0.125) < 0.02
    assert abs(rate(lambda p: p.gamma_inv_on.mean()) - 0.1) < 0.02
    assert abs(rate(lambda p: p.gamma_on.mean()) - 0.3) < 0.02
    assert abs(rate(lambda p: p.flip.mean()) - 0.5) < 0.02
    a = np.concatenate([p.angle[p.rotate] for p in ps])
    assert a.min() >= -np.pi and a.max() <= np.pi
    s = np.concatenate([p.scale[p.scale_on] for p in ps])
    assert s.min() >= 0.7 and s.max() <= 1.4 and abs((s < 1).mean() - 0.5) < 0.1


def test_record_layout():
    p = A.AugmentationParams.identity(2, 3)
    p.blur_sigma[1, 2] = 0.8
    p.lowres_shape[0, 1] = (20, 30)
    p.flip[1] = (False, True)
    r = A.pack_record(p, (40, 40), [True, False, True]).reshape(2, 3, A.REC)
    w = AO.gaussian_kernel1d(0.8)
    assert r[1, 2, A.F_BLUR_R] == 3 and np.array_equal(r[1, 2, A.F_BLUR_W:A.F_BLUR_W + 4], w[3:])
    assert r[0, 1, A.F_LOW_H] == 20 and r[0, 1, A.F_LOW_W] == 30 and r[0, 0, A.F_LOW_H] == 0
    assert r[0, 1, A.F_LOW_Y + 1] == np.float64(AO.PRE.filter_consts(44)[1])
    assert list(r[1, :, A.F_FLIP1]) == [1, 1, 1] and list(r[0, :, A.F_MASK]) == [1, 0, 1]


def test_golden_cases_reproduce():
    from oracle import make_golden_augmentation as MG
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "augmentation_cases.npz"))
    arrays = MG.golden_arrays()
    assert sorted(arrays) == sorted(g.files)
    for k in g.files:
        assert np.array_equal(arrays[k], g[k]), k


def test_bad_configuration_is_rejected():
    with pytest.raises(ValueError):
        A.DeviceTrainingAugmentation((64, 64, 64))
    with pytest.raises(ValueError):
        A.DeviceTrainingAugmentation((64, 64), mirror_axes=(0, 2))
    with pytest.raises(ValueError):
        A.DeviceTrainingAugmentation((64, 64), regions=[(1, 2), 2.5])
    aug = A.DeviceTrainingAugmentation((32, 32), seed=0)
    with pytest.raises(ValueError):   # host tensors are rejected before anything is launched
        aug(torch.zeros(2, 1, 40, 40), torch.zeros(2, 1, 40, 40, dtype=torch.int16))


# ---- the trainer's switch


@pytest.fixture
def switch():
    saved = TR.DinoUNetTrainer._device_augmentation
    yield
    TR.DinoUNetTrainer._device_augmentation = saved


def test_switch_is_stored_like_train_semantics(switch):
    TR.DinoUNetTrainer_s.set_network_config({"architecture": {}}, device_augmentation=True)
    assert TR.DinoUNetTrainer._device_augmentation is True
    TR.DinoUNetTrainer_s.set_network_config({"architecture": {}})
    assert TR.DinoUNetTrainer._device_augmentation is False


def _trainer(monkeypatch):
    tr = TR.DinoUNetTrainer_s.__new__(TR.DinoUNetTrainer_s)
    tr.device, tr.network, tr.is_ddp, tr.local_rank = torch.device("cpu"), object(), False, 0
    tr.loss, tr.optimizer = "loss", "opt"
    tr.label_manager = types.SimpleNamespace(has_regions=True, foreground_regions=[(1, 2), 2], ignore_label=3)
    tr.configuration_manager = types.SimpleNamespace(patch_size=[64, 48], use_mask_for_norm=[True])
    tr.configure_rotation_dummyDA_mirroring_and_inital_patch_size = lambda: ("rot", False, [80, 60], (0, 1))
    steps = []
    import dinounet_b200.train_path as TP
    monkeypatch.setattr(TP, "train_step", lambda net, loss, opt, x, t: steps.append((x, t)) or torch.tensor(1.5))
    return tr, steps


def test_switch_off_passes_through(switch, monkeypatch):
    TR.DinoUNetTrainer_s.set_network_config({"architecture": {}})
    seen = []

    class Base:
        @staticmethod
        def get_training_transforms(*a, **k):
            seen.append((a, k))
            return "reference pipeline"

    monkeypatch.setattr(TR, "_Base", Base)
    assert TR.DinoUNetTrainer_s.get_training_transforms((64, 48), "rot", None, (0, 1), False, order_resampling_data=3) \
        == "reference pipeline"
    assert seen == [(((64, 48), "rot", None, (0, 1), False), {"order_resampling_data": 3})]
    tr, steps = _trainer(monkeypatch)
    x, t = torch.zeros(2, 1, 64, 48), torch.zeros(2, 1, 64, 48)
    assert tr.train_step({"data": x, "target": [t]})["loss"] == 1.5
    assert steps[0][0] is x and steps[0][1] is t and not hasattr(tr, "_device_aug")


def test_switch_on_builds_the_device_augmenter(switch, monkeypatch):
    TR.DinoUNetTrainer_s.set_network_config({"architecture": {}}, device_augmentation=True)
    pipe = TR.DinoUNetTrainer_s.get_training_transforms((64, 48), "rot", None, (0, 1), False)
    out = pipe(data=np.ones((2, 1, 80, 60)), seg=np.full((2, 1, 80, 60), -1), keys=["a"])
    assert out["data"].dtype == torch.float32 and out["target"].dtype == torch.int16 and "seg" not in out
    assert out["keys"] == ["a"]
    built, calls = [], []

    class Recorder:
        def __init__(self, *a, **k):
            built.append((a, k))

        def __call__(self, data, seg):
            calls.append((data, seg))
            return "augmented data", "augmented target"

    monkeypatch.setattr(A, "DeviceTrainingAugmentation", Recorder)
    tr, steps = _trainer(monkeypatch)
    for _ in range(2):
        tr.train_step({"data": out["data"], "target": out["target"]})
    assert len(built) == 1 and len(calls) == 2
    a, k = built[0]
    assert a == ([64, 48], "rot", (0, 1))
    assert k["use_mask_for_norm"] == [True] and k["regions"] == [(1, 2), 2] and k["ignore_label"] == 3
    assert steps[0] == ("augmented data", "augmented target")
    seeds = set()
    for rank in range(3):
        t2, _ = _trainer(monkeypatch)
        t2.is_ddp, t2.local_rank = True, rank
        TR.DinoUNetTrainer._device_augmentation_seed = 5
        try:
            t2._device_augmenter()
        finally:
            TR.DinoUNetTrainer._device_augmentation_seed = None
        seeds.add(built[-1][1]["seed"])
    assert len(seeds) == 3                              # each rank its own stream
