"""Device training augmentation (csrc/augmentation.cu, dinounet_b200/augmentation.py) against the numpy / scipy
restatement (oracle/augmentation_oracle.py) on the same parameter record and noise field.

Targets (label maps and regions, after mirroring, masking and label removal) must be identical.  Data must be identical
unless a gamma step fired: gamma raises to a power with CUDA's `powf` where numpy uses libm's, so those planes are held
to 1e-4 of the plane's value range."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dinounet_b200 import augmentation as A
from oracle import augmentation_oracle as AO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "augmentation_cases.npz")


ct_like = AO.ct_like


def run_both(aug, data, seg, params, seed, patch):
    d_dev, t_dev = aug.apply(torch.from_numpy(data).to(DEV), torch.from_numpy(seg).to(DEV), params, seed)
    noise = A.noise_field(seed, data.shape[0], data.shape[1], patch, DEV).cpu().numpy()
    d_ref, t_ref = AO.augment(data, seg, params, noise, patch, aug.use_mask_for_norm, aug.regions, aug.ignore_label)
    return d_dev.cpu().numpy(), t_dev.cpu().numpy(), d_ref, t_ref


def check(aug, data, seg, params, seed=7):
    patch = aug.patch_size
    d, t, dr, tr = run_both(aug, data, seg, params, seed, patch)
    assert t.shape == tr.shape and np.array_equal(t, tr)
    gamma = params.gamma_on | params.gamma_inv_on
    for b in range(d.shape[0]):
        if gamma[b]:
            rng = max(float(dr[b].max() - dr[b].min()), 1e-6)
            assert np.abs(d[b] - dr[b]).max() <= 1e-4 * rng, b
        else:
            assert np.array_equal(d[b], dr[b]), (b, np.abs(d[b] - dr[b]).max())
    return d, t


def forced(B, C, patch, on: bool, rng=None):
    """Every transform forced on (with seeded values) or off."""
    p = A.AugmentationParams.identity(B, C)
    if not on:
        return p
    rng = rng or np.random.RandomState(0)
    p.spatial[:] = p.rotate[:] = p.scale_on[:] = True
    p.angle[:] = rng.uniform(-np.pi, np.pi, B)
    p.cos[:], p.sin[:] = np.cos(p.angle), np.sin(p.angle)
    p.scale[:] = rng.uniform(0.7, 1.4, B)
    p.noise[:] = True
    p.noise_std[:] = rng.uniform(0, 0.1, B)
    p.blur_sigma[:] = rng.uniform(0.5, 1, (B, C))
    p.brightness_on[:] = True
    p.brightness[:] = rng.uniform(0.75, 1.25, (B, C))
    p.contrast_on[:] = True
    p.contrast[:] = rng.uniform(0.75, 1.25, (B, C))
    p.lowres_shape[:] = np.round(np.array(patch) * rng.uniform(0.5, 1, (B, C, 1))).astype(int)
    p.gamma_inv_on[:] = p.gamma_on[:] = True
    p.gamma_inv[:] = rng.uniform(0.7, 1.5, (B, C))
    p.gamma[:] = rng.uniform(0.7, 1.5, (B, C))
    p.flip[:] = True
    return p


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_sampled_params_match_oracle(seed):
    """Hippocampus-like: 2 channels, a non-square patch, odd in - out; decisions from the sampler."""
    patch = (40, 56)
    aug = A.DeviceTrainingAugmentation(patch, seed=seed)
    data, seg = ct_like(6, 2, 51, 67, 3, seed)
    check(aug, data, seg, aug.sample(6, 2), seed)


@pytest.mark.parametrize("on", [False, True])
@pytest.mark.parametrize("B,C", [(1, 1), (2, 3)])
def test_every_transform_forced(on, B, C):
    patch = (48, 48)
    aug = A.DeviceTrainingAugmentation(patch, use_mask_for_norm=[c % 2 == 0 for c in range(C)], seed=0)
    data, seg = ct_like(B, C, 57, 58, 4, 11 + B + C)
    check(aug, data, seg, forced(B, C, patch, on))


def test_single_transforms():
    """Each step alone on its own sample, so a mismatch names the step."""
    patch = (32, 40)
    B, C = 10, 1
    p = A.AugmentationParams.identity(B, C)
    p.rotate[0] = p.spatial[0] = True
    p.angle[0] = 0.7
    p.cos[0], p.sin[0] = np.cos(0.7), np.sin(0.7)
    p.scale_on[1] = p.spatial[1] = True
    p.scale[1] = 1.31
    p.noise[2] = True
    p.noise_std[2] = 0.05
    p.blur_sigma[3] = 0.83
    p.brightness_on[4] = True
    p.brightness[4] = 1.17
    p.contrast_on[5] = True
    p.contrast[5] = 0.8
    p.lowres_shape[6] = (17, 29)
    p.gamma_inv_on[7] = True
    p.gamma_inv[7] = 1.3
    p.gamma_on[8] = True
    p.gamma[8] = 0.8
    p.flip[9] = (True, False)
    aug = A.DeviceTrainingAugmentation(patch, seed=0)
    data, seg = ct_like(B, C, 41, 47, 2, 5)
    check(aug, data, seg, p)


def test_large_batch_602_to_512():
    """B = 32, C = 1, 602 -> 512 with -1 padding, sampled decisions (the benchmark's setup)."""
    patch = (512, 512)
    aug = A.DeviceTrainingAugmentation(patch, seed=3)
    assert tuple(A.initial_patch_size_2d(patch)) == (602, 602)
    data, seg = ct_like(32, 1, 602, 602, 45, 3)
    params = aug.sample(32, 1)
    params.rotate[:4] = params.spatial[:4] = True          # make sure transformed samples are among them
    params.angle[:4] = [0.3, -2.0, 3.1, 1.0]
    params.cos[:4], params.sin[:4] = np.cos(params.angle[:4]), np.sin(params.angle[:4])
    check(aug, data, seg, params)


def test_all_padding_sample_and_255_labels():
    patch = (40, 40)
    B = 3
    data, seg = ct_like(B, 1, 49, 49, 0, 2)
    data[0] = 0
    seg[0] = -1                                             # a sample that is padding only
    rng = np.random.RandomState(4)
    seg[1, 0] = rng.randint(0, 255, (49, 49))                # 255 labels, many ties
    seg[2, 0] = np.arange(49 * 49).reshape(49, 49) % 255
    aug = A.DeviceTrainingAugmentation(patch, use_mask_for_norm=[True], seed=0)
    for on in (False, True):
        check(aug, data, seg, forced(B, 1, patch, on, np.random.RandomState(9)))


def test_regions_with_ignore_label():
    patch = (44, 36)
    data, seg = ct_like(4, 2, 53, 45, 3, 8, labels=4)
    seg[:, :, 20:25] = 4                                     # the ignore label
    aug = A.DeviceTrainingAugmentation(patch, regions=[(1, 2, 3), (2, 3), 3], ignore_label=4, seed=1)
    for s in range(3):
        d, t = check(aug, data, seg, aug.sample(4, 2) if s else forced(4, 2, patch, True), s)
        assert t.shape == (4, 4, 44, 36)


def test_noise_field_statistics_and_pipeline():
    field = A.noise_field(123, 2, 2, (512, 512), DEV)
    f = field[0, 0].double()
    assert abs(float(f.mean())) < 0.01 and abs(float(f.std()) - 1) < 0.01
    assert not torch.equal(field[0, 0], field[0, 1]) and not torch.equal(field[0, 0], field[1, 0])
    assert torch.equal(field, A.noise_field(123, 2, 2, (512, 512), DEV))
    # the pipeline's noise on zero data is f32(std * field)
    patch = (64, 80)
    p = A.AugmentationParams.identity(2, 2)
    p.noise[:] = True
    p.noise_std[:] = [0.05, 0.1]
    aug = A.DeviceTrainingAugmentation(patch, seed=0)
    x = torch.zeros((2, 2, 64, 80), device=DEV)
    s = torch.zeros((2, 1, 64, 80), dtype=torch.int16, device=DEV)
    d, _ = aug.apply(x, s, p, 99)
    want = (A.noise_field(99, 2, 2, patch, DEV) * torch.tensor([0.05, 0.1], device=DEV, dtype=torch.float64)[:, None,
                                                                                                            None, None])
    assert torch.equal(d, want.float())


def test_same_seed_is_deterministic():
    patch = (96, 96)
    data, seg = ct_like(4, 1, 113, 113, 5, 1)
    x, s = torch.from_numpy(data).to(DEV), torch.from_numpy(seg).to(DEV)
    outs = []
    for _ in range(2):
        aug = A.DeviceTrainingAugmentation(patch, seed=42)
        outs.append([aug(x, s) for _ in range(3)])
    for (d0, t0), (d1, t1) in zip(*outs):
        assert torch.equal(d0, d1) and torch.equal(t0, t1)
    assert not torch.equal(outs[0][0][0], outs[0][1][0])


def test_golden_cases_reproduce():
    g = np.load(GOLDEN, allow_pickle=False)
    from oracle import make_golden_augmentation as MG
    for name, case in MG.cases().items():
        aug, data, seg, params, seed = case
        d, t = aug.apply(torch.from_numpy(data).to(DEV), torch.from_numpy(seg).to(DEV), params, seed)
        assert np.array_equal(t.cpu().numpy().astype(np.int8), g[f"{name}_target"])
        d = d.cpu().numpy()[:, :, ::8, ::8]
        assert np.allclose(d, g[f"{name}_data"], rtol=0, atol=1e-4 * float(np.ptp(g[f"{name}_data"])))


def test_rejects_bad_input_before_launch():
    aug = A.DeviceTrainingAugmentation((32, 32), seed=0)
    x = torch.zeros((2, 1, 40, 40), device=DEV)
    s = torch.zeros((2, 1, 40, 40), dtype=torch.int16, device=DEV)
    for bad in ((x.double(), s), (x, s.int()), (x[:, :, :30], s[:, :, :30]), (x, s[:1]), (x.cpu(), s)):
        with pytest.raises((ValueError, TypeError)):
            aug(*bad)
    with pytest.raises(ValueError):
        aug.apply(x, s, A.AugmentationParams.identity(3, 1), 0)


def test_trainer_train_step_with_device_augmentation():
    """`DinoUNetTrainer.train_step` with the switch on: dinounet_s at 128^2 from a 150^2 batch; finite loss, weights
    move."""
    import dinounet_b200
    from dinounet_b200 import config
    from dinounet_b200.train_path import FusedSGD
    from oracle import dinounet_oracle as O
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, 2, None,
                                             "dinounet_s")
    net.load_state_dict(O.make_state_dict("dinounet_s", 2, seed=0), strict=True)
    net.precision = "fp32"
    net.train_gemm = "fp32"
    net = net.to(DEV).train()
    T = dinounet_b200.DinoUNetTrainer_s
    saved = dinounet_b200.DinoUNetTrainer._device_augmentation
    try:
        dinounet_b200.DinoUNetTrainer._device_augmentation = True
        tr = T.__new__(T)
        tr.device, tr.network, tr.is_ddp = DEV, net, False
        tr.label_manager = SimpleNamespace(has_regions=False, ignore_label=None, foreground_regions=None)
        tr.configuration_manager = SimpleNamespace(batch_dice=True, patch_size=[128, 128], use_mask_for_norm=[False] * 3)
        tr.configure_rotation_dummyDA_mirroring_and_inital_patch_size = lambda: (
            A.rotation_for_da_2d((128, 128)), False, A.initial_patch_size_2d((128, 128)), (0, 1))
        tr.loss = tr._build_loss()
        tr.optimizer = FusedSGD(net.parameters(), lr=1e-2)
        data, seg = ct_like(2, 3, 150, 150, 6, 0, labels=2)
        batch = T.get_training_transforms((128, 128), None, None, (0, 1), False)(data=data, seg=seg)
        before = [p.detach().clone() for p in net.parameters()]
        out = tr.train_step(batch)
        assert np.isfinite(out["loss"]).all()
        assert any(not torch.equal(a, p.detach()) for a, p in zip(before, net.parameters()))
    finally:
        dinounet_b200.DinoUNetTrainer._device_augmentation = saved
