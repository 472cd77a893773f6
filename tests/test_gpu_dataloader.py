"""-m gpu: the 2-D device loader (dinounet_b200/dataloading.py, csrc/dataloading.cu).

* Device batches are bit-identical to the oracle's (oracle/dataloader_oracle.py, pinned to the reference's own loader
  by tests/golden/dataloader_cases.npz) on the golden cases and on seeded sweeps, in train mode (float32 data, int16
  seg padded with -1) and in val mode (the validation transforms' float32 target, label maps and regions), with row
  lengths that take each store width of the kernel.
* Two loaders with the same seed give the same sequence.
* A stand-in trainer's `get_dataloaders` returns device loaders: `train_step(next(dl_tr))` gives the loss bits of
  `train_step` on the host route's batch for the same draws (oracle batch, `PassThroughTransforms`, `.to(device)`)
  with the same augmentation seed, from the same weights (each step starts both sides from the state dict: the backward
  kernels use atomics, so weights after a step differ in the last bits), and `validation_step` on a val batch gives the
  host route's statistics.
* `on_train_end` leaves no read-ahead thread alive.
"""
import os
import threading
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import dinounet_b200
from dinounet_b200 import augmentation as A
from dinounet_b200 import config
from dinounet_b200 import dataloading as DL
from dinounet_b200 import lib as L
from dinounet_b200 import training as TR
from dinounet_b200.loss import DC_and_CE_loss
from dinounet_b200.train_path import FusedSGD
from oracle import dataloader_oracle as DO
from oracle import dinounet_oracle as O
from oracle import make_golden_dataloader as MG

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _bits(t):
    return t.detach().cpu().contiguous().view(torch.int32).numpy() if t.dtype == torch.float32 else t.cpu().numpy()


def _compare(cases, B, patch, final, lm, osp, seed, nb, regions=None, ignore=None):
    """Device batches of both modes against the oracle's, batch by batch."""
    ds = DO.ArrayDataset(sorted(cases.items()))
    rng = np.random.RandomState(seed)
    tr = DL.DeviceDataLoader2D(ds, B, patch, final, lm, osp, seed=seed, device=DEV)
    va = DL.DeviceDataLoader2D(ds, B, patch, final, lm, osp, mode="val", regions=regions, ignore_label=ignore,
                               seed=seed, device=DEV)
    n0 = L.launch_count()
    try:
        for i in range(nb):
            want, _ = DO.generate_train_batch(ds, B, patch, final, lm.all_labels, lm.has_ignore_label, osp, rng)
            got_t, got_v = next(tr), next(va)
            for got in (got_t, got_v):
                assert list(got["keys"]) == list(want["keys"]), i
                assert got["data"].dtype == torch.float32 and got["data"].is_cuda
                assert np.array_equal(_bits(got["data"]), want["data"].view(np.int32)), i
            assert got_t["target"].dtype == torch.int16
            assert np.array_equal(got_t["target"].cpu().numpy(), want["seg"]), i
            vt = DO.val_target(want["seg"], regions, ignore)
            assert got_v["target"].dtype == torch.float32 and tuple(got_v["target"].shape) == vt.shape
            assert np.array_equal(_bits(got_v["target"]), vt.view(np.int32)), i
        torch.cuda.synchronize()
        assert L.launch_count() - n0 == 2 * nb   # one launch per batch
    finally:
        tr.close()
        va.close()


@pytest.mark.parametrize("name", list(MG.CASES))
def test_golden_cases_are_bit_identical(name):
    case = MG.CASES[name]
    patch, final, B, osp, seed, nb = case[7:13]
    _compare(MG.case_arrays(name), B, patch, final, MG.label_manager(case), osp, seed, nb,
             regions=case[4], ignore=case[3])


@pytest.mark.parametrize("seed", range(8))
def test_seeded_sweeps_are_bit_identical(seed):
    r = np.random.RandomState(200 + seed)
    ignore = 4 if seed % 2 else None
    regions = [(1, 2, 3), (2, 3), (3,)] if seed % 4 == 3 else None
    labels = [1, 2, 3] if regions else ([1, 2, 130] if seed % 4 == 2 else [1, 2])
    dtype = np.int16 if 130 in labels else np.int8
    C = 1 + seed % 2
    cases = {f"s{i}": DO.ct_like_case(C, int(r.randint(1, 6)), int(r.randint(20, 150)), int(r.randint(20, 150)),
                                      labels, 70 * seed + i, dtype, empty=(i == 3), ignore_label=ignore,
                                      regions=regions)
             for i in range(5)}
    final = (int(r.randint(16, 120)), int(r.randint(16, 120)) | (seed % 3 == 0))   # odd, 2 mod 4 and 0 mod 4 rows
    patch = (final[0] + int(r.randint(0, 30)), final[1] + 2 * int(r.randint(0, 15)))
    lm = SimpleNamespace(all_labels=[0] + labels, has_ignore_label=ignore is not None)
    B, osp = int(r.randint(1, 12)), float(r.choice([0.0, 0.33, 0.5, 1.0]))
    _compare(cases, B, patch, final, lm, osp, seed, 3, regions=regions, ignore=ignore)


def test_same_seed_same_sequence():
    cases = MG.case_arrays("ignore_b3")
    lm = MG.label_manager(MG.CASES["ignore_b3"])
    ds = DO.ArrayDataset(sorted(cases.items()))
    a = DL.DeviceDataLoader2D(ds, 4, (40, 44), (32, 36), lm, 0.33, seed=11, device=DEV)
    b = DL.DeviceDataLoader2D(ds, 4, (40, 44), (32, 36), lm, 0.33, seed=11, device=DEV)
    try:
        for _ in range(6):
            x, y = next(a), next(b)
            assert list(x["keys"]) == list(y["keys"])
            assert torch.equal(x["data"], y["data"]) and torch.equal(x["target"], y["target"])
    finally:
        a.close()
        b.close()


# ------------------------------------------------------------------------------------------------ stand-in trainer
PATCH = (128, 128)


def _net(state_dict):
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 1, 3, None,
                                             "dinounet_s")
    net.load_state_dict(state_dict, strict=True)
    return net.to(DEV)


def _reset(tr, state_dict):
    tr.network = _net(state_dict).train()
    tr.optimizer = FusedSGD(tr.network.parameters(), lr=1e-2, weight_decay=3e-5, momentum=0.99, max_norm=12.0)


def _trainer(net, datasets):
    initial = tuple(int(v) for v in A.initial_patch_size_2d(PATCH))
    lm = SimpleNamespace(all_labels=[0, 1, 2], has_ignore_label=False, has_regions=False, foreground_regions=None,
                         ignore_label=None, foreground_labels=[1, 2])
    tr = TR.DinoUNetTrainer_s.__new__(TR.DinoUNetTrainer_s)
    tr.network, tr.device, tr.is_ddp, tr.local_rank = net, DEV, False, 0
    tr.loss = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, weight_ce=1,
                             weight_dice=1)
    tr.optimizer = FusedSGD(net.parameters(), lr=1e-2, weight_decay=3e-5, momentum=0.99, max_norm=12.0)
    tr.label_manager = lm
    tr.configuration_manager = SimpleNamespace(patch_size=list(PATCH), use_mask_for_norm=[False])
    tr.configure_rotation_dummyDA_mirroring_and_inital_patch_size = \
        lambda: (A.rotation_for_da_2d(PATCH), False, initial, (0, 1))
    tr.get_tr_and_val_datasets = lambda: datasets
    tr.batch_size, tr.oversample_foreground_percent = 2, 0.33
    tr._device_augmentation_seed, tr._device_dataloading_seed = 5, 9
    return tr, initial, lm


def _cases(n, seed):
    return DO.ArrayDataset(sorted((f"c{i}", DO.ct_like_case(1, 3, 150 + 10 * i, 170 - 10 * i, [1, 2], seed + i))
                                  for i in range(n)))


def test_trainer_steps_on_device_batches_equal_the_host_route(monkeypatch):
    monkeypatch.setattr(TR.DinoUNetTrainer, "_device_augmentation", True)
    monkeypatch.setattr(TR.DinoUNetTrainer, "_device_dataloading", True)
    sd = O.make_state_dict("dinounet_s", 3, seed=0)
    ds_tr, ds_val = _cases(3, 10), _cases(2, 20)
    dev_tr, initial, lm = _trainer(_net(sd).train(), (ds_tr, ds_val))
    host_tr, _, _ = _trainer(_net(sd).train(), (ds_tr, ds_val))
    dl_tr, dl_val = dev_tr.get_dataloaders()
    assert isinstance(dl_tr, DL.DeviceDataLoader2D) and isinstance(dl_val, DL.DeviceDataLoader2D)
    assert dl_tr.patch_size == initial and dl_val.patch_size == PATCH and dl_val.mode == "val"
    dev_tr.dataloader_train, dev_tr.dataloader_val = dl_tr, dl_val
    seeds = [int(np.random.SeedSequence(9, spawn_key=(0, i)).generate_state(1)[0]) for i in (0, 1)]
    rng_tr, rng_val = np.random.RandomState(seeds[0]), np.random.RandomState(seeds[1])
    try:
        for step in range(2):
            _reset(dev_tr, sd)
            _reset(host_tr, sd)
            batch = next(dl_tr)
            want, _ = DO.generate_train_batch(ds_tr, 2, initial, PATCH, [0, 1, 2], False, 0.33, rng_tr)
            host = TR.PassThroughTransforms()(data=want["data"], seg=want["seg"])
            host = {k: host[k].to(DEV) for k in ("data", "target")}
            assert torch.equal(batch["data"], host["data"]) and torch.equal(batch["target"], host["target"])
            got = dev_tr.train_step(batch)["loss"]
            ref = host_tr.train_step(host)["loss"]
            print(f"step {step}: loss {float(got):.7f} (device loader) {float(ref):.7f} (host route)")
            assert np.asarray(got).tobytes() == np.asarray(ref).tobytes(), step
        dev_tr.network.eval()
        batch = next(dl_val)
        want, _ = DO.generate_train_batch(ds_val, 2, PATCH, PATCH, [0, 1, 2], False, 0.33, rng_val)
        host = {"data": torch.from_numpy(want["data"]), "target": torch.from_numpy(DO.val_target(want["seg"]))}
        got, ref = dev_tr.validation_step(batch), dev_tr.validation_step(host)
        assert float(got["loss"]) == float(ref["loss"])
        for key in ("tp_hard", "fp_hard", "fn_hard"):
            assert np.array_equal(np.asarray(got[key]), np.asarray(ref[key])), key
    finally:
        dev_tr.on_train_end()
    assert not any(t.name == "DeviceDataLoader2D" and t.is_alive() for t in threading.enumerate())
    assert not dl_tr._thread.is_alive() and not dl_val._thread.is_alive()
