"""CPU: the 2-D device loader's host side (dinounet_b200/dataloading.py).

* The oracle (oracle/dataloader_oracle.py) reproduces the reference's own `nnUNetDataLoader2D` bit for bit on every
  golden case: keys, data and seg (tests/golden/dataloader_cases.npz, oracle/make_golden_dataloader.py).
* The loader's draws (keys, slices, boxes) equal the oracle's on the golden cases and on seeded sweeps, and the
  reference's errors come from the same draws.
* Every rejection happens in the constructor, before any native call (recording stand-in for the library).
* The trainer's `device_dataloading` switch.
* A pinned slot goes back to the read-ahead thread only after the event behind its launch has completed.
"""
import threading
import time
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dinounet_b200 import dataloading as DL
from dinounet_b200 import lib as L
from oracle import dataloader_oracle as DO
from oracle import make_golden_dataloader as MG

GOLDEN = np.load(__import__("os").path.join(__import__("os").path.dirname(__file__), "golden", "dataloader_cases.npz"))


def _loader(cases, B, patch, final, lm, osp, seed, **kw):
    return DL.DeviceDataLoader2D(DO.ArrayDataset(sorted(cases.items())), B, patch, final, lm, osp, seed=seed, **kw)


@pytest.mark.parametrize("name", list(MG.CASES))
def test_oracle_matches_the_reference_golden(name):
    case = MG.CASES[name]
    patch, final, B, osp, seed, nb = case[7:13]
    cases = MG.case_arrays(name)
    assert np.array_equal(MG.checksum(cases), GOLDEN[f"{name}_checksum"])
    lm = MG.label_manager(case)
    rng = np.random.RandomState(seed)
    ds = DO.ArrayDataset(sorted(cases.items()))
    for i in range(nb):
        batch, _ = DO.generate_train_batch(ds, B, patch, final, lm.all_labels, lm.has_ignore_label, osp, rng)
        assert list(batch["keys"]) == list(GOLDEN[f"{name}_{i}_keys"]), i
        assert batch["data"].dtype == np.float32 and batch["seg"].dtype == np.int16
        assert np.array_equal(batch["data"].view(np.int32), GOLDEN[f"{name}_{i}_data"].view(np.int32)), i
        assert np.array_equal(batch["seg"], GOLDEN[f"{name}_{i}_seg"]), i


def _draws_equal(loader, ds, B, patch, final, lm, osp, seed, nb):
    rng = np.random.RandomState(seed)
    for i in range(nb):
        batch, draws = DO.generate_train_batch(ds, B, patch, final, lm.all_labels, lm.has_ignore_label, osp, rng)
        keys, samples = loader.draw()
        assert list(keys) == list(batch["keys"]), i
        assert [(s.slice, list(s.bbox_lbs)) for s in samples] == draws, i
        assert all(tuple(s.bbox_ubs) == tuple(s.bbox_lbs[d] + patch[d] for d in range(2)) for s in samples)


@pytest.mark.parametrize("name", list(MG.CASES))
def test_loader_draws_equal_the_oracle_on_the_golden_cases(name):
    case = MG.CASES[name]
    patch, final, B, osp, seed, nb = case[7:13]
    cases = MG.case_arrays(name)
    lm = MG.label_manager(case)
    loader = _loader(cases, B, patch, final, lm, osp, seed)
    _draws_equal(loader, DO.ArrayDataset(sorted(cases.items())), B, patch, final, lm, osp, seed, nb)


@pytest.mark.parametrize("seed", range(6))
def test_loader_draws_equal_the_oracle_on_seeded_sweeps(seed):
    r = np.random.RandomState(100 + seed)
    ignore = 4 if seed % 2 else None
    labels = [1, 2, 3][: 1 + seed % 3]
    cases = {f"k{i}": DO.ct_like_case(1 + seed % 2, int(r.randint(1, 5)), int(r.randint(12, 60)),
                                      int(r.randint(12, 60)), labels, 50 * seed + i, np.int8,
                                      empty=(i == 2 and ignore is None), ignore_label=ignore)
             for i in range(4)}
    final = (int(r.randint(8, 40)), int(r.randint(8, 40)))
    patch = (final[0] + int(r.randint(0, 12)), final[1] + int(r.randint(0, 12)))
    lm = SimpleNamespace(all_labels=[0] + labels, has_ignore_label=ignore is not None)
    B, osp = int(r.randint(1, 9)), float(r.choice([0.0, 0.33, 0.5, 1.0]))
    loader = _loader(cases, B, patch, final, lm, osp, seed)
    _draws_equal(loader, DO.ArrayDataset(sorted(cases.items())), B, patch, final, lm, osp, seed, 4)


def test_python_round_decides_oversampling():
    """round(5 * 0.5) = 2 (banker's rounding): samples 2, 3 and 4 of a batch of 5 are foreground-forced."""
    cases = MG.case_arrays("round_b5")
    lm = MG.label_manager(MG.CASES["round_b5"])
    loader = _loader(cases, 5, (40, 40), (32, 32), lm, 0.5, 0)
    assert [not j < round(5 * (1 - 0.5)) for j in range(5)] == [False, False, True, True, True]
    keys, samples = loader.draw()
    for s in samples[2:]:   # every forced sample of a case with foreground holds a voxel of a class in its box
        if not any(len(v) for v in s.properties["class_locations"].values()):
            continue
        lo, hi = s.bbox_lbs, s.bbox_ubs
        seg = s.seg[0, s.slice]
        window = seg[max(0, lo[0]):max(0, hi[0]), max(0, lo[1]):max(0, hi[1])]
        assert (window > 0).any()


def test_reference_errors_come_from_the_same_draws():
    """An ignore-label dataset whose all-labels key has no rows: the reference's choice() raises ValueError."""
    data, seg, props = DO.ct_like_case(1, 2, 20, 20, [1], 0, np.int8, ignore_label=2)
    key = (0, 1)
    props["class_locations"][key] = np.zeros((0, 4), np.int64)
    lm = SimpleNamespace(all_labels=[0, 1], has_ignore_label=True)
    loader = _loader({"a": (data, seg, props)}, 2, (16, 16), (16, 16), lm, 0.0, 0)
    with pytest.raises(ValueError):
        loader.draw()
    with pytest.raises(ValueError):
        DO.generate_train_batch(DO.ArrayDataset([("a", (data, seg, props))]), 2, (16, 16), (16, 16), [0, 1], True, 0.0,
                                np.random.RandomState(0))


class _Recorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*a):
            self.calls.append((name, a))
            return 0
        return fn


def _lm():
    return SimpleNamespace(all_labels=[0, 1], has_ignore_label=False)


@pytest.mark.parametrize("change, exc", [
    (dict(patch=(8, 16, 16), final=(8, 16, 16)), ValueError),
    (dict(seg_channels=2), ValueError),
    (dict(data_dtype=np.float64), TypeError),
    (dict(seg_dtype=np.int32), TypeError),
    (dict(seg_dtype=np.uint8), TypeError),
    (dict(B=65536), ValueError),
    (dict(sampling_probabilities=[1.0]), NotImplementedError),
    (dict(pad_sides=[1, 1]), NotImplementedError),
    (dict(probabilistic_oversampling=True), NotImplementedError),
    (dict(mode="test"), ValueError),
    (dict(regions=[(1,)]), ValueError),   # regions belong to val mode
])
def test_rejections_before_any_native_call(monkeypatch, change, exc):
    rec = _Recorder()
    monkeypatch.setattr(L, "load", lambda: rec)
    data, seg, props = DO.ct_like_case(1, 2, 20, 20, [1], 0, np.int8)
    data = data.astype(change.get("data_dtype", np.float32))
    seg = np.repeat(seg, change.get("seg_channels", 1), 0).astype(change.get("seg_dtype", np.int8))
    kw = {k: change[k] for k in ("sampling_probabilities", "pad_sides", "probabilistic_oversampling", "mode",
                                 "regions") if k in change}
    with pytest.raises(exc):
        DL.DeviceDataLoader2D(DO.ArrayDataset([("a", (data, seg, props))]), change.get("B", 2),
                              change.get("patch", (16, 16)), change.get("final", (16, 16)), _lm(), 0.33, **kw)
    assert rec.calls == []


def test_set_network_config_switch():
    from dinounet_b200 import config
    from dinounet_b200.training import DinoUNetTrainer, DinoUNetTrainer_s
    arch = {"architecture": dict(config.DEFAULT_ARCHITECTURE)}
    try:
        assert DinoUNetTrainer._device_dataloading is False
        with pytest.raises(ValueError, match="device_augmentation"):
            DinoUNetTrainer_s.set_network_config(arch, device_dataloading=True)
        with pytest.raises(ValueError, match="device_dataloading"):
            DinoUNetTrainer_s.set_network_config(arch, device_augmentation=True, device_dataloading=1)
        DinoUNetTrainer_s.set_network_config(arch, device_augmentation=True, device_dataloading=True)
        assert DinoUNetTrainer._device_dataloading is True and DinoUNetTrainer_s._device_dataloading is True
        DinoUNetTrainer_s.set_network_config(arch, device_augmentation=True)
        assert DinoUNetTrainer._device_dataloading is False
    finally:
        DinoUNetTrainer_s.set_network_config(None)


class _Event:
    def __init__(self):
        self.done = False

    def query(self):
        return self.done

    def synchronize(self):
        self.done = True


def test_a_slot_is_not_reused_before_its_event_completes(monkeypatch):
    cases = MG.case_arrays("labels_b2")
    lm = MG.label_manager(MG.CASES["labels_b2"])
    loader = _loader(cases, 2, (48, 40), (40, 32), lm, 0.33, 0, device="cpu")
    in_flight, events, staged = {}, [], []
    lock = threading.Lock()

    def alloc():
        host = [np.zeros(loader.slot_bytes, np.uint8) for _ in range(DL.SLOTS)]
        return None, host, None

    stage = loader._stage

    def checked_stage(buf, samples):
        slot = next(i for i, h in enumerate(loader._host) if h is buf)
        with lock:
            ev = in_flight.get(slot)
            assert ev is None or ev.done, f"slot {slot} restaged while its launch is in flight"
            staged.append(slot)
        return stage(buf, samples)

    def launch(slot, nbytes):
        ev = _Event()
        with lock:
            in_flight[slot] = ev
            events.append(ev)
        return None, None, ev

    monkeypatch.setattr(loader, "_alloc", alloc)
    monkeypatch.setattr(loader, "_stage", checked_stage)
    monkeypatch.setattr(loader, "_launch", launch)
    try:
        for _ in range(DL.SLOTS):
            next(loader)
        time.sleep(0.3)
        assert len(staged) == DL.SLOTS          # every slot in flight: the thread waits
        assert loader._free.qsize() == 0
        events[0].done = True
        next(loader)                            # releases slot 0 (completed) and takes the next batch
        deadline = time.time() + 5
        while len(staged) < DL.SLOTS + 1 and time.time() < deadline:
            time.sleep(0.01)
        assert staged[DL.SLOTS] == 0
        next(loader)                            # all slots in flight again: waits for the oldest, then reuses it
        assert events[1].done
    finally:
        loader.close()
    assert not loader._thread.is_alive()
