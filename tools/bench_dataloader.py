"""The 2-D device loader (dataloading.DeviceDataLoader2D) on CT-like preprocessed cases, at the trainer's setup:

    python tools/bench_dataloader.py [--cases 16] [--slices 48] [--batch 32] [--patch 512] [--batches 30] [--steps 10]

Writes seeded cases (1 x slices x 512 x 512, unpacked `.npy` data and int8 seg plus a `.pkl` with class locations, as
the reference's unpacked dataset) into a temporary directory, removed at the end, and reads them back with
`np.load(mmap_mode='r')` as `nnUNetDataset.load_case` does.  Batch 32, patch 512 (initial 602), oversample 0.33:

* device loader: batches per second seen by a consumer that only calls `next()` and synchronises (after 3 warm-up
  batches), the read-ahead thread's host time per batch (draws, loads, copies into the pinned slot), how often the
  consumer found the queue empty, and the pinned bytes; the H2D copy and the `b2u_dl_crop` kernel of one staged batch
  timed apart with CUDA events (median of 20);
* the reference's algorithm (oracle/dataloader_oracle.py) in this one process, then `PassThroughTransforms` and
  `.to(device)`, per batch.  A single-process restatement, not a measurement of the reference's multi-process
  augmenter;
* a dinounet_b training step at the same batch (device augmentation, TF32 tier, extractors recomputed in the backward)
  fed by the device loader against the same step on a batch already on the device, alternated, median of --steps
  after two warm-ups: what the loader costs the step, including the read-ahead thread's contention for the GIL.

Prints one JSON line with the card's name and power limit and the CPU model, read in the same run."""
import argparse
import json
import os
import pickle
import shutil
import statistics
import sys
import tempfile
import time
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dinounet_b200 import augmentation as A  # noqa: E402
from dinounet_b200 import dataloading as DL  # noqa: E402
from dinounet_b200 import lib as L  # noqa: E402
from dinounet_b200.training import PassThroughTransforms  # noqa: E402
from oracle import dataloader_oracle as DO  # noqa: E402
from tools.bench_evaluation import cpu_info, gpu_info  # noqa: E402


class NpyDataset:
    """nnUNetDataset.load_case on unpacked cases: `<key>.npy`, `<key>_seg.npy` (memory-mapped), `<key>.pkl`."""

    def __init__(self, folder, keys):
        self.folder, self._keys = folder, sorted(keys)

    def keys(self):
        return list(self._keys)

    def load_case(self, key):
        f = os.path.join(self.folder, str(key))
        with open(f + ".pkl", "rb") as fh:
            props = pickle.load(fh)
        return np.load(f + ".npy", mmap_mode="r"), np.load(f + "_seg.npy", mmap_mode="r"), props


def write_cases(folder, n, Z, S, seed):
    """CT-like cases: a body disc (label 0 inside, -1 outside), two organs drifting over the slices (1, 2)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:S, 0:S].astype(np.float32) / S - 0.5
    for i in range(n):
        seg = np.full((Z, S, S), -1, np.int8)
        for z in range(Z):
            seg[z][yy ** 2 + xx ** 2 < 0.2] = 0
            for lab, (cy, cx, r) in ((1, (0.1, -0.1, 0.12)), (2, (-0.12, 0.1, 0.06))):
                dz = (z - Z / 2) / Z
                seg[z][(yy - cy - 0.1 * dz) ** 2 + (xx - cx) ** 2 < (r * (1 - dz * dz)) ** 2] = lab
        data = (seg.astype(np.float32) * 0.8 + rng.standard_normal(seg.shape, dtype=np.float32) * 0.2)[None]
        data[:, seg < 0] = 0
        locs = {}
        for lab in (1, 2):
            rows = np.argwhere(seg[None] == lab)
            take = min(len(rows), max(5000, int(np.ceil(len(rows) * 0.01))))
            locs[lab] = rows[np.sort(rng.choice(len(rows), take, replace=False))] if len(rows) else []
        k = os.path.join(folder, f"case_{i:03d}")
        np.save(k + ".npy", data)
        np.save(k + "_seg.npy", seg[None])
        with open(k + ".pkl", "wb") as fh:
            pickle.dump({"class_locations": locs}, fh)
    return [f"case_{i:03d}" for i in range(n)]


def loader_rates(ds, B, initial, patch, lm, n, dev):
    dl = DL.DeviceDataLoader2D(ds, B, initial, patch, lm, 0.33, seed=0, device=dev)
    try:
        for _ in range(3):
            next(dl)
        torch.cuda.synchronize()
        s0 = dict(dl.stats)
        t0 = time.perf_counter()
        for _ in range(n):
            next(dl)
            torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        s1 = dict(dl.stats)
    finally:
        dl.close()
    return {"batches_per_s": n / dt, "ms_per_batch": 1e3 * dt / n,
            "thread_host_ms_per_batch": 1e3 * (s1["host_s"] - s0["host_s"]) / n,
            "consumer_waits": s1["waits"] - s0["waits"], "consumer_wait_ms_per_batch": 1e3 * (s1["wait_s"] - s0["wait_s"]) / n,
            "pinned_bytes": DL.SLOTS * dl.slot_bytes, "slot_bytes": dl.slot_bytes}


def copy_and_kernel(ds, B, initial, patch, lm, dev, reps=20):
    dl = DL.DeviceDataLoader2D(ds, B, initial, patch, lm, 0.33, seed=1, device=dev)
    pinned = torch.empty(dl.slot_bytes, dtype=torch.uint8, pin_memory=True)
    _, samples = dl.draw()
    nbytes = dl._stage(pinned.numpy(), samples)
    staged = torch.empty(dl.slot_bytes, dtype=torch.uint8, device=dev)
    H, W = dl.patch_size
    data = torch.empty((B, 1, H, W), dtype=torch.float32, device=dev)
    target = torch.empty((B, 1, H, W), dtype=torch.int16, device=dev)
    stream = torch.cuda.current_stream(dev)
    t_copy, t_kernel = [], []
    for _ in range(reps + 3):
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record()
        staged[:nbytes].copy_(pinned[:nbytes], non_blocking=True)
        e[1].record()
        L.check(L.load().b2u_dl_crop(staged.data_ptr(), staged.data_ptr(), B, 1, H, W, 0, None, 0, data.data_ptr(),
                                     target.data_ptr(), stream.cuda_stream), "b2u_dl_crop")
        e[2].record()
        e[2].synchronize()
        t_copy.append(e[0].elapsed_time(e[1]))
        t_kernel.append(e[1].elapsed_time(e[2]))
    written = data.numel() * 4 + target.numel() * 2
    read = nbytes
    k = statistics.median(t_kernel[3:])
    c = statistics.median(t_copy[3:])
    return {"staged_bytes": nbytes, "h2d_ms": c, "h2d_GBps": nbytes / c / 1e6, "kernel_ms": k,
            "kernel_bytes": written + read, "kernel_GBps": (written + read) / k / 1e6}


def oracle_route(ds, B, initial, patch, n, dev):
    rng = np.random.RandomState(0)
    times = []
    for _ in range(n):
        t0 = time.perf_counter()
        batch, _ = DO.generate_train_batch(ds, B, initial, patch, [0, 1, 2], False, 0.33, rng)
        b = PassThroughTransforms()(data=batch["data"], seg=batch["seg"])
        b["data"].to(dev), b["target"].to(dev)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return {"ms_per_batch": 1e3 * statistics.median(times), "batches": n}


def train_steps(ds, B, initial, patch, lm, steps, dev):
    import dinounet_b200
    from dinounet_b200 import config
    from dinounet_b200.loss import DC_and_CE_loss
    from dinounet_b200.train_path import FusedSGD, train_step
    os.environ.setdefault("DINOUNET_B200_ALLOW_RANDOM_BACKBONE", "1")
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 1, 3, None,
                                             "dinounet_b").to(dev).train()
    net.train_gemm, net.train_recompute = "tf32", True
    crit = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, weight_ce=1,
                          weight_dice=1)
    opt = FusedSGD(net.parameters(), lr=1e-4)
    aug = A.DeviceTrainingAugmentation(patch, seed=0)
    dl = DL.DeviceDataLoader2D(ds, B, initial, patch, lm, 0.33, seed=2, device=dev)
    fixed = next(dl)
    fixed = (fixed["data"].clone(), fixed["target"].clone())
    times = {"device_loader": [], "resident_batch": []}
    try:
        for i in range(2 + steps):
            for route in times:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if route == "device_loader":
                    b = next(dl)
                    x, t = b["data"], b["target"]
                else:
                    x, t = fixed
                x, t = aug(x, t)
                float(train_step(net, crit, opt, x, t))
                torch.cuda.synchronize()
                if i >= 2:
                    times[route].append(1e3 * (time.perf_counter() - t0))
    finally:
        dl.close()
    med = {k: statistics.median(v) for k, v in times.items()}
    return {"model": "dinounet_b", "tier": "tf32", "recompute": True, "steps": steps,
            "ms_device_loader": med["device_loader"], "ms_resident_batch": med["resident_batch"],
            "loader_cost_ms": med["device_loader"] - med["resident_batch"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", type=int, default=16)
    ap.add_argument("--slices", type=int, default=48)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--patch", type=int, default=512)
    ap.add_argument("--batches", type=int, default=30)
    ap.add_argument("--oracle-batches", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    dev = torch.device("cuda:0")
    patch = (a.patch, a.patch)
    initial = tuple(int(v) for v in A.initial_patch_size_2d(patch))
    lm = SimpleNamespace(all_labels=[0, 1, 2], has_ignore_label=False)
    tmp = tempfile.mkdtemp(prefix="bench_dataloader_")
    try:
        t0 = time.perf_counter()
        keys = write_cases(tmp, a.cases, a.slices, a.patch, 0)
        setup_s = time.perf_counter() - t0
        ds = NpyDataset(tmp, keys)
        out = {"bench": "dataloader", "gpu": gpu_info(), **cpu_info(), "batch": a.batch, "patch": list(patch),
               "initial_patch": list(initial), "oversample": 0.33, "cases": a.cases, "slices": a.slices,
               "queue_depth": DL.QUEUE_DEPTH, "slots": DL.SLOTS, "setup_s": setup_s}
        out["device_loader"] = loader_rates(ds, a.batch, initial, patch, lm, a.batches, dev)
        out["device_copy_and_kernel"] = copy_and_kernel(ds, a.batch, initial, patch, lm, dev)
        out["oracle_single_process_restatement"] = oracle_route(ds, a.batch, initial, patch, a.oracle_batches, dev)
        out["train_step"] = train_steps(ds, a.batch, initial, patch, lm, a.steps, dev)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
