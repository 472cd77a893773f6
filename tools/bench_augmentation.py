"""Device training augmentation (augmentation.DeviceTrainingAugmentation) against the numpy / scipy restatement of
batchgenerators' pipeline (oracle/augmentation_oracle.py) on the trainer's 2-D setup:

    python tools/bench_augmentation.py [--batch 32] [--channels 1] [--patch 512] [--reps 20] [--no-cpu]

Seeded CT-like data with -1 padding (oracle.augmentation_oracle.ct_like) at the initial patch size (602 for 512).
Device time per batch: CUDA events around `__call__` (host sampling, record upload and the launches) on a batch
already on the device, median of --reps after three warm-ups.  Per-transform breakdown: torch.profiler with CUDA
activities in a separate pass over the same batches, every transform forced on, kernel time summed by step.  The CPU
route: the restatement on one batch with the same decisions, once, single process.  Prints one JSON line with the
card's name and power limit and the CPU model read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dinounet_b200 import augmentation as A  # noqa: E402
from oracle import augmentation_oracle as AO  # noqa: E402
from tools.bench_evaluation import cpu_info, gpu_info  # noqa: E402

STEPS = {"spatial": ("spatial_",), "noise": ("noise_kernel",), "blur": ("blur_",), "brightness+contrast+gamma":
         ("pointwise_", "tree_level", "stats_finalize", "minmax_kernel"), "lowres": ("lowres_",),
         "finalize": ("finalize_",)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--channels", type=int, default=1)
    ap.add_argument("--patch", type=int, default=512)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    patch = (a.patch, a.patch)
    h, w = (int(v) for v in A.initial_patch_size_2d(patch))
    data, seg = AO.ct_like(a.batch, a.channels, h, w, (h - a.patch) // 2, 0)
    dev = torch.device("cuda:0")
    x, s = torch.from_numpy(data).to(dev), torch.from_numpy(seg).to(dev)
    aug = A.DeviceTrainingAugmentation(patch, seed=0)
    for _ in range(3):
        aug(x, s)
    torch.cuda.synchronize()
    times = []
    for _ in range(a.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        aug(x, s)
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    # every transform on, for the breakdown
    rng = np.random.RandomState(1)
    p = A.AugmentationParams.identity(a.batch, a.channels)
    p.spatial[:] = p.rotate[:] = p.scale_on[:] = True
    p.angle[:] = rng.uniform(-np.pi, np.pi, a.batch)
    p.cos[:], p.sin[:] = np.cos(p.angle), np.sin(p.angle)
    p.scale[:] = rng.uniform(0.7, 1.4, a.batch)
    p.noise[:], p.noise_std[:] = True, 0.05
    p.blur_sigma[:] = 0.75
    p.brightness_on[:], p.contrast_on[:] = True, True
    p.lowres_shape[:] = np.round(np.array(patch) * 0.7).astype(int)
    p.gamma_on[:] = p.gamma_inv_on[:] = True
    p.gamma[:], p.gamma_inv[:] = 0.8, 1.2
    on_times = []
    for _ in range(a.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        aug.apply(x, s, p, 5)
        e1.record()
        e1.synchronize()
        on_times.append(e0.elapsed_time(e1))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            aug.apply(x, s, p, 5)
        torch.cuda.synchronize()
    steps = {k: 0.0 for k in STEPS}
    other = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        name = ev.key
        hit = [k for k, pats in STEPS.items() if any(pt in name for pt in pats)]
        if hit:
            steps[hit[0]] += t / 5 / 1000
        elif t:
            other += t / 5 / 1000
    res = {"setup": f"B={a.batch} C={a.channels} {h}x{w}->{a.patch}x{a.patch}", "gpu": gpu_info(),
           "device_ms_per_batch_sampled": float(np.median(times)),
           "device_ms_per_batch_sampled_range": [float(min(times)), float(max(times))],
           "device_ms_per_batch_all_on": float(np.median(on_times)),
           "kernel_ms_per_step_all_on": {k: round(v, 4) for k, v in steps.items()}, "kernel_ms_other": round(other, 4)}
    if not a.no_cpu:
        params = aug.sample(a.batch, a.channels)
        noise = A.noise_field(3, a.batch, a.channels, patch, dev).cpu().numpy()
        t0 = time.perf_counter()
        AO.augment(data, seg, params, noise, patch)
        res["cpu_restatement_s_per_batch"] = time.perf_counter() - t0
        res["cpu"] = cpu_info()
        res["torch_threads"] = torch.get_num_threads()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
