"""Device keep-the-largest-component postprocessing (postprocessing.remove_all_but_largest_component_from_segmentation)
against the CPU route (oracle/postprocessing_oracle.py: scipy.ndimage.label with full connectivity and a bincount, as
acvl-utils does with skimage) on a seeded CT-like case:

    python tools/bench_postprocessing.py [--shape 200 512 512] [--reps 10] [--no-cpu]

The case (uint8): three ellipsoid labels, a large fragmented structure of label 2 (spheres along a curve with gaps), and
scattered false-positive blobs of every label.  Device time: CUDA events around one call on a volume already on the
device (median of --reps after two warm-ups), for the foreground union (the first step of determine_postprocessing) and
for each label; the host->device copy of the volume is timed separately.  Peak extra device memory: the allocator's peak
during a call above what was allocated before it, less the output volume.  The CPU route runs once per call, in this
process.  Prints one JSON line with both routes, their agreement, the CPU model and thread count, and the card's name and
power limit read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dinounet_b200 import postprocessing as PP  # noqa: E402
from oracle import postprocessing_oracle as PO  # noqa: E402
from tools.bench_evaluation import cpu_info, gpu_info  # noqa: E402

LABELS = [1, 2, 3]
# label: centre and radii as fractions of the shape
ELLIPSOIDS = [(1, (0.45, 0.5, 0.45), (0.35, 0.3, 0.25)), (3, (0.5, 0.45, 0.55), (0.15, 0.12, 0.1)),
              (2, (0.1, 0.65, 0.35), (0.08, 0.08, 0.09))]


def make_case(shape, seed: int = 0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    zz, yy, xx = (np.arange(s, dtype=np.float32) for s in shape)
    seg = np.zeros(shape, np.uint8)
    for lab, c, r in ELLIPSOIDS:
        cz, cy, cx = (ci * s for ci, s in zip(c, shape))
        rz, ry, rx = (ri * s for ri, s in zip(r, shape))
        sl = tuple(slice(max(0, int(ci - ri) - 1), min(s, int(ci + ri) + 2)) for ci, ri, s in
                   zip((cz, cy, cx), (rz, ry, rx), shape))
        inside = (((zz[sl[0], None, None] - cz) / rz) ** 2 + ((yy[None, sl[1], None] - cy) / ry) ** 2
                  + ((xx[None, None, sl[2]] - cx) / rx) ** 2) <= 1.0
        seg[sl][inside] = lab
    # a fragmented structure of label 2: spheres along a curve, every seventh left out
    for k, t in enumerate(np.linspace(0.05, 0.95, 160)):
        if k % 7 == 3:
            continue
        c = np.array([t * shape[0], (0.2 + 0.6 * t) * shape[1], (0.5 + 0.35 * np.sin(6 * t)) * shape[2]])
        rad = 2.0 + 4.0 * rng.random()
        sl = tuple(slice(max(0, int(ci - rad)), min(s, int(ci + rad) + 1)) for ci, s in zip(c, shape))
        d = ((zz[sl[0], None, None] - c[0]) ** 2 + (yy[None, sl[1], None] - c[1]) ** 2
             + (xx[None, None, sl[2]] - c[2]) ** 2) <= rad ** 2
        seg[sl][d & (seg[sl] == 0)] = 2
    # scattered false positives
    for _ in range(400):
        lab = int(rng.integers(1, 4))
        size = rng.integers(1, 5, 3)
        p = [int(rng.integers(0, s - e)) for s, e in zip(shape, size)]
        box = tuple(slice(a, a + e) for a, e in zip(p, size))
        seg[box][seg[box] == 0] = lab
    return seg


def time_device(seg_d, lr, reps):
    for _ in range(2):
        PP.remove_all_but_largest_component_from_segmentation(seg_d, lr)
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        PP.remove_all_but_largest_component_from_segmentation(seg_d, lr)
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times)), times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", type=int, nargs=3, default=[200, 512, 512])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--no-cpu", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the device route needs a GPU"
    shape = tuple(args.shape)
    seg = make_case(shape)
    out = {"shape": list(shape), "dtype": "uint8", "gpu": gpu_info(), **cpu_info(), "calls": {}}

    torch.cuda.synchronize()
    host = torch.from_numpy(seg)
    ups = []
    for _ in range(3):
        t0 = time.perf_counter()
        seg_d = host.to("cuda")
        torch.cuda.synchronize()
        ups.append((time.perf_counter() - t0) * 1e3)
    out["upload_ms"] = float(np.median(ups))

    calls = [("foreground", LABELS)] + [(f"label_{lab}", lab) for lab in LABELS]
    agree = True
    for name, lr in calls:
        ms, all_ms = time_device(seg_d, lr, args.reps)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        got = PP.remove_all_but_largest_component_from_segmentation(seg_d, lr)
        torch.cuda.synchronize()
        extra = torch.cuda.max_memory_allocated() - base - got.numel() * got.element_size()
        rec = {"device_ms": round(ms, 3), "device_ms_all": [round(t, 3) for t in all_ms],
               "peak_extra_device_bytes": int(extra), "removed_voxels": int((got != seg_d).sum())}
        if not args.no_cpu:
            t0 = time.perf_counter()
            want = PO.remove_all_but_largest_component_from_segmentation(seg, lr)
            rec["cpu_s"] = round(time.perf_counter() - t0, 3)
            rec["equal"] = bool(np.array_equal(got.cpu().numpy(), want))
            agree &= rec["equal"]
        out["calls"][name] = rec
    out["agree"] = agree if not args.no_cpu else None
    out["voxels"] = int(seg.size)
    out["two_int32_volumes_bytes"] = int(8 * seg.size)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
