"""Device evaluation (evaluation.compute_metrics_arrays) against the CPU route (oracle/evaluation_oracle.py: numpy counts,
scipy erosion and distance_transform_edt, medpy's hd95 / asd restated) on a seeded CT-like case:

    python tools/bench_evaluation.py [--shape 200 512 512] [--spacing 2.5 0.78 0.78] [--reps 10] [--no-cpu]

The case: three ellipsoid labels (one touching the first slice) and a prediction with shifted centres and scaled radii,
uint8.  Device time: CUDA events around compute_metrics_arrays on volumes already on the device (median of --reps after
two warm-ups; it includes the per-label scalar copies to the host); the host->device copy of the two volumes is timed
separately.  The CPU route runs once, in this process.  Prints one JSON line with both routes, their agreement, the
CPU model and thread count, and the card's name and power limit read in the same run."""
import argparse
import json
import os
import platform
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dinounet_b200 import evaluation as EV  # noqa: E402
from oracle import evaluation_oracle as EO  # noqa: E402

LABELS = [1, 2, 3]
# label: centre and radii as fractions of the shape, and the prediction's shift (voxels) and radius scale
ELLIPSOIDS = [(1, (0.45, 0.5, 0.45), (0.35, 0.3, 0.25), (1, 3, -2), 1.04),
              (2, (0.5, 0.45, 0.55), (0.15, 0.12, 0.1), (0, -2, 2), 0.95),
              (3, (0.1, 0.65, 0.35), (0.2, 0.08, 0.09), (-1, 1, 1), 1.02)]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def cpu_info():
    model = platform.processor() or platform.machine()
    try:
        with open("/proc/cpuinfo") as f:
            model = next(line.split(":", 1)[1].strip() for line in f if line.startswith("model name"))
    except (OSError, StopIteration):
        pass
    return {"cpu": model, "cpu_threads": os.cpu_count(), "torch_threads": torch.get_num_threads()}


def make_case(shape):
    zz, yy, xx = (np.arange(s, dtype=np.float32) for s in shape)
    ref = np.zeros(shape, np.uint8)
    pred = np.zeros(shape, np.uint8)
    for lab, c, r, shift, scale in ELLIPSOIDS:
        for seg, dc, k in ((ref, (0, 0, 0), 1.0), (pred, shift, scale)):
            cz, cy, cx = (ci * s + d for ci, s, d in zip(c, shape, dc))
            rz, ry, rx = (ri * s * k for ri, s in zip(r, shape))
            inside = (((zz[:, None, None] - cz) / rz) ** 2 + ((yy[None, :, None] - cy) / ry) ** 2
                      + ((xx[None, None, :] - cx) / rx) ** 2) <= 1.0
            seg[inside] = lab
    return ref[None], pred[None]


def agreement(dev, cpu):
    out = {"counts_equal": True, "nan_equal": True, "max_rel_hd95_asd": 0.0}
    for r in cpu:
        for k, w in cpu[r].items():
            g = dev[r][k]
            if np.isnan(w) or np.isnan(g):
                out["nan_equal"] &= bool(np.isnan(w) and np.isnan(g))
            elif k in ("HD95", "ASD"):
                out["max_rel_hd95_asd"] = max(out["max_rel_hd95_asd"], abs(g - w) / abs(w) if w else abs(g))
            else:
                out["counts_equal"] &= bool(g == w)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", type=int, nargs=3, default=[200, 512, 512])
    ap.add_argument("--spacing", type=float, nargs=3, default=[2.5, 0.78, 0.78])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--no-cpu", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_evaluation needs a GPU")
    ref, pred = make_case(tuple(args.shape))
    spacing = tuple(args.spacing)
    res = {"case": "ct_like", "shape": args.shape, "spacing": spacing, "labels": LABELS, "gpu": gpu_info()}

    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ups = []
    for _ in range(3):
        ev0.record()
        ref_d, pred_d = torch.from_numpy(ref).cuda(), torch.from_numpy(pred).cuda()
        ev1.record()
        torch.cuda.synchronize()
        ups.append(ev0.elapsed_time(ev1))
    res["upload_ms"] = float(np.median(ups))

    for _ in range(2):
        dev = EV.compute_metrics_arrays(ref_d, pred_d, LABELS, None, spacing)
    times = []
    for _ in range(args.reps):
        torch.cuda.synchronize()
        ev0.record()
        dev = EV.compute_metrics_arrays(ref_d, pred_d, LABELS, None, spacing)
        ev1.record()
        torch.cuda.synchronize()
        times.append(ev0.elapsed_time(ev1))
    res["device_ms_median"] = float(np.median(times))
    res["device_ms_min_max"] = [float(min(times)), float(max(times))]
    res["peak_device_mb"] = torch.cuda.max_memory_allocated() / 2 ** 20
    res["device_metrics"] = {str(r): {k: float(v) for k, v in m.items()} for r, m in dev.items()}

    if not args.no_cpu:
        res.update(cpu_info())
        t0 = time.perf_counter()
        cpu = EO.compute_metrics_arrays(ref, pred, LABELS, None, spacing)
        res["cpu_s"] = time.perf_counter() - t0
        res["agreement"] = agreement(dev, cpu)
        res["speedup"] = res["cpu_s"] * 1e3 / res["device_ms_median"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
