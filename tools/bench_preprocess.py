"""Device preprocessing (DevicePreprocessor.run_case_npy) against the reference's CPU arithmetic (numpy normalization +
scipy's order-3 zoom with skimage's clip, the same calls run_case_npy makes), per case:

    python tools/bench_preprocess.py [--reps 10] [--cpu-slices 10] [--no-sw]

Device time: CUDA events around run_case_npy on data already on the device (median of --reps after one warm-up); the
host->device copy of the raw case is timed separately.  The CPU path is timed on --cpu-slices slices and reported per
slice.  For scale, the sliding window (dinounet_s, random weights, 4 mirror variants, 512^2 patches) on the same
preprocessed case.  Prints one JSON line per case, with the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dinounet_b200 import preprocess as PP  # noqa: E402

CASES = [  # name, data [C, X, Y, Z], spacing, configuration spacing, scheme: 100 x 256^2 -> 512^2 per slice,
    # 100 x 700^2 -> 512^2 as one 3-D resize (near-isotropic spacing), an RGB 1024 x 768 image
    ("slices_256_to_512", (1, 100, 256, 256), [3.0, 1.0, 1.0], [0.5, 0.5], "ZScoreNormalization"),
    ("volume_700_to_512", (1, 100, 700, 700), [1.0, 0.7, 0.7], [700 * 0.7 / 512, 700 * 0.7 / 512], "ZScoreNormalization"),
    ("rgb_1024x768", (3, 1, 768, 1024), [999.0, 1.0, 1.0], [768 / 512, 1024 / 512], "RGBTo01Normalization"),
]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def managers(C, cfg_spacing, scheme):
    conf = {"preprocessor_name": "DefaultPreprocessor", "resampling_fn_data": PP.DEFAULT_RESAMPLING_FN,
            "resampling_fn_data_kwargs": dict(PP.DEFAULT_RESAMPLING_KWARGS)}
    cm = SimpleNamespace(spacing=list(cfg_spacing), normalization_schemes=[scheme] * C, use_mask_for_norm=[False] * C,
                         configuration=conf, patch_size=[512, 512])
    pm = SimpleNamespace(transpose_forward=[0, 1, 2], foreground_intensity_properties_per_channel={})
    return pm, cm


def cpu_reference(data, spacing, cfg_spacing, scheme):
    """run_case_npy's arithmetic on the host (numpy + scipy), seconds per slice."""
    import scipy.ndimage as ndi
    t0 = time.perf_counter()
    x = data.astype(np.float32)
    for c in range(x.shape[0]):
        if scheme == "ZScoreNormalization":
            x[c] = (x[c] - x[c].mean()) / max(x[c].std(), 1e-8)
        else:
            x[c] = x[c] / np.float32(255.0)
    new = PP.compute_new_shape(x.shape[1:], spacing, [spacing[0], *cfg_spacing])
    path = PP.resampling_path(x.shape[1:], new, spacing, [spacing[0], *cfg_spacing])
    for c in range(x.shape[0]):
        v = x[c].astype(float)
        if path == "3d":
            o = ndi.zoom(v, np.divide(new, v.shape), order=3, mode="nearest", grid_mode=True)
            np.clip(o, v.min(), v.max(), out=o)
        else:
            for z in range(v.shape[0]):
                o = ndi.zoom(v[z], np.divide(new[1:], v.shape[1:]), order=3, mode="nearest", grid_mode=True)
                np.clip(o, v[z].min(), v[z].max(), out=o)
    return (time.perf_counter() - t0) / data.shape[1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--cpu-slices", type=int, default=10)
    ap.add_argument("--no-sw", action="store_true")
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    info = gpu_info()
    rng = np.random.default_rng(0)
    for name, shape, spacing, cfg_spacing, scheme in CASES:
        if scheme == "RGBTo01Normalization":
            data = rng.integers(0, 256, size=shape).astype(np.float32)
        else:
            data = (rng.standard_normal(shape) * 100 + 40).astype(np.float32)
        pm, cm = managers(shape[0], cfg_spacing, scheme)
        pre = PP.DevicePreprocessor(device=dev)
        host = torch.from_numpy(data).pin_memory()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        h2d = []
        for _ in range(3):
            e0.record()
            xd = host.to(dev, non_blocking=True)
            e1.record()
            torch.cuda.synchronize()
            h2d.append(e0.elapsed_time(e1))
        times = []
        for r in range(a.reps + 1):
            e0.record()
            out, _ = pre.run_case_npy(xd, None, {"spacing": list(spacing)}, pm, cm, {})
            e1.record()
            torch.cuda.synchronize()
            if r:
                times.append(e0.elapsed_time(e1))
        k = min(a.cpu_slices, shape[1])
        cpu_s = cpu_reference(data[:, :k], spacing, cfg_spacing, scheme)
        res = {"case": name, "shape": list(shape), "out": list(out.shape), "gpu": info,
               "device_ms_median": float(np.median(times)), "device_ms_min": float(np.min(times)),
               "h2d_ms_median": float(np.median(h2d)), "cpu_ms_per_slice": cpu_s * 1e3,
               "cpu_ms_extrapolated": cpu_s * 1e3 * shape[1], "cpu_slices_timed": k}
        if not a.no_sw:
            res["sliding_window_ms"] = sliding_window_ms(out, dev)
        print(json.dumps(res), flush=True)


def sliding_window_ms(data, dev):
    os.environ.setdefault("DINOUNET_B200_ALLOW_RANDOM_BACKBONE", "1")
    import dinounet_b200
    from dinounet_b200 import config
    from dinounet_b200.sliding_window import SlidingWindowPredictor
    net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, 2, None,
                                             "dinounet_s").to(dev).eval()
    p = SlidingWindowPredictor(tile_step_size=0.5, use_gaussian=True, use_mirroring=True, device=dev, tile_batch=8)
    p.manual_initialization(net, None, SimpleNamespace(patch_size=[512, 512]), None, {}, "bench", (0, 1))
    p.predict_sliding_window_return_logits(data)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    p.predict_sliding_window_return_logits(data)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


if __name__ == "__main__":
    main()
