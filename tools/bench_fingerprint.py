"""Dataset fingerprint on the device (DeviceFingerprintExtractor.run) against the CPU route in one process (the numpy
restatement of oracle/fingerprint_oracle.py: the reference's algorithm without its spawn pool), on a seeded CT-like
dataset held in memory:

    python tools/bench_fingerprint.py [--cases 20] [--shape 200 512 512] [--reps 3]

Cases: integer HU in [-1024, 3071] (air around a body of soft tissue and bone), labels 0..3 in a centred box.  The
reader hands out the preloaded arrays, so reading costs nothing on either route.  Device: wall time of `run()` ending
in its host reads (median, min and max of --reps after one warm-up run), and, separately, the host's RandomState draws
for the same foreground counts (`host_draws_s`), which run inside `run()`.  CPU: one run.  The two JSON texts are
compared.  Prints one JSON line with the card's name and power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dinounet_b200 import fingerprint as F  # noqa: E402
from dinounet_b200 import preprocess as PP  # noqa: E402
from oracle import fingerprint_oracle as FO  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def make_case(i: int, shape):
    rng = np.random.default_rng(100 + i)
    X, Y, Z = shape
    img = np.full(shape, -1024, np.int16)
    yy, zz = np.ogrid[:Y, :Z]
    body = ((yy - Y / 2) / (0.42 * Y)) ** 2 + ((zz - Z / 2) / (0.36 * Z)) ** 2 < 1
    img[:, body] = rng.integers(-150, 250, size=(X, int(body.sum())))
    bone = ((yy - Y / 2) / (0.08 * Y)) ** 2 + ((zz - Z / 2) / (0.08 * Z)) ** 2 < 1
    img[:, bone] = rng.integers(300, 3072, size=(X, int(bone.sum())))
    seg = np.zeros(shape, np.uint8)
    box = (slice(X // 8, 7 * X // 8), slice(Y // 3, 2 * Y // 3), slice(Z // 3, 2 * Z // 3))
    seg[box] = rng.integers(0, 4, size=[s.stop - s.start for s in box]).astype(np.uint8)
    return img[None].astype(np.float32), seg[None]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", type=int, default=20)
    ap.add_argument("--shape", type=int, nargs=3, default=[200, 512, 512])
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    t0 = time.perf_counter()
    cases = {f"case_{i:03d}": make_case(i, tuple(args.shape)) for i in range(args.cases)}
    gen_s = time.perf_counter() - t0

    class MemReader:
        def read_images(self, files):
            return cases[files[0]][0], {"spacing": [2.5, 0.75, 0.75]}

        def read_seg(self, file):
            return cases[file][1], {"spacing": [2.5, 0.75, 0.75]}

    with tempfile.TemporaryDirectory() as tmp:
        name = "Dataset990_Bench"
        os.makedirs(os.path.join(tmp, "raw", name))
        with open(os.path.join(tmp, "raw", name, "dataset.json"), "w") as f:
            json.dump({"channel_names": {"0": "CT"}, "labels": {"background": 0, "a": 1, "b": 2, "c": 3},
                       "file_ending": ".npy"}, f)
        PP._dataset_name = lambda x: x
        PP._raw_and_preprocessed = lambda: (os.path.join(tmp, "raw"), os.path.join(tmp, "pre"))
        PP._get_filenames_of_train_images_and_targets = lambda folder, dj: {k: {"images": [k], "label": k}
                                                                            for k in cases}
        F._determine_reader_writer = lambda dj, f: MemReader
        ext = F.DeviceFingerprintExtractor(name, num_processes=4)
        times = []
        for r in range(args.reps + 1):
            torch.cuda.synchronize()
            t = time.perf_counter()
            ext.run(overwrite_existing=True)
            torch.cuda.synchronize()
            if r:
                times.append(time.perf_counter() - t)
        with open(os.path.join(tmp, "pre", name, "dataset_fingerprint.json")) as f:
            device_json = f.read()

    num_samples = int(10e7 // len(cases))
    counts = [int(np.count_nonzero(seg[0] > 0)) for _, seg in cases.values()]
    t = time.perf_counter()
    for c in counts:
        F._draws(np.random.RandomState(F.SEED), c, 1, num_samples)
    draws_s = time.perf_counter() - t

    t = time.perf_counter()
    fp = FO.fingerprint([(seg, img) for img, seg in cases.values()], [[2.5, 0.75, 0.75]] * len(cases), 1)
    cpu_s = time.perf_counter() - t
    print(json.dumps({
        "gpu": gpu_info(), "cases": args.cases, "shape": args.shape, "samples_per_case": num_samples,
        "foreground_per_case": counts[0], "device_run_s_median": float(np.median(times)),
        "device_run_s_min": min(times), "device_run_s_max": max(times), "host_draws_s": draws_s,
        "cpu_route_s": cpu_s, "json_equal": FO.fingerprint_json(fp) == device_json, "data_gen_s": gen_s}))


if __name__ == "__main__":
    main()
