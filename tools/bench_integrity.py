"""Dataset integrity check on the device against the reference's algorithm in one process, on a seeded CT-like raw
dataset written as `.npy` files (one file per channel, uint8 labels 0..3):

    python tools/bench_integrity.py [--cases 8] [--shape 200 512 512] [--reps 3]

(a) `integrity.verify_dataset_integrity` against oracle/integrity_oracle.py (the reference's verify without its spawn
    pool: `pd.unique` and `np.isnan` over every case, each case read twice);
(b) the fused `extract_fingerprint_dataset(check_dataset_integrity=True)` (one read of each case) against the device
    verify followed by the device fingerprint (`DeviceFingerprintExtractor.run`), alternated in this process;
(c) the `b2u_vi_scan` kernel on one case's device copy: CUDA-event time per launch, the bytes it reads (images and
    seg) over that time, and that rate over the H100 SXM data sheet's 3.35 TB/s.
Wall times are medians (and min / max) of --reps after one warm-up run; the fused and the two-pass routes' JSON texts
are compared.  Prints the card's name and power limit, read in the same run, then one JSON line."""
import argparse
import contextlib
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
from dinounet_b200 import integrity as I  # noqa: E402
from dinounet_b200 import lib as L  # noqa: E402
from dinounet_b200 import preprocess as PP  # noqa: E402
from oracle import integrity_oracle as IO  # noqa: E402
from oracle import make_golden_integrity as MI  # noqa: E402

DATA_SHEET_BYTES_PER_S = 3.35e12
NAME = "Dataset991_IntegrityBench"


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def make_case(i: int, shape):
    """CT-like: integer HU (air, soft tissue, bone) as float32 [1, X, Y, Z], labels 0..3 in a centred box (uint8)."""
    rng = np.random.default_rng(300 + i)
    X, Y, Z = shape
    img = np.full(shape, -1024, np.int16)
    yy, zz = np.ogrid[:Y, :Z]
    body = ((yy - Y / 2) / (0.42 * Y)) ** 2 + ((zz - Z / 2) / (0.36 * Z)) ** 2 < 1
    img[:, body] = rng.integers(-150, 250, size=(X, int(body.sum())))
    seg = np.zeros(shape, np.uint8)
    box = (slice(X // 8, 7 * X // 8), slice(Y // 3, 2 * Y // 3), slice(Z // 3, 2 * Z // 3))
    seg[box] = rng.integers(0, 4, size=[s.stop - s.start for s in box]).astype(np.uint8)
    return img.astype(np.float32), seg


def write_dataset(raw: str, cases: int, shape):
    folder = os.path.join(raw, NAME)
    for d in ("imagesTr", "labelsTr"):
        os.makedirs(os.path.join(folder, d))
    with open(os.path.join(folder, "dataset.json"), "w") as f:
        json.dump({"channel_names": {"0": "CT"}, "labels": {"background": 0, "a": 1, "b": 2, "c": 3},
                   "file_ending": ".npy", "numTraining": cases}, f)
    for i in range(cases):
        img, seg = make_case(i, shape)
        fi, fs = os.path.join(folder, "imagesTr", f"c{i:03d}_0000.npy"), os.path.join(folder, "labelsTr", f"c{i:03d}.npy")
        np.save(fi, img)
        np.save(fs, seg)
        MI.NpyGeoReader.SPACINGS[fi] = MI.NpyGeoReader.SPACINGS[fs] = [2.5, 0.75, 0.75]
    return folder


def timed(fn):
    with open(os.devnull, "w") as null, contextlib.redirect_stdout(null):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ret = fn()
        torch.cuda.synchronize()
    return time.perf_counter() - t0, ret


def stats(ts):
    return {"median_s": float(np.median(ts)), "min_s": float(min(ts)), "max_s": float(max(ts))}


def kernel_time(folder, reps: int = 50):
    img, seg = make_case(0, tuple(np.load(os.path.join(folder, "labelsTr", "c000.npy"), mmap_mode="r").shape))
    dev = torch.device("cuda", torch.cuda.current_device())
    s, x = I.upload(seg, img[None], 0, dev)
    out = torch.empty(2, dtype=torch.int64, device=dev)
    lib = L.load()
    st = torch.cuda.current_stream(dev).cuda_stream

    def launch():
        L.check(lib.b2u_vi_scan(x.data_ptr(), x.numel(), s.data_ptr(), 0, s.numel(), 0, 3, out.data_ptr(), st),
                "b2u_vi_scan")

    for _ in range(5):
        launch()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        launch()
    b.record()
    b.synchronize()
    t = a.elapsed_time(b) / 1e3 / reps
    nbytes = x.numel() * 4 + s.numel()
    return {"kernel_s": t, "bytes": int(nbytes), "bytes_per_s": nbytes / t,
            "fraction_of_3_35_TBps": nbytes / t / DATA_SHEET_BYTES_PER_S, "offenders": int(out[0])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", type=int, default=8)
    ap.add_argument("--shape", type=int, nargs=3, default=[200, 512, 512])
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_integrity measures the device: it needs a GPU"
    print(gpu_info(), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        raw, pre = os.path.join(tmp, "raw"), os.path.join(tmp, "pre")
        folder = write_dataset(raw, args.cases, tuple(args.shape))
        PP._dataset_name = lambda x: x
        PP._raw_and_preprocessed = lambda: (raw, pre)
        PP._get_filenames_of_train_images_and_targets = IO.get_filenames_of_train_images_and_targets
        F._determine_reader_writer = lambda dj, f: MI.NpyGeoReader
        I._label_manager = IO.LabelManager

        def device_verify():
            return I.verify_dataset_integrity(folder, 4)

        def oracle_verify():
            text, exc = IO.verify(folder, MI.NpyGeoReader)
            assert exc is None, exc
            return text

        def fused():
            I.extract_fingerprint_dataset(NAME, F.DeviceFingerprintExtractor, 4, True, True, False)
            with open(os.path.join(pre, NAME, "dataset_fingerprint.json")) as f:
                return f.read()

        def two_pass():
            I.verify_dataset_integrity(folder, 4)
            F.DeviceFingerprintExtractor(NAME, 4).run(overwrite_existing=True)
            with open(os.path.join(pre, NAME, "dataset_fingerprint.json")) as f:
                return f.read()

        timed(device_verify)
        dv = [timed(device_verify)[0] for _ in range(args.reps)]
        t_oracle, text = timed(oracle_verify)
        timed(fused)
        timed(two_pass)
        tf, tt, same = [], [], True
        for _ in range(args.reps):
            t, a = timed(fused)
            tf.append(t)
            t, b = timed(two_pass)
            tt.append(t)
            same = same and a == b
        result = {
            "gpu": gpu_info(), "cases": args.cases, "shape": args.shape,
            "a_device_verify": stats(dv), "a_oracle_verify_s": t_oracle,
            "a_speedup": t_oracle / float(np.median(dv)),
            "b_fused": stats(tf), "b_verify_then_fingerprint": stats(tt),
            "b_speedup": float(np.median(tt)) / float(np.median(tf)), "b_same_json": same,
            "c_scan": kernel_time(folder),
        }
    print(json.dumps(result))


if __name__ == "__main__":
    main()
