"""Prediction export, device route against the CPU route, at the sizes a user exports: C = 3 channels, 200 slices,
512x512 logits resampled to 384x384 and to 768x768, with and without probabilities.

    python tools/bench_export.py [--slices 200] [--repeats 20] [--cpu-repeats 1]

Device route: b2u_export_resample_f16 + b2u_export_segment + the device-to-host copy of the labels (and of the
probabilities when asked), timed with CUDA events after a warm-up, median over repeats; each kernel is also timed alone
and its bytes (resample: one fp16 read per input element and one fp16 write per output element; segment: one read
of every logit plus the label and probability writes) are set against the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s.
CPU route: the oracle restatement of the reference's chain (float64 resampling, fp16, softmax, argmax) on
the host, wall clock, with the thread count and CPU model printed.  The card's name and power limit are read in the
same run.
"""
import argparse
import json
import os
import platform
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dinounet_b200 import lib as L  # noqa: E402
from oracle import export_oracle as EO  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def _cpu_model():
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.startswith("model name"):
                    return line.split(":", 1)[1].strip()
    except OSError:
        pass
    return platform.processor() or "unknown"


def _events_median(fn, repeats):
    times = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slices", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--cpu-repeats", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_export measures the device route: it needs a GPU"
    lib = L.load()
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream(dev).cuda_stream
    C, Z, h, w = 3, args.slices, 512, 512
    print(f"card: {_card()}")
    print(f"host: {_cpu_model()}, torch threads {torch.get_num_threads()}")
    x = (torch.randn(C, Z, h, w, generator=torch.Generator().manual_seed(0)) * 4).half()
    xd = x.to(dev)
    for H in (384, 768):
        W = H
        vox = Z * H * W
        r = torch.empty((C, Z, H, W), dtype=torch.half, device=dev)
        labels = torch.empty(vox, dtype=torch.uint8, device=dev)
        labels_host = torch.empty(vox, dtype=torch.uint8, pin_memory=True)
        probs = torch.empty((C, vox), dtype=torch.float32, device=dev)
        probs_host = torch.empty((C, vox), dtype=torch.float32, pin_memory=True)

        def resample():
            L.check(lib.b2u_export_resample_f16(xd.data_ptr(), r.data_ptr(), C, Z, h, w, H, W, st))

        def segment(with_probs):
            L.check(lib.b2u_export_segment(r.data_ptr(), C, vox, 0, None, labels.data_ptr(), 1,
                                           probs.data_ptr() if with_probs else None, st))

        def route(with_probs):
            resample()
            segment(with_probs)
            labels_host.copy_(labels, non_blocking=True)
            if with_probs:
                probs_host.copy_(probs, non_blocking=True)

        for _ in range(3):
            route(True)
            route(False)
        torch.cuda.synchronize()
        t_res = _events_median(resample, args.repeats)
        res_bytes = C * Z * (h * w + H * W) * 2
        for with_probs in (False, True):
            t_seg = _events_median(lambda: segment(with_probs), args.repeats)
            seg_bytes = C * vox * 2 + vox + (C * vox * 4 if with_probs else 0)
            t_route = _events_median(lambda: route(with_probs), args.repeats)
            t_cpu = None
            if not with_probs:
                t0 = time.perf_counter()
                for _ in range(args.cpu_repeats):
                    for z0 in range(0, Z, 20):    # chunks of slices bound the host memory of the float64 temporaries
                        EO.nonlin_and_segment(EO.resample_f16(x[:, z0:z0 + 20], H, W), False)
                t_cpu = (time.perf_counter() - t0) / args.cpu_repeats * 1e3
            rec = {"shape": f"{C}x{Z}x{h}x{w}->{H}x{W}", "probabilities": with_probs,
                   "device_route_ms": round(t_route, 3), "resample_ms": round(t_res, 3),
                   "resample_GBps": round(res_bytes / t_res / 1e6, 1),
                   "resample_share_of_peak": round(res_bytes / (t_res * 1e-3) / PEAK_BYTES_PER_S, 3),
                   "segment_ms": round(t_seg, 3), "segment_GBps": round(seg_bytes / t_seg / 1e6, 1),
                   "segment_share_of_peak": round(seg_bytes / (t_seg * 1e-3) / PEAK_BYTES_PER_S, 3)}
            if t_cpu is not None:
                rec["cpu_route_ms"] = round(t_cpu, 1)
            print(json.dumps(rec))


if __name__ == "__main__":
    main()
