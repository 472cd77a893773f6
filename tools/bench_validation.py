"""The final validation of a training run (`DinoUNetTrainer.perform_actual_validation`) on the device, against the route
the inherited reference method takes with the native network: N seeded CT-like preprocessed cases (1 channel,
`--slices` slices of 512x512, exported to 460x460 at the original spacing), dinounet_s and dinounet_l, 3 classes.

    python tools/bench_validation.py [--cases 4] [--slices 24] [--baseline-cases 2]

Device route: a stand-in trainer (SimpleNamespace managers, `.npz` reader-writer: compressed files, as the image
writers' are) runs `perform_actual_validation` from the first case read to `summary.json`; wall clock after a
synchronise, after a warm-up call on one case.  Every call packs the network's current weights again, as the end of a
training run must, so the total and the first case's interval include that packing and the CUDA graph capture.
Reported: total, the median of the per-case intervals between the "predicting" log lines, and the time spent inside
`write_seg` (summed over the writer threads, whose file writing overlaps the next prediction) as a share of the
total.
Baseline route: the reference's loop - one 512x512 tile at a time through the native forward (batch 1, no mirroring,
fp16 accumulation in torch, oracle/sliding_window_oracle.py), the logits copied to the host, the export restated on
the host (float64 resampling, softmax, argmax: oracle/export_oracle.py) and the same writer; serial, wall clock per
case, the median over `--baseline-cases` (the mean of two for the default).  The reference runs its export in a
process pool, so this serial time per case is an upper bound of its own.
The card's name and power limit are read in the same run.
"""
import argparse
import os
import pickle
import statistics
import subprocess
import sys
import tempfile
import time
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import dinounet_b200  # noqa: E402
from dinounet_b200 import config, export as EX, training as TR  # noqa: E402
from dinounet_b200.preprocess import _save_case  # noqa: E402
from oracle import dinounet_oracle as O  # noqa: E402
from oracle import export_oracle as EO  # noqa: E402
from oracle import sliding_window_oracle as SWO  # noqa: E402

SIZE, EXPORT_SIZE, CLASSES = 512, 460, 3
TRANSPOSE_BACKWARD = [0, 1, 2]


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


class _NpzRW:
    write_seconds = 0.0

    def write_seg(self, seg, path, props):
        t0 = time.perf_counter()
        np.savez_compressed(path, seg=seg[None])
        _NpzRW.write_seconds += time.perf_counter() - t0

    def read_seg(self, path):
        return np.load(path)["seg"], {"spacing": (2.5, 0.8, 0.8)}


class _Dataset:
    def __init__(self, folder, keys, folder_with_segs_from_previous_stage=None):
        self.folder, self._keys = folder, list(keys)

    def keys(self):
        return list(self._keys)

    def load_case(self, k):
        f = np.load(os.path.join(self.folder, k + ".npz"))
        with open(os.path.join(self.folder, k + ".pkl"), "rb") as fh:
            return f["data"], f["seg"], pickle.load(fh)


def _write_cases(folder, gt, n, slices, seed):
    keys = []
    for i in range(n):
        k = f"case_{seed + i:03d}"
        g = torch.Generator().manual_seed(seed + i)
        body = torch.nn.functional.interpolate(torch.randn(1, 1, slices, 24, 24, generator=g),
                                               size=(slices, SIZE, SIZE), mode="trilinear", align_corners=False)
        data = (body[0] * 1.2 + 0.2 * torch.randn(1, slices, SIZE, SIZE, generator=g)).numpy().astype(np.float32)
        props = {"spacing": [2.5, 0.8, 0.8], "shape_before_cropping": [slices, EXPORT_SIZE + 12, EXPORT_SIZE + 8],
                 "bbox_used_for_cropping": [[0, slices], [6, EXPORT_SIZE + 6], [4, EXPORT_SIZE + 4]],
                 "shape_after_cropping_and_before_resampling": [slices, EXPORT_SIZE, EXPORT_SIZE]}
        _save_case(os.path.join(folder, k), data, np.zeros((1, slices, SIZE, SIZE), dtype=np.int8), props)
        ref = (body[0, 0] > 0.3).numpy().astype(np.uint8) + (body[0, 0] > 1.0).numpy().astype(np.uint8)
        ref = torch.nn.functional.interpolate(torch.from_numpy(ref)[None, None].float(),
                                              size=(slices, EXPORT_SIZE + 12, EXPORT_SIZE + 8), mode="nearest")
        np.savez_compressed(os.path.join(gt, k + ".npz"), seg=ref[0].numpy().astype(np.uint8))
        keys.append(k)
    return keys


def _trainer(net, data_root, out_root, keys):
    lm = SimpleNamespace(has_regions=False, regions_class_order=None, foreground_labels=[1, 2],
                         foreground_regions=None, num_segmentation_heads=CLASSES, ignore_label=None)
    conf = {"resampling_fn_probabilities": EX.DEFAULT_RESAMPLING_FN,
            "resampling_fn_probabilities_kwargs": dict(EX.DEFAULT_RESAMPLING_KWARGS)}
    tr = TR.DinoUNetTrainer_s.__new__(TR.DinoUNetTrainer_s)
    tr.stamps = []
    tr.print_to_log_file = lambda *a, **kw: tr.stamps.append((time.perf_counter(), str(a[0])))
    tr.network, tr.device, tr.is_ddp, tr.local_rank, tr.is_cascaded = net, torch.device("cuda", 0), False, 0, False
    tr.configuration_manager = SimpleNamespace(patch_size=[SIZE, SIZE], next_stage_names=None, spacing=[0.72, 0.72],
                                               configuration=conf)
    tr.plans_manager = SimpleNamespace(transpose_backward=TRANSPOSE_BACKWARD, get_label_manager=lambda dj: lm,
                                       image_reader_writer_class=_NpzRW)
    tr.label_manager, tr.dataset_json = lm, {"file_ending": ".npz"}
    tr.output_folder = os.path.join(out_root, "fold_0")
    tr.preprocessed_dataset_folder = os.path.join(data_root, "pre", "plans_2d")
    tr.preprocessed_dataset_folder_base = os.path.join(data_root, "pre")
    tr.folder_with_segs_from_previous_stage = None
    tr.inference_allowed_mirroring_axes = (0, 1)
    tr.do_split = lambda: ([], list(keys))
    return tr


def _device_route(net, root, out, keys):
    tr = _trainer(net, root, os.path.join(root, out), keys)
    _NpzRW.write_seconds = 0.0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tr.perform_actual_validation()
    torch.cuda.synchronize()
    total = time.perf_counter() - t0
    starts = [t for t, msg in tr.stamps if msg.startswith("predicting ")]
    ends = starts[1:] + [next(t for t, msg in tr.stamps if msg.startswith("Validation complete"))]
    per_case = [b - a for a, b in zip(starts, ends)]
    return total, statistics.median(per_case), _NpzRW.write_seconds / total


def _baseline_route(net, root, keys, folder):
    def network(t):
        with torch.no_grad():
            return net(t).half()
    times = []
    rw = _NpzRW()
    for k in keys:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        data, _, props = _Dataset(folder, [k]).load_case(k)
        logits = SWO.predict_sliding_window_return_logits(network, torch.from_numpy(data).cuda(), [SIZE, SIZE], CLASSES,
                                                          0.5, True, None, results_device=torch.device("cuda", 0)).cpu()
        _, seg, _ = EO.convert(logits, props, TRANSPOSE_BACKWARD, 2, False)
        rw.write_seg(seg, os.path.join(root, "baseline_" + k + ".npz"), props)
        times.append(time.perf_counter() - t0)
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", type=int, default=4)
    ap.add_argument("--slices", type=int, default=24)
    ap.add_argument("--baseline-cases", type=int, default=2)
    ap.add_argument("--models", nargs="*", default=["dinounet_s", "dinounet_l"])
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_validation measures the device route: it needs a GPU"
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    TR._validation_dataset = _Dataset
    print(f"card: {_card()}")
    print(f"{args.cases} cases of 1 x {args.slices} x {SIZE} x {SIZE} -> {EXPORT_SIZE} x {EXPORT_SIZE}, {CLASSES} classes")
    rows = []
    with tempfile.TemporaryDirectory() as root:
        folder, gt = os.path.join(root, "pre", "plans_2d"), os.path.join(root, "pre", "gt_segmentations")
        os.makedirs(folder)
        os.makedirs(gt)
        keys = _write_cases(folder, gt, args.cases, args.slices, 0)
        for model in args.models:
            net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 1, CLASSES,
                                                     None, model)
            net.load_state_dict(O.make_state_dict(model, CLASSES, seed=0), strict=True)
            net = net.cuda().eval()
            _device_route(net, root, "warm", keys[:1])
            total, median, write_share = _device_route(net, root, model, keys)
            base = _baseline_route(net, root, keys[:args.baseline_cases], folder)
            rows.append((model, total, median, write_share, base))
            del net
            torch.cuda.empty_cache()
    print("| model | device route, total | per case (median) | share writing files | reference loop per case (median) |")
    print("|---|---|---|---|---|")
    for model, total, median, share, base in rows:
        print(f"| {model} | {total:.2f} s | {median * 1e3:.0f} ms | {share * 100:.0f}% | {base * 1e3:.0f} ms |")


if __name__ == "__main__":
    main()
