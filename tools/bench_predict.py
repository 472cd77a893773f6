"""Times the fold ensemble of `SlidingWindowPredictor` and the model-folder loop of `predict_from_files`.

Seeded CT-like cases (default 4 cases of 100 x 512^2, one channel, 3 classes) are written to a temporary folder as
`.npy` files; 5 folds share one backbone (fold k's weights after the taps are fold 0's scaled by a seeded factor), the
patch is 512^2 with mirroring on (the predictor's default), tile batch 8.  In one process, with the two sides of each
comparison alternating:

  * per case, `predict_logits_from_preprocessed_data` on the per-fold route (load + repack + whole network for every
    fold) against the shared-backbone route (the ViT once per tile batch), on the same preprocessed data; the two
    results are compared bit for bit;
  * `predict_from_files` over the folder against a loop of `predict_single_npy_array` writing the same outputs.

Prints one JSON line per model with the card's name and power limit.  Usage:
    python tools/bench_predict.py --models dinounet_s dinounet_l [--cases 4 --slices 100 --folds 5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:   # the timing itself needs no nvidia-smi
        return torch.cuda.get_device_name(0), f"unknown ({e})"


def make_folds(model, ncls, n):
    """Fold 0 from the oracle's seeded weights; fold k > 0 shares its backbone and scales every other floating tensor
    by a seeded factor in [0.9, 1.1] (distinct folds, same frozen backbone).  The state dict's duplicate keys of one
    tensor (`decoder.encoder.*`, `all_modules.*`) keep one value, as in a real checkpoint."""
    from oracle import dinounet_oracle as O
    base = O.make_state_dict(model, ncls, seed=0)
    folds = [base]
    for k in range(1, n):
        g = torch.Generator().manual_seed(1000 + k)
        sd, scaled = {}, {}
        for name, t in base.items():
            if ".dinov3_adapter.backbone." in name or not t.is_floating_point() or "running_var" in name:
                sd[name] = t
            else:
                if id(t) not in scaled:
                    scaled[id(t)] = t * (0.9 + 0.2 * torch.rand((), generator=g))
                sd[name] = scaled[id(t)]
        folds.append(sd)
    return folds


class NpyIO:
    spacing = [1.0, 0.8, 0.8]

    def read_images(self, files):
        return np.stack([np.load(f) for f in files]).astype(np.float32), {"spacing": list(self.spacing)}

    def write_seg(self, seg, path, properties):
        np.save(path, seg)


def managers(ncls):
    from dinounet_b200 import export as EX
    from dinounet_b200 import preprocess as PP
    conf = {"preprocessor_name": "DefaultPreprocessor", "resampling_fn_data": PP.DEFAULT_RESAMPLING_FN,
            "resampling_fn_data_kwargs": dict(PP.DEFAULT_RESAMPLING_KWARGS),
            "resampling_fn_probabilities": EX.DEFAULT_RESAMPLING_FN,
            "resampling_fn_probabilities_kwargs": dict(EX.DEFAULT_RESAMPLING_KWARGS)}
    cm = SimpleNamespace(spacing=[0.8, 0.8], patch_size=[512, 512], normalization_schemes=["CTNormalization"],
                         use_mask_for_norm=[False], configuration=conf, previous_stage_name=None)
    lm = SimpleNamespace(has_regions=False, regions_class_order=None, foreground_labels=list(range(1, ncls)),
                         num_segmentation_heads=ncls)
    intensity = {"0": {"mean": 40.0, "std": 180.0, "percentile_00_5": -1000.0, "percentile_99_5": 1500.0}}
    pm = SimpleNamespace(transpose_forward=[0, 1, 2], transpose_backward=[0, 1, 2], get_label_manager=lambda dj: lm,
                         foreground_intensity_properties_per_channel=intensity, image_reader_writer_class=NpyIO,
                         plans={"plans_name": "bench"})
    return pm, cm, {"file_ending": ".npy", "channel_names": {"0": "CT"}}


def write_cases(folder, n, slices, size, seed=0):
    """CT-like volumes: air around a body ellipse of soft tissue with bright inclusions, plus noise (HU)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:size, :size] / size - 0.5
    for c in range(n):
        vol = np.full((slices, size, size), -1000.0, np.float32)
        body = (yy / 0.42) ** 2 + (xx / 0.36) ** 2 < 1
        vol[:, body] = 40.0
        for _ in range(6):
            cy, cx, r = rng.uniform(-0.25, 0.25), rng.uniform(-0.25, 0.25), rng.uniform(0.02, 0.08)
            vol[:, (yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = rng.uniform(200, 1200)
        vol += rng.standard_normal(vol.shape).astype(np.float32) * 20
        np.save(os.path.join(folder, f"case{c:02d}_0000.npy"), vol)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def bench_model(model, args, src, tmp):
    import dinounet_b200
    from dinounet_b200 import config
    from dinounet_b200.preprocess import DevicePreprocessor
    from dinounet_b200.sliding_window import SlidingWindowPredictor
    dev = torch.device("cuda", 0)
    ncls = args.classes
    folds = make_folds(model, ncls, args.folds)

    def network():
        net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 1, ncls, None, model)
        net.load_state_dict(folds[-1])
        return net.to(dev).eval()

    pm, cm, dj = managers(ncls)
    # one network per predictor: the per-fold route reloads its network for every fold, which would make the shared
    # route repack its engine on every case if they shared one
    shared = SlidingWindowPredictor(device=dev, tile_batch=args.tile_batch)
    shared.manual_initialization(network(), pm, cm, folds, dj, f"DinoUNetTrainer_{model.split('_')[1]}", (0, 1))
    per_fold = SlidingWindowPredictor(device=dev, tile_batch=args.tile_batch)
    per_fold.manual_initialization(network(), pm, cm, folds, dj, shared.trainer_name, (0, 1))
    per_fold.list_of_parameters = list(folds)      # a list assigned after initialisation: the per-fold route
    files = sorted(os.path.join(src, f) for f in os.listdir(src))
    rw = NpyIO()
    pre = DevicePreprocessor(False, dev)

    def preprocessed(path):
        img, props = rw.read_images([path])
        data, _ = pre.run_case_npy(img, None, props, pm, cm, dj)
        return data

    # warm-up: plans, CUDA graphs, the fold engine
    d0 = preprocessed(files[0])
    shared.predict_logits_from_preprocessed_data(d0)
    per_fold.predict_logits_from_preprocessed_data(d0)
    fold_mb = [b / 2 ** 20 for b in shared._fold_engine[3].fold_bytes()]
    t_per, t_shared, identical = [], [], True
    for i, f in enumerate(files):
        data = preprocessed(f)
        order = [("per_fold", per_fold), ("shared", shared)] if i % 2 == 0 else [("shared", shared), ("per_fold", per_fold)]
        res = {}
        for name, p in order:
            t, out = timed(lambda: p.predict_logits_from_preprocessed_data(data))
            (t_per if name == "per_fold" else t_shared).append(t)
            res[name] = out
        identical &= bool(torch.equal(res["per_fold"].view(torch.int16), res["shared"].view(torch.int16)))
        assert per_fold.ensemble_route == "per_fold" and shared.ensemble_route == "shared_backbone"
        del res, data

    # predict_from_files over the folder against a loop of predict_single_npy_array
    def loop(out):
        os.makedirs(out, exist_ok=True)
        for f in files:
            img, props = rw.read_images([f])
            shared.predict_single_npy_array(img, props, None, os.path.join(out, os.path.basename(f)[:-9]), False)

    def from_files(out):
        shared.predict_from_files(src, out, save_probabilities=False, overwrite=True, num_processes_preprocessing=3,
                                  num_processes_segmentation_export=3)

    t_loop, t_files = [], []
    for rep in range(args.reps):
        order = [("loop", loop), ("files", from_files)] if rep % 2 == 0 else [("files", from_files), ("loop", loop)]
        for name, fn in order:
            t, _ = timed(lambda: fn(os.path.join(tmp, f"{model}_{name}_{rep}")))
            (t_loop if name == "loop" else t_files).append(t)
    outs = [os.path.basename(f)[:-9] + ".npy" for f in files]
    same_files = all(np.array_equal(np.load(os.path.join(tmp, f"{model}_loop_0", o)),
                                    np.load(os.path.join(tmp, f"{model}_files_0", o))) for o in outs)
    n = len(files)
    return {
        "model": model, "folds": args.folds, "cases": n, "case_shape": [args.slices, args.size, args.size],
        "classes": ncls, "tile_batch": args.tile_batch, "mirroring": True,
        "per_case_s_per_fold_route": [round(t, 3) for t in t_per],
        "per_case_s_shared_route": [round(t, 3) for t in t_shared],
        "median_per_fold_s": round(float(np.median(t_per)), 3), "median_shared_s": round(float(np.median(t_shared)), 3),
        "shared_speedup": round(float(np.median(t_per) / np.median(t_shared)), 3),
        "routes_bit_identical": identical,
        "folder_s_loop_predict_single_npy_array": [round(t, 3) for t in t_loop],
        "folder_s_predict_from_files": [round(t, 3) for t in t_files],
        "files_speedup": round(float(np.median(t_loop) / np.median(t_files)), 3),
        "files_outputs_equal_loop": same_files,
        "packed_MB_per_fold": round(fold_mb[0], 2),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=["dinounet_s", "dinounet_l"])
    ap.add_argument("--cases", type=int, default=4)
    ap.add_argument("--slices", type=int, default=100)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--classes", type=int, default=3)
    ap.add_argument("--folds", type=int, default=5)
    ap.add_argument("--tile-batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_predict needs a CUDA device")
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    name, power = gpu_info()
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "cases")
        os.makedirs(src)
        write_cases(src, args.cases, args.slices, args.size)
        for model in args.models:
            r = bench_model(model, args, src, tmp)
            r.update(gpu=name, power_limit=power)
            line = json.dumps(r)
            print(line, flush=True)
            if args.out:
                with open(args.out, "a") as f:
                    f.write(line + "\n")
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
