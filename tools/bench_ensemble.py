"""Times ensembling on the device against the reference's host arithmetic, and one-pass ensemble prediction against
the two-step route.

Seeded CT-like cases (default 4 cases of 100 x 512^2, one channel, 3 classes; tools/bench_predict.py's generator) and
3 members.  In one process, the two sides of each comparison alternating:

  * `ensemble_folders` on the device against the oracle's `merge_files` (the reference's numpy / torch-CPU arithmetic)
    called case by case on the same `.npz` files.  The device time per case is split into npz read + decompression,
    upload, kernel time (CUDA events around the accumulate and segment kernels, with the bytes they move over the
    3.35 TB/s data-sheet HBM3 figure) and writing.  The reference runs `merge_files` in a process pool, so the host
    column is one case in one process: an upper bound on its time per case, not a measurement of the pool.
  * `predict_ensemble_from_files` with dinounet_s + dinounet_b + dinounet_l (2 folds each, one shared backbone per
    model) against predicting each member with `save_probabilities` and then `ensemble_folders`; the segmentations and
    averaged probabilities are compared bit for bit, and the `.npz` bytes the two-step route wrote and read reported.

Prints one JSON line with the card's name and power limit.  Usage:
    python tools/bench_ensemble.py [--cases 4 --slices 100 --members dinounet_s dinounet_b dinounet_l] [--out FILE]
"""
import argparse
import json
import os
import pickle
import shutil
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_predict import NpyIO, gpu_info, make_folds, managers, write_cases  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def log(msg):
    print(msg, file=sys.stderr, flush=True)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def write_member_npz(folder, n, slices, size, ncls, members, seed=1):
    """Member probability volumes as the export writes them: softmax of seeded fp16 logits, fp32 `.npz` + `.pkl`."""
    rng = np.random.default_rng(seed)
    for m in range(members):
        d = os.path.join(folder, f"member{m}")
        os.makedirs(d)
        for c in range(n):
            x = torch.from_numpy(rng.standard_normal((ncls, slices, size, size), dtype=np.float32) * 4).half().float()
            np.savez_compressed(os.path.join(d, f"case{c:02d}.npz"), probabilities=torch.softmax(x, 0).numpy())
            with open(os.path.join(d, f"case{c:02d}.pkl"), "wb") as f:
                pickle.dump({"spacing": [1.0, 0.8, 0.8]}, f)
        with open(os.path.join(d, "dataset.json"), "w") as f:
            json.dump({"file_ending": ".npy", "labels": {"background": 0, "a": 1, "b": 2}}, f)
        with open(os.path.join(d, "plans.json"), "w") as f:
            json.dump({"plans_name": "bench"}, f)
    return [os.path.join(folder, f"member{m}") for m in range(members)]


def bench_ensemble_folders(args, tmp, pm, lm):
    from dinounet_b200 import ensembling as E
    from dinounet_b200 import lib as L
    from oracle import ensemble_oracle as EN
    folders = write_member_npz(tmp, args.cases, args.slices, args.size, args.classes, args.n_members)
    log("member .npz written")
    names = sorted(f for f in os.listdir(folders[0]) if f.endswith(".npz"))
    lib = L.load()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev).cuda_stream
    split = {"read_s": [], "upload_s": [], "kernel_s": [], "write_s": []}
    kernel_bytes = []

    def device_split(name, out):
        """One case on the device, step by step (what `ensemble_folders` overlaps across threads)."""
        t0 = time.perf_counter()
        members = [np.load(os.path.join(f, name))["probabilities"] for f in folders]
        t1 = time.perf_counter()
        ups = [torch.from_numpy(m).to(dev) for m in members]
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        acc = torch.empty(members[0].shape, dtype=torch.float32, device=dev)
        labels = torch.empty(members[0].shape[1:], dtype=torch.uint8, device=dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for k, u in enumerate(ups):
            L.check(lib.b2u_ensemble_accumulate(u.data_ptr(), 4, acc.data_ptr(), u.numel(), int(k == 0), stream))
        L.check(lib.b2u_ensemble_segment(acc.data_ptr(), acc.shape[0], acc[0].numel(), len(ups), 0, None,
                                         labels.data_ptr(), 1, stream))
        e1.record()
        seg = labels.cpu().numpy()
        t3 = time.perf_counter()
        NpyIO().write_seg(seg, os.path.join(out, name[:-4] + ".npy"), {})
        t4 = time.perf_counter()
        n = acc.numel()
        # accumulate: member reads + acc read/write (first: write only); segment: acc read + write, labels write
        kernel_bytes.append(len(ups) * n * 4 + (len(ups) - 1) * n * 8 + n * 4 + 8 * n + acc[0].numel())
        split["read_s"].append(t1 - t0)
        split["upload_s"].append(t2 - t1)
        split["kernel_s"].append(e0.elapsed_time(e1) / 1e3)
        split["write_s"].append(t4 - t3)

    def host_case(name, out):
        EN.merge_files([os.path.join(f, name) for f in folders], os.path.join(out, name[:-4]), ".npy", NpyIO(), lm)

    device_split(names[0], tmp)          # warm-up
    t_dev, t_host, t_folders = [], [], []
    out_dev, out_host, out_folders = (os.path.join(tmp, d) for d in ("split", "host", "folders"))
    for d in (out_dev, out_host):
        os.makedirs(d)
    for i, name in enumerate(names):
        order = [("dev", device_split), ("host", host_case)] if i % 2 == 0 else [("host", host_case), ("dev", device_split)]
        for side, fn in order:
            t, _ = timed(lambda: fn(name, out_dev if side == "dev" else out_host))
            (t_dev if side == "dev" else t_host).append(t)
            log(f"{name} {side}: {t:.3f} s")
    for rep in range(2):
        t, _ = timed(lambda: E.ensemble_folders(folders, out_folders + str(rep), False, 3))
        t_folders.append(t / len(names))
        log(f"ensemble_folders: {t:.3f} s")
    same_as_host = sum(int(np.sum(np.load(os.path.join(out_folders + "0", n[:-4] + ".npy")) !=
                                  np.load(os.path.join(out_host, n[:-4] + ".npy")))) for n in names)
    kernel = float(np.median(split["kernel_s"]))
    return {
        "ensemble_folders_per_case_s": [round(t, 3) for t in t_folders],
        "device_step_by_step_per_case_s": [round(t, 3) for t in t_dev],
        "host_merge_files_per_case_s_upper_bound": [round(t, 3) for t in t_host],
        "median_split_s": {k: round(float(np.median(v)), 4) for k, v in split.items()},
        "kernel_bytes_per_case": int(kernel_bytes[0]),
        "kernel_TBps": round(kernel_bytes[0] / kernel / 1e12, 3),
        "kernel_share_of_3.35TBps": round(kernel_bytes[0] / kernel / HBM_BYTES_PER_S, 3),
        "label_voxels_differing_from_host": same_as_host,
    }


def bench_one_pass(args, tmp, src):
    from dinounet_b200 import ensembling as E
    from dinounet_b200 import predict as PR
    from dinounet_b200.sliding_window import SlidingWindowPredictor
    import dinounet_b200
    from dinounet_b200 import config
    dev = torch.device("cuda", 0)
    pm, cm, dj = managers(args.classes)
    PR._plans_manager = lambda plans: pm
    predictors = []
    for model in args.members:
        folds = make_folds(model, args.classes, args.folds)
        net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 1, args.classes,
                                                 None, model)
        net.load_state_dict(folds[-1])
        p = SlidingWindowPredictor(device=dev, tile_batch=args.tile_batch)
        p.manual_initialization(net.to(dev).eval(), pm, cm, folds, dj, f"DinoUNetTrainer_{model.split('_')[1]}", (0, 1))
        predictors.append(p)
    files = sorted(os.listdir(src))
    warm = os.path.join(tmp, "warm")
    os.makedirs(warm)
    os.symlink(os.path.join(src, files[0]), os.path.join(warm, files[0]))
    for p in predictors:
        p.predict_from_files(warm, os.path.join(tmp, "warm_out"), save_probabilities=False)
        log(f"warmed up {p.trainer_name}")

    def two_step(out):
        members = []
        for k, p in enumerate(predictors):
            o = os.path.join(out, f"m{k}")
            p.predict_from_files(src, o, save_probabilities=True)
            members.append(o)
        E.ensemble_folders(members, os.path.join(out, "ens"), False, 3)
        return sum(os.path.getsize(os.path.join(m, f)) for m in members for f in os.listdir(m) if f.endswith(".npz"))

    def one_pass(out):
        E.predict_ensemble_from_files(predictors, src, out, save_probabilities=False)

    t_two, t_one, npz_bytes = [], [], 0
    for rep in range(args.reps):
        order = [("two", two_step), ("one", one_pass)] if rep % 2 == 0 else [("one", one_pass), ("two", two_step)]
        for side, fn in order:
            t, r = timed(lambda: fn(os.path.join(tmp, f"{side}_{rep}")))
            (t_two if side == "two" else t_one).append(t / len(files))
            if side == "two":
                npz_bytes = r
            log(f"rep {rep} {side}: {t:.3f} s")
            if rep > 0:     # rep 0's outputs are compared below; the rest would only fill the disk
                shutil.rmtree(os.path.join(tmp, f"{side}_{rep}"))
    outs = [f[:-9] + ".npy" for f in files]
    identical = all(np.array_equal(np.load(os.path.join(tmp, "two_0", "ens", o)), np.load(os.path.join(tmp, "one_0", o)))
                    for o in outs)
    # averaged probabilities: the two routes once more with save_probabilities
    E.ensemble_folders([os.path.join(tmp, "two_0", f"m{k}") for k in range(len(predictors))],
                       os.path.join(tmp, "two_p"), True, 3)
    E.predict_ensemble_from_files(predictors, src, os.path.join(tmp, "one_p"), save_probabilities=True)
    probs_identical = all(np.array_equal(np.load(os.path.join(tmp, "two_p", o[:-4] + ".npz"))["probabilities"].view(np.int32),
                                         np.load(os.path.join(tmp, "one_p", o[:-4] + ".npz"))["probabilities"].view(np.int32))
                          for o in outs)
    return {
        "one_pass_members": args.members, "folds_per_member": args.folds,
        "two_step_per_case_s": [round(t, 3) for t in t_two], "one_pass_per_case_s": [round(t, 3) for t in t_one],
        "one_pass_speedup": round(float(np.median(t_two) / np.median(t_one)), 3),
        "two_step_npz_bytes_written_and_read": npz_bytes,
        "segmentations_bit_identical": identical, "averaged_probabilities_bit_identical": probs_identical,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", type=int, default=4)
    ap.add_argument("--slices", type=int, default=100)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--classes", type=int, default=3)
    ap.add_argument("--n-members", type=int, default=3)
    ap.add_argument("--members", nargs="+", default=["dinounet_s", "dinounet_b", "dinounet_l"])
    ap.add_argument("--folds", type=int, default=2)
    ap.add_argument("--tile-batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--skip-one-pass", action="store_true")
    ap.add_argument("--skip-folders", action="store_true")
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ensemble needs a CUDA device")
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    name, power = gpu_info()
    from types import SimpleNamespace
    lm = SimpleNamespace(has_regions=False, regions_class_order=None, foreground_labels=list(range(1, args.classes)),
                         num_segmentation_heads=args.classes)
    with tempfile.TemporaryDirectory() as tmp:
        pm, _, _ = managers(args.classes)
        from dinounet_b200 import predict as PR
        PR._plans_manager = lambda plans: pm
        r = {"gpu": name, "power_limit": power, "cases": args.cases, "case_shape": [args.slices, args.size, args.size],
             "classes": args.classes, "npz_members": args.n_members}
        if not args.skip_folders:
            os.makedirs(os.path.join(tmp, "folders"))
            r.update(bench_ensemble_folders(args, os.path.join(tmp, "folders"), pm, lm))
            shutil.rmtree(os.path.join(tmp, "folders"))
        if not args.skip_one_pass:
            src = os.path.join(tmp, "cases")
            os.makedirs(src)
            write_cases(src, args.cases, args.slices, args.size)
            r.update(bench_one_pass(args, tmp, src))
    line = json.dumps(r)
    print(line, flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
