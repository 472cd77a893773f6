"""Peak memory and step time of the native training step with the adapter's extractors recomputed in the backward
(`DinoUNet.train_recompute = True`, the reference's `with_cp=True`) against keeping their activations (the default).

For each model at 512^2 (TF32 tier, "oracle" semantics, Dice+CE, FusedSGD):
  * peak `torch.cuda.max_memory_allocated` of one `train_step` (after `reset_peak_memory_stats`; the step's resident
    state - fp32 module, packed 16-bit engine weights and plan, gradients, momentum - included) at two or three batch
    sizes known to fit, both settings;
  * a least-squares line through those peaks, and from it the largest batch whose predicted peak stays under
    MARGIN x the card's memory.  That batch is then run once to confirm the prediction.  No batch is chosen by running
    into an out-of-memory error.  Confirmation runs stay at batches whose largest activation (the decoder's 64-channel
    input at full resolution) has fewer than 2^31 elements; a prediction beyond that is reported as a fit only;
  * ms per step: median of `--steps` steps per setting at `--time-batch`, the two settings alternated step by step
    after a warm-up, in one process, timed with CUDA events.

The network is built on the device (`with torch.device("cuda")`) and filled with bench.py's synthetic on-device weights:
dinounet_7b's 6.95 B fp32 parameters never pass through host memory.  Prints the card's name and power limit and one
JSON line per model.

  python tools/bench_train_memory.py [--models dinounet_s dinounet_b dinounet_l dinounet_7b] [--steps 5]
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

#: share of the card's memory a predicted peak may use; the rest covers allocator fragmentation and the CUDA context
MARGIN = 0.92
FIT_BATCHES = {"dinounet_s": (4, 8, 16), "dinounet_b": (4, 8, 16), "dinounet_l": (4, 8, 16), "dinounet_7b": (1, 2, 4)}
TIME_BATCH = {"dinounet_s": 16, "dinounet_b": 16, "dinounet_l": 16, "dinounet_7b": 2}


def build(model, dev):
    import dinounet_b200
    from bench import SyntheticParams
    from dinounet_b200 import config
    with torch.device(dev):
        net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, 2, None, model)
    gen = SyntheticParams(model, 2, dev)
    with torch.no_grad():
        for k, t in net.state_dict(keep_vars=True).items():
            if k in gen:                       # aliases (decoder.encoder.*, all_modules.*) share these tensors
                t.copy_(gen[k])
    net.repack()
    return net.train()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=["dinounet_s", "dinounet_b", "dinounet_l", "dinounet_7b"])
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-confirm", action="store_true", help="report the fit without running the predicted batch")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    os.environ.setdefault("DINOUNET_B200_ALLOW_RANDOM_BACKBONE", "1")
    from dinounet_b200.loss import DC_and_CE_loss
    from dinounet_b200.train_path import FusedSGD, train_step
    from oracle import dinounet_oracle as O

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    dev = torch.device("cuda", 0)
    total = torch.cuda.get_device_properties(dev).total_memory
    S = a.size
    max_safe_batch = (2 ** 31 - 1) // (S * S * 64)
    crit = DC_and_CE_loss({"batch_dice": True, "smooth": 1e-5, "do_bg": False, "ddp": False}, {}, weight_ce=1, weight_dice=1)

    for model in a.models:
        net = build(model, dev)
        opt = FusedSGD(net.parameters(), lr=1e-2, weight_decay=3e-5)
        eng = net._get_engine(dev)

        def batch(B):
            x = O.make_input(B, S, 100).to(dev)
            t = torch.randint(0, 2, (B, 1, S, S), generator=torch.Generator().manual_seed(B)).float().to(dev)
            return x, t

        def peak(B, recompute, warm=True):
            """Peak bytes of one step at batch B with only this batch's engine plan resident."""
            eng.clear_plans()
            gc.collect()
            torch.cuda.empty_cache()
            net.train_recompute = recompute
            x, t = batch(B)
            if warm:
                train_step(net, crit, opt, x, t)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            loss = train_step(net, crit, opt, x, t)
            torch.cuda.synchronize()
            if not torch.isfinite(loss):   # the synthetic weights are not trained; memory and time do not depend on them
                print(f"{model} B {B}: loss {loss.item()}", flush=True)
            return torch.cuda.max_memory_allocated(dev)

        res = {"model": model, "size": S, "gpu": card, "train_gemm": net.train_gemm, "semantics": net.train_semantics,
               "card_bytes": total, "margin": MARGIN, "settings": {}}
        for recompute in (False, True):
            name = "recompute" if recompute else "keep"
            pts = {}
            for B in FIT_BATCHES[model]:
                pts[B] = peak(B, recompute)
                print(f"{model} {name} B {B}: peak {pts[B] / 2**30:.2f} GiB", flush=True)
            bs = list(pts)
            mb, mp = statistics.fmean(bs), statistics.fmean(pts.values())
            slope = sum((b - mb) * (pts[b] - mp) for b in bs) / sum((b - mb) ** 2 for b in bs)
            icpt = mp - slope * mb
            bmax = int((MARGIN * total - icpt) // slope)
            r = {"peaks_gib": {B: p / 2 ** 30 for B, p in pts.items()}, "fit_gib": {"per_sample": slope / 2 ** 30,
                 "fixed": icpt / 2 ** 30}, "predicted_max_batch": bmax,
                 "predicted_peak_gib": (icpt + slope * bmax) / 2 ** 30}
            run_b = min(bmax, max_safe_batch)
            if not a.no_confirm and run_b > max(bs):
                p = peak(run_b, recompute, warm=False)
                r["confirm"] = {"batch": run_b, "peak_gib": p / 2 ** 30,
                                "predicted_gib": (icpt + slope * run_b) / 2 ** 30,
                                "note": None if run_b == bmax else f"capped at {max_safe_batch}: 2^31-element activations"}
                print(f"{model} {name}: confirmed B {run_b}: peak {p / 2**30:.2f} GiB", flush=True)
            res["settings"][name] = r
        # step time, the two settings alternated step by step
        eng.clear_plans()
        gc.collect()
        torch.cuda.empty_cache()
        B = TIME_BATCH[model]
        x, t = batch(B)
        times = {False: [], True: []}
        for i in range(2 * (a.warmup + a.steps)):
            recompute = bool(i % 2)
            net.train_recompute = recompute
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            train_step(net, crit, opt, x, t)
            e1.record()
            torch.cuda.synchronize()
            if i >= 2 * a.warmup:
                times[recompute].append(e0.elapsed_time(e1))
        res["time"] = {"batch": B, "steps": a.steps, "ms_keep": statistics.median(times[False]),
                       "ms_recompute": statistics.median(times[True]),
                       "all_ms": {"keep": times[False], "recompute": times[True]}}
        print(json.dumps(res), flush=True)
        del net, opt, eng
        gc.collect()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
