"""Microbenchmark: the training path's matrix products on both tiers (b2u_tf32_gemm = TF32 wgmma, b2u_f32_gemm =
fp32 SIMT) at the shapes that dominate the dinounet_b train step.  CUDA events, 1 warm-up + 3 timed launches each.
usage: python tools/bench_tf32_gemm.py [B] [tiers]   (B = images for the conv shapes, default 8; tiers = "tf32,fp32")"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from dinounet_b200 import lib as L          # noqa: E402
from dinounet_b200 import train_path as TP  # noqa: E402


def timeit(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    tiers = tuple(sys.argv[2].split(",")) if len(sys.argv) > 2 else ("tf32", "fp32")
    dev = "cuda"
    rows = []

    def run(name, flops, call):
        r = {"shape": name, "gflop": flops / 1e9}
        for tier in tiers:
            ms = timeit(lambda: call(tier))
            r[tier + "_ms"] = round(ms, 3)
            r[tier + "_tflops"] = round(flops / ms / 1e9, 1)
        if "fp32_ms" in r and "tf32_ms" in r:
            r["speedup"] = round(r["fp32_ms"] / r["tf32_ms"], 2)
        rows.append(r)
        print(json.dumps(r), flush=True)

    # extractor-sized linear: rows = B*5376 tokens, 768 -> 768
    M, N, K = B * 8 * 5376, 768, 768
    x, W = torch.randn(M, K, device=dev), torch.randn(N, K, device=dev) * 0.03
    y, dx, dW = torch.empty(M, N, device=dev), torch.empty(M, K, device=dev), torch.zeros(N, K, device=dev)
    run(f"linear fwd {M}x{N}x{K}", 2.0 * M * N * K, lambda t: TP._gemm(x, W, y, M, N, K, tier=t))
    run(f"linear dgrad {M}x{K}x{N}", 2.0 * M * N * K, lambda t: TP._gemm(y, W, dx, M, K, N, w_mode=1, tier=t))
    run(f"linear wgrad {N}x{K}x{M}", 2.0 * M * N * K, lambda t: TP._gemm(y, x, dW, N, K, M, a_trans=1, w_mode=1, ksplit=TP._ksplit(M), tier=t))
    del x, y, dx
    for (H, Cin, Cout) in ((512, 64, 32), (512, 32, 32), (256, 128, 64), (128, 256, 128)):
        npix = B * H * H
        x = torch.randn(npix, Cin, device=dev)
        Wp = torch.randn(Cout, 9 * Cin, device=dev) * 0.05
        y = torch.empty(npix, Cout, device=dev)
        dx = torch.empty(npix, Cin, device=dev)
        dWp = torch.zeros(Cout, 9 * Cin, device=dev)
        fl = 2.0 * npix * Cout * 9 * Cin
        run(f"conv3x3 fwd B{B} {H}^2 {Cin}->{Cout}", fl,
            lambda t: TP._gemm(x, Wp, y, npix, Cout, 9 * Cin, conv=L.CONV3X3_S1, img=(H, H, Cin), cpad=Cin, tier=t))
        run(f"conv3x3 dgrad B{B} {H}^2 {Cin}->{Cout}", fl,
            lambda t: TP._gemm(y, Wp, dx, npix, Cin, 9 * Cout, conv=L.CONV3X3_S1, img=(H, H, Cout), cpad=Cout, w_mode=2, w_cpad=Cin, ldw=9 * Cin, tier=t))
        run(f"conv3x3 wgrad B{B} {H}^2 {Cin}->{Cout}", fl,
            lambda t: TP._gemm(y, x, dWp, Cout, 9 * Cin, npix, a_trans=1, lda=Cout, w_mode=3, conv=L.CONV3X3_S1, img=(H, H, Cin), cpad=Cin,
                               ksplit=max(1, min(256, npix // 4096)), tier=t))
        del x, y, dx
    print(json.dumps({"rows": rows}))


if __name__ == "__main__":
    main()
