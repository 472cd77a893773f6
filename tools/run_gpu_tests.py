"""Runs every -m gpu test in its OWN process with a timeout, so one hang / sticky CUDA error cannot mask the others.
Usage (on the GPU box):  python tools/run_gpu_tests.py [-k expr] [--timeout 180]  -> gpurun_out/gpu_tests.log"""
import argparse
import os
import subprocess
import sys
import time

ap = argparse.ArgumentParser()
ap.add_argument("-k", default="")
ap.add_argument("--timeout", type=int, default=240)
ap.add_argument("--per-test", action="store_true")
ap.add_argument("--files", nargs="*", default=["tests/test_gpu_kernels.py", "tests/test_gpu_parity.py", "tests/test_gpu_sliding_window.py",
                                          "tests/test_gpu_loss.py", "tests/test_gpu_trainer_loop.py"])
a = ap.parse_args()
os.makedirs("gpurun_out", exist_ok=True)
cmd = [sys.executable, "-m", "pytest", "--collect-only", "-q", "-m", "gpu", *a.files]
if a.k:
    cmd += ["-k", a.k]
ids = [l.strip() for l in subprocess.run(cmd, capture_output=True, text=True).stdout.splitlines() if "::" in l]
if "--per-test" not in sys.argv:
    seen = []
    for t in ids:   # one process per test FUNCTION (all its parametrisations together)
        f = t.split("[")[0]
        if f not in seen:
            seen.append(f)
    ids = seen
print(f"{len(ids)} test groups")
res = []
with open("gpurun_out/gpu_tests.log", "w") as log:
    for tid in ids:
        t0 = time.time()
        try:
            r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-s", "-m", "gpu", tid], capture_output=True,
                               text=True, timeout=a.timeout)
            status = "PASS" if r.returncode == 0 else "FAIL"
            out = r.stdout[-3500:] + r.stderr[-1500:]
        except subprocess.TimeoutExpired as e:
            status, out = "TIMEOUT", ((e.stdout or b"")[-2000:].decode(errors="replace") if isinstance(e.stdout, bytes) else str(e.stdout)[-2000:])
        dt = time.time() - t0
        print(f"{status:8s} {dt:6.1f}s {tid}", flush=True)
        log.write(f"===== {status} {dt:.1f}s {tid}\n")
        log.write("\n".join(l for l in out.splitlines() if "rel err" in l or "stage " in l or "NON-FINITE" in l) + "\n")
        if status != "PASS":
            log.write(out + "\n")
        log.flush()
        res.append(status)
print({s: res.count(s) for s in set(res)})
sys.exit(0 if all(s == "PASS" for s in res) else 1)
