"""Builds libdinounet_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SOURCES = ["gemm_api.cu", ("gemm_tc2.cu", "gemm_tc2_bf16.o", ["-DB2U_GEMM2_TYPE=1"]), ("gemm_tc2.cu", "gemm_tc2_f16.o", ["-DB2U_GEMM2_TYPE=0"]), "attention_tc.cu", "attention_tc3.cu", "elementwise.cu", "fp32_tier.cu", "gemm_tf32.cu", "train_bwd.cu", "train_mode.cu", "msda.cu", "sliding_window.cu", "export.cu", "preprocess.cu", "evaluation.cu", "postprocessing.cu", "augmentation.cu", "loss.cu", "host_util.cu"]
# A/B builds: B2U_EXTRA_FLAGS="-DFOO=1" B2U_OUT_SUFFIX=_foo python build.py -> libdinounet_b200_foo.so (objects under build_foo/);
# run with DINOUNET_B200_LIB=<that file>.  The default build takes neither.
SUFFIX = os.environ.get("B2U_OUT_SUFFIX", "")
EXTRA = os.environ.get("B2U_EXTRA_FLAGS", "").split()
OUT = os.path.join(os.path.dirname(HERE), f"libdinounet_b200{SUFFIX}.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = [*ARCH, "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
         "--use_fast_math=false"]
FLAGS = [f for f in FLAGS if not f.startswith("--use_fast_math")]


def _stale(obj, src):
    if not os.path.exists(obj):
        return True
    t = os.path.getmtime(obj)
    deps = [src, __file__] + [os.path.join(HERE, f) for f in os.listdir(HERE) if f.endswith((".cuh", ".h"))]
    deps.append(os.path.join(HERE, "..", "..", "include", "dinounet_b200.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    objdir = os.path.join(HERE, "build" + SUFFIX)
    os.makedirs(objdir, exist_ok=True)
    objs, procs = [], []
    for s in SOURCES:
        extra = []
        if isinstance(s, tuple):
            s, oname, extra = s
        else:
            oname = s.replace(".cu", ".o")
        src = os.path.join(HERE, s)
        obj = os.path.join(objdir, oname)
        objs.append(obj)
        if force or _stale(obj, src):
            cmd = [NVCC, *FLAGS, *EXTRA, *extra, "-c", src, "-o", obj]
            if verbose:
                print(" ".join(cmd))
            procs.append((oname, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    relink = force or bool(procs) or not os.path.exists(OUT)
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed for {s}:\n{out}")
        if verbose and out.strip():
            print(out)
    if relink:
        cmd = [NVCC, "-shared", "-o", OUT, *objs, *ARCH]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
