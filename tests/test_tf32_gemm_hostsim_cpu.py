"""CPU: the tf32 GEMM kernel's addressing, executed on the host.

csrc/gemm_tf32_addr.h holds every index computation of gemm_tf32_kernel (operand element per loader thread and mode,
swizzled shared-memory offset, K slicing, epilogue placement) as host/device functions; tests/native/tf32_hostsim.cpp runs
them for all 256 threads of every CTA and models the tensor core's read-out of the SWIZZLE_128B K-major tiles.  The test
bodies of tests/test_gpu_tf32_gemm.py (all modes, tails, split-K, remaps) run against that model here, so what is left for
the GPU run is the wgmma plumbing, not the arithmetic of addresses."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import pytest
import torch

import tests.test_gpu_tf32_gemm as G
from dinounet_b200 import lib as L
from tests.test_tf32_gemm_refs_cpu import _cases

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def hostsim():
    if shutil.which("g++") is None or not os.path.exists("/usr/local/cuda/include/vector_types.h"):
        pytest.skip("host model needs g++ and the CUDA headers (vector_types.h)")
    src = os.path.join(HERE, "native", "tf32_hostsim.cpp")
    out = os.path.join(tempfile.mkdtemp(prefix="b2u_hostsim_"), "tf32_hostsim.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I/usr/local/cuda/include", src, "-o", out], check=True)
    lib = C.CDLL(out)
    lib.tf32_hostsim_gemm.restype = C.c_char_p
    lib.tf32_hostsim_gemm.argtypes = [C.POINTER(L.F32GemmParams)]

    def raw_gemm(fn="b2u_tf32_gemm", **f):
        p = L.F32GemmParams()
        for k, v in f.items():
            setattr(p, k, v.data_ptr() if isinstance(v, torch.Tensor) else int(v))
        why = lib.tf32_hostsim_gemm(C.byref(p))
        assert why is None, why
    raw_gemm.modes = lambda reset=1: lib.tf32_hostsim_modes(reset)
    return raw_gemm


def test_kernel_addressing_on_the_host_model_all_modes(hostsim, monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(G, "raw_gemm", hostsim)
    monkeypatch.setattr(G, "TOL", 1e-5)
    ran = 0
    hostsim.modes()
    for fn in (G.test_plain_rows_bias_activation_residual, G.test_unaligned_leading_dimensions_take_the_scalar_paths,
               G.test_transposed_operands_and_split_k, G.test_conv3x3_forward_data_gradient_weight_gradient, G.test_conv3x3_channel_padding_rows_are_zero,
               G.test_pixel_shuffle_and_row_remap_epilogues):
        for kw in _cases(fn):
            fn(**kw)
            ran += 1
    assert ran >= 20
    assert hostsim.modes() == 15, "row AND block staging of both operands must have been exercised"


def test_host_model_rejects_what_the_entry_point_rejects(hostsim):
    A, W, out = torch.zeros(4, 4), torch.zeros(4, 4), torch.zeros(4, 4)
    with pytest.raises(AssertionError):
        hostsim(A=A, W=W, out=out, M=4, N=4, K=4, lda=4, ldw=4, ldc=4, ksplit=2, act1=L.ACT_RELU)     # split-K: raw products only
    with pytest.raises(AssertionError):
        hostsim(A=A, W=W, out=out, M=4, N=4, K=5, lda=4, ldw=4, ldc=4, conv=L.CONV3X3_S1, C=1, Cpad=1, Hin=2, Win=2)
