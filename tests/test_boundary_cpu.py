"""CPU: the C-ABI library loads and exports every symbol include/dinounet_b200.h declares; the host-side mirror has
the reference's state-dict keys and plugin hook; and the product fails loudly (no CPU fallback) without a GPU."""
import os
import re

import pytest
import torch

import dinounet_b200
from dinounet_b200 import config, lib
from oracle import dinounet_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built():
    import __graft_entry__
    __graft_entry__.build()
    return lib.load()


def test_library_exports_every_declared_symbol(built):
    hdr = open(os.path.join(ROOT, "include", "dinounet_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(b2u_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(built, name), f"{name} declared in the header but not exported"
    assert declared == set(lib.SIGNATURES), "ctypes signature table out of sync with the header"
    assert built.b2u_version() >= 1


def test_struct_layouts_match_header(tmp_path):
    """ctypes mirrors vs the real C layout: compile a probe against the header with gcc and compare every offset."""
    import ctypes as C
    import subprocess
    structs = {"b2u_epilogue": lib.Epilogue, "b2u_gemm_params": lib.GemmParams, "b2u_qkv_params": lib.QkvParams,
               "b2u_f32_gemm_params": lib.F32GemmParams}
    lines = []
    for cname, cls in structs.items():
        lines.append(f'printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    src = tmp_path / "probe.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "dinounet_b200.h"\nint main(){' + "".join(lines) + "return 0;}")
    exe = tmp_path / "probe"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    for cname, cls in structs.items():
        assert int(out[cname]) == C.sizeof(cls), cname
        for fname, _ in cls._fields_:
            assert int(out[f"{cname}.{fname}"]) == getattr(cls, fname).offset, f"{cname}.{fname}"


def _build(model):
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    return dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, 2, None, model)


@pytest.mark.parametrize("model", ["dinounet_s", "dinounet_b"])
def test_state_dict_keys_match_reference_spec(model):
    net = _build(model)
    sd = net.state_dict()
    ref = O.make_state_dict(model, 2, 0)
    assert set(sd) == set(ref)
    assert all(tuple(sd[k].shape) == tuple(ref[k].shape) for k in sd)
    net.load_state_dict(ref, strict=True)
    assert net.decoder.deep_supervision is False
    assert net.encoder.output_channels == [32, 64, 128, 256] and net.encoder.strides == [[2, 2]] * 4
    assert not any(p.requires_grad for p in net.encoder.dinov3_adapter.backbone.parameters())


def test_unknown_model_raises_like_reference():
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    with pytest.raises(ValueError):   # dinounet_training.py:737-738 (the default name is not a registry key)
        dinounet_b200.DinoUNet(network_config={"architecture": dict(config.DEFAULT_ARCHITECTURE)})


def test_missing_checkpoint_raises_without_network():
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "0"
    try:
        with pytest.raises(FileNotFoundError):
            dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, 2,
                                               "/nonexistent.pth", "dinounet_s")
    finally:
        os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"


def test_trainer_hook_builds_the_native_model():
    T = dinounet_b200.get_dinov3_trainer("dinounet_s")
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    T.set_network_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, dinov3_pretrained_path=None)
    net = T.build_network_architecture("DinoUNet", {}, [], 3, 2, enable_deep_supervision=False)
    assert isinstance(net, dinounet_b200.DinoUNet) and net.dinov3_model_name == "dinounet_s"
    with pytest.raises(ValueError):
        dinounet_b200.get_dinov3_trainer("dinov3_vits16")


def test_no_cpu_fallback(built):
    net = _build("dinounet_s").eval()
    with torch.no_grad(), pytest.raises(lib.NativeLibraryError):
        net(torch.zeros(1, 3, 64, 64))
    with pytest.raises(lib.NativeLibraryError):   # the training path (train_path.py) is CUDA-only as well
        net.train()(torch.zeros(1, 3, 64, 64))


def test_engine_rejects_unsupported_kernel_choices(built):
    from dinounet_b200.engine import ForwardEngine
    with pytest.raises(NotImplementedError):   # the wgmma attention kernel is the only one
        ForwardEngine("dinounet_7b", {}, 2, torch.device("cpu"), attn_impl="mma")
    with pytest.raises(ValueError):
        ForwardEngine("dinounet_xl", {}, 2, torch.device("cpu"))


def test_training_checkpoint_loads_into_the_b200_model(tmp_path):
    """A checkpoint in the reference's format (nnUNetTrainer.py:1093-1104), with the DataParallel / torch.compile key
    prefixes its loader tolerates (:1116-1121), loads strictly into the native module."""
    import os
    import torch
    import dinounet_b200
    from dinounet_b200 import config
    from oracle import dinounet_oracle as O
    os.environ["DINOUNET_B200_ALLOW_RANDOM_BACKBONE"] = "1"
    sd = O.make_state_dict("dinounet_s", 3, seed=2)
    for prefix in ("", "module.", "_orig_mod."):
        ckpt = {"network_weights": {prefix + k: v for k, v in sd.items()}, "optimizer_state": {}, "grad_scaler_state": None,
                "logging": {}, "_best_ema": 0.5, "current_epoch": 7, "init_args": {"fold": 0}, "trainer_name": "DinoUNetTrainer_s",
                "inference_allowed_mirroring_axes": (0, 1)}
        path = str(tmp_path / f"checkpoint_final{len(prefix)}.pth")
        torch.save(ckpt, path)
        net = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, 3, None, "dinounet_s")
        meta = dinounet_b200.load_network_weights(net, path)
        assert meta["trainer_name"] == "DinoUNetTrainer_s" and meta["inference_allowed_mirroring_axes"] == (0, 1)
        assert meta["current_epoch"] == 7
        got = net.state_dict()
        assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    import pytest
    with pytest.raises(KeyError):
        dinounet_b200.load_network_weights(net, {"state_dict": {}})


def test_engine_rejects_unsupported_patch_sizes_with_a_clear_error():
    """Host-side validation (no kernel runs): sizes the tiling does not cover raise ValueError, not a late kernel error."""
    import os
    import pytest
    import torch
    from dinounet_b200.engine import ForwardEngine
    from oracle import dinounet_oracle as O
    sd = {k: v for k, v in O.make_state_dict("dinounet_s", 2, seed=0).items() if not k.startswith("decoder.encoder.")}
    eng = ForwardEngine.__new__(ForwardEngine)          # build_plan's size check comes before any device work
    for S in (96, 160, 320, 500):
        with pytest.raises(ValueError, match="multiple of 128"):
            ForwardEngine.build_plan(eng, 1, S)


def test_discoverable_trainer_stub_is_found_by_the_reference_lookup(tmp_path):
    """find_class_by_name.py:7-24 walks <pkg>/training/nnUNetTrainer/*.py with pkgutil + importlib: the stub written by
    install_discoverable_trainers must expose the trainer classes there by name (restated lookup, same mechanism)."""
    import importlib
    import pkgutil
    import sys
    import dinounet_b200
    pkg = tmp_path / "fakeunet"
    tdir = pkg / "training" / "nnUNetTrainer"
    tdir.mkdir(parents=True)
    for d in (pkg, pkg / "training", tdir):
        (d / "__init__.py").write_text("")
    path = dinounet_b200.install_discoverable_trainers(str(pkg))
    assert path.endswith("DinoUNetTrainer_b200.py")
    sys.path.insert(0, str(tmp_path))
    try:
        found = None
        for _, modname, ispkg in pkgutil.iter_modules([str(tdir)]):     # == recursive_find_python_class
            if not ispkg:
                m = importlib.import_module("fakeunet.training.nnUNetTrainer." + modname)
                if hasattr(m, "DinoUNetTrainer_l"):
                    found = getattr(m, "DinoUNetTrainer_l")
        assert found is dinounet_b200.DinoUNetTrainer_l
    finally:
        sys.path.remove(str(tmp_path))


def test_label_export_reverts_cropping_and_transpose():
    """export_prediction.py:43-52 on GPU-side label maps."""
    import numpy as np
    from dinounet_b200.export import labels_to_original_geometry, needs_resampling
    rng = np.random.default_rng(0)
    labels = rng.integers(0, 3, size=(4, 6, 5)).astype(np.uint8)
    props = {"shape_after_cropping_and_before_resampling": (4, 6, 5), "shape_before_cropping": (7, 9, 8),
             "bbox_used_for_cropping": [[2, 6], [1, 7], [3, 8]]}
    seg = labels_to_original_geometry(torch.from_numpy(labels), props, (2, 0, 1), 2)
    ref = np.zeros((7, 9, 8), np.uint8)
    ref[2:6, 1:7, 3:8] = labels
    assert seg.dtype == np.uint8 and np.array_equal(seg, ref.transpose(2, 0, 1))
    assert needs_resampling((4, 6, 4), props)
    with pytest.raises(ValueError):
        labels_to_original_geometry(labels[:, :, :4], props, (0, 1, 2))
