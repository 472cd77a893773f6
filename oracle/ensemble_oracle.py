"""numpy / torch-CPU restatement of the reference's ensembling (dinounet/ensembling/ensemble.py:17-46) and the
`LabelManager.convert_logits_to_segmentation` it calls (utilities/label_handling/label_handling.py:128-182).

`GOLDEN_CASES` are the cases of `tests/golden/ensemble_cases.npz` (oracle/make_golden_ensemble.py)."""
import os
import pickle

import numpy as np
import torch

REGION_ORDER = (1, 2, 3)


def average_probabilities(members) -> np.ndarray:
    """ensemble.py:17-29 on arrays: the first member as float32, `+=` of each later one, `/= len`."""
    avg = None
    for m in members:
        if avg is None:
            avg = np.array(m)
            if avg.dtype != np.float32:
                avg = avg.astype(np.float32)
        else:
            avg += m
    avg /= len(members)
    return avg


def convert_logits_to_segmentation(probabilities: np.ndarray, has_regions: bool, regions_class_order=None):
    """apply_inference_nonlin (torch CPU, float32) + convert_probabilities_to_segmentation, numpy in and out: int64
    argmax for label maps, uint16 regions painted in `regions_class_order`."""
    p = torch.from_numpy(probabilities).float()
    if has_regions:
        p = torch.sigmoid(p).numpy()
        seg = np.zeros(p.shape[1:], dtype=np.uint16)
        for i, c in enumerate(regions_class_order):
            seg[p[i] > 0.5] = c
        return seg
    return torch.softmax(p, 0).numpy().argmax(0)


def softmax_top2_ulps(probabilities: np.ndarray) -> np.ndarray:
    """Per voxel, the fp32 ulps between the two largest softmax values of the average (0 = a tie)."""
    p = torch.softmax(torch.from_numpy(probabilities).float(), 0).numpy()
    top = np.sort(p, axis=0)[-2:]
    return np.abs(top[1].view(np.int32).astype(np.int64) - top[0].view(np.int32).astype(np.int64))


def merge_files(list_of_files, output_filename_truncated, output_file_ending, image_reader_writer, label_manager,
                save_probabilities=False):
    """ensemble.py:32-46 with this module's arithmetic: reads the members' `.npz`, writes what the reference writes."""
    with open(list_of_files[0][:-4] + ".pkl", "rb") as f:
        properties = pickle.load(f)
    probabilities = average_probabilities([np.load(f)["probabilities"] for f in list_of_files])
    order = label_manager.regions_class_order if label_manager.has_regions else None
    segmentation = convert_logits_to_segmentation(probabilities, bool(label_manager.has_regions), order)
    image_reader_writer.write_seg(segmentation, output_filename_truncated + output_file_ending, properties)
    if save_probabilities:
        np.savez_compressed(output_filename_truncated + ".npz", probabilities=probabilities)
        with open(output_filename_truncated + ".pkl", "wb") as f:
            pickle.dump(probabilities, f)


# name, channels, regions, member dtypes, shape [Z, Y, X]
GOLDEN_CASES = (
    ("lab2_two", 2, False, ("f4", "f4"), (3, 17, 29)),
    ("lab4_three_f16", 4, False, ("f4", "f2", "f4"), (2, 33, 21)),
    ("lab4_four", 4, False, ("f4", "f4", "f4", "f4"), (4, 16, 40)),
    ("reg3_three", 3, True, ("f4", "f4", "f2"), (3, 24, 31)),
    ("reg3_two", 3, True, ("f4", "f4"), (2, 19, 37)),
)


def golden_members(case, seed: int):
    """Seeded member probabilities of a case: softmax (label maps) or sigmoid (regions) of random logits, with planted
    exact ties and near-ties of the top two channels, all-zero voxels, and region averages on both sides of
    1.5 * 2^-24 (where fp32 sigmoid(x) > 0.5 starts to hold)."""
    name, C, regions, dtypes, shape = case
    rng = np.random.default_rng(seed)
    members = []
    for k, dt in enumerate(dtypes):
        x = torch.from_numpy(rng.standard_normal((C, *shape)).astype(np.float32) * 3)
        p = (torch.sigmoid(x) if regions else torch.softmax(x, 0)).numpy()
        members.append(p)
    flat = [m.reshape(C, -1) for m in members]
    n = flat[0].shape[1]
    if regions:
        tiny = np.float32(1.5 * 2.0 ** -24)
        near = [tiny, np.nextafter(tiny, np.float32(1)), np.nextafter(tiny, np.float32(0)), np.float32(2.0 ** -23),
                np.float32(2.0 ** -24), np.float32(0)]
        for j, v in enumerate(near):
            for c in range(C):
                for m in range(len(flat)):
                    # every member equal: the average is v exactly; or only member 0 nonzero: the average is v / n
                    flat[m][c, j] = v
                    flat[m][c, 10 + j] = v * len(flat) if m == 0 else 0
    else:
        for j in range(8):                       # exact ties of the top two channels in every member
            for m in range(len(flat)):
                flat[m][:, j] = 0.0
                flat[m][0, j] = flat[m][C - 1, j] = 0.5
        for j in range(8, 16):                   # near-ties: a few ulps apart in the average
            for m in range(len(flat)):
                flat[m][:, j] = 0.0
                a = np.float32(0.5)
                flat[m][1, j] = a
                flat[m][0, j] = np.nextafter(a, np.float32(0)) if (m + j) % 2 else a
    for m in range(len(flat)):                   # all-zero voxels
        flat[m][:, n - 4:] = 0
    return [f.reshape(C, *shape).astype(dt) for f, dt in zip(flat, dtypes)]


def load_reference_ensemble_module():
    """The reference's `dinounet.ensembling.ensemble`, importable without its third-party dependencies: acvl_utils and
    batchgenerators' file helpers restated with `os` / pickle / json, and `dinounet.imageio` / `plans_handler` stubs
    (the module only names their classes)."""
    import importlib
    import json
    import sys
    import types
    from oracle import ref_loader
    # the stub packages must not outlive the import: other tests install their own stand-ins
    roots, meta_path, path = {m.split(".")[0] for m in sys.modules}, list(sys.meta_path), list(sys.path)
    try:
        ref_loader.load_reference_module()
        if "acvl_utils" not in sys.modules:
            for name in ("acvl_utils", "acvl_utils.cropping_and_padding"):
                sys.modules[name] = types.ModuleType(name)
            bb = types.ModuleType("acvl_utils.cropping_and_padding.bounding_boxes")
            bb.bounding_box_to_slice = lambda bbox: tuple(slice(*i) for i in bbox)
            sys.modules[bb.__name__] = bb
        if "batchgenerators" not in sys.modules:
            for name in ("batchgenerators", "batchgenerators.utilities"):
                sys.modules[name] = types.ModuleType(name)
            sys.modules[f"batchgenerators.utilities.file_and_folder_operations"] = types.ModuleType(
                "batchgenerators.utilities.file_and_folder_operations")
        fo = sys.modules["batchgenerators.utilities.file_and_folder_operations"]

        def load_json(p):
            with open(p) as f:
                return json.load(f)

        def load_pickle(p):
            with open(p, "rb") as f:
                return pickle.load(f)

        def save_pickle(o, p):
            with open(p, "wb") as f:
                pickle.dump(o, f)

        def subfiles(folder, join=True, prefix=None, suffix=None, sort=True):
            r = [os.path.join(folder, i) if join else i for i in os.listdir(folder)
                 if os.path.isfile(os.path.join(folder, i)) and (prefix is None or i.startswith(prefix))
                 and (suffix is None or i.endswith(suffix))]
            return sorted(r) if sort else r

        for k, v in dict(join=os.path.join, load_json=load_json, load_pickle=load_pickle, save_pickle=save_pickle,
                         subfiles=subfiles, isdir=os.path.isdir, isfile=os.path.isfile,
                         maybe_mkdir_p=lambda p: os.makedirs(p, exist_ok=True)).items():
            if not hasattr(fo, k):
                setattr(fo, k, v)
        for name, attrs in (("dinounet.configuration", {"default_num_processes": 3}),
                            ("dinounet.imageio.base_reader_writer", {"BaseReaderWriter": object}),
                            ("dinounet.utilities.plans_handling.plans_handler", {"PlansManager": object})):
            try:
                importlib.import_module(name)
            except Exception:
                m = types.ModuleType(name)
                for k, v in attrs.items():
                    setattr(m, k, v)
                sys.modules[name] = m
        label_handling = importlib.import_module("dinounet.utilities.label_handling.label_handling")
        return importlib.import_module("dinounet.ensembling.ensemble"), label_handling.LabelManager
    finally:
        for name in [m for m in sys.modules if m.split(".")[0] not in roots]:
            del sys.modules[name]
        sys.meta_path[:], sys.path[:] = meta_path, path
