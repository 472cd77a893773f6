"""Ensembling on the device (reference: `dinounet/ensembling/ensemble.py`).

Drop-ins with the reference's signatures and files: `average_probabilities`, `merge_files`, `ensemble_folders`,
`ensemble_crossvalidations` and `entry_point_ensemble_folders` (also `python -m dinounet_b200.ensembling -i ... -o ...`).
Reader threads decompress the members' `.npz` (zlib releases the GIL); each member goes to the device as soon as it is
read and is added in member order (`b2u_ensemble_accumulate`, bit-identical to numpy's float32 sum); one kernel
divides by the member count and segments the average (`b2u_ensemble_segment`); writer threads write the files.

`predict_ensemble_from_files` predicts with several trained models in one pass: each case is read and preprocessed
once, every member predicts its fold ensemble, and its probabilities are added on the device into one fp32 buffer
(`export.accumulate_probabilities`).  No member's probability volume is written or kept: the result equals predicting
every member with `save_probabilities` and running `ensemble_folders` on the outputs.
"""
import argparse
import os
import pickle
import shutil
import zipfile
from concurrent.futures import ThreadPoolExecutor
from typing import List, Tuple, Union

import numpy as np
import torch

from . import lib as L
from . import predict as PR
from .export import MAX_EXPORT_CHANNELS

default_num_processes = PR.DEFAULT_NUM_PROCESSES


def _load_json(path):
    return PR._load_json(path)


def _load_pickle(path):
    with open(path, "rb") as f:
        return pickle.load(f)


def _save_pickle(obj, path):
    with open(path, "wb") as f:
        pickle.dump(obj, f)


def _subfiles_npz(folder: str) -> List[str]:
    """batchgenerators' `subfiles(folder, suffix='.npz', join=False)`: file names, sorted."""
    return sorted(f for f in os.listdir(folder) if os.path.isfile(os.path.join(folder, f)) and f.endswith(".npz"))


def _npz_header(path: str):
    """(shape, dtype) of the `probabilities` array of an `.npz`, read from its header without decompressing it."""
    with zipfile.ZipFile(path) as z, z.open("probabilities.npy") as f:
        version = np.lib.format.read_magic(f)
        read = np.lib.format.read_array_header_1_0 if version == (1, 0) else np.lib.format.read_array_header_2_0
        shape, _, dtype = read(f)
    return tuple(shape), np.dtype(dtype)


def _check_members(lists_of_files, label_manager):
    """Every rejection before any launch: members must hold fp32 or fp16 probabilities of one shape whose channels are
    the label manager's heads, at most MAX_EXPORT_CHANNELS of them."""
    heads = label_manager.num_segmentation_heads
    for files in lists_of_files:
        assert len(files), 'At least one file must be given in list_of_files'
        headers = [_npz_header(f) for f in files]
        for f, (shape, dtype) in zip(files, headers):
            if dtype not in (np.dtype(np.float32), np.dtype(np.float16)):
                raise NotImplementedError(f"device ensembling takes fp32 or fp16 probabilities, {f} holds {dtype}")
            if len(shape) < 2 or shape[0] > MAX_EXPORT_CHANNELS:
                raise NotImplementedError(f"device ensembling handles [C, ...] probabilities with C <= "
                                          f"{MAX_EXPORT_CHANNELS}, {f} holds {shape}")
            if shape != headers[0][0]:
                raise ValueError(f"members of one case differ in shape: {files[0]} {headers[0][0]}, {f} {shape}")
        assert headers[0][0][0] == heads, \
            f'unexpected number of channels in predicted_probabilities. Expected {heads}, ' \
            f'got {headers[0][0][0]}. Remember that predicted_probabilities should have shape (c, x, y(, z)).'
        if label_manager.has_regions:
            assert label_manager.regions_class_order is not None, 'if region-based training is requested then you ' \
                                                                  'need to define regions_class_order!'


def _device() -> torch.device:
    return torch.device("cuda", torch.cuda.current_device())


def _accumulate(lib, acc: torch.Tensor, member: np.ndarray, first: bool, stream):
    src = torch.from_numpy(np.ascontiguousarray(member)).to(acc.device)
    L.check(lib.b2u_ensemble_accumulate(src.data_ptr(), src.element_size(), acc.data_ptr(), src.numel(), int(first),
                                        stream), "b2u_ensemble_accumulate")


def _segment(lib, acc: torch.Tensor, n_members: int, label_manager, stream) -> np.ndarray:
    """acc /= n_members in place and the segmentation of the average (uint8, or uint16 for >= 255 foreground labels),
    copied to the host."""
    has_regions = bool(label_manager.has_regions)
    label_bytes = 1 if len(label_manager.foreground_labels) < 255 else 2
    labels = torch.empty(acc.shape[1:], dtype=torch.uint8 if label_bytes == 1 else torch.int16, device=acc.device)
    region_labels = None
    if has_regions:
        region_labels = torch.tensor([int(c) for c in label_manager.regions_class_order], dtype=torch.int32,
                                     device=acc.device)
    L.check(lib.b2u_ensemble_segment(acc.data_ptr(), int(acc.shape[0]), int(np.prod(acc.shape[1:])), int(n_members),
                                     int(has_regions), None if region_labels is None else region_labels.data_ptr(),
                                     labels.data_ptr(), label_bytes, stream), "b2u_ensemble_segment")
    seg = labels.cpu().numpy()
    return seg.view(np.uint16) if label_bytes == 2 else seg


def _ensemble_cases(lists_of_files, outputs_truncated, file_ending: str, image_reader_writer, label_manager,
                    save_probabilities: bool, num_processes: int):
    """`merge_files` for every case: members read ahead by `num_processes` threads, accumulated on the device in
    member order as they arrive, each case averaged and segmented there and written by a writer thread (at most two
    cases queued beyond the writers)."""
    _check_members(lists_of_files, label_manager)
    if not lists_of_files:
        return
    lib = L.load()
    dev = _device()
    stream = torch.cuda.current_stream(dev)
    items = [(i, k, f) for i, files in enumerate(lists_of_files) for k, f in enumerate(files)]

    def read(item):
        return item, np.load(item[2])["probabilities"]

    def write(seg, probabilities, properties, ofile):
        image_reader_writer.write_seg(seg, ofile + file_ending, properties)
        if save_probabilities:
            np.savez_compressed(ofile + ".npz", probabilities=probabilities)
            _save_pickle(probabilities, ofile + ".pkl")   # the reference pickles the probabilities, not properties

    n_writers = max(1, int(num_processes))
    with ThreadPoolExecutor(n_writers) as writers, torch.cuda.device(dev):
        pending, acc, properties = [], None, None
        for (i, k, f), member in PR._read_ahead(read, items, num_processes):
            n = len(lists_of_files[i])
            if k == 0:
                properties = _load_pickle(f[:-4] + ".pkl")     # the first member's properties
                acc = torch.empty(member.shape, dtype=torch.float32, device=dev)
            _accumulate(lib, acc, member, k == 0, stream.cuda_stream)
            del member
            if k + 1 < n:
                continue
            while len([p for p in pending if not p.done()]) >= n_writers + 2:
                next(p for p in pending if not p.done()).result()
            seg = _segment(lib, acc, n, label_manager, stream.cuda_stream)
            probabilities = acc.cpu().numpy() if save_probabilities else None
            pending.append(writers.submit(write, seg, probabilities, properties, outputs_truncated[i]))
            acc = None
        for p in pending:
            p.result()


# ---------------------------------------------------------------------------------------------- the reference's API
def average_probabilities(list_of_files: List[str]) -> np.ndarray:
    """ensemble.py:17-29: the float32 mean of the members' `probabilities`, summed in list order."""
    assert len(list_of_files), 'At least one file must be given in list_of_files'
    shape, _ = _npz_header(list_of_files[0])
    lm = _PlainLabels(shape[0])
    _check_members([list_of_files], lm)
    lib = L.load()
    dev = _device()
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        acc = None
        for k, f in enumerate(list_of_files):
            member = np.load(f)["probabilities"]
            if acc is None:
                acc = torch.empty(member.shape, dtype=torch.float32, device=dev)
            _accumulate(lib, acc, member, k == 0, stream)
        _segment(lib, acc, len(list_of_files), lm, stream)
        return acc.cpu().numpy()


class _PlainLabels:
    """A label-map label manager of C heads: `average_probabilities` takes no label manager, and the segmentation the
    averaging kernel also writes is discarded there."""

    def __init__(self, heads: int):
        self.num_segmentation_heads = heads
        self.has_regions = False
        self.regions_class_order = None
        self.foreground_labels = list(range(1, heads))


def merge_files(list_of_files, output_filename_truncated: str, output_file_ending: str, image_reader_writer,
                label_manager, save_probabilities: bool = False):
    """ensemble.py:32-46 for one case: the segmentation of the members' average, written with the first member's
    properties; with `save_probabilities` the average as `.npz` and, as the reference does, pickled as `.pkl`."""
    _ensemble_cases([list(list_of_files)], [output_filename_truncated], output_file_ending, image_reader_writer,
                    label_manager, save_probabilities, 1)


def ensemble_folders(list_of_input_folders: List[str], output_folder: str, save_merged_probabilities: bool = False,
                     num_processes: int = default_num_processes, dataset_json_file_or_dict=None,
                     plans_json_file_or_dict=None):
    """ensemble.py:49-113: every `.npz` that all folders hold, ensembled into `output_folder`; `dataset.json` and
    `plans.json` default to the first folder's (not checked across folders), and the first folder's `dataset.json` is
    copied to the output."""
    if dataset_json_file_or_dict is None:
        dataset_json = _load_json(os.path.join(list_of_input_folders[0], "dataset.json"))
    elif isinstance(dataset_json_file_or_dict, str):
        dataset_json = _load_json(dataset_json_file_or_dict)
    else:
        dataset_json = dataset_json_file_or_dict
    if plans_json_file_or_dict is None:
        plans = _load_json(os.path.join(list_of_input_folders[0], "plans.json"))
    elif isinstance(plans_json_file_or_dict, str):
        plans = _load_json(plans_json_file_or_dict)
    else:
        plans = plans_json_file_or_dict
    plans_manager = PR._plans_manager(plans)

    files_per_folder = [set(_subfiles_npz(i)) for i in list_of_input_folders]
    s = set().union(*files_per_folder)
    for f in files_per_folder:
        assert len(s.difference(f)) == 0, "Not all folders contain the same files for ensembling. Please only " \
                                          "provide folders that contain the predictions"
    names = sorted(s)
    lists_of_lists_of_files = [[os.path.join(fl, fi) for fl in list_of_input_folders] for fi in names]
    output_files_truncated = [os.path.join(output_folder, fi[:-4]) for fi in names]

    image_reader_writer = plans_manager.image_reader_writer_class()
    label_manager = plans_manager.get_label_manager(dataset_json)
    os.makedirs(output_folder, exist_ok=True)
    shutil.copy(os.path.join(list_of_input_folders[0], "dataset.json"), output_folder)
    _ensemble_cases(lists_of_lists_of_files, output_files_truncated, dataset_json["file_ending"], image_reader_writer,
                    label_manager, save_merged_probabilities, num_processes)


def entry_point_ensemble_folders():
    parser = argparse.ArgumentParser()
    parser.add_argument('-i', nargs='+', type=str, required=True, help='list of input folders')
    parser.add_argument('-o', type=str, required=True, help='output folder')
    parser.add_argument('-np', type=int, required=False, default=default_num_processes,
                        help=f"Numbers of reader and writer threads used for ensembling. Default: {default_num_processes}")
    parser.add_argument('--save_npz', action='store_true', required=False, help='Set this flag to store output '
                                                                                'probabilities in separate .npz files')
    args = parser.parse_args()
    ensemble_folders(args.i, args.o, args.save_npz, args.np)


def ensemble_crossvalidations(list_of_trained_model_folders: List[str], output_folder: str,
                              folds: Union[Tuple[int, ...], List[int]] = (0, 1, 2, 3, 4),
                              num_processes: int = default_num_processes, overwrite: bool = True) -> None:
    """ensemble.py:131-206: the validation predictions (`fold_<k>/validation/*.npz`) of several trained model folders,
    ensembled case by case; `plans.json` and `dataset.json` of the first folder are copied to the output."""
    dataset_json = _load_json(os.path.join(list_of_trained_model_folders[0], "dataset.json"))
    plans_manager = PR._plans_manager(_load_json(os.path.join(list_of_trained_model_folders[0], "plans.json")))

    files_per_folder = {}
    unique_filenames = set()
    for tr in list_of_trained_model_folders:
        files_per_folder[tr] = {}
        for f in folds:
            val = os.path.join(tr, f'fold_{f}', 'validation')
            if not os.path.isdir(val):
                raise RuntimeError(f'Expected model output directory does not exist. You must train all requested '
                                   f'folds of the specified model.\nModel: {tr}\nFold: {f}')
            files_here = _subfiles_npz(val)
            if len(files_here) == 0:
                raise RuntimeError(f"No .npz files found in folder {val}. Rerun your "
                                   f"validation with the --npz flag. Use nnUNetv2_train [...] --val --npz.")
            files_per_folder[tr][f] = files_here
            unique_filenames.update(files_here)

    for tr, fi in files_per_folder.items():
        all_files_here = set()
        for f in folds:
            all_files_here.update(fi[f])
        diff = unique_filenames.difference(all_files_here)
        if len(diff) > 0:
            print(f'model {tr} does not seem to contain all predictions. Missing: {diff}')
            raise RuntimeError('There were missing files, see print statements above this one')

    file_mapping = []
    for tr in list_of_trained_model_folders:
        file_mapping.append({})
        for f in folds:
            for fi in files_per_folder[tr][f]:
                assert fi not in file_mapping[-1].keys(), f"Duplicate detected. Case {fi} is present in more than " \
                                                          f"one fold of model {tr}."
                file_mapping[-1][fi] = os.path.join(tr, f'fold_{f}', 'validation', fi)

    names = sorted(unique_filenames)
    lists_of_lists_of_files = [[fm[i] for fm in file_mapping] for i in names]
    output_files_truncated = [os.path.join(output_folder, fi[:-4]) for fi in names]

    image_reader_writer = plans_manager.image_reader_writer_class()
    os.makedirs(output_folder, exist_ok=True)
    label_manager = plans_manager.get_label_manager(dataset_json)

    if not overwrite:
        keep = [i for i, o in enumerate(output_files_truncated) if not os.path.isfile(o + dataset_json['file_ending'])]
        lists_of_lists_of_files = [lists_of_lists_of_files[i] for i in keep]
        output_files_truncated = [output_files_truncated[i] for i in keep]

    _ensemble_cases(lists_of_lists_of_files, output_files_truncated, dataset_json['file_ending'], image_reader_writer,
                    label_manager, False, num_processes)

    shutil.copy(os.path.join(list_of_trained_model_folders[0], 'plans.json'), os.path.join(output_folder, 'plans.json'))
    shutil.copy(os.path.join(list_of_trained_model_folders[0], 'dataset.json'),
                os.path.join(output_folder, 'dataset.json'))


# ---------------------------------------------------------------------------------------------- one-pass prediction
def _label_manager_key(lm):
    return {k: getattr(lm, k, None) for k in ("has_regions", "regions_class_order", "foreground_labels",
                                              "num_segmentation_heads")}


def check_same_setup(predictors):
    """Raises ValueError naming the first difference unless every predictor has the first one's plans, configuration
    and label manager."""
    if not predictors:
        raise ValueError("predict_ensemble_from_files needs at least one predictor")
    p0 = predictors[0]
    for i, p in enumerate(predictors[1:], 1):
        for what, a, b in (("plans", p0.plans_manager.plans, p.plans_manager.plans),
                           ("configuration", getattr(p0.configuration_manager, "configuration", None),
                            getattr(p.configuration_manager, "configuration", None)),
                           ("label manager", _label_manager_key(p0.label_manager), _label_manager_key(p.label_manager))):
            if a != b:
                keys = [k for k in (set(a) | set(b) if isinstance(a, dict) and isinstance(b, dict) else [])
                        if a.get(k) != b.get(k)]
                detail = f" (first differing key: {sorted(keys, key=str)[0]!r})" if keys else ""
                raise ValueError(f"ensemble members must share plans, configuration and label manager: member {i}'s "
                                 f"{what} differs from member 0's{detail}")


def predict_ensemble_from_files(predictors, list_of_lists_or_source_folder,
                                output_folder_or_list_of_truncated_output_files, save_probabilities: bool = False,
                                overwrite: bool = True, num_processes_preprocessing: int = default_num_processes,
                                num_processes_segmentation_export: int = default_num_processes, num_parts: int = 1,
                                part_id: int = 0):
    """`predict_from_files` with several trained models (`SlidingWindowPredictor`s, each initialised from a model
    folder, any variant and folds) in one pass.  Each case is read and preprocessed once with the first member's plans;
    every member predicts its fold ensemble and adds its probabilities (the export's resampling and softmax / sigmoid)
    into one fp32 buffer in member order; the average is segmented on the device and pasted into the original
    geometry.  Writes what `predict_from_files(..., save_probabilities=True)` per member followed by `ensemble_folders`
    writes (the segmentation and, with `save_probabilities`, the averaged probabilities as `.npz`), with the case's
    properties in `<case>.pkl`.  Without output names it returns the segmentations (and probabilities)."""
    from . import export
    from .engine import GRAPH_CAPTURE
    predictors = list(predictors)
    check_same_setup(predictors)
    for p in predictors:
        PR.check_no_previous_stage(p, None)
    p0 = predictors[0]
    args = dict(list_of_lists_or_source_folder=list_of_lists_or_source_folder,
                output_folder_or_list_of_truncated_output_files=output_folder_or_list_of_truncated_output_files,
                save_probabilities=save_probabilities, overwrite=overwrite,
                num_processes_preprocessing=num_processes_preprocessing,
                num_processes_segmentation_export=num_processes_segmentation_export, num_parts=num_parts,
                part_id=part_id, members=[p.trainer_name for p in predictors])
    cases = PR.cases_from_files(p0, list_of_lists_or_source_folder, output_folder_or_list_of_truncated_output_files,
                                save_probabilities, overwrite, num_processes_preprocessing, num_parts, part_id, args)
    if cases is None:
        return None
    pm, cm, lm, dj = p0.plans_manager, p0.configuration_manager, p0.label_manager, p0.dataset_json
    dev = PR._device(p0)
    stream = torch.cuda.current_stream(dev)
    n_fg = len(lm.foreground_labels)
    has_regions = bool(lm.has_regions)

    def predict(data, properties):
        acc = torch.empty((lm.num_segmentation_heads, *properties["shape_after_cropping_and_before_resampling"]),
                          dtype=torch.float32, device=dev)
        for k, p in enumerate(predictors):
            logits = p.predict_logits_from_preprocessed_data(data)
            export.accumulate_probabilities(logits, cm, lm, properties, acc, k == 0)
            del logits
        return acc

    def write(acc, properties, ofile):
        # outside the crop box every member's probabilities are exactly 1 / 0 (label maps) or 0 (regions): their
        # average is the same constants, which segment to 0, so pasting after averaging inside the box is exact
        with GRAPH_CAPTURE.device_work(), torch.cuda.stream(stream):
            seg = _segment(L.load(), acc, len(predictors), lm, stream.cuda_stream)
            probs = acc.cpu().numpy() if save_probabilities else None
        seg = export.labels_to_original_geometry(seg, properties, pm.transpose_backward, n_fg)
        if probs is not None:
            probs = export.probabilities_to_original_geometry(probs, properties, pm.transpose_backward, has_regions)
        if ofile is None:
            return (seg, probs) if save_probabilities else seg
        if save_probabilities:
            np.savez_compressed(ofile + ".npz", probabilities=probs)
            _save_pickle(properties, ofile + ".pkl")
        pm.image_reader_writer_class().write_seg(seg, ofile + dj["file_ending"], properties)
        return None

    return PR.run_cases(p0, cases, predict, write, num_processes_segmentation_export)


if __name__ == "__main__":
    entry_point_ensemble_folders()
