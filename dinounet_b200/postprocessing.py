"""Keep-the-largest-component postprocessing on the device (reference: `dinounet/postprocessing/remove_connected_components.py`).

`remove_all_but_largest_component_from_segmentation` is the reference's function with its signature and output: the
union mask of the given labels or regions (read straight from the stored dtype, compared as numpy's `==`), its
components with full connectivity (skimage's `label(mask, connectivity=None)`: 26 neighbours in 3-D, 8 in 2-D, 2 in
1-D), and every masked voxel outside the largest components set to `background_label`; every component of the largest
size is kept (acvl-utils' `j == max(y)`).  One C-ABI call does it (`b2u_pp_largest_component`, csrc/postprocessing.cu);
its scratch is two int32 volumes.  A numpy array comes back as a numpy array of its dtype, a tensor as a new tensor on
its device, so the device export's labels can be postprocessed and scored (`evaluation.compute_metrics_arrays`) without
a host copy.

`determine_postprocessing` and `apply_postprocessing_to_folder` are drop-ins with the reference's signatures, printed
messages, `postprocessing.pkl`, `postprocessing.json` and `postprocessed/` folder.  They write no temporary folders:
every candidate is scored by one pass over the cases that reads each prediction and its reference once (threads read
the next cases meanwhile), applies the postprocessing accepted so far plus the candidate on the device and scores the
result there.  Only the final `postprocessed/` folder is written.
"""
from __future__ import annotations

import argparse
import json
import os
import pickle
import shutil

import numpy as np
import torch

from . import evaluation as EV
from . import lib as L

REFERENCE_MODULE = "dinounet.postprocessing.remove_connected_components"
MAX_VOXELS = 2 ** 31 - 1  # int32 component indices
NUMPY_DTYPES = {torch.uint8: np.uint8, torch.int8: np.int8, torch.int16: np.int16, torch.uint16: np.uint16,
                torch.int32: np.int32, torch.float32: np.float32}
_BITS = {1: np.uint8, 2: np.uint16, 4: np.uint32}


def _mask_labels(labels_or_regions) -> list:
    """The distinct label values whose union is the mask, ascending (region_or_label_to_mask over the list)."""
    if not isinstance(labels_or_regions, list):
        labels_or_regions = [labels_or_regions]
    values = set()
    for r in labels_or_regions:
        for v in ([r] if np.isscalar(r) else list(r)):
            if not isinstance(v, (int, np.integer)) or isinstance(v, (bool, np.bool_)):
                raise NotImplementedError(f"label {v!r} of {r!r}: only integer labels are supported")
            if not -2 ** 63 <= int(v) < 2 ** 63:
                raise NotImplementedError(f"label {v!r} of {r!r} does not fit in int64")
            values.add(int(v))
    return sorted(values)


def _background_bits(background_label, dtype: torch.dtype) -> int:
    """background_label stored in the segmentation's dtype, as its raw bits.  numpy itself converts it, so a Python int
    the dtype cannot hold raises OverflowError (numpy 2), whether or not a voxel would be written."""
    cell = np.zeros(1, NUMPY_DTYPES[dtype])
    cell[0] = background_label
    return int(cell.view(_BITS[cell.itemsize])[0])


def remove_all_but_largest_component_from_segmentation(segmentation, labels_or_regions, background_label: int = 0):
    """Drop-in for the reference's function (remove_connected_components.py:22-34) on a segmentation of rank 1 to 3:
    numpy arrays are processed on the current device and come back as numpy arrays, tensors come back as new tensors on
    their device.  The input is never modified."""
    t = EV._as_tensor(segmentation, "segmentation")
    if not 1 <= segmentation.ndim <= 3:   # before np.ascontiguousarray lifts a 0-d array to rank 1
        raise NotImplementedError(f"segmentation of rank {segmentation.ndim}: ranks 1 to 3 are supported")
    n = t.numel()
    if n > MAX_VOXELS:
        raise NotImplementedError(f"segmentation of {n} voxels: at most 2^31 - 1 are supported")
    labels = _mask_labels(labels_or_regions)
    background = _background_bits(background_label, t.dtype)
    if n == 0:
        return segmentation.copy() if isinstance(segmentation, np.ndarray) else t.clone()
    Z, Y, X = (1,) * (3 - t.dim()) + tuple(int(s) for s in t.shape)
    device = EV._device(t, t)
    lib = L.load()
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device).cuda_stream
        seg = EV._to_device(t, device)
        out = torch.empty_like(seg)
        work = torch.empty(2 * n + 1, dtype=torch.int32, device=device)
        values = torch.tensor(labels, dtype=torch.int64).to(device)
        L.check(lib.b2u_pp_largest_component(seg.data_ptr(), EV.DTYPE_CODES[t.dtype], Z, Y, X, values.data_ptr(),
                                             len(labels), background, out.data_ptr(), work.data_ptr(), stream),
                "b2u_pp_largest_component")
    if isinstance(segmentation, np.ndarray):
        return out.cpu().numpy()
    return out.to(t.device)


def _resolve(fn):
    """This module's function for the reference's (a postprocessing.pkl written by the reference), else fn."""
    if getattr(fn, "__module__", None) == REFERENCE_MODULE and \
            getattr(fn, "__name__", None) == "remove_all_but_largest_component_from_segmentation":
        return remove_all_but_largest_component_from_segmentation
    return fn


def apply_postprocessing(segmentation, pp_fns, pp_fn_kwargs):
    """The reference's `apply_postprocessing`; other functions than the keep-the-largest-component one receive numpy
    arrays and run as given."""
    for fn, kwargs in zip(pp_fns, pp_fn_kwargs):
        fn = _resolve(fn)
        if fn is not remove_all_but_largest_component_from_segmentation and isinstance(segmentation, torch.Tensor):
            segmentation = segmentation.cpu().numpy()
        segmentation = fn(segmentation, **kwargs)
    return segmentation


def _as_numpy(seg):
    return seg.cpu().numpy() if isinstance(seg, torch.Tensor) else seg


def _upload(seg: np.ndarray):
    """seg on the current device when its dtype is one the kernels read, else as it is."""
    if seg.dtype not in [np.dtype(d) for d in NUMPY_DTYPES.values()]:
        return seg
    return torch.from_numpy(np.ascontiguousarray(seg)).to(torch.device("cuda", torch.cuda.current_device()))


def _postprocess_on_device(seg, pp_fns, pp_fn_kwargs):
    """seg[0] of a case as read, uploaded once, through the chain."""
    return apply_postprocessing(_upload(seg[0]), pp_fns, pp_fn_kwargs)


def load_postprocess_save(segmentation_file: str, output_fname: str, image_reader_writer, pp_fns, pp_fn_kwargs):
    """The reference's `load_postprocess_save`, on the current device."""
    seg, props = image_reader_writer.read_seg(segmentation_file)
    seg = _as_numpy(_postprocess_on_device(seg, pp_fns, pp_fn_kwargs))
    image_reader_writer.write_seg(seg, output_fname, props)


# ---- folders ---------------------------------------------------------------------------------------------------------


def _plans_manager(plans_file_or_dict):
    """The host nnU-Net's PlansManager, which these drop-ins are called from."""
    from dinounet.utilities.plans_handling.plans_handler import PlansManager
    return PlansManager(plans_file_or_dict)


def _load_json(file: str):
    with open(file) as f:
        return json.load(f)


def _plans_and_dataset(folder, plans_file_or_dict, dataset_json_file_or_dict, plans_hint: str, dataset_hint: str):
    """remove_connected_components.py:71-90 / 258-279: the plans manager and dataset.json, from `folder` when None."""
    if plans_file_or_dict is None:
        expected_plans_file = os.path.join(folder, "plans.json")
        if not os.path.isfile(expected_plans_file):
            raise RuntimeError(f"Expected plans file missing: {expected_plans_file}. {plans_hint}")
        plans_file_or_dict = _load_json(expected_plans_file)
    plans_manager = _plans_manager(plans_file_or_dict)
    if dataset_json_file_or_dict is None:
        expected_dataset_json_file = os.path.join(folder, "dataset.json")
        if not os.path.isfile(expected_dataset_json_file):
            raise RuntimeError(f"Expected plans file missing: {expected_dataset_json_file}. {dataset_hint}")
        dataset_json_file_or_dict = _load_json(expected_dataset_json_file)
    if not isinstance(dataset_json_file_or_dict, dict):
        dataset_json = _load_json(dataset_json_file_or_dict)
    else:
        dataset_json = dataset_json_file_or_dict
    return plans_manager, dataset_json


def apply_postprocessing_to_folder(input_folder: str, output_folder: str, pp_fns, pp_fn_kwargs,
                                   plans_file_or_dict=None, dataset_json_file_or_dict=None, num_processes=8) -> None:
    """Drop-in for the reference's `apply_postprocessing_to_folder`: the cases in order on the current device, while
    `num_processes` threads read the next ones.  Accepts a postprocessing.pkl written by the reference (its
    keep-the-largest-component function runs through this module's)."""
    plans_manager, dataset_json = _plans_and_dataset(
        input_folder, plans_file_or_dict, dataset_json_file_or_dict,
        "The plans file should have been created while running nnUNetv2_predict. Sadge. If the folder you want to apply "
        "postprocessing to was create from an ensemble then just specify one of the plans files of the ensemble members "
        "in plans_file_or_dict",
        "The dataset.json should have been copied while running nnUNetv2_predict/nnUNetv2_ensemble. Sadge.")
    rw = plans_manager.image_reader_writer_class()
    os.makedirs(output_folder, exist_ok=True)
    files = EV._subfiles(input_folder, dataset_json["file_ending"])
    for f, (seg, props) in zip(files, EV.read_ahead(len(files), lambda i: rw.read_seg(os.path.join(input_folder, files[i])),
                                                     num_processes)):
        rw.write_seg(_as_numpy(_postprocess_on_device(seg, pp_fns, pp_fn_kwargs)), os.path.join(output_folder, f), props)


def determine_postprocessing(folder_predictions: str, folder_ref: str, plans_file_or_dict, dataset_json_file_or_dict,
                             num_processes: int = EV.DEFAULT_NUM_PROCESSES, keep_postprocessed_files: bool = True):
    """Drop-in for the reference's `determine_postprocessing` (remove_connected_components.py:53-245): the same
    decisions, messages, postprocessing.pkl / .json and postprocessed/ folder, with every candidate scored on the
    current device from the original predictions (see the module docstring)."""
    output_folder = os.path.join(folder_predictions, "postprocessed")
    hint = "The plans files should have been created while running nnUNetv2_predict. Sadge."
    plans_manager, dataset_json = _plans_and_dataset(folder_predictions, plans_file_or_dict, dataset_json_file_or_dict,
                                                     hint, hint)
    rw = plans_manager.image_reader_writer_class()
    label_manager = plans_manager.get_label_manager(dataset_json)
    labels_or_regions = label_manager.foreground_regions if label_manager.has_regions else \
        label_manager.foreground_labels
    file_ending = dataset_json["file_ending"]
    predicted_files = EV._subfiles(folder_predictions, file_ending)
    ref_files = EV._subfiles(folder_ref, file_ending)
    if not all([i in predicted_files for i in ref_files]):
        print("WARNING: Not all files in folder_ref were found in folder_predictions. Determining postprocessing "
              "should always be done on the entire dataset!")
    summary_file = os.path.join(folder_predictions, "summary.json")
    if not os.path.isfile(summary_file):
        EV.compute_metrics_on_folder(folder_ref, folder_predictions, summary_file, rw, file_ending, labels_or_regions,
                                     label_manager.ignore_label, num_processes)

    def evaluate(pp_fns, pp_fn_kwargs, name):
        """The summary the reference computes over its temporary folder `name` (case paths included), and that summary
        as `load_summary_json` returns it."""
        folder_here = os.path.join(output_folder, "temp", name)

        def read(i):
            return (rw.read_seg(os.path.join(folder_ref, predicted_files[i])),
                    rw.read_seg(os.path.join(folder_predictions, predicted_files[i])))

        results = []
        for f, ((seg_ref, ref_props), (seg, props)) in zip(predicted_files,
                                                            EV.read_ahead(len(predicted_files), read, num_processes)):
            seg = _postprocess_on_device(seg, pp_fns, pp_fn_kwargs)
            seg = seg.unsqueeze(0) if isinstance(seg, torch.Tensor) else seg[None]
            results.append(EV._score(os.path.join(folder_ref, f), os.path.join(folder_here, f),
                                     ((seg_ref, ref_props), (seg, props)), labels_or_regions,
                                     label_manager.ignore_label))
        summary = EV.aggregate(results, labels_or_regions)
        return summary, EV.summary_keys_from_json(json.loads(EV.summary_text(summary)))

    pp_fns, pp_fn_kwargs = [], []
    source = None  # (summary, loaded summary) of the accepted postprocessing; None: the predictions as they are

    pp_fn = remove_all_but_largest_component_from_segmentation
    kwargs = {"labels_or_regions": label_manager.foreground_labels}
    summary, pp_results = evaluate([pp_fn], [kwargs], "keep_largest_fg")
    baseline_results = EV.load_summary_json(summary_file)
    do_this = pp_results["foreground_mean"]["Dice"] > baseline_results["foreground_mean"]["Dice"]
    if do_this:
        for class_id in pp_results["mean"].keys():
            if pp_results["mean"][class_id]["Dice"] < baseline_results["mean"][class_id]["Dice"]:
                do_this = False
                break
    if do_this:
        print(f"Results were improved by removing all but the largest foreground region. "
              f"Mean dice before: {round(baseline_results['foreground_mean']['Dice'], 5)} "
              f"after: {round(pp_results['foreground_mean']['Dice'], 5)}")
        source = (summary, pp_results)
        pp_fns.append(pp_fn)
        pp_fn_kwargs.append(kwargs)
    else:
        print("Removing all but the largest foreground region did not improve results!")

    if len(labels_or_regions) > 1:
        for label_or_region in labels_or_regions:
            kwargs = {"labels_or_regions": label_or_region}
            summary, pp_results = evaluate(pp_fns + [pp_fn], pp_fn_kwargs + [kwargs],
                                           "keep_largest_perClassOrRegion")
            baseline_results = EV.load_summary_json(summary_file) if source is None else source[1]
            do_this = pp_results["mean"][label_or_region]["Dice"] > baseline_results["mean"][label_or_region]["Dice"]
            if do_this:
                print(f"Results were improved by removing all but the largest component for {label_or_region}. "
                      f"Dice before: {round(baseline_results['mean'][label_or_region]['Dice'], 5)} "
                      f"after: {round(pp_results['mean'][label_or_region]['Dice'], 5)}")
                source = (summary, pp_results)
                pp_fns.append(pp_fn)
                pp_fn_kwargs.append(kwargs)
            else:
                print(f"Removing all but the largest component for {label_or_region} did not improve results! "
                      f"Dice before: {round(baseline_results['mean'][label_or_region]['Dice'], 5)} "
                      f"after: {round(pp_results['mean'][label_or_region]['Dice'], 5)}")

    if keep_postprocessed_files:
        os.makedirs(output_folder, exist_ok=True)
        if source is None:
            for f in EV._subfiles(folder_predictions, ""):
                shutil.copy(os.path.join(folder_predictions, f), os.path.join(output_folder, f))
        else:
            apply_postprocessing_to_folder(folder_predictions, output_folder, pp_fns, pp_fn_kwargs, plans_file_or_dict,
                                           dataset_json, num_processes)
            EV.save_summary_json(source[0], os.path.join(output_folder, "summary.json"))
    with open(os.path.join(folder_predictions, "postprocessing.pkl"), "wb") as f:
        pickle.dump((pp_fns, pp_fn_kwargs), f)

    baseline_results = EV.load_summary_json(summary_file)
    final_results = baseline_results if source is None else source[1]
    tmp = {
        "input_folder": {i: baseline_results[i] for i in ["foreground_mean", "mean"]},
        "postprocessed": {i: final_results[i] for i in ["foreground_mean", "mean"]},
        "postprocessing_fns": [i.__name__ for i in pp_fns],
        "postprocessing_kwargs": pp_fn_kwargs,
    }
    tmp["input_folder"]["mean"] = {str(k): tmp["input_folder"]["mean"][k] for k in tmp["input_folder"]["mean"].keys()}
    tmp["postprocessed"]["mean"] = {str(k): tmp["postprocessed"]["mean"][k] for k in
                                    tmp["postprocessed"]["mean"].keys()}
    EV.fix_for_json_export(tmp)
    with open(os.path.join(folder_predictions, "postprocessing.json"), "w") as f:
        json.dump(tmp, f, sort_keys=True, indent=4)

    if not keep_postprocessed_files and os.path.isdir(output_folder):
        shutil.rmtree(output_folder)
    return pp_fns, pp_fn_kwargs


# ---- command lines (nnUNetv2_determine_postprocessing / nnUNetv2_apply_postprocessing) --------------------------------


def entry_point_determine_postprocessing_folder():
    parser = argparse.ArgumentParser("Writes postprocessing.pkl and postprocessing.json in input_folder.")
    parser.add_argument("-i", type=str, required=True, help="Input folder")
    parser.add_argument("-ref", type=str, required=True, help="Folder with gt labels")
    parser.add_argument("-plans_json", type=str, required=False, default=None,
                        help="plans file to use. If not specified we will look for the plans.json file in the "
                             "input folder (input_folder/plans.json)")
    parser.add_argument("-dataset_json", type=str, required=False, default=None,
                        help="dataset.json file to use. If not specified we will look for the dataset.json file in the "
                             "input folder (input_folder/dataset.json)")
    parser.add_argument("-np", type=int, required=False, default=EV.DEFAULT_NUM_PROCESSES,
                        help=f"number of processes to use. Default: {EV.DEFAULT_NUM_PROCESSES}")
    parser.add_argument("--remove_postprocessed", action="store_true", required=False,
                        help="set this is you don't want to keep the postprocessed files")
    args = parser.parse_args()
    determine_postprocessing(args.i, args.ref, args.plans_json, args.dataset_json, args.np,
                             not args.remove_postprocessed)


def entry_point_apply_postprocessing():
    parser = argparse.ArgumentParser("Apples postprocessing specified in pp_pkl_file to input folder.")
    parser.add_argument("-i", type=str, required=True, help="Input folder")
    parser.add_argument("-o", type=str, required=True, help="Output folder")
    parser.add_argument("-pp_pkl_file", type=str, required=True, help="postprocessing.pkl file")
    parser.add_argument("-np", type=int, required=False, default=EV.DEFAULT_NUM_PROCESSES,
                        help=f"number of processes to use. Default: {EV.DEFAULT_NUM_PROCESSES}")
    parser.add_argument("-plans_json", type=str, required=False, default=None,
                        help="plans file to use. If not specified we will look for the plans.json file in the "
                             "input folder (input_folder/plans.json)")
    parser.add_argument("-dataset_json", type=str, required=False, default=None,
                        help="dataset.json file to use. If not specified we will look for the dataset.json file in the "
                             "input folder (input_folder/dataset.json)")
    args = parser.parse_args()
    with open(args.pp_pkl_file, "rb") as f:
        pp_fns, pp_fn_kwargs = pickle.load(f)
    apply_postprocessing_to_folder(args.i, args.o, pp_fns, pp_fn_kwargs, args.plans_json, args.dataset_json, args.np)
