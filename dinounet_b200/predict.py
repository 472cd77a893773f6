"""Predicting new cases with a trained model folder: the model-folder and file handling of the reference's
`nnUNetPredictor` (inference/predict_from_raw_data.py:67-130, 158-266, 343-424) around `SlidingWindowPredictor`.

`initialize_from_trained_model_folder` builds the native `DinoUNet` from `plans.json`, `dataset.json` and the fold
checkpoints, `predict_from_files` / `predict_from_list_of_npy_arrays` run a list of cases: threads read the images
ahead with the plans' reader-writer, `DevicePreprocessor.run_case_npy` preprocesses on the device, the fold ensemble runs
there too (one ViT pass per tile batch for folds that share the backbone), and writer threads export each case on the
prediction's stream while the next one is predicted.  2-D configurations only; the cascade is not implemented.
"""
import copy
import json
import os
import re
from concurrent.futures import ThreadPoolExecutor
from typing import List, Sequence

import numpy as np
import torch

#: writer / reader threads when the caller does not say (the reference's `default_num_processes`)
DEFAULT_NUM_PROCESSES = 3


def _plans_manager(plans: dict):
    """The reference's `PlansManager` for a plans dict.  Tests substitute it."""
    from dinounet.utilities.plans_handling.plans_handler import PlansManager
    return PlansManager(plans)


def _load_json(path: str):
    with open(path) as f:
        return json.load(f)


def _save_json(obj, path: str, sort_keys: bool = True):
    with open(path, "w") as f:
        json.dump(obj, f, sort_keys=sort_keys, indent=4)


def auto_detect_available_folds(model_training_output_dir: str, checkpoint_name: str) -> List[int]:
    """The `fold_<k>` folders (not `fold_all`) that hold `checkpoint_name`, in name order."""
    names = sorted(n for n in os.listdir(model_training_output_dir)
                   if n.startswith("fold_") and os.path.isdir(os.path.join(model_training_output_dir, n)))
    names = [n for n in names if n != "fold_all"
             and os.path.isfile(os.path.join(model_training_output_dir, n, checkpoint_name))]
    return [int(n.split("_")[-1]) for n in names]


def variant_from_trainer_name(trainer_name: str) -> str:
    """The model variant of a native trainer class name (`DinoUNetTrainer_l` -> `dinounet_l`)."""
    from .training import DINOV3_TRAINERS
    for variant, cls in DINOV3_TRAINERS.items():
        if cls.__name__ == trainer_name:
            return variant
    raise ValueError(f"unknown trainer {trainer_name!r}: the checkpoints must come from one of "
                     f"{[c.__name__ for c in DINOV3_TRAINERS.values()]}")


def network_config_from_configuration(configuration_manager) -> dict:
    """The `network_config` the Dino U-Net trainers are given for a configuration (dinounet/api.py:91-110): the
    architecture entries of `network_arch_init_kwargs`, with the same defaults, and the data configuration."""
    arch_kwargs = dict(configuration_manager.network_arch_init_kwargs or {})
    return {
        "architecture": {
            "network_class_name": configuration_manager.network_arch_class_name or "",
            "n_stages": arch_kwargs.get("n_stages", 0),
            "features_per_stage": arch_kwargs.get("features_per_stage", []),
            "kernel_sizes": arch_kwargs.get("kernel_sizes", []),
            "strides": arch_kwargs.get("strides", []),
            "n_conv_per_stage": arch_kwargs.get("n_conv_per_stage", []),
            "n_conv_per_stage_decoder": arch_kwargs.get("n_conv_per_stage_decoder", []),
            "conv_op": arch_kwargs.get("conv_op", ""),
            "norm_op": arch_kwargs.get("norm_op", ""),
            "nonlin": arch_kwargs.get("nonlin", ""),
            "conv_bias": arch_kwargs.get("conv_bias", True),
            "dropout_op": arch_kwargs.get("dropout_op", None),
            "norm_op_kwargs": arch_kwargs.get("norm_op_kwargs", {}),
            "nonlin_kwargs": arch_kwargs.get("nonlin_kwargs", {}),
            "dropout_op_kwargs": arch_kwargs.get("dropout_op_kwargs", {}),
        },
        "data_config": {
            "batch_size": getattr(configuration_manager, "batch_size", None),
            "patch_size": getattr(configuration_manager, "patch_size", []),
            "spacing": getattr(configuration_manager, "spacing", []),
            "median_image_size_in_voxels": getattr(configuration_manager, "median_image_size_in_voxels", []),
        },
    }


def num_input_channels(dataset_json: dict) -> int:
    """Input channels of a configuration without a previous stage: one per `channel_names` (or legacy `modality`)."""
    names = dataset_json["channel_names"] if "channel_names" in dataset_json else dataset_json["modality"]
    return len(names)


def load_model_folder(model_training_output_dir: str, use_folds, checkpoint_name: str = "checkpoint_final.pth"):
    """(plans_manager, configuration_manager, dataset_json, parameters, trainer_name, configuration name,
    mirroring axes) of a trained model folder.  use_folds: None = every fold found, "all" = `fold_all`, or a sequence of
    fold numbers / "all"."""
    if use_folds is None:
        use_folds = auto_detect_available_folds(model_training_output_dir, checkpoint_name)
        if not use_folds:
            raise FileNotFoundError(f"no fold_<k>/{checkpoint_name} in {model_training_output_dir}")
    if isinstance(use_folds, str):
        use_folds = [use_folds]
    dataset_json = _load_json(os.path.join(model_training_output_dir, "dataset.json"))
    plans = _load_json(os.path.join(model_training_output_dir, "plans.json"))
    parameters, trainer_name, configuration, mirror_axes = [], None, None, None
    for i, f in enumerate(use_folds):
        f = int(f) if f != "all" else f
        path = os.path.join(model_training_output_dir, f"fold_{f}", checkpoint_name)
        if not os.path.isfile(path):
            raise FileNotFoundError(f"fold {f}: {path} does not exist")
        ckpt = torch.load(path, map_location=torch.device("cpu"), weights_only=False)
        if i == 0:
            trainer_name = ckpt["trainer_name"]
            configuration = ckpt["init_args"]["configuration"]
            mirror_axes = ckpt.get("inference_allowed_mirroring_axes")
        parameters.append(ckpt["network_weights"])
    plans_manager = _plans_manager(plans)
    configuration_manager = plans_manager.get_configuration(configuration)
    return plans_manager, configuration_manager, dataset_json, parameters, trainer_name, configuration, mirror_axes


def build_network(trainer_name: str, configuration_manager, input_channels: int, num_heads: int):
    """The native `DinoUNet` a trainer of that name trains for that configuration, without deep supervision.  Its
    backbone is not read from a pretrained file: the checkpoints carry it."""
    from .network_architecture import DinoUNet
    from .network_architecture.modules import BACKBONE_FROM_CHECKPOINT
    variant = variant_from_trainer_name(trainer_name)
    config = network_config_from_configuration(configuration_manager)
    config["architecture"]["deep_supervision"] = False
    return DinoUNet.from_config(network_config=config, input_channels=input_channels, num_classes=num_heads,
                                dinov3_pretrained_path=BACKBONE_FROM_CHECKPOINT, dinov3_model_name=variant)


# ---------------------------------------------------------------------------------------------- input / output lists
def create_lists_from_splitted_dataset_folder(folder: str, file_ending: str) -> List[List[str]]:
    """One list per case identifier of `folder`: its files `<id>_<4 digits><file_ending>`, in name order, identifiers
    in name order."""
    files = sorted(f for f in os.listdir(folder) if f.endswith(file_ending) and os.path.isfile(os.path.join(folder, f)))
    crop = len(file_ending) + 5
    identifiers = sorted({f[:-crop] for f in files})
    out = []
    for case in identifiers:
        pattern = re.compile(re.escape(case) + r"_\d\d\d\d" + re.escape(file_ending))
        out.append([os.path.join(folder, f) for f in files if pattern.fullmatch(f)])
    return out


def manage_input_and_output_lists(list_of_lists_or_source_folder, output_folder_or_list_of_truncated_output_files,
                                  file_ending: str, overwrite: bool = True, part_id: int = 0, num_parts: int = 1,
                                  save_probabilities: bool = False):
    """(list of input file lists, truncated output names) of this part (`[part_id::num_parts]`), without the cases
    whose outputs exist when `overwrite` is False (with `save_probabilities`, the `.npz` must exist too)."""
    if isinstance(list_of_lists_or_source_folder, str):
        list_of_lists_or_source_folder = create_lists_from_splitted_dataset_folder(list_of_lists_or_source_folder,
                                                                                   file_ending)
    lists = list(list_of_lists_or_source_folder)[part_id::num_parts]
    caseids = [os.path.basename(files[0])[:-(len(file_ending) + 5)] for files in lists]
    outputs = output_folder_or_list_of_truncated_output_files
    if isinstance(outputs, str):
        outputs = [os.path.join(outputs, c) for c in caseids]
    if not overwrite and outputs is not None:
        done = [os.path.isfile(o + file_ending) and (not save_probabilities or os.path.isfile(o + ".npz"))
                for o in outputs]
        keep = [i for i, d in enumerate(done) if not d]
        lists = [lists[i] for i in keep]
        outputs = [outputs[i] for i in keep]
    return lists, outputs


# ---------------------------------------------------------------------------------------------- the prediction loop
def predict_cases(predictor, cases, save_probabilities: bool, num_writers: int):
    """cases yields (image [C, X, Y, Z] numpy, properties, truncated output name or None).  Each case is preprocessed
    and predicted on the device; a case with an output name is exported by a writer thread on the prediction's
    stream (at most two cases queued beyond the writers), one without is converted and returned as the reference
    returns it: the segmentation, or (segmentation, probabilities) with `save_probabilities`."""
    from . import export
    from .engine import GRAPH_CAPTURE
    stream = torch.cuda.current_stream(_device(predictor))
    pm, cm, dj = predictor.plans_manager, predictor.configuration_manager, predictor.dataset_json

    def write(logits, properties, ofile):
        # a case whose weights must be repacked captures new CUDA graphs while earlier cases are being exported
        with GRAPH_CAPTURE.device_work(), torch.cuda.stream(stream):
            if ofile is not None:
                export.export_prediction_from_logits(logits, properties, cm, pm, dj, ofile, save_probabilities)
                return None
            return export.convert_predicted_logits_to_segmentation_with_correct_shape(
                logits, pm, cm, predictor.label_manager, properties, return_probabilities=save_probabilities)

    return run_cases(predictor, cases, lambda data, properties: predictor.predict_logits_from_preprocessed_data(data),
                     write, num_writers)


def _device(predictor) -> torch.device:
    return predictor.device if predictor.device.index is not None else torch.device("cuda", torch.cuda.current_device())


def run_cases(predictor, cases, predict, write, num_writers: int):
    """The prediction loop: each case of `cases` ((image, properties, truncated output name or None)) is preprocessed
    on the device with `predictor`'s plans, `predict(data, properties)` runs on the main thread, and
    `write(result, properties, output name)` in one of `num_writers` writer threads, with at most two cases queued
    beyond the writers.  Returns the writers' results in case order."""
    from .preprocess import DevicePreprocessor
    pre = DevicePreprocessor(predictor.verbose_preprocessing, _device(predictor))
    pm, cm, dj = predictor.plans_manager, predictor.configuration_manager, predictor.dataset_json
    with ThreadPoolExecutor(max(1, num_writers)) as writers:
        pending = []
        for image, properties, ofile in cases:
            while len([p for p in pending if not p.done()]) >= max(1, num_writers) + 2:
                next(p for p in pending if not p.done()).result()
            if predictor.verbose:
                print(f"predicting {os.path.basename(ofile) if ofile is not None else 'image'} of shape {image.shape}")
            data, _ = pre.run_case_npy(image, None, properties, pm, cm, dj)
            result = predict(data, properties)
            pending.append(writers.submit(write, result, properties, ofile))
            del result, data
        results = [p.result() for p in pending]
    return results


def check_no_previous_stage(predictor, segs_from_prev_stage):
    """Raises NotImplementedError for the cascade: a configuration with a previous stage, or segmentations of one (a
    folder, an array, or a list holding anything but None; a list of Nones means none, as in the reference)."""
    segs = segs_from_prev_stage
    if isinstance(segs, (list, tuple)) and all(s is None for s in segs):
        segs = None
    if segs is not None or getattr(predictor.configuration_manager, "previous_stage_name", None) is not None:
        raise NotImplementedError("the cascade (segmentations of a previous stage) is not implemented on the device")


def _read_ahead(read, items: Sequence, num_threads: int):
    """Yields read(item) in order, with `num_threads` threads reading up to that many items ahead."""
    n = max(1, int(num_threads))
    with ThreadPoolExecutor(n) as pool:
        futures = [pool.submit(read, item) for item in items[:n]]
        for i in range(len(items)):
            if i + n < len(items):
                futures.append(pool.submit(read, items[i + n]))
            yield futures[i].result()
            futures[i] = None


def predict_from_files(predictor, list_of_lists_or_source_folder, output_folder_or_list_of_truncated_output_files,
                       save_probabilities: bool = False, overwrite: bool = True,
                       num_processes_preprocessing: int = DEFAULT_NUM_PROCESSES,
                       num_processes_segmentation_export: int = DEFAULT_NUM_PROCESSES,
                       folder_with_segs_from_prev_stage: str = None, num_parts: int = 1, part_id: int = 0):
    check_no_previous_stage(predictor, folder_with_segs_from_prev_stage)
    args = dict(list_of_lists_or_source_folder=list_of_lists_or_source_folder,
                output_folder_or_list_of_truncated_output_files=output_folder_or_list_of_truncated_output_files,
                save_probabilities=save_probabilities, overwrite=overwrite,
                num_processes_preprocessing=num_processes_preprocessing,
                num_processes_segmentation_export=num_processes_segmentation_export,
                folder_with_segs_from_prev_stage=folder_with_segs_from_prev_stage, num_parts=num_parts, part_id=part_id)
    cases = cases_from_files(predictor, list_of_lists_or_source_folder, output_folder_or_list_of_truncated_output_files,
                             save_probabilities, overwrite, num_processes_preprocessing, num_parts, part_id, args)
    if cases is None:
        return None
    return predict_cases(predictor, cases, save_probabilities, num_processes_segmentation_export)


def cases_from_files(predictor, list_of_lists_or_source_folder, output_folder_or_list_of_truncated_output_files,
                     save_probabilities: bool, overwrite: bool, num_processes_preprocessing: int, num_parts: int,
                     part_id: int, args: dict):
    """The file side of `predict_from_files`: writes `args`, `dataset.json` and `plans.json` to the output folder,
    selects this part's cases (skipping finished ones unless `overwrite`) and returns the read-ahead generator of
    (image, properties, truncated output name or None) that `run_cases` takes, or None when no case is left."""
    outputs = output_folder_or_list_of_truncated_output_files
    if isinstance(outputs, str):
        output_folder = outputs
    elif isinstance(outputs, list):
        output_folder = os.path.dirname(outputs[0])
    else:
        output_folder = None
    if output_folder is not None:
        os.makedirs(output_folder, exist_ok=True)
        _save_json(_jsonable(copy.deepcopy(args)), os.path.join(output_folder, "predict_from_raw_data_args.json"))
        _save_json(predictor.dataset_json, os.path.join(output_folder, "dataset.json"), sort_keys=False)
        _save_json(predictor.plans_manager.plans, os.path.join(output_folder, "plans.json"), sort_keys=False)
    lists, ofiles = manage_input_and_output_lists(list_of_lists_or_source_folder, outputs,
                                                  predictor.dataset_json["file_ending"], overwrite, part_id, num_parts,
                                                  save_probabilities)
    if not lists:
        return None
    if ofiles is None:
        ofiles = [None] * len(lists)
    rw = predictor.plans_manager.image_reader_writer_class()

    def read(item):
        files, ofile = item
        data, properties = rw.read_images(files)
        return np.asarray(data, dtype=np.float32), properties, ofile

    return _read_ahead(read, list(zip(lists, ofiles)), num_processes_preprocessing)


def predict_from_list_of_npy_arrays(predictor, image_or_list_of_images, segs_from_prev_stage_or_list_of_segs_from_prev_stage,
                                    properties_or_list_of_properties, truncated_ofname, num_processes: int = 3,
                                    save_probabilities: bool = False,
                                    num_processes_segmentation_export: int = DEFAULT_NUM_PROCESSES):
    check_no_previous_stage(predictor, segs_from_prev_stage_or_list_of_segs_from_prev_stage)
    images = image_or_list_of_images if isinstance(image_or_list_of_images, list) else [image_or_list_of_images]
    props = properties_or_list_of_properties
    props = [props] if isinstance(props, dict) else list(props)
    names = [truncated_ofname] if isinstance(truncated_ofname, str) else truncated_ofname
    names = [None] * len(images) if names is None else list(names)
    if not len(images) == len(props) == len(names):
        raise ValueError(f"{len(images)} images, {len(props)} properties and {len(names)} output names")
    cases = ((np.asarray(im, dtype=np.float32), copy.deepcopy(p), o) for im, p, o in zip(images, props, names))
    return predict_cases(predictor, cases, save_probabilities, num_processes_segmentation_export)


def _jsonable(obj):
    """Tuples to lists, numpy scalars and arrays to Python values, so that the arguments can be written as JSON."""
    if isinstance(obj, dict):
        return {k: _jsonable(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return [_jsonable(v) for v in obj]
    if isinstance(obj, np.ndarray):
        return obj.tolist()
    if isinstance(obj, np.generic):
        return obj.item()
    return obj
