"""Trainer plugin hook (the primary drop-in boundary, SURVEY.md section 8b).

Mirrors `DinoUNetTrainer` and its four subclasses (dinounet_training.py:833-930): `set_network_config` stores the
planner's architecture dict on the class, and the static `build_network_architecture` hook
(nnUNetTrainer.py:265-298) returns the native `DinoUNet`.  When the reference's nnU-Net package is importable the
trainers derive from its `nnUNetTrainerNoDeepSupervision`, so `api.training(trainer_class=DinoUNetTrainer_l, ...)`
works unchanged; otherwise they derive from `object` (the hook itself is a staticmethod and needs no base class).
"""
import os
import warnings
from concurrent.futures import ThreadPoolExecutor
from typing import List, Tuple, Union

import numpy as np
import torch
from torch import distributed as dist
from torch import nn

from . import config as cfg
from . import deep_supervision as DS
from .loss import DC_and_BCE_loss, DC_and_CE_loss, DeepSupervisionWrapper, validation_statistics
from .network_architecture import DinoUNet

try:  # the reference package (needs batchgenerators etc.); optional
    from dinounet.training.nnUNetTrainer.nnUNetTrainerNoDeepSupervision import nnUNetTrainerNoDeepSupervision as _Base
except Exception:  # pragma: no cover - reference stack absent
    _Base = object


class DinoUNetTrainer(_Base):
    _network_config = None
    _dinov3_pretrained_path = None
    _dinov3_model_name = None
    _train_semantics = None
    _device_augmentation = False
    _train_recompute = False
    _device_dataloading = False

    @classmethod
    def set_network_config(cls, network_config, dinov3_pretrained_path=None, dinov3_model_name=None,
                           adapter_type="default", train_semantics=None, device_augmentation=False, train_recompute=False,
                           device_dataloading=False):
        """train_semantics: `DinoUNet.train_semantics` of the networks `build_network_architecture` returns ("oracle" or
        "reference"); None keeps the module default.  device_augmentation: run the training transforms on the device
        (dinounet_b200/augmentation.py) instead of batchgenerators' worker processes; off by default.  train_recompute:
        `DinoUNet.train_recompute` of those networks, recomputing the adapter's extractors in the backward (the reference's
        checkpointing; what lets the large variants train at a useful batch); off by default.  device_dataloading: draw
        the 2-D batches in one read-ahead thread and assemble them on the device (dinounet_b200/dataloading.py) instead
        of batchgenerators' worker processes; needs device_augmentation, off by default."""
        if not isinstance(train_recompute, bool):
            raise ValueError(f"train_recompute must be True or False, got {train_recompute!r}")
        if not isinstance(device_dataloading, bool):
            raise ValueError(f"device_dataloading must be True or False, got {device_dataloading!r}")
        if device_dataloading and not device_augmentation:
            raise ValueError("device_dataloading=True needs device_augmentation=True: the host transforms cannot take "
                             "the device loader's CUDA tensors")
        cls._network_config = network_config
        cls._train_semantics = train_semantics
        cls._device_augmentation = bool(device_augmentation)
        cls._train_recompute = train_recompute
        cls._device_dataloading = device_dataloading
        if dinov3_pretrained_path is not None:
            cls._dinov3_pretrained_path = dinov3_pretrained_path
        if dinov3_model_name is not None:
            cls._dinov3_model_name = dinov3_model_name
        # the static hook reads the base class (dinounet_training.py:851-855)
        DinoUNetTrainer._network_config = cls._network_config
        DinoUNetTrainer._dinov3_model_name = cls._dinov3_model_name
        DinoUNetTrainer._dinov3_pretrained_path = cls._dinov3_pretrained_path
        DinoUNetTrainer._train_semantics = cls._train_semantics
        DinoUNetTrainer._device_augmentation = cls._device_augmentation
        DinoUNetTrainer._train_recompute = cls._train_recompute
        DinoUNetTrainer._device_dataloading = cls._device_dataloading

    @staticmethod
    def build_network_architecture(architecture_class_name: str, arch_init_kwargs: dict,
                                   arch_init_kwargs_req_import: Union[List[str], Tuple[str, ...]],
                                   num_input_channels: int, num_output_channels: int,
                                   enable_deep_supervision: bool = True) -> nn.Module:
        if DinoUNetTrainer._network_config is None:
            raise RuntimeError("call set_network_config(network_config) before build_network_architecture")
        config = DinoUNetTrainer._network_config.copy()
        config["architecture"] = config["architecture"].copy()
        config["architecture"]["deep_supervision"] = enable_deep_supervision
        net = DinoUNet.from_config(network_config=config, input_channels=num_input_channels,
                                   num_classes=num_output_channels,
                                   dinov3_pretrained_path=DinoUNetTrainer._dinov3_pretrained_path,
                                   dinov3_model_name=DinoUNetTrainer._dinov3_model_name)
        if DinoUNetTrainer._train_semantics is not None:
            net.train_semantics = DinoUNetTrainer._train_semantics
        net.train_recompute = DinoUNetTrainer._train_recompute
        return net


    # ---- training transforms (nnUNetTrainer.py:684-775)
    @staticmethod
    def get_training_transforms(patch_size, rotation_for_DA, deep_supervision_scales, mirror_axes,
                                do_dummy_2d_data_aug, *args, **kwargs):
        """With device augmentation on, the host pipeline only renames `seg` to `target` and makes tensors of the
        batch at the initial patch size (float32 data, int16 seg); `train_step` augments it on the device.  Otherwise
        the reference's pipeline."""
        if DinoUNetTrainer._device_augmentation:
            return PassThroughTransforms()
        return _Base.get_training_transforms(patch_size, rotation_for_DA, deep_supervision_scales, mirror_axes,
                                             do_dummy_2d_data_aug, *args, **kwargs)

    def _device_augmenter(self):
        """The device pipeline with the trainer's configuration, built once.  Under DDP each rank seeds its own stream
        of draws: the seed is derived from the rank."""
        aug = getattr(self, "_device_aug", None)
        if aug is None:
            from .augmentation import DeviceTrainingAugmentation
            rotation_for_DA, do_dummy_2d, _, mirror_axes = self.configure_rotation_dummyDA_mirroring_and_inital_patch_size()
            if do_dummy_2d or len(self.configuration_manager.patch_size) != 2:
                raise NotImplementedError("device augmentation covers 2-D configurations only")
            lm = self.label_manager
            rank = getattr(self, "local_rank", 0) if getattr(self, "is_ddp", False) else 0
            seed = int(np.random.SeedSequence(self._device_augmentation_seed, spawn_key=(rank,)).generate_state(1)[0])
            aug = DeviceTrainingAugmentation(self.configuration_manager.patch_size, rotation_for_DA, mirror_axes,
                                             use_mask_for_norm=self.configuration_manager.use_mask_for_norm,
                                             regions=lm.foreground_regions if lm.has_regions else None,
                                             ignore_label=lm.ignore_label, seed=seed)
            self._device_aug = aug
        return aug

    # None: fresh entropy per run; an int makes every rank's draws reproducible
    _device_augmentation_seed = None

    # ---- data loading on the device (nnUNetTrainer.py:652-690)
    def get_dataloaders(self):
        """With device data loading on: a train loader at the initial patch size and a val loader at the patch size
        (with the trainer's regions and ignore label) in this process, each with one read-ahead thread; otherwise the
        reference's augmenters.  Under DDP each rank seeds its own loaders from `_device_dataloading_seed` and its
        rank."""
        if not DinoUNetTrainer._device_dataloading:
            return _Base.get_dataloaders(self)
        from .dataloading import DeviceDataLoader2D
        patch_size = self.configuration_manager.patch_size
        if len(patch_size) != 2:
            raise NotImplementedError("device data loading covers 2-D configurations only")
        _, _, initial_patch_size, _ = self.configure_rotation_dummyDA_mirroring_and_inital_patch_size()
        dataset_tr, dataset_val = self.get_tr_and_val_datasets()
        lm = self.label_manager
        rank = getattr(self, "local_rank", 0) if getattr(self, "is_ddp", False) else 0
        seeds = [int(np.random.SeedSequence(self._device_dataloading_seed, spawn_key=(rank, i)).generate_state(1)[0])
                 for i in (0, 1)]
        dl_tr = DeviceDataLoader2D(dataset_tr, self.batch_size, initial_patch_size, patch_size, lm,
                                   oversample_foreground_percent=self.oversample_foreground_percent, mode="train",
                                   seed=seeds[0], device=self.device)
        dl_val = DeviceDataLoader2D(dataset_val, self.batch_size, patch_size, patch_size, lm,
                                    oversample_foreground_percent=self.oversample_foreground_percent, mode="val",
                                    regions=lm.foreground_regions if lm.has_regions else None,
                                    ignore_label=lm.ignore_label, seed=seeds[1], device=self.device)
        return dl_tr, dl_val

    # None: fresh entropy per run; an int makes every rank's batches reproducible
    _device_dataloading_seed = None

    def on_train_end(self):
        """Stops the device loaders' read-ahead threads, then the reference's end of training."""
        from .dataloading import DeviceDataLoader2D
        for dl in (getattr(self, "dataloader_train", None), getattr(self, "dataloader_val", None)):
            if isinstance(dl, DeviceDataLoader2D):
                dl.close()
        base = getattr(super(), "on_train_end", None)   # absent without the reference package
        if base is not None:
            base()

    # ---- forward-only callers of the path that the trainer owns (nnUNetTrainer.py:355-365, :945-1005)
    def _build_loss(self):
        """The fused native losses with the reference's arguments.  Region-based datasets: sigmoid Dice (batch_dice from
        the plans, every region, smooth 1e-5) + BCE, ignore channel when the dataset has an ignore label.  Label maps:
        Dice (no background) + CE, weights 1:1.  `ddp` follows the trainer, so under DDP the batch Dice sums are taken
        over every rank.  With `enable_deep_supervision` (off in the base trainer, which derives from
        nnUNetTrainerNoDeepSupervision; a subclass sets it in its constructor) the loss is wrapped in a
        `DeepSupervisionWrapper` with the reference's weights (nnUNetTrainer.py:370-390); a plan whose scales do not
        match the network's three outputs raises here, before training starts."""
        if self.label_manager.has_regions:
            loss = DC_and_BCE_loss({}, {"batch_dice": self.configuration_manager.batch_dice, "do_bg": True,
                                        "smooth": 1e-5, "ddp": self.is_ddp},
                                   use_ignore_label=self.label_manager.ignore_label is not None)
        else:
            loss = DC_and_CE_loss({"batch_dice": self.configuration_manager.batch_dice, "smooth": 1e-5, "do_bg": False,
                                   "ddp": self.is_ddp}, {}, weight_ce=1, weight_dice=1,
                                  ignore_label=self.label_manager.ignore_label)
        if getattr(self, "enable_deep_supervision", False):
            weights = DS.deep_supervision_weights(len(self._ds_scales()), self.is_ddp)
            loss = DeepSupervisionWrapper(loss, weights)
        return loss

    def _ds_scales(self):
        """The plan's deep-supervision scales (nnUNetTrainer.py:300-306), checked against the network's outputs."""
        return DS.deep_supervision_scales(self.configuration_manager.pool_op_kernel_sizes)

    def _target_to_device(self, target, keep_list: bool):
        """The batch's target on the device: the list of the host transforms' scales when `keep_list`, else its first
        (full-resolution) entry."""
        if isinstance(target, list):
            if keep_list:
                return [t.to(self.device, non_blocking=True) for t in target]
            target = target[0]
        return target.to(self.device, non_blocking=True)

    def _ds_targets(self, target):
        """With deep supervision, a target made on the device (one tensor) as the list of the plan's scales, highest
        resolution first, from one target-kernel launch; anything else as it is."""
        if getattr(self, "enable_deep_supervision", False) and not isinstance(target, list):
            return DS.downsample_targets(target, self._ds_scales())
        return target

    def set_deep_supervision_enabled(self, enabled: bool):
        """Switches the network's deep-supervision outputs, as the reference trainer does around its final validation
        (nnUNetTrainer.py:1147, :1292); a trainer without deep supervision keeps them off whatever `enabled` says."""
        mod = self.network.module if getattr(self, "is_ddp", False) else self.network
        mod = getattr(mod, "_orig_mod", mod)
        mod.decoder.deep_supervision = bool(enabled and getattr(self, "enable_deep_supervision", False))

    # ---- training step on the native path (nnUNetTrainer.py:486-489, 899-929)
    def configure_optimizers(self):
        """SGD(momentum 0.99, nesterov, weight decay) + the reference's PolyLRScheduler (it only writes param_groups[0]['lr'])
        on the fused kernels; gradient clipping (12) is part of the fused step.  Without the reference package there is
        no scheduler; a scheduler that fails to construct raises."""
        from .train_path import FusedSGD
        optimizer = FusedSGD(self.network.parameters(), self.initial_lr, weight_decay=self.weight_decay, momentum=0.99, max_norm=12.0)
        try:
            from dinounet.training.lr_scheduler.polylr import PolyLRScheduler
        except ImportError:  # pragma: no cover - reference stack absent
            return optimizer, None
        return optimizer, PolyLRScheduler(optimizer, self.initial_lr, self.num_epochs)

    def train_step(self, batch: dict) -> dict:
        from .train_path import train_step
        data = batch["data"].to(self.device, non_blocking=True)
        ds = getattr(self, "enable_deep_supervision", False)
        target = self._target_to_device(batch["target"], ds and not DinoUNetTrainer._device_augmentation)
        if DinoUNetTrainer._device_augmentation:
            data, target = self._device_augmenter()(data, target)
        # the device pipeline's target is downsampled after it (the host pipeline made no scales, PassThroughTransforms)
        target = self._ds_targets(target)
        net = self.network.module if hasattr(self.network, "module") else self.network
        loss = train_step(net, self.loss, self.optimizer, data, target)
        return {"loss": loss.cpu().numpy()}

    def validation_step(self, batch: dict) -> dict:
        """One online-validation batch: native forward, then loss + hard tp/fp/fn in one fused pass over the logits
        (argmax per class for label maps, sigmoid > 0.5 per region with the ignore channel as a weight for regions).
        With deep supervision: the loss over every scale, the counts from the full-resolution output and target."""
        data = batch["data"].to(self.device, non_blocking=True)
        target = self._target_to_device(batch["target"], getattr(self, "enable_deep_supervision", False))
        target = self._ds_targets(target)
        with torch.no_grad():
            output = self.network(data)
        del data
        return validation_statistics(self.loss, output, target)

    # ---- final validation on the device (nnUNetTrainer.py:1146-1293)
    def _validation_keys(self):
        """`do_split()`'s validation keys, under DDP this rank's share `val_keys[rank::world]`, and the last case index
        after which the periodic barrier stops (every rank reaches it), as nnUNetTrainer.py:1174-1180."""
        _, val_keys = self.do_split()
        last_barrier_at_idx = None
        if self.is_ddp:
            world = dist.get_world_size()
            last_barrier_at_idx = len(val_keys) // world - 1
            val_keys = val_keys[self.local_rank::world]
        return val_keys, last_barrier_at_idx

    def perform_actual_validation(self, save_probabilities: bool = False):
        """The validation at the end of training on the device: each validation case is predicted by
        `SlidingWindowPredictor` (tile step 0.5, gaussian, no mirroring) on the network's current weights, and its fp16
        logits go to the device export without leaving the GPU.  `VALIDATION_WRITERS` threads run the export, with at
        most two cases queued beyond them: its kernels and its copy of the labels to the host are ordered after the
        prediction work already queued on the stream, and its host part (geometry, file writing) overlaps the next
        case's prediction.  Rank 0 then scores `validation/` against `gt_segmentations/` with the device evaluation into
        `validation/summary.json`.  The cascade and next-stage predictions are not implemented: they raise before
        anything runs."""
        from . import evaluation, export
        from .engine import GRAPH_CAPTURE
        from .sliding_window import SlidingWindowPredictor
        if self.is_cascaded:
            raise NotImplementedError("the final validation on the device does not implement the cascade")
        if self.configuration_manager.next_stage_names is not None:
            raise NotImplementedError("the final validation on the device does not predict for next stages "
                                      f"({self.configuration_manager.next_stage_names})")
        self.set_deep_supervision_enabled(False)
        self.network.eval()
        net = self.network.module if self.is_ddp else self.network
        net.repack()   # the optimizer changed the weights in place since the engine packed them
        predictor = SlidingWindowPredictor(tile_step_size=0.5, use_gaussian=True, use_mirroring=False,
                                           perform_everything_on_device=True, device=self.device)
        predictor.manual_initialization(net, self.plans_manager, self.configuration_manager, None, self.dataset_json,
                                        self.__class__.__name__, self.inference_allowed_mirroring_axes)
        validation_output_folder = os.path.join(self.output_folder, "validation")
        os.makedirs(validation_output_folder, exist_ok=True)
        val_keys, last_barrier_at_idx = self._validation_keys()
        dataset_val = _validation_dataset(self.preprocessed_dataset_folder, val_keys,
                                          self.folder_with_segs_from_previous_stage)
        # the writers enqueue the export on the stream the logits were computed on
        stream = torch.cuda.current_stream(predictor.device if predictor.device.index is not None else None)

        def write(logits, properties, output_filename_truncated):
            with GRAPH_CAPTURE.device_work(), torch.cuda.stream(stream):
                export.export_prediction_from_logits(logits, properties, self.configuration_manager, self.plans_manager,
                                                     self.dataset_json, output_filename_truncated, save_probabilities)

        with ThreadPoolExecutor(VALIDATION_WRITERS) as writers:
            pending = []
            for i, k in enumerate(dataset_val.keys()):
                while len(pending) >= VALIDATION_WRITERS + 2:   # allowed_num_queued=2 (nnUNetTrainer.py:1194-1199)
                    pending.pop(0).result()
                self.print_to_log_file(f"predicting {k}")
                data, _, properties = dataset_val.load_case(k)
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")   # 'The given NumPy array is not writable'
                    data = torch.from_numpy(data)
                self.print_to_log_file(f"{k}, shape {data.shape}, rank {self.local_rank}")
                logits = predictor.predict_sliding_window_return_logits(data)
                pending.append(writers.submit(write, logits, properties, os.path.join(validation_output_folder, k)))
                del logits
                if self.is_ddp and i < last_barrier_at_idx and (i + 1) % 20 == 0:
                    dist.barrier()
            for f in pending:
                f.result()
        if self.is_ddp:
            dist.barrier()
        if self.local_rank == 0:
            lm = self.label_manager
            metrics = evaluation.compute_metrics_on_folder(
                os.path.join(self.preprocessed_dataset_folder_base, "gt_segmentations"), validation_output_folder,
                os.path.join(validation_output_folder, "summary.json"), self.plans_manager.image_reader_writer_class(),
                self.dataset_json["file_ending"], lm.foreground_regions if lm.has_regions else lm.foreground_labels,
                lm.ignore_label, chill=True,
                num_processes=evaluation.DEFAULT_NUM_PROCESSES * (dist.get_world_size() if self.is_ddp else 1))
            self.print_to_log_file("Validation complete", also_print_to_console=True)
            self.print_to_log_file("Mean Validation Dice: ", (metrics["foreground_mean"]["Dice"]),
                                   also_print_to_console=True)
        self.set_deep_supervision_enabled(True)


#: threads that export and write the final validation's cases; their host work overlaps the next prediction
VALIDATION_WRITERS = 2


def _validation_dataset(folder: str, keys, folder_with_segs_from_previous_stage):
    """The reference's dataset of preprocessed cases (`<key>.npz` / `<key>.pkl`), loaded with `load_case(key)` ->
    (data, seg, properties).  Tests substitute it."""
    from dinounet.training.dataloading.nnunet_dataset import nnUNetDataset
    return nnUNetDataset(folder, keys, folder_with_segs_from_previous_stage=folder_with_segs_from_previous_stage,
                         num_images_properties_loading_threshold=0)


class PassThroughTransforms:
    """The host side of device augmentation: `seg` renamed to `target`, data and seg as tensors (NumpyToTensor without
    the cast of the labels to float, so that they stay int16 for the device pipeline)."""

    def __call__(self, **data_dict):
        data_dict["data"] = torch.as_tensor(np.asarray(data_dict["data"], dtype=np.float32))
        data_dict["target"] = torch.as_tensor(np.asarray(data_dict.pop("seg"), dtype=np.int16))
        return data_dict


class DinoUNetTrainer_s(DinoUNetTrainer):
    _dinov3_model_name = "dinounet_s"
    _dinov3_pretrained_path = cfg.CHECKPOINTS["dinounet_s"]


class DinoUNetTrainer_b(DinoUNetTrainer):
    _dinov3_model_name = "dinounet_b"
    _dinov3_pretrained_path = cfg.CHECKPOINTS["dinounet_b"]


class DinoUNetTrainer_l(DinoUNetTrainer):
    _dinov3_model_name = "dinounet_l"
    _dinov3_pretrained_path = cfg.CHECKPOINTS["dinounet_l"]


class DinoUNetTrainer_7b(DinoUNetTrainer):
    _dinov3_model_name = "dinounet_7b"
    _dinov3_pretrained_path = cfg.CHECKPOINTS["dinounet_7b"]


DINOV3_TRAINERS = {"dinounet_s": DinoUNetTrainer_s, "dinounet_b": DinoUNetTrainer_b, "dinounet_l": DinoUNetTrainer_l,
                   "dinounet_7b": DinoUNetTrainer_7b}


_DISCOVERABLE_STUB = '''"""Makes the native Dino U-Net trainers visible to nnU-Net's name-based trainer lookup.

`recursive_find_python_class` (dinounet/utilities/find_class_by_name.py:7-24) walks dinounet/training/nnUNetTrainer/*.py;
the reference's own `DinoUNetTrainer_*` classes live in the top-level script dinounet_training.py and are therefore
invisible to `get_trainer_from_args` (run/run_training.py:39-47) and to the standalone predictor
(`nnUNetPredictor.initialize_from_trained_model_folder`, predict_from_raw_data.py:99-100).  This file is written by
`dinounet_b200.training.install_discoverable_trainers()`.
"""
from dinounet_b200.training import (DinoUNetTrainer, DinoUNetTrainer_s, DinoUNetTrainer_b, DinoUNetTrainer_l,  # noqa: F401
                                    DinoUNetTrainer_7b)
'''


def install_discoverable_trainers(dinounet_package_dir: str = None, filename: str = "DinoUNetTrainer_b200.py") -> str:
    """Writes a one-import module into `<dinounet>/training/nnUNetTrainer/` so that the reference's filesystem-based class
    lookup (find_class_by_name.py:7-24) finds `DinoUNetTrainer_s/_b/_l/_7b` by name - what the standalone predictor and
    `nnUNetv2_train -tr DinoUNetTrainer_l` need (SURVEY.md section 8a, quirk list).  Returns the path written."""
    import os
    if dinounet_package_dir is None:
        import importlib.util
        spec = importlib.util.find_spec("dinounet")
        if spec is None or not spec.submodule_search_locations:
            raise ModuleNotFoundError("the reference package `dinounet` is not importable; pass its directory")
        dinounet_package_dir = list(spec.submodule_search_locations)[0]
    target = os.path.join(dinounet_package_dir, "training", "nnUNetTrainer")
    if not os.path.isdir(target):
        raise FileNotFoundError(f"{target} does not exist (not a dinounet package directory?)")
    path = os.path.join(target, filename)
    with open(path, "w") as f:
        f.write(_DISCOVERABLE_STUB)
    return path


def get_dinov3_trainer(model_name: str):
    if model_name not in DINOV3_TRAINERS:
        raise ValueError(f"Unsupported model: {model_name}. Supported models: {list(DINOV3_TRAINERS)}")
    return DINOV3_TRAINERS[model_name]
