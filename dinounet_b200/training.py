"""Trainer plugin hook (the primary drop-in boundary, SURVEY.md section 8b).

Mirrors `DinoUNetTrainer` and its four subclasses (dinounet_training.py:833-930): `set_network_config` stores the
planner's architecture dict on the class, and the static `build_network_architecture` hook
(nnUNetTrainer.py:265-298) returns the native `DinoUNet`.  When the reference's nnU-Net package is importable the
trainers derive from its `nnUNetTrainerNoDeepSupervision`, so `api.training(trainer_class=DinoUNetTrainer_l, ...)`
works unchanged; otherwise they derive from `object` (the hook itself is a staticmethod and needs no base class).
"""
from typing import List, Tuple, Union

import torch
from torch import nn

from . import config as cfg
from .loss import DC_and_CE_loss, validation_statistics
from .network_architecture import DinoUNet

try:  # the reference package (needs batchgenerators etc.); optional
    from dinounet.training.nnUNetTrainer.nnUNetTrainerNoDeepSupervision import nnUNetTrainerNoDeepSupervision as _Base
except Exception:  # pragma: no cover - reference stack absent
    _Base = object


class DinoUNetTrainer(_Base):
    _network_config = None
    _dinov3_pretrained_path = None
    _dinov3_model_name = None

    @classmethod
    def set_network_config(cls, network_config, dinov3_pretrained_path=None, dinov3_model_name=None,
                           adapter_type="default"):
        cls._network_config = network_config
        if dinov3_pretrained_path is not None:
            cls._dinov3_pretrained_path = dinov3_pretrained_path
        if dinov3_model_name is not None:
            cls._dinov3_model_name = dinov3_model_name
        # the static hook reads the base class (dinounet_training.py:851-855)
        DinoUNetTrainer._network_config = cls._network_config
        DinoUNetTrainer._dinov3_model_name = cls._dinov3_model_name
        DinoUNetTrainer._dinov3_pretrained_path = cls._dinov3_pretrained_path

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
        return DinoUNet.from_config(network_config=config, input_channels=num_input_channels,
                                    num_classes=num_output_channels,
                                    dinov3_pretrained_path=DinoUNetTrainer._dinov3_pretrained_path,
                                    dinov3_model_name=DinoUNetTrainer._dinov3_model_name)


    # ---- forward-only callers of the path that the trainer owns (nnUNetTrainer.py:355-365, :945-1005)
    def _build_loss(self):
        """Label-map training: Dice (batch_dice from the plans, smooth 1e-5, no background) + CE, weights 1:1 — the
        fused native loss.  No deep-supervision wrapper (the trainer derives from nnUNetTrainerNoDeepSupervision)."""
        if self.label_manager.has_regions:
            raise NotImplementedError("region-based (sigmoid/BCE) training is not covered by the fused native loss")
        return DC_and_CE_loss({"batch_dice": self.configuration_manager.batch_dice, "smooth": 1e-5, "do_bg": False,
                               "ddp": self.is_ddp}, {}, weight_ce=1, weight_dice=1,
                              ignore_label=self.label_manager.ignore_label)

    # ---- training step on the native path (nnUNetTrainer.py:486-489, 899-929)
    def configure_optimizers(self):
        """SGD(momentum 0.99, nesterov, weight decay) + the reference's PolyLRScheduler (it only writes param_groups[0]['lr'])
        on the fused kernels; gradient clipping (12) is part of the fused step."""
        from .train_path import FusedSGD
        optimizer = FusedSGD(self.network.parameters(), self.initial_lr, weight_decay=self.weight_decay, momentum=0.99, max_norm=12.0)
        try:
            from dinounet.training.lr_scheduler.polylr import PolyLRScheduler
            lr_scheduler = PolyLRScheduler(optimizer, self.initial_lr, self.num_epochs)
        except Exception:  # pragma: no cover - reference stack absent
            lr_scheduler = None
        return optimizer, lr_scheduler

    def train_step(self, batch: dict) -> dict:
        from .train_path import train_step
        data = batch["data"].to(self.device, non_blocking=True)
        target = batch["target"]
        if isinstance(target, list):
            target = target[0]
        target = target.to(self.device, non_blocking=True)
        net = self.network.module if hasattr(self.network, "module") else self.network
        loss = train_step(net, self.loss, self.optimizer, data, target)
        return {"loss": loss.cpu().numpy()}

    def validation_step(self, batch: dict) -> dict:
        """One online-validation batch: native forward, then loss + hard tp/fp/fn in one fused pass over the logits."""
        data = batch["data"].to(self.device, non_blocking=True)
        target = batch["target"]
        if isinstance(target, list):
            target = target[0]
        target = target.to(self.device, non_blocking=True)
        with torch.no_grad():
            output = self.network(data)
        del data
        return validation_statistics(self.loss, output, target)


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
