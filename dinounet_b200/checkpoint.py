"""Loading nnU-Net / Dino U-Net training checkpoints (`checkpoint_final.pth`, `checkpoint_best.pth`) into the native model.

The reference writes `{'network_weights': state_dict, 'optimizer_state', 'grad_scaler_state', 'logging', '_best_ema',
'current_epoch', 'init_args', 'trainer_name', 'inference_allowed_mirroring_axes'}` (nnUNetTrainer.py:1083-1104) and reads
it back with a key heuristic for DataParallel / torch.compile wrappers (nnUNetTrainer.py:1108-1140,
predict_from_raw_data.py:99-118).  `dinounet_b200.DinoUNet` has the reference's state-dict keys (including the
duplicated `decoder.encoder.*` entries), so the weights load with `strict=True`; this helper applies the same prefix
heuristic, refreshes the packed kernel weights and hands back the metadata the predictor needs.
"""
from typing import Union

import torch

_PREFIXES = ("module.", "_orig_mod.", "module._orig_mod.")


def load_network_weights(network: torch.nn.Module, filename_or_checkpoint: Union[dict, str], strict: bool = True) -> dict:
    """Returns {'trainer_name', 'init_args', 'current_epoch', 'inference_allowed_mirroring_axes'} (None where absent)."""
    ckpt = filename_or_checkpoint
    if isinstance(ckpt, str):
        ckpt = torch.load(ckpt, map_location="cpu", weights_only=False)     # the reference pickles plain python objects too
    if "network_weights" not in ckpt:
        raise KeyError("not an nnU-Net checkpoint: no 'network_weights' entry")
    weights = match_keys(ckpt["network_weights"], set(network.state_dict().keys()))
    network.load_state_dict(weights, strict=strict)
    if hasattr(network, "repack"):
        network.repack()          # packed K-major kernel weights are rebuilt on the next forward
    return {k: ckpt.get(k) for k in ("trainer_name", "init_args", "current_epoch", "inference_allowed_mirroring_axes")}


def match_keys(network_weights: dict, own: set) -> dict:
    """The checkpoint's weights under the network's own keys: a key the network lacks loses a DataParallel /
    torch.compile prefix when that names one of the network's keys."""
    weights = {}
    for k, v in network_weights.items():
        key = k
        if key not in own:
            for p in _PREFIXES:
                if key.startswith(p) and key[len(p):] in own:
                    key = key[len(p):]
                    break
        weights[key] = v
    return weights
