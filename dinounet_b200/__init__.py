"""dinounet_b200 — H100-native (sm_90a) implementation of the Dino U-Net forward segmentation path.

Public surface (drop-in for the reference's `dinounet_training.py` model + trainer hook):
    from dinounet_b200 import DinoUNet, DinoUNetTrainer_s/_b/_l/_7b, get_dinov3_trainer
The compute path is hand-written CUDA behind the C-ABI of include/dinounet_b200.h (libdinounet_b200.so); importing the
package does not need a GPU, running a forward does, and there is no CPU / PyTorch fallback.
"""
from . import config  # noqa: F401
from .network_architecture import DinoUNet, DINOv3EncoderAdapter, FAPM, UNetDecoder, DINOv3_Adapter, MSDeformAttn  # noqa: F401
from .training import (  # noqa: F401
    DinoUNetTrainer, DinoUNetTrainer_s, DinoUNetTrainer_b, DinoUNetTrainer_l, DinoUNetTrainer_7b, DINOV3_TRAINERS,
    get_dinov3_trainer, install_discoverable_trainers,
)

__version__ = "0.1.0"
from .sliding_window import SlidingWindowPredictor, compute_gaussian, compute_steps_for_sliding_window  # noqa: F401,E402
from .inference import StreamedPredictor  # noqa: F401,E402
from .checkpoint import load_network_weights  # noqa: F401,E402
from .export import labels_to_original_geometry  # noqa: F401,E402
