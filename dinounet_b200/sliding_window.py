"""Sliding-window prediction on the native forward engine (SURVEY.md section 8f rank 1).

Mirror of the reference's `nnUNetPredictor` sliding-window surface (inference/predict_from_raw_data.py:39-64,
132-146, 502-553, 572-621, 680-726) and of `inference/sliding_window_prediction.py:11-61`:
same constructor arguments, attribute names, `manual_initialization`, `_internal_get_sliding_window_slicers`,
`predict_sliding_window_return_logits`, same results (fp16 logits, the reference's fp16 accumulation sequence
reproduced bit for bit by the kernels in csrc/sliding_window.cu), same errors.

What is different is the schedule.  The reference handles one tile at a time: slice, upload, 1 + 3 mirrored forwards
of batch 1, flip back, multiply, accumulate (eight torch ops per tile).  Here the padded volume is resident in HBM,
`tile_batch` tiles x their mirror variants are cropped/mirrored/channel-adapted by ONE gather kernel straight into
the engine's input buffer, run as ONE batched forward (CUDA-graph replay), and each tile's variants are un-mirrored,
averaged, gaussian-weighted and accumulated by one small kernel.  Nothing crosses PCIe between the upload of the
volume and the download of the result.
"""
import itertools
from types import SimpleNamespace
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import lib as L

_GAUSSIAN_CACHE = {}


def compute_steps_for_sliding_window(image_size: Sequence[int], tile_size: Sequence[int],
                                     tile_step_size: float) -> List[List[int]]:
    """sliding_window_prediction.py:35-61: evenly spread tile origins, at most tile*step apart, last tile flush with
    the border."""
    if any(i < t for i, t in zip(image_size, tile_size)):
        raise AssertionError("image size must be as large or larger than patch_size")
    if not 0 < tile_step_size <= 1:
        raise AssertionError("step_size must be larger than 0 and smaller or equal to 1")
    out = []
    for size, tile in zip(image_size, tile_size):
        n = int(np.ceil((size - tile) / (tile * tile_step_size))) + 1
        span = size - tile
        stride = span / (n - 1) if n > 1 else 99999999999
        out.append([int(np.round(stride * k)) for k in range(n)])
    return out


def compute_gaussian(tile_size: Sequence[int], sigma_scale: float = 1. / 8, value_scaling_factor: float = 1,
                     dtype=torch.float16, device=torch.device("cuda", 0)) -> torch.Tensor:
    """sliding_window_prediction.py:11-32.  The reference filters a unit impulse at the tile centre with
    scipy's truncated (4 sigma) gaussian; that equals the outer product of per-axis kernel lines, built here directly."""
    key = (tuple(tile_size), sigma_scale, value_scaling_factor, dtype, str(device))
    if key in _GAUSSIAN_CACHE:
        return _GAUSSIAN_CACHE[key]
    lines = []
    for n in tile_size:
        sigma = n * sigma_scale
        radius = int(4.0 * sigma + 0.5)
        taps = np.arange(-radius, radius + 1)
        kern = np.exp(-0.5 / (sigma * sigma) * taps ** 2)
        kern = kern / kern.sum()
        off = n // 2 - np.arange(n)
        inside = np.abs(off) <= radius
        line = np.zeros(n)
        line[inside] = kern[off[inside] + radius]
        lines.append(line)
    g = lines[0]
    for ln in lines[1:]:
        g = np.multiply.outer(g, ln)
    g = torch.from_numpy(g)
    g = (g / g.max() * value_scaling_factor).to(dtype).to(device)
    g[g == 0] = g[g != 0].min()          # the importance map must not contain zeros (:29-30)
    while len(_GAUSSIAN_CACHE) >= 2:     # the reference keeps two (lru_cache(maxsize=2), sliding_window_prediction.py:10)
        _GAUSSIAN_CACHE.pop(next(iter(_GAUSSIAN_CACHE)))
    _GAUSSIAN_CACHE[key] = g
    return g


def pad_to_patch_size(image: torch.Tensor, patch_size: Sequence[int]):
    """What the reference obtains from acvl_utils' `pad_nd_image(image, patch_size, 'constant', {'value': 0}, True)`
    (predict_from_raw_data.py:703-705): zero-pad the trailing dims, centred, up to the patch size; plus the slicer
    that undoes it."""
    lead = image.ndim - len(patch_size)
    target = list(image.shape[:lead]) + [max(p, s) for p, s in zip(patch_size, image.shape[lead:])]
    lo = [(t - s) // 2 for t, s in zip(target, image.shape)]
    hi = [(t - s) - l for t, s, l in zip(target, image.shape, lo)]
    if any(lo) or any(hi):
        pads = [v for l, h in zip(reversed(lo), reversed(hi)) for v in (l, h)]
        image = torch.nn.functional.pad(image, pads, mode="constant", value=0)
    return image, tuple(slice(l, t - h) for l, h, t in zip(lo, hi, target))


class SlidingWindowPredictor:
    """Drop-in for the sliding-window part of `nnUNetPredictor` (2D configurations, which is what `main_dinov3` forces,
    dinounet_training.py:991-999)."""

    def __init__(self, tile_step_size: float = 0.5, use_gaussian: bool = True, use_mirroring: bool = True,
                 perform_everything_on_device: bool = True, device: torch.device = torch.device("cuda"),
                 verbose: bool = False, verbose_preprocessing: bool = False, allow_tqdm: bool = False,
                 tile_batch: int = 8, use_graph: bool = True):
        self.verbose = verbose
        self.verbose_preprocessing = verbose_preprocessing
        self.allow_tqdm = allow_tqdm
        self.plans_manager = self.configuration_manager = self.list_of_parameters = self.network = None
        self.dataset_json = self.trainer_name = self.allowed_mirroring_axes = self.label_manager = None
        self.tile_step_size = tile_step_size
        self.use_gaussian = use_gaussian
        self.use_mirroring = use_mirroring
        if device.type != "cuda":
            raise L.NativeLibraryError("dinounet_b200.SlidingWindowPredictor runs on CUDA devices only (no CPU path)")
        self.device = device
        self.perform_everything_on_device = perform_everything_on_device
        self.tile_batch = int(tile_batch)
        self.use_graph = use_graph

    def manual_initialization(self, network, plans_manager, configuration_manager, parameters: Optional[List[dict]],
                              dataset_json: dict, trainer_name: str,
                              inference_allowed_mirroring_axes: Optional[Tuple[int, ...]]):
        """predict_from_raw_data.py:132-146.  `configuration_manager` needs `.patch_size`; `plans_manager` may be None,
        in which case the number of segmentation heads is taken from the network."""
        self.plans_manager = plans_manager
        self.configuration_manager = configuration_manager
        self.list_of_parameters = parameters
        self.network = network
        self.dataset_json = dataset_json
        self.trainer_name = trainer_name
        self.allowed_mirroring_axes = inference_allowed_mirroring_axes
        if plans_manager is not None:
            self.label_manager = plans_manager.get_label_manager(dataset_json)
        else:
            self.label_manager = SimpleNamespace(num_segmentation_heads=network.num_classes)

    def initialize_from_checkpoint(self, network, filename_or_checkpoint, patch_size=(512, 512)):
        """Weights + mirroring axes from a training checkpoint (`checkpoint_final.pth`), the part of
        `initialize_from_trained_model_folder` (predict_from_raw_data.py:66-130) that concerns the network."""
        from .checkpoint import load_network_weights
        meta = load_network_weights(network, filename_or_checkpoint)
        self.manual_initialization(network.to(self.device), None, SimpleNamespace(patch_size=list(patch_size)), None, {},
                                   meta.get("trainer_name"), meta.get("inference_allowed_mirroring_axes"))
        return meta

    def _internal_get_sliding_window_slicers(self, image_size: Tuple[int, ...]):
        patch = self.configuration_manager.patch_size
        if len(patch) != len(image_size) - 1:
            raise AssertionError("2D patch size expects a (slices, H, W) image (only dimension discrepancy of 1 allowed)")
        steps = compute_steps_for_sliding_window(image_size[1:], patch, self.tile_step_size)
        if self.verbose:
            print(f"n_steps {image_size[0] * len(steps[0]) * len(steps[1])}, image size is {image_size}, "
                  f"tile_size {patch}, tile_step_size {self.tile_step_size}\nsteps:\n{steps}")
        return [(slice(None), d, slice(sx, sx + patch[0]), slice(sy, sy + patch[1]))
                for d in range(image_size[0]) for sx in steps[0] for sy in steps[1]]

    def _mirror_variants(self) -> List[int]:
        """flip bits per forward of one tile, in the reference's order (:545-550): bit0 = tensor dim 2, bit1 = dim 3."""
        axes = self.allowed_mirroring_axes if self.use_mirroring else None
        variants = [0]
        if axes is not None:
            if max(axes) > 1:
                raise AssertionError("mirror_axes does not match the dimension of the input!")
            dims = [m + 2 for m in axes]
            for k in range(len(dims)):
                for combo in itertools.combinations(dims, k + 1):
                    variants.append(sum(1 << (a - 2) for a in combo))
        return variants

    @torch.no_grad()
    def predict_sliding_window_return_logits(self, input_image: torch.Tensor) -> torch.Tensor:
        """input_image [c, slices, H, W] -> fp16 logits [heads, slices, H, W] (on the device, or on the CPU when
        `perform_everything_on_device` is False — the accumulation itself always happens in HBM)."""
        assert isinstance(input_image, torch.Tensor)
        assert input_image.ndim == 4, "input_image must be a 4D np.ndarray or torch.Tensor (c, x, y, z)"
        net = self.network
        net.eval()
        patch = [int(p) for p in self.configuration_manager.patch_size]
        if len(patch) != 2 or patch[0] != patch[1]:
            raise NotImplementedError("the native engine runs square 2D patches (main_dinov3 forces 512x512)")
        lib = L.load()
        dev = self.device if self.device.index is not None else torch.device("cuda", torch.cuda.current_device())
        heads = int(self.label_manager.num_segmentation_heads)
        data, revert = pad_to_patch_size(input_image, patch)
        slicers = self._internal_get_sliding_window_slicers(tuple(data.shape[1:]))
        data = data.to(dev, dtype=torch.float32, non_blocking=True).contiguous()
        Cin, D, H, W = data.shape
        th = tw = patch[0]
        variants = self._mirror_variants()
        nvar = len(variants)
        tiles = [(s[1], s[2].start, s[3].start) for s in slicers]
        per = max(1, self.tile_batch)
        nb = per * nvar
        n_batches = (len(tiles) + per - 1) // per
        desc = np.zeros((n_batches, nb, 4), dtype=np.int32)
        for t, (d, y0, x0) in enumerate(tiles):
            for v, bits in enumerate(variants):
                desc[t // per, (t % per) * nvar + v] = (d, y0, x0, bits)
        for t in range(len(tiles), n_batches * per):      # fill the last batch with repeats of tile 0 (never accumulated)
            desc[t // per, (t % per) * nvar:(t % per + 1) * nvar] = desc[0, :nvar]
        desc_dev = torch.from_numpy(desc).to(dev)
        acc = torch.zeros((heads, D, H, W), dtype=torch.half, device=dev)
        npred = torch.zeros((D, H, W), dtype=torch.half, device=dev)
        flag = torch.zeros(1, dtype=torch.int32, device=dev)
        gaussian = compute_gaussian(tuple(patch), sigma_scale=1. / 8, value_scaling_factor=10,
                                    device=dev) if self.use_gaussian else None
        eng = net._get_engine(dev)
        if eng.ncls != heads:
            raise ValueError(f"network produces {eng.ncls} heads, label manager expects {heads}")
        _, bufs = eng.get_plan(nb, th)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            for b in range(n_batches):
                dptr = desc_dev[b].data_ptr()
                L.check(lib.b2u_sw_gather_tiles(data.data_ptr(), bufs["x"].data_ptr(), dptr, nb, Cin, D, H, W, th, tw,
                                                stream), "sw_gather_tiles")
                logits, _ = eng.run_resident(nb, th, self.use_graph)
                for t in range(min(per, len(tiles) - b * per)):
                    L.check(lib.b2u_sw_accumulate(logits.data_ptr(), dptr, t * nvar, nvar,
                                                  gaussian.data_ptr() if gaussian is not None else None,
                                                  acc.data_ptr(), npred.data_ptr(), heads, D, H, W, th, tw, stream),
                            "sw_accumulate")
            L.check(lib.b2u_sw_finalize(acc.data_ptr(), npred.data_ptr(), heads, D * H * W, flag.data_ptr(), stream),
                    "sw_finalize")
        if int(flag.item()):
            raise RuntimeError("Encountered inf in predicted array. Aborting... If this problem persists, "
                               "reduce value_scaling_factor in compute_gaussian or increase the dtype of "
                               "predicted_logits to fp32")
        out = acc[(slice(None), *revert[1:])]
        return out if self.perform_everything_on_device else out.cpu()

    @torch.no_grad()
    def predict_logits_from_preprocessed_data(self, data: torch.Tensor) -> torch.Tensor:
        """predict_from_raw_data.py:466-501: the sliding window once per entry of `list_of_parameters` (loaded into the
        network), summed and divided by the number of folds in fp16 with the bits of the reference's CPU fp16 ops
        (`b2u_pre_ensemble_f16`).  The fp16 logits [heads, *data.shape[1:]] stay on the device.  With
        `list_of_parameters` None the network's current weights make the single prediction."""
        from .preprocess import ensemble_logits
        lib = L.load()
        params = self.list_of_parameters

        def runs():
            for p in (params or [None]):
                if p is not None:
                    self.network.load_state_dict(p)
                    if hasattr(self.network, "repack"):
                        self.network.repack()   # the engine packs the weights it was built with
                logits = self.predict_sliding_window_return_logits(data)
                yield logits if logits.is_cuda else logits.to(self.device)

        def add(acc, x, divisor):
            with torch.cuda.device(acc.device):
                L.check(lib.b2u_pre_ensemble_f16(acc.data_ptr(), None if x is None else x.data_ptr(), acc.numel(),
                                                 divisor, torch.cuda.current_stream(acc.device).cuda_stream),
                        "b2u_pre_ensemble_f16")

        return ensemble_logits(runs(), len(params) if params else 1, add)

    def predict_single_npy_array(self, input_image: np.ndarray, image_properties: dict,
                                 segmentation_previous_stage: np.ndarray = None, output_file_truncated: str = None,
                                 save_or_return_probabilities: bool = False):
        """predict_from_raw_data.py:429-464 on the device: DevicePreprocessor.run_case_npy -> the fold ensemble ->
        the device export.  Only the input goes up, and only the segmentation (and the probabilities, when asked) comes
        down.  `image_properties` needs the 'spacing' key; the preprocessing adds its keys to it, as the reference's."""
        from . import export
        from .preprocess import DevicePreprocessor
        if segmentation_previous_stage is not None:
            raise NotImplementedError("the cascade (segmentation_previous_stage) is not implemented on the device")
        if self.plans_manager is None:
            raise ValueError("predict_single_npy_array needs a plans_manager (manual_initialization)")
        dev = self.device if self.device.index is not None else torch.device("cuda", torch.cuda.current_device())
        data, _ = DevicePreprocessor(self.verbose_preprocessing, dev).run_case_npy(
            input_image, None, image_properties, self.plans_manager, self.configuration_manager, self.dataset_json)
        logits = self.predict_logits_from_preprocessed_data(data)
        if output_file_truncated is not None:
            export.export_prediction_from_logits(logits, image_properties, self.configuration_manager,
                                                 self.plans_manager, self.dataset_json, output_file_truncated,
                                                 save_or_return_probabilities)
            return None
        return export.convert_predicted_logits_to_segmentation_with_correct_shape(
            logits, self.plans_manager, self.configuration_manager, self.label_manager, image_properties,
            return_probabilities=save_or_return_probabilities)
