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
import math
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


def backbones_identical(list_of_parameters) -> bool:
    """True when there are at least two state dicts and every one holds the same DINOv3 backbone, bit for bit: the
    `*.dinov3_adapter.backbone.*` tensors, the `decoder.encoder.` duplicates included.  Training freezes the backbone,
    so the folds of one run pass this."""
    if not list_of_parameters or len(list_of_parameters) < 2:
        return False

    def backbone(sd):
        return {k: t for k, t in sd.items() if ".dinov3_adapter.backbone." in k}

    first = backbone(list_of_parameters[0])
    if not first:
        return False
    for sd in list_of_parameters[1:]:
        other = backbone(sd)
        if other.keys() != first.keys():
            return False
        for k, a in first.items():
            b = other[k]
            if a.dtype != b.dtype or a.shape != b.shape:
                return False
            a8 = a.detach().contiguous().reshape(-1).view(torch.uint8)
            b8 = b.detach().to(a.device).contiguous().reshape(-1).view(torch.uint8)
            if not torch.equal(a8, b8):
                return False
    return True


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
        #: slices per chunk of the shared-backbone fold route; None = the fewest slices that fill whole tile batches,
        #: times the multiple that makes about four batches
        self.fold_chunk_slices = None
        #: the fold ensemble route the last `predict_logits_from_preprocessed_data` took: "shared_backbone" (one ViT
        #: pass per tile batch for every fold) or "per_fold" (the weights reloaded for each fold)
        self.ensemble_route = None
        self._shared_backbone_params = None
        self._fold_engine = None

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
        self._select_ensemble_route()

    def _select_ensemble_route(self):
        """Folds that share the backbone bit for bit run it once per tile batch; decided once, for this
        `list_of_parameters` (a list assigned later takes the per-fold route)."""
        params = self.list_of_parameters
        self._shared_backbone_params = params if backbones_identical(params) else None
        self._fold_engine = None

    def initialize_from_trained_model_folder(self, model_training_output_dir: str, use_folds,
                                             checkpoint_name: str = "checkpoint_final.pth"):
        """predict_from_raw_data.py:67-130: plans, dataset.json and the fold checkpoints of a trained model folder
        (use_folds None = every `fold_<k>` with the checkpoint, "all" = `fold_all`).  The trainer name, configuration and
        mirroring axes come from the first checkpoint; the network is the native `DinoUNet` of that trainer's variant,
        built on the device with the first fold's weights.  Folds that share the backbone (the folds of one run) run it
        once per tile batch."""
        from . import predict as PR
        from .checkpoint import match_keys
        pm, cm, dj, parameters, trainer_name, _, mirror_axes = PR.load_model_folder(
            model_training_output_dir, use_folds, checkpoint_name)
        heads = pm.get_label_manager(dj).num_segmentation_heads
        network = PR.build_network(trainer_name, cm, PR.num_input_channels(dj), heads)
        own = set(network.state_dict().keys())
        parameters = [match_keys(p, own) for p in parameters]
        network.load_state_dict(parameters[0])
        self.manual_initialization(network.to(self.device), pm, cm, parameters, dj, trainer_name, mirror_axes)

    def predict_from_files(self, list_of_lists_or_source_folder, output_folder_or_list_of_truncated_output_files,
                           save_probabilities: bool = False, overwrite: bool = True, num_processes_preprocessing: int = 3,
                           num_processes_segmentation_export: int = 3, folder_with_segs_from_prev_stage: str = None,
                           num_parts: int = 1, part_id: int = 0):
        """predict_from_raw_data.py:207-266 on the device (see dinounet_b200/predict.py): cases `<id>_<4 digits>` of a
        folder, or lists of files, to `<output>/<id><file_ending>` (and `.npz` / `.pkl` with `save_probabilities`),
        this part's share `[part_id::num_parts]`, finished cases skipped when `overwrite` is False."""
        from . import predict as PR
        return PR.predict_from_files(self, list_of_lists_or_source_folder, output_folder_or_list_of_truncated_output_files,
                                     save_probabilities, overwrite, num_processes_preprocessing,
                                     num_processes_segmentation_export, folder_with_segs_from_prev_stage, num_parts,
                                     part_id)

    def predict_from_list_of_npy_arrays(self, image_or_list_of_images, segs_from_prev_stage_or_list_of_segs_from_prev_stage,
                                        properties_or_list_of_properties, truncated_ofname, num_processes: int = 3,
                                        save_probabilities: bool = False, num_processes_segmentation_export: int = 3):
        """predict_from_raw_data.py:343-359 on the device: images [C, X, Y, Z] with their properties ('spacing') to the
        truncated output names, or, where there is none, the segmentation (and probabilities) returned."""
        from . import predict as PR
        return PR.predict_from_list_of_npy_arrays(self, image_or_list_of_images,
                                                  segs_from_prev_stage_or_list_of_segs_from_prev_stage,
                                                  properties_or_list_of_properties, truncated_ofname, num_processes,
                                                  save_probabilities, num_processes_segmentation_export)

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
        if params and params is self._shared_backbone_params:
            self.ensemble_route = "shared_backbone"
            return self._predict_folds_shared_backbone(data)
        self.ensemble_route = "per_fold"

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

    def _shared_fold_engine(self, dev: torch.device):
        """An engine of its own with the shared backbone packed once and every fold's weights after the taps, kept
        across calls for this `list_of_parameters` while the network's weights stay as this method left them.  It
        loads the last fold into the network (so the network holds it, as after the per-fold route) and packs the
        backbone from the network's own parameters, as the network's engine does."""
        params = self.list_of_parameters
        net = self.network
        cached = self._fold_engine
        if (cached is not None and cached[0] is params and cached[1] is net and cached[2] == net.weights_version
                and not net._repack_before_eval and cached[3].device == dev):
            return cached[3]
        self._fold_engine = None
        net.load_state_dict(params[-1])
        net._repack_before_eval = False     # the load already dropped the network's packed weights

        # the folds are packed from device copies of their weights after the taps, one fold at a time: BatchNorm folded
        # on the host rounds differently in the last bit from the network's engine, which packs device tensors
        def after_taps_on_device(sd):
            return {k: t.to(dev) for k, t in sd.items() if ".dinov3_adapter.backbone." not in k}

        eng = net.new_engine(net.state_dict(), dev)
        eng.pack_folds(after_taps_on_device(p) for p in params)
        self._fold_engine = (params, net, net.weights_version, eng)
        return eng

    def _fold_chunk(self, tiles_per_slice: int, D: int) -> int:
        if self.fold_chunk_slices is not None:
            return max(1, min(int(self.fold_chunk_slices), D))
        per = max(1, self.tile_batch)
        k0 = per // math.gcd(per, tiles_per_slice)     # slices whose tiles fill whole batches
        return max(1, min(k0 * max(1, (4 * per) // (k0 * tiles_per_slice)), D))

    @torch.no_grad()
    def _predict_folds_shared_backbone(self, input_image: torch.Tensor) -> torch.Tensor:
        """The fold ensemble when every fold holds the same backbone.  Per tile batch: one gather, one ViT pass, then
        each fold's SPM .. seg head on the shared taps, its logits accumulated before the next fold overwrites them.
        2-D tiles never mix slices, so the case runs in chunks of slices: each fold's fp16 accumulator covers one chunk,
        the gaussian weight count (the same for every fold) is kept once, and after the chunk each fold is finalized and
        the folds are combined in the order of `ensemble_logits`.  Every voxel sees the operations of the per-fold route,
        so the result has its bits.  Afterwards the network holds the last fold's weights, as after the per-fold route."""
        assert isinstance(input_image, torch.Tensor)
        assert input_image.ndim == 4, "input_image must be a 4D np.ndarray or torch.Tensor (c, x, y, z)"
        params = self.list_of_parameters
        net = self.network
        net.eval()
        patch = [int(p) for p in self.configuration_manager.patch_size]
        if len(patch) != 2 or patch[0] != patch[1]:
            raise NotImplementedError("the native engine runs square 2D patches (main_dinov3 forces 512x512)")
        lib = L.load()
        dev = self.device if self.device.index is not None else torch.device("cuda", torch.cuda.current_device())
        heads = int(self.label_manager.num_segmentation_heads)
        nf = len(params)
        data, revert = pad_to_patch_size(input_image, patch)
        slicers = self._internal_get_sliding_window_slicers(tuple(data.shape[1:]))
        data = data.to(dev, dtype=torch.float32, non_blocking=True).contiguous()
        Cin, D, H, W = data.shape
        th = tw = patch[0]
        variants = self._mirror_variants()
        nvar = len(variants)
        tiles = [(s[1], s[2].start, s[3].start) for s in slicers]
        tps = len(tiles) // D
        per = max(1, self.tile_batch)
        nb = per * nvar
        chunk = self._fold_chunk(tps, D)
        gaussian = compute_gaussian(tuple(patch), sigma_scale=1. / 8, value_scaling_factor=10,
                                    device=dev) if self.use_gaussian else None
        eng = self._shared_fold_engine(dev)
        if eng.ncls != heads:
            raise ValueError(f"network produces {eng.ncls} heads, label manager expects {heads}")
        _, bufs = eng.get_plan(nb, th)
        hs, ws = revert[2], revert[3]
        out = torch.empty((heads, D, hs.stop - hs.start, ws.stop - ws.start), dtype=torch.half, device=dev)
        acc_all = torch.empty(nf * heads * chunk * H * W, dtype=torch.half, device=dev)
        npred_all = torch.empty(chunk * H * W, dtype=torch.half, device=dev)
        flag = torch.zeros(1, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            for d0 in range(0, D, chunk):
                dc = min(chunk, D - d0)
                plane = dc * H * W
                ctiles = tiles[d0 * tps:(d0 + dc) * tps]
                n_batches = (len(ctiles) + per - 1) // per
                desc = np.zeros((n_batches, nb, 4), dtype=np.int32)
                for t, (d, y0, x0) in enumerate(ctiles):        # slices relative to the chunk
                    for v, bits in enumerate(variants):
                        desc[t // per, (t % per) * nvar + v] = (d - d0, y0, x0, bits)
                for t in range(len(ctiles), n_batches * per):   # fill the last batch with repeats of the chunk's first tile
                    desc[t // per, (t % per) * nvar:(t % per + 1) * nvar] = desc[0, :nvar]
                desc_dev = torch.from_numpy(desc).to(dev)
                accs = [acc_all[f * heads * plane:(f + 1) * heads * plane].view(heads, dc, H, W) for f in range(nf)]
                acc_all[:nf * heads * plane].zero_()
                npred = npred_all[:plane].zero_()
                vol = data.data_ptr() + d0 * H * W * data.element_size()   # slice d0 of channel 0; channel stride D*H*W
                for b in range(n_batches):
                    dptr = desc_dev[b].data_ptr()
                    L.check(lib.b2u_sw_gather_tiles(vol, bufs["x"].data_ptr(), dptr, nb, Cin, D, H, W, th, tw, stream),
                            "sw_gather_tiles")
                    eng.run_resident(nb, th, self.use_graph, part="vit")
                    for f in range(nf):
                        logits, _ = eng.run_fold_rest(nb, th, f, self.use_graph)
                        for t in range(min(per, len(ctiles) - b * per)):
                            L.check(lib.b2u_sw_accumulate(logits.data_ptr(), dptr, t * nvar, nvar,
                                                          gaussian.data_ptr() if gaussian is not None else None,
                                                          accs[f].data_ptr(), npred.data_ptr() if f == 0 else None,
                                                          heads, dc, H, W, th, tw, stream), "sw_accumulate")
                for f in range(nf):
                    L.check(lib.b2u_sw_finalize(accs[f].data_ptr(), npred.data_ptr(), heads, plane, flag.data_ptr(),
                                                stream), "sw_finalize")
                for f in range(1, nf):
                    L.check(lib.b2u_pre_ensemble_f16(accs[0].data_ptr(), accs[f].data_ptr(), heads * plane, 0, stream),
                            "b2u_pre_ensemble_f16")
                L.check(lib.b2u_pre_ensemble_f16(accs[0].data_ptr(), None, heads * plane, nf, stream),
                        "b2u_pre_ensemble_f16")
                out[:, d0:d0 + dc].copy_(accs[0][:, :, hs, ws])
        if int(flag.item()):
            raise RuntimeError("Encountered inf in predicted array. Aborting... If this problem persists, "
                               "reduce value_scaling_factor in compute_gaussian or increase the dtype of "
                               "predicted_logits to fp32")
        return out

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
