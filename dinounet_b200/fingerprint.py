"""Dataset fingerprint on the device (reference: `DatasetFingerprintExtractor`,
experiment_planning/dataset_fingerprint/fingerprint_extractor.py), a drop-in the reference's own functions take:

    extract_fingerprint_dataset(d, DeviceFingerprintExtractor, num_processes, check_dataset_integrity, clean, verbose)

`DeviceFingerprintExtractor.run` writes the same `dataset_fingerprint.json`, byte for byte, and returns the same dict:
* the crop is the whole volume (cropping.py:34 marks every voxel of the nonzero mask, so its `binary_fill_holes` has no
  effect): `shapes_after_crop` are the images' shapes and `median_relative_size_after_cropping` is 1.0;
* per case, the foreground `seg[0] > 0` is compacted on the device in C order (`b2u_fp_fg_compact`) and the
  `num_samples` intensities per channel are gathered in place into the dataset's vector of that channel
  (`b2u_fp_gather`).  The ranks are the reference's draws: `RandomState(1234).choice(fg, k, replace=True)` is
  `fg[randint(0, len(fg), k)]`, one stream across the channels; they run on the host while the device reads and
  compacts the next case;
* the dataset statistics come from one exact multi-rank radix select per channel (`b2u_fp_select`: min, max, the
  median's and both percentiles' neighbours) and numpy's pairwise sums (`b2u_fp_moments`), read once per vector and
  finished on the host with numpy's formulas (`quantile_positions`, `lerp`, `median_of`) in the vector's dtype.  A case
  without foreground contributes the reference's `[]`, which promotes the concatenation to float64: every statistic is
  then computed in float64 (the select runs on the float32 values, which the promotion maps exactly and monotonically).

Rejected before any launch: images that are not float32 (every reader delivers float32), a seg dtype other than uint8,
int8, int16, uint16, int32, float32, shapes that differ, 2^31 voxels or more in a case, and +-inf in the images
(NotImplementedError: the reference would write inf / nan statistics).  NaN gives the reference's AssertionError and a
dataset without foreground numpy's ValueError.  -0.0 and +0.0 are one value to the select, which returns +0.0.

Peak device memory of `run`: the dataset vectors, 4 * C * num_samples * n_cases bytes (about 4e8 bytes per channel at
the default budget of 1e8 samples; float64 statistics add a converted copy of one channel, 8 bytes per sample, plus
its tree slots), and two cases in flight, each its images, seg and one int32 index per voxel.
"""
import ctypes
import json
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import lib as L
from . import preprocess as PP

SEED = 1234
PERCENTILES = (99.5, 0.5)
NAN_SEG = "Segmentation contains NaN values. grrrr.... :-("
NAN_IMAGES = "Images contains NaN values. grrrr.... :-("


# ---- numpy's order-statistic formulas (numpy/lib/_function_base_impl.py), for the host finishing ---------------------


def quantile_positions(n: int, q: float, dtype):
    """np.percentile(x, q, method="linear") of n values of `dtype`: (previous rank, next rank, gamma), the ranks
    0-based in ascending order.  q / 100 and the virtual index (n - 1) * q are computed in the array's dtype, as
    `percentile` and `_quantile` do; `_get_indexes` and `_get_gamma` follow."""
    dtype = np.dtype(dtype)
    quantiles = np.true_divide(q, dtype.type(100), out=...)
    virtual = np.asanyarray((n - 1) * quantiles)
    previous = np.asanyarray(np.floor(virtual))
    nxt = np.asanyarray(previous + 1)
    above = virtual >= n - 1
    if above.any():
        previous[above] = -1
        nxt[above] = -1
    below = virtual < 0
    if below.any():
        previous[below] = 0
        nxt[below] = 0
    previous = previous.astype(np.intp)
    nxt = nxt.astype(np.intp)
    gamma = np.asanyarray(np.asanyarray(virtual - previous), dtype=virtual.dtype)
    return int(previous) % n, int(nxt) % n, gamma


def lerp(a, b, t):
    """numpy's `_lerp` on the two neighbours (scalars of the array's dtype) and gamma."""
    diff_b_a = np.subtract(b, a)
    res = np.asanyarray(np.add(a, diff_b_a * t))
    np.subtract(b, diff_b_a * (1 - t), out=res, where=t >= 0.5, casting="unsafe", dtype=type(res.dtype))
    return res[()]


def median_ranks(n: int) -> list:
    """The ranks np.median averages."""
    return [n // 2 - 1, n // 2] if n % 2 == 0 else [(n - 1) // 2]


def median_of(values, dtype):
    """np.median's `mean` of the middle value(s), ascending, in `dtype`."""
    return np.mean(np.asarray(values, dtype=dtype))


def finish_mean(total, n: int, dtype):
    """numpy's `_mean` from the pairwise sum: the sum divided by the intp count in float64, then `dtype`."""
    return np.dtype(dtype).type(np.float64(total) / np.intp(n))


def finish_std(sq_total, n: int, dtype):
    """numpy's std from `_var`'s pairwise sum of (x - mean)^2 (no clamp)."""
    t = np.dtype(dtype).type
    return t(np.sqrt(t(np.float64(sq_total) / np.intp(n))))


def statistic_ranks(n: int, dtype) -> list:
    """The distinct ranks the dataset statistics read: min, max, the median's and both percentiles' neighbours."""
    ranks = [0, n - 1, *median_ranks(n)]
    for q in PERCENTILES:
        ranks += quantile_positions(n, q, dtype)[:2]
    return sorted(set(ranks))


def statistics_from(values: dict, n: int, dtype, mean, std=None) -> dict:
    """The reference's statistics of one vector from its order statistics {rank: value} (and mean / std), in `dtype`."""
    t = np.dtype(dtype).type
    v = {r: t(x) for r, x in values.items()}
    pct = {}
    for q in PERCENTILES:
        lo, hi, gamma = quantile_positions(n, q, dtype)
        pct[q] = lerp(v[lo], v[hi], gamma)
    out = {"mean": t(mean), "median": median_of([v[r] for r in median_ranks(n)], dtype)}
    if std is not None:
        out["std"] = t(std)
    out.update({"min": v[0], "max": v[n - 1], "percentile_99_5": pct[99.5], "percentile_00_5": pct[0.5]})
    return out


# ---- input checks (before any launch) --------------------------------------------------------------------------------


def _seg_code(seg) -> int:
    if isinstance(seg, torch.Tensor):
        if seg.dtype not in PP._TORCH_SEG_DTYPES:
            raise NotImplementedError(f"seg dtype {seg.dtype} is not implemented on the device (implemented: uint8, "
                                      "int8, int16, uint16, int32, float32)")
        return PP.SEG_DTYPE_CODES[np.dtype(PP._TORCH_SEG_DTYPES[seg.dtype])]
    if seg.dtype not in PP.SEG_DTYPE_CODES:
        raise NotImplementedError(f"seg dtype {seg.dtype} is not implemented on the device (implemented: uint8, int8, "
                                  "int16, uint16, int32, float32)")
    return PP.SEG_DTYPE_CODES[seg.dtype]


def check_case(segmentation, images) -> int:
    """The reference's assertions and this module's scope, before any launch; returns the seg's dtype code."""
    assert images.ndim == 4
    assert segmentation.ndim == 4
    tensor = isinstance(images, torch.Tensor)
    if images.dtype != (torch.float32 if tensor else np.float32):
        raise NotImplementedError(f"images of dtype {images.dtype}: the device fingerprint takes float32 images (what "
                                  "every reader delivers)")
    code = _seg_code(segmentation)
    if tuple(images.shape[1:]) != tuple(segmentation.shape[1:]):
        raise IndexError(f"the segmentation {tuple(segmentation.shape)} and the images {tuple(images.shape)} differ "
                         "in shape")
    if int(np.prod(images.shape[1:])) >= 2 ** 31:
        raise NotImplementedError(f"a case of {tuple(images.shape[1:])} has 2^31 voxels or more")
    if code == PP.SEG_DTYPE_CODES[np.dtype(np.float32)]:
        assert not bool((torch.isnan(segmentation) if tensor else np.isnan(segmentation)).any()), NAN_SEG
    if not bool((torch.isfinite(images) if tensor else np.isfinite(images)).all()):   # one pass for finite input
        assert not bool((torch.isnan(images) if tensor else np.isnan(images)).any()), NAN_IMAGES
        raise NotImplementedError("the images hold +-inf: the reference would write inf / nan statistics")
    return code


def _as_input(segmentation, images):
    """(seg, images, device or None): CUDA tensors stay where they are, anything else becomes numpy."""
    if isinstance(images, torch.Tensor) and images.is_cuda:
        if not isinstance(segmentation, torch.Tensor) or segmentation.device != images.device:
            raise ValueError("the segmentation must be a tensor on the images' device")
        return segmentation.detach(), images.detach(), images.device
    if isinstance(segmentation, torch.Tensor):
        segmentation = segmentation.detach().cpu().numpy()
    if isinstance(images, torch.Tensor):
        images = images.detach().cpu().numpy()
    return np.asarray(segmentation), np.asarray(images), None


# ---- one case on the device ------------------------------------------------------------------------------------------


class _Case:
    """A case uploaded and its foreground compacted (asynchronously); `count()` reads the foreground size once."""

    def __init__(self, segmentation, images, code: int, dev, lib, stream):
        self.C = int(images.shape[0])
        self.n = int(np.prod(images.shape[1:]))
        s = segmentation[0]
        if isinstance(s, torch.Tensor):
            s = (s.view(torch.int16) if code == 3 else s).contiguous()
            self.seg = s if s.device == dev else s.to(dev)
            self.img = images.contiguous().to(dev)
        else:
            s = s.view(np.int16) if code == 3 else s
            self.seg = torch.from_numpy(np.ascontiguousarray(s)).to(dev, non_blocking=True)
            self.img = torch.from_numpy(np.ascontiguousarray(images)).to(dev, non_blocking=True)
        self.lib, self.stream, self.dev = lib, stream, dev
        self.idx = torch.empty(self.n, dtype=torch.int32, device=dev)
        work = torch.empty(int(lib.b2u_pre_seg_compact_work_ints(self.n)), dtype=torch.int32, device=dev)
        self._count = torch.empty(1, dtype=torch.int64, device=dev)
        L.check(lib.b2u_fp_fg_compact(self.seg.data_ptr(), code, self.n, work.data_ptr(), self.idx.data_ptr(),
                                      self._count.data_ptr(), stream), "b2u_fp_fg_compact")
        self._count_host = torch.empty(1, dtype=torch.int64, pin_memory=True)
        self._count_host.copy_(self._count, non_blocking=True)
        self._ready = torch.cuda.Event()
        self._ready.record(torch.cuda.current_stream(dev))
        self._fg = None

    def count(self) -> int:
        self._ready.synchronize()
        return int(self._count_host[0])

    def gather_samples(self, ranks: np.ndarray, out: torch.Tensor, offset: int):
        """out[c, offset + j] = fg_c[ranks[c, j]]; ranks [C, m] int64 from the host."""
        r = torch.from_numpy(ranks).to(self.dev)
        m = int(ranks.shape[1])
        L.check(self.lib.b2u_fp_gather(self.img.data_ptr(), self.C, self.n, self.idx.data_ptr(), r.data_ptr(), m,
                                       out[:, offset:].data_ptr(), int(out.stride(0)), self.stream), "b2u_fp_gather")

    def foreground(self, count: int) -> torch.Tensor:
        """fp32 [C, count]: every channel's foreground in C order (images[c][mask])."""
        fg = torch.empty((self.C, count), dtype=torch.float32, device=self.dev)
        L.check(self.lib.b2u_fp_gather(self.img.data_ptr(), self.C, self.n, self.idx.data_ptr(), None, count,
                                       fg.data_ptr(), count, self.stream), "b2u_fp_gather")
        return fg


def _launch_statistics(x: torch.Tensor, n: int, f64: bool, with_std: bool, lib, stream):
    """Launches the select and the moments of x[:n] (fp32, contiguous); returns (ranks, values fp32 [R], stats [2],
    work buffers).  Buffers freed before the stream has run reuse only on this stream, after it."""
    dtype = np.float64 if f64 else np.float32
    ranks = statistic_ranks(n, dtype)
    host = (ctypes.c_int64 * len(ranks))(*ranks)
    vals = torch.empty(len(ranks), dtype=torch.float32, device=x.device)
    work = torch.empty(int(lib.b2u_fp_select_work_bytes()), dtype=torch.uint8, device=x.device)
    L.check(lib.b2u_fp_select(x.data_ptr(), n, host, len(ranks), work.data_ptr(), vals.data_ptr(), stream),
            "b2u_fp_select")
    stats = torch.empty(2, dtype=torch.float64 if f64 else torch.float32, device=x.device)
    mwork = torch.empty(int(lib.b2u_fp_moments_work_bytes(n, int(f64))), dtype=torch.uint8, device=x.device)
    L.check(lib.b2u_fp_moments(x.data_ptr(), n, int(f64), int(with_std), mwork.data_ptr(), stats.data_ptr(), stream),
            "b2u_fp_moments")
    return ranks, vals, stats, (work, mwork)


def _draws(rs: np.random.RandomState, count: int, C: int, num_samples: int) -> np.ndarray:
    """rs.choice(fg, num_samples, replace=True) per channel is fg[rs.randint(0, count, num_samples)]."""
    return np.stack([rs.randint(0, count, num_samples) for _ in range(C)]).astype(np.int64, copy=False)


# ---- the extractor ---------------------------------------------------------------------------------------------------


class DeviceFingerprintExtractor:
    """Drop-in for the reference's DatasetFingerprintExtractor: the same constructor, attributes, `run`, and the static
    `collect_foreground_intensities` and `analyze_case`."""

    def __init__(self, dataset_name_or_id, num_processes: int = 8, verbose: bool = False):
        dataset_name = PP._dataset_name(dataset_name_or_id)
        self.verbose = verbose
        self.dataset_name = dataset_name
        raw, _ = PP._raw_and_preprocessed()
        self.input_folder = os.path.join(raw, dataset_name)
        self.num_processes = num_processes
        with open(os.path.join(self.input_folder, "dataset.json")) as f:
            self.dataset_json = json.load(f)
        self.dataset = PP._get_filenames_of_train_images_and_targets(self.input_folder, self.dataset_json)
        self.num_foreground_voxels_for_intensitystats = 10e7

    @staticmethod
    def collect_foreground_intensities(segmentation, images, seed: int = 1234, num_samples: int = 10000):
        """The reference's (fingerprint_extractor.py:41-80): per channel the `num_samples` drawn foreground intensities
        and the case's statistics (mean, median, min, max, percentile_99_5, percentile_00_5 in float32; `[]` and NaN
        without foreground).  numpy input gives numpy results; CUDA tensors give tensors on their device."""
        segmentation, images, dev = _as_input(segmentation, images)
        code = check_case(segmentation, images)
        target = dev or torch.device("cuda", torch.cuda.current_device())
        lib = L.load()
        with torch.cuda.device(target):
            stream = torch.cuda.current_stream(target).cuda_stream
            case = _Case(segmentation, images, code, target, lib, stream)
            count = case.count()
            C = case.C
            if count == 0:
                nan = {"mean": np.nan, "median": np.nan, "min": np.nan, "max": np.nan, "percentile_99_5": np.nan,
                       "percentile_00_5": np.nan}
                return [[] for _ in range(C)], [dict(nan) for _ in range(C)]
            fg = case.foreground(count)
            launched = [_launch_statistics(fg[c], count, False, False, lib, stream) for c in range(C)]
            ranks = _draws(np.random.RandomState(seed), count, C, num_samples)   # while the device works
            samples = torch.empty((C, num_samples), dtype=torch.float32, device=target)
            case.gather_samples(ranks, samples, 0)
            stats = [statistics_from(dict(zip(rk, v.cpu().numpy())), count, np.float32, st.cpu().numpy()[0])
                     for rk, v, st, _ in launched]
            if dev is None:
                return [s for s in samples.cpu().numpy()], stats
            return [samples[c] for c in range(C)], [{k: torch.tensor(v, device=dev) for k, v in s.items()}
                                                    for s in stats]

    @staticmethod
    def analyze_case(image_files, segmentation_file, reader_writer_class, num_samples: int = 10000):
        """The reference's (lines 82-105): (shape after crop, spacing, intensities, statistics, relative size 1.0)."""
        rw = reader_writer_class()
        images, properties_images = rw.read_images(image_files)
        segmentation, _ = rw.read_seg(segmentation_file)
        intensities, stats = DeviceFingerprintExtractor.collect_foreground_intensities(segmentation, images,
                                                                                      num_samples=num_samples)
        shape = images.shape[1:]
        return shape, properties_images["spacing"], intensities, stats, np.prod(shape) / np.prod(shape)

    def run(self, overwrite_existing: bool = False) -> dict:
        """The reference's `run` (lines 107-194): `<nnUNet_preprocessed>/<dataset>/dataset_fingerprint.json`, written
        with sort_keys and indent 4 (or loaded when it exists and overwrite_existing is False)."""
        return self._run(overwrite_existing)

    def _run(self, overwrite_existing: bool, check=None) -> dict:
        """`run`, with `check` (integrity._FusedCheck) verifying the dataset in the same read of each case."""
        _, preprocessed = PP._raw_and_preprocessed()
        out_folder = os.path.join(preprocessed, self.dataset_name)
        os.makedirs(out_folder, exist_ok=True)
        properties_file = os.path.join(out_folder, "dataset_fingerprint.json")
        if os.path.isfile(properties_file) and not overwrite_existing:
            with open(properties_file) as f:
                return json.load(f)
        keys = list(self.dataset.keys())
        rw_class = _determine_reader_writer(self.dataset_json, self.dataset[keys[0]]["images"][0])
        num_samples = int(self.num_foreground_voxels_for_intensitystats // len(self.dataset))
        shapes, spacings, vectors, total, promoted = self._sample_dataset(keys, rw_class, num_samples, check)
        num_channels = len(self.dataset_json["channel_names"].keys() if "channel_names" in self.dataset_json.keys()
                           else self.dataset_json["modality"].keys())
        if total == 0:
            raise ValueError("zero-size array to reduction operation minimum which has no identity")
        dtype = np.float64 if promoted else np.float32
        lib = L.load()
        dev = vectors.device
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            launched = [_launch_statistics(vectors[i], total, promoted, True, lib, stream) for i in range(num_channels)]
            intensity_statistics_per_channel = {}
            for i, (rk, v, st, _) in enumerate(launched):
                s = st.cpu().numpy()
                stats = statistics_from(dict(zip(rk, v.cpu().numpy())), total, dtype, s[0], s[1])
                intensity_statistics_per_channel[i] = {k: float(stats[k]) for k in (
                    "mean", "median", "std", "min", "max", "percentile_99_5", "percentile_00_5")}
        fingerprint = {
            "spacings": spacings,
            "shapes_after_crop": shapes,
            "foreground_intensity_properties_per_channel": intensity_statistics_per_channel,
            "median_relative_size_after_cropping": np.median([np.prod(s) / np.prod(s) for s in shapes], 0),
        }
        try:
            with open(properties_file, "w") as f:
                json.dump(fingerprint, f, sort_keys=True, indent=4)
        except Exception:
            if os.path.isfile(properties_file):
                os.remove(properties_file)
            raise
        return fingerprint

    def _sample_dataset(self, keys, rw_class, num_samples, check=None):
        """Reads and checks the cases ahead on `num_processes` threads and processes them in order on the current
        device: each case's draws run on the host while the device uploads and compacts the next case.  Returns
        (shapes, spacings, the dataset vectors fp32 [C, cap], the samples written per channel, whether the
        concatenation promotes).  With `check`, every case is also verified on its device copy, the cases are
        sampled only while the check and the fingerprint's own checks pass, and `check.finish()` reports (and
        raises) before anything is returned."""
        def read(k):   # and check, off the thread that drives the device
            rw = rw_class()
            images, props = rw.read_images(self.dataset[k]["images"])
            if check is not None:
                seg, props_seg = rw.read_seg(self.dataset[k]["label"])
                seg, images, _ = _as_input(seg, images)
                return images, seg, props, check.read(images, seg, props_seg)
            seg, _ = rw.read_seg(self.dataset[k]["label"])
            seg, images, _ = _as_input(seg, images)
            return images, seg, props, check_case(seg, images)

        lib = L.load()
        dev = torch.device("cuda", torch.cuda.current_device())
        shapes, spacings = [], []
        vectors, total, promoted = None, 0, False
        workers = max(1, int(self.num_processes))
        with torch.cuda.device(dev), ThreadPoolExecutor(workers) as pool:
            stream = torch.cuda.current_stream(dev).cuda_stream
            reads = [pool.submit(read, k) for k in keys[:workers]]
            pending = None
            for i, k in enumerate(keys + [None]):
                case = None
                if k is not None:
                    images, seg, props, code = reads[i].result()
                    reads[i] = None
                    if i + workers < len(keys):
                        reads.append(pool.submit(read, keys[i + workers]))
                    shapes.append(images.shape[1:])
                    spacings.append(props["spacing"])
                    if vectors is None:
                        vectors = torch.empty((images.shape[0], num_samples * len(keys)), dtype=torch.float32,
                                              device=dev)
                    if check is None:
                        case = _Case(seg, images, code, dev, lib, stream)
                    else:
                        case = check.case(k, images, seg, props, code,
                                          lambda c: _Case(seg, images, c, dev, lib, stream))
                if pending is not None and (check is None or check.sampling):   # the previous case's draws, while the device compacts this one
                    count = pending.count()
                    if count == 0:
                        promoted = True
                    else:
                        ranks = _draws(np.random.RandomState(SEED), count, pending.C, num_samples)
                        pending.gather_samples(ranks, vectors, total)
                        total += num_samples
                pending = case
            if check is not None:
                check.finish()
        return shapes, spacings, vectors, total, promoted


def _determine_reader_writer(dataset_json: dict, example_file: str):
    """The host nnU-Net's reader registry (tests substitute it)."""
    from dinounet.imageio.reader_writer_registry import determine_reader_writer_from_dataset_json
    return determine_reader_writer_from_dataset_json(dataset_json, example_file)
