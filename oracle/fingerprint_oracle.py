"""A numpy restatement of the device fingerprint (dinounet_b200/fingerprint.py), step for step: the foreground's C-order
indices, the host draws `RandomState(1234).randint(0, n_fg, num_samples)` per channel on one stream, the gathers, the
order statistics at the ranks the device selects (here from `np.partition`), numpy's pairwise sums (`np.sum`) finished
by `finish_mean` / `finish_std`, and the host finishing of `fingerprint.statistics_from`.  tests/test_fingerprint_cpu.py
pins it to the reference's own `DatasetFingerprintExtractor` (tests/golden/fingerprint_cases.npz)."""
import json

import numpy as np

from dinounet_b200 import fingerprint as F


def order_statistics(x: np.ndarray, ranks) -> dict:
    part = np.partition(x, list(ranks))
    return {r: part[r] for r in ranks}


def vector_statistics(x: np.ndarray, with_std: bool) -> dict:
    """The reference's statistics of one vector, computed the device's way."""
    dtype, n = x.dtype, len(x)
    mean = F.finish_mean(np.sum(x), n, dtype)
    std = F.finish_std(np.sum(np.square(x - mean)), n, dtype) if with_std else None
    return F.statistics_from(order_statistics(x, F.statistic_ranks(n, dtype)), n, dtype, mean, std)


def collect_foreground_intensities(segmentation, images, seed: int = 1234, num_samples: int = 10000):
    idx = np.flatnonzero(segmentation[0] > 0)
    rs = np.random.RandomState(seed)
    samples, stats = [], []
    for c in range(len(images)):
        fg = images[c].ravel()[idx]
        if len(idx) == 0:
            samples.append([])
            stats.append({k: np.nan for k in ("mean", "median", "min", "max", "percentile_99_5", "percentile_00_5")})
            continue
        samples.append(fg[rs.randint(0, len(idx), num_samples)])
        stats.append(vector_statistics(fg, with_std=False))
    return samples, stats


def dataset_vectors(cases, num_samples: int) -> list:
    """Each channel's samples concatenated in case order, as `run` concatenates them (float64 once a case is empty)."""
    per_case = [collect_foreground_intensities(seg, images, num_samples=num_samples)[0] for seg, images in cases]
    return [np.concatenate([r[c] for r in per_case]) for c in range(len(per_case[0]))]


def fingerprint(cases, spacings, num_channels: int, budget: float = 10e7) -> dict:
    """`run`'s dict for cases [(seg, images)] in key order."""
    vectors = dataset_vectors(cases, int(budget // len(cases)))
    stats = {}
    for i in range(num_channels):
        x = vectors[i]
        if len(x) == 0:
            raise ValueError("zero-size array to reduction operation minimum which has no identity")
        s = vector_statistics(x, with_std=True)
        stats[i] = {k: float(s[k]) for k in ("mean", "median", "std", "min", "max", "percentile_99_5",
                                             "percentile_00_5")}
    shapes = [images.shape[1:] for _, images in cases]
    return {"spacings": spacings, "shapes_after_crop": shapes, "foreground_intensity_properties_per_channel": stats,
            "median_relative_size_after_cropping": np.median([np.prod(s) / np.prod(s) for s in shapes], 0)}


def fingerprint_json(fp: dict) -> str:
    """batchgenerators' save_json: json.dump with sort_keys and indent 4."""
    return json.dumps(fp, sort_keys=True, indent=4)
