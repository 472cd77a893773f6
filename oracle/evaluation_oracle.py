"""CPU restatement of the reference's per-case evaluation (dinounet/evaluation/evaluate_predictions.py:76-230
`compute_metrics`) with numpy and scipy, including medpy's `hd95` / `asd` (medpy 0.4/0.5 `__surface_distances`), which
the reference imports and which is not installed here.  Test-only: it is the yardstick for dinounet_b200.evaluation.

GOLDEN_CASES / make_case define the seeded cases of tests/golden/evaluation_cases.npz (oracle/make_golden_evaluation.py).
"""
import numpy as np
from scipy import ndimage as ndi

METRIC_KEYS = ("Dice", "IoU", "Sensitivity", "Specificity", "Precision", "HD95", "ASD", "FP", "TP", "FN", "TN",
               "n_pred", "n_ref")


# ---- medpy.metric.binary


def surface_distances(result, reference, voxelspacing=None, connectivity=1):
    """medpy's `__surface_distances`: the distances of result's border voxels to reference's border, in C order."""
    result = np.atleast_1d(result.astype(bool))
    reference = np.atleast_1d(reference.astype(bool))
    if voxelspacing is not None:
        voxelspacing = tuple(voxelspacing)
        if len(voxelspacing) != result.ndim:
            raise RuntimeError("sequence argument must have length equal to input rank")
        voxelspacing = np.asarray(voxelspacing, dtype=np.float64)
    footprint = ndi.generate_binary_structure(result.ndim, connectivity)
    if np.count_nonzero(result) == 0:
        raise RuntimeError("The first supplied array does not contain any binary object.")
    if np.count_nonzero(reference) == 0:
        raise RuntimeError("The second supplied array does not contain any binary object.")
    result_border = result ^ ndi.binary_erosion(result, structure=footprint, iterations=1)
    reference_border = reference ^ ndi.binary_erosion(reference, structure=footprint, iterations=1)
    dt = ndi.distance_transform_edt(~reference_border, sampling=voxelspacing)
    return dt[result_border]


def hd95(result, reference, voxelspacing=None, connectivity=1):
    hd1 = surface_distances(result, reference, voxelspacing, connectivity)
    hd2 = surface_distances(reference, result, voxelspacing, connectivity)
    return np.percentile(np.hstack((hd1, hd2)), 95)


def asd(result, reference, voxelspacing=None, connectivity=1):
    return surface_distances(result, reference, voxelspacing, connectivity).mean()


def brute_force_distances(result_border, reference_border, spacing):
    """All pairs, float64, scipy's formula: sqrt of ((d0 s0)^2 + (d1 s1)^2) + (d2 s2)^2 minimised over the reference's
    border voxels, for each of result's border voxels in C order."""
    src = np.argwhere(result_border)
    dst = np.argwhere(reference_border)
    acc = None
    for a in range(result_border.ndim):
        t = (dst[None, :, a] - src[:, None, a]).astype(np.float64) * float(spacing[a])
        acc = t * t if acc is None else acc + t * t
    return np.sqrt(acc.min(axis=1))


# ---- evaluate_predictions.compute_metrics on arrays


def region_or_label_to_mask(seg, r):
    if np.isscalar(r):
        return seg == r
    mask = np.zeros_like(seg, dtype=bool)
    for v in r:
        mask[seg == v] = True
    return mask


def surface_spacing(spacing, ndim):
    """evaluate_predictions.py:123-136 (the spacing medpy receives)."""
    if len(spacing) == ndim or len(spacing) == ndim - 1:
        return tuple(float(s) for s in spacing)
    if len(spacing) > ndim:
        return tuple(float(s) for s in spacing[-ndim:])
    return tuple(float(s) for s in spacing) + (1.0,) * (ndim - len(spacing))


def surface_metrics(mask_ref, mask_pred, spacing):
    if not np.any(mask_ref) or not np.any(mask_pred):
        return np.nan, np.nan
    sp = surface_spacing(spacing, mask_ref.ndim)
    try:
        return float(hd95(mask_pred, mask_ref, sp)), float(asd(mask_pred, mask_ref, sp))
    except RuntimeError:
        return np.nan, np.nan


def compute_metrics_arrays(seg_ref, seg_pred, labels_or_regions, ignore_label=None, spacing=None):
    """The reference's `results['metrics']` for two arrays shaped (1, *spatial)."""
    if spacing is None:
        spacing = (1.0,) * (seg_ref.ndim - 1)
    ignore_mask = seg_ref == ignore_label if ignore_label is not None else None
    use = np.ones_like(seg_ref, dtype=bool) if ignore_mask is None else ~ignore_mask
    out = {}
    for r in labels_or_regions:
        mr, mp = region_or_label_to_mask(seg_ref, r), region_or_label_to_mask(seg_pred, r)
        tp = np.sum((mr & mp) & use)
        fp = np.sum(((~mr) & mp) & use)
        fn = np.sum((mr & (~mp)) & use)
        tn = np.sum(((~mr) & (~mp)) & use)
        m = {}
        if tp + fp + fn == 0:
            m["Dice"], m["IoU"] = np.nan, np.nan
        else:
            m["Dice"] = 2 * tp / (2 * tp + fp + fn)
            m["IoU"] = tp / (tp + fp + fn)
        m["Sensitivity"] = tp / (tp + fn) if tp + fn > 0 else np.nan
        m["Specificity"] = tn / (tn + fp) if tn + fp > 0 else np.nan
        m["Precision"] = tp / (tp + fp) if tp + fp > 0 else np.nan
        if mr.shape[0] == 1:
            mr, mp = np.squeeze(mr, axis=0), np.squeeze(mp, axis=0)
        m["HD95"], m["ASD"] = surface_metrics(mr, mp, spacing)
        m["FP"], m["TP"], m["FN"], m["TN"] = fp, tp, fn, tn
        m["n_pred"], m["n_ref"] = fp + tp, fn + tp
        out[r] = m
    return out


def pair_distances(seg_ref, seg_pred, r, spacing):
    """(surf(pred, ref), surf(ref, pred)) of one label or region, or two empty arrays when a mask is empty."""
    mr = np.squeeze(region_or_label_to_mask(seg_ref, r), axis=0)
    mp = np.squeeze(region_or_label_to_mask(seg_pred, r), axis=0)
    if not mr.any() or not mp.any():
        return np.zeros(0), np.zeros(0)
    sp = surface_spacing(spacing, mr.ndim)
    return surface_distances(mp, mr, sp), surface_distances(mr, mp, sp)


# ---- seeded golden cases


def _blobs(rng, shape, labels, count=2):
    seg = np.zeros(shape, np.uint8)
    grid = np.indices(shape).astype(np.float64)
    for lab in labels:
        for _ in range(count):
            c = [rng.uniform(0.2, 0.8) * s for s in shape]
            rad = [max(1.0, rng.uniform(0.12, 0.3) * s) for s in shape]
            inside = sum(((g - ci) / ri) ** 2 for g, ci, ri in zip(grid, c, rad)) <= 1.0
            seg[inside] = lab
    return seg


def _perturb(rng, seg, labels):
    pred = np.roll(seg, int(rng.integers(-2, 3)), axis=int(rng.integers(0, seg.ndim)))
    flip = rng.random(seg.shape) < 0.01
    pred[flip] = rng.choice(np.asarray([0, *labels], np.uint8), size=int(flip.sum()))
    return pred


# name, spatial shape, spacing, labels_or_regions, ignore_label, ref dtype, pred dtype
GOLDEN_CASES = [
    ("labels3_spacing311", (20, 40, 48), (3.0, 1.0, 1.0), [1, 2, 3], None, np.uint8, np.uint8),
    ("labels2_fractional", (16, 32, 36), (2.5, 0.7, 0.7), [1, 2], None, np.float32, np.float32),
    ("regions_overlapping", (18, 30, 34), (3.0, 1.0, 1.0), [(1, 2, 3), (2, 3), (3,)], None, np.uint8, np.uint8),
    ("ignore_label", (14, 36, 30), (2.5, 0.7, 0.7), [1, 2], 4, np.uint8, np.uint8),
    ("empty_masks", (12, 24, 28), (3.0, 1.0, 1.0), [1, 2, 3, 4], None, np.uint8, np.float32),
    ("slice2d", (1, 64, 80), (999.0, 1.0, 1.0), [1, 2], None, np.float32, np.float32),
    ("touching_faces", (10, 14, 16), (1.0, 1.0, 1.0), [1, 2], None, np.float32, np.uint8),
]


def make_case(name):
    """Seeded (seg_ref, seg_pred) shaped (1, *spatial) of one golden case."""
    i = [c[0] for c in GOLDEN_CASES].index(name)
    _, shape, _, regions, ignore, dt_ref, dt_pred = GOLDEN_CASES[i]
    rng = np.random.default_rng(1000 + i)
    labels = sorted({v for r in regions for v in (r if isinstance(r, tuple) else (r,))})
    if name == "touching_faces":
        ref = np.ones(shape, np.uint8)                 # label 1 fills the volume but for a label-2 core
        ref[3:7, 4:10, 5:11] = 2
        pred = ref.copy()
        pred[:, :, -1] = 2                             # label 2 reaches the last x face in the prediction only
        pred[4:6, 6:8, 7:9] = 0
    else:
        ref = _blobs(rng, shape, labels)
        pred = _perturb(rng, ref, labels)
    if name == "ignore_label":
        ref[rng.random(shape) < 0.05] = ignore
    if name == "empty_masks":
        ref[ref == 2] = 0                              # 2: empty reference, 3: empty prediction, 4: both empty
        pred[pred == 3] = 0
        ref[ref == 4] = 0
        pred[pred == 4] = 0
    return ref[None].astype(dt_ref), pred[None].astype(dt_pred)
