"""CPU restatement of the reference's keep-the-largest-component postprocessing
(`dinounet/postprocessing/remove_connected_components.py`), for tests only.

The reference labels with acvl-utils' `remove_all_but_largest_component` (acvl-utils >=0.2.3,<0.3, as pinned by the
reference's requirements; `acvl_utils/morphology/morphology_helper.py` of 0.2.x): `label_with_component_sizes` is
skimage's `label(binary_image, return_num=True, connectivity=None)` followed by `np.bincount`, and
`generic_filter_components` keeps the component ids the filter returns.  skimage's default connectivity is full
(`ndim` hops), which is `scipy.ndimage.label` with a structure of ones; neither acvl-utils nor skimage is needed.

`determine_postprocessing_arrays` restates `determine_postprocessing` on in-memory cases, scored by
`oracle/evaluation_oracle.compute_metrics_arrays`.  The folder scenarios (`make_scenario`) are shared by the CPU test that
pins this restatement and the device module to the reference, the GPU test and the golden file.
"""
import json

import numpy as np
from scipy import ndimage as ndi

from . import evaluation_oracle as EO

SCENARIOS = ("fg_accepted", "fg_rejected_one_label_worse", "regions_overlapping", "existing_summary",
             "tied_components")


# ---- acvl-utils 0.2.x morphology_helper ------------------------------------------------------------------------------


def label_with_component_sizes(binary_image: np.ndarray, connectivity=None):
    assert connectivity is None
    labeled_image, _ = ndi.label(binary_image, structure=np.ones((3,) * binary_image.ndim, dtype=bool))
    component_sizes = {i + 1: j for i, j in enumerate(np.bincount(labeled_image.ravel())[1:])}
    return labeled_image, component_sizes


def generic_filter_components(binary_image: np.ndarray, filter_fn, connectivity=None):
    labeled_image, component_sizes = label_with_component_sizes(binary_image, connectivity)
    component_ids = list(component_sizes.keys())
    component_sizes = list(component_sizes.values())
    keep = filter_fn(component_ids, component_sizes)
    return np.isin(labeled_image.ravel(), keep).reshape(labeled_image.shape)


def remove_all_but_largest_component(binary_image: np.ndarray, connectivity=None) -> np.ndarray:
    filter_fn = lambda x, y: [i for i, j in zip(x, y) if j == max(y)]  # noqa: E731
    return generic_filter_components(binary_image, filter_fn, connectivity)


# ---- remove_connected_components.py ----------------------------------------------------------------------------------


def region_or_label_to_mask(segmentation: np.ndarray, region_or_label) -> np.ndarray:
    if np.isscalar(region_or_label):
        return segmentation == region_or_label
    mask = np.zeros_like(segmentation, dtype=bool)
    for r in region_or_label:
        mask[segmentation == r] = True
    return mask


def remove_all_but_largest_component_from_segmentation(segmentation, labels_or_regions, background_label=0):
    mask = np.zeros_like(segmentation, dtype=bool)
    if not isinstance(labels_or_regions, list):
        labels_or_regions = [labels_or_regions]
    for l_or_r in labels_or_regions:
        mask |= region_or_label_to_mask(segmentation, l_or_r)
    mask_keep = remove_all_but_largest_component(mask)
    ret = np.copy(segmentation)
    ret[mask & ~mask_keep] = background_label
    return ret


def _aggregate(cases_metrics, labels_or_regions) -> dict:
    """evaluate_predictions.py:269-286: np.nanmean per key and metric, the mean over every key but 0."""
    metric_list = list(cases_metrics[0][labels_or_regions[0]].keys())
    means = {r: {m: float(np.nanmean([c[r][m] for c in cases_metrics])) for m in metric_list}
             for r in labels_or_regions}
    foreground_mean = {m: float(np.mean([means[k][m] for k in means if not (k == 0 or k == "0")]))
                       for m in metric_list}
    return {"mean": means, "foreground_mean": foreground_mean}


def determine_postprocessing_arrays(cases, labels_or_regions, foreground_labels, ignore_label, spacing,
                                    baseline=None):
    """determine_postprocessing on cases [(ref, pred)] shaped (1, *spatial).  `baseline`: the summary means to start
    from (a pre-existing summary.json), else the predictions' own.  Returns the accepted kwargs, the final predictions,
    the baseline and the final summary means."""
    def summarize(preds):
        return _aggregate([EO.compute_metrics_arrays(ref, p, labels_or_regions, ignore_label, spacing)
                           for (ref, _), p in zip(cases, preds)], labels_or_regions)

    current = [pred for _, pred in cases]
    baseline = summarize(current) if baseline is None else baseline
    accepted, current_summary = [], baseline
    candidate = [remove_all_but_largest_component_from_segmentation(p[0], foreground_labels)[None] for p in current]
    s = summarize(candidate)
    do_this = s["foreground_mean"]["Dice"] > baseline["foreground_mean"]["Dice"]
    if do_this:
        do_this = not any(s["mean"][k]["Dice"] < baseline["mean"][k]["Dice"] for k in s["mean"])
    if do_this:
        accepted.append({"labels_or_regions": foreground_labels})
        current, current_summary = candidate, s
    if len(labels_or_regions) > 1:
        for r in labels_or_regions:
            candidate = [remove_all_but_largest_component_from_segmentation(p[0], r)[None] for p in current]
            s = summarize(candidate)
            if s["mean"][r]["Dice"] > current_summary["mean"][r]["Dice"]:
                accepted.append({"labels_or_regions": r})
                current, current_summary = candidate, s
    return accepted, current, baseline, current_summary


# ---- folder scenarios ------------------------------------------------------------------------------------------------


def _box(a, z, y, x, v):
    a[0, z[0]:z[1], y[0]:y[1], x[0]:x[1]] = v


def make_scenario(name: str) -> dict:
    """Two cases shaped (1, 6, 16, 16) (uint8 predictions, float32 references as an image reader returns them), the
    label setup and the expected kind of outcome:

    fg_accepted                  a spurious label-1 blob: removing all but the largest foreground component helps
    fg_rejected_one_label_worse  a spurious label-1 blob and a detached true part of label 2: the foreground step
                                 raises the mean Dice but lowers label 2's, so it is rejected; per label, 1 is
                                 accepted and 2 rejected
    regions_overlapping          the same volumes as regions (1, 2) and (2,)
    existing_summary             fg_accepted with a summary.json already present whose Dice values are 1
    tied_components              one label with two equal largest components, both kept, and a smaller blob
    """
    cases = []
    for c in range(2):
        ref = np.zeros((1, 6, 16, 16), np.uint8)
        if name == "tied_components":
            _box(ref, (1, 3), (2, 5), (2, 5), 1)
            _box(ref, (1, 3), (9, 12), (9 + c, 12 + c), 1)
            pred = ref.copy()
            _box(pred, (4, 6), (13, 15), (1, 3), 1)
        else:
            _box(ref, (1, 5), (2, 8), (2, 8), 1)
            _box(ref, (1, 5), (8, 12), (2, 8), 2)
            pred = ref.copy()
            pred[0, 1 + c, 4, 4] = 2   # a wrong voxel inside label 1, so Dice differs between the cases
            _box(pred, (1, 4), (13, 16), (12, 15), 1)
            if name != "fg_accepted" and name != "existing_summary":
                _box(ref, (1, 3), (13, 15), (2, 4), 2)
                _box(pred, (1, 3), (13, 15), (2, 4), 2)
        cases.append((f"case_{c}.npy", ref.astype(np.float32), pred))
    labels = [1] if name == "tied_components" else [1, 2]
    regions = [(1, 2), (2,)] if name == "regions_overlapping" else None
    return {"cases": cases, "foreground_labels": labels, "regions": regions,
            "labels_or_regions": regions if regions else labels, "ignore_label": None, "spacing": (2.0, 1.0, 1.0),
            "existing_summary": name == "existing_summary"}


def existing_summary_text(scenario: dict) -> str:
    """A summary.json as save_summary_json writes it, for the scenario's predictions, with every Dice set to 1."""
    lr = scenario["labels_or_regions"]
    per_case, results = [], []
    for f, ref, pred in scenario["cases"]:
        m = EO.compute_metrics_arrays(ref, pred, lr, scenario["ignore_label"], scenario["spacing"])
        results.append(m)
        per_case.append({"metrics": {str(k): {kk: float(vv) for kk, vv in v.items()} for k, v in m.items()},
                         "prediction_file": f, "reference_file": f})
    agg = _aggregate(results, lr)
    for k in agg["mean"]:
        agg["mean"][k]["Dice"] = 1.0
    agg["foreground_mean"]["Dice"] = 1.0
    return json.dumps({"foreground_mean": agg["foreground_mean"], "mean": {str(k): v for k, v in agg["mean"].items()},
                       "metric_per_case": per_case}, sort_keys=True, indent=4)


def scenario_baseline(scenario: dict):
    """The baseline means of a scenario with a pre-existing summary.json, else None."""
    if not scenario["existing_summary"]:
        return None
    d = json.loads(existing_summary_text(scenario))
    key = {str(k): k for k in scenario["labels_or_regions"]}
    return {"mean": {key[k]: v for k, v in d["mean"].items()},
            "foreground_mean": d["foreground_mean"]}


def run_scenario(name: str):
    s = make_scenario(name)
    return determine_postprocessing_arrays([(ref, pred) for _, ref, pred in s["cases"]], s["labels_or_regions"],
                                           s["foreground_labels"], s["ignore_label"], s["spacing"],
                                           scenario_baseline(s))


# ---- single-volume cases ---------------------------------------------------------------------------------------------


def random_mask_case(shape, density, seed, dtype=np.uint8, labels=(1, 2, 3)):
    """A label volume whose foreground has the given density, labels drawn uniformly."""
    rng = np.random.default_rng(seed)
    seg = np.where(rng.random(shape) < density, rng.choice(np.array(labels), size=shape), 0)
    return seg.astype(dtype)


GOLDEN_MASKS = [  # name, shape, density, seed, dtype, labels_or_regions, background
    ("u8_3d_p020", (9, 21, 37), 0.2, 1, np.uint8, [1, 2, 3], 0),
    ("i16_3d_p012_label2", (11, 9, 67), 0.12, 2, np.int16, 2, 0),
    ("f32_2d_p030_region", (45, 71), 0.3, 3, np.float32, [(1, 3)], 7),
    ("i32_1d_p050", (257,), 0.5, 4, np.int32, [1, 2], 0),
    ("u16_3d_p025_bg9", (5, 33, 33), 0.25, 5, np.uint16, [3, (1,)], 9),
]


def golden_mask(name: str):
    _, shape, density, seed, dtype, lr, bg = next(c for c in GOLDEN_MASKS if c[0] == name)
    seg = random_mask_case(shape, density, seed, dtype)
    return seg, lr, bg
