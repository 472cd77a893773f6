"""Writes tests/golden/evaluation_cases.npz: the seeded segmentation pairs of oracle/evaluation_oracle.GOLDEN_CASES with
their expected metrics (the oracle's `compute_metrics_arrays`, one row of METRIC_KEYS per label or region, NaN kept) and
surface-distance arrays (`{name}_sd{i}_pred_ref`, `{name}_sd{i}_ref_pred`).

    python -m oracle.make_golden_evaluation
"""
import os

import numpy as np

from . import evaluation_oracle as EO

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                   "evaluation_cases.npz")


def golden_arrays() -> dict:
    arrays = {}
    for name, _, spacing, regions, ignore, _, _ in EO.GOLDEN_CASES:
        ref, pred = EO.make_case(name)
        arrays[f"{name}_ref"], arrays[f"{name}_pred"] = ref, pred
        metrics = EO.compute_metrics_arrays(ref, pred, regions, ignore, spacing)
        arrays[f"{name}_metrics"] = np.array([[float(metrics[r][k]) for k in EO.METRIC_KEYS] for r in regions])
        for i, r in enumerate(regions):
            a, b = EO.pair_distances(ref, pred, r, spacing)
            arrays[f"{name}_sd{i}_pred_ref"], arrays[f"{name}_sd{i}_ref_pred"] = a, b
    return arrays


if __name__ == "__main__":
    np.savez_compressed(OUT, **golden_arrays())
    print(OUT, os.path.getsize(OUT), "bytes")
