"""Writes tests/golden/export_cases.npz: the reference's export chain (oracle/export_oracle.py with scipy's float64
zoom as the resampler) on the cases of `GOLDEN_CASES`: label maps with 2 and 4 classes and regions with 3 overlapping
classes; up-, down-, mixed and identity resampling; non-trivial boxes and transposes; with and without probabilities.

    python oracle/make_golden_export.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import export_oracle as EO  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "export_cases.npz")


def main():
    arrays = {}
    for seed, case in enumerate(EO.GOLDEN_CASES):
        name, C, regions, order, shape, _, _, _, tb, save_probs = case
        logits = EO.golden_logits(C, shape, seed)
        props = EO.golden_properties(case)
        r, seg, probs = EO.convert(logits, props, tb, 3 if regions else C - 1, regions, order, save_probs, resampler="scipy")
        arrays[f"{name}_logits"] = logits.numpy()
        arrays[f"{name}_resampled"] = r.numpy()
        arrays[f"{name}_seg"] = seg
        if probs is not None:
            arrays[f"{name}_probs"] = probs
    np.savez_compressed(OUT, **arrays)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
