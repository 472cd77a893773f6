"""Writes tests/golden/postprocessing_cases.npz: the seeded label volumes of oracle/postprocessing_oracle.GOLDEN_MASKS
with the oracle's `remove_all_but_largest_component_from_segmentation` output (`{name}_seg`, `{name}_out`), and per
folder scenario the accepted kwargs (`{name}_accepted`, their repr), the final predictions (`{name}_final{i}`) and the
final foreground mean Dice (`{name}_fg_dice`).

    python -m oracle.make_golden_postprocessing
"""
import os

import numpy as np

from . import postprocessing_oracle as PO

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                   "postprocessing_cases.npz")


def golden_arrays() -> dict:
    arrays = {}
    for name, *_ in PO.GOLDEN_MASKS:
        seg, lr, bg = PO.golden_mask(name)
        arrays[f"{name}_seg"] = seg
        arrays[f"{name}_out"] = PO.remove_all_but_largest_component_from_segmentation(seg, lr, bg)
    for name in PO.SCENARIOS:
        accepted, final, _, final_summary = PO.run_scenario(name)
        arrays[f"{name}_accepted"] = np.array(repr(accepted))
        for i, f in enumerate(final):
            arrays[f"{name}_final{i}"] = f
        arrays[f"{name}_fg_dice"] = np.float64(final_summary["foreground_mean"]["Dice"])
    return arrays


if __name__ == "__main__":
    np.savez_compressed(OUT, **golden_arrays())
    print(OUT, os.path.getsize(OUT), "bytes")
