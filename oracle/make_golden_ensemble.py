"""Writes tests/golden/ensemble_cases.npz: the reference's own `merge_files` (dinounet/ensembling/ensemble.py) with
its `LabelManager` on the seeded members of `ensemble_oracle.GOLDEN_CASES` (2 to 4 members, fp32 and fp16; label maps
with 2 and 4 classes and 3 overlapping regions; ties, near-ties, region averages around 1.5 * 2^-24, all-zero voxels).
Stores the members, the averaged probabilities and the segmentation the reference wrote.

    python oracle/make_golden_ensemble.py
"""
import os
import pickle
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ensemble_oracle as EN  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ensemble_cases.npz")


class NpyWriter:
    def write_seg(self, seg, path, properties):
        np.save(path, seg)


def label_dict(C, regions):
    if regions:
        return {"background": 0, "whole": [1, 2, 3], "core": [2, 3], "enh": [3]}
    return {"background": 0, **{f"c{i}": i for i in range(1, C)}}


def run_reference(ensemble, LabelManager, case, members, tmp):
    name, C, regions, _, _ = case
    files = []
    for k, m in enumerate(members):
        f = os.path.join(tmp, f"{name}_m{k}.npz")
        np.savez_compressed(f, probabilities=m)
        with open(f[:-4] + ".pkl", "wb") as fh:
            pickle.dump({"member": k}, fh)
        files.append(f)
    lm = LabelManager(label_dict(C, regions), list(EN.REGION_ORDER) if regions else None)
    out = os.path.join(tmp, f"{name}_out")
    ensemble.merge_files(files, out, ".npy", NpyWriter(), lm, True)
    return np.load(out + ".npz")["probabilities"], np.load(out + ".npy")


def main():
    ensemble, LabelManager = EN.load_reference_ensemble_module()
    arrays = {}
    with tempfile.TemporaryDirectory() as tmp:
        for seed, case in enumerate(EN.GOLDEN_CASES):
            name = case[0]
            members = EN.golden_members(case, seed)
            avg, seg = run_reference(ensemble, LabelManager, case, members, tmp)
            for k, m in enumerate(members):
                arrays[f"{name}_m{k}"] = m
            arrays[f"{name}_avg"] = avg
            arrays[f"{name}_seg"] = seg
    np.savez_compressed(OUT, **arrays)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
