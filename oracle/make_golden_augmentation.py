"""Writes tests/golden/augmentation_cases.npz: three seeded augmentation cases run through the restatement
(oracle/augmentation_oracle.py) with noise off (the noise field comes from the device's Philox generator, and is
tested on its own).  Per case: the target (`{name}_target`, int8) and every 8th pixel of the data (`{name}_data`);
the inputs and decisions are rebuilt from seeds by `cases()`.

    python -m oracle.make_golden_augmentation
"""
import os

import numpy as np

from . import augmentation_oracle as AO

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                   "augmentation_cases.npz")


def cases() -> dict:
    """name -> (DeviceTrainingAugmentation, data, seg, params, noise seed)."""
    from dinounet_b200.augmentation import DeviceTrainingAugmentation
    out = {}
    specs = {   # name: (patch, B, C, in shape, pad, seed, augmentation kwargs)
        "hippocampus_2ch": ((40, 56), 3, 2, (51, 67), 3, 0, {"use_mask_for_norm": [True, False]}),
        "ct_602_to_512": ((512, 512), 1, 1, (602, 602), 45, 1, {}),
        "regions_ignore": ((44, 36), 2, 1, (53, 45), 3, 2, {"regions": [(1, 2), 2], "ignore_label": 3}),
    }
    for name, (patch, B, C, shape, pad, seed, kw) in specs.items():
        aug = DeviceTrainingAugmentation(patch, seed=seed, **kw)
        data, seg = AO.ct_like(B, C, *shape, pad, seed, labels=4 if "regions" in kw else 3)
        if "regions" in kw:
            seg[:, :, 10:14] = kw["ignore_label"]
        params = aug.sample(B, C)
        while not params.spatial.any():   # every case has a rotated or scaled sample
            params = aug.sample(B, C)
        params.noise[:] = False
        out[name] = (aug, data, seg, params, 0)
    return out


def golden_arrays() -> dict:
    arrays = {}
    for name, (aug, data, seg, params, seed) in cases().items():
        noise = np.zeros((data.shape[0], data.shape[1], *aug.patch_size))
        d, t = AO.augment(data, seg, params, noise, aug.patch_size, aug.use_mask_for_norm, aug.regions,
                          aug.ignore_label)
        arrays[f"{name}_target"] = t.astype(np.int8)
        arrays[f"{name}_data"] = d[:, :, ::8, ::8].copy()
    return arrays


if __name__ == "__main__":
    np.savez_compressed(OUT, **golden_arrays())
    print(OUT, os.path.getsize(OUT), "bytes")
