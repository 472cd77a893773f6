"""CPU restatement of nnU-Net's 2-D data loader (`nnUNetDataLoader2D.generate_train_batch`, data_loader_2d.py:7-91,
`nnUNetDataLoaderBase.get_bbox`, base_data_loader.py:64-134, batchgenerators 0.25's infinite `get_indices`) on a
`np.random.RandomState`, and the validation transforms' target (nnUNetTrainer.py:778-805), for tests only.

`generate_train_batch` returns the reference's batch (data float32, seg int16, padded by np.pad with 0 and -1) and
every draw it made: the keys, and per sample the slice and the box.  tests/golden/dataloader_cases.npz pins it to the
reference's own loader (oracle/make_golden_dataloader.py).
"""
import numpy as np


def get_bbox(rng, data_shape, force_fg, class_locations, patch_size, need_to_pad, annotated_key, has_ignore,
             overwrite_class=None):
    need = np.array(need_to_pad).copy()
    dim = len(data_shape)
    for d in range(dim):
        if need[d] + data_shape[d] < patch_size[d]:
            need[d] = patch_size[d] - data_shape[d]
    lbs = [- need[i] // 2 for i in range(dim)]
    ubs = [data_shape[i] + need[i] // 2 + need[i] % 2 - patch_size[i] for i in range(dim)]
    if not force_fg and not has_ignore:
        return [rng.randint(lbs[i], ubs[i] + 1) for i in range(dim)]
    if not force_fg and has_ignore:
        selected = annotated_key
        if len(class_locations[selected]) == 0:
            print('Warning! No annotated pixels in image!')
            selected = None
    elif force_fg:
        assert class_locations is not None
        if overwrite_class is not None:
            assert overwrite_class in class_locations.keys()
        eligible = [i for i in class_locations.keys() if len(class_locations[i]) > 0]
        tmp = [i == annotated_key if isinstance(i, tuple) else False for i in eligible]
        if any(tmp) and len(eligible) > 1:
            eligible.pop(np.where(tmp)[0][0])
        if not eligible:
            selected = None
        elif overwrite_class is None or overwrite_class not in eligible:
            selected = eligible[rng.choice(len(eligible))]
        else:
            selected = overwrite_class
    else:
        raise RuntimeError('lol what!?')
    voxels = class_locations[selected] if selected is not None else None
    if voxels is not None and len(voxels) > 0:
        v = voxels[rng.choice(len(voxels))]
        return [max(lbs[i], v[i + 1] - patch_size[i] // 2) for i in range(dim)]
    return [rng.randint(lbs[i], ubs[i] + 1) for i in range(dim)]


def generate_train_batch(dataset, batch_size, patch_size, final_patch_size, all_labels, has_ignore, oversample, rng):
    """(batch {"data", "seg", "keys", "properties"}, draws [(slice, bbox_lbs)] per sample)."""
    keys = list(dataset.keys())
    annotated_key = tuple(all_labels)
    need_to_pad = (np.array(patch_size) - np.array(final_patch_size)).astype(int)
    selected_keys = rng.choice(keys, batch_size, replace=True, p=None)
    d0, s0, _ = dataset.load_case(keys[0])
    data_all = np.zeros((batch_size, d0.shape[0], *patch_size), dtype=np.float32)
    seg_all = np.zeros((batch_size, s0.shape[0], *patch_size), dtype=np.int16)
    props, draws = [], []
    for j, key in enumerate(selected_keys):
        force_fg = not j < round(batch_size * (1 - oversample))
        data, seg, p = dataset.load_case(key)
        props.append(p)
        if not force_fg:
            sel = annotated_key if has_ignore else None
        else:
            locs = p['class_locations']
            eligible = [i for i in locs.keys() if len(locs[i]) > 0]
            tmp = [i == annotated_key if isinstance(i, tuple) else False for i in eligible]
            if any(tmp) and len(eligible) > 1:
                eligible.pop(np.where(tmp)[0][0])
            sel = eligible[rng.choice(len(eligible))] if eligible else None
        sl = rng.choice(p['class_locations'][sel][:, 1]) if sel is not None else rng.choice(len(data[0]))
        data, seg = data[:, sl], seg[:, sl]
        cl = None
        if sel is not None:
            rows = p['class_locations'][sel]
            cl = {sel: rows[rows[:, 1] == sl][:, (0, 2, 3)]}
        shape = data.shape[1:]
        lbs = get_bbox(rng, shape, force_fg if sel is not None else None, cl, patch_size, need_to_pad, annotated_key,
                       has_ignore, overwrite_class=sel)
        ubs = [lbs[i] + patch_size[i] for i in range(2)]
        lo = [max(0, lbs[i]) for i in range(2)]
        hi = [min(shape[i], ubs[i]) for i in range(2)]
        pad = [(-min(0, lbs[i]), max(ubs[i] - shape[i], 0)) for i in range(2)]
        data_all[j] = np.pad(data[:, lo[0]:hi[0], lo[1]:hi[1]], ((0, 0), *pad), 'constant', constant_values=0)
        seg_all[j] = np.pad(seg[:, lo[0]:hi[0], lo[1]:hi[1]], ((0, 0), *pad), 'constant', constant_values=-1)
        draws.append((int(sl), [int(v) for v in lbs]))
    return {"data": data_all, "seg": seg_all, "keys": selected_keys, "properties": props}, draws


def val_target(seg, regions=None, ignore_label=None):
    """RemoveLabelTransform(-1, 0), ConvertSegmentationToRegionsTransform(regions (+ [ignore_label])) and
    NumpyToTensor(float): float32 [B, 1 or R, *patch]."""
    s = np.array(seg, copy=True)
    s[s == -1] = 0
    if regions is None:
        return s.astype(np.float32)
    regs = list(regions) + [ignore_label] if ignore_label is not None else list(regions)
    out = np.zeros((s.shape[0], len(regs), *s.shape[2:]), dtype=s.dtype)
    for b in range(s.shape[0]):
        for r, labels in enumerate(regs):
            for v in (labels if isinstance(labels, (list, tuple)) else (labels,)):
                out[b, r][s[b, 0] == v] = 1
    return out.astype(np.float32)


class ArrayDataset:
    """`keys()` / `load_case(key)` over in-memory (data, seg, properties) per key (nnUNetDataset's interface)."""

    def __init__(self, cases):
        self.cases = dict(cases)

    def keys(self):
        return list(self.cases.keys())

    def load_case(self, key):
        return self.cases[str(key)]


def ct_like_case(C, Z, X, Y, labels, seed, seg_dtype=np.int8, empty=False, ignore_label=None, regions=None):
    """A seeded preprocessed case: data float32 [C, Z, X, Y] (CT-like: labels times 80 plus noise, z-scored), seg
    [1, Z, X, Y] with -1 in a border of the crop, and class_locations as DefaultPreprocessor writes them: per class
    (or region, or the all-labels key with an ignore label) int64 rows (c, z, x, y), an empty list for a class absent."""
    rng = np.random.RandomState(seed)
    zz, yy, xx = np.meshgrid(np.linspace(-1, 1, Z), np.linspace(-1, 1, X), np.linspace(-1, 1, Y), indexing="ij")
    seg = np.zeros((Z, X, Y), np.int64)
    if not empty:
        for lab in labels:
            c = rng.uniform(-.5, .5, 3)
            r = np.sqrt(((zz - c[0]) * 0.3) ** 2 + ((yy - c[1]) * 1.3) ** 2 + (xx - c[2]) ** 2)
            seg[r < rng.uniform(0.25, 0.6)] = lab
    if ignore_label is not None and not empty:
        seg[:, :, :2] = ignore_label
    seg[:, :1, :] = -1
    data = np.stack([((seg * 80.0 - 500 + rng.normal(0, 40, seg.shape)) / 300.0 + c) for c in range(C)])
    data[:, seg < 0] = 0
    if regions is not None:
        classes = [tuple(r) if isinstance(r, (list, tuple)) else r for r in regions]
    else:
        classes = [lab for lab in labels]
    if ignore_label is not None:
        classes.append(tuple(lab for lab in [0] + list(labels)))
    locs = {}
    for c in classes:
        mask = np.isin(seg, c if isinstance(c, tuple) else [c])
        rows = np.argwhere(mask[None])
        if len(rows) == 0:
            locs[c] = []
            continue
        take = min(len(rows), max(10000 // len(classes), int(np.ceil(len(rows) * 0.01))))
        locs[c] = rows[np.sort(rng.choice(len(rows), take, replace=False))]
    return data.astype(np.float32), seg[None].astype(seg_dtype), {"class_locations": locs}
