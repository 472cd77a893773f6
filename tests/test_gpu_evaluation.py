"""Device evaluation on the GPU (csrc/evaluation.cu, dinounet_b200/evaluation.py) against numpy / scipy, the golden
cases (tests/golden/evaluation_cases.npz) and the in-tree oracle (oracle/evaluation_oracle.py)."""
import ctypes
import os

import numpy as np
import pytest
import torch
from scipy import ndimage as ndi

from dinounet_b200 import evaluation as EV
from dinounet_b200 import lib as L
from oracle import evaluation_oracle as EO

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "evaluation_cases.npz"))
DTYPES = [np.uint8, np.int8, np.int16, np.uint16, np.int32, np.float32]
INTEGER_SPACINGS = [(1.0, 1.0, 1.0), (3.0, 1.0, 1.0), (999.0, 1.0, 1.0)]


def _masks(ref, pred, labels, ignore=None):
    """b2u_eval_masks on (1, *spatial) arrays: (border_ref, border_pred, counts)."""
    ndim = ref.ndim - 1
    Z, Y, X = (1,) * (3 - ndim) + ref.shape[1:]
    r, p = torch.from_numpy(ref).cuda(), torch.from_numpy(pred).cuda()
    br = torch.empty(ref.size, dtype=torch.uint8, device="cuda")
    bp = torch.empty_like(br)
    counts = torch.empty(6, dtype=torch.int64, device="cuda")
    lab = (ctypes.c_int64 * len(labels))(*labels)
    L.check(L.load().b2u_eval_masks(r.data_ptr(), EV.DTYPE_CODES[r.dtype], p.data_ptr(), EV.DTYPE_CODES[p.dtype], ndim,
                                    Z, Y, X, lab, len(labels), int(ignore is not None), ignore or 0, br.data_ptr(),
                                    bp.data_ptr(), counts.data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return br.cpu().numpy().reshape(ref.shape[1:]), bp.cpu().numpy().reshape(ref.shape[1:]), counts.cpu().numpy()


def _edt(border, spacing):
    Z, Y, X = border.shape
    b = torch.from_numpy(border.astype(np.uint8)).cuda()
    dt, tmp = (torch.empty(border.size, dtype=torch.float64, device="cuda") for _ in range(2))
    scratch = torch.empty(border.size, dtype=torch.int32, device="cuda")
    L.check(L.load().b2u_eval_edt(b.data_ptr(), Z, Y, X, *spacing, tmp.data_ptr(), scratch.data_ptr(), dt.data_ptr(),
                                  torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return dt.cpu().numpy().reshape(border.shape)


def _border(m):
    return m ^ ndi.binary_erosion(m, ndi.generate_binary_structure(m.ndim, 1))


# ---- counts and borders


@pytest.mark.parametrize("dt_ref", DTYPES)
def test_counts_exact_over_dtype_pairs(dt_ref):
    rng = np.random.default_rng(3)
    base_ref = rng.integers(0, 5, (1, 9, 17, 23))
    base_pred = rng.integers(0, 5, (1, 9, 17, 23))
    for dt_pred in DTYPES:
        ref, pred = base_ref.astype(dt_ref), base_pred.astype(dt_pred)
        for labels, ignore in [([1], None), ([2, 3], 4), ([4], 4), ([0, 1, 2, 3], 1)]:
            r = labels[0] if len(labels) == 1 else tuple(labels)
            mr, mp = EO.region_or_label_to_mask(ref, r), EO.region_or_label_to_mask(pred, r)
            use = np.ones_like(mr) if ignore is None else ref != ignore
            want = [np.sum(mr & mp & use), np.sum(~mr & mp & use), np.sum(mr & ~mp & use), np.sum(~mr & ~mp & use),
                    mr.sum(), mp.sum()]
            br, bp, counts = _masks(ref, pred, labels, ignore)
            assert counts.tolist() == [int(w) for w in want], (dt_ref, dt_pred, labels, ignore)
            assert np.array_equal(br.astype(bool), _border(mr[0])) and np.array_equal(bp.astype(bool), _border(mp[0]))


def test_float_labels_compare_as_numpy():
    ref = np.array([[[[1.0, 1.5, 2.0, 16777216.0, -1.0]]]], np.float32)
    for labels in ([1], [2], [16777217], [-1], [255]):
        _, _, counts = _masks(ref, ref, labels)
        assert counts[4] == np.sum(ref == labels[0]), labels
    u = np.array([[[[255, 44, 1]]]], np.uint8)
    for labels in ([-1], [300], [255]):
        assert _masks(u, u, labels)[2][4] == np.sum(u == labels[0])


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 6, 7), (5, 1, 9), (1, 1, 13), (4, 6, 1), (7, 9, 11)])
def test_borders_match_scipy(shape):
    rng = np.random.default_rng(sum(shape))
    seg = (rng.random(shape) < 0.7).astype(np.uint8)[None]
    br, _, _ = _masks(seg, seg, [1])
    assert np.array_equal(br.astype(bool), _border(seg[0].astype(bool)))
    # rank 2: the mask (y, x) is eroded in-plane only
    seg2 = seg[:, 0]
    br2, _, _ = _masks(seg2, seg2, [1])
    assert np.array_equal(br2.astype(bool).reshape(seg2.shape[1:]), _border(seg2[0].astype(bool)))


# ---- the distance transform


def _edt_cases():
    rng = np.random.default_rng(11)
    yield "random", rng.random((9, 13, 17)) < 0.05
    yield "odd", rng.random((7, 11, 31)) < 0.01
    single = np.zeros((6, 8, 10), bool)
    single[2, 5, 7] = True
    yield "single", single
    lines = np.zeros((1, 1, 1), bool)
    lines[0, 0, 0] = True
    yield "one_voxel", lines
    long_x = np.zeros((2, 3, 1500), bool)
    long_x[0, 1, 3] = long_x[1, 2, 1400] = True
    yield "long_x", long_x
    long_z = np.zeros((1100, 2, 3), bool)
    long_z[5, 0, 0] = long_z[1000, 1, 2] = True
    yield "long_z", long_z
    long_y = np.zeros((2, 1300, 2), bool)
    long_y[1, 7, 1] = True
    yield "long_y", long_y
    yield "line1", rng.random((1, 40, 1)) < 0.2


@pytest.mark.parametrize("name,border", list(_edt_cases()), ids=[c[0] for c in _edt_cases()])
def test_edt_matches_scipy(name, border):
    if not border.any():
        border.flat[0] = True
    for spacing in INTEGER_SPACINGS + [(2.5, 0.7, 0.7), (0.3, 1.7, 1.1)]:
        want = ndi.distance_transform_edt(~border, sampling=spacing)
        got = _edt(border, spacing)
        if spacing in INTEGER_SPACINGS:
            assert np.array_equal(got, want), (name, spacing)
        else:
            np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)


# ---- end to end


def _check(got, want, integer):
    assert list(got) == list(want)
    for r in want:
        assert list(got[r]) == list(want[r])
        for k, w in want[r].items():
            g = got[r][k]
            assert type(g) is type(w), (r, k)
            if np.isnan(w):
                assert np.isnan(g), (r, k)
            elif k in ("HD95", "ASD") and not integer:
                assert abs(g - w) <= 1e-12 * abs(w), (r, k, g, w)
            else:
                assert g == w, (r, k, g, w)


@pytest.mark.parametrize("case", EO.GOLDEN_CASES, ids=[c[0] for c in EO.GOLDEN_CASES])
def test_compute_metrics_arrays_golden_and_oracle(case):
    name, _, spacing, regions, ignore, _, _ = case
    ref, pred = GOLDEN[f"{name}_ref"], GOLDEN[f"{name}_pred"]
    integer = all(float(s).is_integer() for s in spacing)
    got = EV.compute_metrics_arrays(ref, pred, regions, ignore, spacing)
    _check(got, EO.compute_metrics_arrays(ref, pred, regions, ignore, spacing), integer)
    rows = np.array([[float(got[r][k]) for k in EV.METRIC_KEYS] for r in regions])
    want = GOLDEN[f"{name}_metrics"]
    if integer:
        assert np.array_equal(rows, want, equal_nan=True)
    else:
        np.testing.assert_allclose(rows, want, rtol=1e-12, atol=0)
    again = EV.compute_metrics_arrays(torch.from_numpy(ref).cuda(), torch.from_numpy(pred).cuda(), regions, ignore,
                                      spacing)
    assert repr(again) == repr(got)


def test_ct_like_case_against_oracle():
    """A larger anisotropic case with every label touching the volume's faces, label maps and a region."""
    rng = np.random.default_rng(5)
    shape = (24, 96, 80)
    ref = EO._blobs(rng, shape, [1, 2, 3], count=3)
    ref[:, :, :4] = 1
    pred = EO._perturb(rng, ref, [1, 2, 3])
    for spacing in [(3.0, 1.0, 1.0), (2.5, 0.78, 0.78)]:
        regions = [1, 2, 3, (2, 3)]
        got = EV.compute_metrics_arrays(ref[None], pred[None].astype(np.float32), regions, 0, spacing)
        _check(got, EO.compute_metrics_arrays(ref[None], pred[None].astype(np.float32), regions, 0, spacing),
               spacing[1] == 1.0)


def test_folder(tmp_path):
    class NpyReader:
        def read_seg(self, path):
            return np.load(path), {"spacing": (3.0, 1.0, 1.0)}

    (tmp_path / "gt").mkdir()
    (tmp_path / "pred").mkdir()
    for name, *_ in EO.GOLDEN_CASES[:3]:
        np.save(tmp_path / "gt" / f"{name}.npy", GOLDEN[f"{name}_ref"].astype(np.float32))
        np.save(tmp_path / "pred" / f"{name}.npy", GOLDEN[f"{name}_pred"].astype(np.uint8))
    got = EV.compute_metrics_on_folder(str(tmp_path / "gt"), str(tmp_path / "pred"), str(tmp_path / "s.json"),
                                       NpyReader(), ".npy", [1, 2], None, 2)
    real = EV.compute_metrics_arrays
    try:
        EV.compute_metrics_arrays = EO.compute_metrics_arrays
        want = EV.compute_metrics_on_folder(str(tmp_path / "gt"), str(tmp_path / "pred"), str(tmp_path / "o.json"),
                                            NpyReader(), ".npy", [1, 2], None, 2)
    finally:
        EV.compute_metrics_arrays = real
    assert (tmp_path / "s.json").read_text() == (tmp_path / "o.json").read_text()
    assert repr(got) == repr(want)
