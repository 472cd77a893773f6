"""nnU-Net's 2-D data loader with the batch assembled on the device (reference: `nnUNetDataLoader2D`,
data_loader_2d.py:7-91, with `nnUNetDataLoaderBase.get_bbox`, base_data_loader.py:64-134, and batchgenerators 0.25's
`DataLoader.get_indices`), for the Dino U-Net trainer's `device_dataloading` route.

    dl = DeviceDataLoader2D(dataset, batch_size, initial_patch_size, patch_size, label_manager, 0.33, seed=0)
    batch = next(dl)   # {"data": fp32 [B, C, *patch] CUDA, "target": int16 [B, 1, *patch] CUDA, "properties", "keys"}
    dl.close()

One read-ahead thread makes every random draw of the reference, in its order, on a `np.random.RandomState`: the keys
(`choice(keys, B, replace=True)`), then per sample the class (oversampling the last `round(B * (1 - p))` samples onward,
Python's round), the slice, and the voxel or the `randint` per axis of the box.  With the reference's global `np.random`
seeded to s, `RandomState(s)` gives the same keys, slices and boxes, and the reference's errors (the ValueError of
`choice` on an empty row set, the TypeError of an empty class stored as a list) are raised where it raises them.  The
thread loads each case with `load_case(key)`, copies only the part of each box inside its slice (`valid_bbox_lbs/ubs`)
into one of three pinned slots (data float32, seg as stored, and a descriptor per sample) and makes no CUDA call.

`next()` runs on the caller's thread: one non-blocking host-to-device copy of the slot and one `b2u_dl_crop` launch
(csrc/dataloading.cu) on the current stream, which pads with 0 (data) and -1 (seg) as `np.pad` does.  A slot returns
to the thread only after the event recorded behind that launch has completed.  mode="val" writes the target of the
reference's validation transforms (nnUNetTrainer.py:778-805): -1 -> 0, then the label map or the region planes, float32.
"""
from __future__ import annotations

import queue
import threading
import time
from typing import NamedTuple, Optional

import numpy as np
import torch

from . import lib as L
from .augmentation import _region_table

DESC = 8           # int64 per sample: data offset, seg offset, y0, x0, h, w, seg bytes, 0 (B2U_DL_DESC)
SLOTS = 3          # pinned slots: one being filled, at most two queued
QUEUE_DEPTH = 2
_ALIGN = 16


class Sample(NamedTuple):
    """One sample's draws: the case, the slice and the box [lbs, ubs) in the slice's coordinates."""
    key: str
    data: np.ndarray
    seg: np.ndarray
    properties: dict
    slice: int
    bbox_lbs: tuple
    bbox_ubs: tuple


def _align(n: int) -> int:
    return (n + _ALIGN - 1) // _ALIGN * _ALIGN


class DeviceDataLoader2D:
    """Infinite iterator over 2-D training (mode="train") or validation (mode="val") batches on a CUDA device (module
    docstring).  `data` needs only `keys()` and `load_case(key) -> (data [C, Z, X, Y] float32, seg [1, Z, X, Y] int8 or
    int16, properties)`."""

    def __init__(self, data, batch_size, patch_size, final_patch_size, label_manager, oversample_foreground_percent=0.0,
                 sampling_probabilities=None, pad_sides=None, probabilistic_oversampling=False, *, mode="train",
                 regions=None, ignore_label=None, seed: Optional[int] = None, device=None):
        if sampling_probabilities is not None:
            raise NotImplementedError("the device loader draws keys uniformly; sampling_probabilities is not implemented")
        if pad_sides is not None:
            raise NotImplementedError("pad_sides is not implemented by the device loader")
        if probabilistic_oversampling:
            raise NotImplementedError("probabilistic_oversampling is not implemented by the device loader")
        if mode not in ("train", "val"):
            raise ValueError(f"mode must be 'train' or 'val', got {mode!r}")
        if mode == "train" and regions is not None:
            raise ValueError("regions are converted in val mode only; train batches keep the label map")
        self.patch_size = tuple(int(v) for v in patch_size)
        self.final_patch_size = tuple(int(v) for v in final_patch_size)
        if len(self.patch_size) != 2 or len(self.final_patch_size) != 2 or min(self.patch_size) < 1:
            raise ValueError(f"the device loader is 2-D only; got patch_size {tuple(patch_size)} and final_patch_size "
                             f"{tuple(final_patch_size)}")
        self.batch_size = int(batch_size)
        if self.batch_size < 1:
            raise ValueError(f"batch_size must be >= 1, got {batch_size}")
        self.mode = mode
        self.oversample_foreground_percent = oversample_foreground_percent
        self.need_to_pad = (np.array(self.patch_size) - np.array(self.final_patch_size)).astype(int)
        self._data = data
        self.indices = list(data.keys())
        if not self.indices:
            raise ValueError("the dataset has no cases")
        self.annotated_classes_key = tuple(label_manager.all_labels)
        self.has_ignore = label_manager.has_ignore_label
        self.regions = None if regions is None else list(regions)
        self._R, self._table = (0, None) if regions is None else _region_table(regions, ignore_label)
        d0, s0, _ = data.load_case(self.indices[0])   # determine_shapes (base_data_loader.py:55-62)
        self._check_case(self.indices[0], d0, s0)
        self.num_channels = int(d0.shape[0])
        if self.batch_size * self.num_channels > 65535:
            raise ValueError(f"B={self.batch_size}, C={self.num_channels}: need B*C <= 65535")
        self.rng = np.random.RandomState(seed)
        self.device = None if device is None else torch.device(device)
        H, W = self.patch_size
        B, C = self.batch_size, self.num_channels
        self.slot_bytes = _align(B * DESC * 8) + B * (_align(C * H * W * 4) + _align(H * W * 2))
        self.stats = {"batches": 0, "host_s": 0.0, "wait_s": 0.0, "waits": 0}
        self._thread = None
        self._stop = threading.Event()
        self._free: queue.Queue = queue.Queue()
        self._ready: queue.Queue = queue.Queue(maxsize=QUEUE_DEPTH)
        self._pending = []
        self._failed = False

    # ---- validation of a case ---------------------------------------------------------------------------------------
    def _check_case(self, key, data, seg):
        if data.ndim != 4 or seg.ndim != 4 or tuple(seg.shape[1:]) != tuple(data.shape[1:]):
            raise ValueError(f"case {key}: data [C, Z, X, Y] and seg [1, Z, X, Y] expected, got {tuple(data.shape)} and "
                             f"{tuple(seg.shape)}")
        if seg.shape[0] != 1:
            raise ValueError(f"case {key}: the seg has {seg.shape[0]} channels; the device loader takes one (no "
                             "segmentation from a previous stage)")
        if data.dtype != np.float32:
            raise TypeError(f"case {key}: data must be float32, got {data.dtype}")
        if seg.dtype not in (np.int8, np.int16):
            raise TypeError(f"case {key}: seg must be int8 or int16 as the preprocessor stores it, got {seg.dtype}")
        if hasattr(self, "num_channels") and data.shape[0] != self.num_channels:
            raise ValueError(f"case {key}: {data.shape[0]} channels, the first case has {self.num_channels}")

    # ---- the reference's draws ------------------------------------------------------------------------------------
    def _bbox(self, data_shape, force_fg, class_locations, overwrite_class=None):
        """nnUNetDataLoaderBase.get_bbox on self.rng."""
        rng = self.rng
        need_to_pad = self.need_to_pad.copy()
        dim = len(data_shape)
        for d in range(dim):
            if need_to_pad[d] + data_shape[d] < self.patch_size[d]:
                need_to_pad[d] = self.patch_size[d] - data_shape[d]
        lbs = [- need_to_pad[i] // 2 for i in range(dim)]
        ubs = [data_shape[i] + need_to_pad[i] // 2 + need_to_pad[i] % 2 - self.patch_size[i] for i in range(dim)]
        if not force_fg and not self.has_ignore:
            bbox_lbs = [rng.randint(lbs[i], ubs[i] + 1) for i in range(dim)]
        else:
            if not force_fg and self.has_ignore:
                selected_class = self.annotated_classes_key
                if len(class_locations[selected_class]) == 0:
                    print('Warning! No annotated pixels in image!')
                    selected_class = None
            elif force_fg:
                assert class_locations is not None, 'if force_fg is set class_locations cannot be None'
                if overwrite_class is not None:
                    assert overwrite_class in class_locations.keys(), 'desired class ("overwrite_class") does not ' \
                                                                      'have class_locations (missing key)'
                eligible = [i for i in class_locations.keys() if len(class_locations[i]) > 0]
                tmp = [i == self.annotated_classes_key if isinstance(i, tuple) else False for i in eligible]
                if any(tmp) and len(eligible) > 1:
                    eligible.pop(np.where(tmp)[0][0])
                if len(eligible) == 0:
                    selected_class = None
                else:
                    selected_class = eligible[rng.choice(len(eligible))] if \
                        (overwrite_class is None or (overwrite_class not in eligible)) else overwrite_class
            else:
                raise RuntimeError('lol what!?')
            voxels = class_locations[selected_class] if selected_class is not None else None
            if voxels is not None and len(voxels) > 0:
                selected_voxel = voxels[rng.choice(len(voxels))]
                bbox_lbs = [max(lbs[i], selected_voxel[i + 1] - self.patch_size[i] // 2) for i in range(dim)]
            else:
                bbox_lbs = [rng.randint(lbs[i], ubs[i] + 1) for i in range(dim)]
        bbox_ubs = [bbox_lbs[i] + self.patch_size[i] for i in range(dim)]
        return tuple(int(v) for v in bbox_lbs), tuple(int(v) for v in bbox_ubs)

    def draw(self):
        """One batch's draws in the reference's order (generate_train_batch): (keys, [Sample])."""
        rng = self.rng
        keys = rng.choice(self.indices, self.batch_size, replace=True, p=None)
        samples = []
        for j, key in enumerate(keys):
            force_fg = not j < round(self.batch_size * (1 - self.oversample_foreground_percent))
            data, seg, properties = self._data.load_case(key)
            self._check_case(key, data, seg)
            if not force_fg:
                selected = self.annotated_classes_key if self.has_ignore else None
            else:
                locs = properties['class_locations']
                eligible = [i for i in locs.keys() if len(locs[i]) > 0]
                tmp = [i == self.annotated_classes_key if isinstance(i, tuple) else False for i in eligible]
                if any(tmp) and len(eligible) > 1:
                    eligible.pop(np.where(tmp)[0][0])
                selected = eligible[rng.choice(len(eligible))] if len(eligible) > 0 else None
            if selected is not None:
                selected_slice = rng.choice(properties['class_locations'][selected][:, 1])
            else:
                selected_slice = rng.choice(len(data[0]))
            rows = properties['class_locations'][selected] if selected is not None else None
            class_locations = {selected: rows[rows[:, 1] == selected_slice][:, (0, 2, 3)]} \
                if selected is not None else None
            lbs, ubs = self._bbox(data.shape[2:], force_fg if selected is not None else None, class_locations,
                                  overwrite_class=selected)
            samples.append(Sample(key, data, seg, properties, int(selected_slice), lbs, ubs))
        return keys, samples

    # ---- staging (read-ahead thread) ------------------------------------------------------------------------------
    def _stage(self, buf: np.ndarray, samples) -> int:
        """Writes the descriptor table and every sample's valid box into `buf` (uint8); returns the bytes used."""
        C = self.num_channels
        desc = buf[:len(samples) * DESC * 8].view(np.int64).reshape(len(samples), DESC)
        off = _align(len(samples) * DESC * 8)
        for b, s in enumerate(samples):
            shape = s.data.shape[2:]
            lo = [max(0, s.bbox_lbs[i]) for i in range(2)]
            hi = [min(shape[i], s.bbox_ubs[i]) for i in range(2)]
            h, w = max(0, hi[0] - lo[0]), max(0, hi[1] - lo[1])
            nd = C * h * w * 4
            np.copyto(buf[off:off + nd].view(np.float32).reshape(C, h, w),
                      s.data[:, s.slice, lo[0]:lo[0] + h, lo[1]:lo[1] + w])
            es = s.seg.dtype.itemsize
            ns = h * w * es
            np.copyto(buf[off + _align(nd):off + _align(nd) + ns].view(s.seg.dtype).reshape(h, w),
                      s.seg[0, s.slice, lo[0]:lo[0] + h, lo[1]:lo[1] + w])
            desc[b] = (off, off + _align(nd), -min(0, s.bbox_lbs[0]), -min(0, s.bbox_lbs[1]), h, w, es, 0)
            off += _align(nd) + _align(ns)
        return off

    def _get(self, q: queue.Queue):
        while not self._stop.is_set():
            try:
                return q.get(timeout=0.05)
            except queue.Empty:
                pass
        return None

    def _put(self, q: queue.Queue, item) -> bool:
        while not self._stop.is_set():
            try:
                q.put(item, timeout=0.05)
                return True
            except queue.Full:
                pass
        return False

    def _run(self):
        try:
            while not self._stop.is_set():
                t0 = time.perf_counter()
                keys, samples = self.draw()
                t1 = time.perf_counter()
                slot = self._get(self._free)
                if slot is None:
                    return
                t2 = time.perf_counter()
                nbytes = self._stage(self._host[slot], samples)
                self.stats["host_s"] += (t1 - t0) + (time.perf_counter() - t2)
                if not self._put(self._ready, (slot, nbytes, keys, [s.properties for s in samples])):
                    return
        except BaseException as e:  # noqa: BLE001 - handed to the consumer, which raises it
            self._put(self._ready, e)

    # ---- consumer side --------------------------------------------------------------------------------------------
    def _alloc(self):
        """The pinned host slots (as uint8 numpy views) and their device copies."""
        pinned = [torch.empty(self.slot_bytes, dtype=torch.uint8, pin_memory=True) for _ in range(SLOTS)]
        dev = [torch.empty(self.slot_bytes, dtype=torch.uint8, device=self.device) for _ in range(SLOTS)]
        return pinned, [p.numpy() for p in pinned], dev

    def _start(self):
        if self._thread is not None:
            return
        if self.device is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self._pinned, self._host, self._dev = self._alloc()
        if self._table is not None:
            self._table_dev = torch.from_numpy(self._table).to(self.device)
        for s in range(SLOTS):
            self._free.put(s)
        self._thread = threading.Thread(target=self._run, name="DeviceDataLoader2D", daemon=True)
        self._thread.start()

    def _release(self):
        """Returns to the thread every slot whose copy and kernel have completed; when all slots are in flight, waits
        for the oldest (the thread could not stage the next batch otherwise)."""
        keep = []
        for ev, slot in self._pending:
            if ev.query():
                self._free.put(slot)
            else:
                keep.append((ev, slot))
        self._pending = keep
        if len(self._pending) == SLOTS:
            ev, slot = self._pending.pop(0)
            ev.synchronize()
            self._free.put(slot)

    def _launch(self, slot: int, nbytes: int):
        """H2D copy of the slot and the crop kernel on the current stream; returns (data, target, event)."""
        B, C = self.batch_size, self.num_channels
        H, W = self.patch_size
        dev = self.device
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev)
            staged = self._dev[slot]
            staged[:nbytes].copy_(self._pinned[slot][:nbytes], non_blocking=True)
            data = torch.empty((B, C, H, W), dtype=torch.float32, device=dev)
            if self.mode == "train":
                target = torch.empty((B, 1, H, W), dtype=torch.int16, device=dev)
            else:
                target = torch.empty((B, self._R or 1, H, W), dtype=torch.float32, device=dev)
            table = self._table_dev.data_ptr() if self._table is not None else None
            L.check(L.load().b2u_dl_crop(staged.data_ptr(), staged.data_ptr(), B, C, H, W, int(self.mode == "val"),
                                         table, self._R, data.data_ptr(), target.data_ptr(), stream.cuda_stream),
                    "b2u_dl_crop")
            ev = torch.cuda.Event()
            ev.record(stream)
        return data, target, ev

    def __iter__(self):
        return self

    def __next__(self):
        if self._failed:
            raise RuntimeError("the loader's read-ahead thread stopped after an error")
        if self._stop.is_set():
            raise RuntimeError("the loader is closed")
        self._start()
        self._release()
        t0 = time.perf_counter()
        try:
            item = self._ready.get_nowait()
        except queue.Empty:
            self.stats["waits"] += 1
            item = self._get(self._ready)
        self.stats["wait_s"] += time.perf_counter() - t0
        if isinstance(item, BaseException):
            self._failed = True
            raise item
        slot, nbytes, keys, properties = item
        data, target, ev = self._launch(slot, nbytes)
        self._pending.append((ev, slot))
        self.stats["batches"] += 1
        return {"data": data, "target": target, "properties": properties, "keys": keys}

    def close(self):
        """Stops and joins the read-ahead thread (no process is ever started)."""
        self._stop.set()
        if self._thread is not None:
            self._thread.join()
        for ev, _ in self._pending:
            ev.synchronize()
        self._pending = []
