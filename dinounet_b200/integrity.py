"""Dataset integrity check on the device (reference: experiment_planning/verify_dataset_integrity.py), drop-ins for
the reference's own functions:

    verify_dataset_integrity(folder, num_processes)
    extract_fingerprint_dataset(dataset_id, fingerprint_extractor_class, num_processes, check_dataset_integrity,
                                clean, verbose)
    extract_fingerprints(dataset_ids, fingerprint_extractor_class_name, num_processes, check_dataset_integrity,
                         clean, verbose)

`verify_dataset_integrity` prints the reference's text and raises its exceptions.  The host part (dataset.json, its
keys, the files, numTraining, the label manager's consecutive labels, the reader from the first image; per case the
shapes, spacings, channel count and the nibabel / SimpleITK geometry warnings) follows the reference line for line.
The two array checks are one device read per case (`b2u_vi_scan`): NaN in the images, NaN in the seg, and the seg
voxels outside the expected labels, which the reference asserts are consecutive, so membership is a range test.  Only
a failing case sorts its seg's distinct values on the device for the reference's `Found: [...]` line.  Cases are read
ahead on `num_processes` threads and scanned in order on the current device; the reference's two stages stay
observable: unexpected labels are reported (and raise) alone, otherwise the per-case errors and warnings follow, in
case order.

With the check on and `DeviceFingerprintExtractor` as the extractor, `extract_fingerprint_dataset` reads every case
once for both: the scan runs on the device copy the fingerprint uploads.  A dataset that fails the check prints the
reference's text, raises its RuntimeError and writes no fingerprint; an exception the fingerprint would raise for a
case (e.g. +-inf in the images) is raised only after the check has passed, as the reference runs the two in turn.

Rejected before any launch: a seg dtype other than uint8, int8, int16, uint16, int32, float32, and 2^31 voxels or more
in a case (NotImplementedError).
"""
import json
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import fingerprint as F
from . import lib as L
from . import preprocess as PP

REQUIRED_KEYS = ['labels', "channel_names", "numTraining", "file_ending"]
DEFAULT_NUM_PROCESSES = 8 if 'nnUNet_def_n_proc' not in os.environ else int(os.environ['nnUNet_def_n_proc'])
LABELS_ERROR = ('Some segmentation images contained unexpected labels. Please check text output above to see which '
                'one(s).')
CASES_ERROR = 'Some images have errors. Please check text output above to see which one(s) and what\'s going on.'
IMAGE_NAN, IMAGE_INF, SEG_NAN = 1, 2, 4   # B2U_VI_* flags
_F32 = PP.SEG_DTYPE_CODES[np.dtype(np.float32)]
_U16 = PP.SEG_DTYPE_CODES[np.dtype(np.uint16)]


def _label_manager(labels: dict, regions_class_order):
    """The host nnU-Net's LabelManager (tests substitute it)."""
    from dinounet.utilities.label_handling.label_handling import LabelManager
    return LabelManager(labels, regions_class_order=regions_class_order)


def _subfiles(folder: str, suffix: str) -> list:
    """batchgenerators' subfiles(folder, suffix=suffix, join=False): sorted file names."""
    return sorted(i for i in os.listdir(folder) if os.path.isfile(os.path.join(folder, i)) and i.endswith(suffix))


class _Plan:
    """What the reference establishes before its pool (verify_dataset_integrity.py:128-200)."""

    def __init__(self, folder: str):
        join = os.path.join
        assert os.path.isfile(join(folder, "dataset.json")), \
            f"There needs to be a dataset.json file in folder, folder={folder}"
        with open(join(folder, "dataset.json")) as f:
            dataset_json = json.load(f)
        if 'dataset' not in dataset_json.keys():
            assert os.path.isdir(join(folder, "imagesTr")), \
                f"There needs to be a imagesTr subfolder in folder, folder={folder}"
            assert os.path.isdir(join(folder, "labelsTr")), \
                f"There needs to be a labelsTr subfolder in folder, folder={folder}"
        dataset_keys = list(dataset_json.keys())
        assert all([i in dataset_keys for i in REQUIRED_KEYS]), \
            'not all required keys are present in dataset.json.\n\nRequired: \n%s\n\nPresent: \n%s\n\nMissing: ' \
            '\n%s\n\nUnused by nnU-Net:\n%s' % (str(REQUIRED_KEYS), str(dataset_keys),
                                               str([i for i in REQUIRED_KEYS if i not in dataset_keys]),
                                               str([i for i in dataset_keys if i not in REQUIRED_KEYS]))
        expected_num_training = dataset_json['numTraining']
        self.num_modalities = len(dataset_json['channel_names'].keys() if 'channel_names' in dataset_json.keys()
                                  else dataset_json['modality'].keys())
        file_ending = dataset_json['file_ending']
        dataset = PP._get_filenames_of_train_images_and_targets(folder, dataset_json)
        assert len(dataset) == expected_num_training, \
            'Did not find the expected number of training cases (%d). Found %d instead.\nExamples: %s' % \
            (expected_num_training, len(dataset), list(dataset.keys())[:5])
        if 'dataset' in dataset_json.keys():
            ok = True
            missing_images, missing_labels = [], []
            for k in dataset:
                for i in dataset[k]['images']:
                    if not os.path.isfile(i):
                        missing_images.append(i)
                        ok = False
                if not os.path.isfile(dataset[k]['label']):
                    missing_labels.append(dataset[k]['label'])
                    ok = False
            if not ok:
                raise FileNotFoundError(f"Some expected files were missing. Make sure you are properly referencing "
                                        f"them in the dataset.json. Or use imagesTr & labelsTr folders!\nMissing "
                                        f"images:\n{missing_images}\n\nMissing labels:\n{missing_labels}")
        else:
            labelfiles = _subfiles(join(folder, 'labelsTr'), file_ending)
            label_identifiers = [i[:-len(file_ending)] for i in labelfiles]
            labels_present = [i in label_identifiers for i in dataset.keys()]
            missing = [i for j, i in enumerate(dataset.keys()) if not labels_present[j]]
            assert all(labels_present), \
                f'not all training cases have a label file in labelsTr. Fix that. Missing: {missing}'
        label_manager = _label_manager(dataset_json['labels'], dataset_json.get('regions_class_order'))
        expected_labels = list(label_manager.all_labels)
        if label_manager.has_ignore_label:
            expected_labels.append(label_manager.ignore_label)
        labels_valid_consecutive = np.ediff1d(expected_labels) == 1
        assert all(labels_valid_consecutive), \
            f'Labels must be in consecutive order (0, 1, 2, ...). The labels ' \
            f'{np.array(expected_labels)[1:][~labels_valid_consecutive]} do not satisfy this restriction'
        self.rw_class = F._determine_reader_writer(dataset_json, dataset[next(iter(dataset.keys()))]['images'][0])
        self.folder, self.dataset, self.expected_labels = folder, dataset, expected_labels
        self.lo, self.hi = int(expected_labels[0]), int(expected_labels[-1])


def seg_code(seg, images) -> int:
    """This module's scope, before any launch: the seg's dtype code."""
    code = F._seg_code(seg)
    for shape in (seg.shape[1:], images.shape[1:]):
        if int(np.prod(shape)) >= 2 ** 31:
            raise NotImplementedError(f"a case of {tuple(shape)} has 2^31 voxels or more")
    return code


def found_labels(seg: torch.Tensor, code: int, np_dtype, seg_nan: bool) -> np.ndarray:
    """np.sort(pd.unique(seg.ravel())) of a device seg (int16 bits for uint16): one NaN, last, and a zero with the sign
    of the seg's first zero, as pd.unique keeps the first of values that compare equal."""
    seg = seg.reshape(-1)
    values = seg[~torch.isnan(seg)] if seg_nan else seg
    u = torch.unique(values).cpu().numpy()
    u = u.view(np.uint16) if code == _U16 else u
    u = np.sort(u.astype(np_dtype, copy=False))
    if code == _F32:
        zero = u == 0
        if zero.any():
            first = seg[int(torch.argmax((seg == 0).to(torch.uint8)))]
            u[zero] = np.float32(-0.0) if bool(torch.signbit(first)) else np.float32(0.0)
        if seg_nan:
            u = np.append(u, np.float32(np.nan))
    return u


class _Scan:
    """b2u_vi_scan of one case; `result()` reads (offenders, flags) once."""

    def __init__(self, img, seg, code: int, lo: int, hi: int, lib, stream):
        self.out = torch.empty(2, dtype=torch.int64, device=seg.device)
        L.check(lib.b2u_vi_scan(img.data_ptr() if img is not None else None, img.numel() if img is not None else 0,
                                seg.data_ptr(), code, seg.numel(), lo, hi, self.out.data_ptr(), stream),
                "b2u_vi_scan")
        self.host = torch.empty(2, dtype=torch.int64, pin_memory=True)
        self.host.copy_(self.out, non_blocking=True)
        self.ready = torch.cuda.Event()
        self.ready.record(torch.cuda.current_stream(seg.device))

    def result(self):
        self.ready.synchronize()
        return int(self.host[0]), int(self.host[1]) & 0xffffffff


def upload(seg: np.ndarray, images: np.ndarray, code: int, dev):
    """(seg [n] in its stored dtype, int16 bits for uint16; images fp32 [C * n]) on `dev`."""
    s = seg.view(np.int16) if code == _U16 else seg
    s = torch.from_numpy(np.ascontiguousarray(s).reshape(-1)).to(dev, non_blocking=True)
    img = torch.from_numpy(np.ascontiguousarray(images, dtype=np.float32).reshape(-1)).to(dev, non_blocking=True)
    return s, img


class _Verifier:
    """Scans the cases in order, reads each result one case later, and keeps the reference's messages of both
    stages.  `failed` turns true as soon as a case is known to fail."""

    def __init__(self, plan: _Plan):
        self.plan = plan
        self.dev = self.lib = self.stream = None   # the current device, at the first case
        self.label_errors, self.case_messages = [], []
        self.cases_failed = False
        self.inf_keys = []   # cases whose images hold +-inf (no verify error; the fingerprint rejects them)
        self.pending = None

    @property
    def failed(self) -> bool:
        return bool(self.label_errors) or self.cases_failed

    def submit(self, key, images, seg, props_images, props_seg, code: int, device_case=None) -> None:
        """Launches the scan of one case, on `device_case`'s buffers (a fingerprint `_Case`) or on an upload of its
        own, and finishes the previous case."""
        if self.lib is None:
            self.lib = L.load()
            self.dev = torch.device("cuda", torch.cuda.current_device())
            self.stream = torch.cuda.current_stream(self.dev).cuda_stream
        if device_case is not None:
            s, img = device_case.seg, device_case.img
        else:
            s, img = upload(seg, images, code, self.dev)
        scan = _Scan(img, s, code, self.plan.lo, self.plan.hi, self.lib, self.stream)
        self._finish_pending()
        self.pending = (key, images.shape, seg.shape, seg.dtype, props_images, props_seg, code, s, scan)
        if not self.host_checks_pass(images, seg, props_images, props_seg):
            self.cases_failed = True

    def host_checks_pass(self, images, seg, props_images, props_seg) -> bool:
        return (images.shape[1:] == seg.shape[1:] and bool(np.allclose(props_seg['spacing'], props_images['spacing']))
                and len(images) == self.plan.num_modalities)

    def _finish_pending(self) -> None:
        if self.pending is None:
            return
        key, img_shape, seg_shape, seg_dtype, props_images, props_seg, code, s, scan = self.pending
        self.pending = None
        offenders, flags = scan.result()
        join = os.path.join
        image_files, label_file = self.plan.dataset[key]['images'], self.plan.dataset[key]['label']
        if offenders:
            found = found_labels(s, code, seg_dtype, bool(flags & SEG_NAN))
            self.label_errors.append("Error: Unexpected labels found in file %s.\nExpected: %s\nFound: %s" % (
                join(self.plan.folder, 'labelsTr', label_file), self.plan.expected_labels, found))
        ok = True
        out = self.case_messages
        if flags & IMAGE_NAN:
            out.append(f'Images contain NaN pixel values. You need to fix that by replacing NaN values with something '
                       f'that makes sense for your images!\nImages:\n{image_files}')
            ok = False
        if flags & SEG_NAN:
            out.append(f'Segmentation contains NaN pixel values. You need to fix that.\nSegmentation:\n{label_file}')
            ok = False
        shape_image, shape_seg = img_shape[1:], seg_shape[1:]
        if shape_image != shape_seg:
            out.append('Error: Shape mismatch between segmentation and corresponding images. \nShape images: %s. '
                       '\nShape seg: %s. \nImage files: %s. \nSeg file: %s\n' %
                       (shape_image, shape_seg, image_files, label_file))
            ok = False
        spacing_images, spacing_seg = props_images['spacing'], props_seg['spacing']
        if not np.allclose(spacing_seg, spacing_images):
            out.append('Error: Spacing mismatch between segmentation and corresponding images. \nSpacing images: %s. '
                       '\nSpacing seg: %s. \nImage files: %s. \nSeg file: %s\n' %
                       (spacing_images, spacing_seg, image_files, label_file))
            ok = False
        if not img_shape[0] == self.plan.num_modalities:
            out.append('Error: Unexpected number of modalities. \nExpected: %d. \nGot: %d. \nImages: %s\n'
                       % (self.plan.num_modalities, img_shape[0], image_files))
            ok = False
        if 'nibabel_stuff' in props_images.keys():
            affine_image = props_images['nibabel_stuff']['original_affine']
            affine_seg = props_seg['nibabel_stuff']['original_affine']
            if not np.allclose(affine_image, affine_seg):
                out.append('WARNING: Affine is not the same for image and seg! \nAffine image: %s \nAffine seg: %s\n'
                           'Image files: %s. \nSeg file: %s.\nThis can be a problem but doesn\'t have to be. Please '
                           'run nnUNet_plot_dataset_pngs to verify if everything is OK!\n'
                           % (affine_image, affine_seg, image_files, label_file))
        if 'sitk_stuff' in props_images.keys():
            origin_image, origin_seg = props_images['sitk_stuff']['origin'], props_seg['sitk_stuff']['origin']
            if not np.allclose(origin_image, origin_seg):
                out.append('Warning: Origin mismatch between segmentation and corresponding images. \nOrigin images: '
                           '%s. \nOrigin seg: %s. \nImage files: %s. \nSeg file: %s\n' %
                           (origin_image, origin_seg, image_files, label_file))
            direction_image = props_images['sitk_stuff']['direction']
            direction_seg = props_seg['sitk_stuff']['direction']
            if not np.allclose(direction_image, direction_seg):
                out.append('Warning: Direction mismatch between segmentation and corresponding images. \nDirection '
                           'images: %s. \nDirection seg: %s. \nImage files: %s. \nSeg file: %s\n' %
                           (direction_image, direction_seg, image_files, label_file))
        if not ok:
            self.cases_failed = True
        if flags & IMAGE_INF:
            self.inf_keys.append(key)

    def finish(self) -> None:
        """Prints the reference's text for the dataset and raises its RuntimeError when a case failed."""
        self._finish_pending()
        if self.label_errors:
            for m in self.label_errors:
                print(m)
            raise RuntimeError(LABELS_ERROR)
        for m in self.case_messages:
            print(m)
        if self.cases_failed:
            raise RuntimeError(CASES_ERROR)
        print('\n####################')
        print('verify_dataset_integrity Done. \nIf you didn\'t see any error messages then your dataset is most likely '
              'OK!')
        print('####################\n')


def _read(plan: _Plan, key):
    rw = plan.rw_class()
    images, props_images = rw.read_images(plan.dataset[key]['images'])
    seg, props_seg = rw.read_seg(plan.dataset[key]['label'])
    seg, images, _ = F._as_input(seg, images)
    return images, seg, props_images, props_seg, seg_code(seg, images)


def verify_dataset_integrity(folder: str, num_processes: int = 8) -> None:
    """The reference's verify_dataset_integrity (verify_dataset_integrity.py:119-227): the same text on stdout, the same
    exceptions, None."""
    plan = _Plan(folder)
    keys = list(plan.dataset.keys())
    workers = max(1, int(num_processes))
    with ThreadPoolExecutor(workers) as pool:
        verifier = _Verifier(plan)
        reads = [pool.submit(_read, plan, k) for k in keys[:workers]]
        for i, k in enumerate(keys):
            images, seg, props_images, props_seg, code = reads[i].result()
            reads[i] = None
            if i + workers < len(keys):
                reads.append(pool.submit(_read, plan, keys[i + workers]))
            verifier.submit(k, images, seg, props_images, props_seg, code)
        verifier.finish()


# ---- the fused route: one read of each case for the check and the fingerprint ----------------------------------------


class _FusedCheck:
    """The fingerprint's per-case hooks (DeviceFingerprintExtractor._sample_dataset) that verify the dataset on the
    way.  A case the fingerprint could not take, or any case once the check or the fingerprint has failed, is only
    verified; the fingerprint's exception for the first such case is raised after the check has passed."""

    def __init__(self, plan: _Plan):
        self.plan = plan
        self.verifier = _Verifier(plan)
        self.order = {k: i for i, k in enumerate(plan.dataset)}
        self.fingerprint_errors = {}

    def read(self, images, seg, props_seg):
        """On a reader thread: (the seg's properties, the verify's seg code, the fingerprint's seg code or the
        exception its check raises).  The fingerprint's NaN and +-inf checks come from the scan's flags instead of a
        host pass: NaN fails the verify, +-inf is the fingerprint's NotImplementedError."""
        code = seg_code(seg, images)
        try:
            assert images.ndim == 4
            assert seg.ndim == 4
            if images.dtype != np.float32:
                raise NotImplementedError(f"images of dtype {images.dtype}: the device fingerprint takes float32 "
                                          "images (what every reader delivers)")
            if tuple(images.shape[1:]) != tuple(seg.shape[1:]):
                raise IndexError(f"the segmentation {tuple(seg.shape)} and the images {tuple(images.shape)} differ "
                                 "in shape")
            fp = code
        except (AssertionError, NotImplementedError, IndexError) as e:
            fp = e
        return props_seg, code, fp

    def _errors(self) -> dict:
        inf = NotImplementedError("the images hold +-inf: the reference would write inf / nan statistics")
        return {**{self.order[k]: inf for k in self.verifier.inf_keys}, **self.fingerprint_errors}

    @property
    def sampling(self) -> bool:
        return not self.verifier.failed and not self._errors()

    def case(self, key, images, seg, props_images, read, make_case):
        """Scans the case, on the fingerprint's device copy (`make_case(code)`) when the fingerprint takes it;
        returns that copy or None."""
        props_seg, code, fp = read
        device_case = None
        if isinstance(fp, Exception):
            self.fingerprint_errors[self.order[key]] = fp
        elif self.sampling and self.verifier.host_checks_pass(images, seg, props_images, props_seg):
            device_case = make_case(fp)
        self.verifier.submit(key, images, seg, props_images, props_seg, code, device_case)
        return device_case

    def finish(self) -> None:
        self.verifier.finish()
        errors = self._errors()
        if errors:
            raise errors[min(errors)]


def extract_fingerprint_dataset(dataset_id, fingerprint_extractor_class=F.DeviceFingerprintExtractor,
                                num_processes: int = DEFAULT_NUM_PROCESSES, check_dataset_integrity: bool = False,
                                clean: bool = True, verbose: bool = True):
    """The reference's extract_fingerprint_dataset (plan_and_preprocess_api.py:17-32): returns the fingerprint (and
    writes it).  With the check on and DeviceFingerprintExtractor, the check and the fingerprint share one read of each
    case; with any other extractor the check runs first, then the extractor."""
    dataset_name = PP._dataset_name(dataset_id)
    print(dataset_name)
    raw, _ = PP._raw_and_preprocessed()
    folder = os.path.join(raw, dataset_name)
    if check_dataset_integrity and isinstance(fingerprint_extractor_class, type) and \
            issubclass(fingerprint_extractor_class, F.DeviceFingerprintExtractor):
        plan = _Plan(folder)   # the reference's host checks raise before the extractor is made
        fpe = fingerprint_extractor_class(dataset_id, num_processes, verbose=verbose)
        _, preprocessed = PP._raw_and_preprocessed()
        stored = os.path.join(preprocessed, fpe.dataset_name, "dataset_fingerprint.json")
        if not clean and os.path.isfile(stored):
            verify_dataset_integrity(folder, num_processes)
            return fpe.run(overwrite_existing=False)
        return fpe._run(True, _FusedCheck(plan))
    if check_dataset_integrity:
        verify_dataset_integrity(folder, num_processes)
    fpe = fingerprint_extractor_class(dataset_id, num_processes, verbose=verbose)
    return fpe.run(overwrite_existing=clean)


def _find_extractor_class(name: str):
    """The reference's lookup of an extractor class by name under dinounet.experiment_planning; this module's
    DeviceFingerprintExtractor by its own name."""
    if name == F.DeviceFingerprintExtractor.__name__:
        return F.DeviceFingerprintExtractor
    import dinounet
    from dinounet.utilities.find_class_by_name import recursive_find_python_class
    return recursive_find_python_class(os.path.join(dinounet.__path__[0], "experiment_planning"), name,
                                       current_module="dinounet.experiment_planning")


def extract_fingerprints(dataset_ids, fingerprint_extractor_class_name: str = 'DatasetFingerprintExtractor',
                         num_processes: int = DEFAULT_NUM_PROCESSES, check_dataset_integrity: bool = False,
                         clean: bool = True, verbose: bool = True):
    """The reference's extract_fingerprints (plan_and_preprocess_api.py:35-47), with this module's
    extract_fingerprint_dataset."""
    fingerprint_extractor_class = _find_extractor_class(fingerprint_extractor_class_name)
    for d in dataset_ids:
        extract_fingerprint_dataset(d, fingerprint_extractor_class, num_processes, check_dataset_integrity, clean,
                                    verbose)
