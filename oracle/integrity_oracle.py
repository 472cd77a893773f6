"""A numpy / pandas restatement of the reference's `verify_dataset_integrity`
(experiment_planning/verify_dataset_integrity.py:32-227) in one process: `verify(folder, reader_class)` returns the
stdout text and the exception (or None).  The spawn pool becomes a loop in case order, so the per-case messages come in
that order.  Restated with it: `get_filenames_of_train_images_and_targets` (utilities/utils.py:26-65) and the
LabelManager properties the check reads (label_handling.py: all labels as np.int64 from np.unique, the ignore label
and its assertions, and the regions' `regions_class_order` assertions).
"""
import contextlib
import io
import json
import os
import re

import numpy as np
import pandas as pd

REQUIRED_KEYS = ['labels', "channel_names", "numTraining", "file_ending"]


class LabelManager:
    """The parts of label_handling.LabelManager that verify_dataset_integrity reads."""

    def __init__(self, label_dict: dict, regions_class_order=None):
        if 'background' not in label_dict.keys():
            raise RuntimeError('Background label not declared (remember that this should be label 0!)')
        bg = label_dict['background']
        if isinstance(bg, (tuple, list)):
            raise RuntimeError(f"Background label must be 0. Not a list. Not a tuple. Your background label: {bg}")
        assert int(bg) == 0, f"Background label must be 0. Your background label: {bg}"
        has_regions = any(isinstance(i, (tuple, list)) and len(i) > 1 for i in label_dict.values())
        self.ignore_label = label_dict.get('ignore')
        if self.ignore_label is not None:
            assert isinstance(self.ignore_label, int), f'Ignore label has to be an integer. It cannot be a region ' \
                                                       f'(list/tuple). Got {type(self.ignore_label)}.'
        labels = [int(v) for k, r in label_dict.items() if k != 'ignore'
                  for v in (r if isinstance(r, (tuple, list)) else [r])]
        self.all_labels = sorted(list(np.unique(labels)))
        if has_regions:
            assert regions_class_order is not None, \
                'if region-based training is requested then you need to define regions_class_order!'
            regions = [r for k, r in label_dict.items() if k != 'ignore' and not (
                (np.isscalar(r) and r == 0) or
                (isinstance(r, (tuple, list)) and len(np.unique(r)) == 1 and np.unique(r)[0] == 0))]
            assert len(regions_class_order) == len(regions), \
                'regions_class_order must have as many entries as there are regions'
        self.has_ignore_label = self.ignore_label is not None
        if self.has_ignore_label:
            assert self.ignore_label == max(self.all_labels) + 1, \
                'If you use the ignore label it must have the highest label value! It cannot be 0 or in between ' \
                'other labels. Sorry bro.'


def subfiles(folder: str, suffix: str) -> list:
    return sorted(i for i in os.listdir(folder) if os.path.isfile(os.path.join(folder, i)) and i.endswith(suffix))


def get_filenames_of_train_images_and_targets(folder: str, dataset_json: dict) -> dict:
    join = os.path.join
    if 'dataset' in dataset_json.keys():
        dataset = dataset_json['dataset']
        for k in dataset.keys():
            lab = dataset[k]['label']
            dataset[k]['label'] = lab if os.path.isabs(lab) else os.path.abspath(join(folder, lab))
            dataset[k]['images'] = [i if os.path.isabs(i) else os.path.abspath(join(folder, i))
                                    for i in dataset[k]['images']]
        return dataset
    ending = dataset_json['file_ending']
    images_dir = join(folder, 'imagesTr')
    files = subfiles(images_dir, ending)
    identifiers = np.unique([i[:-(len(ending) + 5)] for i in files])
    dataset = {}
    for i in identifiers:
        p = re.compile(re.escape(i) + r"_\d\d\d\d" + re.escape(ending))
        dataset[i] = {'images': [join(images_dir, f) for f in files if p.fullmatch(f)],
                      'label': join(folder, 'labelsTr', i + ending)}
    return dataset


def _verify_labels(label_file, rw, expected_labels) -> bool:
    seg, _ = rw().read_seg(label_file)
    found = np.sort(pd.unique(seg.ravel()))
    if any(i not in expected_labels for i in found):
        print("Error: Unexpected labels found in file %s.\nExpected: %s\nFound: %s" % (label_file, expected_labels,
                                                                                       found))
        return False
    return True


def _check_case(image_files, label_file, expected_num_channels, rw) -> bool:
    r = rw()
    images, pi = r.read_images(image_files)
    seg, ps = r.read_seg(label_file)
    ok = True
    if np.any(np.isnan(images)):
        print(f'Images contain NaN pixel values. You need to fix that by replacing NaN values with something that '
              f'makes sense for your images!\nImages:\n{image_files}')
        ok = False
    if np.any(np.isnan(seg)):
        print(f'Segmentation contains NaN pixel values. You need to fix that.\nSegmentation:\n{label_file}')
        ok = False
    if images.shape[1:] != seg.shape[1:]:
        print('Error: Shape mismatch between segmentation and corresponding images. \nShape images: %s. \nShape seg: '
              '%s. \nImage files: %s. \nSeg file: %s\n' % (images.shape[1:], seg.shape[1:], image_files, label_file))
        ok = False
    if not np.allclose(ps['spacing'], pi['spacing']):
        print('Error: Spacing mismatch between segmentation and corresponding images. \nSpacing images: %s. '
              '\nSpacing seg: %s. \nImage files: %s. \nSeg file: %s\n' % (pi['spacing'], ps['spacing'], image_files,
                                                                         label_file))
        ok = False
    if len(images) != expected_num_channels:
        print('Error: Unexpected number of modalities. \nExpected: %d. \nGot: %d. \nImages: %s\n'
              % (expected_num_channels, len(images), image_files))
        ok = False
    if 'nibabel_stuff' in pi.keys():
        a, b = pi['nibabel_stuff']['original_affine'], ps['nibabel_stuff']['original_affine']
        if not np.allclose(a, b):
            print('WARNING: Affine is not the same for image and seg! \nAffine image: %s \nAffine seg: %s\nImage files: '
                  '%s. \nSeg file: %s.\nThis can be a problem but doesn\'t have to be. Please run '
                  'nnUNet_plot_dataset_pngs to verify if everything is OK!\n' % (a, b, image_files, label_file))
    if 'sitk_stuff' in pi.keys():
        a, b = pi['sitk_stuff']['origin'], ps['sitk_stuff']['origin']
        if not np.allclose(a, b):
            print('Warning: Origin mismatch between segmentation and corresponding images. \nOrigin images: %s. '
                  '\nOrigin seg: %s. \nImage files: %s. \nSeg file: %s\n' % (a, b, image_files, label_file))
        a, b = pi['sitk_stuff']['direction'], ps['sitk_stuff']['direction']
        if not np.allclose(a, b):
            print('Warning: Direction mismatch between segmentation and corresponding images. \nDirection images: %s. '
                  '\nDirection seg: %s. \nImage files: %s. \nSeg file: %s\n' % (a, b, image_files, label_file))
    return ok


def _verify(folder: str, rw) -> None:
    join = os.path.join
    assert os.path.isfile(join(folder, "dataset.json")), f"There needs to be a dataset.json file in folder, folder={folder}"
    with open(join(folder, "dataset.json")) as f:
        dj = json.load(f)
    if 'dataset' not in dj.keys():
        assert os.path.isdir(join(folder, "imagesTr")), f"There needs to be a imagesTr subfolder in folder, folder={folder}"
        assert os.path.isdir(join(folder, "labelsTr")), f"There needs to be a labelsTr subfolder in folder, folder={folder}"
    keys = list(dj.keys())
    assert all(i in keys for i in REQUIRED_KEYS), \
        'not all required keys are present in dataset.json.\n\nRequired: \n%s\n\nPresent: \n%s\n\nMissing: \n%s\n\n' \
        'Unused by nnU-Net:\n%s' % (str(REQUIRED_KEYS), str(keys), str([i for i in REQUIRED_KEYS if i not in keys]),
                                   str([i for i in keys if i not in REQUIRED_KEYS]))
    n_train = dj['numTraining']
    n_channels = len(dj['channel_names'].keys() if 'channel_names' in dj.keys() else dj['modality'].keys())
    dataset = get_filenames_of_train_images_and_targets(folder, dj)
    assert len(dataset) == n_train, 'Did not find the expected number of training cases (%d). Found %d instead.\n' \
                                    'Examples: %s' % (n_train, len(dataset), list(dataset.keys())[:5])
    if 'dataset' in dj.keys():
        missing_images = [i for k in dataset for i in dataset[k]['images'] if not os.path.isfile(i)]
        missing_labels = [dataset[k]['label'] for k in dataset if not os.path.isfile(dataset[k]['label'])]
        if missing_images or missing_labels:
            raise FileNotFoundError(f"Some expected files were missing. Make sure you are properly referencing them "
                                    f"in the dataset.json. Or use imagesTr & labelsTr folders!\nMissing images:"
                                    f"\n{missing_images}\n\nMissing labels:\n{missing_labels}")
    else:
        ending = dj['file_ending']
        ids = [i[:-len(ending)] for i in subfiles(join(folder, 'labelsTr'), ending)]
        missing = [k for k in dataset.keys() if k not in ids]
        assert not missing, f'not all training cases have a label file in labelsTr. Fix that. Missing: {missing}'
    lm = LabelManager(dj['labels'], dj.get('regions_class_order'))
    expected = list(lm.all_labels)
    if lm.has_ignore_label:
        expected.append(lm.ignore_label)
    consecutive = np.ediff1d(expected) == 1
    assert all(consecutive), f'Labels must be in consecutive order (0, 1, 2, ...). The labels ' \
                             f'{np.array(expected)[1:][~consecutive]} do not satisfy this restriction'
    if not all([_verify_labels(join(folder, 'labelsTr', v['label']), rw, expected) for v in dataset.values()]):
        raise RuntimeError('Some segmentation images contained unexpected labels. Please check text output above to '
                           'see which one(s).')
    if not all([_check_case(v['images'], v['label'], n_channels, rw) for v in dataset.values()]):
        raise RuntimeError('Some images have errors. Please check text output above to see which one(s) and what\'s '
                           'going on.')
    print('\n####################')
    print('verify_dataset_integrity Done. \nIf you didn\'t see any error messages then your dataset is most likely OK!')
    print('####################\n')


def verify(folder: str, reader_class):
    """(stdout, exception or None) of the reference's verify_dataset_integrity(folder)."""
    out = io.StringIO()
    exc = None
    with contextlib.redirect_stdout(out):
        try:
            _verify(folder, reader_class)
        except Exception as e:   # noqa: BLE001 - the exception is the result
            exc = e
    return out.getvalue(), exc
