#!/usr/bin/env python
"""Golden outputs of the REAL reference's transformation classes (data_generator/object_detection_2d_geometric_ops.py,
_patch_sampling_ops.py, _photometric_ops.py), unmodified, with cv2: each class of tests/transformations_cases.py ``SINGLES``
applied alone to seeded images and labels, and the custom chains of ``CHAINS`` through the reference's own
``DataGenerator.generate`` with shuffling and a short last batch.

- ``single_<name>_<k>_x`` / ``_labels`` / ``_pos``: image k (``single_images``) of ``chain_dataset.variable_dataset('float')``
  through the case's list, its labels and ``np.random``'s position after it; ``single_<name>_state``: the state after the
  case's last image (one seed, ``SINGLE_SEED``, before its first);
- ``<chain>_digest``, ``<chain>_b<k>_x`` (uint8 images), ``_labels`` with ``_counts``, ``_files`` and ``_state`` / ``_pos`` per
  batch, as tests/golden/make_augmentation_chains_golden.py writes them.

The inputs come from tests/chain_dataset.py.  cv2 runs with IPP off; ``np.int`` / ``np.float`` are put back for the
reference's Scale and Rotate.  Needs the reference tree, cv2, sklearn and tqdm; run once, the .npz is data."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.environ.get('SSD_REFERENCE_ROOT', '/root/reference'))
np.int = int
np.float = float

import cv2  # noqa: E402

sys.path.insert(0, os.path.dirname(HERE))
import chain_dataset as ds  # noqa: E402
import transformations_cases as tc  # noqa: E402

from data_generator import object_detection_2d_geometric_ops as geo  # noqa: E402
from data_generator import object_detection_2d_image_boxes_validation_utils as valid  # noqa: E402
from data_generator import object_detection_2d_patch_sampling_ops as patch  # noqa: E402
from data_generator import object_detection_2d_photometric_ops as photo  # noqa: E402
from data_generator.object_detection_2d_data_generator import DataGenerator  # noqa: E402


class Modules:
    pass


M = Modules()
M.geo, M.patch, M.photo, M.valid = geo, patch, photo, valid
SINGLE_IMAGES = (1, 2, 5)                  # a gray, an RGBA and a one-channel image


def singles(out):
    images, labels = ds.variable_dataset('float')
    for name, make in tc.SINGLES.items():
        np.random.seed(tc.SINGLE_SEED)
        chain = [photo.ConvertTo3Channels()] + make(M)
        for k in SINGLE_IMAGES:
            x, y = images[k].copy(), labels[k].copy()
            for t in chain:
                x, y = t(x, y)
            p = 'single_%s_%d_' % (name, k)
            out[p + 'x'] = np.asarray(x, np.uint8)
            out[p + 'labels'] = np.asarray(y, np.float64).reshape(-1, 5)
            out[p + 'pos'] = np.int64(np.random.get_state()[2])
        out['single_%s_state' % name] = np.random.get_state()[1]
        print('single', name, [out['single_%s_%d_x' % (name, k)].shape for k in SINGLE_IMAGES])


def chains(out):
    for name, (make, dataset, dtype, seed, n_batches) in tc.CHAINS.items():
        images, labels = dataset(dtype)
        out[name + '_digest'] = ds.digest(images, labels)
        gen = DataGenerator(load_images_into_memory=False, filenames=['%d' % i for i in range(len(images))], labels=[l.copy() for l in labels])
        gen.images = images
        np.random.seed(seed)
        it = gen.generate(batch_size=tc.BATCH, shuffle=True, transformations=make(M), label_encoder=None,
                          returns={'processed_images', 'processed_labels', 'filenames'}, keep_images_without_gt=False)
        for k in range(n_batches):
            x, y, files = next(it)
            p = '%s_b%d_' % (name, k)
            out[p + 'x'] = np.asarray(x, np.uint8)
            out[p + 'labels'] = np.concatenate([np.asarray(a, np.float64).reshape(-1, 5) for a in y])
            out[p + 'counts'] = np.array([len(a) for a in y], np.int64)
            out[p + 'files'] = np.array([int(f) for f in files], np.int64)
            state = np.random.get_state()
            out[p + 'state'], out[p + 'pos'] = state[1], np.int64(state[2])
            print(name, 'batch', k, 'images', out[p + 'files'].tolist(), 'boxes', out[p + 'counts'].tolist())


def main():
    cv2.ipp.setUseIPP(False)
    out = {'batch_size': tc.BATCH, 'single_images': np.array(SINGLE_IMAGES)}
    singles(out)
    chains(out)
    np.savez_compressed(os.path.join(HERE, 'ref_transformations_golden.npz'), **out)


if __name__ == '__main__':
    main()
