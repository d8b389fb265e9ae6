#!/usr/bin/env python
"""Golden batches of the REAL reference's ``DataGenerator.generate`` with ``SSDDataAugmentation``
(data_generator/object_detection_2d_data_generator.py, data_augmentation_chain_original_ssd.py): a seeded global ``np.random``,
nine images in memory (gray, RGB and RGBA; smaller and larger than the 90 x 120 output, two of them larger than 300), label sets that are empty, hold one
box, many boxes or boxes at the edges, batches of 4 with shuffling, so that the first pass ends in a short batch and the
second starts with a reshuffle.  The dataset comes from tests/augmentation_dataset.py (a seed and NumPy), so the file holds
the outputs and a digest of the inputs only.  cv2 runs with IPP off, i.e. OpenCV's own resize code (IPP's INTER_CUBIC differs from it in
the last bit at a few pixels in 10^5 and from CPU to CPU).  Writes tests/golden/ref_ssd_augmentation_golden.npz:
``n_images`` and ``digest`` (the dataset), per batch ``b<k>_x`` (uint8 processed images), ``b<k>_labels`` (the processed
labels, stacked) with ``b<k>_counts``, ``b<k>_files`` (the dataset indices of the batch) and ``b<k>_state`` / ``b<k>_pos``
(``np.random``'s state after the batch).  Needs the reference tree, cv2, PIL, sklearn and tqdm; run once, the .npz is data."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.environ.get('SSD_REFERENCE_ROOT', '/root/reference'))

import cv2  # noqa: E402

sys.path.insert(0, os.path.dirname(HERE))
import augmentation_dataset as ds  # noqa: E402

from data_generator.data_augmentation_chain_original_ssd import SSDDataAugmentation  # noqa: E402
from data_generator.object_detection_2d_data_generator import DataGenerator  # noqa: E402

SEED = ds.SEED
OUT_H, OUT_W = 90, 120
BATCH, N_BATCHES = 4, 7


def main():
    cv2.ipp.setUseIPP(False)
    images, labels = ds.dataset()
    out = {'n_images': len(images), 'digest': ds.digest(images)}
    gen = DataGenerator(load_images_into_memory=False, filenames=['%d' % i for i in range(len(images))], labels=[l.copy() for l in labels])
    gen.images = images
    aug = SSDDataAugmentation(img_height=OUT_H, img_width=OUT_W, background=(123, 117, 104))
    np.random.seed(SEED)
    it = gen.generate(batch_size=BATCH, shuffle=True, transformations=[aug], label_encoder=None,
                      returns={'processed_images', 'processed_labels', 'filenames'}, keep_images_without_gt=False)
    for k in range(N_BATCHES):
        x, y, files = next(it)
        out['b%d_x' % k] = np.asarray(x, np.uint8)
        out['b%d_labels' % k] = np.concatenate([np.asarray(a, np.float64).reshape(-1, 5) for a in y])
        out['b%d_counts' % k] = np.array([len(a) for a in y], np.int64)
        out['b%d_files' % k] = np.array([int(f) for f in files], np.int64)
        state = np.random.get_state()
        out['b%d_state' % k], out['b%d_pos' % k] = state[1], np.int64(state[2])
        print('batch', k, 'images', out['b%d_files' % k].tolist(), 'boxes', out['b%d_counts' % k].tolist())
    out['n_batches'], out['seed'], out['batch_size'], out['out_hw'] = N_BATCHES, SEED, BATCH, np.array([OUT_H, OUT_W])
    np.savez_compressed(os.path.join(HERE, 'ref_ssd_augmentation_golden.npz'), **out)


if __name__ == '__main__':
    main()
