#!/usr/bin/env python
"""Golden batches of the REAL reference's ``DataGenerator.generate`` with its SSD7, variable-input-size and satellite chains
(data_generator/data_augmentation_chain_constant_input_size.py, _variable_input_size.py, _satellite.py), and of its
``parse_csv``.

Each run seeds both the global ``np.random`` and Python's ``random`` (``RandomRotate`` draws its angle from the latter) and
takes batches of 4 with shuffling, so that a pass ends in a short batch and the next starts with a reshuffle:

- ``ssd7_int``: the SSD7 notebook's chain arguments on ten 60 x 96 images with int64 labels, images without boxes dropped;
- ``ssd7_float``: the same chain with a non-black background on float labels, images without boxes kept;
- ``variable``: ``DataAugmentationVariableInputSize(48, 64)``, int64 labels, images without boxes dropped;
- ``satellite``: ``DataAugmentationSatellite(48, 64)`` with a non-black ``background`` (its patches still pad black, as the
  reference does not hand it to ``RandomPatch``), float labels, images without boxes kept.

The inputs come from tests/chain_dataset.py (a seed and NumPy), so the file holds the outputs and a digest of the inputs only:
per run ``<run>_digest``, and per batch ``<run>_b<k>_x`` (uint8 images), ``_labels`` (processed labels, stacked, float64)
with ``_counts``, ``_files`` (dataset indices), ``_state`` / ``_pos`` (``np.random``'s state after the batch) and ``_pystate``
(Python ``random``'s).  ``csv_*``: ``parse_csv`` of ``chain_dataset.csv_text()`` with ``include_classes`` and a seeded
``random_sample``: the file names relative to the image directory, the image ids, the labels and ``np.random``'s state.

cv2 runs with IPP off.  NumPy >= 1.24 has no ``np.int`` / ``np.float``, which the reference's Scale and Rotate use, so they are
put back as the builtins they aliased.  Needs the reference tree, cv2, PIL, sklearn and tqdm; run once, the .npz is data."""
import os
import random
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.environ.get('SSD_REFERENCE_ROOT', '/root/reference'))
np.int = int
np.float = float

import cv2  # noqa: E402

sys.path.insert(0, os.path.dirname(HERE))
import chain_dataset as ds  # noqa: E402

from data_generator.data_augmentation_chain_constant_input_size import DataAugmentationConstantInputSize  # noqa: E402
from data_generator.data_augmentation_chain_satellite import DataAugmentationSatellite  # noqa: E402
from data_generator.data_augmentation_chain_variable_input_size import DataAugmentationVariableInputSize  # noqa: E402
from data_generator.object_detection_2d_data_generator import DataGenerator  # noqa: E402

BATCH = 4
SSD7_ARGS = dict(random_brightness=(-48, 48, 0.5), random_contrast=(0.5, 1.8, 0.5), random_saturation=(0.5, 1.8, 0.5),
                 random_hue=(18, 0.5), random_flip=0.5, random_translate=((0.03, 0.5), (0.03, 0.5), 0.5), random_scale=(0.5, 2.0, 0.5),
                 n_trials_max=3, clip_boxes=True, overlap_criterion='area', bounds_box_filter=(0.3, 1.0), bounds_validator=(0.5, 1.0),
                 n_boxes_min=1, background=(0, 0, 0))
# name: (dataset, labels dtype, chain, keep_images_without_gt, batches, seed)
RUNS = {
    'ssd7_int': (ds.ssd7_dataset, 'int', lambda: DataAugmentationConstantInputSize(**SSD7_ARGS), False, 8, 11),
    'ssd7_float': (ds.ssd7_dataset, 'float', lambda: DataAugmentationConstantInputSize(**dict(SSD7_ARGS, background=(123, 117, 104))),
                   True, 8, 12),
    'variable': (ds.variable_dataset, 'int', lambda: DataAugmentationVariableInputSize(48, 64), False, 7, 13),
    'satellite': (ds.variable_dataset, 'float', lambda: DataAugmentationSatellite(48, 64, background=(200, 100, 50)), True, 8, 14),
}
CSV_SEED = 15


def run(name, out):
    dataset, dtype, chain, keep, n_batches, seed = RUNS[name]
    images, labels = dataset(dtype)
    out[name + '_digest'] = ds.digest(images, labels)
    gen = DataGenerator(load_images_into_memory=False, filenames=['%d' % i for i in range(len(images))], labels=[l.copy() for l in labels])
    gen.images = images
    np.random.seed(seed)
    random.seed(seed)
    it = gen.generate(batch_size=BATCH, shuffle=True, transformations=[chain()], label_encoder=None,
                      returns={'processed_images', 'processed_labels', 'filenames'}, keep_images_without_gt=keep)
    for k in range(n_batches):
        x, y, files = next(it)
        p = '%s_b%d_' % (name, k)
        out[p + 'x'] = np.asarray(x, np.uint8)
        out[p + 'labels'] = np.concatenate([np.asarray(a, np.float64).reshape(-1, 5) for a in y])
        out[p + 'counts'] = np.array([len(a) for a in y], np.int64)
        out[p + 'files'] = np.array([int(f) for f in files], np.int64)
        state = np.random.get_state()
        out[p + 'state'], out[p + 'pos'] = state[1], np.int64(state[2])
        out[p + 'pystate'] = np.array(random.getstate()[1], np.int64)
        print(name, 'batch', k, 'images', out[p + 'files'].tolist(), 'boxes', out[p + 'counts'].tolist())
    out[name + '_n_batches'], out[name + '_seed'] = n_batches, seed


def parse(out):
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, 'labels.csv')
        with open(path, 'w') as f:
            f.write(ds.csv_text())
        gen = DataGenerator()
        np.random.seed(CSV_SEED)
        _, filenames, labels, image_ids = gen.parse_csv(images_dir='images', labels_filename=path, input_format=ds.CSV_INPUT_FORMAT,
                                                        include_classes=ds.CSV_INCLUDE, random_sample=ds.CSV_SAMPLE, ret=True, verbose=False)
    out['csv_filenames'] = np.array([os.path.relpath(f, 'images') for f in filenames])
    out['csv_image_ids'] = np.array(image_ids)
    out['csv_labels'] = np.concatenate(labels)
    out['csv_counts'] = np.array([len(a) for a in labels], np.int64)
    out['csv_dtype'] = str(labels[0].dtype)
    state = np.random.get_state()
    out['csv_state'], out['csv_pos'], out['csv_seed'] = state[1], np.int64(state[2]), CSV_SEED
    print('parse_csv', len(filenames), 'images', out['csv_counts'].tolist())


def main():
    cv2.ipp.setUseIPP(False)
    out = {'batch_size': BATCH}
    for name in RUNS:
        run(name, out)
    parse(out)
    np.savez_compressed(os.path.join(HERE, 'ref_augmentation_chains_golden.npz'), **out)


if __name__ == '__main__':
    main()
