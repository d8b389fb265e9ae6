#!/usr/bin/env python
"""Time the VOC evaluation notebook's pipeline (ssd300_evaluation.ipynb) on a VOC2007-test-shaped set built from a seed: JPEG
files of VOC's sizes (around 500 x 375, quality 90) and one Pascal VOC XML per image with 1-6 objects.

  python tools/time_voc_evaluation.py [--images N] [--out DIR]

Prints the card's name and power limit, then:
  - the host time of ``DataGenerator.parse_xml`` over the N annotation files;
  - the notebook's ``Evaluator`` call (SSD300, 20 classes, batch 8, 'resize', 11 recall points) in images/s, including the JPEG
    decoding, once from the files (PIL on the thread pool) and once with ``load_images_into_memory=True`` (the decoding into
    memory timed on its own).
The model has seeded random weights, so with ``confidence_thresh=0.01`` every image keeps its ``top_k=200`` boxes, as a
trained model does on most VOC images.  Writes the numbers as JSON to DIR/time_voc_evaluation.json when --out is given."""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CLASSES = ['background', 'aeroplane', 'bicycle', 'bird', 'boat', 'bottle', 'bus', 'car', 'cat', 'chair', 'cow', 'diningtable', 'dog',
           'horse', 'motorbike', 'person', 'pottedplant', 'sheep', 'sofa', 'train', 'tvmonitor']
SIZES = [(375, 500), (500, 375), (333, 500), (500, 333), (281, 500), (366, 500), (500, 400), (338, 500)]


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:                                           # noqa: BLE001
        return 'unknown (%s)' % e


def write_dataset(root, n, seed=0):
    """N JPEGs (8 x 8 blocks of colour over a ramp, with noise so that they do not compress to nothing), their XMLs and
    ImageSets/Main/test.txt."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    for d in ('JPEGImages', 'Annotations', os.path.join('ImageSets', 'Main')):
        os.makedirs(os.path.join(root, d), exist_ok=True)
    ids = ['%06d' % (i + 1) for i in range(n)]
    for image_id in ids:
        h, w = SIZES[int(rng.integers(len(SIZES)))]
        base = rng.integers(0, 220, (h // 8 + 1, w // 8 + 1, 3), dtype=np.int64)
        img = np.repeat(np.repeat(base, 8, 0), 8, 1)[:h, :w] + rng.integers(0, 36, (h, w, 3))
        Image.fromarray(img.astype(np.uint8)).save(os.path.join(root, 'JPEGImages', image_id + '.jpg'), quality=90)
        objects = ''
        for _ in range(int(rng.integers(1, 7))):
            x0, y0 = int(rng.integers(1, w - 40)), int(rng.integers(1, h - 40))
            x1, y1 = int(rng.integers(x0 + 20, w + 1)), int(rng.integers(y0 + 20, h + 1))
            objects += ('\t<object>\n\t\t<name>%s</name>\n\t\t<pose>Unspecified</pose>\n\t\t<truncated>%d</truncated>\n'
                        '\t\t<difficult>%d</difficult>\n\t\t<bndbox>\n\t\t\t<xmin>%d</xmin>\n\t\t\t<ymin>%d</ymin>\n\t\t\t<xmax>%d</xmax>\n'
                        '\t\t\t<ymax>%d</ymax>\n\t\t</bndbox>\n\t</object>\n'
                        % (CLASSES[int(rng.integers(1, 21))], int(rng.integers(3) == 0), int(rng.integers(5) == 0), x0, y0, x1, y1))
        with open(os.path.join(root, 'Annotations', image_id + '.xml'), 'w') as f:
            f.write('<annotation>\n\t<folder>VOC2007</folder>\n\t<filename>%s.jpg</filename>\n\t<size>\n\t\t<width>%d</width>\n'
                    '\t\t<height>%d</height>\n\t\t<depth>3</depth>\n\t</size>\n%s</annotation>\n' % (image_id, w, h, objects))
    with open(os.path.join(root, 'ImageSets', 'Main', 'test.txt'), 'w') as f:
        f.write(''.join(i + '\n' for i in ids))


def model():
    from oracle import synth
    from oracle.model import SSD300_AR, vgg_weight_shapes
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    m = ssd_300(image_size=(300, 300, 3), n_classes=20, mode='inference', l2_regularization=0.0005,
                scales=[0.1, 0.2, 0.37, 0.54, 0.71, 0.88, 1.05], aspect_ratios_per_layer=SSD300_AR, two_boxes_for_ar1=True,
                steps=[8, 16, 32, 64, 100, 300], offsets=[0.5] * 6, clip_boxes=False, variances=[0.1, 0.1, 0.2, 0.2],
                normalize_coords=True, subtract_mean=[123, 117, 104], swap_channels=[2, 1, 0], confidence_thresh=0.01,
                iou_threshold=0.45, top_k=200, nms_max_output_size=400)
    w = synth.synth_weights(0, vgg_weight_shapes(300, 20), bias_scale=0.02)
    w['conv4_3_norm/gamma'] = np.full((512,), 20.0, np.float32)
    m.set_weights(w)
    return m


def parse(root, load_images_into_memory):
    from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator
    dataset = DataGenerator(load_images_into_memory=load_images_into_memory)
    dataset.parse_xml(images_dirs=[os.path.join(root, 'JPEGImages')], image_set_filenames=[os.path.join(root, 'ImageSets', 'Main', 'test.txt')],
                      annotations_dirs=[os.path.join(root, 'Annotations')], classes=CLASSES, include_classes='all',
                      exclude_truncated=False, exclude_difficult=False, ret=False)
    return dataset


def sweep(m, dataset):
    """The notebook's Evaluator call, up to its returned mAP -> (seconds, mAP)."""
    import torch
    from ssd_keras_b200.eval_utils.average_precision_evaluator import Evaluator
    torch.cuda.synchronize()
    t = time.perf_counter()
    evaluator = Evaluator(model=m, n_classes=20, data_generator=dataset, model_mode='inference')
    with contextlib.redirect_stdout(io.StringIO()):
        results = evaluator(img_height=300, img_width=300, batch_size=8, data_generator_mode='resize', round_confidences=False,
                            matching_iou_threshold=0.5, border_pixels='include', sorting_algorithm='quicksort',
                            average_precision_mode='sample', num_recall_points=11, ignore_neutral_boxes=True, return_precisions=True,
                            return_recalls=True, return_average_precisions=True, verbose=False)
    torch.cuda.synchronize()
    return time.perf_counter() - t, float(results[0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=4952, help='images in the set (VOC2007 test has 4952)')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), 'needs a CUDA device'
    import __graft_entry__ as entry
    entry.build()
    n = args.images
    res = {'images': n, 'card': card()}
    with tempfile.TemporaryDirectory() as tmp:
        write_dataset(tmp, n)
        t = time.perf_counter()
        files = parse(tmp, False)
        res['parse_xml_s'] = time.perf_counter() - t
        m = model()
        warm = parse(tmp, False)
        for attr in ('filenames', 'labels', 'image_ids', 'eval_neutral'):
            setattr(warm, attr, getattr(warm, attr)[:32])
        warm.dataset_size, warm.dataset_indices = 32, warm.dataset_indices[:32]
        sweep(m, warm)                                               # module loads, plans and every batch shape once
        s, res['map_files'] = sweep(m, files)
        res['sweep_files_img_per_s'] = n / s
        t = time.perf_counter()
        memory = parse(tmp, True)
        res['parse_xml_and_decode_into_memory_s'] = time.perf_counter() - t
        s, res['map_memory'] = sweep(m, memory)
        res['sweep_memory_img_per_s'] = n / s
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'time_voc_evaluation.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
