#!/usr/bin/env python
"""Time the reference evaluation notebook's call on a synthetic VOC07-sized dataset: ``Evaluator(model, 20, dg)(img_height=300,
img_width=300, batch_size=8, data_generator_mode=...)`` with SSD300 ('inference' mode, seeded weights, inputs normalised as in
bench.py so that the boxes stay finite), over 4952 seeded images of VOC-like sizes, from memory and from JPEG files written to
the output directory.  Prints images/s end to end and the split predict / match / AP, and, in the same run, the host path a
user has without the device chain: cv2.resize on the host, then the same-size path and its Python loops.  Prints the GPU name
and power limit.  Needs a GPU.

    python tools/time_evaluate.py [--images 4952] [--out DIR (default: a temporary directory)]"""
import argparse
import os
import subprocess
import sys
import tempfile
import time
import types

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)

VOC_SIZES = [(375, 500), (500, 375), (333, 500), (500, 333), (281, 500), (500, 500), (366, 500), (375, 499), (335, 500), (480, 640)]


def gpu_info():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                   # noqa: BLE001
        return 'nvidia-smi unavailable (%s)' % e


def dataset(n, seed=0):
    rng = np.random.default_rng(seed)
    imgs, labels = [], []
    for i in range(n):
        h, w = VOC_SIZES[int(rng.integers(0, len(VOC_SIZES)))]
        # smooth content: a small random image upsampled, cheap to make and to compress
        small = rng.integers(0, 256, (h // 25 + 1, w // 25 + 1, 3), dtype=np.uint8)
        imgs.append(np.ascontiguousarray(np.repeat(np.repeat(small, 25, 0), 25, 1)[:h, :w]))
        k = int(rng.integers(1, 4))
        x0 = rng.integers(0, w - 60, k); y0 = rng.integers(0, h - 60, k)
        labels.append(np.stack([rng.integers(1, 21, k), x0, y0, x0 + rng.integers(20, 60, k), y0 + rng.integers(20, 60, k)], 1).astype(np.float64))
    return imgs, labels


def ssd300():
    from oracle import synth
    from oracle.model import vgg_weight_shapes
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    model = ssd_300((300, 300, 3), 20, mode='inference', scales=[0.1, 0.2, 0.37, 0.54, 0.71, 0.88, 1.05], divide_by_stddev=[127.5] * 3)
    w = synth.synth_weights(1, vgg_weight_shapes(300, 20), bias_scale=0.0)
    w['conv4_3_norm/gamma'] = np.full((512,), 20.0, np.float32)
    model.set_weights(w)
    return model


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t


def run_device(model, dg, mode):
    from ssd_keras_b200.eval_utils.average_precision_evaluator import Evaluator
    ev = Evaluator(model, 20, dg)
    np.random.seed(0)
    _, tp = timed(lambda: ev.predict_on_dataset(300, 300, 8, data_generator_mode=mode, verbose=False))
    _, tm = timed(lambda: (ev.get_num_gt_per_class(), ev.match_predictions(verbose=False)))
    mAP, ta = timed(lambda: (ev.compute_precision_recall(verbose=False), ev.compute_average_precisions(verbose=False),
                             ev.compute_mean_average_precision())[-1])
    return ev, mAP, tp, tm, ta


def run_host(model, imgs, labels):
    """Today's path without the device chain: cv2.resize on the host, then the same-size path and its loops."""
    import cv2
    from ssd_keras_b200.eval_utils.average_precision_evaluator import Evaluator

    def prep():
        out = []
        for im in imgs:
            out.append(cv2.resize(im, (300, 300), interpolation=cv2.INTER_LINEAR))
        return out
    small, t_resize = timed(prep)
    ev = Evaluator(model, 20, types.SimpleNamespace(images=small, image_ids=list(range(len(imgs))), labels=labels, eval_neutral=None))
    _, tp = timed(lambda: ev.predict_on_dataset(300, 300, 8, verbose=False))
    _, tm = timed(lambda: (ev.get_num_gt_per_class(), ev.match_predictions(verbose=False)))
    _, ta = timed(lambda: (ev.compute_precision_recall(verbose=False), ev.compute_average_precisions(verbose=False)))
    return t_resize, tp, tm, ta


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=4952)
    ap.add_argument('--out', default=None, help='where the JPEG files go')
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('time_evaluate.py needs a GPU')
    import __graft_entry__ as entry
    entry.build()
    a.out = a.out or tempfile.mkdtemp(prefix='time_evaluate_')
    os.makedirs(a.out, exist_ok=True)
    print('gpu:', gpu_info())
    imgs, labels = dataset(a.images)
    files = []
    from PIL import Image
    for i, im in enumerate(imgs):
        f = os.path.join(a.out, '%06d.jpg' % i)
        Image.fromarray(im).save(f, quality=90)
        files.append(f)
    model = ssd300()
    n = len(imgs)
    # warm-up: every shape of the timed window
    warm = types.SimpleNamespace(images=imgs[:16], image_ids=list(range(16)), labels=labels[:16], eval_neutral=None)
    for mode in ('resize', 'pad'):
        run_device(model, warm, mode)
    for src in ('memory', 'jpeg'):
        for mode in ('resize', 'pad'):
            dg = types.SimpleNamespace(images=imgs if src == 'memory' else None, filenames=None if src == 'memory' else files,
                                       image_ids=list(range(n)), labels=labels, eval_neutral=None)
            ev, mAP, tp, tm, ta = run_device(model, dg, mode)
            tot = tp + tm + ta
            print('device  %-6s %-6s: %7.1f images/s end to end (%.3f s: predict %.3f, match %.3f, AP %.3f), %d detections, mAP %.6f'
                  % (src, mode, n / tot, tot, tp, tm, ta, len(ev._detections), mAP))
    t_resize, tp, tm, ta = run_host(model, imgs, labels)
    tot = t_resize + tp + tm + ta
    print('host    memory resize: %7.1f images/s end to end (%.3f s: cv2.resize %.3f, predict + tuple loop %.3f, match + '
          'flattening loop %.3f, AP %.3f)' % (n / tot, tot, t_resize, tp, tm, ta))
    print('gpu:', gpu_info())


if __name__ == '__main__':
    main()
