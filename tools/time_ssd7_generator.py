#!/usr/bin/env python
"""Time the SSD7 notebook's input pipeline: DataGenerator.generate with DataAugmentationConstantInputSize (the notebook's chain
arguments) at B=16, 300x480, against the SSD7 training step it feeds.

  python tools/time_ssd7_generator.py [--out DIR] [--batches N]

Prints the card's name and power limit, then:
  - the host planner alone (shuffle, slices and every draw of the chain, validators included), ms per batch;
  - batches per second of generate() with the encoder, from memory and from PNG files (PIL on the thread pool);
  - the device assembly of one batch (images, boxes and encoder: assemble_training_batch), as the summed device time of its
    kernels (torch.profiler, median over the timed calls) and as host wall time up to a synchronise;
  - the SSD7 training step at the same batch (train_on_batch up to a synchronise, median), for comparison.
Writes the numbers as JSON to DIR/time_ssd7_generator.json when --out is given."""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
B, H, W, N_CLASSES, N_IMAGES = 16, 300, 480, 5, 160
SCALES, ARS = [0.08, 0.16, 0.32, 0.64, 0.96], [0.5, 1.0, 2.0]
CHAIN_ARGS = dict(random_brightness=(-48, 48, 0.5), random_contrast=(0.5, 1.8, 0.5), random_saturation=(0.5, 1.8, 0.5),
                  random_hue=(18, 0.5), random_flip=0.5, random_translate=((0.03, 0.5), (0.03, 0.5), 0.5), random_scale=(0.5, 2.0, 0.5),
                  n_trials_max=3, clip_boxes=True, overlap_criterion='area', bounds_box_filter=(0.3, 1.0), bounds_validator=(0.5, 1.0),
                  n_boxes_min=1, background=(0, 0, 0))


def traffic_like(n, seed=0):
    """Udacity-traffic-sized frames (300 x 480) with 1-8 boxes of 5 classes, int64 labels as parse_csv gives them."""
    rng = np.random.default_rng(seed)
    images, labels = [], []
    for _ in range(n):
        base = rng.integers(0, 256, (H // 16 + 2, W // 16 + 2, 3), dtype=np.uint8)
        images.append(np.ascontiguousarray(np.repeat(np.repeat(base, 16, 0), 16, 1)[:H, :W]))
        k = int(rng.integers(1, 9))
        x0, y0 = rng.integers(0, W - 60, k), rng.integers(0, H - 60, k)
        labels.append(np.stack([rng.integers(1, N_CLASSES + 1, k), x0, y0, x0 + rng.integers(8, 60, k), y0 + rng.integers(8, 60, k)], 1))
    return images, labels


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:                                           # noqa: BLE001
        return 'unknown (%s)' % e


def chain():
    from ssd_keras_b200.data_generator.data_augmentation_chain_constant_input_size import DataAugmentationConstantInputSize
    return DataAugmentationConstantInputSize(**CHAIN_ARGS)


def planner_ms(gen, n_batches):
    np.random.seed(3)
    random.seed(3)
    it = gen.plan_batches(B, True, [chain()], False)
    t = time.perf_counter()
    for _ in range(n_batches):
        next(it)
    return (time.perf_counter() - t) / n_batches * 1e3


def generate_rate(gen, n_batches, encoder):
    import torch
    np.random.seed(2)
    random.seed(2)
    it = gen.generate(batch_size=B, shuffle=True, transformations=[chain()], label_encoder=encoder, returns={'processed_images', 'encoded_labels'})
    for _ in range(2):
        next(it)
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(n_batches):
        next(it)
    torch.cuda.synchronize()
    return n_batches / (time.perf_counter() - t)


def assembly_ms(gen, encoder, reps=40):
    """Device time (summed kernels per call) and wall time of assemble_training_batch on planned batches."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from ssd_keras_b200.data_generator import batch_assembly as ba
    np.random.seed(4)
    random.seed(4)
    it = gen.plan_batches(B, True, [chain()], False)
    batches = []
    for _ in range(8):
        b = next(it)
        batches.append(([b['images'][i] for i in b['keep']], [b['labels'][i] for i in b['keep']], b['ops']))
    for x, y, o in batches:
        ba.assemble_training_batch(encoder, x, y, o, H, W)
    torch.cuda.synchronize()
    wall = []
    for r in range(reps):
        x, y, o = batches[r % len(batches)]
        t = time.perf_counter()
        ba.assemble_training_batch(encoder, x, y, o, H, W)
        torch.cuda.synchronize()
        wall.append(time.perf_counter() - t)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for r in range(reps):
            x, y, o = batches[r % len(batches)]
            ba.assemble_training_batch(encoder, x, y, o, H, W)
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.events():
        if e.device_time > 0 and 'Memcpy' not in e.name and 'Memset' not in e.name:
            kernels.setdefault(e.name, []).append(e.device_time)
    per_call = sum(float(np.sum(v)) for v in kernels.values()) / reps / 1000.0
    names = {k: float(np.median(v)) / 1000.0 for k, v in kernels.items()}
    return per_call, float(np.median(wall)) * 1e3, names


def train_step_ms(model, gen, encoder, steps=30):
    import torch
    np.random.seed(5)
    random.seed(5)
    it = gen.generate(batch_size=B, shuffle=True, transformations=[chain()], label_encoder=encoder, returns={'processed_images', 'encoded_labels'})
    batches = [next(it) for _ in range(4)]
    for x, y in batches:
        model.train_on_batch(x, y)
    torch.cuda.synchronize()
    times = []
    for s in range(steps):
        x, y = batches[s % len(batches)]
        t = time.perf_counter()
        model.train_on_batch(x, y)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t)
    return float(np.median(times)) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--batches', type=int, default=20)
    args = ap.parse_args()
    import __graft_entry__ as entry
    entry.build()
    from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator
    from ssd_keras_b200.keras_loss_function.keras_ssd_loss import SSDLoss
    from ssd_keras_b200.models.keras_ssd7 import build_model
    from ssd_keras_b200.optimizers import Adam
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    images, labels = traffic_like(N_IMAGES)
    res = {'batch': B, 'height': H, 'width': W, 'images': 'synthetic %dx%d frames, 1-8 boxes' % (H, W), 'card': card()}
    model, predictor_sizes = build_model((H, W, 3), N_CLASSES, mode='training', l2_regularization=0.0005, scales=SCALES,
                                         aspect_ratios_global=ARS, two_boxes_for_ar1=True, variances=[1.0, 1.0, 1.0, 1.0],
                                         normalize_coords=True, subtract_mean=127.5, divide_by_stddev=127.5, return_predictor_sizes=True)
    model.compile(optimizer=Adam(lr=0.001), loss=SSDLoss(neg_pos_ratio=3, alpha=1.0).compute_loss)
    encoder = SSDInputEncoder(img_height=H, img_width=W, n_classes=N_CLASSES, predictor_sizes=predictor_sizes, scales=SCALES,
                              aspect_ratios_global=ARS, two_boxes_for_ar1=True, steps=None, offsets=None, clip_boxes=False,
                              variances=[1.0, 1.0, 1.0, 1.0], matching_type='multi', pos_iou_threshold=0.5, neg_iou_limit=0.3,
                              normalize_coords=True)
    mem = DataGenerator(filenames=['%d' % i for i in range(N_IMAGES)], labels=[l.copy() for l in labels])
    mem.images = images
    res['host_planner_ms_per_batch'] = planner_ms(mem, args.batches)
    res['generate_memory_batches_per_s'] = generate_rate(mem, args.batches, encoder)
    with tempfile.TemporaryDirectory() as d:
        from PIL import Image
        files = []
        for i, im in enumerate(images):
            files.append(os.path.join(d, '%d.png' % i))
            Image.fromarray(im).save(files[-1])
        png = DataGenerator(filenames=files, labels=[l.copy() for l in labels])
        res['generate_png_batches_per_s'] = generate_rate(png, args.batches, encoder)
    res['assembly_device_ms'], res['assembly_wall_ms'], res['assembly_kernels_ms'] = assembly_ms(mem, encoder)
    res['train_step_ms'] = train_step_ms(model, mem, encoder)
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'time_ssd7_generator.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
