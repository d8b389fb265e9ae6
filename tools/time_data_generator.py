#!/usr/bin/env python
"""Time DataGenerator.generate with SSDDataAugmentation at B=32 -> 300x300 on VOC-sized images (333-500 x 375-500).

  python tools/time_data_generator.py [--out DIR] [--reference PATH]

Prints the card's name and power limit, then:
  - image_assemble_kernel's device time (torch.profiler, median over the timed calls) on the original SSD chain with all five
    interpolation modes drawn, and on the same chain with the modes restricted to nearest / linear, with the algorithmic bytes
    (uint8 source read + float32 batch written) and their share of the 3.35 TB/s data-sheet HBM bandwidth;
  - batches per second of generate() from memory and from JPEG files (PIL on the thread pool), and the host planner alone
    (shuffle, slices and every np.random draw of the chain) and PIL decoding alone, per batch;
  - with --reference, the reference's own host generate() with the same chain and images (run where its tree exists).
Writes the numbers as JSON to DIR/time_data_generator.json when --out is given."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
B, OUT, N_IMAGES = 32, 300, 256
HBM_GBS = 3350.0


def voc_like(n, seed=0):
    rng = np.random.default_rng(seed)
    images, labels = [], []
    for _ in range(n):
        h, w = int(rng.integers(333, 501)), int(rng.integers(375, 501))
        base = rng.integers(0, 256, (h // 16 + 2, w // 16 + 2, 3), dtype=np.uint8)
        images.append(np.ascontiguousarray(np.repeat(np.repeat(base, 16, 0), 16, 1)[:h, :w]))
        k = int(rng.integers(1, 6))
        x0, y0 = rng.integers(0, w - 40, k), rng.integers(0, h - 40, k)
        x1, y1 = x0 + rng.integers(20, 40, k), y0 + rng.integers(20, 40, k)
        labels.append(np.stack([rng.integers(1, 21, k), x0, y0, x1, y1], 1).astype(np.int64))
    return images, labels


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:                                           # noqa: BLE001
        return 'unknown (%s)' % e


def kernel_ms(images, labels, modes, reps=50):
    """Median device time of image_assemble_kernel over ``reps`` assemblies of planned batches."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from ssd_keras_b200.data_generator import batch_assembly as ba
    from ssd_keras_b200.data_generator.data_augmentation_chain_original_ssd import SSDDataAugmentation
    aug = SSDDataAugmentation(OUT, OUT)
    aug.resize.interpolation_modes = modes
    np.random.seed(1)
    batches = []
    for r in range(8):
        idx = np.random.choice(len(images), B, replace=False)
        batches.append(([images[i] for i in idx], [aug.plan(images[i].shape[0], images[i].shape[1], labels[i])[0] for i in idx]))
    out = torch.empty((B, OUT, OUT, 3), dtype=torch.float32, device='cuda')
    for x, o in batches:
        ba.assemble_images_device(x, o, OUT, OUT, out=out)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for r in range(reps):
            x, o = batches[r % len(batches)]
            ba.assemble_images_device(x, o, OUT, OUT, out=out)
        torch.cuda.synchronize()
    times = [e.device_time for e in prof.events() if 'image_assemble_kernel' in e.name]
    src = np.mean([sum(a.nbytes for a in x) for x, _ in batches])
    return float(np.median(times)) / 1000.0, float(src + B * OUT * OUT * 3 * 4), len(times)


def generate_rate(gen, n_batches, label_encoder):
    from ssd_keras_b200.data_generator.data_augmentation_chain_original_ssd import SSDDataAugmentation
    import torch
    np.random.seed(2)
    it = gen.generate(batch_size=B, shuffle=True, transformations=[SSDDataAugmentation(OUT, OUT)], label_encoder=label_encoder,
                      returns={'processed_images', 'encoded_labels'})
    for _ in range(2):
        next(it)
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(n_batches):
        x, y = next(it)
    torch.cuda.synchronize()
    return n_batches / (time.perf_counter() - t)


def host_parts(gen, files, n_batches):
    from ssd_keras_b200.data_generator.data_augmentation_chain_original_ssd import SSDDataAugmentation
    from ssd_keras_b200.eval_utils.dataset_predict import load_image
    np.random.seed(3)
    it = gen.plan_batches(B, True, [SSDDataAugmentation(OUT, OUT)], False)
    t = time.perf_counter()
    for _ in range(n_batches):
        next(it)
    plan = (time.perf_counter() - t) / n_batches
    t = time.perf_counter()
    for f in files[:B]:
        load_image(f)
    return plan, time.perf_counter() - t


def reference_rate(path, images, labels, n_batches):
    sys.path.insert(0, path)
    from data_generator.data_augmentation_chain_original_ssd import SSDDataAugmentation as RefAug
    from data_generator.object_detection_2d_data_generator import DataGenerator as RefGen
    gen = RefGen(filenames=['%d' % i for i in range(len(images))], labels=[l.copy() for l in labels])
    gen.images = images
    np.random.seed(2)
    it = gen.generate(batch_size=B, shuffle=True, transformations=[RefAug(OUT, OUT)], returns={'processed_images', 'processed_labels'})
    next(it)
    t = time.perf_counter()
    for _ in range(n_batches):
        next(it)
    return n_batches / (time.perf_counter() - t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--reference', default=None, help='a reference tree: time its host generate() instead of the device path')
    ap.add_argument('--batches', type=int, default=20)
    args = ap.parse_args()
    images, labels = voc_like(N_IMAGES)
    res = {'batch': B, 'out': OUT, 'images': 'synthetic VOC-sized, 333-500 x 375-500'}
    if args.reference:
        res['reference_generate_batches_per_s'] = reference_rate(args.reference, images, labels, max(2, args.batches // 4))
        print(json.dumps(res))
        return
    import torch
    import __graft_entry__ as entry
    entry.build()
    from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    from oracle.model import SSD300_AR
    res['card'] = card()
    for name, modes in (('all_modes', [0, 1, 2, 3, 4]), ('nearest_linear', [0, 1])):
        ms, nbytes, n = kernel_ms(images, labels, modes)
        res['kernel_ms_' + name] = ms
        res['kernel_bytes_' + name] = nbytes
        res['kernel_share_hbm_' + name] = nbytes / (ms * 1e-3) / (HBM_GBS * 1e9)
    encoder = SSDInputEncoder(img_height=OUT, img_width=OUT, n_classes=20, predictor_sizes=[(38, 38), (19, 19), (10, 10), (5, 5), (3, 3), (1, 1)],
                              scales=[0.1, 0.2, 0.37, 0.54, 0.71, 0.88, 1.05], aspect_ratios_per_layer=SSD300_AR, two_boxes_for_ar1=True,
                              steps=[8, 16, 32, 64, 100, 300], offsets=[0.5] * 6, clip_boxes=False, variances=[0.1, 0.1, 0.2, 0.2],
                              matching_type='multi', pos_iou_threshold=0.5, neg_iou_limit=0.5, normalize_coords=True)
    mem = DataGenerator(filenames=['%d' % i for i in range(N_IMAGES)], labels=[l.copy() for l in labels])
    mem.images = images
    res['generate_memory_batches_per_s'] = generate_rate(mem, args.batches, encoder)
    with tempfile.TemporaryDirectory() as d:
        from PIL import Image
        files = []
        for i, im in enumerate(images):
            files.append(os.path.join(d, '%d.jpg' % i))
            Image.fromarray(im).save(files[-1], quality=90)
        jpg = DataGenerator(filenames=files, labels=[l.copy() for l in labels])
        res['generate_jpeg_batches_per_s'] = generate_rate(jpg, args.batches, encoder)
        res['host_planner_ms_per_batch'], decode = host_parts(mem, files, args.batches)
        res['pil_decode_ms_per_batch_one_thread'] = decode * 1e3
    res['host_planner_ms_per_batch'] *= 1e3
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'time_data_generator.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
