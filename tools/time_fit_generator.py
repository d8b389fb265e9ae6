#!/usr/bin/env python
"""Time training on generate()'s batches: a serial train_on_batch loop (pull a batch, train, read the loss, then the next
batch) against fit_generator, which pulls batch i+1 while step i runs.

  python tools/time_fit_generator.py [--out DIR] [--steps N] [--rounds R]

Workloads:
  - ssd7_memory: the SSD7 notebook's chain (DataAugmentationConstantInputSize) at B=16, 300x480, images in memory, Adam;
  - ssd7_png:    the same from PNG files, decoded with PIL on the generator's thread pool;
  - ssd300_memory: SSD300 with SSDDataAugmentation at B=32, VOC-sized images in memory, SGD.
Each workload runs R rounds of N steps of each loop, alternating, after a warm-up.  CUDA events recorded on the stream before
and after each step's enqueue give, per loop:
  - ms per step: the median time from the end of one step's kernels to the end of the next one's;
  - GPU idle between steps: the median time from the end of one step's kernels to the start of the next one's (it includes
    the next batch's assembly kernels, about 0.1 ms, and is the host's planning time the loop leaves exposed);
and the host wall time per step of the whole run.  Prints the card's name and power limit with the numbers, and writes them
as JSON to DIR/time_fit_generator.json when --out is given."""
import argparse
import json
import os
import random
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import time_data_generator as tdg                                    # noqa: E402  (voc_like images)
import time_ssd7_generator as t7                                     # noqa: E402  (the SSD7 notebook's chain and frames)


class StepEvents:
    """Wraps a model's step enqueue: an event before it and one after it on the current stream."""

    def __init__(self, model):
        import torch
        self.torch, self.starts, self.ends = torch, [], []
        enqueue = model._enqueue_train_step

        def timed(x, y):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            loss = enqueue(x, y)
            e.record()
            self.starts.append(s)
            self.ends.append(e)
            return loss
        model._enqueue_train_step = timed

    def take(self):
        """(step periods, idle gaps) in ms of the steps recorded since the last call."""
        self.torch.cuda.synchronize()
        s, e = self.starts, self.ends
        self.starts, self.ends = [], []
        period = [e[i - 1].elapsed_time(e[i]) for i in range(1, len(e))]
        idle = [e[i - 1].elapsed_time(s[i]) for i in range(1, len(e))]
        return period, idle


def run_serial(model, it, steps):
    for _ in range(steps):
        x, y = next(it)[:2]
        model.train_on_batch(x, y)


def run_fit(model, it, steps):
    model.fit_generator(it, steps_per_epoch=steps, epochs=1)


def measure(model, it, steps, rounds):
    ev = StepEvents(model)
    run_fit(model, it, 6)                                           # warm-up: plans, trainer, encoder, pinned buffers
    run_serial(model, it, 4)
    ev.take()
    out = {name: {'period': [], 'idle': [], 'wall': []} for name in ('serial', 'fit_generator')}
    for _ in range(rounds):
        for name, fn in (('serial', run_serial), ('fit_generator', run_fit)):
            t = time.perf_counter()
            fn(model, it, steps)
            ev.torch.cuda.synchronize()
            out[name]['wall'].append((time.perf_counter() - t) * 1e3 / steps)
            period, idle = ev.take()
            out[name]['period'] += period
            out[name]['idle'] += idle
    res = {}
    for name, d in out.items():
        res[name] = {'ms_per_step': float(np.median(d['period'])), 'gpu_idle_ms_between_steps': float(np.median(d['idle'])),
                     'wall_ms_per_step': float(np.median(d['wall'])), 'steps_timed': len(d['period'])}
    res['speedup'] = res['serial']['ms_per_step'] / res['fit_generator']['ms_per_step']
    return res


def ssd7(files):
    from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator
    from ssd_keras_b200.keras_loss_function.keras_ssd_loss import SSDLoss
    from ssd_keras_b200.models.keras_ssd7 import build_model
    from ssd_keras_b200.optimizers import Adam
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    H, W = t7.H, t7.W
    model, sizes = build_model((H, W, 3), t7.N_CLASSES, mode='training', l2_regularization=0.0005, scales=t7.SCALES,
                               aspect_ratios_global=t7.ARS, two_boxes_for_ar1=True, variances=[1.0, 1.0, 1.0, 1.0], normalize_coords=True,
                               subtract_mean=127.5, divide_by_stddev=127.5, return_predictor_sizes=True)
    model.compile(optimizer=Adam(lr=0.001), loss=SSDLoss(neg_pos_ratio=3, alpha=1.0).compute_loss)
    enc = SSDInputEncoder(img_height=H, img_width=W, n_classes=t7.N_CLASSES, predictor_sizes=sizes, scales=t7.SCALES,
                          aspect_ratios_global=t7.ARS, two_boxes_for_ar1=True, clip_boxes=False, variances=[1.0, 1.0, 1.0, 1.0],
                          matching_type='multi', pos_iou_threshold=0.5, neg_iou_limit=0.3, normalize_coords=True)
    images, labels = t7.traffic_like(t7.N_IMAGES)
    if files is None:
        data = DataGenerator(filenames=['%d' % i for i in range(len(images))], labels=[l.copy() for l in labels])
        data.images = images
    else:
        from PIL import Image
        names = []
        for i, im in enumerate(images):
            names.append(os.path.join(files, '%d.png' % i))
            Image.fromarray(im).save(names[-1])
        data = DataGenerator(filenames=names, labels=[l.copy() for l in labels])
    it = data.generate(batch_size=t7.B, shuffle=True, transformations=[t7.chain()], label_encoder=enc,
                       returns={'processed_images', 'encoded_labels'}, keep_images_without_gt=True)
    return model, it


def ssd300():
    from oracle import synth
    from oracle.model import SSD300_AR, vgg_weight_shapes
    from ssd_keras_b200.data_generator.data_augmentation_chain_original_ssd import SSDDataAugmentation
    from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator
    from ssd_keras_b200.keras_loss_function.keras_ssd_loss import SSDLoss
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    from ssd_keras_b200.optimizers import SGD
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    scales = [0.1, 0.2, 0.37, 0.54, 0.71, 0.88, 1.05]
    model = ssd_300((300, 300, 3), 20, mode='training', l2_regularization=0.0005, scales=scales, subtract_mean=[123, 117, 104],
                    swap_channels=[2, 1, 0])
    model.set_weights(synth.synth_weights(0, vgg_weight_shapes(300, 20), bias_scale=0.02))
    model.compile(optimizer=SGD(lr=1e-4, momentum=0.9), loss=SSDLoss(neg_pos_ratio=3, alpha=1.0).compute_loss)
    enc = SSDInputEncoder(img_height=300, img_width=300, n_classes=20, predictor_sizes=model.predictor_sizes, scales=scales,
                          aspect_ratios_per_layer=SSD300_AR, two_boxes_for_ar1=True, steps=[8, 16, 32, 64, 100, 300], offsets=[0.5] * 6,
                          clip_boxes=False, variances=[0.1, 0.1, 0.2, 0.2], matching_type='multi', pos_iou_threshold=0.5,
                          neg_iou_limit=0.5, normalize_coords=True)
    images, labels = tdg.voc_like(tdg.N_IMAGES)
    data = DataGenerator(filenames=['%d' % i for i in range(len(images))], labels=[l.copy() for l in labels])
    data.images = images
    it = data.generate(batch_size=tdg.B, shuffle=True, transformations=[SSDDataAugmentation(300, 300)], label_encoder=enc,
                       returns={'processed_images', 'encoded_labels'})
    return model, it


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--rounds', type=int, default=2)
    args = ap.parse_args()
    import __graft_entry__ as entry
    entry.build()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('time_fit_generator.py needs a CUDA device')
    np.random.seed(1)
    random.seed(1)
    res = {'card': t7.card(), 'steps': args.steps, 'rounds': args.rounds}
    res['ssd7_memory'] = dict(batch=t7.B, height=t7.H, width=t7.W, **measure(*ssd7(None), args.steps, args.rounds))
    print(json.dumps(res, indent=1), flush=True)
    with tempfile.TemporaryDirectory() as d:
        res['ssd7_png'] = dict(batch=t7.B, height=t7.H, width=t7.W, **measure(*ssd7(d), args.steps, args.rounds))
    print(json.dumps(res['ssd7_png'], indent=1), flush=True)
    res['ssd300_memory'] = dict(batch=tdg.B, height=300, width=300, **measure(*ssd300(), max(args.steps // 2, 8), args.rounds))
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'time_fit_generator.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
