#!/usr/bin/env python
"""Time COCOeval for iouType 'bbox' (eval_utils/coco_eval.py) on a seeded synthetic val2017-sized set: 5000 images, 80
categories, about 7 ground truths per image of every size with about 1 % crowd, and 200 detections per image jittered from the
ground truths plus noise, scores on a 0.001 grid (ties, as the results file's rounding to 3 decimals gives).

Prints the GPU name and power limit, then, each as the median over the repeats after a warm-up call:
- the kernel times of coco_match_kernel (evaluate) and coco_accumulate_kernel (accumulate), as torch.profiler reports them
  (the device time of each kernel, from a separate profiled run);
- the span of each call on the stream between two CUDA events recorded before and after it (its uploads, sorts, kernel and
  read-back, and any gap while the host packs);
- the whole calls by the host clock, ending in a device synchronise;
and the CPU time of the NumPy restatement (oracle/cocoeval.py, pycocotools' own
per-image loops) on the first --oracle-images images, extrapolated linearly to the whole set and labelled as such.  For scale,
the reference's COCO notebook stores pycocotools' own times on val2017 on its author's machine: 64.15 s for evaluate() and
10.58 s for accumulate().  Needs a GPU: without one it stops with the device error after the oracle part.

    python tools/time_cocoeval.py [--images 5000] [--repeats 5] [--oracle-images 100] [--seed 0]"""
import argparse
import contextlib
import copy
import io
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                   # noqa: BLE001
        return 'nvidia-smi unavailable (%s)' % e


def synthetic(n_images, n_cats=80, gt_per_image=7, det_per_image=200, crowd=0.01, seed=0):
    """(ground-truth dataset, results list), seeded."""
    rng = np.random.default_rng(seed)
    img_ids = np.sort(rng.choice(600000, n_images, replace=False)).tolist()
    cat_ids = [c for c in range(1, 91) if c not in (12, 26, 29, 30, 45, 66, 68, 69, 71, 83)][:n_cats]
    n_gt = rng.poisson(gt_per_image, n_images)
    g_img = np.repeat(np.arange(n_images), n_gt)
    G = len(g_img)
    side = np.exp(rng.uniform(np.log(6), np.log(400), G))                # small, medium and large
    g_wh = np.round(side[:, None] * rng.uniform(.6, 1.4, (G, 2)), 2)
    g_xy = np.round(rng.uniform(0, 640, (G, 2)) - g_wh / 4, 2)
    g_cat = rng.integers(0, n_cats, G)
    g_crowd = rng.random(G) < crowd
    g_area = g_wh[:, 0] * g_wh[:, 1] * rng.uniform(.5, 1.0, G)
    anns = [{'image_id': img_ids[i], 'category_id': cat_ids[c], 'bbox': [x, y, w, h], 'area': float(a), 'iscrowd': int(k), 'id': n + 1}
            for n, (i, c, (x, y), (w, h), a, k) in enumerate(zip(g_img.tolist(), g_cat.tolist(), g_xy.tolist(), g_wh.tolist(),
                                                                  g_area.tolist(), g_crowd.tolist()))]
    gt = {'images': [{'id': i} for i in img_ids], 'categories': [{'id': c, 'name': str(c)} for c in cat_ids], 'annotations': anns}
    D = n_images * det_per_image
    d_img = np.repeat(np.arange(n_images), det_per_image)
    first = np.concatenate([[0], np.cumsum(n_gt)[:-1]])
    from_gt = (rng.random(D) < .5) & (n_gt[d_img] > 0)
    src = first[d_img] + (rng.random(D) * np.maximum(n_gt[d_img], 1)).astype(np.int64)
    src = np.where(from_gt, np.minimum(src, G - 1), 0)
    wh = np.where(from_gt[:, None], g_wh[src] * (1 + rng.normal(0, .1, (D, 2))), rng.uniform(4, 300, (D, 2)))
    xy = np.where(from_gt[:, None], g_xy[src] + rng.normal(0, .08, (D, 2)) * g_wh[src], rng.uniform(0, 600, (D, 2)))
    cat = np.where(from_gt & (rng.random(D) < .85), g_cat[src], rng.integers(0, n_cats, D))
    score = np.round(rng.beta(1.2, 4, D), 3)
    box = np.round(np.concatenate([xy, np.maximum(wh, .5)], 1), 1)
    res = [{'image_id': img_ids[i], 'category_id': cat_ids[c], 'bbox': b, 'score': s}
           for i, c, b, s in zip(d_img.tolist(), cat.tolist(), box.tolist(), score.tolist())]
    return gt, res


def subset(gt, res, n):
    keep = {im['id'] for im in gt['images'][:n]}
    return ({'images': gt['images'][:n], 'categories': gt['categories'],
             'annotations': [a for a in gt['annotations'] if a['image_id'] in keep]},
            [r for r in res if r['image_id'] in keep])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=5000)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--oracle-images', type=int, default=100)
    ap.add_argument('--seed', type=int, default=0)
    args = ap.parse_args()
    gt, res = synthetic(args.images, seed=args.seed)
    print('set: %d images, %d categories, %d ground truths (%d crowd), %d detections'
          % (len(gt['images']), len(gt['categories']), len(gt['annotations']), sum(a['iscrowd'] for a in gt['annotations']), len(res)))

    from oracle import cocoeval as oc
    sg, sr = subset(gt, res, args.oracle_images)
    og = oc.COCO(copy.deepcopy(sg))
    oev = oc.COCOeval(og, og.loadRes(copy.deepcopy(sr)))
    t0 = time.perf_counter()
    oev.evaluate()
    t1 = time.perf_counter()
    oev.accumulate()
    t2 = time.perf_counter()
    scale = len(gt['images']) / len(sg['images'])
    print('oracle (NumPy restatement, CPU) on %d images: evaluate %.2f s, accumulate %.2f s; extrapolated x%.0f to the whole set '
          '(not measured): evaluate ~%.0f s, accumulate ~%.0f s' % (len(sg['images']), t1 - t0, t2 - t1, scale, (t1 - t0) * scale,
                                                                   (t2 - t1) * scale))

    import torch
    if not torch.cuda.is_available():
        raise SystemExit('time_cocoeval.py: no CUDA device; the device timings need an H100')
    import __graft_entry__ as entry
    entry.build()
    from ssd_keras_b200.eval_utils.coco_eval import COCO, COCOeval
    print('gpu:', gpu_info())
    with contextlib.redirect_stdout(io.StringIO()):
        g = COCO()
        g.dataset = gt
        g.createIndex()
        d = g.loadRes(res)

    def run():
        ev = COCOeval(g, d, iouType='bbox')
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        with contextlib.redirect_stdout(io.StringIO()):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            e[0].record()
            ev.evaluate()
            e[1].record()
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            ev.accumulate()
            e[2].record()
            torch.cuda.synchronize()
            t2 = time.perf_counter()
        run.events.append((e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2])))
        return ev, t1 - t0, t2 - t1
    run.events = []

    ev, c0, c1 = run()                                        # warm-up: module load, allocator, the COCO objects' column arrays
    print('first call (columns extracted from the annotation dicts): evaluate() %.3f s, accumulate() %.3f s' % (c0, c1))
    run.events.clear()
    walls = [run()[1:] for _ in range(args.repeats)]
    events = list(run.events)
    kern = {'coco_match_kernel': [], 'coco_accumulate_kernel': []}
    from torch.profiler import ProfilerActivity, profile
    for _ in range(args.repeats):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run()
        for e in prof.key_averages():
            for k in kern:
                if k in e.key:
                    kern[k].append(e.device_time_total / 1e3)
    med = lambda v: statistics.median(v) if v else float('nan')
    print('kernels (torch.profiler device time, median of %d): coco_match_kernel %.3f ms, coco_accumulate_kernel %.3f ms'
          % (args.repeats, med(kern['coco_match_kernel']), med(kern['coco_accumulate_kernel'])))
    print('calls on the stream (CUDA events, median of %d): evaluate() %.3f ms, accumulate() %.3f ms'
          % (args.repeats, med([v[0] for v in events]), med([v[1] for v in events])))
    print('whole call incl. host packing (median of %d): evaluate() %.3f s, accumulate() %.3f s'
          % (args.repeats, med([w[0] for w in walls]), med([w[1] for w in walls])))
    with contextlib.redirect_stdout(io.StringIO()) as buf:
        ev.summarize()
    print('summary of the synthetic set:\n' + buf.getvalue().rstrip())


if __name__ == '__main__':
    main()
