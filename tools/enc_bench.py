#!/usr/bin/env python
"""Encoder timing sweep (one GPU): config 5 (P=1e5, G=128, B=256) and config 3 (SSD300, B=32, G=8) over the tile-set /
tiles-per-CTA knobs.  CUDA events around back-to-back calls into a preallocated output; prints one JSON line per variant."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..')); sys.path.insert(0, ROOT)
import __graft_entry__; __graft_entry__.build()
import bench
from oracle import synth
from oracle.model import SSD300_AR
from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder

peaks, _ = bench._peaks()
hbm = peaks['hbm_gbs']


def run(tag, enc, gdev, offs, ybuf, bytes_, inner, env):
    for k in ('SSDK_ENC_SPATIAL_MIN', 'SSDK_ENC_TPC', 'SSDK_ENC_DEBUG', 'SSDK_ENC_LB_MIN'):
        os.environ.pop(k, None)
    os.environ.update(env)
    ms = bench._time_cuda(lambda: enc.encode_device(gdev, offs, out=ybuf), iters=7, warm=3, inner=inner)
    print(json.dumps({'case': tag, 'env': env, 'ms': round(ms, 5), 'GBps': round(bytes_ / ms / 1e6, 1), 'frac_hbm': round(bytes_ / ms / 1e6 / hbm, 4)}), flush=True)


def main():
    Bm = int(sys.argv[1]) if len(sys.argv) > 1 else 256
    encm = SSDInputEncoder(1000, 1600, 20, [(125, 200)], scales=[0.1, 0.2], aspect_ratios_global=[0.5, 1.0, 2.0], pos_iou_threshold=0.5,
                           neg_iou_limit=0.5)
    gtm = synth.synth_gt(4, Bm, 128, 1600, 1000, 20)
    offm = np.cumsum([0] + [g.shape[0] for g in gtm]).astype(np.int32)
    gm = torch.from_numpy(np.concatenate(gtm)).cuda()
    ybuf = torch.empty((Bm, 100000, 33), dtype=torch.float32, device='cuda')
    bytes_ = Bm * (100000 * 16 + 128 * 20 + 100000 * 4 * 33)
    for env in ({}, {'SSDK_ENC_SPATIAL_MIN': '1000000'}, {'SSDK_ENC_TPC': '1'}, {'SSDK_ENC_TPC': '2'}, {'SSDK_ENC_TPC': '8'},
                {'SSDK_ENC_SPATIAL_MIN': '1000000', 'SSDK_ENC_TPC': '1'}, {'SSDK_ENC_DEBUG': '1'}):
        run('micro_b%d' % Bm, encm, gm, offm, ybuf, bytes_, 1, env)
    # memory-bound floor of the same output: a plain fill of the target tensor
    ms = bench._time_cuda(lambda: ybuf.fill_(1.0), iters=7, warm=2)
    print(json.dumps({'case': 'fill_same_bytes', 'ms': round(ms, 5), 'GBps': round(ybuf.numel() * 4 / ms / 1e6, 1)}), flush=True)
    del ybuf, encm
    ps = [(38, 38), (19, 19), (10, 10), (5, 5), (3, 3), (1, 1)]
    enc = SSDInputEncoder(300, 300, 20, ps, scales=bench.SC300, aspect_ratios_per_layer=SSD300_AR, steps=[8, 16, 32, 64, 100, 300],
                          offsets=[0.5] * 6, pos_iou_threshold=0.5, neg_iou_limit=0.5)
    gt = synth.synth_gt(2, 32, 8, 300, 300, 20)
    offs = np.cumsum([0] + [g.shape[0] for g in gt]).astype(np.int32)
    gdev = torch.from_numpy(np.concatenate(gt)).cuda()
    y300 = torch.empty((32, 8732, 33), dtype=torch.float32, device='cuda')
    b300 = 32 * (8732 * 16 + 8 * 20 + 8732 * 4 * 33)
    for env in ({}, {'SSDK_ENC_SPATIAL_MIN': '0'}, {'SSDK_ENC_TPC': '2'}, {'SSDK_ENC_DEBUG': '1'}):
        run('ssd300_b32', enc, gdev, offs, y300, b300, 50, env)
    ms = bench._time_cuda(lambda: y300.fill_(1.0), iters=7, warm=2, inner=50)
    print(json.dumps({'case': 'fill_same_bytes_ssd300', 'ms': round(ms, 5), 'GBps': round(y300.numel() * 4 / ms / 1e6, 1)}), flush=True)


if __name__ == '__main__':
    main()
