#!/usr/bin/env python
"""Time histogram equalisation in ssdk_assemble_images at B=32 on VOC-sized images (333-500 x 375-500, uint8 RGB).

CUDA events around `--iters` calls of ssdk_assemble_images on sources already on the device, three op lists alternating:
``plain`` (resize to 300 x 300), ``hsv`` (RGB -> HSV -> RGB, then the resize: one photometric pass) and ``equalize``
(RGB -> HSV, EQUALIZE_V, HSV -> RGB, then the resize: two passes with the histogram and table kernels between them).  The
per-call device time of each, the cost of the equalisation (equalize - hsv) and the spread over `--rounds`; prints the card's
name and power limit with the record (one JSON line); fails without a GPU."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), '..')))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    import torch
    from ssd_keras_b200 import _ffi
    from ssd_keras_b200.data_generator import batch_assembly as ba
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: nothing to time')
    try:
        smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                      # noqa: BLE001
        smi = 'nvidia-smi unavailable (%s)' % e
    B = args.batch
    rng = np.random.default_rng(2026)
    images = [rng.integers(0, 256, (int(rng.integers(333, 501)), int(rng.integers(375, 501)), 3), dtype=np.uint8) for _ in range(B)]
    geo = [[ba.resize(im.shape[0], im.shape[1], 300, 300)] for im in images]
    hsv, rgb = ba.convert_color('RGB', 'HSV'), ba.convert_color('HSV', 'RGB')
    lists = {'plain': geo, 'hsv': [[hsv, rgb] + g for g in geo], 'equalize': [[hsv, ba.equalize_hist(), rgb] + g for g in geo]}
    L, ctx, stream = _ffi.lib(), _ffi.context(), _ffi.stream_ptr()
    offs = np.concatenate([[0], np.cumsum([im.size for im in images])]).astype(np.int64)
    hwc = np.asarray([im.shape for im in images], np.int32)
    src = torch.from_numpy(np.concatenate([im.reshape(-1) for im in images])).cuda()
    out = torch.empty((B, 300, 300, 3), dtype=torch.float32, device='cuda')
    packed = {k: ba._pack_ops(v, B) for k, v in lists.items()}

    def launches(which, n):
        arr, max_ops = packed[which]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            _ffi.check(L.ssdk_assemble_images(ctx, _ffi.dptr(src), _ffi.np_ptr(offs, C.c_longlong), _ffi.np_ptr(hwc, C.c_int), B, arr,
                                              max_ops, 300, 300, _ffi.dptr(out), stream))
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    for which in lists:
        launches(which, 20)
    ms = {k: [] for k in lists}
    for _ in range(args.rounds):                              # alternating, so that all three see the same machine
        for which in lists:
            ms[which].append(launches(which, args.iters))
    med = {k: float(np.median(v)) for k, v in ms.items()}
    n_px = int(sum(im.shape[0] * im.shape[1] for im in images))
    print(json.dumps(dict(card=smi, batch=B, source_pixels=n_px, output='300x300', iters=args.iters, rounds=args.rounds,
                          ms_per_call={k: round(v, 4) for k, v in med.items()},
                          spread_ms={k: round(float(np.max(v) - np.min(v)), 4) for k, v in ms.items()},
                          equalize_ms=round(med['equalize'] - med['hsv'], 4))))


if __name__ == '__main__':
    main()
