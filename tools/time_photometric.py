#!/usr/bin/env python
"""Time the photometric pre-pass of ssdk_assemble_images at B=32 on VOC-like images (333-500 x 375-500, uint8 RGB).

  kernel      photometric_kernel alone: CUDA events around `--iters` calls of ssdk_assemble_images with and without the
              photometric prefix on sources already on the device, alternating; the difference of the two per-call times is the
              pre-pass (the assembly kernel runs in both).  Algorithmic bytes: 3 read + 3 written per source pixel, over that
              time, and the rate's share of the H100 SXM's 3.35 TB/s data-sheet bandwidth.
  call        the whole `assemble_images_device` call (host packing, upload, launches; synchronised) with and without the
              prefix, alternating, for the SSD300 chain (expand -> crop -> flip -> resize to 300x300) and the SSD7 chain
              (translate -> scale -> flip at 300x480).
  host        with cv2 importable: the same photometric sequences with the reference's NumPy + cv2 arithmetic on the host.

Prints the card's name and power limit with every record (one JSON line each); fails without a GPU."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), '..')))

HBM_PEAK = 3.35e12
MEAN = (123, 117, 104)


def chains(rng, B, kind):
    """(images, photometric op lists, geometric op lists, output size)"""
    from ssd_keras_b200.data_generator import batch_assembly as ba
    images, photo, geo = [], [], []
    for b in range(B):
        h, w = (300, 480) if kind == 'ssd7' else (int(rng.integers(333, 501)), int(rng.integers(375, 501)))
        images.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        draw = lambda lo, hi: float(rng.uniform(lo, hi)) if rng.random() < 0.5 else None      # noqa: E731
        photo.append(ba.photometric_ops(1 + b % 2, brightness=draw(-32, 32), contrast=draw(0.5, 1.5), saturation=draw(0.5, 1.5),
                                        hue=draw(-18, 18)))
        if kind == 'ssd7':
            lst = [ba.translate(h, w, rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3))] if rng.random() < 0.5 else []
            lst += [ba.scale(h, w, rng.uniform(0.5, 2.0))] if rng.random() < 0.5 else []
            geo.append(lst + ([ba.flip(w)] if rng.random() < 0.5 else []))
            continue
        r = rng.uniform(1, 4)
        ph, pw = int(h * r), int(w * r)
        lst = [ba.crop_pad(-int(rng.integers(0, ph - h + 1)), -int(rng.integers(0, pw - w + 1)), ph, pw, clip_boxes=False, background=MEAN)]
        ch, cw = max(1, int(ph * rng.uniform(0.3, 1))), max(1, int(pw * rng.uniform(0.3, 1)))
        lst.append(ba.crop_pad(int(rng.integers(0, ph - ch + 1)), int(rng.integers(0, pw - cw + 1)), ch, cw, center_point_filter=True))
        geo.append(lst + ([ba.flip(cw)] if b % 2 else []) + [ba.resize(ch, cw, 300, 300, interpolation_mode=b % 2)])
    return images, photo, geo, ((300, 480) if kind == 'ssd7' else (300, 300))


def host_photometric(images, photo, cv2):
    """The reference's arithmetic per image: float32 NumPy steps and uint8 cv2.cvtColor."""
    from ssd_keras_b200 import _ffi
    out = []
    for img, lst in zip(images, photo):
        x = img
        for o in lst:
            if o[0] == _ffi.BOXOP_TO_FLOAT32:
                x = x.astype(np.float32)
            elif o[0] == _ffi.BOXOP_TO_UINT8:
                x = np.round(x, decimals=0).astype(np.uint8)
            elif o[0] == _ffi.BOXOP_BRIGHTNESS:
                x = np.clip(x + o[2], 0, 255)
            elif o[0] == _ffi.BOXOP_CONTRAST:
                x = np.clip(127.5 + o[2] * (x - 127.5), 0, 255)
            elif o[0] == _ffi.BOXOP_SATURATION:
                x[:, :, 1] = np.clip(x[:, :, 1] * o[2], 0, 255)
            elif o[0] == _ffi.BOXOP_HUE:
                x[:, :, 0] = (x[:, :, 0] + o[2]) % 180.0
            elif o[0] == _ffi.BOXOP_RGB2HSV:
                x = cv2.cvtColor(x, cv2.COLOR_RGB2HSV)
            elif o[0] == _ffi.BOXOP_HSV2RGB:
                x = cv2.cvtColor(x, cv2.COLOR_HSV2RGB)
        out.append(x)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--host-iters', type=int, default=3)
    args = ap.parse_args()
    import torch
    from ssd_keras_b200 import _ffi
    from ssd_keras_b200.data_generator.batch_assembly import _pack_ops, assemble_images_device
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: nothing to time')
    try:
        smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                      # noqa: BLE001
        smi = 'nvidia-smi unavailable (%s)' % e
    try:
        import cv2
    except ImportError:
        cv2 = None
        print('cv2 is not importable: the host sequences are not timed')
    B = args.batch
    rng = np.random.default_rng(2026)
    L, ctx, stream = _ffi.lib(), _ffi.context(), _ffi.stream_ptr()
    for kind in ('ssd', 'ssd7'):
        images, photo, geo, (oh, ow) = chains(rng, B, kind)
        offs = np.concatenate([[0], np.cumsum([im.size for im in images])]).astype(np.int64)
        hwc = np.asarray([im.shape for im in images], np.int32)
        src = torch.from_numpy(np.concatenate([im.reshape(-1) for im in images])).cuda()
        out = torch.empty((B, oh, ow, 3), dtype=torch.float32, device='cuda')
        lists = {'plain': geo, 'photo': [p + g for p, g in zip(photo, geo)]}
        packed = {k: _pack_ops(v, B) for k, v in lists.items()}

        def launches(which, n):
            arr, max_ops = packed[which]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                _ffi.check(L.ssdk_assemble_images(ctx, _ffi.dptr(src), _ffi.np_ptr(offs, C.c_longlong), _ffi.np_ptr(hwc, C.c_int), B, arr,
                                                  max_ops, oh, ow, _ffi.dptr(out), stream))
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / n

        def calls(which, n):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(n):
                assemble_images_device(images, lists[which], oh, ow, out=out)
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3 / n

        for which in lists:
            launches(which, 20)
            calls(which, 3)
        dev = {k: [] for k in lists}
        call = {k: [] for k in lists}
        for _ in range(args.rounds):                              # alternating, so that both see the same machine
            for which in lists:
                dev[which].append(launches(which, args.iters))
                call[which].append(calls(which, max(5, args.iters // 20)))
        med = lambda v: float(np.median(v))                        # noqa: E731
        pre_ms = med(dev['photo']) - med(dev['plain'])
        nbytes = 6 * sum(im.shape[0] * im.shape[1] for im in images)
        rec = dict(chain=kind, batch=B, gpu=smi, source_pixels=nbytes // 6,
                   assemble_only_device_ms=round(med(dev['plain']), 4), with_photometric_device_ms=round(med(dev['photo']), 4),
                   photometric_kernel_ms=round(pre_ms, 4), device_ms_spread=[round(min(dev['photo']), 4), round(max(dev['photo']), 4)],
                   photometric_algorithmic_bytes=nbytes, photometric_gbps=round(nbytes / pre_ms / 1e6, 1),
                   hbm_fraction=round(nbytes / (pre_ms * 1e-3) / HBM_PEAK, 3),
                   call_ms_plain=round(med(call['plain']), 3), call_ms_with_photometric=round(med(call['photo']), 3))
        if cv2 is not None:
            t0 = time.perf_counter()
            for _ in range(args.host_iters):
                host_photometric(images, photo, cv2)
            rec['host_numpy_cv2_photometric_ms'] = round((time.perf_counter() - t0) * 1e3 / args.host_iters, 2)
            rec['host_threads'] = cv2.getNumThreads()
        print(json.dumps(rec))


if __name__ == '__main__':
    main()
