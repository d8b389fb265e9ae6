#!/usr/bin/env python
"""Time ssdk_assemble_images at B=32 on two chains, and the same chains on the host with cv2 for comparison.

  validation  VOC-like sizes around 500x375 -> 300x300, INTER_LINEAR (ConvertTo3Channels -> Resize)
  ssd         the geometric part of the original SSD chain: expand (ratio up to 4, mean colour) -> crop -> flip -> resize,
              alternating INTER_NEAREST and INTER_LINEAR per image
  ssd7        the geometric part of the SSD7 chain (DataAugmentationConstantInputSize) at 300x480: sequence 1 (translate ->
              zoom in -> flip) and sequence 2 (zoom out -> translate -> flip) on alternate images, each step taken with
              probability 0.5 as there, so about half the images are zoomed (cv2.warpAffine)

For each chain: the kernel alone (CUDA events around `--iters` launches on sources already on the device), the whole call
(`assemble_images_device`: host packing into pinned memory, one upload, the launch; synchronised), algorithmic bytes (uint8
source bytes read + float32 bytes written) over kernel time, and that rate's share of the H100 SXM's 3.35 TB/s.  With cv2
importable, the host chain per batch (numpy crop / pad / flip + cv2.resize + float32 stack).  Prints one JSON line per chain."""
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


SIZES = {'validation': (300, 300), 'ssd': (300, 300), 'ssd7': (300, 480)}


def ssd7_chains(rng, B, H, W):
    from ssd_keras_b200.data_generator import batch_assembly as ba
    images, ops = [], []
    for b in range(B):
        images.append(rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
        lst = []
        translate = ba.translate(H, W, rng.uniform(0.03, 0.5) * rng.choice([-1, 1]), rng.uniform(0.03, 0.5) * rng.choice([-1, 1]))
        zoom = ba.scale(H, W, rng.uniform(1.0, 2.0) if b % 2 == 0 else rng.uniform(0.5, 1.0))
        steps = [translate, zoom] if b % 2 == 0 else [zoom, translate]
        lst += [o for o in steps if rng.random() < 0.5]
        if rng.random() < 0.5:
            lst.append(ba.flip(W))
        ops.append(lst)
    return images, ops


def chains(rng, B, kind):
    from ssd_keras_b200.data_generator import batch_assembly as ba
    if kind == 'ssd7':
        return ssd7_chains(rng, B, *SIZES['ssd7'])
    images, ops = [], []
    for b in range(B):
        h, w = int(rng.integers(333, 501)), int(rng.integers(375, 501))
        images.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        if kind == 'validation':
            ops.append([ba.resize(h, w, 300, 300)])
            continue
        lst, ch, cw = [], h, w
        r = rng.uniform(1, 4)
        ph, pw = int(ch * r), int(cw * r)
        lst.append(ba.crop_pad(-int(rng.integers(0, ph - ch + 1)), -int(rng.integers(0, pw - cw + 1)), ph, pw, clip_boxes=False,
                               background=MEAN))
        ch, cw = ph, pw
        ph, pw = max(1, int(ch * rng.uniform(0.3, 1))), max(1, int(cw * rng.uniform(0.3, 1)))
        lst.append(ba.crop_pad(int(rng.integers(0, ch - ph + 1)), int(rng.integers(0, cw - pw + 1)), ph, pw, center_point_filter=True))
        ch, cw = ph, pw
        if b % 2:
            lst.append(ba.flip(cw))
        lst.append(ba.resize(ch, cw, 300, 300, interpolation_mode=b % 2))
        ops.append(lst)
    return images, ops


def host_chain(images, ops, cv2):
    """The per-image host chain the device replaces: ConvertTo3Channels, CropPad's canvas copy, Flip, cv2.resize, and
    Translate / Scale's cv2.warpAffine."""
    out = []
    for img, lst in zip(images, ops):
        x = img
        for o in lst:
            f = int(o[1]) & 0xFFFFFFFF
            bg = ((f >> 8) & 255, (f >> 16) & 255, (f >> 24) & 255)
            if o[0] == 6:
                h, w = x.shape[:2]
                x = cv2.warpAffine(x, np.float32([[1, 0, o[3]], [0, 1, o[2]]]), (w, h), borderMode=cv2.BORDER_CONSTANT, borderValue=bg)
            elif o[0] == 7:
                h, w = x.shape[:2]
                x = cv2.warpAffine(x, cv2.getRotationMatrix2D((w / 2, h / 2), 0, o[2]), (w, h), borderMode=cv2.BORDER_CONSTANT,
                                   borderValue=bg)
            elif o[0] == 1:
                py, px, ph, pw = (int(v) for v in o[2:])
                canvas = np.empty((ph, pw, 3), np.uint8)
                canvas[:, :] = ((f >> 8) & 255, (f >> 16) & 255, (f >> 24) & 255)
                H, W = x.shape[:2]
                r0, r1, c0, c1 = max(0, -py), min(ph, H - py), max(0, -px), min(pw, W - px)
                if r1 > r0 and c1 > c0:
                    canvas[r0:r1, c0:c1] = x[r0 + py:r1 + py, c0 + px:c1 + px]
                x = canvas
            elif o[0] == 2:
                x = x[:, ::-1]
            elif o[0] == 4:
                x = cv2.resize(np.ascontiguousarray(x), (int(o[5]), int(o[4])), interpolation=(int(o[1]) >> 8) & 255)
        out.append(x)
    return np.stack(out).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--host-iters', type=int, default=5)
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
        print('cv2 is not importable: the host chain is not timed')
    B = args.batch
    rng = np.random.default_rng(2026)
    for kind in ('validation', 'ssd', 'ssd7'):
        images, ops = chains(rng, B, kind)
        oh, ow = SIZES[kind]
        offs = np.concatenate([[0], np.cumsum([im.size for im in images])]).astype(np.int64)
        hwc = np.asarray([im.shape for im in images], np.int32)
        arr, max_ops = _pack_ops(ops, B)
        src = torch.from_numpy(np.concatenate([im.reshape(-1) for im in images])).cuda()
        out = torch.empty((B, oh, ow, 3), dtype=torch.float32, device='cuda')
        L, ctx, stream = _ffi.lib(), _ffi.context(), _ffi.stream_ptr()

        def launch():
            _ffi.check(L.ssdk_assemble_images(ctx, _ffi.dptr(src), _ffi.np_ptr(offs, C.c_longlong), _ffi.np_ptr(hwc, C.c_int), B, arr,
                                              max_ops, oh, ow, _ffi.dptr(out), stream))
        for _ in range(20):
            launch()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            launch()
        e1.record()
        torch.cuda.synchronize()
        kernel_ms = e0.elapsed_time(e1) / args.iters
        # whole call: pack into pinned memory, upload, launch, synchronised
        for _ in range(5):
            assemble_images_device(images, ops, oh, ow, out=out)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n_call = max(10, args.iters // 10)
        for _ in range(n_call):
            assemble_images_device(images, ops, oh, ow, out=out)
        torch.cuda.synchronize()
        call_ms = (time.perf_counter() - t0) * 1e3 / n_call
        nbytes = int(offs[-1]) + B * oh * ow * 3 * 4
        rec = dict(chain=kind, batch=B, gpu=smi, kernel_ms=round(kernel_ms, 4), call_ms=round(call_ms, 3),
                   algorithmic_bytes=nbytes, kernel_gbps=round(nbytes / kernel_ms / 1e6, 1),
                   hbm_fraction=round(nbytes / (kernel_ms * 1e-3) / HBM_PEAK, 3))
        if cv2 is not None:
            ref = host_chain(images, ops, cv2)
            assert np.array_equal(ref, out.cpu().numpy()), 'device and host chains differ'
            t0 = time.perf_counter()
            for _ in range(args.host_iters):
                host_chain(images, ops, cv2)
            rec['host_cv2_ms'] = round((time.perf_counter() - t0) * 1e3 / args.host_iters, 2)
            rec['host_threads'] = cv2.getNumThreads()
        print(json.dumps(rec))


if __name__ == '__main__':
    main()
