#!/usr/bin/env python
"""Time the focal loss (ssdk_focal_loss: focal_count_kernel + focal_loss_kernel) next to SSDLoss (ssdk_ssd_loss) at the
benchmark's shapes: SSD300 at B=32 (C=21, P=8732) and SSD512 at B=16 (C=81, P=24564), on seeded encoder-like inputs (about 2 %
positives, 5 % neutral boxes, softmax class scores).

Prints the GPU name and power limit, then per shape and call the median over --repeats of the span between two CUDA events
recorded around the call on its stream (loss and gradient, and the loss alone), after --warmup calls.  Bytes: the least any loss
and gradient call must move, reading y_true and y_pred once and writing the gradient once (3 B P (C+12) 4 bytes; the loss alone
reads the two inputs, 2 B P (C+12) 4), over the median time, and that rate as a share of the H100 SXM data sheet's 3.35 TB/s.
Needs a GPU.

    python tools/time_focal_loss.py [--repeats 50] [--warmup 5] [--seed 0]"""
import argparse
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
SHAPES = (('ssd300', 32, 8732, 21), ('ssd512', 16, 24564, 81))


def gpu_info():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                   # noqa: BLE001
        return 'nvidia-smi unavailable (%s)' % e


def make_inputs(rng, B, P, C):
    import torch
    W = C + 12
    kind = rng.choice(3, size=(B, P), p=[0.93, 0.02, 0.05])
    yt = np.zeros((B, P, W), np.float32)
    yt[..., 0] = kind == 0
    bi, pi = np.nonzero(kind == 1)
    yt[bi, pi, rng.integers(1, C, bi.size)] = 1
    yt[..., C:C + 4] = rng.normal(0, 1, (B, P, 4))
    z = rng.normal(0, 2, (B, P, C)).astype(np.float32)
    e = np.exp(z - z.max(-1, keepdims=True))
    yp = np.zeros_like(yt)
    yp[..., :C] = e / e.sum(-1, keepdims=True)
    yp[..., C:C + 4] = yt[..., C:C + 4] + rng.normal(0, 0.5, (B, P, 4))
    return torch.from_numpy(yt).cuda(), torch.from_numpy(yp).cuda()


def time_call(fn, repeats, warmup):
    import torch
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--repeats', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--seed', type=int, default=0)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as entry
    entry.build()
    from ssd_keras_b200 import _ffi
    if not torch.cuda.is_available():
        raise SystemExit('time_focal_loss.py needs a CUDA device')
    print('GPU: %s (name, power limit, max SM clock)' % gpu_info())
    lib, ctx, d = _ffi.lib(), _ffi.context(), _ffi.dptr
    rng = np.random.default_rng(args.seed)
    for name, B, P, C in SHAPES:
        yt, yp = make_inputs(rng, B, P, C)
        loss = torch.empty((B,), dtype=torch.float32, device='cuda')
        grad = torch.empty_like(yp)

        def focal(g):
            return lambda: _ffi.check(lib.ssdk_focal_loss(ctx, d(yt), d(yp), B, P, C, 2.0, 0.25, 1.0, None, d(loss), d(g),
                                                          _ffi.stream_ptr()))

        def ssd(g):
            return lambda: _ffi.check(lib.ssdk_ssd_loss(ctx, d(yt), d(yp), B, P, C, 3, 0, 1.0, None, d(loss), None, d(g),
                                                        _ffi.stream_ptr()))
        W = C + 12
        for label, fn, n_tensors in (('focal loss + gradient', focal(grad), 3), ('SSDLoss loss + gradient', ssd(grad), 3),
                                     ('focal loss', focal(None), 2), ('SSDLoss loss', ssd(None), 2)):
            ms = time_call(fn, args.repeats, args.warmup)
            nbytes = n_tensors * B * P * W * 4
            rate = nbytes / (ms * 1e-3)
            print('%s B=%d C=%d P=%d  %-24s median %.4f ms  %6.1f MB  %.3f TB/s = %.3f of 3.35 TB/s'
                  % (name, B, C, P, label, ms, nbytes / 1e6, rate / 1e12, rate / HBM_BYTES_PER_S), flush=True)
        del yt, yp, grad
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
