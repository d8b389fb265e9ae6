#!/usr/bin/env python
"""Golden vectors for the photometric ops: the REAL reference's ConvertDataType, Brightness, Contrast, Saturation, Hue,
ConvertColor and ChannelSwap (data_generator/object_detection_2d_photometric_ops.py, i.e. NumPy and uint8 cv2.cvtColor), each
alone and in the order of SSDPhotometricDistortions.sequence1 / sequence2 (data_augmentation_chain_original_ssd.py:165-191; the
photometric part of the SSD7 chain's sequences is the same) with fixed parameters, on seeded uint8 images, gray and RGBA included.
Writes tests/golden/ref_photo_golden.npz: per case the input ``in<k>``, the op list ``ops<k>`` as (n, 6) float64 rows
(op, flags, a0, a1, a2, a3) in the encoding of ssd_keras_b200.data_generator.batch_assembly, and the reference output ``out<k>``
(uint8, or float32 where the case ends in the float state).  Needs the reference tree and cv2; run once, the .npz is data."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.environ.get('SSD_REFERENCE_ROOT', '/root/reference'))

from data_generator.object_detection_2d_photometric_ops import (Brightness, ChannelSwap, Contrast, ConvertColor,     # noqa: E402
                                                                 ConvertDataType, ConvertTo3Channels, Hue, Saturation)

TO_FLOAT32, TO_UINT8, BRIGHTNESS, CONTRAST, SATURATION, HUE, RGB2HSV, HSV2RGB, CHANNEL_SWAP = range(16, 25)


def op(code, a0=0.0, a1=0.0, a2=0.0):
    """(the reference transform, its row)"""
    ref = {TO_FLOAT32: lambda: ConvertDataType('float32'), TO_UINT8: lambda: ConvertDataType('uint8'),
           BRIGHTNESS: lambda: Brightness(a0), CONTRAST: lambda: Contrast(a0), SATURATION: lambda: Saturation(a0),
           HUE: lambda: Hue(a0), RGB2HSV: lambda: ConvertColor('RGB', 'HSV'), HSV2RGB: lambda: ConvertColor('HSV', 'RGB'),
           CHANNEL_SWAP: lambda: ChannelSwap((int(a0), int(a1), int(a2)))}[code]()
    return ref, [code, 0, a0, a1, a2, 0.0]


def sequence(which, brightness=None, contrast=None, saturation=None, hue=None, swap=None):
    f32, u8 = op(TO_FLOAT32), op(TO_UINT8)
    b = [op(BRIGHTNESS, brightness)] if brightness is not None else []
    c = [op(CONTRAST, contrast)] if contrast is not None else []
    hsv = ([op(RGB2HSV), f32] + ([op(SATURATION, saturation)] if saturation is not None else [])
           + ([op(HUE, hue)] if hue is not None else []) + [u8, op(HSV2RGB)])
    s = [op(CHANNEL_SWAP, *swap)] if swap is not None else []
    return [f32] + b + c + [u8] + hsv + s if which == 1 else [f32] + b + [u8] + hsv + [f32] + c + [u8] + s


def main():
    rng = np.random.default_rng(1912)
    out, k = {}, 0

    def image(h, w, c):
        return rng.integers(0, 256, (h, w) if c == 0 else (h, w, c), dtype=np.uint8)

    def case(img, steps):
        nonlocal k
        x = ConvertTo3Channels()(img)
        for ref, _ in steps:
            x = ref(x)
        out['in%d' % k] = img
        out['ops%d' % k] = np.asarray([row for _, row in steps], np.float64).reshape(-1, 6)
        out['out%d' % k] = x
        k += 1

    f32, u8 = op(TO_FLOAT32), op(TO_UINT8)
    # each class alone (between the conversions it needs)
    for delta in (32.0, -32.0, 84.0, -84.0, 0.5, 17.5, -3.25):
        case(image(37, 50, 3), [f32, op(BRIGHTNESS, delta), u8])
        case(image(9, 33, 3), [f32, op(BRIGHTNESS, delta)])
    for factor in (0.5, 1.5, 0.7310585786300049, 1.2345678):
        case(image(37, 50, 3), [f32, op(CONTRAST, factor), u8])
        case(image(9, 33, 3), [f32, op(CONTRAST, factor)])
    for factor in (0.3, 0.5, 1.5, 2.0, 1.1):
        case(image(21, 40, 3), [f32, op(SATURATION, factor), u8])
    for delta in (18.0, -18.0, 179.99999, -1e-6, 180.0, -180.0, 0.0, 77.7):
        img = image(21, 40, 3)
        img[..., 0] = rng.integers(0, 181, img.shape[:2])
        img[0, :8, 0] = (0, 1, 179, 180, 90, 2, 178, 0)
        case(img, [f32, op(HUE, delta), u8])
        case(img, [f32, op(HUE, delta)])
    for w in (1, 7, 31, 32, 33, 50, 64, 95, 130):
        case(image(13, w, 3), [op(RGB2HSV)])
        case(image(13, w, 3), [op(HSV2RGB)])
        case(image(5, w, 3), [op(RGB2HSV), op(HSV2RGB)])
    for order in ((0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)):
        case(image(11, 19, 3), [op(CHANNEL_SWAP, *order)])
    case(image(11, 19, 3), [f32, u8])
    # the sequences: every op present / absent / the extremes, random, gray and RGBA
    params = [dict(), dict(brightness=32.0, contrast=1.5, saturation=1.5, hue=18.0, swap=(2, 0, 1)),
              dict(brightness=-32.0, contrast=0.5, saturation=0.5, hue=-18.0), dict(brightness=84.0, saturation=2.0, hue=-1e-6),
              dict(brightness=-84.0, saturation=0.3, hue=179.99999), dict(brightness=12.5, contrast=0.9), dict(hue=7.25, swap=(1, 0, 2))]
    for _ in range(8):
        params.append(dict(brightness=float(rng.uniform(-32, 32)), contrast=float(rng.uniform(0.5, 1.5)),
                           saturation=float(rng.uniform(0.5, 1.5)), hue=float(rng.uniform(-18, 18))))
    for i, p in enumerate(params):
        for which in (1, 2):
            c = (3, 0, 4, 1)[(i + which) % 4]
            case(image(int(rng.integers(8, 40)), int(rng.integers(20, 110)), c), sequence(which, **p))
    out['n'] = np.int64(k)
    np.savez_compressed(os.path.join(HERE, 'ref_photo_golden.npz'), **out)
    print('wrote %d cases' % k)


if __name__ == '__main__':
    main()
