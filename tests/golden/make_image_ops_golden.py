#!/usr/bin/env python
"""Golden vectors for the image half of the geometric ops: the REAL reference's ConvertTo3Channels
(data_generator/object_detection_2d_photometric_ops.py), CropPad (..._patch_sampling_ops.py), Flip / Resize
(..._geometric_ops.py, i.e. uint8 cv2.resize) and SSDExpand (data_augmentation_chain_original_ssd.py) on seeded uint8 images.
Writes tests/golden/ref_image_ops_golden.npz: per case the input image ``in<k>``, the op list ``ops<k>`` as (n, 6) int64 rows
(op, flags, a0, a1, a2, a3) in the encoding of ssd_keras_b200.data_generator.batch_assembly, and the reference output
``out<k>``.  Needs the reference tree and cv2; run once, the .npz is data."""
import os
import sys

import numpy as np

np.float = float   # noqa
np.int = int       # noqa
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.environ.get('SSD_REFERENCE_ROOT', '/root/reference'))

import cv2                                                                                         # noqa: E402
from data_generator.data_augmentation_chain_original_ssd import SSDExpand                          # noqa: E402
from data_generator.object_detection_2d_geometric_ops import Flip, Resize                          # noqa: E402
from data_generator.object_detection_2d_patch_sampling_ops import CropPad                          # noqa: E402
from data_generator.object_detection_2d_photometric_ops import ConvertTo3Channels                  # noqa: E402

CROP_PAD, FLIP_H, FLIP_V, RESIZE = 1, 2, 3, 4
MEAN = (123, 117, 104)


def _crop_row(py, px, ph, pw, bg):
    return [CROP_PAD, (2 | (bg[0] << 8) | (bg[1] << 16) | (bg[2] << 24)) - (1 << 32 if bg[2] >= 128 else 0), py, px, ph, pw]


class Chain:
    def __init__(self, image):
        self.image = image
        self.img = ConvertTo3Channels()(image)
        self.ops = []

    def crop_pad(self, py, px, ph, pw, bg=(0, 0, 0)):
        self.img = CropPad(py, px, ph, pw, clip_boxes=False, box_filter=None, background=bg)(self.img, np.zeros((0, 5), np.int64))[0]
        self.ops.append(_crop_row(py, px, ph, pw, bg))

    def expand(self, rng):
        """SSDExpand with a seeded np.random; the patch it chose is read back from a box spanning the image."""
        h, w = self.img.shape[:2]
        np.random.seed(int(rng.integers(1 << 30)))
        img, lab = SSDExpand(background=MEAN)(self.img, np.array([[1, 0, 0, w, h]], np.int64))
        if img.shape[:2] != (h, w) or lab[0, 1] != 0 or lab[0, 2] != 0:
            self.ops.append(_crop_row(-int(lab[0, 2]), -int(lab[0, 1]), img.shape[0], img.shape[1], MEAN))
        self.img = img

    def flip(self, dim):
        self.ops.append([FLIP_H, 0, self.img.shape[1], 0, 0, 0] if dim == 'horizontal' else [FLIP_V, 0, self.img.shape[0], 0, 0, 0])
        self.img = Flip(dim=dim)(self.img)

    def resize(self, oh, ow, mode):
        self.ops.append([RESIZE, 1 | (mode << 8), self.img.shape[0], self.img.shape[1], oh, ow])
        self.img = Resize(height=oh, width=ow, interpolation_mode=mode)(self.img)


def _image(rng, h, w, c):
    shape = (h, w) if c == 0 else (h, w, c)
    return rng.integers(0, 256, shape, dtype=np.uint8)


def main():
    rng = np.random.default_rng(4711)
    cases = []
    # resize alone: upscale, downscale, exact 2x, non-integer ratios, identity, one axis only, 1-pixel inputs, every channel layout
    sizes = [((14, 20), (33, 31)), ((36, 28), (17, 11)), ((28, 28), (14, 14)), ((25, 33), (19, 19)), ((30, 30), (30, 30)),
             ((1, 57), (33, 40)), ((49, 1), (50, 7)), ((1, 1), (5, 4)), ((27, 31), (27, 50)), ((41, 27), (20, 27)),
             ((29, 37), (11, 14)), ((32, 32), (16, 16)), ((33, 31), (16, 15)), ((2, 2), (1, 1)), ((12, 16), (29, 29)),
             ((7, 5), (30, 30))]
    for k, ((h, w), (oh, ow)) in enumerate(sizes):
        for mode in (cv2.INTER_NEAREST, cv2.INTER_LINEAR):
            c = (0, 1, 3, 4)[(k + mode) % 4]
            ch = Chain(_image(rng, h, w, c))
            ch.resize(oh, ow, mode)
            cases.append(ch)
    # patches: pad every side, crop every side, both; then flips and a resize
    H, W = 30, 40
    patches = [(-4, -6, 40, 52), (5, 8, 18, 22), (-4, 10, 40, 20), (7, -5, 18, 52), (0, 0, H, W), (-2, -3, 14, 17),
               (20, 33, 17, 14), (H, W, 4, 4), (-10, -13, 12, 15), (0, -7, H, W + 13)]
    for k, (py, px, ph, pw) in enumerate(patches):
        c = (0, 1, 3, 4)[k % 4]
        ch = Chain(_image(rng, H, W, c))
        bg = MEAN if k % 2 else (0, 0, 0)
        ch.crop_pad(py, px, ph, pw, bg)
        if k % 3 == 0:
            ch.flip('horizontal')
        if k % 3 == 1:
            ch.flip('vertical')
        ch.resize(24, 18, k % 2)
        cases.append(ch)
    # the geometric part of the original SSD chain: expand (mean colour) -> crop inside the canvas -> flip -> resize
    for k in range(20):
        h, w = int(rng.integers(8, 36)), int(rng.integers(8, 36))
        ch = Chain(_image(rng, h, w, (3, 3, 1, 0, 4)[k % 5]))
        ch.expand(rng)
        ih, iw = ch.img.shape[:2]
        if k % 4 != 3:
            ph, pw = int(ih * rng.uniform(0.3, 1.0)) or 1, int(iw * rng.uniform(0.3, 1.0)) or 1
            ch.crop_pad(int(rng.integers(0, ih - ph + 1)), int(rng.integers(0, iw - pw + 1)), ph, pw)
        if k % 2:
            ch.flip('horizontal')
        ch.resize(32, 32, k % 2)
        cases.append(ch)
    # validation chain: ConvertTo3Channels -> Resize
    for k in range(6):
        h, w = int(rng.integers(24, 48)), int(rng.integers(28, 52))
        ch = Chain(_image(rng, h, w, (3, 0, 4)[k % 3]))
        ch.resize(20, 20, cv2.INTER_LINEAR)
        cases.append(ch)
    arrays = {'n': np.int64(len(cases))}
    for k, ch in enumerate(cases):
        arrays['in%d' % k] = ch.image
        arrays['ops%d' % k] = np.asarray(ch.ops, np.int64).reshape(-1, 6)
        arrays['out%d' % k] = ch.img
        assert ch.img.dtype == np.uint8 and ch.img.ndim == 3 and ch.img.shape[2] == 3
    out = os.path.join(HERE, 'ref_image_ops_golden.npz')
    np.savez_compressed(out, **arrays)
    print('wrote %d cases to %s (cv2 %s)' % (len(cases), out, cv2.__version__))


if __name__ == '__main__':
    main()
