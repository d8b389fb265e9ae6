#!/usr/bin/env python
"""Golden vectors for Translate / Scale / Rotate and BoxFilter's overlap test: the REAL reference's ConvertTo3Channels
(data_generator/object_detection_2d_photometric_ops.py), Translate / Scale / Rotate / Flip / Resize (..._geometric_ops.py, i.e.
uint8 cv2.warpAffine and cv2.resize), CropPad (..._patch_sampling_ops.py) and BoxFilter (..._image_boxes_validation_utils.py)
on seeded uint8 images and label arrays.  Per case: the input image ``in<k>`` and labels ``lin<k>``, the op list ``ops<k>`` as
(n, 6) float64 rows (op, flags, a0, a1, a2, a3) in the encoding of ssd_keras_b200.data_generator.batch_assembly, the
reference's image ``out<k>`` and labels ``lout<k>``, and ``kind<k>``.  Covers both geometric sequences of the SSD7 chain
(DataAugmentationConstantInputSize, the notebook's filter settings), the satellite chain's geometric list, every overlap
criterion and border_pixels mode, and a Scale corner that lands on an exact .5 tie.  Writes
tests/golden/ref_warp_golden.npz.  Needs the reference tree and cv2; run once, the .npz is data."""
import os
import sys
from fractions import Fraction

import numpy as np

np.float = float   # noqa
np.int = int       # noqa
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.environ.get('SSD_REFERENCE_ROOT', '/root/reference'))

import cv2                                                                                          # noqa: E402
from data_generator.object_detection_2d_geometric_ops import Flip, Resize, Rotate, Scale, Translate  # noqa: E402
from data_generator.object_detection_2d_image_boxes_validation_utils import BoxFilter               # noqa: E402
from data_generator.object_detection_2d_patch_sampling_ops import CropPad                           # noqa: E402
from data_generator.object_detection_2d_photometric_ops import ConvertTo3Channels                   # noqa: E402

CROP_PAD, FLIP_H, FLIP_V, RESIZE, FILTER, TRANSLATE, SCALE, ROTATE, OVERLAP, CLIP = 1, 2, 3, 4, 5, 6, 7, 8, 9, 10
CRIT = {'center_point': 0, 'area': 1, 'iou': 2}
BORD = {'half': 0, 'include': 1, 'exclude': 2}
SSD7_FILTER = dict(check_overlap=True, check_min_area=True, check_degenerate=True, overlap_criterion='area',
                   overlap_bounds=(0.3, 1.0), min_area=16)


def _i32(v):
    return v - (1 << 32) if v >= (1 << 31) else v


def _bg(bg):
    return (bg[0] << 8) | (bg[1] << 16) | (bg[2] << 24)


def _filter_rows(kw, h, w):
    rows = []
    if kw.get('check_degenerate', True) or kw.get('check_min_area', True):
        ma = kw.get('check_min_area', True)
        rows.append([FILTER, (1 if kw.get('check_degenerate', True) else 0) | (2 if ma else 0), kw.get('min_area', 16) if ma else 0, 0, 0, 0])
    if kw.get('check_overlap', True):
        lo, up = kw.get('overlap_bounds', (0.3, 1.0))
        rows.append([OVERLAP, CRIT[kw.get('overlap_criterion', 'center_point')] | (BORD[kw.get('border_pixels', 'half')] << 2), lo, up, h, w])
    return rows


class Chain:
    def __init__(self, image, labels, kind):
        self.image, self.labels, self.kind = image, labels.astype(np.float64), kind
        self.img = ConvertTo3Channels()(image)
        self.lab = self.labels.copy()
        self.ops = []

    def translate(self, dy, dx, kw=None, clip=True, bg=(0, 0, 0)):
        h, w = self.img.shape[:2]
        bf = BoxFilter(**kw) if kw else None
        self.img, self.lab = Translate(dy, dx, clip_boxes=clip, box_filter=bf, background=bg)(self.img, self.lab)
        self.ops.append([TRANSLATE, _i32(_bg(bg)), int(round(h * dy)), int(round(w * dx)), h, w])
        self.ops += _filter_rows(kw, h, w) if kw else []
        if clip:
            self.ops.append([CLIP, 0, h, w, 0, 0])

    def scale(self, f, kw=None, clip=True, bg=(0, 0, 0)):
        h, w = self.img.shape[:2]
        bf = BoxFilter(**kw) if kw else None
        self.img, self.lab = Scale(f, clip_boxes=clip, box_filter=bf, background=bg)(self.img, self.lab)
        self.ops.append([SCALE, _i32(_bg(bg)), f, h, w, 0])
        self.ops += _filter_rows(kw, h, w) if kw else []
        if clip:
            self.ops.append([CLIP, 0, h, w, 0, 0])

    def rotate(self, angle):
        h, w = self.img.shape[:2]
        self.img, self.lab = Rotate(angle)(self.img, self.lab)
        self.ops.append([ROTATE, 0, angle, h, w, 0])

    def flip(self, dim):
        self.ops.append([FLIP_H, 0, self.img.shape[1], 0, 0, 0] if dim == 'horizontal' else [FLIP_V, 0, self.img.shape[0], 0, 0, 0])
        self.img, self.lab = Flip(dim=dim)(self.img, self.lab)

    def patch(self, py, px, ph, pw, kw):
        self.img, self.lab = CropPad(py, px, ph, pw, clip_boxes=True, box_filter=BoxFilter(**kw))(self.img, self.lab)
        self.ops.append([CROP_PAD, 0, py, px, ph, pw])
        self.ops += _filter_rows(kw, ph, pw)
        self.ops.append([CLIP, 0, ph, pw, 0, 0])

    def resize(self, oh, ow, kw):
        ih, iw = self.img.shape[:2]
        self.img, self.lab = Resize(oh, ow, box_filter=BoxFilter(**kw))(self.img, self.lab)
        self.ops.append([RESIZE, 1 << 8, ih, iw, oh, ow])
        self.ops += _filter_rows(kw, oh, ow)


def _image(rng, h, w, c):
    return rng.integers(0, 256, (h, w) if c == 0 else (h, w, c), dtype=np.uint8)


def _labels(rng, h, w, n, halves=False):
    x0 = rng.integers(-w // 4, w, n); y0 = rng.integers(-h // 4, h, n)
    bw = rng.integers(0, max(2, w // 2), n); bh = rng.integers(0, max(2, h // 2), n)
    lab = np.stack([rng.integers(1, 21, n), x0, y0, x0 + bw, y0 + bh], axis=1).astype(np.float64)
    if halves:
        lab[:, 1:] += rng.integers(0, 2, (n, 4)) * 0.5
    return lab


def _tie():
    """(h, w, factor, x): Scale's corner x lands on round(f*x) + m2 == k + 0.5 exactly, where the exact f*x + m2 is not a tie."""
    for f in (1.1, 1.3, 0.7, 1.7, 0.9, 1.9, 0.55):
        for w in range(20, 400):
            M = cv2.getRotationMatrix2D((w / 2, 50), 0, f)
            for x in range(w):
                two = (M[0, 0] * x + M[0, 1] * 0.0) + M[0, 2]
                exact = Fraction(M[0, 0]) * x + Fraction(M[0, 2])
                if two - np.floor(two) == 0.5 and exact != Fraction(two) and np.round(two) != np.round(float(exact)):
                    return 100, w, f, x
    raise RuntimeError('no tie found')


def main():
    rng = np.random.default_rng(8128)
    cases = []
    bg7 = (0, 0, 0)
    # SSD7, sequence 1: translate -> zoom in -> flip; sequence 2: zoom out -> translate -> flip (each step taken or not)
    for k in range(24):
        h, w = int(rng.integers(12, 44)), int(rng.integers(12, 44))
        c = (3, 3, 0, 4, 1)[k % 5]
        bg = bg7 if k % 3 else (int(rng.integers(256)), int(rng.integers(256)), int(rng.integers(256)))
        ch = Chain(_image(rng, h, w, c), _labels(rng, h, w, int(rng.integers(0, 9))), 'ssd7_seq%d' % (1 + k % 2))
        dy = float(rng.uniform(0.03, 0.5)) * rng.choice([-1, 1]); dx = float(rng.uniform(0.03, 0.5)) * rng.choice([-1, 1])
        if k % 2 == 0:
            if k % 8 != 6:
                ch.translate(dy, dx, SSD7_FILTER, bg=bg)
            if k % 8 != 4:
                ch.scale(float(rng.uniform(1.0, 2.0)), SSD7_FILTER, bg=bg)
        else:
            if k % 8 != 7:
                ch.scale(float(rng.uniform(0.5, 1.0)), SSD7_FILTER, bg=bg)
            if k % 8 != 5:
                ch.translate(dy, dx, SSD7_FILTER, bg=bg)
        if k % 4 < 2:
            ch.flip('horizontal')
        cases.append(ch)
    # satellite: flips -> rotate -> patch ('area' filter, clip) -> resize (degenerate + min area)
    for k in range(12):
        h, w = int(rng.integers(12, 40)), int(rng.integers(12, 40))
        ch = Chain(_image(rng, h, w, (3, 0, 4)[k % 3]), _labels(rng, h, w, int(rng.integers(1, 8))), 'satellite')
        if k % 2:
            ch.flip('horizontal')
        if k % 3 == 1:
            ch.flip('vertical')
        if k % 4 != 3:
            ch.rotate((90, 180, 270)[k % 3])
        ih, iw = ch.img.shape[:2]
        ph, pw = max(1, int(ih * rng.uniform(0.3, 1.5))), max(1, int(iw * rng.uniform(0.3, 1.5)))
        py, px = int(rng.integers(min(0, ih - ph), max(0, ih - ph) + 1)), int(rng.integers(min(0, iw - pw), max(0, iw - pw) + 1))
        ch.patch(py, px, ph, pw, dict(check_overlap=True, check_min_area=False, check_degenerate=False, overlap_criterion='area',
                                      overlap_bounds=(0.3, 1.0)))
        ch.resize(24, 30, dict(check_overlap=False, check_min_area=True, check_degenerate=True, min_area=16))
        cases.append(ch)
    # single ops: factors below, above and exactly 1, translations beyond the image, rotations of odd / even / 1-pixel sizes
    sizes = [(1, 1), (1, 17), (23, 1), (15, 21), (16, 16), (31, 12), (2, 3), (19, 26)]
    for k, (h, w) in enumerate(sizes):
        for j, f in enumerate((0.5, 1.0, 1.37, 2.0, 0.73)):
            ch = Chain(_image(rng, h, w, (3, 0, 4, 1)[(k + j) % 4]), _labels(rng, h, w, 3, halves=j % 2 == 1), 'scale')
            ch.scale(f, None, clip=False, bg=(10 * j, 200, 7))
            cases.append(ch)
        for j, (dy, dx) in enumerate(((1.5, 0.0), (-0.2, 0.6), (0.0, -1.3), (0.35, 0.35))):
            ch = Chain(_image(rng, h, w, (0, 3, 1, 4)[(k + j) % 4]), _labels(rng, h, w, 3), 'translate')
            ch.translate(dy, dx, None, clip=j % 2 == 0, bg=(255, 1, 128))
            cases.append(ch)
        for j, a in enumerate((90, 180, 270)):
            ch = Chain(_image(rng, h, w, (4, 3, 0)[(k + j) % 3]), _labels(rng, h, w, 3, halves=True), 'rotate')
            ch.rotate(a)
            cases.append(ch)
    # every overlap criterion and border_pixels mode, through Translate's box filter; 'area' with lower == 0 too
    for k, (crit, bp, bounds) in enumerate([(c, b, lb) for c in ('center_point', 'area', 'iou') for b in ('half', 'include', 'exclude')
                                            for lb in ((0.3, 1.0), (0.0, 0.6))]):
        h, w = 24, 30
        ch = Chain(_image(rng, h, w, 3), _labels(rng, h, w, 12, halves=k % 2 == 1), 'overlap')
        kw = dict(check_overlap=True, check_min_area=k % 3 == 0, check_degenerate=k % 2 == 0, overlap_criterion=crit,
                  overlap_bounds=bounds, border_pixels=bp, min_area=9)
        ch.translate(float(rng.uniform(-0.4, 0.4)), float(rng.uniform(-0.4, 0.4)), kw, clip=k % 2 == 0)
        cases.append(ch)
    # a corner tie for np.round: (m0*x + m1*y) + m2 rounded twice is k + 0.5; a fused f*x + m2 would round the other way
    th, tw, tf, tx = _tie()
    ch = Chain(_image(rng, th, tw, 3), np.array([[1, tx, 10, tw - 1, 60], [2, 0, 0, tx, 30]], np.float64), 'tie')
    ch.scale(tf, None, clip=False)
    cases.append(ch)
    arrays = {'n': np.int64(len(cases)), 'tie': np.array([th, tw, tf, tx], np.float64)}
    for k, ch in enumerate(cases):
        arrays['in%d' % k] = ch.image
        arrays['lin%d' % k] = ch.labels
        arrays['ops%d' % k] = np.asarray(ch.ops, np.float64).reshape(-1, 6)
        arrays['out%d' % k] = ch.img
        arrays['lout%d' % k] = np.asarray(ch.lab, np.float64).reshape(-1, 5)
        arrays['kind%d' % k] = np.array(ch.kind)
        assert ch.img.dtype == np.uint8 and ch.img.ndim == 3 and ch.img.shape[2] == 3
    out = os.path.join(HERE, 'ref_warp_golden.npz')
    np.savez_compressed(out, **arrays)
    print('wrote %d cases to %s (cv2 %s, numpy %s); tie h=%d w=%d f=%r x=%d' % (len(cases), out, cv2.__version__, np.__version__, th, tw, tf, tx))


if __name__ == '__main__':
    main()
