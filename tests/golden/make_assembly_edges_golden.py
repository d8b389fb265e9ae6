#!/usr/bin/env python
"""Golden vectors for the edges of the box half of the op lists: the REAL reference's CropPad (data_generator/
object_detection_2d_patch_sampling_ops.py), Flip / Resize / Translate / Scale / Rotate (..._geometric_ops.py) and BoxFilter
(..._image_boxes_validation_utils.py) on hand-made float64 label arrays.  Per case: the labels ``lin<k>``, the op list ``ops<k>``
as (n, 6) float64 rows (op, flags, a0, a1, a2, a3) in the encoding of ssd_keras_b200.data_generator.batch_assembly, the
reference's labels ``lout<k>``, ``kind<k>`` and the reference's calls ``calls<k>`` (a repr, so that the CPU test can run them
again where the reference is present).

Covers coordinates that land exactly on .5 after a Resize ratio and one float64 ulp either side, 'center_point' centres on 0 and
on h-1 / w-1, 'area' on its lower bound (lower == 0 and lower > 0), 'iou' on both bounds in every border_pixels mode, min_area
and degenerate equality, the -0.0 that Resize keeps and that Scale / Rotate turn into +0 (their ``astype(int)``), with and
without a following clip, NaN and +-inf in every coordinate through every op but Scale and Rotate (``astype(int)`` of a NaN or
an infinity is platform-defined, so those are left out), empty label arrays, lists that drop every box, and fractional and
negative class ids.  Writes tests/golden/ref_assembly_edges_golden.npz.  Needs the reference tree and cv2; run once, the .npz
is data."""
import os
import sys

import numpy as np

np.float = float   # noqa
np.int = int       # noqa
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.environ.get('SSD_REFERENCE_ROOT', '/root/reference'))

import cv2                                                                                          # noqa: E402,F401
from data_generator.object_detection_2d_geometric_ops import Flip, Resize, Rotate, Scale, Translate  # noqa: E402
from data_generator.object_detection_2d_image_boxes_validation_utils import BoxFilter               # noqa: E402
from data_generator.object_detection_2d_patch_sampling_ops import CropPad                           # noqa: E402

CROP_PAD, FLIP_H, FLIP_V, RESIZE, FILTER, TRANSLATE, SCALE, ROTATE, OVERLAP, CLIP = 1, 2, 3, 4, 5, 6, 7, 8, 9, 10
CRIT = {'center_point': 0, 'area': 1, 'iou': 2}
BORD = {'half': 0, 'include': 1, 'exclude': 2}
NAN, INF = float('nan'), float('inf')


def filter_rows(kw, h, w):
    """The op rows of one BoxFilter(**kw) call against an h x w image (batch_assembly.box_filter_ops)."""
    rows = []
    deg, ma = kw.get('check_degenerate', True), kw.get('check_min_area', True)
    if deg or ma:
        rows.append([FILTER, (1 if deg else 0) | (2 if ma else 0), kw.get('min_area', 16) if ma else 0, 0, 0, 0])
    if kw.get('check_overlap', True):
        lo, up = kw.get('overlap_bounds', (0.3, 1.0))
        rows.append([OVERLAP, CRIT[kw.get('overlap_criterion', 'center_point')] | (BORD[kw.get('border_pixels', 'half')] << 2), lo, up, h, w])
    return rows


def run(calls, labels, h, w):
    """calls: ('crop_pad', py, px, ph, pw, clip, filter_kw) | ('flip', dim) | ('resize', oh, ow, filter_kw) | ('filter', kw) |
    ('translate', dy, dx, clip, filter_kw) | ('scale', f, clip, filter_kw) | ('rotate', angle), in order, on an h x w image.
    -> (reference labels, op rows)."""
    img = np.zeros((h, w, 3), np.uint8)
    lab = np.array(labels, np.float64).reshape(-1, 5)
    rows = []
    for c in calls:
        h, w = img.shape[:2]
        kind = c[0]
        if kind == 'crop_pad':
            _, py, px, ph, pw, clip, kw = c
            if kw == 'center':              # CropPad's own center_point filter: op flag 1
                bf = BoxFilter(check_overlap=True, check_min_area=False, check_degenerate=False, overlap_criterion='center_point')
                rows.append([CROP_PAD, 1 | (2 if clip else 0), py, px, ph, pw])
            else:
                bf = BoxFilter(**kw) if kw else None
                rows.append([CROP_PAD, 0, py, px, ph, pw])
                rows += filter_rows(kw, ph, pw) if kw else []
                rows += [[CLIP, 0, ph, pw, 0, 0]] if clip else []
            img, lab = CropPad(py, px, ph, pw, clip_boxes=clip, box_filter=bf)(img, lab)
        elif kind == 'flip':
            rows.append([FLIP_H, 0, w, 0, 0, 0] if c[1] == 'horizontal' else [FLIP_V, 0, h, 0, 0, 0])
            img, lab = Flip(dim=c[1])(img, lab)
        elif kind == 'resize':
            _, oh, ow, kw = c
            if kw == 'degenerate':          # Resize's degenerate filter: op flag 1
                bf = BoxFilter(check_overlap=False, check_min_area=False, check_degenerate=True)
                rows.append([RESIZE, 1 | (1 << 8), h, w, oh, ow])
            else:
                bf = BoxFilter(**kw) if kw else None
                rows.append([RESIZE, 1 << 8, h, w, oh, ow])
                rows += filter_rows(kw, oh, ow) if kw else []
            img, lab = Resize(oh, ow, box_filter=bf)(img, lab)
        elif kind == 'filter':
            lab = BoxFilter(**c[1])(lab, image_height=h, image_width=w)
            rows += filter_rows(c[1], h, w)
        elif kind == 'translate':
            _, dy, dx, clip, kw = c
            rows.append([TRANSLATE, 0, int(round(h * dy)), int(round(w * dx)), h, w])
            rows += filter_rows(kw, h, w) if kw else []
            rows += [[CLIP, 0, h, w, 0, 0]] if clip else []
            img, lab = Translate(dy, dx, clip_boxes=clip, box_filter=BoxFilter(**kw) if kw else None)(img, lab)
        elif kind == 'scale':
            _, f, clip, kw = c
            rows.append([SCALE, 0, f, h, w, 0])
            rows += filter_rows(kw, h, w) if kw else []
            rows += [[CLIP, 0, h, w, 0, 0]] if clip else []
            img, lab = Scale(f, clip_boxes=clip, box_filter=BoxFilter(**kw) if kw else None)(img, lab)
        elif kind == 'rotate':
            rows.append([ROTATE, 0, c[1], h, w, 0])
            img, lab = Rotate(c[1])(img, lab)
        else:
            raise ValueError(kind)
    return np.asarray(lab, np.float64).reshape(-1, 5), np.asarray(rows, np.float64).reshape(-1, 6)


def _half_ties(r, n=4):
    """Coordinates x >= 0 whose float64 product x * r is exactly k + 0.5 (np.round's half-even tie)."""
    out = []
    for i in range(1, 4000):
        x = i / 4
        p = x * r
        if p - np.floor(p) == 0.5:
            out.append(x)
            if len(out) == n:
                break
    return out


def _ulps(x):
    return [np.nextafter(x, -INF), x, np.nextafter(x, INF)]


def _nonfinite_rows():
    """Per coordinate: NaN, +inf, -inf, with a finite box around it; plus two ordinary boxes."""
    base = [3.0, 5.0, 4.0, 20.0, 18.0]
    rows = [[1, 2, 2, 12, 10], [2, 6, 1, 25, 15]]
    for j in range(1, 5):
        for v in (NAN, INF, -INF):
            r = list(base)
            r[j] = v
            rows.append(r)
    rows.append([4, NAN, NAN, NAN, NAN])
    return np.asarray(rows, np.float64)


def cases():
    out = []

    def add(kind, calls, labels, h, w):
        out.append((kind, calls, np.asarray(labels, np.float64).reshape(-1, 5), h, w))

    # Resize ratios whose products land on .5, and one ulp either side; ratios above and below 1, dyadic and not
    for (ih, iw, oh, ow) in ((40, 40, 60, 60), (30, 70, 300, 300), (300, 300, 7, 3), (3, 7, 300, 300), (299, 500, 300, 300)):
        ry, rx = oh / ih, ow / iw
        xs = [u for x in _half_ties(rx) for u in _ulps(x)]
        ys = [u for y in _half_ties(ry) for u in _ulps(y)]
        n = min(len(xs), len(ys))
        lab = [[1 + k % 3, xs[k], ys[k], xs[k] + 1.5, ys[n - 1 - k] + 7.0] for k in range(n)]
        add('resize_tie', [('resize', oh, ow, None)], lab, ih, iw)
        add('resize_tie', [('resize', oh, ow, 'degenerate')], lab, ih, iw)
    # 'center_point' centres exactly on 0 and on h-1 / w-1 (and an ulp outside), CropPad's own filter and BoxFilter's
    h, w = 24, 30
    lab = []
    for cy in (0.0, h - 1.0, np.nextafter(0.0, -1), np.nextafter(h - 1.0, INF)):
        for cx in (0.0, w - 1.0, np.nextafter(0.0, -1), np.nextafter(w - 1.0, INF)):
            lab.append([1, cx - 3, cy - 2, cx + 3, cy + 2])
    lab = np.asarray(lab)
    add('center', [('filter', dict(check_overlap=True, check_min_area=False, check_degenerate=False, overlap_criterion='center_point'))],
        lab, h, w)
    sh = lab.copy()
    sh[:, [2, 4]] += 5
    sh[:, [1, 3]] += 7
    add('center', [('crop_pad', 5, 7, h, w, True, 'center')], sh, 40, 50)
    add('center', [('crop_pad', 5, 7, h, w, False, 'center')], sh, 40, 50)
    # 'area' on the lower bound: lower == 0 with zero intersections; lower > 0 with inter == lower * area exactly
    for bp in BORD:
        d = {'half': 0, 'include': 1, 'exclude': -1}[bp]
        h, w = 20, 20
        zero = [[1, -10, 2, -10 + (1 - d) * 0 + 0, 12], [1, 25, 3, 30, 9], [2, 19 + 0, 0, 25, 5], [3, 2, 2, 6, 6], [1, -8, -8, 0, 0]]
        add('area_lower0', [('filter', dict(check_overlap=True, check_min_area=False, check_degenerate=False, overlap_criterion='area',
                                             overlap_bounds=(0.0, 1.0), border_pixels=bp))], zero, h, w)
        # [-5, 0, 5, 10]: inter (5 + d) * (10 + d) of area (10 + d) * (10 + d): lower = the quotient in float64, and its ulps
        lab = [[1, -5, 0, 5, 10], [2, 10, -5, 30, 5], [3, -4, 4, 8, 12]]
        for lo in _ulps((5.0 + d) / (10.0 + d)):
            add('area_lower', [('filter', dict(check_overlap=True, check_min_area=False, check_degenerate=False, overlap_criterion='area',
                                                overlap_bounds=(lo, 1.0), border_pixels=bp))], lab, h, w)
        # upper bound: a box inside the image has inter == area
        add('area_upper', [('filter', dict(check_overlap=True, check_min_area=False, check_degenerate=False, overlap_criterion='area',
                                            overlap_bounds=(0.2, 0.5), border_pixels=bp))], lab + [[4, 2, 2, 9, 9]], h, w)
    # 'iou' on both bounds, every border mode: a box inside the image, v = inter / (ap + aq - inter), inter without border_pixels
    for bp in BORD:
        d = {'half': 0, 'include': 1, 'exclude': -1}[bp]
        H, W = 16, 16
        lab = [[1, 4, 4, 12, 12], [2, 0, 0, 16, 16], [3, -4, -4, 4, 4], [4, 8, 2, 24, 6]]
        inter, aq, ap = 64.0, (8.0 + d) ** 2, (W + d) * (H + d)
        v = inter / ((ap + aq) - inter)
        for lo, up in ((v, 1.0), (np.nextafter(v, -1), 1.0), (0.0, v), (0.0, np.nextafter(v, -1)), (v, v)):
            add('iou_bound', [('filter', dict(check_overlap=True, check_min_area=False, check_degenerate=False, overlap_criterion='iou',
                                               overlap_bounds=(lo, up), border_pixels=bp))], lab, H, W)
    # min_area equality and degenerate equality
    lab = [[1, 0, 0, 4, 4], [2, 0, 0, 4, 3.9999999999999996], [3, 5, 5, 5, 9], [4, 5, 5, 9, 5], [5, 1, 1, 2, 17], [6, 3, 3, 2, 8]]
    for kw in (dict(check_overlap=False, check_min_area=True, check_degenerate=False, min_area=16),
               dict(check_overlap=False, check_min_area=True, check_degenerate=True, min_area=16),
               dict(check_overlap=False, check_min_area=False, check_degenerate=True),
               dict(check_overlap=False, check_min_area=True, check_degenerate=False, min_area=0)):
        add('min_area', [('filter', kw)], lab, 20, 20)
    # -0.0: Resize keeps it; Scale and Rotate store np.round(...).astype(int), so +0; a following clip keeps what it is given
    neg = [[1, -0.2, -0.4, 10, 12], [2, -0.0, 3, 5, -0.0], [3, 9.9, 6.6, 30, 30]]
    add('negzero', [('resize', 30, 50, None)], neg, 40, 60)
    add('negzero', [('resize', 30, 50, None), ('crop_pad', 0, 0, 30, 50, True, None)], neg, 40, 60)
    add('negzero', [('resize', 30, 50, None), ('translate', 0.0, 0.0, True, None)], neg, 40, 60)
    add('negzero', [('scale', 1.5, False, None)], [[1, 9.9, 6.6, 30, 30], [2, 10.1, 6.8, 12, 20]], 40, 60)
    add('negzero', [('scale', 1.5, True, None)], [[1, 9.9, 6.6, 30, 30], [2, 10.1, 6.8, 12, 20]], 40, 60)
    for a in (90, 180, 270):
        add('negzero', [('rotate', a)], [[1, 0.3, 0.4, 5, 6], [2, 10, 12, 19.6, 29.7], [3, -0.4, -0.3, 0.4, 0.3]], 30, 20)
    add('negzero', [('crop_pad', 0, 0, 20, 20, True, None)], [[1, -0.0, -0.0, 5, 5], [2, -3, -0.0, -0.0, 4]], 20, 20)
    # NaN and +-inf in every coordinate through every op but Scale and Rotate
    nf = _nonfinite_rows()
    ssd7 = dict(check_overlap=True, check_min_area=True, check_degenerate=True, overlap_criterion='area', overlap_bounds=(0.3, 1.0),
                min_area=16)
    for calls in ([('crop_pad', 2, 3, 20, 24, True, None)], [('crop_pad', 2, 3, 20, 24, False, None)],
                  [('crop_pad', 0, 0, 30, 30, True, 'center')], [('crop_pad', -4, -3, 40, 40, True, dict(check_overlap=True,
                   check_min_area=False, check_degenerate=False, overlap_criterion='area', overlap_bounds=(0.3, 1.0)))],
                  [('flip', 'horizontal')], [('flip', 'vertical')], [('resize', 45, 20, None)], [('resize', 45, 20, 'degenerate')],
                  [('crop_pad', 0, 0, 30, 30, True, None), ('resize', 60, 60, 'degenerate')],
                  [('translate', 0.1, -0.2, True, None)], [('translate', -0.3, 0.25, False, ssd7)],
                  [('filter', ssd7)], [('filter', dict(check_overlap=False, check_min_area=False, check_degenerate=True))]) + tuple(
                  [('filter', dict(check_overlap=True, check_min_area=False, check_degenerate=False, overlap_criterion=c,
                                   overlap_bounds=(0.0, 1.0), border_pixels=b))] for c in CRIT for b in ('half', 'include')):
        add('nonfinite', calls, nf, 30, 30)
    # empty label arrays, lists that drop every box, fractional and negative class ids
    for calls in ([('crop_pad', 2, 3, 20, 24, True, 'center')], [('resize', 10, 10, 'degenerate'), ('filter', ssd7)],
                  [('flip', 'horizontal'), ('translate', 0.5, 0.5, True, None)]):
        add('empty', calls, np.zeros((0, 5)), 30, 30)
    add('drop_all', [('crop_pad', 0, 0, 10, 10, True, 'center')], [[1, 20, 20, 29, 29], [2, -9, -9, -1, -1], [3, 15, 1, 25, 8]], 30, 30)
    add('drop_all', [('filter', ssd7)], [[1, 0, 0, 2, 2], [2, 5, 5, 5, 9], [3, -10, -10, -1, -1]], 30, 30)
    add('drop_all', [('resize', 3, 3, 'degenerate')], [[1, 0, 0, 4, 4], [2, 10, 10, 14, 30]], 30, 30)
    cls = [[1.5, 1, 1, 9, 9], [-1, 2, 2, 12, 8], [-0.0, 3, 3, 7, 7], [0.25, 4, 4, 20, 20], [1e9, 1, 2, 3, 4], [-2.5, 0, 0, 1, 1]]
    add('class_ids', [('flip', 'horizontal'), ('resize', 60, 60, 'degenerate')], cls, 30, 30)
    add('class_ids', [('scale', 1.25, True, None), ('rotate', 90)], cls, 30, 30)
    return out


def main():
    arrays = {}
    cs = cases()
    for k, (kind, calls, lab, h, w) in enumerate(cs):
        ref, rows = run(calls, lab, h, w)
        arrays['lin%d' % k] = lab
        arrays['ops%d' % k] = rows
        arrays['lout%d' % k] = ref
        arrays['kind%d' % k] = np.array(kind)
        arrays['calls%d' % k] = np.array(repr((calls, h, w)))
    arrays['n'] = np.int64(len(cs))
    out = os.path.join(HERE, 'ref_assembly_edges_golden.npz')
    np.savez_compressed(out, **arrays)
    print('wrote %d cases to %s (numpy %s, %d bytes)' % (len(cs), out, np.__version__, os.path.getsize(out)))


if __name__ == '__main__':
    main()
