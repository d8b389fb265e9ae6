"""Cases for the evaluator's matching (csrc/evaluate.cu: eval_match_kernel, eval_cumsum_kernel, driven by
Evaluator.match_predictions) and a model of which kernel paths each case reaches.

Two tables, both seeded:
- EDGES: small cases the reference's own Evaluator was run on (tests/golden/make_eval_edges_golden.py writes
  tests/golden/ref_eval_edges_golden.npz): every label dtype, the three border modes, thresholds 0.5 / 0.45 / 0.7 / 0.0,
  predictions bisected onto the threshold in both arithmetic types, dyadic boxes with an IoU of exactly 0.5, NaN overlaps,
  non-finite coordinates, ties and NaNs across lanes, neutral arg-maxes, duplicates, an empty class, images without labels,
  integer image ids, a permuted gt_format, a fractional class id, equal confidences, and overlaps below -1.
- CASES: large generated cases for the GPU, held to oracle/evalops.py: more than 32 boxes per image (several lane passes),
  thousands of images x 20 classes (thousands of CTAs), classes of 1023 / 1024 / 1025 / 5000 predictions (1 to 5 cumsum
  chunks), an empty class, float32 and float64 images in one call, and tens of thousands of near-threshold predictions.

``paths(case)`` restates the kernels' structure (32 lanes striding an image's boxes, 8 warps per CTA, 1024-element cumsum
chunks, read from the source) and names the paths the case reaches."""
import math
import os
import re
from fractions import Fraction

import numpy as np

from oracle import evalops as eo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EVALUATE_CU = os.path.join(ROOT, 'ssd_keras_b200', 'csrc', 'evaluate.cu')


def _constants():
    with open(EVALUATE_CU) as f:
        src = f.read()
    lanes = int(re.search(r'for \(int g = g0 \+ lane; g < g1; g \+= (\d+)\)', src).group(1))
    warps = int(re.search(r'launch\(ctx, eval_match_kernel, ceil_div\(n_seg, (\d+)\), (\d+),', src).group(1))
    chunk = int(re.search(r'for \(int base = lo; base < hi; base \+= (\d+)\)', src).group(1))
    return lanes, warps, chunk


LANES, WARPS_PER_CTA, CHUNK = _constants()


def case(name, labels, preds, n_classes, thr=0.5, border='include', neutral=None, ids=None, gt_format=None):
    return dict(name=name, labels=labels, preds=preds, n_classes=n_classes, thr=thr, border=border, neutral=neutral,
                ids=list(range(len(labels))) if ids is None else ids, gt_format=gt_format)


def oracle(c):
    return eo.evaluate(c['labels'], c['preds'], c['n_classes'], c['ids'], c['neutral'], c['thr'], c['border'], c['gt_format'])


def old_overlaps(gt, pred_box, d):
    """The arithmetic the kernel had before: float64 throughout, the predicted area included."""
    g, b = np.asarray(gt, np.float64), np.asarray(pred_box, np.float32).astype(np.float64)[None, :]
    with np.errstate(invalid='ignore', divide='ignore', over='ignore'):
        return _old_iou(g, b, d)


def _old_iou(g, b, d):
    side = np.maximum(0, np.minimum(g[:, [2, 3]], b[:, [2, 3]]) - np.maximum(g[:, [0, 1]], b[:, [0, 1]]))
    inter = side[:, 0] * side[:, 1]
    return inter / ((g[:, 2] - g[:, 0] + d) * (g[:, 3] - g[:, 1] + d) + (b[:, 2] - b[:, 0] + d) * (b[:, 3] - b[:, 1] + d) - inter)


# -- builders ------------------------------------------------------------------------------------------------------------
def _bisect_onto(gt, thr, d, rng, f32):
    """A float32 predicted box whose IoU with ``gt`` (4,) lies on ``thr``: a jittered copy slid right, the slide bisected in
    float64 to the threshold, then rounded to float32.  With ``f32`` the box is nudged by a few float32 ulps of xmax to an IoU
    exactly equal to float32(thr) in float32 arithmetic where one exists (the case a float64 threshold gets wrong)."""
    g = np.asarray(gt, np.float64)
    w, h = g[2] - g[0], g[3] - g[1]
    base = g + rng.normal(0, 0.03, 4) * np.array([w, h, w, h])
    iou = lambda t: old_overlaps(g[None], np.array([base[0] + t, base[1], base[2] + t, base[3]]), d)[0]   # noqa: E731
    lo, hi = 0.0, 2.0 * w + 4.0
    if not iou(lo) > thr:
        return None
    for _ in range(80):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if iou(mid) > thr else (lo, mid)
    p = np.array([base[0] + lo, base[1], base[2] + lo, base[3]], np.float32)
    if f32:
        gt32 = g.astype(np.float32)[None]
        for k in range(-6, 7):
            q = p.copy()
            q[2] = np.nextafter(p[2], np.float32(np.inf if k > 0 else -np.inf)) if k else p[2]
            for _ in range(abs(k) - 1):
                q[2] = np.nextafter(q[2], np.float32(np.inf if k > 0 else -np.inf))
            if eo.overlaps(gt32, q, d)[0] == np.float32(thr):
                return q
    return p


def near_threshold(name, n, dtype, thr, border, seed, decimals=None):
    """``n`` images with one class-1 box each and one prediction bisected onto ``thr``."""
    rng = np.random.default_rng(seed)
    d = eo.BORDER_D[border]
    labels, preds = [], [[], []]
    f32 = np.result_type(dtype, np.float32) == np.float32
    while len(labels) < n:
        x0, y0 = rng.uniform(0, 200, 2)
        g = np.array([x0, y0, x0 + rng.uniform(20, 180), y0 + rng.uniform(20, 180)])
        g = np.round(g, decimals) if decimals is not None else np.floor(g)
        lab = np.array([[1, *g]]).astype(dtype)
        p = _bisect_onto(lab[0, 1:], thr, d, rng, f32)
        if p is None:
            continue
        preds[1].append((len(labels), float(np.float32(rng.uniform(0.01, 1))), *(float(v) for v in p)))
        labels.append(lab)
    return case(name, labels, preds, 1, thr, border)


def regression_example():
    """One prediction on which the float64 predicted area gave FP where the reference gives TP (IoU 0.5000000034554928 in
    the reference's arithmetic, 0.4999999962302931 with a float64 predicted area)."""
    lab = [np.array([[1, 32, 89, 208, 234]], np.int64)]
    p = [[], [(0, 0.9, 30.85151481628418, 91.00242614746094, 124.6299819946289, 236.61366271972656)]]
    return case('regression_i64', lab, p, 1, 0.5, 'include')


def mixed_dtypes(name, thr, border, seed=11):
    """Images of every label dtype in one dataset, int16 boxes past sqrt(32767) so that their areas wrap."""
    rng = np.random.default_rng(seed)
    dtypes = [np.int64, np.int32, np.int16, np.float16, np.float32, np.float64]
    labels, preds = [], [[] for _ in range(4)]
    for i in range(36):
        dt = dtypes[i % len(dtypes)]
        g = int(rng.integers(1, 6))
        if dt is np.int16:
            x0, y0 = rng.integers(0, 40, g), rng.integers(0, 40, g)
            b = np.stack([x0, y0, x0 + rng.integers(180, 260, g), y0 + rng.integers(180, 260, g)], 1).astype(np.float64)
        else:
            x0, y0 = rng.uniform(0, 200, g), rng.uniform(0, 200, g)
            b = np.stack([x0, y0, x0 + rng.uniform(8, 120, g), y0 + rng.uniform(8, 120, g)], 1)
            b = np.round(b * 2) / 2 if dt in (np.float16, np.float32, np.float64) else np.floor(b)
        lab = np.concatenate([rng.integers(1, 4, (g, 1)), b], 1).astype(dt)
        labels.append(lab)
        for _ in range(int(rng.integers(2, 8))):
            j = int(rng.integers(0, g))
            q = lab[j, 1:].astype(np.float64) + rng.normal(0, 4, 4)
            c = int(lab[j, 0]) if rng.uniform() < 0.85 else int(rng.integers(1, 4))
            preds[c].append((i, float(np.float32(rng.uniform(0.01, 1))), *(round(float(v), 1) for v in q)))
    return case(name, labels, preds, 3, thr, border)


def _exact_iou(g, p, d):
    side = [max(Fraction(0), min(g[2 + k], p[2 + k]) - max(g[k], p[k])) for k in (0, 1)]
    inter = side[0] * side[1]
    union = (g[2] - g[0] + d) * (g[3] - g[1] + d) + (p[2] - p[0] + d) * (p[3] - p[1] + d) - inter
    return None if union == 0 else inter / union


def dyadic(name, border, dtype, seed):
    """Boxes on a (half-)pixel grid whose IoU is exactly 1/2 in rational arithmetic, so every step is exact in both types:
    a prediction sharing the ground truth's y range and its left edge, its width c solved from 3 c h = (a + c + 2 d)(h + d)
    for the ground truth's width a; then shifted, x and y swapped at random, and sometimes the two boxes exchanged."""
    rng = np.random.default_rng(seed)
    d = eo.BORDER_D[border]
    s = 1 if np.issubdtype(dtype, np.integer) else 2
    labels, preds = [], [[], []]
    while len(labels) < 40:
        h, c = Fraction(int(rng.integers(2, 24 * s)), s), Fraction(int(rng.integers(1, 24 * s)), s)
        if h + d <= 0:
            continue
        a = 3 * c * h / (h + d) - c - 2 * d
        if (a * s).denominator != 1 or not c < a < 40:
            continue
        x, y = Fraction(int(rng.integers(0, 80 * s)), s), Fraction(int(rng.integers(0, 80 * s)), s)
        g, p = [x, y, x + a, y + h], [x, y, x + c, y + h]
        if rng.uniform() < 0.5:
            g, p = [g[1], g[0], g[3], g[2]], [p[1], p[0], p[3], p[2]]
        if rng.uniform() < 0.5:
            g, p = p, g
        assert _exact_iou(g, p, d) == Fraction(1, 2)
        labels.append(np.array([[1] + [float(v) for v in g]]).astype(dtype))
        preds[1].append((len(labels) - 1, 0.5, *(float(v) for v in p)))
    return case(name, labels, preds, 1, 0.5, border)


def lanes_nan_tie(name, border):
    """Ties and NaNs across lanes, neutral arg-maxes, duplicates (float64 labels, class 1 unless said otherwise).
    image 0: 70 boxes; zero-area boxes at 34 (lane 2) and 65 (lane 1) give NaN overlaps with a zero-area prediction under
             'half', every other box overlaps it by 0: the first NaN, 34, wins, then is a duplicate.
    image 1: identical boxes at 3, 35 (the same lane, a later pass) and 36 (another lane), 35 and 36 neutral: the first
             maximum, 3, is a TP, then a duplicate.
    image 2: a neutral box as the only maximum: neither TP nor FP, twice.
    image 3: width-1 boxes apart: under 'exclude' inter 0 and union 0, NaN.
    image 4: non-finite coordinates in labels and predictions."""
    labels, neutral = [], []
    b = np.array([[1, 100 + 3 * k, 100, 102 + 3 * k, 103] for k in range(70)], np.float64)
    b[34, 1:] = [5, 5, 5, 5]
    b[65, 1:] = [5, 5, 5, 5]
    labels.append(b); neutral.append(np.zeros(70, bool))
    b = np.array([[1, 50 + 2 * k, 50, 60 + 2 * k, 60] for k in range(40)], np.float64)
    b[35] = b[3]
    b[36] = b[3]
    n = np.zeros(40, bool); n[35] = n[36] = True
    labels.append(b); neutral.append(n)
    labels.append(np.array([[1, 0, 0, 10, 10], [1, 20, 20, 30, 30], [2, 0, 0, 10, 10]], np.float64))
    neutral.append(np.array([True, False, False]))
    labels.append(np.array([[1, 0, 0, 1, 3], [1, 7, 0, 8, 3]], np.float64)); neutral.append(np.zeros(2, bool))
    inf, nan = np.inf, np.nan
    labels.append(np.array([[1, 0, 0, inf, 10], [1, -inf, 0, 10, 10], [1, 0, 0, 10, nan], [1, 20, 20, 30, 30]], np.float64))
    neutral.append(np.zeros(4, bool))
    preds = [[], [(0, 0.9, 5, 5, 5, 5), (0, 0.8, 5, 5, 5, 5), (1, 0.9, 56, 50, 66, 60), (1, 0.7, 56, 50, 66, 60),
                  (2, 0.9, 0, 0, 10, 10), (2, 0.6, 0, 0, 10, 10), (3, 0.9, 2, 0, 3, 3), (3, 0.5, 0, 0, 1, 3),
                  (4, 0.9, 0, 0, 10, 10), (4, 0.8, nan, 0, 10, 10), (4, 0.7, -inf, 0, 10, 10), (4, 0.6, 20, 20, inf, 30),
                  (4, 0.5, 20, 20, 30, 30)],
             [(2, 0.4, 1, 1, 10, 10)]]
    return case(name, labels, preds, 2, 0.5, border, neutral=neutral)


def misc(name, thr=0.5):
    """An empty class (3), images with (0, 5) labels, integer image ids, a permuted gt_format (class id last), a fractional
    class id (1.5: no class, so the prediction on it is FP), equal confidences (input order decides)."""
    fmt = {'xmin': 0, 'ymin': 1, 'xmax': 2, 'ymax': 3, 'class_id': 4}
    labels = [np.array([[10, 10, 50, 50, 1], [60, 60, 90, 90, 2]], np.float32),
              np.zeros((0, 5), np.float32),
              np.array([[10, 10, 50, 50, 1.5], [0, 0, 5, 5, 2]], np.float32),
              np.array([[0, 0, 40, 40, 4], [2, 2, 40, 40, 4], [100, 100, 140, 140, 1]], np.int64),
              np.zeros((0, 5), np.int64)]
    ids = [101, 7, 33, 2024, 5]
    preds = [[], [(101, 0.5, 11, 11, 50, 50), (101, 0.5, 10, 10, 50, 50), (101, 0.5, 10, 10, 49, 50), (7, 0.5, 1, 1, 9, 9),
                  (33, 0.9, 10, 10, 50, 50), (2024, 0.3, 100, 100, 140, 140), (5, 0.2, 0, 0, 9, 9)],
             [(101, 0.8, 60, 60, 90, 90), (33, 0.8, 0, 0, 5, 5), (7, 0.1, 0, 0, 5, 5)],
             [],
             [(2024, 0.6, 1, 1, 40, 40), (2024, 0.6, 1, 1, 40, 40), (2024, 0.6, 0, 0, 40, 40), (33, 0.6, 0, 0, 5, 5)]]
    return case(name, labels, preds, 4, thr, 'include', ids=ids, gt_format=fmt)


def below_minus_one(name):
    """'exclude' with sub-pixel boxes: the union is negative and smaller than the intersection, so every overlap is below
    -1 (2.25 / (0.25 + 0.25 - 2.25)); with a threshold below that the arg-max must still name a box."""
    labels = [np.array([[1, 0, 0, 1.5, 1.5], [1, 0.25, 0.25, 1.75, 1.75]], np.float64),
              np.array([[1, 0, 0, 1.5, 1.5]], np.float32)]
    preds = [[], [(0, 0.9, 0, 0, 1.5, 1.5), (0, 0.8, 0, 0, 1.5, 1.5), (0, 0.7, 0, 0, 1.5, 1.5), (1, 0.9, 0, 0, 1.5, 1.5)]]
    return case(name, labels, preds, 1, -5.0, 'exclude')


EDGE_BUILDERS = {}
for _b in ('include', 'half', 'exclude'):
    for _t in (0.5, 0.45, 0.7, 0.0):
        EDGE_BUILDERS['dtypes_%s_%s' % (_b, _t)] = (lambda b=_b, t=_t: mixed_dtypes('dtypes_%s_%s' % (b, t), t, b))
EDGE_BUILDERS.update({
    'near_i64_include': lambda: near_threshold('near_i64_include', 300, np.int64, 0.5, 'include', 21),
    'near_i64_half_045': lambda: near_threshold('near_i64_half_045', 300, np.int64, 0.45, 'half', 22),
    'near_f32_include': lambda: near_threshold('near_f32_include', 300, np.float32, 0.5, 'include', 23, decimals=1),
    'near_f32_half_045': lambda: near_threshold('near_f32_half_045', 300, np.float32, 0.45, 'half', 24, decimals=1),
    'near_f32_exclude_07': lambda: near_threshold('near_f32_exclude_07', 300, np.float32, 0.7, 'exclude', 25, decimals=1),
    'near_i16_include': lambda: near_threshold('near_i16_include', 200, np.int16, 0.5, 'include', 26),
    'regression_i64': regression_example,
    'dyadic_include_i64': lambda: dyadic('dyadic_include_i64', 'include', np.int64, 31),
    'dyadic_half_f32': lambda: dyadic('dyadic_half_f32', 'half', np.float32, 32),
    'dyadic_exclude_f16': lambda: dyadic('dyadic_exclude_f16', 'exclude', np.float16, 33),
    'lanes_nan_tie_half': lambda: lanes_nan_tie('lanes_nan_tie_half', 'half'),
    'lanes_nan_tie_exclude': lambda: lanes_nan_tie('lanes_nan_tie_exclude', 'exclude'),
    'lanes_nan_tie_thr0': lambda: dict(lanes_nan_tie('lanes_nan_tie_thr0', 'include'), thr=0.0),
    'misc': lambda: misc('misc'),
    'misc_thr0': lambda: misc('misc_thr0', 0.0),
    'below_minus_one': lambda: below_minus_one('below_minus_one'),
})
EDGES = sorted(EDGE_BUILDERS)
# overlaps below -1: the kernel before the arg-max fix indexed its flags at INT_MAX here, so it only runs on a fixed kernel
NEEDS_ARGMAX_FIX = ('below_minus_one',)


def edge(name):
    return EDGE_BUILDERS[name]()


# -- large generated cases (GPU) -----------------------------------------------------------------------------------------
def many_images(name, n_images, n_classes, seed):
    """Thousands of images x 20 classes, mixed float32 / int64 labels: tens of thousands of (class, image) segments."""
    rng = np.random.default_rng(seed)
    labels, preds = [], [[] for _ in range(n_classes + 1)]
    for i in range(n_images):
        g = int(rng.integers(0, 6))
        x0, y0 = rng.integers(0, 250, g), rng.integers(0, 250, g)
        lab = np.stack([rng.integers(1, n_classes + 1, g), x0, y0, x0 + rng.integers(8, 120, g), y0 + rng.integers(8, 120, g)], 1)
        lab = lab.reshape(-1, 5).astype(np.float32 if i % 2 else np.int64)
        labels.append(lab)
        for _ in range(int(rng.integers(0, 24))):
            if g and rng.uniform() < 0.6:
                j = int(rng.integers(0, g))
                q = lab[j, 1:].astype(np.float64) + rng.normal(0, 5, 4)
                c = int(lab[j, 0])
            else:
                xy = rng.uniform(0, 250, 2); q = np.concatenate([xy, xy + rng.uniform(8, 120, 2)])
                c = int(rng.integers(1, n_classes + 1))
            preds[c].append((i, float(np.float32(rng.uniform(0.01, 1))), *(round(float(v), 1) for v in q)))
    return case(name, labels, preds, n_classes, 0.5, 'include')


def crowded(name, seed):
    """Images of 100 same-class boxes (four lane passes) plus a few of other classes, with jittered and exact copies."""
    rng = np.random.default_rng(seed)
    labels, preds = [], [[] for _ in range(4)]
    for i in range(24):
        g = 100 + int(rng.integers(0, 12))
        x0, y0 = rng.uniform(0, 280, g), rng.uniform(0, 280, g)
        cls = np.where(np.arange(g) < 100, 1, rng.integers(2, 4, g))
        lab = np.stack([cls, x0, y0, x0 + rng.uniform(6, 40, g), y0 + rng.uniform(6, 40, g)], 1)
        lab = np.round(lab, 1).astype(np.float64 if i % 3 else np.float32)
        if i % 4 == 0:
            lab[71] = lab[6]                               # a tie across lanes (6 and 71: lanes 6 and 7)
        labels.append(lab)
        for _ in range(60):
            j = int(rng.integers(0, g))
            q = lab[j, 1:].astype(np.float64) + (0 if rng.uniform() < 0.2 else rng.normal(0, 2, 4))
            preds[int(lab[j, 0])].append((i, float(np.float32(rng.uniform(0.01, 1))), *(round(float(v), 1) for v in q)))
    return case(name, labels, preds, 3, 0.5, 'half')


def cumsum_sizes(name, seed):
    """Classes of exactly 1023, 1024, 1025 and 5000 predictions (1, 1, 2 and 5 cumsum chunks), class 5 empty; half of the
    images float32, half int64."""
    rng = np.random.default_rng(seed)
    sizes = {1: 1023, 2: 1024, 3: 1025, 4: 5000, 5: 0}
    n_images = 300
    labels = []
    for i in range(n_images):
        g = int(rng.integers(1, 8))
        x0, y0 = rng.integers(0, 250, g), rng.integers(0, 250, g)
        lab = np.stack([rng.integers(1, 6, g), x0, y0, x0 + rng.integers(8, 100, g), y0 + rng.integers(8, 100, g)], 1)
        labels.append(lab.astype(np.float32 if i % 2 else np.int64))
    preds = [[] for _ in range(6)]
    for c, k in sizes.items():
        for _ in range(k):
            i = int(rng.integers(0, n_images))
            lab = labels[i]
            own = np.nonzero(lab[:, 0] == c)[0]
            if len(own) and rng.uniform() < 0.7:
                q = lab[own[int(rng.integers(0, len(own)))], 1:].astype(np.float64) + rng.normal(0, 4, 4)
            else:
                xy = rng.uniform(0, 250, 2); q = np.concatenate([xy, xy + rng.uniform(8, 100, 2)])
            conf = float(np.float32(round(rng.uniform(0.01, 1), 2)))     # many equal confidences
            preds[c].append((i, conf, *(round(float(v), 1) for v in q)))
    return case(name, labels, preds, 5, 0.5, 'include')


CASE_BUILDERS = {
    'crowded': lambda: crowded('crowded', 41),
    'many_images': lambda: many_images('many_images', 3000, 20, 42),
    'cumsum_sizes': lambda: cumsum_sizes('cumsum_sizes', 43),
    'near_i64_big': lambda: near_threshold('near_i64_big', 6000, np.int64, 0.5, 'include', 44),
    'near_f32_big': lambda: near_threshold('near_f32_big', 6000, np.float32, 0.5, 'half', 45, decimals=1),
    'near_f32_big_07': lambda: near_threshold('near_f32_big_07', 4000, np.float32, 0.7, 'include', 46, decimals=1),
    'regression_i64': regression_example,
    'below_minus_one': lambda: below_minus_one('below_minus_one'),
}
CASES = sorted(CASE_BUILDERS)


def build(name):
    return CASE_BUILDERS[name]()


# -- path model ------------------------------------------------------------------------------------------------------------
REQUIRED = {                                   # path -> the case that reaches it
    'lane_passes_gt_1': 'crowded',
    'tie_across_lanes': 'crowded',
    'nan_across_lanes': 'lanes_nan_tie_half',
    'ctas_over_1024': 'many_images',
    'class_1023': 'cumsum_sizes', 'class_1024': 'cumsum_sizes', 'class_1025': 'cumsum_sizes', 'class_5000': 'cumsum_sizes',
    'cumsum_chunks_1': 'cumsum_sizes', 'cumsum_chunks_2': 'cumsum_sizes', 'cumsum_chunks_5': 'cumsum_sizes',
    'empty_class': 'cumsum_sizes',
    'both_types_one_call': 'many_images',
    'old_arithmetic_flips_f64': 'near_i64_big',
    'old_arithmetic_flips_f32': 'near_f32_big',
    'on_float32_threshold': 'near_f32_big_07',
    'overlap_below_minus_one': 'below_minus_one',
}


def paths(c):
    """The kernel paths case ``c`` reaches, and the number of predictions the kernel's former arithmetic (float64
    throughout, float64 threshold) decided differently, under the names of REQUIRED."""
    f = eo.GT_FORMAT if c['gt_format'] is None else c['gt_format']
    ci, cols = f['class_id'], [f['xmin'], f['ymin'], f['xmax'], f['ymax']]
    d = eo.BORDER_D[c['border']]
    index = {str(i): k for k, i in enumerate(c['ids'])}
    out = set()
    segs, types = set(), set()
    flips = {'f64': 0, 'f32': 0}
    for cls in range(1, c['n_classes'] + 1):
        k = len(c['preds'][cls])
        if k == 0:
            out.add('empty_class')
            continue
        out.add('cumsum_chunks_%d' % math.ceil(k / CHUNK))
        if k in (1023, 1024, 1025, 5000):
            out.add('class_%d' % k)
        for p in c['preds'][cls]:
            img = index[str(p[0])]
            lab = np.asarray(c['labels'][img])
            segs.add((cls, img))
            f32 = np.result_type(lab.dtype, np.float32) == np.float32
            types.add(bool(f32))
            if len(lab) > LANES:
                out.add('lane_passes_gt_1')
            if lab.size == 0:
                continue
            rows = np.nonzero(eo.class_mask(lab[:, ci], cls))[0]
            if len(rows) == 0:
                continue
            box = np.asarray(p[2:6], np.float64).astype(np.float32)
            ov = eo.overlaps(lab[rows][:, cols], box, d)
            j = eo.best_index(ov)
            lanes = rows % LANES
            if np.isnan(ov[j]):
                if (lanes != lanes[j]).any() and lanes[j] != 0:
                    out.add('nan_across_lanes')
            elif len(np.unique(lanes[ov == ov[j]])) > 1:
                out.add('tie_across_lanes')
            if ov[j] < -1 and not eo.below(ov[j], c['thr']):
                out.add('overlap_below_minus_one')
            if f32 and ov[j] == np.float32(c['thr']) and float(ov[j]) < c['thr']:
                out.add('on_float32_threshold')
            old = old_overlaps(lab[rows][:, cols], box, d)
            if eo.below(ov[j], c['thr']) != bool(old[int(np.argmax(old))] < c['thr']):
                flips['f32' if f32 else 'f64'] += 1
    if math.ceil(len(segs) / WARPS_PER_CTA) > 1024:
        out.add('ctas_over_1024')
    if types == {True, False}:
        out.add('both_types_one_call')
    for t, n in flips.items():
        if n:
            out.add('old_arithmetic_flips_' + t)
    return out, flips


def device(c):
    """The package's Evaluator on case ``c``: flags, cumulative counts, counts per class, precisions, recalls, both AP
    modes and both mAPs, under the oracle's keys."""
    import types
    from ssd_keras_b200.eval_utils.average_precision_evaluator import Evaluator
    dg = types.SimpleNamespace(labels=c['labels'], image_ids=c['ids'], eval_neutral=c['neutral'])
    ev = Evaluator(model=None, n_classes=c['n_classes'], data_generator=dg, gt_format=c['gt_format'] or dict(eo.GT_FORMAT))
    ev.prediction_results = c['preds']
    num = ev.get_num_gt_per_class(ret=True)
    tp, fp, ctp, cfp = ev.match_predictions(matching_iou_threshold=c['thr'], border_pixels=c['border'], sorting_algorithm='mergesort',
                                            ret=True)
    prec, rec = ev.compute_precision_recall(verbose=False, ret=True)
    ap_s = ev.compute_average_precisions(mode='sample', verbose=False, ret=True)
    m_s = ev.compute_mean_average_precision()
    ap_i = ev.compute_average_precisions(mode='integrate', verbose=False, ret=True)
    m_i = ev.compute_mean_average_precision()
    return dict(tp=tp, fp=fp, ctp=ctp, cfp=cfp, num_gt=num, prec=prec, rec=rec, ap_sample=ap_s, ap_integrate=ap_i,
                map=np.asarray([m_s, m_i]))


def assert_same(got, want, n_classes, what=''):
    """Bit for bit: the flags and counts are integers, and precision, recall and AP are the same NumPy expressions on them."""
    np.testing.assert_array_equal(got['num_gt'], want['num_gt'], err_msg=what + ' num_gt')
    for k in range(1, n_classes + 1):
        for key in ('tp', 'fp', 'ctp', 'cfp', 'prec', 'rec'):
            np.testing.assert_array_equal(np.asarray(got[key][k]), np.asarray(want[key][k]), err_msg='%s %s class %d' % (what, key, k))
    for key in ('ap_sample', 'ap_integrate', 'map'):
        np.testing.assert_array_equal(np.asarray(got[key], np.float64), np.asarray(want[key], np.float64), err_msg=what + ' ' + key)


def golden(G, name, n_classes):
    """The stored results of edge case ``name`` under the oracle's keys."""
    out = {key: [np.zeros(0, np.int64)] + [G['%s/%s%d' % (name, key, k)] for k in range(1, n_classes + 1)]
           for key in ('tp', 'fp', 'ctp', 'cfp', 'prec', 'rec')}
    for key in ('num_gt', 'ap_sample', 'ap_integrate', 'map'):
        out[key] = G['%s/%s' % (name, key)]
    return out
