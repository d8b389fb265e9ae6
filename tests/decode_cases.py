"""Case table of the decoder tests (tests/test_gpu_decode_paths.py) and a restatement, in Python, of the launch decisions
csrc/decode.cu makes for each case (tests/test_decode_paths_cpu.py checks that together the cases reach every path).

The decoder (``ssdk_decode``) runs one NMS CTA per (image, class) segment.  Each segment takes its candidates (scores that pass
the confidence threshold) in (score descending, index ascending) order, in bands of at most kNmsCap.  A first band of at most
kMaskN candidates is resolved through a pairwise suppression bit matrix; every other band by the general scan, whose kept
boxes are cached in shared memory up to kKeptSm and read from global memory beyond.  With a top_k, stage 1 scans one band of
``stage1_band`` candidates per class and records the key where it stopped; the top-k stage flags the classes that stopped at
or above the image's top_k-th score, and those classes and images are redone with the full scan.  ``SSDK_NMS_TWO_STAGE=0``
always runs the full scan.

Every case is plain data plus a seeded generator, so the GPU test and the CPU model see the same inputs."""
import functools
import os
import re

import numpy as np

from oracle import decoder as odec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DECODE_CU = os.path.join(ROOT, 'ssd_keras_b200', 'csrc', 'decode.cu')


def kernel_constants():
    """The launch constants of csrc/decode.cu, read from the source so that this model cannot drift from the kernel."""
    with open(DECODE_CU) as f:
        src = f.read()
    return {k: int(v) for k, v in re.findall(r'constexpr int (k\w+) = (\d+);', src)}


_K = kernel_constants()
NMS_CAP, KEPT_SM, MASK_N, TOP_CAP = _K['kNmsCap'], _K['kKeptSm'], _K['kMaskN'], _K['kTopCap']
VAR = (0.1, 0.1, 0.2, 0.2)


# ------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def ssd300_anchors():
    """The 8732 normalised centroid anchors of SSD300 (the layout of models/keras_ssd300.py), float32."""
    from oracle.anchors import all_anchors
    from oracle.model import SSD300_AR
    a = all_anchors(300, 300, [(38, 38), (19, 19), (10, 10), (5, 5), (3, 3), (1, 1)], [0.1, 0.2, 0.37, 0.54, 0.71, 0.88, 1.05],
                    SSD300_AR, two_boxes_for_ar1=True, steps=[8, 16, 32, 64, 100, 300], offsets=[0.5] * 6).astype(np.float32)
    a.setflags(write=False)
    return a


def corners_of(anc):
    """Centroid anchors (cx, cy, w, h) -> corners (x0, y0, x1, y1), float32."""
    c = np.empty_like(anc)
    c[:, 0] = anc[:, 0] - anc[:, 2] / 2; c[:, 1] = anc[:, 1] - anc[:, 3] / 2
    c[:, 2] = anc[:, 0] + anc[:, 2] / 2; c[:, 3] = anc[:, 1] + anc[:, 3] / 2
    return c


def minmax_of(anc):
    c = corners_of(anc)
    return c[:, [0, 2, 1, 3]].copy()


def make_y(scores, offsets, anc, variances=VAR):
    """y_pred (B, P, C + 12) float32 from scores (B, P, C), offsets (B, P, 4) and anchors (P, 4) or (B, P, 4)."""
    B, P, _ = scores.shape
    anc = np.broadcast_to(np.asarray(anc, np.float32), (B, P, 4))
    var = np.broadcast_to(np.asarray(variances, np.float32), (B, P, 4))
    return np.concatenate([scores, offsets, anc, var], axis=-1).astype(np.float32)


def _rescan_batch():
    """SSD300, 21 classes, three images.  Image 0: 1100 priors share one box (jitter 1e-3) and hold the 1100 best class-1
    scores, so stage 1 keeps 1 of its 256 class-1 candidates and must re-scan that class.  Image 1: plain random scores, every
    class is cut short but stops far below the image's 200th detection.  Image 2: class 7 in image 0's role."""
    rng = np.random.default_rng(71)
    anc = ssd300_anchors()
    B, P, C = 3, anc.shape[0], 21
    sc = rng.uniform(0.0, 0.5, (B, P, C)).astype(np.float32)
    sc[1] = rng.uniform(0.0, 1.0, (P, C))
    off = (rng.standard_normal((B, P, 4)) * 0.3).astype(np.float32)
    a = np.broadcast_to(anc, (B, P, 4)).copy()
    for b, cls in ((0, 1), (2, 7)):
        pri = rng.choice(P, 1100, replace=False)
        sc[b, pri, cls] = rng.uniform(0.9, 0.95, 1100)
        a[b, pri] = anc[pri[0]]
        off[b, pri] = rng.standard_normal((1100, 4)) * 1e-3
    return make_y(sc, off, a)


def _random_ssd300(seed, B=1, C=21, lo=0.0, hi=1.0, loc=0.3):
    rng = np.random.default_rng(seed)
    anc = ssd300_anchors()
    sc = rng.uniform(lo, hi, (B, anc.shape[0], C)).astype(np.float32)
    off = (rng.standard_normal((B, anc.shape[0], 4)) * loc).astype(np.float32)
    return make_y(sc, off, anc)


def _flat(seed, coords, C=3, levels=4, B=1):
    """Every prior passes the threshold in every class; scores take one of ``levels`` values, so runs of thousands of equal
    scores straddle every band edge.  Anchors in the given coordinate format."""
    rng = np.random.default_rng(seed)
    anc = ssd300_anchors()
    P = anc.shape[0]
    a = {'centroids': anc, 'corners': corners_of(anc), 'minmax': minmax_of(anc)}[coords]
    sc = (np.float32(0.25) + rng.integers(0, levels, (B, P, C)).astype(np.float32) * np.float32(1 / 64)).astype(np.float32)
    off = (rng.standard_normal((B, P, 4)) * 0.3).astype(np.float32)
    return make_y(sc, off, a)


def _grid_boxes(n, coords):
    """n disjoint unit-spaced boxes as anchors in ``coords`` format with zero offsets: they decode to themselves exactly."""
    x0 = (np.arange(n) * 4).astype(np.float32)
    c = np.stack([x0, np.zeros(n, np.float32), x0 + 2, np.full(n, 2, np.float32)], 1)
    return _anchor_rows(c, coords)


def _anchor_rows(c, coords):
    c = np.asarray(c, np.float32)
    if coords == 'corners':
        return c
    if coords == 'minmax':
        return c[:, [0, 2, 1, 3]].copy()
    return np.stack([(c[:, 0] + c[:, 2]) / 2, (c[:, 1] + c[:, 3]) / 2, c[:, 2] - c[:, 0], c[:, 3] - c[:, 1]], 1).astype(np.float32)


THRESHOLDS = (0.5, 0.3, 0.01)


def threshold_scores(thr):
    """Scores at, just below and just above float32(thr), and thr's two float32 neighbours."""
    t = np.float32(thr)
    dn, up = np.nextafter(t, np.float32(0)), np.nextafter(t, np.float32(1))
    return np.array([t, dn, up, t, np.nextafter(dn, np.float32(0)), np.nextafter(up, np.float32(1))], np.float32)


def threshold_input(thr, coords):
    """Twelve disjoint boxes: the first six take threshold_scores(thr) in class 1, the last six in class 2; everything else 0."""
    s = threshold_scores(thr)
    P = 2 * s.size
    sc = np.zeros((1, P, 3), np.float32)
    sc[0, :s.size, 1] = s
    sc[0, s.size:, 2] = s
    return make_y(sc, np.zeros((1, P, 4), np.float32), _grid_boxes(P, coords), (1.0, 1.0, 1.0, 1.0))


def nan_score_input(coords):
    """Rows whose class vector holds a NaN: before, after and instead of the largest score, and in the background slot."""
    rows = np.array([[0.1, np.nan, 0.9, 0.2],
                     [0.1, 0.9, np.nan, 0.2],
                     [np.nan, 0.9, 0.2, 0.1],
                     [0.1, 0.2, 0.3, np.nan],
                     [0.0, 0.8, 0.1, 0.1],                    # a plain row, for contrast
                     [0.1, np.nan, np.nan, 0.7]], np.float32)
    P = rows.shape[0]
    return make_y(rows[None], np.zeros((1, P, 4), np.float32), _grid_boxes(P, coords), (1.0, 1.0, 1.0, 1.0))


def iou_half_input(coords):
    """Box A = [0,0,2,1] (0.9), B = [0,0,1,1] (0.8), IoU(A, B) = 0.5 exactly with border 'half'; C far away (0.7)."""
    c = np.array([[0, 0, 2, 1], [0, 0, 1, 1], [10, 10, 12, 11]], np.float32)
    sc = np.zeros((1, 3, 3), np.float32)
    sc[0, :, 1] = [0.9, 0.8, 0.7]
    sc[0, :, 2] = [0.6, 0.7, 0.8]
    return make_y(sc, np.zeros((1, 3, 4), np.float32), _anchor_rows(c, coords), (1.0, 1.0, 1.0, 1.0))


def one_pixel_input():
    """1-pixel and 0-pixel corner boxes: their IoU depends on border_pixels (areas use d, the intersection does not)."""
    c = np.array([[10, 10, 11, 11], [10, 10, 11, 11], [10, 10, 10, 11], [11, 10, 12, 11], [10, 10, 12, 12], [10, 11, 11, 11],
                  [10, 10, 10, 10]], np.float32)
    n = c.shape[0]
    sc = np.zeros((1, n, 3), np.float32)
    sc[0, :, 1] = np.linspace(0.9, 0.3, n)
    sc[0, :, 2] = np.linspace(0.3, 0.9, n)
    return make_y(sc, np.zeros((1, n, 4), np.float32), c, (1.0, 1.0, 1.0, 1.0))


def nonfinite_input(coords):
    """exp overflow (w and h infinite), NaN offsets, NaN scores, zero-area boxes and swapped corners among ordinary boxes."""
    rng = np.random.default_rng(91)
    P = 64
    base = np.concatenate([rng.uniform(0, 20, (P, 2)), rng.uniform(0, 20, (P, 2))], 1).astype(np.float32)
    c = np.concatenate([base[:, :2], base[:, :2] + 1 + np.abs(base[:, 2:]) / 4], 1)
    anc = _anchor_rows(c, coords)
    sc = rng.uniform(0, 1, (1, P, 3)).astype(np.float32)
    off = (rng.standard_normal((1, P, 4)) * 0.1).astype(np.float32)
    off[0, 0:4, 2:] = 500.0                                   # centroids: exp(100) = inf
    off[0, 4:6, 3] = -500.0                                   # centroids: exp(-100) = 0 -> zero height
    off[0, 6:8, :] = np.nan                                   # NaN box
    off[0, 8:10, 0] = 300.0                                   # corners / minmax: x0 far beyond x1 (swapped)
    sc[0, 10:13, 1] = np.nan                                  # NaN scores
    sc[0, 13, :] = np.nan
    sc[0, 14, 0] = np.nan
    anc[14:16] = anc[16]                                      # duplicates of one box
    sc[0, 0:16, 1] += 0.5                                     # the odd rows lead class 1
    return make_y(sc, off, anc, (1.0, 1.0, 1.0, 1.0))


# ------------------------------------------------------------------------------------------------
# the case table
# ------------------------------------------------------------------------------------------------
def case(name, api, fast, make, conf, iou, top_k, cap=400, coords='centroids', norm=True, H=300, W=300, border='half'):
    """api: 'layer' (DecodeDetections / DecodeDetectionsFast) or 'numpy' (decode_detections / decode_detections_fast)."""
    return dict(name=name, api=api, fast=fast, make=make, conf=conf, iou=iou, top_k=top_k, cap=cap, coords=coords, norm=norm,
                H=H, W=W, border=border)


def _cases():
    out = [
        case('rescan_mixed', 'layer', False, _rescan_batch, 0.01, 0.45, 200),
        case('rescan_mixed_fast', 'layer', True, _rescan_batch, 0.01, 0.45, 200),
        case('rescan_mixed_numpy', 'numpy', False, _rescan_batch, 0.01, 0.45, 200),
        case('cap10', 'layer', False, lambda: _random_ssd300(72), 0.01, 0.45, 200, cap=10),
        case('cap10_fast', 'layer', True, lambda: _random_ssd300(72), 0.01, 0.45, 200, cap=10),
        case('flat_all_corners', 'numpy', False, lambda: _flat(73, 'corners'), 0.01, 0.45, 'all', coords='corners'),
        case('flat_all_centroids', 'numpy', False, lambda: _flat(73, 'centroids'), 0.01, 0.45, 'all'),
        case('flat_all_fast_minmax', 'numpy', True, lambda: _flat(74, 'minmax', C=4), 0.01, 0.45, 'all', coords='minmax'),
        case('flat_topk3000_centroids', 'numpy', False, lambda: _flat(73, 'centroids'), 0.01, 0.45, 3000),
        case('ties_fast_topk3000', 'layer', True, lambda: _flat(75, 'centroids', C=21, levels=3), 0.01, 0.45, 3000, cap=3000),
        case('topk16384', 'layer', False, lambda: _random_ssd300(76, lo=0.02, hi=0.06), 0.01, 0.45, TOP_CAP),
        case('topk16384_numpy_fast', 'numpy', True, lambda: _random_ssd300(77, C=5), 0.01, 0.45, TOP_CAP),
        case('nms_off_topk200_fast', 'numpy', True, lambda: _random_ssd300(79, C=5), 0.01, 0.0, 200),
        case('small_topk_class_major', 'numpy', False, lambda: _random_ssd300(78, B=2, C=4, lo=0.0, hi=0.2), 0.19, 0.45, 200),
    ]
    for thr in THRESHOLDS:
        for coords in ('centroids', 'corners', 'minmax'):
            for fast in (False, True):
                out.append(case('thr%g_numpy_%s%s' % (thr, coords, '_fast' if fast else ''), 'numpy', fast,
                                functools.partial(threshold_input, thr, coords), thr, 0.45, 200, coords=coords, norm=False))
        for fast in (False, True):
            out.append(case('thr%g_layer%s' % (thr, '_fast' if fast else ''), 'layer', fast,
                            functools.partial(threshold_input, thr, 'centroids'), thr, 0.45, 20, norm=False))
    for coords in ('centroids', 'corners'):
        for fast in (False, True):
            for api in ('numpy', 'layer'):
                if api == 'layer' and coords != 'centroids':
                    continue
                sfx = '%s_%s%s' % (api, coords, '_fast' if fast else '')
                out.append(case('nan_scores_' + sfx, api, fast, functools.partial(nan_score_input, coords), 0.01, 0.45, 20,
                                coords=coords, norm=False))
                out.append(case('nonfinite_' + sfx, api, fast, functools.partial(nonfinite_input, coords), 0.05, 0.45, 50,
                                coords=coords, norm=False))
                if api == 'numpy' and fast:                   # iou_threshold 0: no NMS, non-finite boxes stay
                    out.append(case('nonfinite_iou0_' + sfx, api, fast, functools.partial(nonfinite_input, coords), 0.05, 0.0,
                                    50, coords=coords, norm=False))
                for iou in (0.5, 0.0, -0.1):
                    out.append(case('iou_half_%g_%s' % (iou, sfx), api, fast, functools.partial(iou_half_input, coords), 0.01,
                                    iou, 20, coords=coords, norm=False))
    for border in ('half', 'include', 'exclude'):
        for fast in (False, True):
            out.append(case('one_pixel_%s%s' % (border, '_fast' if fast else ''), 'numpy', fast, one_pixel_input, 0.01, 0.45,
                            20, coords='corners', norm=False, border=border))
    return out


CASES = _cases()
BY_NAME = {c['name']: c for c in CASES}
assert len(BY_NAME) == len(CASES)


@functools.lru_cache(maxsize=None)
def inputs(name):
    y = BY_NAME[name]['make']()
    y.setflags(write=False)
    return y


# ------------------------------------------------------------------------------------------------
# exact references
# ------------------------------------------------------------------------------------------------
def reference(c, y):
    """The exact expected output of one case: (rows (B, max_out, 6) float32, prior index (B, max_out), counts (B,)), shaped as
    ssdk_decode writes them.  Layer: the oracle's layer restatement with the kernel's exp.  NumPy API: the oracle's full survivor
    list (class-major, NMS order); when more than top_k survive, the kernel's documented choice among them -- confidence
    descending, ties in that class-major order."""
    if c['api'] == 'layer':
        fn = odec.decode_layer_fast if c['fast'] else odec.decode_layer
        out, idx = fn(y, c['conf'], c['iou'], c['top_k'], c['cap'], c['norm'], c['H'], c['W'], return_indices=True,
                      nms=odec.tf_nms_c, exp=odec.exp_cr)
        return out, idx, (idx >= 0).sum(axis=1)
    B, P, Wd = y.shape
    fn = odec.decode_detections_fast if c['fast'] else odec.decode_detections
    with np.errstate(all='ignore'):
        full, fidx = fn(y, c['conf'], c['iou'], 'all', c['coords'], c['norm'], c['H'], c['W'], c['border'], exp=odec.exp_cr,
                        return_index=True)
    if c['top_k'] == 'all':
        max_out = P * (Wd - 13) if not c['fast'] else P
    else:
        max_out = c['top_k']
    out = np.zeros((B, max_out, 6), np.float32)
    idx = np.full((B, max_out), -1, np.int64)
    counts = np.zeros(B, np.int64)
    for b in range(B):
        rows = np.asarray(full[b], np.float64).reshape(-1, 6)
        ri = np.asarray(fidx[b], np.int64)
        if c['top_k'] != 'all' and rows.shape[0] > c['top_k']:
            o = np.argsort(-rows[:, 1], kind='stable')[:c['top_k']]
            rows, ri = rows[o], ri[o]
        k = rows.shape[0]
        out[b, :k] = rows.astype(np.float32)
        idx[b, :k] = ri
        counts[b] = k
    return out, idx, counts


# ------------------------------------------------------------------------------------------------
# the launch decisions of csrc/decode.cu, restated
# ------------------------------------------------------------------------------------------------
def stage1_band(S, top_k):
    want, b = 4 * top_k // max(S, 1), 256
    while b < want and b < NMS_CAP:
        b <<= 1
    return b


def okey(s):
    """The order-preserving key of a float32 score (okey in decode.cu)."""
    b = np.asarray(s, np.float32).view(np.uint32).astype(np.uint64)
    return np.where(b & 0x80000000, ~b & 0xFFFFFFFF, b | 0x80000000).astype(np.uint64)


def launch(c, y):
    """Host-side decisions of run_nms_topk: S, cap, kmax, the stage-1 band and whether the two stages run."""
    B, P, Wd = y.shape
    Ctot = Wd - 12
    layer = c['api'] == 'layer'
    S = 1 if c['fast'] else Ctot - 1
    top_k = 0 if c['top_k'] == 'all' else int(c['top_k'])
    cap = int(c['cap']) if layer else P
    if 0 < top_k < cap:
        cap = top_k
    band1 = stage1_band(S, top_k)
    two_stage = top_k > 0 and P > band1 and band1 < NMS_CAP
    if layer:
        inst = 'float,layer'
    else:
        inst = 'float,numpy' if c['coords'] == 'corners' else 'double,numpy'
    return dict(B=B, P=P, S=S, layer=layer, top_k=top_k, cap=cap, kmax=cap, band1=band1, two_stage=two_stage, inst=inst)


def segments(c, y):
    """Per image and segment: candidate prior indices in scan order, their float32 scores, and the boxes in the NMS's dtype."""
    L = launch(c, y)
    Ctot = y.shape[2] - 12
    with np.errstate(all='ignore'):
        if L['layer']:
            boxes = odec._layer_boxes(y, c['norm'], c['H'], c['W'], odec.exp_cr)
        else:
            boxes = odec._decode_boxes_inplace(np.copy(y[:, :, -12:-8]), y, c['coords'], (0, 1, 2, 3), odec.exp_cr)
            if c['norm']:
                boxes[:, :, [0, 2]] *= c['W']
                boxes[:, :, [1, 3]] *= c['H']
    dt = boxes.dtype
    out = []
    for b in range(L['B']):
        if c['fast']:
            cls = np.argmax(y[b, :, :Ctot], axis=-1)
            scs = [np.max(y[b, :, :Ctot], axis=-1)]
            lab_ok = [cls != 0]
        else:
            scs = [y[b, :, k] for k in range(1, Ctot)]
            lab_ok = [np.ones(y.shape[1], bool)] * (Ctot - 1)
        segs = []
        for s, ok in zip(scs, lab_ok):
            with np.errstate(invalid='ignore'):
                if L['layer']:
                    pas = s > np.float32(c['conf'])
                elif c['fast']:
                    pas = s.astype(dt) >= c['conf']
                else:
                    pas = s.astype(dt) > c['conf']
            m = np.nonzero(pas & ok)[0]
            m = m[np.lexsort((m, -s[m].astype(np.float64)))]
            segs.append((m, s[m]))
        out.append(segs)
    return L, boxes, out


def _nms_order(c, L, boxes_b, m, sc):
    """Greedy NMS over candidates already in scan order; returns the positions (into m) that survive, capped at L['cap']."""
    if m.size == 0:
        return np.zeros(0, np.int64)
    if L['layer']:
        return np.asarray(odec.tf_nms_c(boxes_b[m], sc, L['cap'], c['iou']), np.int64)
    if c['fast'] and not c['iou']:
        return np.arange(min(m.size, L['cap']))
    rows = np.concatenate([np.arange(m.size, dtype=boxes_b.dtype)[:, None], sc.astype(boxes_b.dtype)[:, None], boxes_b[m]], 1)
    with np.errstate(all='ignore'):
        kept = odec._nms_rows(rows, 1, 2, c['iou'], 'corners', c['border'])
    return np.asarray(kept, np.float64).reshape(-1, 6)[:, 0].astype(np.int64)[:L['cap']]


def _scan(L, sc, surv, band_cap, max_bands):
    """One segment's scan: bands of band_cap (stop after max_bands if > 0), given the survivors of the full greedy order."""
    R, cap = sc.size, L['cap']
    p = {}
    first = min(R, band_cap)
    if first == 0:
        return p, surv[:0], 0, 0
    p['bitmatrix' if first <= MASK_N else 'general'] = True
    reach = first if max_bands else R                        # candidates the scan may look at
    kept = surv[surv < reach][:cap]
    if kept.size >= cap:                                     # cap reached: the scan stops after that candidate's band
        last = int(kept[cap - 1])
        bands = last // band_cap + 1
        if first <= MASK_N and last % 32 != 31 and last < first - 1:
            p['cap_in_chunk'] = True
        p['cap_hit'] = True
    else:
        bands = -(-reach // band_cap)
    p['bands'] = bands
    for e in range(band_cap, min(bands * band_cap, R - 1) + 1, band_cap):
        if e < R and sc[e - 1] == sc[e]:
            p['tie_band_edge'] = True
    if kept.size > KEPT_SM:
        p['kept_gt_512'] = True
    cut = 0
    if max_bands and R > first and kept.size < cap:
        cut = int(okey(sc[first - 1]))
        cut = cut if cut else 1
    return p, kept, cut, bands


def paths(c, y):
    """Every path of csrc/decode.cu one case reaches, with the default two-stage scan and with SSDK_NMS_TWO_STAGE=0."""
    L, boxes, segs = segments(c, y)
    reached = {'inst:' + L['inst'], 'sem:%s/%s' % ('fast' if c['fast'] else 'per_class', c['api'])}
    if not L['layer'] and c['fast'] and not c['iou']:
        reached.add('nms_off')
    per_image = []
    for b, ss in enumerate(segs):
        full = [_nms_order(c, L, boxes[b], m, sc) for m, sc in ss]
        M = 0
        stage1, cuts = [], []
        for (m, sc), surv in zip(ss, full):
            p, kept, _, bands = _scan(L, sc, surv, NMS_CAP, 0)
            M += kept.size
            reached |= {k for k in p if k != 'bands'}
            if bands >= 3:
                reached.add('bands_ge_3')
            if L['two_stage']:
                p1, kept1, cut, _ = _scan(L, sc, surv, L['band1'], 1)
                reached |= {k for k in p1 if k != 'bands'}
                stage1.append(sc[kept1])
                cuts.append(cut)
                if cut:
                    reached.add('stage1_cut')
                    if sc.size > L['band1'] and sc[L['band1'] - 1] == sc[L['band1']]:
                        reached.add('tie_band_edge')
        top_k = L['top_k']
        if top_k <= 0 or (not L['layer'] and M <= top_k):
            reached.add('emit_class_major' if top_k > 0 else 'emit_all')
        else:
            reached.add('emit_sorted')
            if min(top_k, M) > NMS_CAP:
                reached.add('topk_gt_%d' % NMS_CAP)
            if top_k == TOP_CAP:
                reached.add('topk_%d' % TOP_CAP)
        redo = []
        if L['two_stage']:
            cat = np.concatenate(stage1) if stage1 else np.zeros(0, np.float32)
            M1 = cat.size
            sigma = 0
            if M1 >= top_k and (L['layer'] or M1 > top_k):
                sigma = int(np.sort(okey(cat))[::-1][top_k - 1])
            redo = [bool(ck and not ck < sigma) for ck in cuts]
            if any(redo):
                reached.add('redo')
            if any(ck and not r for ck, r in zip(cuts, redo)):
                reached.add('cut_without_redo')
        per_image.append(any(redo))
    if L['two_stage'] and any(per_image) and not all(per_image):
        reached.add('redo_mixed_batch')
    return L, reached, per_image


# every path the decoder can take, and the case expected to reach it first
REQUIRED = {
    'redo': 'rescan_mixed',
    'cut_without_redo': 'rescan_mixed',
    'redo_mixed_batch': 'rescan_mixed',
    'stage1_cut': 'rescan_mixed',
    'bitmatrix': 'cap10',
    'general': 'cap10',
    'cap_hit': 'cap10',
    'cap_in_chunk': 'cap10',
    'kept_gt_512': 'flat_all_corners',
    'bands_ge_3': 'flat_all_corners',
    'tie_band_edge': 'flat_all_corners',
    'topk_gt_%d' % NMS_CAP: 'flat_topk3000_centroids',
    'topk_%d' % TOP_CAP: 'topk16384',
    'emit_all': 'flat_all_corners',
    'emit_class_major': 'thr0.5_numpy_centroids',
    'emit_sorted': 'rescan_mixed',
    'inst:float,layer': 'rescan_mixed',
    'inst:float,numpy': 'flat_all_corners',
    'inst:double,numpy': 'flat_all_centroids',
    'sem:per_class/layer': 'rescan_mixed',
    'sem:fast/layer': 'rescan_mixed_fast',
    'sem:per_class/numpy': 'rescan_mixed_numpy',
    'sem:fast/numpy': 'flat_all_fast_minmax',
    'nms_off': 'nonfinite_iou0_numpy_centroids_fast',
}
