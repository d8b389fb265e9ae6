"""NumPy restatement of pycocotools' COCO evaluation for iouType 'bbox' (cocoapi ``PythonAPI/pycocotools/coco.py``,
``cocoeval.py`` and the ``bbIou`` of ``common/maskApi.c``), with the per-image Python loops of the original.  Test
infrastructure only: ``ssd_keras_b200.eval_utils.coco_eval`` is held to it.

pycocotools is not installed here and cannot be fetched offline, so this restatement is not compared against the library.  It
is pinned instead by hand-derived cases (``tests/cocoeval_cases.py``), one per rule below, and by the summary lines the
reference's COCO notebook stores.  The rules, each cited to the function it restates:

- ``Params.setDetParams``: ``iouThrs = np.linspace(.5, .95, 10)``, ``recThrs = np.linspace(0, 1, 101)`` (NumPy's exact float64
  values), ``maxDets = [1, 10, 100]``, ``areaRng = [[0, 1e10], [0, 32**2], [32**2, 96**2], [96**2, 1e10]]`` labelled all /
  small / medium / large, ``useCats = 1``; ``COCOeval.__init__`` sets ``imgIds`` / ``catIds`` to the sorted ids of the ground
  truth; ``evaluate`` replaces them by ``np.unique`` of themselves and sorts ``maxDets``.
- ``COCOeval._prepare``: ground truths and detections of ``imgIds`` x ``catIds`` grouped per (image, category), in
  annotation-file order (results order for detections); a ground truth's ``ignore`` is overwritten by
  ``'iscrowd' in gt and gt['iscrowd']``.
- ``COCO.loadRes`` (bbox results from a file name, a list of dicts or an N x 7 array ``[image_id, x, y, w, h, score,
  category_id]``): ``area = bb[2] * bb[3]``, ``id = index + 1``, ``iscrowd = 0``; an image id outside the ground truth fails
  with "Results do not correspond to current coco set".
- ``maskApi.c bbIou``, float64: ``w = fmin(Dx + Dw, Gx + Gw) - fmax(Dx, Gx)``, IoU 0 if ``w <= 0``, ``h`` likewise,
  ``i = w * h``, ``u = crowd ? Dw * Dh : Dw * Dh + Gw * Gh - i``, IoU ``i / u``.  The ground truth's box area is used, not its
  ``'area'``.  ``fmin`` / ``fmax`` ignore a NaN operand.  Python's float arithmetic is IEEE double without contraction, which
  is what the usual x86-64 build of the C extension computes (no FMA).
- ``COCOeval.computeIoU``: detections stable-sorted by ``-score`` and cut to ``maxDets[-1]``.
- ``COCOeval.evaluateImg``: ``None`` for a pair with neither ground truths nor detections; a ground truth is ignored when it is
  a crowd box or ``area < lo or area > hi`` (both bounds inclusive); ground truths stable-sorted ignored-last; per threshold
  ``iou = min(t, 1 - 1e-10)`` and the greedy walk: skip a matched non-crowd box, break from a non-ignored candidate at the
  first ignored box, skip ``ious < iou`` (so the last of equal IoUs wins), else take it.  ``dtIg = gtIg[m]``, ``dtm = gt id``,
  ``gtm = det id``; an unmatched (``dtm == 0``, so also one matched to a ground truth with id 0) detection outside the range is
  ignored.
- ``COCOeval.accumulate``: per (category, area, maxDet) the first ``maxDet`` detections of each image in ``imgIds`` order,
  stable-sorted by ``-score`` (ties: image order, then rank; -0.0 equals 0.0, NaN last); ``npig == 0`` leaves -1;
  ``tp`` / ``fp`` cumulative sums over non-ignored detections, ``rc = tp / npig``, ``pr = tp / (fp + tp + np.spacing(1))``,
  ``recall = rc[-1]`` (0 without detections), ``pr`` made non-increasing from the right, ``precision`` / ``scores`` at
  ``searchsorted(rc, recThrs, 'left')`` until the first index past the end.
- ``COCOeval.summarize``: the twelve ``_summarize`` selections (``stats[0]`` asks for the literal ``maxDets=100``), the mean
  over entries > -1 or -1, and pycocotools' line format.
"""
import copy
import datetime
import json
import time
from collections import defaultdict

import numpy as np


def fmin(a, b):
    """C's fmin: a NaN operand is ignored."""
    if a != a:
        return b
    if b != b:
        return a
    return a if a <= b else b


def fmax(a, b):
    if a != a:
        return b
    if b != b:
        return a
    return a if a >= b else b


def bb_iou(dt, gt, iscrowd):
    """maskApi.c bbIou: (len(dt), len(gt)) float64 IoUs of [x, y, w, h] boxes, one pair at a time."""
    m, n = len(dt), len(gt)
    o = np.zeros((m, n))
    for g in range(n):
        G = [float(v) for v in gt[g]]
        ga = G[2] * G[3]
        crowd = bool(iscrowd[g]) if iscrowd is not None else False
        for d in range(m):
            D = [float(v) for v in dt[d]]
            da = D[2] * D[3]
            w = fmin(D[2] + D[0], G[2] + G[0]) - fmax(D[0], G[0])
            if w <= 0:
                continue
            h = fmin(D[3] + D[1], G[3] + G[1]) - fmax(D[1], G[1])
            if h <= 0:
                continue
            i = w * h
            u = da if crowd else da + ga - i
            with np.errstate(divide='ignore', invalid='ignore'):
                o[d, g] = np.float64(i) / np.float64(u)        # C's division: x / 0 is inf or NaN, not an exception
    return o


class COCO:
    """pycocotools.coco.COCO: the index and the calls COCOeval makes."""

    def __init__(self, dataset=None):
        self.dataset = dataset if dataset is not None else {}
        self.anns, self.imgs, self.cats = {}, {}, {}
        self.imgToAnns = defaultdict(list)
        if dataset is not None:
            self.createIndex()

    def createIndex(self):
        for ann in self.dataset.get('annotations', []):
            self.imgToAnns[ann['image_id']].append(ann)
            self.anns[ann['id']] = ann
        for img in self.dataset.get('images', []):
            self.imgs[img['id']] = img
        for cat in self.dataset.get('categories', []):
            self.cats[cat['id']] = cat

    def getAnnIds(self, imgIds=[], catIds=[]):
        if len(imgIds) != 0:
            anns = [a for i in imgIds if i in self.imgToAnns for a in self.imgToAnns[i]]
        else:
            anns = self.dataset['annotations']
        anns = anns if len(catIds) == 0 else [a for a in anns if a['category_id'] in catIds]
        return [a['id'] for a in anns]

    def getCatIds(self):
        return [c['id'] for c in self.dataset['categories']]

    def getImgIds(self):
        return list(self.imgs.keys())

    def loadAnns(self, ids):
        return [self.anns[i] for i in ids]

    def loadRes(self, resFile):
        res = COCO()
        res.dataset['images'] = [img for img in self.dataset['images']]
        if isinstance(resFile, str):
            with open(resFile) as f:
                anns = json.load(f)
        elif isinstance(resFile, np.ndarray):
            anns = [{'image_id': int(r[0]), 'bbox': [r[1], r[2], r[3], r[4]], 'score': r[5], 'category_id': int(r[6])}
                    for r in resFile]
        else:
            anns = copy.deepcopy(resFile)
        assert type(anns) == list, 'results in not an array of objects'
        annsImgIds = [ann['image_id'] for ann in anns]
        assert set(annsImgIds) == (set(annsImgIds) & set(self.getImgIds())), 'Results do not correspond to current coco set'
        res.dataset['categories'] = copy.deepcopy(self.dataset['categories'])
        for id, ann in enumerate(anns):
            bb = ann['bbox']
            ann['area'] = bb[2] * bb[3]
            ann['id'] = id + 1
            ann['iscrowd'] = 0
        res.dataset['annotations'] = anns
        res.createIndex()
        return res


class Params:
    def __init__(self):
        self.imgIds = []
        self.catIds = []
        self.iouThrs = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
        self.recThrs = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
        self.maxDets = [1, 10, 100]
        self.areaRng = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
        self.areaRngLbl = ['all', 'small', 'medium', 'large']
        self.useCats = 1
        self.iouType = 'bbox'


class COCOeval:
    def __init__(self, cocoGt, cocoDt):
        self.cocoGt, self.cocoDt = cocoGt, cocoDt
        self.evalImgs = []
        self.eval = {}
        self.params = Params()
        self.params.imgIds = sorted(cocoGt.getImgIds())
        self.params.catIds = sorted(cocoGt.getCatIds())
        self.stats = []
        self.ious = {}

    def _prepare(self):
        p = self.params
        gts = self.cocoGt.loadAnns(self.cocoGt.getAnnIds(imgIds=p.imgIds, catIds=p.catIds))
        dts = self.cocoDt.loadAnns(self.cocoDt.getAnnIds(imgIds=p.imgIds, catIds=p.catIds))
        for gt in gts:
            gt['ignore'] = gt['ignore'] if 'ignore' in gt else 0
            gt['ignore'] = 'iscrowd' in gt and gt['iscrowd']
        self._gts = defaultdict(list)
        self._dts = defaultdict(list)
        for gt in gts:
            self._gts[gt['image_id'], gt['category_id']].append(gt)
        for dt in dts:
            self._dts[dt['image_id'], dt['category_id']].append(dt)

    def evaluate(self):
        p = self.params
        p.imgIds = list(np.unique(p.imgIds))
        p.catIds = list(np.unique(p.catIds))
        p.maxDets = sorted(p.maxDets)
        self._prepare()
        self.ious = {(i, c): self.computeIoU(i, c) for i in p.imgIds for c in p.catIds}
        maxDet = p.maxDets[-1]
        self.evalImgs = [self.evaluateImg(i, c, a, maxDet) for c in p.catIds for a in p.areaRng for i in p.imgIds]
        self._paramsEval = copy.deepcopy(self.params)

    def computeIoU(self, imgId, catId):
        p = self.params
        gt, dt = self._gts[imgId, catId], self._dts[imgId, catId]
        if len(gt) == 0 and len(dt) == 0:
            return []
        inds = np.argsort([-d['score'] for d in dt], kind='mergesort')
        dt = [dt[i] for i in inds]
        if len(dt) > p.maxDets[-1]:
            dt = dt[0:p.maxDets[-1]]
        if len(dt) == 0 or len(gt) == 0:
            return []
        return bb_iou([d['bbox'] for d in dt], [g['bbox'] for g in gt], [int(o['iscrowd']) for o in gt])

    def evaluateImg(self, imgId, catId, aRng, maxDet):
        p = self.params
        gt, dt = self._gts[imgId, catId], self._dts[imgId, catId]
        if len(gt) == 0 and len(dt) == 0:
            return None
        for g in gt:
            g['_ignore'] = 1 if (g['ignore'] or (g['area'] < aRng[0] or g['area'] > aRng[1])) else 0
        gtind = np.argsort([g['_ignore'] for g in gt], kind='mergesort')
        gt = [gt[i] for i in gtind]
        dtind = np.argsort([-d['score'] for d in dt], kind='mergesort')
        dt = [dt[i] for i in dtind[0:maxDet]]
        iscrowd = [int(o['iscrowd']) for o in gt]
        ious = self.ious[imgId, catId][:, gtind] if len(self.ious[imgId, catId]) > 0 else self.ious[imgId, catId]
        T, G, D = len(p.iouThrs), len(gt), len(dt)
        gtm = np.zeros((T, G))
        dtm = np.zeros((T, D))
        gtIg = np.array([g['_ignore'] for g in gt])
        dtIg = np.zeros((T, D))
        if not len(ious) == 0:
            for tind, t in enumerate(p.iouThrs):
                for dind, d in enumerate(dt):
                    iou = min([t, 1 - 1e-10])
                    m = -1
                    for gind, g in enumerate(gt):
                        if gtm[tind, gind] > 0 and not iscrowd[gind]:
                            continue
                        if m > -1 and gtIg[m] == 0 and gtIg[gind] == 1:
                            break
                        if ious[dind, gind] < iou:
                            continue
                        iou = ious[dind, gind]
                        m = gind
                    if m == -1:
                        continue
                    dtIg[tind, dind] = gtIg[m]
                    dtm[tind, dind] = gt[m]['id']
                    gtm[tind, m] = d['id']
        a = np.array([d['area'] < aRng[0] or d['area'] > aRng[1] for d in dt]).reshape((1, len(dt)))
        dtIg = np.logical_or(dtIg, np.logical_and(dtm == 0, np.repeat(a, T, 0)))
        return {'image_id': imgId, 'category_id': catId, 'aRng': aRng, 'maxDet': maxDet,
                'dtIds': [d['id'] for d in dt], 'gtIds': [g['id'] for g in gt], 'dtMatches': dtm, 'gtMatches': gtm,
                'dtScores': [d['score'] for d in dt], 'gtIgnore': gtIg, 'dtIgnore': dtIg}

    def accumulate(self, p=None):
        if p is None:
            p = self.params
        T, R, K, A, M = len(p.iouThrs), len(p.recThrs), len(p.catIds), len(p.areaRng), len(p.maxDets)
        precision = -np.ones((T, R, K, A, M))
        recall = -np.ones((T, K, A, M))
        scores = -np.ones((T, R, K, A, M))
        _pe = self._paramsEval
        setK, setA, setM, setI = set(_pe.catIds), set(map(tuple, _pe.areaRng)), set(_pe.maxDets), set(_pe.imgIds)
        k_list = [n for n, k in enumerate(p.catIds) if k in setK]
        m_list = [m for n, m in enumerate(p.maxDets) if m in setM]
        a_list = [n for n, a in enumerate(map(lambda x: tuple(x), p.areaRng)) if a in setA]
        i_list = [n for n, i in enumerate(p.imgIds) if i in setI]
        I0, A0 = len(_pe.imgIds), len(_pe.areaRng)
        for k, k0 in enumerate(k_list):
            Nk = k0 * A0 * I0
            for a, a0 in enumerate(a_list):
                Na = a0 * I0
                for m, maxDet in enumerate(m_list):
                    E = [self.evalImgs[Nk + Na + i] for i in i_list]
                    E = [e for e in E if e is not None]
                    if len(E) == 0:
                        continue
                    dtScores = np.concatenate([e['dtScores'][0:maxDet] for e in E])
                    inds = np.argsort(-dtScores, kind='mergesort')
                    dtScoresSorted = dtScores[inds]
                    dtm = np.concatenate([e['dtMatches'][:, 0:maxDet] for e in E], axis=1)[:, inds]
                    dtIg = np.concatenate([e['dtIgnore'][:, 0:maxDet] for e in E], axis=1)[:, inds]
                    gtIg = np.concatenate([e['gtIgnore'] for e in E])
                    npig = np.count_nonzero(gtIg == 0)
                    if npig == 0:
                        continue
                    tps = np.logical_and(dtm, np.logical_not(dtIg))
                    fps = np.logical_and(np.logical_not(dtm), np.logical_not(dtIg))
                    tp_sum = np.cumsum(tps, axis=1).astype(dtype=np.float64)
                    fp_sum = np.cumsum(fps, axis=1).astype(dtype=np.float64)
                    for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                        tp, fp = np.array(tp), np.array(fp)
                        nd = len(tp)
                        rc = tp / npig
                        pr = tp / (fp + tp + np.spacing(1))
                        q = np.zeros((R,))
                        ss = np.zeros((R,))
                        recall[t, k, a, m] = rc[-1] if nd else 0
                        pr = pr.tolist()
                        q = q.tolist()
                        for i in range(nd - 1, 0, -1):
                            if pr[i] > pr[i - 1]:
                                pr[i - 1] = pr[i]
                        inds = np.searchsorted(rc, p.recThrs, side='left')
                        try:
                            for ri, pi in enumerate(inds):
                                q[ri] = pr[pi]
                                ss[ri] = dtScoresSorted[pi]
                        except IndexError:
                            pass
                        precision[t, :, k, a, m] = np.array(q)
                        scores[t, :, k, a, m] = np.array(ss)
        self.eval = {'params': p, 'counts': [T, R, K, A, M], 'date': datetime.datetime.now().strftime('%Y-%m-%d %H:%M:%S'),
                     'precision': precision, 'recall': recall, 'scores': scores}

    def summarize(self):
        self.stats = summarize(self.params, self.eval)


def summarize(p, ev, out=print):
    """COCOeval.summarize for 'bbox': the twelve stats, each printed with pycocotools' line format."""
    def _summarize(ap=1, iouThr=None, areaRng='all', maxDets=100):
        iStr = ' {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}'
        titleStr = 'Average Precision' if ap == 1 else 'Average Recall'
        typeStr = '(AP)' if ap == 1 else '(AR)'
        iouStr = '{:0.2f}:{:0.2f}'.format(p.iouThrs[0], p.iouThrs[-1]) if iouThr is None else '{:0.2f}'.format(iouThr)
        aind = [i for i, aRng in enumerate(p.areaRngLbl) if aRng == areaRng]
        mind = [i for i, mDet in enumerate(p.maxDets) if mDet == maxDets]
        if ap == 1:
            s = ev['precision']
            if iouThr is not None:
                s = s[np.where(iouThr == p.iouThrs)[0]]
            s = s[:, :, :, aind, mind]
        else:
            s = ev['recall']
            if iouThr is not None:
                s = s[np.where(iouThr == p.iouThrs)[0]]
            s = s[:, :, aind, mind]
        mean_s = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
        out(iStr.format(titleStr, typeStr, iouStr, areaRng, maxDets, mean_s))
        return mean_s
    stats = np.zeros((12,))
    stats[0] = _summarize(1)
    stats[1] = _summarize(1, iouThr=.5, maxDets=p.maxDets[2])
    stats[2] = _summarize(1, iouThr=.75, maxDets=p.maxDets[2])
    stats[3] = _summarize(1, areaRng='small', maxDets=p.maxDets[2])
    stats[4] = _summarize(1, areaRng='medium', maxDets=p.maxDets[2])
    stats[5] = _summarize(1, areaRng='large', maxDets=p.maxDets[2])
    stats[6] = _summarize(0, maxDets=p.maxDets[0])
    stats[7] = _summarize(0, maxDets=p.maxDets[1])
    stats[8] = _summarize(0, maxDets=p.maxDets[2])
    stats[9] = _summarize(0, areaRng='small', maxDets=p.maxDets[2])
    stats[10] = _summarize(0, areaRng='medium', maxDets=p.maxDets[2])
    stats[11] = _summarize(0, areaRng='large', maxDets=p.maxDets[2])
    return stats
