"""MS COCO box evaluation on the device: pycocotools' ``COCO`` / ``COCOeval`` for ``iouType='bbox'``, bit for bit.

A drop-in for the last cell of the reference's ``ssd300_evaluation_COCO.ipynb``::

    from ssd_keras_b200.eval_utils.coco_eval import COCO, COCOeval
    coco_gt = COCO(annotations_file)
    coco_dt = coco_gt.loadRes(results_file)
    cocoEval = COCOeval(cocoGt=coco_gt, cocoDt=coco_dt, iouType='bbox')
    cocoEval.params.imgIds = sorted(coco_gt.getImgIds())
    cocoEval.evaluate(); cocoEval.accumulate(); cocoEval.summarize()

``evaluate()`` is ``evaluateImg`` for every (image, category, area range) in one launch of ``ssdk_cocoeval_match``;
``accumulate()`` is one launch of ``ssdk_cocoeval_accumulate``.  The host groups the columns of the two annotation sets with
stable sorts on the device; the match results stay there between the two calls, and only ``precision`` / ``recall`` /
``scores`` come back.  ``evalImgs`` (pycocotools' list of per-(category, area, image) dicts, ``None`` for absent pairs) is
built from the device arrays when it is first read.  ``summarize()`` is pycocotools' NumPy code on those arrays.

``COCO`` holds what this evaluation uses: ``dataset``, ``getImgIds()``, ``getCatIds()`` and ``loadRes()`` (bbox results from a
file name, a list of dicts or an N x 7 array).  Segmentation and keypoint evaluation and ``useCats = 0`` are not implemented.
Annotation ids are taken to be unique, as pycocotools' index assumes."""
import copy
import ctypes
import datetime
import json
import time

import numpy as np

from .. import _ffi


def _columns(anns, results):
    """The fields evaluation reads, one array per field, in annotation order.  A ground truth without 'iscrowd' counts as not
    crowd (pycocotools' computeIoU would raise KeyError on it)."""
    n = len(anns)
    box = np.asarray([a['bbox'] for a in anns], dtype=np.float64).reshape(n, 4) if n else np.zeros((0, 4))
    cols = {'image_id': np.asarray([a['image_id'] for a in anns]), 'category_id': np.asarray([a['category_id'] for a in anns]),
            'bbox': box, 'id': np.asarray([a['id'] for a in anns], dtype=np.int64)}
    if results:
        with np.errstate(all='ignore'):                   # a non-finite box gives a NaN area, silently, as Python floats do
            cols['area'] = box[:, 2] * box[:, 3]
        cols['score'] = np.asarray([a['score'] for a in anns], dtype=np.float64)
        cols['crowd'] = np.zeros(n, bool)
    else:
        cols['area'] = np.asarray([a['area'] for a in anns], dtype=np.float64)
        cols['crowd'] = np.asarray([bool('iscrowd' in a and a['iscrowd']) for a in anns], dtype=bool)
    return cols


class COCO:
    """The part of pycocotools.coco.COCO that COCOeval and the notebook use."""

    def __init__(self, annotation_file=None):
        self.dataset = {}
        self._results = False
        self._cols = None
        if annotation_file is not None:
            print('loading annotations into memory...')
            tic = time.time()
            with open(annotation_file, 'r') as f:
                dataset = json.load(f)
            assert type(dataset) == dict, 'annotation file format {} not supported'.format(type(dataset))
            print('Done (t={:0.2f}s)'.format(time.time() - tic))
            self.dataset = dataset
            self.createIndex()

    def createIndex(self):
        print('creating index...')
        self._img_ids = list({img['id']: None for img in self.dataset.get('images', [])})
        self._cols = None
        print('index created!')

    def getImgIds(self):
        """The ids of ``dataset['images']`` in file order (the first of repeated ids)."""
        return list(self._img_ids)

    def getCatIds(self):
        return [c['id'] for c in self.dataset.get('categories', [])]

    def columns(self):
        if self._cols is None:
            self._cols = _columns(self.dataset.get('annotations', []), self._results)
        return self._cols

    def loadRes(self, resFile):
        """Detection results as a COCO object: ``area = w * h``, ``id = index + 1``, ``iscrowd = 0``."""
        res = COCO()
        res.dataset['images'] = [img for img in self.dataset['images']]
        print('Loading and preparing results...')
        tic = time.time()
        if isinstance(resFile, str):
            with open(resFile) as f:
                anns = json.load(f)
        elif isinstance(resFile, np.ndarray):
            data = np.asarray(resFile)
            assert data.ndim == 2 and data.shape[1] == 7, 'results array must be N x 7'
            anns = [{'image_id': int(r[0]), 'bbox': [r[1], r[2], r[3], r[4]], 'score': r[5], 'category_id': int(r[6])} for r in data]
        else:
            anns = resFile
        assert type(anns) == list, 'results in not an array of objects'
        if anns and not ('bbox' in anns[0] and anns[0]['bbox'] != []):
            raise NotImplementedError('only bbox results can be evaluated here (segmentation, keypoints and captions cannot)')
        res_ids = np.unique(np.asarray([a['image_id'] for a in anns]))
        assert np.isin(res_ids, np.asarray(self.getImgIds())).all(), 'Results do not correspond to current coco set'
        res.dataset['categories'] = copy.deepcopy(self.dataset['categories'])
        box = np.asarray([a['bbox'] for a in anns], dtype=np.float64).reshape(-1, 4)
        with np.errstate(all='ignore'):
            area = (box[:, 2] * box[:, 3]).tolist()
        for i, ann in enumerate(anns):
            ann['area'] = area[i]
            ann['id'] = i + 1
            ann['iscrowd'] = 0
        print('DONE (t={:0.2f}s)'.format(time.time() - tic))
        res.dataset['annotations'] = anns
        res._results = True
        res.createIndex()
        return res


class Params:
    """COCOeval's parameters for iouType 'bbox' (Params.setDetParams)."""

    def __init__(self, iouType='bbox'):
        if iouType != 'bbox':
            raise NotImplementedError("iouType '{}' is not implemented: only 'bbox' evaluation runs on the device".format(iouType))
        self.imgIds = []
        self.catIds = []
        self.iouThrs = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
        self.recThrs = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
        self.maxDets = [1, 10, 100]
        self.areaRng = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
        self.areaRngLbl = ['all', 'small', 'medium', 'large']
        self.useCats = 1
        self.iouType = iouType
        self.useSegm = None


def _positions(ids, values):
    """Position of each of values in the sorted unique ids, -1 where it is not there."""
    pos = np.searchsorted(ids, values) if len(ids) else np.zeros(len(values), np.int64)
    pos = np.minimum(pos, max(len(ids) - 1, 0))
    ok = (ids[pos] == values) if len(ids) else np.zeros(len(values), bool)
    return np.where(ok, pos, -1)


class COCOeval:
    """pycocotools.cocoeval.COCOeval for iouType 'bbox' with useCats = 1, on the device."""

    def __init__(self, cocoGt=None, cocoDt=None, iouType='bbox'):
        self.cocoGt, self.cocoDt = cocoGt, cocoDt
        self.params = Params(iouType=iouType)
        self.eval = {}
        self.stats = []
        self._paramsEval = {}
        self._dev = None
        self._evalImgs = None
        if cocoGt is not None:
            self.params.imgIds = sorted(cocoGt.getImgIds())
            self.params.catIds = sorted(cocoGt.getCatIds())

    def _check_params(self, p):
        if p.useCats != 1:
            raise NotImplementedError('useCats = 0 is not implemented: evaluation is per category')
        if p.iouType != 'bbox':
            raise NotImplementedError("iouType '{}' is not implemented: only 'bbox' evaluation runs on the device".format(p.iouType))

    # -- evaluate ---------------------------------------------------------------------------------
    def evaluate(self):
        """evaluateImg for every (image, category, area range) of the parameters, as one device launch."""
        import torch
        tic = time.time()
        print('Running per image evaluation...')
        p = self.params
        self._check_params(p)
        print('Evaluate annotation type *{}*'.format(p.iouType))
        p.imgIds = list(np.unique(p.imgIds))
        p.catIds = list(np.unique(p.catIds))
        p.maxDets = sorted(p.maxDets)
        self.params = p
        img_ids, cat_ids = np.asarray(p.imgIds), np.asarray(p.catIds)
        K, A, T = len(cat_ids), len(p.areaRng), len(p.iouThrs)
        max_det = int(p.maxDets[-1])
        dev = torch.device('cuda', torch.cuda.current_device())
        ctx = _ffi.context(dev.index)

        def keyed(cols):
            """Annotations of imgIds x catIds: their indices in file order and their (image position, category position) keys."""
            ip, kp = _positions(img_ids, cols['image_id']), _positions(cat_ids, cols['category_id'])
            sel = np.nonzero((ip >= 0) & (kp >= 0))[0]
            return sel, ip[sel].astype(np.int64) * max(K, 1) + kp[sel]

        gc, dc = self.cocoGt.columns(), self.cocoDt.columns()
        g_sel, g_key = keyed(gc)
        d_sel, d_key = keyed(dc)
        up = lambda a, dt=None: torch.from_numpy(np.ascontiguousarray(a if dt is None else np.asarray(a, dt))).to(dev)
        # ground truths: stable by key, so file order inside a segment
        t_gkey = up(g_key, np.int64)
        g_ord = torch.sort(t_gkey, stable=True).indices
        g_sorted_key = t_gkey[g_ord]
        g_idx = up(g_sel, np.int64)[g_ord]
        gflags = gc['crowd'].astype(np.uint8) | ((gc['id'] == 0).astype(np.uint8) << 1)
        t_gbox = up(gc['bbox'])[g_idx].contiguous()
        t_garea = up(gc['area'])[g_idx].contiguous()
        t_gflags = up(gflags)[g_idx].contiguous()
        # detections: -score stable (-0.0 as 0.0, NaN last), then by segment key, so results order among equal scores
        t_dkey, t_dsel = up(d_key, np.int64), up(d_sel, np.int64)
        t_score = up(dc['score'])[t_dsel]
        o = _score_order(t_score)
        o = o[torch.sort(t_dkey[o] * 2 + torch.isnan(t_score[o]).long(), stable=True).indices]
        d_sorted_key = t_dkey[o]
        n_all = int(o.numel())
        first = torch.ones(n_all, dtype=torch.bool, device=dev)
        if n_all:
            first[1:] = d_sorted_key[1:] != d_sorted_key[:-1]
        pos = torch.arange(n_all, device=dev)
        rank = pos - torch.cummax(torch.where(first, pos, torch.zeros_like(pos)), 0).values if n_all else pos
        keep = rank < max_det
        o_kept, d_rank, d_key_kept = o[keep], rank[keep], d_sorted_key[keep]
        d_idx = t_dsel[o_kept]
        t_dbox = up(dc['bbox'])[d_idx].contiguous()
        t_darea = up(dc['area'])[d_idx].contiguous()
        d_score = t_score[o_kept].contiguous()
        # segments: every key with a ground truth or a detection (before the cut to maxDets[-1])
        seg_key = torch.unique(torch.cat([g_sorted_key, d_sorted_key]))
        n_seg, n_gt, n_det = int(seg_key.numel()), int(g_idx.numel()), int(d_idx.numel())
        i32 = lambda t: t.to(torch.int32).contiguous()
        bound = lambda keys, n: i32(torch.cat([torch.searchsorted(keys, seg_key), torch.tensor([n], device=dev)]))
        seg_gt, seg_det = bound(g_sorted_key, n_gt), bound(d_key_kept, n_det)
        seg_cat = i32(seg_key % max(K, 1))
        # accumulate's order per category: -score stable over the segment order (image, rank), then by category
        d_cat = d_key_kept % max(K, 1)
        a_ord = _score_order(d_score)
        a_ord = a_ord[torch.sort(d_cat[a_ord] * 2 + torch.isnan(d_score[a_ord]).long(), stable=True).indices]
        cat_off = i32(torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), torch.cumsum(torch.bincount(d_cat, minlength=K), 0)]))
        area_rng = up(np.asarray(p.areaRng, np.float64).reshape(A, 2))
        iou_thrs = up(np.asarray(p.iouThrs, np.float64).reshape(T))
        AT = A * T
        r = dict(
            gt_matched=torch.zeros(max(AT * n_gt, 1), dtype=torch.uint8, device=dev),
            det_flags=torch.empty(max(AT * n_det, 1), dtype=torch.uint8, device=dev),
            det_match=torch.empty(max(AT * n_det, 1), dtype=torch.int32, device=dev),
            seg_npig=torch.empty(max(n_seg * A, 1), dtype=torch.int32, device=dev),
            npig=torch.zeros(max(K * A, 1), dtype=torch.int32, device=dev))
        args = _ffi.CocoMatch(n_seg, n_gt, n_det, A, T, *[_ffi.dptr(x).value for x in (
            seg_gt, seg_det, seg_cat, t_gbox, t_garea, t_gflags, t_dbox, t_darea, area_rng, iou_thrs, r['gt_matched'],
            r['det_flags'], r['det_match'], r['seg_npig'], r['npig'])])
        _ffi.check(_ffi.lib().ssdk_cocoeval_match(ctx, ctypes.byref(args), _ffi.stream_ptr()))
        self._dev = dict(r, K=K, A=A, T=T, n_gt=n_gt, n_det=n_det, seg_key=seg_key, seg_gt=seg_gt, seg_det=seg_det,
                         g_idx=g_idx, d_idx=d_idx, d_score=d_score, cat_off=cat_off, ord_det=i32(a_ord),
                         ord_rank=i32(d_rank[a_ord]), ord_score=d_score[a_ord].contiguous())
        self._evalImgs = None
        self._paramsEval = copy.deepcopy(self.params)
        print('DONE (t={:0.2f}s).'.format(time.time() - tic))

    # -- accumulate -------------------------------------------------------------------------------
    def accumulate(self, p=None):
        """Precision [T, R, K, A, M], recall [T, K, A, M] and scores, as one device launch."""
        import torch
        print('Accumulating evaluation results...')
        tic = time.time()
        if self._dev is None:
            raise RuntimeError('Please run evaluate() first')
        if p is None:
            p = self.params
        self._check_params(p)
        _pe, dv = self._paramsEval, self._dev
        if list(p.imgIds) != list(_pe.imgIds) or len(p.iouThrs) != len(_pe.iouThrs):
            raise NotImplementedError('accumulate() takes the image ids and the number of IoU thresholds that evaluate() used')
        T, R, K, A, M = len(p.iouThrs), len(p.recThrs), len(p.catIds), len(p.areaRng), len(p.maxDets)
        setK, setA, setM = set(_pe.catIds), set(map(tuple, _pe.areaRng)), set(_pe.maxDets)
        k_list = [n for n, k in enumerate(p.catIds) if k in setK]
        m_list = [m for n, m in enumerate(p.maxDets) if m in setM]
        a_list = [n for n, a in enumerate(map(lambda x: tuple(x), p.areaRng)) if a in setA]
        if any(k >= dv['K'] for k in k_list) or any(a >= dv['A'] for a in a_list):
            raise IndexError('list index out of range')      # pycocotools indexes its evalImgs with these positions
        dev = dv['npig'].device
        precision = torch.full((T, R, K, A, M), -1.0, dtype=torch.float64, device=dev)
        scores = torch.full((T, R, K, A, M), -1.0, dtype=torch.float64, device=dev)
        recall = torch.full((T, K, A, M), -1.0, dtype=torch.float64, device=dev)
        rec = np.asarray(p.recThrs, np.float64).reshape(R)
        perm = np.argsort(rec, kind='stable')
        small = [torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (
            rec, rec[perm], perm.astype(np.int32), np.asarray(k_list + [0], np.int32), np.asarray(a_list + [0], np.int32),
            np.asarray(m_list + [0], np.int32))]
        args = _ffi.CocoAccumulate(dv['T'], dv['A'], dv['n_det'], R, len(k_list), len(a_list), len(m_list), K, A, M, *[
            _ffi.dptr(x).value for x in (dv['cat_off'], dv['ord_det'], dv['ord_rank'], dv['ord_score'], dv['det_flags'], dv['npig'],
                                         *small, precision, scores, recall)])
        _ffi.check(_ffi.lib().ssdk_cocoeval_accumulate(_ffi.context(dev.index), ctypes.byref(args), _ffi.stream_ptr()))
        self.eval = {'params': p, 'counts': [T, R, K, A, M], 'date': datetime.datetime.now().strftime('%Y-%m-%d %H:%M:%S'),
                     'precision': precision.cpu().numpy(), 'recall': recall.cpu().numpy(), 'scores': scores.cpu().numpy()}
        print('DONE (t={:0.2f}s).'.format(time.time() - tic))

    # -- summarize --------------------------------------------------------------------------------
    def summarize(self):
        """The twelve standard numbers (pycocotools' _summarizeDets), printed in its format; stored in ``stats``."""
        if not self.eval:
            raise Exception('Please run accumulate() first')
        p = self.params

        def _summarize(ap=1, iouThr=None, areaRng='all', maxDets=100):
            iStr = ' {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}'
            titleStr = 'Average Precision' if ap == 1 else 'Average Recall'
            typeStr = '(AP)' if ap == 1 else '(AR)'
            iouStr = '{:0.2f}:{:0.2f}'.format(p.iouThrs[0], p.iouThrs[-1]) if iouThr is None else '{:0.2f}'.format(iouThr)
            aind = [i for i, aRng in enumerate(p.areaRngLbl) if aRng == areaRng]
            mind = [i for i, mDet in enumerate(p.maxDets) if mDet == maxDets]
            if ap == 1:
                s = self.eval['precision']
                if iouThr is not None:
                    s = s[np.where(iouThr == p.iouThrs)[0]]
                s = s[:, :, :, aind, mind]
            else:
                s = self.eval['recall']
                if iouThr is not None:
                    s = s[np.where(iouThr == p.iouThrs)[0]]
                s = s[:, :, aind, mind]
            mean_s = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
            print(iStr.format(titleStr, typeStr, iouStr, areaRng, maxDets, mean_s))
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
        self.stats = stats

    # -- evalImgs ---------------------------------------------------------------------------------
    @property
    def evalImgs(self):
        """pycocotools' per-(category, area range, image) dicts in its order, None for a pair without ground truths or
        detections; built from the device results on first access."""
        if self._evalImgs is None and self._dev is not None:
            self._evalImgs = self._build_eval_imgs()
        return self._evalImgs if self._evalImgs is not None else []

    @evalImgs.setter
    def evalImgs(self, value):
        """An assigned list is what evalImgs returns from then on; accumulate() still reads evaluate()'s device results."""
        self._evalImgs = value

    def _build_eval_imgs(self):
        p, dv = self._paramsEval, self._dev
        K, A, T = dv['K'], dv['A'], dv['T']
        I = len(p.imgIds)
        max_det = p.maxDets[-1]
        host = lambda k: dv[k].cpu().numpy()
        seg_key, seg_gt, seg_det = host('seg_key'), host('seg_gt'), host('seg_det')
        g_idx, d_idx, d_score = host('g_idx'), host('d_idx'), host('d_score')
        n_det = dv['n_det']
        flags = host('det_flags')[:A * T * n_det].reshape(A, T, n_det)
        match = host('det_match')[:A * T * n_det].reshape(A, T, n_det)
        gc, dc = self.cocoGt.columns(), self.cocoDt.columns()
        g_id, g_area, g_crowd = gc['id'][g_idx], gc['area'][g_idx], gc['crowd'][g_idx]
        d_id = dc['id'][d_idx]
        out = [None] * (K * A * I)
        for s, key in enumerate(seg_key.tolist()):
            i, k = divmod(key, K)
            g0, g1, d0, d1 = int(seg_gt[s]), int(seg_gt[s + 1]), int(seg_det[s]), int(seg_det[s + 1])
            for a, rng in enumerate(p.areaRng):
                ig = (g_crowd[g0:g1] | (g_area[g0:g1] < rng[0]) | (g_area[g0:g1] > rng[1])).astype(np.int64)
                gtind = np.argsort(ig, kind='mergesort')
                where = np.empty(len(gtind), np.int64)
                where[gtind] = np.arange(len(gtind))
                m = match[a, :, d0:d1]
                dtm = np.where(m >= 0, g_id[np.maximum(m, g0)].astype(np.float64), 0.0) if g1 > g0 else np.zeros((T, d1 - d0))
                gtm = np.zeros((T, g1 - g0))
                for t in range(T):
                    for dd in range(d1 - d0):
                        if m[t, dd] >= 0:
                            gtm[t, where[m[t, dd] - g0]] = d_id[d0 + dd]
                out[(k * A + a) * I + i] = {
                    'image_id': p.imgIds[i], 'category_id': p.catIds[k], 'aRng': rng, 'maxDet': max_det,
                    'dtIds': d_id[d0:d1].tolist(), 'gtIds': g_id[g0:g1][gtind].tolist(), 'dtMatches': dtm, 'gtMatches': gtm,
                    'dtScores': d_score[d0:d1].tolist(), 'gtIgnore': ig[gtind] if g1 > g0 else np.array([]),
                    'dtIgnore': (flags[a, :, d0:d1] & 2) != 0}
        return out


def _score_order(score):
    """Indices sorting a float64 device tensor by -score, stable, with -0.0 equal to 0.0 and NaN last (np.argsort of -score,
    'mergesort').  The NaN positions are moved last by the caller's next stable sort; here they sort as 0."""
    import torch
    s = score + 0.0                                   # -0.0 + 0.0 is +0.0: one key for both zeros
    key = torch.where(torch.isnan(s), torch.zeros_like(s), -s)
    return torch.sort(key, stable=True).indices
