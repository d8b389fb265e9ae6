"""COCO evaluation cases shared by the CPU tests of the oracle (oracle/cocoeval.py) and the GPU tests of
ssd_keras_b200.eval_utils.coco_eval: small hand-derived datasets, one per rule of pycocotools' COCOeval, and seeded random
COCO-like sets.

A case is a dict: ``gt`` (a COCO ground-truth dataset), ``res`` (a list of bbox results), ``params`` (attributes set on
``COCOeval.params`` before ``evaluate()``) and ``check(ev)``, the hand-derived expectations on an evaluated and accumulated
oracle ``COCOeval``."""
import copy

import numpy as np


def dataset(img_ids, cat_ids, anns):
    """A ground-truth dataset; each ann is (image_id, category_id, [x, y, w, h]) plus optional fields, ids from 1 unless set."""
    out = []
    for n, a in enumerate(anns):
        img, cat, box = a[:3]
        d = {'image_id': img, 'category_id': cat, 'bbox': list(box), 'area': float(box[2] * box[3]), 'iscrowd': 0, 'id': n + 1}
        if len(a) > 3:
            d.update(a[3])
        out.append(d)
    return {'images': [{'id': i} for i in img_ids], 'categories': [{'id': c, 'name': 'c%d' % c} for c in cat_ids],
            'annotations': out}


def det(img, cat, box, score):
    return {'image_id': img, 'category_id': cat, 'bbox': list(box), 'score': score}


def ev_img(ev, img, cat, area=0):
    """The oracle's evalImgs entry of (image id, category id, area index)."""
    p = ev.params
    I, A = len(p.imgIds), len(p.areaRng)
    return ev.evalImgs[(list(p.catIds).index(cat) * A + area) * I + list(p.imgIds).index(img)]


def _equal_ious():
    def check(ev):
        e = ev_img(ev, 1, 1)
        assert (e['dtMatches'] == 2).all()                       # two equal IoUs of 1.0: the later ground truth wins
        assert (e['gtMatches'][:, 0] == 0).all() and (e['gtMatches'][:, 1] == 1).all()
    return dict(gt=dataset([1], [1], [(1, 1, [0, 0, 10, 10]), (1, 1, [0, 0, 10, 10])]), res=[det(1, 1, [0, 0, 10, 10], .9)],
                check=check)


def _iou_at_threshold():
    def check(ev):
        e = ev_img(ev, 1, 1)                                     # IoU 50 / 100 = 0.5 exactly: matched at 0.5 only
        assert e['dtMatches'][:, 0].tolist() == [1] + [0] * 9
        assert ev.eval['recall'][:, 0, 0, 2].tolist() == [1.0] + [0.0] * 9
    return dict(gt=dataset([1], [1], [(1, 1, [0, 0, 10, 10])]), res=[det(1, 1, [0, 0, 10, 5], .9)], check=check)


def _crowd():
    # category 1: one crowd box matched by two detections inside it (IoU = i / det area = 1), both ignored, npig 0
    # category 2: a non-ignored box A (IoU 100 / 110) and a crowd box B (IoU 1) behind it: below 0.95 the walk takes A and
    # breaks at B; at 0.95 it skips A and takes B
    def check(ev):
        e = ev_img(ev, 1, 1)
        assert (e['dtMatches'] == 1).all() and e['dtIgnore'].all() and e['gtIgnore'].tolist() == [1]
        assert (ev.eval['precision'][:, :, 0] == -1).all() and (ev.eval['recall'][:, 0] == -1).all()
        e = ev_img(ev, 1, 2)
        assert e['dtMatches'][:, 0].tolist() == [2] * 9 + [3] and e['dtIgnore'][:, 0].tolist() == [False] * 9 + [True]
    return dict(gt=dataset([1], [1, 2], [(1, 1, [0, 0, 20, 20], {'iscrowd': 1}), (1, 2, [0, 0, 10, 11]),
                                         (1, 2, [0, 0, 10, 10], {'iscrowd': 1})]),
                res=[det(1, 1, [0, 0, 10, 10], .9), det(1, 1, [5, 5, 10, 10], .8), det(1, 2, [0, 0, 10, 10], .7)], check=check)


def _ignore_overwritten():
    def check(ev):                                               # 'ignore': 1 without iscrowd counts; 'ignore': 0 with it does not
        e = ev_img(ev, 1, 1)
        assert e['gtIds'] == [1, 2] and e['gtIgnore'].tolist() == [0, 1]
    return dict(gt=dataset([1], [1], [(1, 1, [0, 0, 10, 10], {'ignore': 1}), (1, 1, [50, 50, 10, 10], {'ignore': 0, 'iscrowd': 1})]),
                res=[det(1, 1, [0, 0, 10, 10], .9)], check=check)


def _area_bounds():
    def check(ev):                                               # areas 32^2 and 96^2: in both neighbouring ranges
        for a, want in enumerate([[0, 0], [0, 1], [0, 0], [1, 0]]):
            e = ev_img(ev, 1, 1, a)
            assert sorted(zip(e['gtIds'], e['gtIgnore'].tolist())) == [(1, want[0]), (2, want[1])], (a, e['gtIgnore'])
    return dict(gt=dataset([1], [1], [(1, 1, [0, 0, 32, 32]), (1, 1, [100, 100, 96, 96])]), res=[], check=check)


def _unmatched_outside():
    def check(ev):                                               # an unmatched detection of area 2000 is ignored in 'small' only
        assert not ev_img(ev, 1, 1, 0)['dtIgnore'].any()
        assert ev_img(ev, 1, 1, 1)['dtIgnore'].all()
        assert not ev_img(ev, 1, 1, 2)['dtIgnore'].any()
    return dict(gt=dataset([1], [1], [(1, 1, [0, 0, 10, 10])]), res=[det(1, 1, [200, 200, 40, 50], .9)], check=check)


def _gt_id_zero():
    def check(ev):                                               # matched to id 0: dtm == 0 reads as a false positive
        e = ev_img(ev, 1, 1)
        assert (e['dtMatches'] == 0).all() and (e['gtMatches'] == 1).all() and not e['dtIgnore'].any()
        assert (ev.eval['recall'][:, 0, :2] == 0).all() and (ev.eval['precision'][:, :, 0, :2] == 0).all()
    return dict(gt=dataset([1], [1], [(1, 1, [0, 0, 10, 10], {'id': 0})]), res=[det(1, 1, [0, 0, 10, 10], .9)], check=check)


def _no_detections():
    def check(ev):                                               # category 2 has a ground truth and no detection: recall 0
        assert (ev.eval['recall'][:, 1, :2] == 0).all() and (ev.eval['recall'][:, 1, 2:] == -1).all()
        assert (ev.eval['precision'][:, :, 1, :2] == 0).all() and (ev.eval['scores'][:, :, 1, :2] == 0).all()
    return dict(gt=dataset([1], [1, 2], [(1, 1, [0, 0, 10, 10]), (1, 2, [0, 0, 10, 10])]), res=[det(1, 1, [0, 0, 10, 10], .9)],
                check=check)


def _searchsorted_end():
    def check(ev):                                               # recall reaches 0.5: thresholds 0 .. 0.5 filled, the rest 0
        q = ev.eval['precision'][0, :, 0, 0, 2]
        assert (q[:51] == 1 / (1 + np.spacing(1))).all() and (q[51:] == 0).all()
        assert (ev.eval['scores'][0, :51, 0, 0, 2] == .9).all() and (ev.eval['scores'][0, 51:, 0, 0, 2] == 0).all()
    return dict(gt=dataset([1], [1], [(1, 1, [0, 0, 10, 10]), (1, 1, [50, 50, 10, 10])]), res=[det(1, 1, [0, 0, 10, 10], .9)],
                check=check)


def _ties_across_images():
    def check(ev):                                               # equal scores: image 3 (a false positive) before image 5
        assert (ev.eval['precision'][0, :, 0, 0, 2] == 0.5).all()
    return dict(gt=dataset([5, 3], [1], [(5, 1, [0, 0, 10, 10])]),
                res=[det(5, 1, [0, 0, 10, 10], .5), det(3, 1, [0, 0, 10, 10], .5)], check=check)


def _many_detections():
    rng = np.random.default_rng(7)
    s = rng.permutation(120) / 200 + .1
    res = [det(1, 1, [float(i % 11), float(i % 7), 10.0, 10.0], float(s[i])) for i in range(120)]

    def check(ev):                                               # 120 detections in one pair: the best 100 are kept
        e = ev_img(ev, 1, 1)
        assert e['dtIds'] == (np.argsort(-s, kind='stable')[:100] + 1).tolist()
    return dict(gt=dataset([1], [1], [(1, 1, [0, 0, 10, 10]), (1, 1, [5, 3, 10, 10])]), res=res, check=check)


def _custom_max_dets():
    def check(ev):                                               # stats[0] asks for maxDets=100, which is not there
        assert ev.stats[0] == -1 and ev.stats[1] > 0
    return dict(gt=dataset([1], [1], [(1, 1, [0, 0, 10, 10])]), res=[det(1, 1, [0, 0, 10, 10], .9)],
                params={'maxDets': [1, 5, 20]}, check=check)


def _signed_zero_and_nan():
    def check(ev):                                               # -0.0 equals 0.0 (results order), NaN last
        assert ev_img(ev, 1, 1)['dtIds'] == [4, 1, 2, 3]
    return dict(gt=dataset([1], [1], [(1, 1, [0, 0, 10, 10])]),
                res=[det(1, 1, [0, 0, 10, 10], 0.0), det(1, 1, [0, 0, 10, 10], -0.0), det(1, 1, [0, 0, 9, 9], float('nan')),
                     det(1, 1, [1, 1, 10, 10], .5)], check=check)


CASES = {'equal_ious': _equal_ious, 'iou_at_threshold': _iou_at_threshold, 'crowd': _crowd,
         'ignore_overwritten': _ignore_overwritten, 'area_bounds': _area_bounds, 'unmatched_outside': _unmatched_outside,
         'gt_id_zero': _gt_id_zero, 'no_detections': _no_detections, 'searchsorted_end': _searchsorted_end,
         'ties_across_images': _ties_across_images, 'many_detections': _many_detections, 'custom_max_dets': _custom_max_dets,
         'signed_zero_and_nan': _signed_zero_and_nan}


def case(name):
    return CASES[name]()


def random_set(seed, n_images=300, n_cats=80, gt_per_image=7, det_per_image=60, crowd=0.02, big_segment=0):
    """A COCO-like set: ground truths of every size (some crowd, a few with 'ignore'), detections jittered from them plus noise,
    scores on a coarse grid (ties), exact duplicates, images without annotations, categories without detections, detections of
    an unknown category; big_segment > 0 adds one (image, category) pair with that many ground truths and 100 detections."""
    rng = np.random.default_rng(seed)
    img_ids = [int(i) for i in rng.choice(100000, n_images, replace=False)]
    cat_ids = [int(c) for c in np.sort(rng.choice(np.arange(1, 200), n_cats, replace=False))]
    anns, res = [], []
    for n, img in enumerate(img_ids):
        if n % 17 == 5:
            continue                                                      # no annotations, no detections
        k = int(rng.poisson(gt_per_image))
        for _ in range(k):
            side = float(np.exp(rng.uniform(np.log(4), np.log(300))))
            w, h = side * rng.uniform(.6, 1.4), side * rng.uniform(.6, 1.4)
            x, y = float(rng.uniform(0, 500)), float(rng.uniform(0, 400))
            extra = {'iscrowd': int(rng.random() < crowd)}
            if rng.random() < .02:
                extra['ignore'] = 1
            area = w * h * rng.uniform(.5, 1.0)
            if rng.random() < .05:
                area = float(rng.choice([32 ** 2, 96 ** 2]))
            extra['area'] = area
            anns.append((img, int(rng.choice(cat_ids[:n_cats - 3])), [round(x, 2), round(y, 2), round(w, 2), round(h, 2)], extra))
    gt = dataset(img_ids, cat_ids, anns)
    by_img = {}
    for a in gt['annotations']:
        by_img.setdefault(a['image_id'], []).append(a)
    for n, img in enumerate(img_ids):
        if n % 17 == 5:
            continue
        own = by_img.get(img, [])
        for _ in range(int(rng.integers(det_per_image // 2, det_per_image + 1))):
            score = float(np.round(rng.uniform(0, 1), 2))
            if own and rng.random() < .6:
                a = own[int(rng.integers(len(own)))]
                x, y, w, h = a['bbox']
                j = rng.normal(0, .08, 4) * [w, h, w, h]
                box = [x + j[0], y + j[1], max(w + j[2], .5), max(h + j[3], .5)]
                cat = a['category_id'] if rng.random() < .9 else int(rng.choice(cat_ids))
            else:
                box = [float(rng.uniform(0, 500)), float(rng.uniform(0, 400)), float(rng.uniform(2, 200)), float(rng.uniform(2, 200))]
                cat = int(rng.choice(cat_ids))
            res.append(det(img, cat, [round(float(v), 2) for v in box], score))
            if rng.random() < .03:
                res.append(copy.deepcopy(res[-1]))                         # an exact duplicate
        if rng.random() < .02:
            res.append(det(img, 1000, [1.0, 1.0, 5.0, 5.0], .5))             # a category outside the parameters
    if big_segment:
        img, cat = img_ids[0], cat_ids[0]
        base = len(gt['annotations'])
        for i in range(big_segment):
            x, y = float(i % 20) * 12, float(i // 20) * 12
            gt['annotations'].append({'image_id': img, 'category_id': cat, 'bbox': [x, y, 11.0, 11.0], 'area': 121.0,
                                      'iscrowd': int(i % 37 == 3), 'id': base + i + 1})
        for i in range(100):
            x, y = float((i * 7) % 20) * 12 + .5, float((i * 3) % (big_segment // 20)) * 12 + .5
            res.append(det(img, cat, [x, y, 11.0, 11.0], float(np.round(rng.uniform(0, 1), 2))))
    return gt, res
