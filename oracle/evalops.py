"""CPU restatement of the dataset half of the reference's evaluation (never imported by the package): the patch
``RandomPadFixedAR`` draws (patch_sampling_ops.py:180-193, :508, :859-881), the inverters of ``Resize`` and ``CropPad``
(geometric_ops.py:74-79, patch_sampling_ops.py:315-320) in the generator's reversed order, the rounding of confidences and
coordinates (``round(numpy_scalar, n)``), the collection order of ``Evaluator.predict_on_dataset`` (:374-419), the VOC txt lines
of ``write_predictions_to_txt`` (:426-475) and the JSON of ``coco_utils.predict_all_to_json`` (:177-198).  Plain NumPy, every
step in the dtype NumPy itself would use."""
import json

import numpy as np


def pad_draws(shapes, img_height, img_width, seed):
    """Per image ``(patch_ymin, patch_xmin, patch_height, patch_width)``: ``np.random.seed(seed)``, then per image one
    ``uniform(0, 1)`` and the y and x ``randint`` draws."""
    rs = np.random.RandomState(seed)
    ar = img_width / img_height
    out = []
    for h, w in shapes:
        if w < h:
            ph, pw = h, int(round(h * ar))
        else:
            pw, ph = w, int(round(w / ar))
        rs.uniform(0, 1)
        yr, xr = h - ph, w - pw
        py = rs.randint(0, yr + 1) if yr >= 0 else rs.randint(yr, 1)
        px = rs.randint(0, xr + 1) if xr >= 0 else rs.randint(xr, 1)
        out.append((py, px, ph, pw))
    return out


def round_scalar(v, n, dtype):
    """``round(dtype(v), n)`` for NumPy scalars: ``rint(v * 10**n) / 10**n`` in ``dtype``."""
    f = dtype(10.0 ** n)
    return (np.rint(np.asarray(v, dtype) * f) / f).astype(dtype)


def invert(rows, canvas_hw, out_hw, patch_origin, dtype, cols=(3, 5, 2, 4)):
    """The inverters of one image on its kept rows (k, 6), in ``dtype``: Resize's, then (``patch_origin`` given) CropPad's."""
    r = np.array(rows, dtype=dtype, copy=True)
    y, x = [cols[0], cols[1]], [cols[2], cols[3]]
    r[:, y] = np.round(r[:, y] * dtype(canvas_hw[0] / out_hw[0]), 0)        # float32 * Python float: the ratio rounded to float32
    r[:, x] = np.round(r[:, x] * dtype(canvas_hw[1] / out_hw[1]), 0)
    if patch_origin is not None:
        r[:, y] += dtype(patch_origin[0])
        r[:, x] += dtype(patch_origin[1])
    return r


def collect(batches, dtype, round_confidences=False):
    """``batches``: per batch a list of per-image ``(rows (k, 6) decoded, canvas_hw, out_hw, patch_origin or None)``.
    Returns ``(image index, class, conf, box (n, 4))`` in collection order, conf and box in ``dtype``."""
    img, cls, conf, box = [], [], [], []
    i = 0
    for batch in batches:
        for rows, canvas, out, origin in batch:
            rows = np.asarray(rows, dtype=dtype).reshape(-1, 6)
            rows = rows[rows[:, 0] != 0]
            r = invert(rows, canvas, out, origin, dtype)
            c = r[:, 1]
            if round_confidences:
                c = round_scalar(c, round_confidences, dtype)
            img.append(np.full(len(r), i, np.int64)); cls.append(r[:, 0].astype(np.int64)); conf.append(c)
            box.append(round_scalar(r[:, 2:6], 1, dtype))
            i += 1
    cat = lambda a, t, s: np.concatenate(a).astype(t) if a else np.zeros(s, t)  # noqa: E731
    return cat(img, np.int64, (0,)), cat(cls, np.int64, (0,)), cat(conf, dtype, (0,)), cat(box, dtype, (0, 4))


def per_class(img, cls, conf, box, image_ids, n_classes):
    results = [list() for _ in range(n_classes + 1)]
    for k in range(len(img)):
        results[int(cls[k])].append((image_ids[img[k]], conf[k], box[k, 0], box[k, 1], box[k, 2], box[k, 3]))
    return results


def txt_texts(results, n_classes):
    """The text of every class file of ``write_predictions_to_txt``."""
    out = []
    for c in range(1, n_classes + 1):
        lines = []
        for p in results[c]:
            p = list(p)
            p[0] = '{:06d}'.format(int(p[0]))
            p[1] = round(p[1], 4)
            lines.append(' '.join(map(str, p)) + '\n')
        out.append(''.join(lines))
    return out


def json_text(img, cls, conf, box, image_ids, classes_to_cats):
    res = []
    for k in range(len(img)):
        xmin, ymin, xmax, ymax = (float(round(box[k, j], 1)) for j in range(4))
        res.append({'image_id': image_ids[img[k]], 'category_id': classes_to_cats[int(cls[k])], 'score': float(round(conf[k], 3)),
                    'bbox': [xmin, ymin, xmax - xmin, ymax - ymin]})
    return json.dumps(res)


# -- Evaluator.match_predictions and what follows it (reference :490-905) ---------------------------------------------------
# Per prediction, the reference takes its box from a structured array with 'f4' fields (a float32 array) and the ground truth
# as np.asarray(labels), in the labels' own dtype, so NumPy runs its element-wise iou in mixed types: the predicted area in
# float32, the ground-truth area in the labels' dtype (an int16 area wraps), intersection, union and quotient in
# result_type(labels, float32), and on a float32 overlap ``overlap < threshold`` rounds the threshold to float32 (NumPy >= 2).
# The helpers below are the steps a kernel could get subtly wrong, one function each so that a test can swap one out.
# Two deliberate departures from the reference, kept by the package: every prediction is matched (the reference's
# verbose=False loop matches only the first of each class), and a class without predictions has empty cumulative arrays (the
# reference's cumulative lists skip it, which shifts every later class).
BORDER_D = {'half': 0, 'include': 1, 'exclude': -1}
GT_FORMAT = {'class_id': 0, 'xmin': 1, 'ymin': 2, 'xmax': 3, 'ymax': 4}


def class_mask(classes, class_id):
    """``gt[:, class_id] == class_id`` in the labels' dtype: a class of 1.5 is no class."""
    return classes == class_id


def pred_area(b, d):
    """The predicted box's area, ``b`` (1, 4) float32: float32 arithmetic."""
    return (b[:, 2] - b[:, 0] + d) * (b[:, 3] - b[:, 1] + d)


def gt_area(g, d):
    """The ground-truth areas, ``g`` (k, 4) in the labels' dtype: that dtype's arithmetic."""
    return (g[:, 2] - g[:, 0] + d) * (g[:, 3] - g[:, 1] + d)


def best_index(overlaps):
    """np.argmax: the first maximum, and the first NaN wins over every number."""
    return int(np.argmax(overlaps))


def below(overlap, threshold):
    """``overlap < threshold`` with a NumPy scalar overlap and a Python float threshold (NaN < thr is False)."""
    return bool(overlap < threshold)


def cumulative(flags):
    """np.cumsum: inclusive."""
    return np.cumsum(flags)


def overlaps(gt, pred_box, d):
    """Element-wise iou (corners) of ``gt`` (k, 4) in the labels' dtype with one ``pred_box`` (4,) float32: intersection
    without the border term (the reference's iou() calls intersection_area_ with its default), areas with it."""
    b = pred_box[None, :]
    with np.errstate(invalid='ignore', divide='ignore', over='ignore'):
        return _iou(gt, b, d)


def _iou(gt, b, d):
    side = np.maximum(0, np.minimum(gt[:, [2, 3]], b[:, [2, 3]]) - np.maximum(gt[:, [0, 1]], b[:, [0, 1]]) + 0)
    inter = side[:, 0] * side[:, 1]
    return inter / (gt_area(gt, d) + pred_area(b, d) - inter)


def match_predictions(labels, predictions, n_classes, image_ids, eval_neutral=None, ignore_neutral_boxes=True,
                      matching_iou_threshold=0.5, border_pixels='include', gt_format=None):
    """``labels``: per image an array in its own dtype; ``predictions``: per class (index 0 unused) a list of
    ``(image_id, confidence, xmin, ymin, xmax, ymax)``.  Returns the true and false positive flags per class (index 0 empty),
    in descending confidence, equal confidences in input order (the reference with 'mergesort')."""
    f = GT_FORMAT if gt_format is None else gt_format
    ci, cols = f['class_id'], [f['xmin'], f['ymin'], f['xmax'], f['ymax']]
    d = BORDER_D[border_pixels]
    index = {str(i): k for k, i in enumerate(image_ids)}
    use_neutral = ignore_neutral_boxes and eval_neutral is not None
    tps, fps = [np.zeros(0, np.int64)], [np.zeros(0, np.int64)]
    for c in range(1, n_classes + 1):
        preds = predictions[c]
        tp, fp = np.zeros(len(preds), np.int64), np.zeros(len(preds), np.int64)
        if len(preds):
            conf = np.asarray([p[1] for p in preds], np.float32)
            boxes = np.asarray([p[2:6] for p in preds], np.float64).astype(np.float32)
            matched = {}                                    # per image of this class
            for i, k in enumerate(np.argsort(-conf, kind='mergesort')):
                img = index[str(preds[k][0])]
                gt = np.asarray(labels[img])
                mask = class_mask(gt[:, ci], c)
                gt = gt[mask]
                if gt.size == 0:
                    fp[i] = 1
                    continue
                ov = overlaps(gt[:, cols], boxes[k], d)
                j = best_index(ov)
                if below(ov[j], matching_iou_threshold):
                    fp[i] = 1
                    continue
                if use_neutral and not (np.asarray(eval_neutral[img])[mask][j] == False):     # noqa: E712 (the reference's test)
                    continue                                # a neutral box: neither, and not marked matched
                m = matched.setdefault(img, np.zeros(len(gt), bool))
                if m[j]:
                    fp[i] = 1
                else:
                    tp[i] = 1
                    m[j] = True
        tps.append(tp)
        fps.append(fp)
    return tps, fps


def num_gt_per_class(labels, n_classes, eval_neutral=None, ignore_neutral_boxes=True, class_col=0):
    """Evaluator.get_num_gt_per_class as the package counts: class ids cast to int (the reference indexes with the raw value
    and so raises on float labels)."""
    num = np.zeros(n_classes + 1, dtype=int)
    for i, boxes in enumerate(labels):
        boxes = np.asarray(boxes)
        if boxes.size == 0:
            continue
        cls = boxes[:, class_col].astype(int)
        if ignore_neutral_boxes and eval_neutral is not None:
            cls = cls[~np.asarray(eval_neutral[i], dtype=bool)]
        np.add.at(num, cls, 1)
    return num


def precision_recall(ctp, cfp, num_gt, n_classes):
    """Cumulative precision (0 where nothing was predicted yet) and recall per class (index 0 empty)."""
    prec, rec = [[]], [[]]
    for c in range(1, n_classes + 1):
        t, f = ctp[c], cfp[c]
        with np.errstate(divide='ignore', invalid='ignore'):
            prec.append(np.where(t + f > 0, t / (t + f), 0))
            rec.append(t / num_gt[c])
    return prec, rec


def average_precisions(prec, rec, n_classes, mode='sample', num_recall_points=11):
    """Per class (index 0 is 0.0): the maximum precision at recall >= t over ``num_recall_points`` t in [0, 1] averaged
    ('sample'), or the sum over unique recalls of the recall step times the best precision from there on ('integrate')."""
    aps = [0.0]
    for c in range(1, n_classes + 1):
        p, r = prec[c], rec[c]
        ap = 0.0
        if mode == 'sample':
            for t in np.linspace(start=0, stop=1, num=num_recall_points, endpoint=True):
                sel = p[r >= t]
                ap += 0.0 if sel.size == 0 else np.amax(sel)
            ap /= num_recall_points
        else:
            ur, ui = np.unique(r, return_index=True)
            mp, dr = np.zeros_like(ur), np.zeros_like(ur)
            for i in range(len(ur) - 2, -1, -1):
                mp[i] = np.maximum(np.amax(p[ui[i]:ui[i + 1]]), mp[i + 1])
                dr[i] = ur[i + 1] - ur[i]
            ap = np.sum(mp * dr)
        aps.append(ap)
    return aps


def evaluate(labels, predictions, n_classes, image_ids, eval_neutral=None, matching_iou_threshold=0.5, border_pixels='include',
             gt_format=None):
    """Everything the golden files hold: flags, cumulative counts, precisions, recalls, both AP modes and both mAPs."""
    f = GT_FORMAT if gt_format is None else gt_format
    tp, fp = match_predictions(labels, predictions, n_classes, image_ids, eval_neutral, True, matching_iou_threshold, border_pixels, f)
    ctp, cfp = [tp[0]] + [cumulative(t) for t in tp[1:]], [fp[0]] + [cumulative(x) for x in fp[1:]]
    num = num_gt_per_class(labels, n_classes, eval_neutral, True, f['class_id'])
    prec, rec = precision_recall(ctp, cfp, num, n_classes)
    ap_s = average_precisions(prec, rec, n_classes, 'sample')
    ap_i = average_precisions(prec, rec, n_classes, 'integrate')
    return dict(tp=tp, fp=fp, ctp=ctp, cfp=cfp, num_gt=num, prec=prec, rec=rec, ap_sample=ap_s, ap_integrate=ap_i,
                map=np.asarray([np.average(ap_s[1:]), np.average(ap_i[1:])]))
