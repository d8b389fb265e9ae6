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
