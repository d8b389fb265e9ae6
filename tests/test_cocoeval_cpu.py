"""The COCO evaluation's oracle (oracle/cocoeval.py) against hand-derived values, one case per rule of pycocotools'
COCOeval; its bbIou against an independent vectorised IoU; the summary text against the lines the reference's COCO notebook
stores; and the host-only parts of ssd_keras_b200.eval_utils.coco_eval (loading, parameters, summary)."""
import contextlib
import copy
import io
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import cocoeval_cases as cc                                                     # noqa: E402
from oracle import cocoeval as oc                                               # noqa: E402


def run_oracle(case):
    gt = oc.COCO(copy.deepcopy(case['gt']))
    ev = oc.COCOeval(gt, gt.loadRes(copy.deepcopy(case['res'])))
    for k, v in case.get('params', {}).items():
        setattr(ev.params, k, v)
    with contextlib.redirect_stdout(io.StringIO()):
        ev.evaluate()
        ev.accumulate()
        ev.summarize()
    return ev


@pytest.mark.parametrize('name', sorted(cc.CASES))
def test_oracle_hand_derived(name):
    case = cc.case(name)
    case['check'](run_oracle(case))


def vectorised_iou(d, g, crowd):
    d, g = np.asarray(d, np.float64)[:, None, :], np.asarray(g, np.float64)[None, :, :]
    w = np.fmin(d[..., 2] + d[..., 0], g[..., 2] + g[..., 0]) - np.fmax(d[..., 0], g[..., 0])
    h = np.fmin(d[..., 3] + d[..., 1], g[..., 3] + g[..., 1]) - np.fmax(d[..., 1], g[..., 1])
    i = w * h
    da, ga = d[..., 2] * d[..., 3], g[..., 2] * g[..., 3]
    with np.errstate(invalid='ignore', divide='ignore'):
        u = np.where(np.asarray(crowd, bool)[None, :], da, da + ga - i)
        return np.where((w <= 0) | (h <= 0), 0.0, i / u)           # a NaN width or height is not <= 0


def test_bb_iou_matches_vectorised():
    rng = np.random.default_rng(3)
    boxes = np.concatenate([
        np.c_[rng.uniform(0, 50, (40, 2)), rng.uniform(0, 30, (40, 2))],            # random
        [[0, 0, 10, 10], [10, 0, 5, 5], [0, 10, 5, 5], [10, 10, 3, 3], [-5, -5, 5, 5]],   # touching [0, 0, 10, 10]
        [[3, 3, 0, 4], [3, 3, 4, 0], [3, 3, 0, 0], [3, 3, -2, 4], [0, 0, 1e-300, 1e-300]],  # degenerate
        [[np.nan, 0, 10, 10], [0, 0, np.nan, 10], [0, 0, np.inf, 10]],             # NaN / inf: fmin / fmax ignore NaN
    ])
    crowd = (np.arange(len(boxes)) % 5 == 2).astype(int)
    got = oc.bb_iou(boxes, boxes, crowd)
    want = vectorised_iou(boxes, boxes, crowd)
    assert np.array_equal(got, want, equal_nan=True)
    assert got[40, 41] == 0 and got[40, 42] == 0 and got[40, 40] == 1.0


def golden_lines():
    with open(os.path.join(HERE, 'golden', 'ref_cocoeval_summary.txt')) as f:
        return f.read().splitlines()


def fed_eval(values):
    """precision / recall arrays whose twelve summary selections average to the given values."""
    v = values
    prec = -np.ones((10, 1, 1, 4, 3))
    rec = -np.ones((10, 1, 4, 3))
    prec[:, 0, 0, 0, 2] = (10 * v[0] - v[1] - v[2]) / 8
    prec[0, 0, 0, 0, 2], prec[5, 0, 0, 0, 2] = v[1], v[2]
    for a in range(1, 4):
        prec[:, 0, 0, a, 2] = v[2 + a]
        rec[:, 0, a, 2] = v[8 + a]
    for m in range(3):
        rec[:, 0, 0, m] = v[6 + m]
    return {'precision': prec, 'recall': rec}


@pytest.mark.parametrize('which', ['oracle', 'product'])
def test_summary_text_matches_notebook(which):
    lines = golden_lines()
    values = [float(l.rsplit('=', 1)[1]) for l in lines]
    if which == 'oracle':
        out = []
        stats = oc.summarize(oc.Params(), fed_eval(values), out=out.append)
    else:
        from ssd_keras_b200.eval_utils.coco_eval import COCOeval
        ev = COCOeval()
        ev.eval = fed_eval(values)
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            ev.summarize()
        out, stats = buf.getvalue().splitlines(), ev.stats
    assert out == lines
    assert np.allclose(stats, values, atol=1e-12)


def test_product_params_and_load_res(tmp_path):
    import json
    from ssd_keras_b200.eval_utils.coco_eval import COCO, COCOeval
    case = cc.case('crowd')
    path = tmp_path / 'gt.json'
    path.write_text(json.dumps(case['gt']))
    with contextlib.redirect_stdout(io.StringIO()):
        gt = COCO(str(path))
        dt = gt.loadRes(copy.deepcopy(case['res']))
        arr = gt.loadRes(np.array([[1, 0, 0, 10, 10, .9, 1], [1, 5, 5, 2, 3, .8, 2]]))
        with pytest.raises(AssertionError, match='Results do not correspond to current coco set'):
            gt.loadRes([cc.det(99, 1, [0, 0, 1, 1], .5)])
    assert gt.getImgIds() == [1] and gt.getCatIds() == [1, 2]
    assert [a['id'] for a in dt.dataset['annotations']] == [1, 2, 3] and all(a['iscrowd'] == 0 for a in dt.dataset['annotations'])
    assert [a['area'] for a in arr.dataset['annotations']] == [100.0, 6.0]
    ev = COCOeval(gt, dt, iouType='bbox')
    p, o = ev.params, oc.Params()
    assert np.array_equal(p.iouThrs, o.iouThrs) and np.array_equal(p.recThrs, o.recThrs)
    assert p.maxDets == [1, 10, 100] and p.areaRng == o.areaRng and p.areaRngLbl == o.areaRngLbl
    assert p.imgIds == [1] and p.catIds == [1, 2] and ev.evalImgs == []
    ev.evalImgs = [None, {'image_id': 1}]                     # a plain attribute in pycocotools: user code may assign it
    assert ev.evalImgs == [None, {'image_id': 1}]
    for kind in ('segm', 'keypoints'):
        with pytest.raises(NotImplementedError):
            COCOeval(gt, dt, iouType=kind)
    ev.params.useCats = 0
    with pytest.raises(NotImplementedError, match='useCats'), contextlib.redirect_stdout(io.StringIO()):
        ev.evaluate()
