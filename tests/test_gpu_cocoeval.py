"""COCO box evaluation on the device (eval_utils/coco_eval.py, csrc/cocoeval.cu) against the NumPy restatement of pycocotools'
COCOeval (oracle/cocoeval.py): every evalImgs entry, the device's per-(segment, area) non-ignored counts, and precision /
recall / scores / stats bit for bit, on the hand-derived cases, seeded random COCO-like sets, a segment larger than the shared
IoU tile, changed parameters and an SSD300 results file written by predict_all_to_json."""
import contextlib
import copy
import io
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import cocoeval_cases as cc                                                     # noqa: E402
from oracle import cocoeval as oc                                               # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def built():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    import __graft_entry__ as entry
    entry.build()


def evaluate_both(gt, res, params=None):
    """(device COCOeval, oracle COCOeval), each evaluated, accumulated and summarised on its own copy of the data."""
    from ssd_keras_b200.eval_utils import coco_eval as ce
    out = []
    for mod, make in ((ce, lambda d: _device_coco(d)), (oc, oc.COCO)):
        g = make(copy.deepcopy(gt))
        ev = mod.COCOeval(g, g.loadRes(copy.deepcopy(res) if not isinstance(res, str) else res))
        for k, v in (params or {}).items():
            setattr(ev.params, k, copy.deepcopy(v))
        with contextlib.redirect_stdout(io.StringIO()):
            ev.evaluate()
            ev.accumulate()
            ev.summarize()
        out.append(ev)
    return out


def _device_coco(dataset):
    from ssd_keras_b200.eval_utils.coco_eval import COCO
    with contextlib.redirect_stdout(io.StringIO()):
        c = COCO()
        c.dataset = dataset
        c.createIndex()
    return c


def assert_same(dev, ref):
    assert len(dev.evalImgs) == len(ref.evalImgs)
    n = 0
    for a, b in zip(dev.evalImgs, ref.evalImgs):
        assert (a is None) == (b is None)
        if a is None:
            continue
        n += 1
        for k in ('image_id', 'category_id', 'aRng', 'maxDet', 'dtIds', 'gtIds'):
            assert a[k] == b[k], (k, a[k], b[k])
        assert np.array_equal(np.asarray(a['dtScores']), np.asarray(b['dtScores']), equal_nan=True)
        for k in ('dtMatches', 'gtMatches', 'gtIgnore', 'dtIgnore'):
            assert a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k]), (k, a, b)
    assert n == sum(e is not None for e in ref.evalImgs)
    # the kernel's non-ignored counts per (segment, area) against the oracle's gtIgnore
    dv, p = dev._dev, ref.params
    I, A = len(p.imgIds), len(p.areaRng)
    seg_key, npig = dv['seg_key'].cpu().numpy(), dv['seg_npig'].cpu().numpy().reshape(-1, A)[:len(dv['seg_key'])]
    for s, key in enumerate(seg_key.tolist()):
        i, k = divmod(key, dv['K'])
        for a in range(A):
            assert npig[s, a] == np.count_nonzero(ref.evalImgs[(k * A + a) * I + i]['gtIgnore'] == 0)
    for k in ('precision', 'recall', 'scores'):
        x, y = dev.eval[k], ref.eval[k]
        assert x.shape == y.shape and x.dtype == y.dtype, k
        assert np.array_equal(x, y, equal_nan=True) and np.array_equal(np.signbit(x), np.signbit(y)), k
    assert dev.eval['counts'] == ref.eval['counts']
    assert np.array_equal(dev.stats, ref.stats)


@pytest.mark.parametrize('name', sorted(cc.CASES))
def test_cases(name):
    case = cc.case(name)
    dev, ref = evaluate_both(case['gt'], case['res'], case.get('params'))
    case['check'](ref)
    assert_same(dev, ref)


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_random_sets(seed):
    gt, res = cc.random_set(seed)
    assert_same(*evaluate_both(gt, res))


def test_segment_larger_than_the_tile():
    gt, res = cc.random_set(5, n_images=40, big_segment=400)          # 100 detections x 400 ground truths in one segment
    assert_same(*evaluate_both(gt, res))


def test_categories_longer_than_one_accumulate_chunk():
    """Five categories with ground truths and about 1 400 detections each: each of their accumulate CTAs walks several
    256-detection chunks, so the counts and the running precision maximum carried from one chunk into the next are compared
    with the oracle."""
    gt, res = cc.random_set(13, n_images=150, n_cats=8, gt_per_image=6, det_per_image=80)
    dev, ref = evaluate_both(gt, res)
    dv = dev._dev
    per_cat = np.diff(dv['cat_off'].cpu().numpy())
    with_gt = dv['npig'].cpu().numpy()[:dv['K'] * dv['A']].reshape(dv['K'], dv['A'])[:, 0] > 0
    assert with_gt.sum() == 5 and per_cat[with_gt].min() > 3 * 256, (per_cat, with_gt)
    assert_same(dev, ref)


def test_changed_params():
    gt, res = cc.random_set(9, n_images=150)
    img_ids = sorted(i['id'] for i in gt['images'])
    cat_ids = sorted(c['id'] for c in gt['categories'])
    variants = [
        {'imgIds': img_ids[::3], 'catIds': cat_ids[5:40]},
        {'maxDets': [20, 1, 5]},
        {'iouThrs': np.array([.3, .5, .85])},
        {'iouThrs': np.linspace(.05, .95, 19)},                          # 4 x 19 scans: a thread owns two of them
        {'areaRng': [[0, 1e10], [0, 500.5], [400, 4096], [4096, 5e4]], 'areaRngLbl': ['all', 'small', 'medium', 'large']},
        {'recThrs': np.linspace(0, 1, 11)},
    ]
    for params in variants:
        assert_same(*evaluate_both(gt, res, params))


def test_ssd300_results_file_end_to_end(tmp_path):
    """A random-weight SSD300 through predict_all_to_json on a small synthetic COCO-format dataset; the file then goes to both
    COCOevals."""
    import types
    from oracle import synth
    from oracle.model import vgg_weight_shapes
    from ssd_keras_b200.eval_utils.coco_utils import predict_all_to_json
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    n_classes = 80
    model = ssd_300((300, 300, 3), n_classes, mode='inference', scales=[0.07, 0.15, 0.33, 0.51, 0.69, 0.87, 1.05],
                    confidence_thresh=0.01, iou_threshold=0.45, top_k=200)
    w = synth.synth_weights(4, vgg_weight_shapes(300, n_classes), bias_scale=0.02)
    w['conv4_3_norm/gamma'] = np.full((512,), 20.0, np.float32)
    model.set_weights(w)
    rng = np.random.default_rng(11)
    shapes = [(480, 640), (427, 640), (640, 480), (300, 300), (375, 500), (512, 512), (333, 500), (240, 320)]
    ids = [int(v) for v in rng.choice(600000, len(shapes), replace=False)]
    images = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in shapes]
    cat_ids = [c for c in range(1, 91) if c not in (12, 26, 29, 30, 45, 66, 68, 69, 71, 83)]
    classes_to_cats = {i + 1: c for i, c in enumerate(cat_ids)}
    anns = []
    for img, (h, w_) in zip(ids, shapes):
        for _ in range(int(rng.integers(0, 12))):
            bw, bh = float(rng.uniform(4, w_ / 2)), float(rng.uniform(4, h / 2))
            box = [round(float(rng.uniform(0, w_ - bw)), 2), round(float(rng.uniform(0, h - bh)), 2), round(bw, 2), round(bh, 2)]
            anns.append((img, int(rng.choice(cat_ids)), box, {'iscrowd': int(rng.random() < .05)}))
    gt = cc.dataset(ids, cat_ids, anns)
    for im, (h, w_) in zip(gt['images'], shapes):
        im.update(height=h, width=w_, file_name='%012d.jpg' % im['id'])
    dg = types.SimpleNamespace(images=images, filenames=None, image_ids=ids, labels=[np.zeros((0, 5)) for _ in ids], eval_neutral=None)
    f = str(tmp_path / 'results.json')
    with contextlib.redirect_stdout(io.StringIO()):
        predict_all_to_json(f, model, 300, 300, classes_to_cats, dg, 4, model_mode='inference', top_k=200)
    res = json.load(open(f))
    assert len(res) > 100
    dev, ref = evaluate_both(gt, f)
    assert_same(dev, ref)


def test_launch_count_is_independent_of_the_dataset_size():
    from ssd_keras_b200 import _ffi
    counts = []
    for n in (50, 500):
        gt, res = cc.random_set(21, n_images=n, n_cats=20, det_per_image=20)
        from ssd_keras_b200.eval_utils.coco_eval import COCOeval
        g = _device_coco(gt)
        with contextlib.redirect_stdout(io.StringIO()):
            ev = COCOeval(g, g.loadRes(res))
            before = _ffi.launch_count()
            ev.evaluate()
            ev.accumulate()
        counts.append(_ffi.launch_count() - before)
    assert counts == [2, 2]
