"""Evaluator on the GPU (ssdk_eval_match / ssdk_eval_cumsum) against the REAL reference's match_predictions /
compute_precision_recall / compute_average_precisions / compute_mean_average_precision on synthetic predictions
(tests/golden/make_eval_golden.py): true / false positive flags and cumulative counts bit-exact per class, precisions,
recalls, APs and mAP to float64 round-off; and on the edge cases of tests/eval_cases.py (ref_eval_edges_golden.npz), all of
it bit for bit."""
import os
import types

import numpy as np
import pytest

import eval_cases as xc

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_eval_golden.npz'))
E = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_eval_edges_golden.npz'))


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()


def _inputs(name):
    n_images, n_classes = [int(v) for v in G[name + '/cfg']]
    ids = [str(v) for v in G[name + '/ids']]
    labels = [G[name + '/labels%d' % i] for i in range(n_images)]
    neutral = [G[name + '/neutral%d' % i] for i in range(n_images)]
    preds = [list() for _ in range(n_classes + 1)]
    for c in range(1, n_classes + 1):
        for i, p in zip(G[name + '/pred_ids%d' % c], G[name + '/pred%d' % c]):
            preds[c].append((str(i), float(p[0]), float(p[1]), float(p[2]), float(p[3]), float(p[4])))
    return n_classes, ids, labels, neutral, preds


@pytest.mark.parametrize('name', ['a', 'neutral', 'ties'])
@pytest.mark.parametrize('use_neutral', [False, True])
@pytest.mark.parametrize('bp', ['include', 'half'])
def test_evaluator_vs_reference(name, use_neutral, bp):
    from ssd_keras_b200.eval_utils.average_precision_evaluator import Evaluator
    n_classes, ids, labels, neutral, preds = _inputs(name)
    dg = types.SimpleNamespace(labels=labels, image_ids=ids, eval_neutral=neutral if use_neutral else None)
    ev = Evaluator(model=None, n_classes=n_classes, data_generator=dg)
    ev.prediction_results = preds
    key = '%s/%d/%s' % (name, int(use_neutral), bp)
    np.testing.assert_array_equal(ev.get_num_gt_per_class(ret=True), G[key + '/num_gt'])
    tp, fp, ctp, cfp = ev.match_predictions(ignore_neutral_boxes=True, matching_iou_threshold=0.5, border_pixels=bp, sorting_algorithm='mergesort',
                                            ret=True)
    prec, rec = ev.compute_precision_recall(ret=True)
    for c in range(1, n_classes + 1):
        np.testing.assert_array_equal(tp[c], G[key + '/tp%d' % c])
        np.testing.assert_array_equal(fp[c], G[key + '/fp%d' % c])
        np.testing.assert_array_equal(ctp[c], G[key + '/ctp%d' % c])
        np.testing.assert_array_equal(cfp[c], G[key + '/cfp%d' % c])
        np.testing.assert_allclose(prec[c], G[key + '/prec%d' % c], rtol=1e-15)
        np.testing.assert_allclose(rec[c], G[key + '/rec%d' % c], rtol=1e-15)
    np.testing.assert_allclose(ev.compute_average_precisions(mode='sample', ret=True), G[key + '/ap_sample'], rtol=1e-14)
    m_s = ev.compute_mean_average_precision()
    np.testing.assert_allclose(ev.compute_average_precisions(mode='integrate', ret=True), G[key + '/ap_integrate'], rtol=1e-14)
    m_i = ev.compute_mean_average_precision()
    np.testing.assert_allclose([m_s, m_i], G[key + '/map'], rtol=1e-14)


@pytest.mark.parametrize('name', xc.EDGES)
def test_evaluator_edges_vs_reference(name):
    """The edge cases of tests/eval_cases.py (every label dtype, border mode and threshold, predictions on the threshold in
    both arithmetic types, NaN and non-finite overlaps, ties and NaNs across lanes, neutral arg-maxes, an empty class,
    integer ids, a permuted gt_format, a fractional class id) against the reference's own results, bit for bit."""
    c = xc.edge(name)
    xc.assert_same(xc.device(c), xc.golden(E, name, c['n_classes']), c['n_classes'], name)


def test_evaluator_end_to_end_on_a_model():
    """Predictions that are the ground truth itself score an 11-point mAP of exactly 1 (precision 1 at every recall level).
    ('integrate' mode would give 1 - 1/n_gt per class: the reference's integration starts at the first recall value, :869-876.)"""
    from ssd_keras_b200.eval_utils.average_precision_evaluator import Evaluator
    n_classes, ids, labels, neutral, _ = _inputs('a')
    preds = [list() for _ in range(n_classes + 1)]
    for i, lab in zip(ids, labels):
        for r in lab:
            preds[int(r[0])].append((i, 0.9, float(r[1]), float(r[2]), float(r[3]), float(r[4])))
    dg = types.SimpleNamespace(labels=labels, image_ids=ids, eval_neutral=None)
    ev = Evaluator(model=None, n_classes=n_classes, data_generator=dg)
    ev.prediction_results = preds
    ev.get_num_gt_per_class()
    ev.match_predictions()
    ev.compute_precision_recall()
    ev.compute_average_precisions(mode='sample')
    assert abs(ev.compute_mean_average_precision() - 1.0) < 1e-12
    ng = ev.num_gt_per_class[1:]
    ev.compute_average_precisions(mode='integrate')
    np.testing.assert_allclose(ev.average_precisions[1:], 1.0 - 1.0 / ng, rtol=1e-12)
