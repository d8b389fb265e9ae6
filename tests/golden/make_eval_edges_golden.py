"""Regenerates tests/golden/ref_eval_edges_golden.npz: the reference's own Evaluator (match_predictions with verbose=True and
'mergesort', compute_precision_recall, compute_average_precisions in both modes, compute_mean_average_precision) on the edge
cases of tests/eval_cases.py (EDGES).  Stored per case and class: the true / false positive flags, np.cumsum of each (the
reference's cumulative lists skip a class without predictions and so shift every later one; those are not stored), the
precisions and recalls computed by the reference from those sums, both AP modes and both mAPs, and a digest of the inputs.
The reference's get_num_gt_per_class indexes with the raw class value and raises on float labels; the counts come from
oracle.evalops.num_gt_per_class (class ids cast to int, as the package counts) for every case.  Needs a checkout of the
reference:
    python tests/golden/make_eval_edges_golden.py /path/to/ssd_keras"""
import contextlib
import hashlib
import io
import os
import sys
import types
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))


def digest(c):
    """Of the inputs a case is made of, so that a changed generator shows as a changed case rather than a kernel bug."""
    h = hashlib.sha256()
    for lab in c['labels']:
        lab = np.ascontiguousarray(lab)
        h.update(str(lab.dtype).encode()); h.update(str(lab.shape).encode()); h.update(lab.tobytes())
    h.update(repr([c['preds'], c['n_classes'], c['thr'], c['border'], c['ids'], c['gt_format']]).encode())
    if c['neutral'] is not None:
        for e in c['neutral']:
            h.update(np.asarray(e, bool).tobytes())
    return h.hexdigest()[:16]


def main(ref_root):
    sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), ref_root]
    np.float = float    # noqa  the reference targets NumPy < 1.24
    np.int = int        # noqa
    warnings.simplefilter('ignore')
    from eval_utils.average_precision_evaluator import Evaluator
    import eval_cases as xc
    from oracle import evalops as eo
    out = {}
    for name in xc.EDGES:
        c = xc.edge(name)
        f = eo.GT_FORMAT if c['gt_format'] is None else c['gt_format']
        dg = types.SimpleNamespace(labels=c['labels'], image_ids=c['ids'], eval_neutral=c['neutral'])
        ev = Evaluator(model=None, n_classes=c['n_classes'], data_generator=dg, gt_format=f)
        ev.prediction_results = c['preds']
        n = c['n_classes']
        with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
            tp, fp, _, _ = ev.match_predictions(ignore_neutral_boxes=True, matching_iou_threshold=c['thr'], border_pixels=c['border'],
                                                sorting_algorithm='mergesort', verbose=True, ret=True)
            ev.num_gt_per_class = eo.num_gt_per_class(c['labels'], n, c['neutral'], True, f['class_id'])
            ev.cumulative_true_positives = [[]] + [np.cumsum(tp[k]) for k in range(1, n + 1)]
            ev.cumulative_false_positives = [[]] + [np.cumsum(fp[k]) for k in range(1, n + 1)]
            prec, rec = ev.compute_precision_recall(verbose=False, ret=True)
            ap_s = ev.compute_average_precisions(mode='sample', num_recall_points=11, verbose=False, ret=True)
            map_s = ev.compute_mean_average_precision()
            ap_i = ev.compute_average_precisions(mode='integrate', verbose=False, ret=True)
            map_i = ev.compute_mean_average_precision()
        out[name + '/digest'] = np.asarray(digest(c))
        out[name + '/num_gt'] = np.asarray(ev.num_gt_per_class)
        for k in range(1, n + 1):
            out['%s/tp%d' % (name, k)] = np.asarray(tp[k], np.int64)
            out['%s/fp%d' % (name, k)] = np.asarray(fp[k], np.int64)
            out['%s/ctp%d' % (name, k)] = np.asarray(ev.cumulative_true_positives[k], np.int64)
            out['%s/cfp%d' % (name, k)] = np.asarray(ev.cumulative_false_positives[k], np.int64)
            out['%s/prec%d' % (name, k)] = np.asarray(prec[k], np.float64)
            out['%s/rec%d' % (name, k)] = np.asarray(rec[k], np.float64)
        out[name + '/ap_sample'] = np.asarray(ap_s, np.float64)
        out[name + '/ap_integrate'] = np.asarray(ap_i, np.float64)
        out[name + '/map'] = np.asarray([map_s, map_i], np.float64)
        print('%-24s %5d predictions, %4d TP, %4d FP' % (name, sum(len(p) for p in c['preds']),
                                                      sum(int(np.sum(t)) for t in tp[1:]), sum(int(np.sum(x)) for x in fp[1:])))
    np.savez_compressed(os.path.join(HERE, 'ref_eval_edges_golden.npz'), **out)


if __name__ == '__main__':
    main(sys.argv[1])
