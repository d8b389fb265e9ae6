"""Regenerates tests/golden/ref_decode_edges_golden.npz: the reference's own ``decode_detections`` / ``decode_detections_fast`` on
the threshold and NaN-score inputs of tests/decode_cases.py -- scores at and around float32(confidence_thresh) in every input
coordinate format, and class vectors that hold a NaN.  Needs a checkout of the reference:
    python tests/golden/make_decode_edges_golden.py /path/to/ssd_keras"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))


def edge_inputs():
    """(key, y_pred, kwargs) of every stored case; the inputs come from tests/decode_cases.py."""
    import decode_cases as dc
    out = []
    for coords in ('centroids', 'corners', 'minmax'):
        for thr in dc.THRESHOLDS:
            out.append(('thr%g/%s' % (thr, coords), dc.threshold_input(thr, coords), dict(confidence_thresh=thr, input_coords=coords)))
        out.append(('nan/%s' % coords, dc.nan_score_input(coords), dict(confidence_thresh=0.01, input_coords=coords)))
    for key, y, kw in out:
        kw.update(iou_threshold=0.45, top_k='all', normalize_coords=False)
    return out


def main(ref_root):
    sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), ref_root]
    np.float = float    # noqa  the reference targets NumPy < 1.24 (caller-side aliases, SURVEY.md section 8c)
    np.int = int        # noqa
    from ssd_encoder_decoder.ssd_output_decoder import decode_detections, decode_detections_fast
    out = {}
    with np.errstate(all='ignore'):
        for key, y, kw in edge_inputs():
            for name, fn in (('per_class', decode_detections), ('fast', decode_detections_fast)):
                out['%s/%s' % (key, name)] = np.asarray(fn(y, **kw)[0], np.float64).reshape(-1, 6)
    np.savez_compressed(os.path.join(HERE, 'ref_decode_edges_golden.npz'), **out)


if __name__ == '__main__':
    main(sys.argv[1])
