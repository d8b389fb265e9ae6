"""Regenerates tests/golden/ref_encode_edges_golden.npz: the reference's own ``SSDInputEncoder`` on the threshold, conflict,
zero-row and thr <= 0 cases of tests/encode_cases.py -- IoUs exactly at and one float64 ulp below pos_iou_threshold and
neg_iou_limit in every coordinate format, chains of boxes that want the same prior, rows that fall to zero, boxes that overlap
no prior, and neg_iou_limit <= 0 with a box of the background class.  Needs a checkout of the reference:
    python tests/golden/make_encode_edges_golden.py /path/to/ssd_keras"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

EDGE_CASES = ('thr_at_centroids', 'thr_below_centroids', 'thr_at_corners', 'thr_below_corners', 'thr_at_minmax',
              'thr_below_minmax', 'thr_at_corners_f64', 'thr_below_centroids_f64', 'thr0_neg0', 'thr0_negative',
              'no_multi_pos', 'bipartite_only', 'chain4', 'tozero', 'c1_other_tile', 'zero_rows')


def main(ref_root):
    sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), ref_root]
    np.float = float    # noqa  the reference targets NumPy < 1.24 (caller-side aliases, SURVEY.md section 8c)
    np.int = int        # noqa
    from ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    import encode_cases as ec
    out = {}
    for name in EDGE_CASES:
        c = ec.BY_NAME[name]
        out[name] = np.asarray(SSDInputEncoder(**ec.config(c))(ec.inputs(name)), np.float64)
    np.savez_compressed(os.path.join(HERE, 'ref_encode_edges_golden.npz'), **out)


if __name__ == '__main__':
    main(sys.argv[1])
