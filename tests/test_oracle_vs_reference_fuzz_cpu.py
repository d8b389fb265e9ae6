"""Differential fuzzing of the NumPy half of the oracle against the REAL reference, beyond the fixed golden vectors: random
encoder configurations and ground truth, random prediction tensors for the two NumPy decoders, random box sets for iou /
convert_coordinates.  The reference's results on these seeded inputs are stored in tests/golden/ref_fuzz_golden.npz
(tests/golden/make_fuzz_golden.py runs the reference checkout and calls the reference_* functions below); the inputs are
regenerated here from the same seeds.  Bit-exact float64 equality is required, as in tests/test_oracle_golden.py."""
import os

import numpy as np
import pytest

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_fuzz_golden.npz')


@pytest.fixture(scope='module')
def gold():
    with np.load(GOLD) as z:
        return {k: z[k] for k in z.files}


def _results(gold, prefix):
    """The stored results of one case, in the order the reference_* function produced them."""
    n = int(gold[prefix + '/n'])
    return [gold['%s/%d' % (prefix, i)] for i in range(n)]


def _random_encoder_cfg(rng):
    n_layers = int(rng.integers(1, 4))
    H, W = int(rng.integers(60, 200)), int(rng.integers(60, 200))
    sizes = [(int(rng.integers(1, 7)), int(rng.integers(1, 7))) for _ in range(n_layers)]
    scales = sorted(rng.uniform(0.05, 1.0, n_layers + 1).tolist())
    per_layer = bool(rng.integers(0, 2))
    pool = [0.5, 1.0, 2.0, 3.0, 1.0 / 3.0, 1.5]
    ars = [list(rng.choice(pool, size=int(rng.integers(1, 5)), replace=False)) for _ in range(n_layers)]
    cfg = dict(img_height=H, img_width=W, n_classes=int(rng.integers(1, 6)), predictor_sizes=sizes, scales=scales,
               aspect_ratios_global=ars[0] if not per_layer else None, aspect_ratios_per_layer=ars if per_layer else None,
               two_boxes_for_ar1=bool(rng.integers(0, 2)), clip_boxes=bool(rng.integers(0, 2)),
               variances=rng.choice([0.1, 0.2, 1.0], size=4).tolist(), matching_type=str(rng.choice(['multi', 'bipartite'])),
               pos_iou_threshold=float(rng.choice([0.3, 0.5, 0.7])), neg_iou_limit=float(rng.choice([0.2, 0.3, 0.5])),
               border_pixels=str(rng.choice(['half', 'include', 'exclude'])), coords=str(rng.choice(['centroids', 'minmax', 'corners'])),
               normalize_coords=bool(rng.integers(0, 2)))
    cfg['neg_iou_limit'] = min(cfg['neg_iou_limit'], cfg['pos_iou_threshold'])
    if rng.integers(0, 2):
        cfg['steps'] = [(float(rng.uniform(8, 40)), float(rng.uniform(8, 40))) if rng.integers(0, 2) else float(rng.uniform(8, 40))
                        for _ in range(n_layers)]
    if rng.integers(0, 2):
        cfg['offsets'] = [float(rng.uniform(0.2, 0.8)) for _ in range(n_layers)]
    cfg['background_id'] = int(rng.integers(0, cfg['n_classes'] + 1)) if rng.integers(0, 3) == 0 else 0
    return cfg


def _random_gt(rng, cfg, B):
    out = []
    for _ in range(B):
        G = int(rng.integers(0, 6))
        x0 = rng.uniform(0, 0.7 * cfg['img_width'], G); y0 = rng.uniform(0, 0.7 * cfg['img_height'], G)
        w = rng.uniform(5, 0.6 * cfg['img_width'], G); h = rng.uniform(5, 0.6 * cfg['img_height'], G)
        ids = [c for c in range(cfg['n_classes'] + 1) if c != cfg['background_id']]
        g = np.stack([rng.choice(ids, G) if G else np.zeros(0), x0, y0, np.minimum(x0 + w, cfg['img_width'] - 1),
                      np.minimum(y0 + h, cfg['img_height'] - 1)], axis=1) if G else np.zeros((0, 5))
        if G >= 2 and rng.integers(0, 3) == 0:
            g[1] = g[0]                                    # duplicate box: exercises the tie rules
        out.append(g.astype(np.float64))
    return out


def _encoder_case(seed):
    rng = np.random.default_rng(1000 + seed)
    cfg = _random_encoder_cfg(rng)
    return cfg, _random_gt(rng, cfg, int(rng.integers(1, 4)))


def reference_encoder(ref, seed):
    cfg, gt = _encoder_case(seed)
    r = ref['SSDInputEncoder'](**cfg)
    tpl = r.generate_encoding_template(2)
    assert (tpl[1] == tpl[0]).all()                                          # one image's template is stored
    return [tpl[0][:, -8:-4], r(gt), tpl[0]] + list(r.boxes_list)


@pytest.mark.parametrize('seed', range(40))
def test_encoder_fuzz(gold, seed):
    from oracle.encoder import OracleEncoder
    cfg, gt = _encoder_case(seed)
    want = _results(gold, 'encoder/%d' % seed)
    o = OracleEncoder(**cfg)
    np.testing.assert_array_equal(o.anchors, want[0])
    np.testing.assert_array_equal(o(gt), want[1])


def _decoder_case(seed):
    from oracle import synth
    rng = np.random.default_rng(2000 + seed)
    P, C, B = int(rng.integers(20, 200)), int(rng.integers(2, 7)), int(rng.integers(1, 3))
    anchors = np.concatenate([rng.uniform(0.1, 0.9, (P, 2)), rng.uniform(0.05, 0.5, (P, 2))], axis=1)
    y = synth.synth_y_pred(seed, B, anchors, C, sharp=float(rng.uniform(1, 5)), loc_scale=float(rng.uniform(0.3, 1.5)))
    kw = dict(confidence_thresh=float(rng.choice([0.01, 0.2, 0.5])), iou_threshold=float(rng.choice([0.3, 0.45, 0.6])),
              top_k=int(rng.choice([5, 20, 200])), normalize_coords=bool(rng.integers(0, 2)), img_height=120, img_width=160,
              border_pixels=str(rng.choice(['half', 'include', 'exclude'])))
    return y, kw


def reference_decoders(ref, seed):
    y, kw = _decoder_case(seed)
    out = []
    for name in ('decode_detections', 'decode_detections_fast'):
        out += [np.asarray(b, np.float64).reshape(-1, 6) for b in ref[name](y, **kw)]
    return out


@pytest.mark.parametrize('seed', range(25))
def test_numpy_decoders_fuzz(gold, seed):
    from oracle.decoder import decode_detections, decode_detections_fast
    y, kw = _decoder_case(seed)
    want = _results(gold, 'decoders/%d' % seed)
    got = []
    for fn in (decode_detections, decode_detections_fast):
        res = fn(y, **kw)
        assert len(res) == y.shape[0]
        got += [np.asarray(a, np.float64).reshape(-1, 6) for a in res]
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert a.shape == b.shape
        # top-k of the reference is an unordered argpartition set: compare as sorted rows
        ka = np.lexsort(a.T[::-1]); kb = np.lexsort(b.T[::-1])
        np.testing.assert_array_equal(a[ka], b[kb])


def _box_case(seed):
    rng = np.random.default_rng(3000 + seed)
    m, n = int(rng.integers(1, 9)), int(rng.integers(1, 9))

    def boxes(k):
        xy = rng.uniform(0, 80, (k, 2)); wh = rng.uniform(0, 40, (k, 2))
        return np.concatenate([xy, xy + wh], axis=1)
    b1, b2 = boxes(m), boxes(n)
    wide = np.concatenate([rng.standard_normal((m, 2)), b1], axis=1)          # conversion in the middle of a wider row
    return b1, b2, wide


_CONVS = ('minmax2centroids', 'centroids2minmax', 'corners2centroids', 'centroids2corners', 'minmax2corners', 'corners2minmax')


def _box_calls(fns, seed):
    """Every box-math call of one case, in a fixed order; fns supplies convert_coordinates / convert_coordinates2 / iou."""
    b1, b2, wide = _box_case(seed)
    k = min(len(b1), len(b2))
    out = [fns['convert_coordinates2'](wide, 2, conv) for conv in ('minmax2centroids', 'centroids2minmax')]
    for border in ('half', 'include', 'exclude'):
        out += [fns['convert_coordinates'](b1, 0, conv, border) for conv in _CONVS]
        for coords in ('corners', 'minmax', 'centroids'):
            c1 = b1 if coords == 'corners' else fns['convert_coordinates'](b1, 0, 'corners2' + coords)
            c2 = b2 if coords == 'corners' else fns['convert_coordinates'](b2, 0, 'corners2' + coords)
            out += [fns['iou'](c1, c2, coords, 'outer_product', border), fns['iou'](c1[:k], c2[:k], coords, 'element-wise', border)]
    return out


def reference_box_math(ref, seed):
    return _box_calls(ref, seed)


@pytest.mark.parametrize('seed', range(10))
def test_box_math_fuzz(gold, seed):
    from oracle.boxes import convert_coordinates, iou
    from ssd_keras_b200.bounding_box_utils.bounding_box_utils import convert_coordinates as mirror_cc
    from ssd_keras_b200.bounding_box_utils.bounding_box_utils import convert_coordinates2 as mirror_cc2
    want = _results(gold, 'box_math/%d' % seed)
    oracle = _box_calls(dict(convert_coordinates=convert_coordinates, convert_coordinates2=mirror_cc2, iou=iou), seed)
    product = _box_calls(dict(convert_coordinates=mirror_cc, convert_coordinates2=mirror_cc2, iou=iou), seed)   # product (host side)
    assert len(oracle) == len(want)
    for a, p, w in zip(oracle, product, want):
        np.testing.assert_array_equal(a, w)
        np.testing.assert_array_equal(p, w)


@pytest.mark.parametrize('seed', range(40))
def test_product_anchor_generation_fuzz(gold, seed):
    """PRODUCT code: the library's host-side anchor generator (`ssdk_anchors_generate`, csrc/api.cu) behind the mirror's
    SSDInputEncoder constructor against the real reference on the same random configurations (no GPU needed)."""
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    cfg, _ = _encoder_case(seed)
    want = _results(gold, 'encoder/%d' % seed)
    m = SSDInputEncoder(**cfg)
    np.testing.assert_array_equal(m.anchors, want[0])
    tpl = m.generate_encoding_template(2)
    np.testing.assert_array_equal(tpl[0], want[2])
    np.testing.assert_array_equal(tpl[1], want[2])
    assert len(m.boxes_list) == len(want) - 3
    for a, b in zip(m.boxes_list, want[3:]):
        np.testing.assert_array_equal(a, b)
