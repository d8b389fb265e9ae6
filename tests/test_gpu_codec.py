"""GPU parity tests (run with -m gpu on an H100): CUDA encode / decode / loss / IoU through the C-ABI,
checked against the oracle and the committed golden fixtures.  Bars: bit-exact for match assignments, class
ids and NMS survivor indices; every encoded float column is the oracle rounded once to float32 (centroid log columns: either
neighbour of a value within 4 float64 ulps of a float32 midpoint); 1e-6..1e-4 relative (stated per test) for decoded
coordinates and losses."""
import numpy as np
import pytest

import encode_cases as ec
from oracle import synth
from oracle import decoder as odec
from oracle.boxes import iou as oracle_iou
from oracle.encoder import OracleEncoder
from oracle.loss import ssd_loss, ssd_loss_grad

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


def _enc(cfg):
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    return SSDInputEncoder(**cfg)


def _check_encode(cfg, gts):
    import torch
    enc = _enc(cfg)
    y = enc(gts)
    y_ref, m_ref, n_ref = OracleEncoder(**cfg)(gts, return_matches=True)
    assert y.shape == y_ref.shape and y.dtype == np.float64
    C = enc.n_classes
    # class vectors (incl. neutral rows) bit-exact
    np.testing.assert_array_equal(y[:, :, :C], y_ref[:, :, :C])
    # float32 kernel output vs float64 oracle
    ec.assert_float_columns(y[:, :, C:].astype(np.float32), y_ref[:, :, C:], C, cfg.get('coords', 'centroids'))
    # integer match assignments through the device entry point
    rows = [np.asarray(g, np.float32).reshape(-1, 5) for g in gts]
    offs = np.cumsum([0] + [r.shape[0] for r in rows]).astype(np.int32)
    flat = np.concatenate(rows, axis=0) if offs[-1] else np.zeros((0, 5), np.float32)
    gdev = torch.from_numpy(flat).cuda() if offs[-1] else None
    yd, match = enc.encode_device(gdev, offs, return_matches=True)
    match = match.cpu().numpy()
    exp = np.where(m_ref >= 0, m_ref, np.where(n_ref, -2, -1))
    np.testing.assert_array_equal(match, exp)
    assert int(enc.last_status.item()) == 0
    return y, y_ref


@pytest.mark.parametrize('key,cfg_name', [('tiny', 'tiny'), ('tiny_corners', 'tiny'), ('tiny_minmax', 'tiny'),
                                          ('tiny_bip', 'tiny_clip_abs'), ('tiny_bg3', 'tiny'), ('tiny_incl', 'tiny')])
def test_encode_golden_small(golden, configs, key, cfg_name):
    arr, meta = golden
    m = meta['enc/' + key]
    cfg = dict(configs[cfg_name]); cfg.update(m['over'])
    gts = [arr['enc/%s/gt%d' % (key, i)] for i in range(m['n_gt'])]
    y, _ = _check_encode(cfg, gts)
    # and directly against the tensor the real reference produced
    ref = arr['enc/%s/y' % key]
    C = cfg['n_classes'] + 1
    np.testing.assert_array_equal(y[:, :, :C], ref[:, :, :C])
    ec.assert_float_columns(y[:, :, C:].astype(np.float32), ref[:, :, C:], C, cfg.get('coords', 'centroids'))


def test_encode_ssd300_config3(configs):
    """SURVEY 8d config 3: B=32, G=8, SSD300/VOC -> 2397 positives, 0 neutral."""
    gts = synth.synth_gt(2, 32, 8, 300, 300, 20)
    y, _ = _check_encode(configs['ssd300'], gts)
    assert int((y[:, :, 1:21].max(-1) > 0).sum()) == 2397
    cfg = dict(configs['ssd300']); cfg['neg_iou_limit'] = 0.3
    y, _ = _check_encode(cfg, gts)
    assert int((y[:, :, :21].sum(-1) == 0).sum()) == 15743


def test_encode_ssd512_coco(configs):
    _check_encode(configs['ssd512'], synth.synth_gt(7, 4, 24, 512, 512, 80))


def test_encode_micro_golden(golden, configs):
    """P = 100000 priors x G = 128 (config 5), first image, against the real reference's match list."""
    arr, meta = golden
    gts = [arr['enc/micro/gt0']]
    y, y_ref = _check_encode(configs['micro'], gts)
    pos = np.argwhere(y[:, :, 1:21].max(-1) > 0)
    np.testing.assert_array_equal(pos, arr['enc/micro/pos'])
    np.testing.assert_array_equal(y[pos[:, 0], pos[:, 1], :21].argmax(-1), arr['enc/micro/pos_cls'])
    np.testing.assert_allclose(y[pos[:, 0], pos[:, 1], 21:25], arr['enc/micro/pos_off'], rtol=1e-6, atol=1e-6)
    np.testing.assert_array_equal(np.argwhere(y[:, :, :21].sum(-1) == 0), arr['enc/micro/neutral'])


def test_encode_edge_cases(configs):
    cfg = configs['tiny']
    gts = synth.synth_gt(5, 6, 3, 160, 120, 3)
    gts[0] = np.zeros((0, 5), np.float32)                         # empty images
    gts[5] = np.zeros((0, 5), np.float32)
    gts[2] = np.repeat(gts[2][:1], 4, axis=0)                     # identical boxes -> ties, bipartite collisions
    gts[3] = np.array([[1, 0, 0, 3, 3], [2, 1, 1, 2.5, 2.5], [3, 150, 110, 159, 119]], np.float32)   # all-zero IoU rows (quirk)
    _check_encode(cfg, gts)
    _check_encode(cfg, [np.zeros((0, 5), np.float32)] * 3)        # nothing at all
    big = synth.synth_gt(9, 2, 300, 160, 120, 3)                  # many boxes per image
    _check_encode(cfg, big)


@pytest.mark.parametrize('spatial_min', ['0', '100000'])
def test_encode_both_tile_sets(configs, monkeypatch, spatial_min):
    """The encoder groups priors either into runs of 256 consecutive priors or into compact blocks of feature-map cells
    (picked by the number of boxes per image); both groupings must give the reference's result on every kind of input."""
    monkeypatch.setenv('SSDK_ENC_SPATIAL_MIN', spatial_min)
    gts = synth.synth_gt(2, 4, 8, 300, 300, 20)
    _check_encode(configs['ssd300'], gts)
    cfg = dict(configs['ssd300']); cfg['neg_iou_limit'] = 0.3
    _check_encode(cfg, synth.synth_gt(12, 3, 40, 300, 300, 20))
    _check_encode(configs['ssd512'], synth.synth_gt(7, 2, 30, 512, 512, 80))
    _check_encode(configs['ssd7'], synth.synth_gt(8, 3, 12, 300, 300, 5))
    tiny = synth.synth_gt(5, 6, 3, 160, 120, 3)
    tiny[0] = np.zeros((0, 5), np.float32)
    tiny[2] = np.repeat(tiny[2][:1], 4, axis=0)
    tiny[3] = np.array([[1, 0, 0, 3, 3], [2, 1, 1, 2.5, 2.5], [3, 150, 110, 159, 119]], np.float32)
    _check_encode(configs['tiny'], tiny)
    _check_encode(configs['tiny_clip_abs'], tiny)
    _check_encode(configs['tiny'], synth.synth_gt(9, 2, 300, 160, 120, 3))      # 300 boxes on 240 priors: contested priors
    for tpc in ('1', '4'):
        monkeypatch.setenv('SSDK_ENC_TPC', tpc)
        _check_encode(configs['ssd300'], synth.synth_gt(13, 2, 60, 300, 300, 20))
    monkeypatch.delenv('SSDK_ENC_TPC')


def test_encode_integer_pixel_labels_ties(configs):
    """Integer pixel coordinates on a regular prior grid produce exact IoU ties between neighbouring priors (and between
    tiles): np.argmax's first-index rule must hold in both matching stages."""
    rng = np.random.default_rng(77)
    gts = []
    for _ in range(4):
        n = 12
        x0 = rng.integers(0, 200, n) // 4 * 4; y0 = rng.integers(0, 200, n) // 4 * 4
        w = rng.integers(2, 20, n) * 8; h = rng.integers(2, 20, n) * 8
        gts.append(np.stack([rng.integers(1, 21, n), x0, y0, np.minimum(x0 + w, 299), np.minimum(y0 + h, 299)], 1).astype(np.float32))
    _check_encode(configs['ssd300'], gts)
    cfg = dict(configs['ssd7']); cfg['neg_iou_limit'] = 0.3
    g7 = []
    for g in gts:
        g = g.copy(); g[:, 0] = (g[:, 0] - 1) % 5 + 1
        g7.append(g)
    _check_encode(cfg, g7)


def test_encode_float64_labels(configs):
    """Labels that float32 cannot hold: the reference computes on float64 copies (:330) and so does ssdk_encode with gt_f64 = 1."""
    rng = np.random.default_rng(3)
    gts = []
    for _ in range(3):
        n = 6
        x0 = rng.uniform(0, 200, n); y0 = rng.uniform(0, 200, n)
        gts.append(np.stack([rng.integers(1, 21, n).astype(np.float64), x0, y0, x0 + rng.uniform(10, 90, n),
                             y0 + rng.uniform(10, 90, n)], 1))
    assert any((g.astype(np.float32).astype(np.float64) != g).any() for g in gts)
    enc = _enc(configs['ssd300'])
    y = enc(gts)
    y_ref = OracleEncoder(**configs['ssd300'])(gts)
    np.testing.assert_array_equal(y[:, :, :21], y_ref[:, :, :21])
    ec.assert_float_columns(y[:, :, 21:].astype(np.float32), y_ref[:, :, 21:], 21, 'centroids')
    with pytest.raises(IndexError):
        enc([np.array([[21, 10., 10., 50., 60.]])])               # class id outside [0, n_classes]: np.eye row gather fails


def test_encode_large_batch_and_device_offsets(configs):
    """B > 1024: the offsets no longer fit the launch arguments and travel through the pinned ring; and the entry that
    takes offsets which already live on the device."""
    import torch
    cfg = configs['tiny']
    gts = synth.synth_gt(21, 1100, 2, 160, 120, 3)
    enc = _enc(cfg)
    y = enc(gts)
    y_ref = OracleEncoder(**cfg)(gts)
    np.testing.assert_array_equal(y[:, :, :4], y_ref[:, :, :4])
    ec.assert_float_columns(y[:, :, 4:].astype(np.float32), y_ref[:, :, 4:], 4, 'centroids')
    gts = synth.synth_gt(22, 5, 7, 160, 120, 3)
    offs = np.cumsum([0] + [g.shape[0] for g in gts]).astype(np.int32)
    gd = torch.from_numpy(np.concatenate(gts)).cuda()
    yd = enc.encode_device_offsets(gd, torch.from_numpy(offs).cuda(), int(offs[-1]), 7).cpu().numpy()
    np.testing.assert_array_equal(yd, enc.encode_device(gd, offs).cpu().numpy())
    with pytest.raises(ValueError, match='float64 rows need host offsets'):
        enc.encode_device_offsets(gd.double(), torch.from_numpy(offs).cuda(), int(offs[-1]), 7)
    out = torch.empty((5, enc.anchors.shape[0], enc.n_classes + 12), dtype=torch.float32, device='cuda')
    assert enc.encode_device(gd, offs, out=out) is out
    np.testing.assert_array_equal(out.cpu().numpy(), yd)
    # repeated launches reuse the per-image tickets
    for _ in range(3):
        np.testing.assert_array_equal(enc.encode_device(gd, offs).cpu().numpy(), yd)


def test_encode_degenerate_raises(configs):
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import DegenerateBoxError
    enc = _enc(configs['tiny'])
    with pytest.raises(DegenerateBoxError):
        enc([np.array([[1, 10., 10., 10., 20.]])])
    import torch
    g = torch.tensor([[1, 5., 5., 50., 60.], [1, 10., 10., 10., 20.]], dtype=torch.float32).cuda()
    enc.encode_device(g, np.array([0, 1, 2], np.int32))
    assert int(enc.last_status.item()) == 2                        # 1-based index of the offending image


def test_iou_matches_reference_arithmetic(golden):
    from ssd_keras_b200.bounding_box_utils.bounding_box_utils import convert_coordinates, iou
    arr, _ = golden
    b1, b2 = arr['iou/b1'], arr['iou/b2']
    for bp in ('half', 'include', 'exclude'):
        np.testing.assert_array_equal(iou(b1, b2, coords='corners', border_pixels=bp), arr['iou/outer/corners/' + bp])
        np.testing.assert_array_equal(iou(b2, b1[0], coords='corners', mode='element-wise', border_pixels=bp),
                                      arr['iou/elem/corners/' + bp])
    c1 = convert_coordinates(b1, 0, 'corners2centroids'); c2 = convert_coordinates(b2, 0, 'corners2centroids')
    np.testing.assert_array_equal(iou(c1, c2, coords='centroids'), arr['iou/outer/centroids'])
    rng = np.random.default_rng(0)
    a = rng.uniform(0, 1, (300, 4)); a[:, 2:] += a[:, :2]
    b = rng.uniform(0, 1, (700, 4)); b[:, 2:] += b[:, :2]
    np.testing.assert_array_equal(iou(a, b, coords='corners'), oracle_iou(a, b, coords='corners'))


# ------------------------------------------------------------------------------------------------
# decoders
# ------------------------------------------------------------------------------------------------
def _rows_equal_as_sets(a, b, rtol=1e-6, atol=1e-4):
    a = np.asarray(a, np.float64).reshape(-1, 6); b = np.asarray(b, np.float64).reshape(-1, 6)
    assert a.shape == b.shape, (a.shape, b.shape)
    ka = np.lexsort((a[:, 2], a[:, 0], -a[:, 1])); kb = np.lexsort((b[:, 2], b[:, 0], -b[:, 1]))
    a, b = a[ka], b[kb]
    np.testing.assert_array_equal(a[:, 0], b[:, 0])
    np.testing.assert_allclose(a[:, 1:], b[:, 1:], rtol=rtol, atol=atol)


@pytest.mark.parametrize('key,fast', [('tiny', False), ('tiny_topk', False), ('tiny_nonorm', False), ('tiny_empty', False),
                                      ('tiny_fast', True), ('tiny_fast_topk', True)])
def test_decode_numpy_api_golden(golden, key, fast):
    from ssd_keras_b200.ssd_encoder_decoder.ssd_output_decoder import decode_detections, decode_detections_fast
    arr, meta = golden
    m = meta['dec/' + key]
    res = (decode_detections_fast if fast else decode_detections)(arr['dec/%s/y_pred' % key], **m['kw'])
    assert [int(np.asarray(r).reshape(-1, 6).shape[0]) for r in res] == m['counts']
    for i, r in enumerate(res):
        _rows_equal_as_sets(r, arr['dec/%s/out%d' % (key, i)])


def test_decode_numpy_api_ssd300(golden, configs):
    from ssd_keras_b200.ssd_encoder_decoder.ssd_output_decoder import decode_detections, decode_detections_fast
    arr, meta = golden
    enc = OracleEncoder(**configs['ssd300'])
    yp = synth.synth_y_pred(23, 1, enc.anchors, 21, sharp=6.0, loc_scale=1.0)
    res = decode_detections(yp, confidence_thresh=0.5, iou_threshold=0.45, top_k=200, img_height=300, img_width=300)
    _rows_equal_as_sets(res[0], arr['dec/ssd300/out0'])
    res = decode_detections_fast(yp, confidence_thresh=0.5, iou_threshold=0.45, top_k=200, img_height=300, img_width=300)
    _rows_equal_as_sets(res[0], arr['dec/ssd300_fast/out0'])


@pytest.mark.parametrize('coords', ['centroids', 'corners', 'minmax'])
def test_decode_numpy_api_all_coords(configs, coords):
    from ssd_keras_b200.ssd_encoder_decoder.ssd_output_decoder import decode_detections, decode_detections_fast
    cfg = dict(configs['tiny']); cfg['coords'] = coords
    enc = OracleEncoder(**cfg)
    yp = synth.synth_y_pred(31, 3, enc.anchors.astype(np.float32), 4, sharp=3.0, loc_scale=0.3)
    kw = dict(confidence_thresh=0.05, iou_threshold=0.45, top_k=200, input_coords=coords, img_height=120, img_width=160)
    for r, e in zip(decode_detections(yp, **kw), odec.decode_detections(yp, **kw)):
        _rows_equal_as_sets(r, e)
    kw['confidence_thresh'] = 0.4
    for r, e in zip(decode_detections_fast(yp, **kw), odec.decode_detections_fast(yp, **kw)):
        _rows_equal_as_sets(r, e)


def _layer_check(y_pred, fast, H, W, conf=0.01, iou=0.45, top_k=200, cap=400):
    import torch
    from ssd_keras_b200.keras_layers.keras_layer_DecodeDetections import DecodeDetections
    from ssd_keras_b200.keras_layers.keras_layer_DecodeDetectionsFast import DecodeDetectionsFast
    cls = DecodeDetectionsFast if fast else DecodeDetections
    layer = cls(confidence_thresh=conf, iou_threshold=iou, top_k=top_k, nms_max_output_size=cap, img_height=H, img_width=W)
    out, idx = layer(torch.from_numpy(y_pred).cuda(), return_index=True)
    out, idx = out.cpu().numpy(), idx.cpu().numpy()
    ref, ridx = (odec.decode_layer_fast if fast else odec.decode_layer)(y_pred, conf, iou, top_k, cap, True, H, W, return_indices=True)
    assert out.shape == ref.shape == (y_pred.shape[0], top_k, 6)
    np.testing.assert_array_equal(idx, ridx)                       # survivor prior indices, in output order: bit-exact
    np.testing.assert_array_equal(out[:, :, :2], ref[:, :, :2])    # class ids and confidences
    np.testing.assert_allclose(out[:, :, 2:], ref[:, :, 2:], rtol=1e-6, atol=1e-4)
    return out


@pytest.mark.parametrize('fast', [False, True])
def test_decode_layer_ssd300(configs, fast):
    enc = OracleEncoder(**configs['ssd300'])
    # sharp predictions (few survivors) and flat ones (every prior passes 0.01 in every class: worst case)
    yp = synth.synth_y_pred(41, 2, enc.anchors.astype(np.float32), 21, sharp=5.0, loc_scale=1.0)
    _layer_check(yp, fast, 300, 300)
    yp = synth.synth_y_pred(42, 1, enc.anchors.astype(np.float32), 21, sharp=0.5, loc_scale=0.5)
    out = _layer_check(yp, fast, 300, 300)
    assert (out[:, :, 1] > 0).all()                                # 200 real detections


def test_decode_layer_ssd512_two_bands(configs):
    """P = 24564 > band capacity (16384): exercises the multi-band path."""
    enc = OracleEncoder(**configs['ssd512'])
    yp = synth.synth_y_pred(43, 1, enc.anchors.astype(np.float32), 81, sharp=0.3, loc_scale=0.5)
    _layer_check(yp, True, 512, 512, conf=0.0125)


def test_decode_layer_ties_and_empty(configs):
    enc = OracleEncoder(**configs['tiny'])
    anc = enc.anchors.astype(np.float32)
    yp = synth.synth_y_pred(44, 2, anc, 4, sharp=0.0, loc_scale=0.2)       # uniform softmax: every score ties
    _layer_check(yp, False, 120, 160, conf=0.01, top_k=20, cap=10)
    _layer_check(yp, False, 120, 160, conf=0.9, top_k=20, cap=10)          # nothing passes -> all zero rows


def test_nms_microbench_semantics():
    """config 5 NMS part at a reduced size: anchors as boxes, uniform scores, cap 400, top_k 200."""
    import torch
    from ssd_keras_b200.ssd_encoder_decoder.ssd_output_decoder import nms_device
    cfg = dict(img_height=1000, img_width=1600, n_classes=20, predictor_sizes=[(50, 80)], scales=[0.1, 0.2],
               aspect_ratios_global=[0.5, 1.0, 2.0], coords='corners', normalize_coords=False)
    anc = OracleEncoder(**cfg).anchors.astype(np.float32)
    n = anc.shape[0]
    B = 3
    scores = np.stack([np.random.default_rng(5 + i).uniform(0, 1, n) for i in range(B)]).astype(np.float32)
    boxes = np.broadcast_to(anc[None], (B, n, 4)).copy()
    out, cnt, idx = nms_device(torch.from_numpy(boxes).cuda(), torch.from_numpy(scores).cuda(), 0.01, 0.45, 400, 200, return_index=True)
    out, cnt, idx = out.cpu().numpy(), cnt.cpu().numpy(), idx.cpu().numpy()
    for b in range(B):
        m = np.nonzero(scores[b] > np.float32(0.01))[0]
        sel = odec.tf_nms_fast(boxes[b, m], scores[b, m], 400, 0.45)
        keep = m[sel]
        order = np.lexsort((np.arange(len(keep)), -scores[b, keep].astype(np.float64)))[:200]
        np.testing.assert_array_equal(idx[b, :len(order)], keep[order])
        assert cnt[b] == len(order)


def test_nms_config5_full_size():
    """config 5 NMS part at its stated size: 100 000 boxes per image (the micro-benchmark's prior grid as corner boxes),
    uniform scores, conf 0.01 / iou 0.45, cap 400, top_k 200."""
    import torch
    from ssd_keras_b200.ssd_encoder_decoder.ssd_output_decoder import nms_device
    cfg = dict(img_height=1000, img_width=1600, n_classes=20, predictor_sizes=[(125, 200)], scales=[0.1, 0.2],
               aspect_ratios_global=[0.5, 1.0, 2.0], coords='corners', normalize_coords=False)
    anc = OracleEncoder(**cfg).anchors.astype(np.float32)
    n = anc.shape[0]
    assert n == 100000
    B = 2
    scores = np.stack([np.random.default_rng(5 + i).uniform(0, 1, n) for i in range(B)]).astype(np.float32)
    boxes = np.broadcast_to(anc[None], (B, n, 4)).copy()
    out, cnt, idx = nms_device(torch.from_numpy(boxes).cuda(), torch.from_numpy(scores).cuda(), 0.01, 0.45, 400, 200, return_index=True)
    out, cnt, idx = out.cpu().numpy(), cnt.cpu().numpy(), idx.cpu().numpy()
    for b in range(B):
        m = np.nonzero(scores[b] > np.float32(0.01))[0]
        sel = odec.tf_nms_fast(boxes[b, m], scores[b, m], 400, 0.45)
        keep = m[sel]
        order = np.lexsort((np.arange(len(keep)), -scores[b, keep].astype(np.float64)))[:200]
        np.testing.assert_array_equal(idx[b, :len(order)], keep[order])
        assert cnt[b] == len(order)
        np.testing.assert_array_equal(out[b, :len(order), 1], scores[b, keep[order]])
        np.testing.assert_array_equal(out[b, :len(order), 2:], boxes[b, keep[order]])


def test_nms_large_n_multi_band():
    """n = 40000 random boxes > band capacity; uncapped enough to need several bands."""
    import torch
    from ssd_keras_b200.ssd_encoder_decoder.ssd_output_decoder import nms_device
    rng = np.random.default_rng(11)
    n = 40000
    xy = rng.uniform(0, 2000, (n, 2)); wh = rng.uniform(5, 40, (n, 2))
    boxes = np.concatenate([xy, xy + wh], axis=1).astype(np.float32)[None]
    scores = rng.uniform(0, 1, (1, n)).astype(np.float32)
    scores[0, ::7] = 0.5                                           # a block of exact ties across the band boundary
    out, cnt, idx = nms_device(torch.from_numpy(boxes).cuda(), torch.from_numpy(scores).cuda(), 0.01, 0.45, 30000, 200, return_index=True)
    m = np.nonzero(scores[0] > np.float32(0.01))[0]
    sel = odec.tf_nms_fast(boxes[0, m], scores[0, m], 30000, 0.45)
    keep = m[sel]
    order = np.lexsort((np.arange(len(keep)), -scores[0, keep].astype(np.float64)))[:200]
    np.testing.assert_array_equal(idx.cpu().numpy()[0], keep[order])


# ------------------------------------------------------------------------------------------------
# loss
# ------------------------------------------------------------------------------------------------
def _loss_case(cfg, seed, B, G, ncls, sharp, ratio=3, n_neg_min=0, alpha=1.0, tol=1e-4):
    import torch
    from ssd_keras_b200.keras_loss_function.keras_ssd_loss import SSDLoss
    enc = OracleEncoder(**cfg)
    y_true, y_pred = synth.synth_y_true_pred_for_loss(seed, enc, B, G, ncls, sharp=sharp)
    L = SSDLoss(neg_pos_ratio=ratio, n_neg_min=n_neg_min, alpha=alpha)
    loss, stats = L.loss_and_stats(y_true, y_pred)
    ref, parts = ssd_loss(y_true, y_pred, ratio, n_neg_min, alpha, return_parts=True)
    stats = stats.cpu().numpy()
    assert stats[0] == parts['n_positive'] and stats[2] == parts['k']            # integers: bit-exact
    np.testing.assert_allclose(loss.cpu().numpy(), ref, rtol=tol)
    # gradient through autograd (hand-written backward kernel)
    yp = torch.from_numpy(y_pred).cuda().requires_grad_(True)
    L.compute_loss(torch.from_numpy(y_true).cuda(), yp).mean().backward()
    g_ref = ssd_loss_grad(y_true, y_pred, ratio, n_neg_min, alpha)
    np.testing.assert_allclose(yp.grad.cpu().numpy(), g_ref, rtol=1e-4, atol=1e-7)
    return stats


def test_loss_tiny(configs):
    _loss_case(configs['tiny'], 51, 4, 3, 3, sharp=2.0)
    _loss_case(configs['tiny'], 52, 2, 1, 3, sharp=0.5, ratio=1, n_neg_min=7, alpha=0.5)


def test_loss_ssd300_config3(configs):
    stats = _loss_case(configs['ssd300'], 2, 32, 8, 20, sharp=2.0)
    assert stats[0] > 2000 and stats[2] == 3 * stats[0]


def test_loss_ties_and_no_positives(configs):
    import torch
    from ssd_keras_b200.keras_loss_function.keras_ssd_loss import SSDLoss
    enc = OracleEncoder(**configs['tiny'])
    B, P, W = 3, enc.anchors.shape[0], enc.n_classes + 12
    # every negative has exactly the same loss: the k kept ones must be the lowest flat indices
    y_true, _ = synth.synth_y_true_pred_for_loss(61, enc, B, 2, 3, sharp=1.0)
    y_pred = np.zeros((B, P, W), np.float32); y_pred[:, :, :4] = 0.25
    loss = SSDLoss().compute_loss(y_true, y_pred).cpu().numpy()
    np.testing.assert_allclose(loss, ssd_loss(y_true, y_pred), rtol=1e-5)
    g = ssd_loss_grad(y_true, y_pred)
    yp = torch.from_numpy(y_pred).cuda().requires_grad_(True)
    SSDLoss().compute_loss(torch.from_numpy(y_true).cuda(), yp).mean().backward()
    np.testing.assert_allclose(yp.grad.cpu().numpy(), g, rtol=1e-5, atol=1e-8)
    # no positives at all: k = n_neg_min = 0 -> zero loss (tf.cond branch f1)
    y_true0 = enc([np.zeros((0, 5))] * B).astype(np.float32)
    loss0 = SSDLoss().compute_loss(y_true0, y_pred).cpu().numpy()
    np.testing.assert_allclose(loss0, ssd_loss(y_true0, y_pred), atol=1e-7)
    loss1 = SSDLoss(n_neg_min=10).compute_loss(y_true0, y_pred).cpu().numpy()
    np.testing.assert_allclose(loss1, ssd_loss(y_true0, y_pred, n_neg_min=10), rtol=1e-5)


def _global_loss_by_hand(y_true, y_pred, shards, ratio=3, n_neg_min=0, alpha=1.0):
    """The phase-wise loss of `shards` ranks on ONE GPU: the NCCL all-reduces / all-gather replaced by adding the tensors."""
    import torch
    from ssd_keras_b200.distributed import GlobalLossRun
    B = y_true.shape[0]
    per = B // shards
    runs = [GlobalLossRun(torch.from_numpy(y_true[r * per:(r + 1) * per]).cuda(), torch.from_numpy(y_pred[r * per:(r + 1) * per]).cuda(),
                          ratio, n_neg_min, alpha, shards, r, True) for r in range(shards)]
    for r in runs:
        r.phase(0)
    for name in ('counts', 'hist1'):
        tot = sum(getattr(r, name).clone() for r in runs)
        for r in runs:
            getattr(r, name).copy_(tot)
    for r in runs:
        r.phase(1)
    tot = sum(r.hist2.clone() for r in runs)
    for r in runs:
        r.hist2.copy_(tot)
    for r in runs:
        r.phase(2); r.phase(3)
    ties = torch.cat([r.ties.clone() for r in runs])
    for r in runs:
        r.ties_all.copy_(ties); r.phase(4)
    return (np.concatenate([r.loss.cpu().numpy() for r in runs]), np.concatenate([r.grad.cpu().numpy() for r in runs]),
            runs[0].stats.cpu().numpy())


@pytest.mark.parametrize('shards', [1, 2, 4])
def test_loss_global_batch_exact_phases(configs, shards):
    """The multi-GPU loss mode (n_positive and the top-k over the whole sharded batch): its phase-wise launches, with the
    collectives emulated, give the single-process loss and gradient of the full batch -- also when every negative ties."""
    enc = OracleEncoder(**configs['ssd300'])
    y_true, y_pred = synth.synth_y_true_pred_for_loss(2, enc, 8, 8, 20, sharp=2.0)
    loss, grad, stats = _global_loss_by_hand(y_true, y_pred, shards)
    ref, parts = ssd_loss(y_true, y_pred, 3, 0, 1.0, return_parts=True)
    assert stats[0] == parts['n_positive'] and stats[2] == parts['k']
    np.testing.assert_allclose(loss, ref, rtol=1e-5)
    np.testing.assert_allclose(grad, ssd_loss_grad(y_true, y_pred, 3, 0, 1.0), rtol=1e-4, atol=1e-7)
    tiny = OracleEncoder(**configs['tiny'])
    yt, _ = synth.synth_y_true_pred_for_loss(61, tiny, 4, 2, 3, sharp=1.0)
    yp = np.zeros_like(yt); yp[:, :, :4] = 0.25                    # every negative has the same loss: global flat-index order decides
    loss, grad, _ = _global_loss_by_hand(yt, yp, shards)
    np.testing.assert_allclose(loss, ssd_loss(yt, yp), rtol=1e-5)
    np.testing.assert_allclose(grad, ssd_loss_grad(yt, yp), rtol=1e-5, atol=1e-8)
    yt0 = tiny([np.zeros((0, 5))] * 4).astype(np.float32)          # no positives anywhere
    loss, _, _ = _global_loss_by_hand(yt0, yp, shards, n_neg_min=10)
    np.testing.assert_allclose(loss, ssd_loss(yt0, yp, n_neg_min=10), rtol=1e-5)


def test_ssd_loss_with_loss_and_gradient_is_one_launch(configs):
    """ssdk_ssd_loss with the loss and the gradient (what the training step calls): one launch, the loss and gradient of the
    reference."""
    import ctypes as C
    import torch
    from ssd_keras_b200 import _ffi
    enc = OracleEncoder(**configs['ssd300'])
    y_true, y_pred = synth.synth_y_true_pred_for_loss(5, enc, 4, 8, 20, sharp=2.0)
    yt, yp = torch.from_numpy(y_true).cuda(), torch.from_numpy(y_pred).cuda()
    loss = torch.empty((4,), dtype=torch.float32, device='cuda'); grad = torch.empty_like(yp)
    n0 = _ffi.launch_count()
    _ffi.check(_ffi.lib().ssdk_ssd_loss(_ffi.context(), _ffi.dptr(yt), _ffi.dptr(yp), 4, yp.shape[1], 21, 3, 0, 1.0, _ffi.dptr(None),
                                        _ffi.dptr(loss), _ffi.dptr(None), _ffi.dptr(grad), _ffi.stream_ptr()))
    assert _ffi.launch_count() - n0 == 1
    np.testing.assert_allclose(loss.cpu().numpy(), ssd_loss(y_true, y_pred), rtol=1e-5)
    np.testing.assert_allclose(grad.cpu().numpy(), ssd_loss_grad(y_true, y_pred), rtol=1e-4, atol=1e-7)
