"""The CUDA path against golden vectors produced by THE REFERENCE'S OWN SOURCE, directly (no oracle in between).

``tests/golden/ref_tf_shim_golden.npz`` holds the outputs of the reference's ``SSDLoss.compute_loss``, ``DecodeDetections`` /
``DecodeDetectionsFast`` / ``L2Normalization`` / ``AnchorBoxes`` ``.call`` and of the builders ``ssd_300`` / ``ssd_512`` /
``build_model`` (incl. ``mode='inference'`` / ``'inference_fast'``), executed unmodified over the NumPy stand-in of the
TensorFlow primitives (``tests/golden/make_tf_golden.py``).  Inputs that are not stored are regenerated from their seeds."""
import os

import numpy as np
import pytest

from oracle import synth
from oracle.model import ssd7_weight_shapes, vgg_weight_shapes

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_tf_shim_golden.npz'))
PRE = dict(subtract_mean=[123, 117, 104], divide_by_stddev=[64, 64, 64], swap_channels=[2, 1, 0])
SC300 = [0.1, 0.2, 0.37, 0.54, 0.71, 0.88, 1.05]
SC512 = [0.04, 0.1, 0.26, 0.42, 0.58, 0.74, 0.9, 1.06]


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


@pytest.mark.parametrize('key', ['plain', 'ratio2_alpha', 'no_pos', 'no_pos_negmin', 'ties', 'neutral', 'zero_neg_losses'])
def test_ssd_loss_kernel_vs_reference_code(key):
    from ssd_keras_b200.keras_loss_function.keras_ssd_loss import SSDLoss
    ratio, n_neg_min, alpha = G['loss/%s/kw' % key]
    out = SSDLoss(int(ratio), int(n_neg_min), float(alpha)).compute_loss(G['loss/%s/y_true' % key], G['loss/%s/y_pred' % key])
    ref = G['loss/%s/out' % key]
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-5, atol=1e-6)     # float32 summation order is the only freedom


@pytest.mark.parametrize('fast', [False, True])
@pytest.mark.parametrize('case', ['default', 'cap', 'topk_small', 'nonorm', 'none'])
def test_decode_layer_kernels_vs_reference_code(case, fast):
    import torch
    from ssd_keras_b200.keras_layers.keras_layer_DecodeDetections import DecodeDetections
    from ssd_keras_b200.keras_layers.keras_layer_DecodeDetectionsFast import DecodeDetectionsFast
    key = ('fast_' if fast else 'layer_') + case
    conf, iou, top_k, cap, norm = G['dec/%s/kw' % key]
    layer = (DecodeDetectionsFast if fast else DecodeDetections)(confidence_thresh=float(conf), iou_threshold=float(iou), top_k=int(top_k),
                                                                 nms_max_output_size=int(cap), normalize_coords=bool(norm),
                                                                 img_height=120, img_width=160)
    out = layer(torch.from_numpy(G['dec/y_pred']).cuda()).cpu().numpy()
    ref = G['dec/%s/out' % key]
    assert out.shape == ref.shape
    np.testing.assert_array_equal(out[..., 0], ref[..., 0])         # class ids, row by row (same order, same zero padding)
    np.testing.assert_array_equal(out[..., 1], ref[..., 1])         # confidences are copied, not computed
    np.testing.assert_allclose(out[..., 2:], ref[..., 2:], rtol=1e-6, atol=1e-4)


def test_l2_normalization_kernel_vs_reference_code():
    from ssd_keras_b200.keras_layers.keras_layer_L2Normalization import L2Normalization
    out = L2Normalization(gamma_init=20)(G['l2norm/x'])
    np.testing.assert_allclose(np.asarray(out), G['l2norm/out'], rtol=2e-6, atol=1e-6)


@pytest.mark.parametrize('key,fmap,kw', [
    ('tiny0', (6, 8), dict(img_height=120, img_width=160, this_scale=0.2, next_scale=0.45, aspect_ratios=[0.5, 1.0, 2.0],
                           two_boxes_for_ar1=True, coords='centroids', normalize_coords=True)),
    ('tiny1_clip_corners', (3, 4), dict(img_height=120, img_width=160, this_scale=0.45, next_scale=0.8, aspect_ratios=[0.5, 3.0],
                                        two_boxes_for_ar1=False, this_steps=(40, 41), this_offsets=(0.4, 0.6), clip_boxes=True,
                                        coords='corners', normalize_coords=False)),
    ('ssd300_conv4_3', (38, 38), dict(img_height=300, img_width=300, this_scale=0.1, next_scale=0.2, aspect_ratios=[1.0, 2.0, 0.5],
                                      two_boxes_for_ar1=True, this_steps=8, this_offsets=0.5, clip_boxes=False,
                                      coords='centroids', normalize_coords=True)),
])
def test_anchor_boxes_layer_vs_reference_code(key, fmap, kw):
    from ssd_keras_b200.keras_layers.keras_layer_AnchorBoxes import AnchorBoxes
    ref = G['anchors/%s/out' % key]
    out = AnchorBoxes(variances=[0.1, 0.1, 0.2, 0.2], **kw)(np.zeros((ref.shape[0],) + fmap + (8,), np.float32))
    np.testing.assert_array_equal(np.asarray(out), ref)               # float64 math, one rounding to float32: bit-exact


def _vgg_w(seed, variant, n_cls):
    w = synth.synth_weights(seed, vgg_weight_shapes(variant, n_cls), bias_scale=0.02)
    w['conv4_3_norm/gamma'] = np.random.default_rng(seed).uniform(10, 30, 512).astype(np.float32)
    return w


def _close_to_builder(y, rows, colsum, stride):
    """Element-wise: the oracle's own pin against the builders is rtol 2e-3 / atol 1e-4 (two float32 evaluation orders through
    ~23 layers); the wgmma path adds its own <= 1.5e-4 on the probabilities (tests/test_gpu_model.py), hence atol 3e-4.
    Column sums over all P rows: the bf16x3 accumulation error is systematic (truncating fp32 adds), so it does not average
    out -- bounded by 3e-5 per row on top of the float32 summation noise."""
    np.testing.assert_allclose(y[:, ::stride], rows, rtol=2e-3, atol=3e-4)
    np.testing.assert_allclose(y.astype(np.float64).sum(axis=1), colsum, rtol=1e-5, atol=1e-3 + 3e-5 * y.shape[1])


def test_ssd300_model_vs_reference_builder():
    """ssd_300 in all three modes against the real builder's outputs on the same image and weights."""
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    x = synth.synth_images(41, 1, 300, 300)
    w = _vgg_w(42, 300, 20)
    m = ssd_300((300, 300, 3), 20, mode='training', scales=SC300, **PRE)
    m.set_weights(w)
    y = m.predict(x)
    assert y.shape == (1, 8732, 33)
    _close_to_builder(y, G['model/ssd300/rows7'], G['model/ssd300/colsum'], 7)
    for mode in ('inference', 'inference_fast'):
        mi = ssd_300((300, 300, 3), 20, mode=mode, scales=SC300, confidence_thresh=0.01, iou_threshold=0.45, top_k=200,
                     nms_max_output_size=400, **PRE)
        mi.set_weights(w)
        out = mi.predict(x)
        ref = G['model/ssd300/' + mode]
        assert out.shape == ref.shape == (1, 200, 6)
        _same_detections(out[0], ref[0])


def _same_detections(out, ref, min_match=0.97):
    """Two float32 evaluations of a 23-layer network (the builder's run over torch-CPU convolutions, ours over bf16x3 tensor-core
    tiles) agree to ~1e-4 on the confidences.  Detections whose confidences are closer than that can swap places in the sorted
    output, and a near-threshold suppression can go the other way; everything else must be the same detection: same class, same
    confidence (5e-4), same box (0.5 px).  Required: the sorted confidence sequences agree row by row and at least 97 % of
    the reference's rows have such a partner."""
    np.testing.assert_allclose(out[:, 1], ref[:, 1], rtol=5e-4, atol=1e-6)          # both sorted by confidence
    used = np.zeros(len(out), bool)
    hit = 0
    for r in ref:
        cand = np.nonzero(~used & (out[:, 0] == r[0]) & (np.abs(out[:, 1] - r[1]) <= 5e-4 * max(abs(r[1]), 1e-3))
                          & (np.abs(out[:, 2:] - r[2:]).max(axis=1) <= 0.5))[0]
        if len(cand):
            used[cand[0]] = True
            hit += 1
    assert hit >= min_match * len(ref), 'only %d of %d reference detections found' % (hit, len(ref))


def test_ssd512_model_vs_reference_builder():
    from ssd_keras_b200.models.keras_ssd512 import ssd_512
    x = synth.synth_images(43, 1, 512, 512)
    m = ssd_512((512, 512, 3), 20, mode='training', scales=SC512, **PRE)
    m.set_weights(_vgg_w(44, 512, 20))
    y = m.predict(x)
    assert y.shape == (1, 24564, 33)
    _close_to_builder(y, G['model/ssd512/rows16'], G['model/ssd512/colsum'], 16)


def test_ssd7_model_vs_reference_builder():
    """300 x 480 input: also pins the height / width order of every anchor and reshape in the CUDA plan."""
    from ssd_keras_b200.models.keras_ssd7 import build_model
    x = synth.synth_images(45, 1, 300, 480)
    w = synth.synth_weights(46, ssd7_weight_shapes(5), bias_scale=0.05)
    rng = np.random.default_rng(47)
    for i in range(1, 8):
        c = w['conv%d/bias' % i].shape[0]
        w['bn%d/gamma' % i] = rng.uniform(0.8, 1.2, c).astype(np.float32)
        w['bn%d/beta' % i] = (rng.standard_normal(c) * 0.1).astype(np.float32)
        w['bn%d/moving_mean' % i] = (rng.standard_normal(c) * 0.1).astype(np.float32)
        w['bn%d/moving_variance' % i] = rng.uniform(0.5, 1.5, c).astype(np.float32)
    m = build_model((300, 480, 3), 5, mode='training', scales=[0.08, 0.16, 0.32, 0.64, 0.96], normalize_coords=True,
                    subtract_mean=127.5, divide_by_stddev=127.5)
    m.set_weights(w)
    y = m.predict(x)
    assert tuple(G['model/ssd7/shape']) == y.shape
    _close_to_builder(y, G['model/ssd7/rows5'], G['model/ssd7/colsum'], 5)
