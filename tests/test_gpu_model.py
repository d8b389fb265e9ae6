"""GPU parity tests for the wgmma convolution plan: SSD7 / SSD300 / SSD512 forward against the float32
torch-CPU oracle graphs (oracle/model.py) on identical synthetic weights and images.

Tolerances (north star: float32 box coordinates and loss within 1e-4): the default 'bf16x3' mode splits every operand into
bf16 hi+lo and issues hi*hi + hi*lo + lo*hi with fp32 accumulation.
  * every conv layer and the box offsets: 1e-4 of the tensor's max magnitude (CONV_TOL / OFF_TOL);
  * class probabilities on inputs that do not saturate the softmax (images normalised by the preprocessing lambdas, logits
    of order 10-20): a FIXED absolute bound PROB_ATOL = 1.5e-4;
  * one deliberately saturated case per model family (raw 0..255 images on he_normal weights, logits in the hundreds,
    exp() overflowing in float32 for some rows): there a relative logit error of 1e-5 already moves a probability by more
    than 1e-4, so the bound scales with max|logit| (SAT_REL) -- stated as what it is, a conditioning limit, not a precision
    claim.
The single-pass 'bf16' mode is checked at 5e-2.  Measured errors are appended to gpurun_out/model_errors.jsonl."""
import json
import os

import numpy as np
import pytest

from oracle import synth
from oracle import decoder as odec
from oracle.model import ssd7_forward, ssd7_weight_shapes, ssd_vgg_forward, vgg_weight_shapes

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
SC300 = [0.1, 0.2, 0.37, 0.54, 0.71, 0.88, 1.05]
SC512 = [0.04, 0.1, 0.26, 0.42, 0.58, 0.74, 0.9, 1.06]
SC7 = [0.08, 0.16, 0.32, 0.64, 0.96]
CONV_TOL = 1e-4
OFF_TOL = 1e-4
PROB_ATOL = 1.5e-4
SAT_REL = 3e-5
# preprocessing that keeps the network out of saturation: (x - mean) / 64, BGR swap (the reference's own lambdas)
PRE = dict(subtract_mean=[123, 117, 104], divide_by_stddev=[64, 64, 64], swap_channels=[2, 1, 0])


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


def _record(test, **kv):
    try:
        os.makedirs(os.path.join(ROOT, 'gpurun_out'), exist_ok=True)
        with open(os.path.join(ROOT, 'gpurun_out', 'model_errors.jsonl'), 'a') as f:
            f.write(json.dumps(dict(test=test, **{k: float(v) for k, v in kv.items()})) + '\n')
    except OSError:
        pass


def _ssd7_weights(seed, n_classes=5):
    w = synth.synth_weights(seed, ssd7_weight_shapes(n_classes), bias_scale=0.05)
    rng = np.random.default_rng(seed + 100)
    for i in range(1, 8):
        c = w['conv%d/bias' % i].shape[0]
        w['bn%d/gamma' % i] = rng.uniform(0.8, 1.2, c).astype(np.float32)
        w['bn%d/beta' % i] = (rng.standard_normal(c) * 0.1).astype(np.float32)
        w['bn%d/moving_mean' % i] = (rng.standard_normal(c) * 0.1).astype(np.float32)
        w['bn%d/moving_variance' % i] = rng.uniform(0.5, 1.5, c).astype(np.float32)
    return w


def _vgg_weights(seed, variant, n_classes):
    w = synth.synth_weights(seed, vgg_weight_shapes(variant, n_classes), bias_scale=0.02)
    w['conv4_3_norm/gamma'] = np.full((512,), 20.0, np.float32)
    return w


def _cmp_layers(test, model, feats, B, names, tol, rows=None):
    """Every named layer within `tol` of its max magnitude.  Returns {layer: error / max}; asserts after measuring all."""
    errs = {}
    for n in names:
        got = model.read_layer(n, B)
        ref = feats[n]
        if rows is not None:
            got = got[rows]
        assert got.shape == ref.shape, (n, got.shape, ref.shape)
        errs[n] = float(np.abs(got - ref).max() / max(float(np.abs(ref).max()), 1e-30))
    _record(test, **errs)
    bad = {k: v for k, v in errs.items() if not v <= tol}
    assert not bad, 'layers beyond %.1e of their max: %s (all: %s)' % (tol, bad, errs)
    return errs


def _cmp_pred(test, y, y_ref, feats, C, prob_atol=PROB_ATOL, off_tol=OFF_TOL):
    """Class probabilities at a fixed absolute bound, offsets relative to their max, anchors + variances bit-exact."""
    e_prob = float(np.abs(y[:, :, :C] - y_ref[:, :, :C]).max())
    e_off = float(np.abs(y[:, :, C:C + 4] - y_ref[:, :, C:C + 4]).max() / np.abs(y_ref[:, :, C:C + 4]).max())
    _record(test + ':pred', prob_abs=e_prob, off_rel=e_off, max_logit=np.abs(feats['logits']).max())
    np.testing.assert_array_equal(y[:, :, C + 4:], y_ref[:, :, C + 4:])
    assert e_prob <= prob_atol, 'class probabilities off by %.3e (bound %.1e, max|logit| %.1f)' % (e_prob, prob_atol, np.abs(feats['logits']).max())
    assert e_off <= off_tol, 'box offsets off by %.3e of their max (bound %.1e)' % (e_off, off_tol)


def _sat_atol(feats):
    return max(PROB_ATOL, SAT_REL * float(np.abs(feats['logits']).max()))


def _rows_equal_as_sets(a, b, rtol=1e-6, atol=1e-4):
    a = np.asarray(a, np.float64).reshape(-1, 6); b = np.asarray(b, np.float64).reshape(-1, 6)
    assert a.shape == b.shape, (a.shape, b.shape)
    ka = np.lexsort((a[:, 2], a[:, 0], -a[:, 1])); kb = np.lexsort((b[:, 2], b[:, 0], -b[:, 1]))
    a, b = a[ka], b[kb]
    np.testing.assert_array_equal(a[:, 0], b[:, 0])
    np.testing.assert_allclose(a[:, 1:], b[:, 1:], rtol=rtol, atol=atol)


def test_ssd7_config0_forward_and_decode():
    """BASELINE config 0: SSD7 forward + decode_detections on one synthetic 300x300 image (raw 0..255 pixels: the
    saturated case of this family), then the same network behind the normalising lambdas at the fixed bounds."""
    from ssd_keras_b200.models.keras_ssd7 import build_model
    from ssd_keras_b200.ssd_encoder_decoder.ssd_output_decoder import decode_detections
    w = _ssd7_weights(1)
    x = synth.synth_images(0, 1, 300, 300)
    model = build_model((300, 300, 3), 5, mode='training', scales=SC7, normalize_coords=True)
    model.set_weights(w)
    y = model.predict(x)
    y_ref, feats = ssd7_forward(x, w, n_classes=5, scales=SC7, normalize_coords=True, return_features=True)
    assert y.shape == (1, 7160, 18)
    _cmp_layers('ssd7_raw', model, feats, 1, ['conv1', 'conv4', 'conv7'], CONV_TOL)
    _cmp_pred('ssd7_raw', y, y_ref, feats, 6, prob_atol=_sat_atol(feats))
    # decode on identical inputs (the oracle's y_pred): the same detections, value for value, as the NumPy reference path
    kw = dict(confidence_thresh=0.3, iou_threshold=0.45, top_k=200, img_height=300, img_width=300)
    got = decode_detections(y_ref, **kw)
    exp = odec.decode_detections(y_ref, **kw)
    assert len(got) == len(exp) == 1
    _rows_equal_as_sets(got[0], exp[0])
    # ... and decoding the CUDA forward's own output gives the same detections as decoding it with the NumPy reference path
    got = decode_detections(y, **kw)
    exp = odec.decode_detections(y, **kw)
    _rows_equal_as_sets(got[0], exp[0])
    # normalised inputs: fixed bounds
    pre = dict(subtract_mean=[127.5] * 3, divide_by_stddev=[127.5] * 3, swap_channels=[2, 1, 0])
    m2 = build_model((300, 300, 3), 5, mode='training', scales=SC7, normalize_coords=True, **pre)
    m2.set_weights(w)
    y2 = m2.predict(x)
    y2_ref, f2 = ssd7_forward(x, w, n_classes=5, scales=SC7, normalize_coords=True, return_features=True, **pre)
    _cmp_layers('ssd7_norm', m2, f2, 1, ['conv1', 'conv4', 'conv7'], CONV_TOL)
    _cmp_pred('ssd7_norm', y2, y2_ref, f2, 6)


LAYERS300 = ['conv1_1', 'conv1_2', 'conv2_2', 'conv3_3', 'conv4_3', 'conv5_3', 'fc6', 'fc7', 'conv6_2', 'conv7_2', 'conv8_2',
             'conv9_2', 'conv4_3_norm']


def test_ssd300_forward_layers():
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    B = 2
    w = _vgg_weights(1, 300, 20)
    x = synth.synth_images(0, B, 300, 300)
    model = ssd_300((300, 300, 3), 20, mode='training', scales=SC300, **PRE)
    model.set_weights(w)
    y = model.predict(x)
    y_ref, feats = ssd_vgg_forward(x, w, 300, 20, scales=SC300, return_features=True, **PRE)
    assert y.shape == (B, 8732, 33)
    _cmp_layers('ssd300_b2', model, feats, B, LAYERS300, CONV_TOL)
    _cmp_pred('ssd300_b2', y, y_ref, feats, 21)


def test_ssd300_forward_saturated_raw_pixels():
    """The reference's default preprocessing (mean subtraction only) on he_normal weights: logits in the hundreds."""
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    B = 2
    w = _vgg_weights(1, 300, 20)
    x = synth.synth_images(0, B, 300, 300)
    model = ssd_300((300, 300, 3), 20, mode='training', scales=SC300)
    model.set_weights(w)
    y = model.predict(x)
    y_ref, feats = ssd_vgg_forward(x, w, 300, 20, scales=SC300, return_features=True)
    _cmp_layers('ssd300_raw', model, feats, B, LAYERS300, CONV_TOL)
    _cmp_pred('ssd300_raw', y, y_ref, feats, 21, prob_atol=_sat_atol(feats))


def test_ssd300_single_pass_bf16_mode():
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    B = 2
    w = _vgg_weights(1, 300, 20)
    x = synth.synth_images(0, B, 300, 300)
    model = ssd_300((300, 300, 3), 20, mode='training', scales=SC300, precision='bf16', **PRE)
    model.set_weights(w)
    y = model.predict(x)
    y_ref, feats = ssd_vgg_forward(x, w, 300, 20, scales=SC300, return_features=True, **PRE)
    _cmp_layers('ssd300_bf16', model, feats, B, LAYERS300, 5e-2)
    np.testing.assert_array_equal(y[:, :, 25:], y_ref[:, :, 25:])


def test_ssd300_batch32_layers():
    """The benchmark configuration itself (BASELINE configs[1]: batch 32): at this size the 64/128-channel layers run with
    two m-tiles per work unit and the deep layers with the cross-term accumulator, plans that small batches do not select."""
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    import torch
    B = 32
    w = _vgg_weights(5, 300, 20)
    x = synth.synth_images(6, B, 300, 300)
    model = ssd_300((300, 300, 3), 20, mode='training', scales=SC300, **PRE)
    model.set_weights(w)
    y = model.predict(x)
    threads = torch.get_num_threads()
    torch.set_num_threads(min(32, os.cpu_count() or 1))        # torch's CPU convolutions are slowest with every core of a big host
    try:
        y_ref, feats = ssd_vgg_forward(x, w, 300, 20, scales=SC300, return_features=True, **PRE)
    finally:
        torch.set_num_threads(threads)
    assert y.shape == (B, 8732, 33)
    _cmp_layers('ssd300_b32', model, feats, B, ['conv1_1', 'conv1_2', 'conv2_1', 'conv2_2', 'conv3_1', 'conv3_3', 'conv4_3', 'conv4_3_norm',
                                               'fc7', 'conv6_2', 'conv9_2'], CONV_TOL)
    _cmp_pred('ssd300_b32', y, y_ref, feats, 21)


def test_ssd300_inference_mode_matches_layer_oracle():
    """mode='inference' / 'inference_fast': (B,200,6).  Decoded from identical y_pred the output equals the layer oracle: class
    ids and confidences bit for bit, row by row; all four coordinates at 1e-6 relative."""
    import torch
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    B = 2
    w = _vgg_weights(1, 300, 20)
    x = synth.synth_images(0, B, 300, 300)
    model = ssd_300((300, 300, 3), 20, mode='inference', scales=SC300, **PRE)
    model.set_weights(w)
    xd = torch.from_numpy(x).cuda()
    y_pred = model.forward_device(xd).cpu().numpy()
    out = model.predict(x)
    assert out.shape == (B, 200, 6)
    ref = odec.decode_layer(y_pred, 0.01, 0.45, 200, 400, True, 300, 300)
    np.testing.assert_array_equal(out[:, :, :2], ref[:, :, :2])
    np.testing.assert_allclose(out[:, :, 2:], ref[:, :, 2:], rtol=1e-6, atol=1e-4)
    fast = ssd_300((300, 300, 3), 20, mode='inference_fast', scales=SC300, **PRE)
    fast.set_weights(w)
    outf = fast.predict(x)
    reff = odec.decode_layer_fast(y_pred, 0.01, 0.45, 200, 400, True, 300, 300)
    np.testing.assert_array_equal(outf[:, :, :2], reff[:, :, :2])
    np.testing.assert_allclose(outf[:, :, 2:], reff[:, :, 2:], rtol=1e-6, atol=1e-4)      # all six columns


def test_ssd512_forward():
    from ssd_keras_b200.models.keras_ssd512 import ssd_512
    B = 1
    w = _vgg_weights(2, 512, 80)
    x = synth.synth_images(3, B, 512, 512)
    model = ssd_512((512, 512, 3), 80, mode='training', scales=SC512, **PRE)
    model.set_weights(w)
    y = model.predict(x)
    y_ref, feats = ssd_vgg_forward(x, w, 512, 80, scales=SC512, return_features=True, **PRE)
    assert y.shape == (B, 24564, 93)
    _cmp_layers('ssd512_b1', model, feats, B, ['conv1_2', 'conv4_3', 'fc7', 'conv8_2', 'conv9_2', 'conv10_2'], CONV_TOL)
    _cmp_pred('ssd512_b1', y, y_ref, feats, 81)


def test_ssd512_config4_inference_fast_batch16():
    """BASELINE config 4 as stated: SSD512, 81 classes (COCO), 24564 priors, batch 16, mode='inference_fast'
    (DecodeDetectionsFast 0.01 / 0.45 / 200 / 400) through the model.  The forward of the first and last image is checked
    against the float32 oracle (the batch dimension is independent), the decoded (16,200,6) output against the layer
    oracle applied to the very same predictions: ids and confidences bit-exact, coordinates 1e-6."""
    import torch
    from ssd_keras_b200.models.keras_ssd512 import ssd_512
    B = 16
    w = _vgg_weights(4, 512, 80)
    x = synth.synth_images(8, B, 512, 512)
    model = ssd_512((512, 512, 3), 80, mode='inference_fast', scales=SC512, **PRE)
    model.set_weights(w)
    xd = torch.from_numpy(x).cuda()
    y_pred = model.forward_device(xd).cpu().numpy()
    assert y_pred.shape == (B, 24564, 93)
    sel = [0, B - 1]
    threads = torch.get_num_threads()
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    try:
        y_ref, feats = ssd_vgg_forward(x[sel], w, 512, 80, scales=SC512, return_features=True, **PRE)
    finally:
        torch.set_num_threads(threads)
    _cmp_layers('ssd512_b16', model, feats, B, ['conv1_2', 'conv3_3', 'conv4_3', 'fc7', 'conv6_2', 'conv10_2'], CONV_TOL, rows=sel)
    _cmp_pred('ssd512_b16', y_pred[sel], y_ref, feats, 81)
    out = model.predict(x)
    assert out.shape == (B, 200, 6)
    with np.errstate(all='ignore'):
        ref = odec.decode_layer_fast(y_pred, 0.01, 0.45, 200, 400, True, 512, 512)
    np.testing.assert_array_equal(out[:, :, :2], ref[:, :, :2])
    np.testing.assert_allclose(out[:, :, 2:], ref[:, :, 2:], rtol=1e-6, atol=1e-4)
    assert (out[:, :, 1] > 0).any()


def test_l2_normalization_layer():
    import torch
    from ssd_keras_b200.keras_layers.keras_layer_L2Normalization import L2Normalization
    rng = np.random.default_rng(0)
    x = rng.standard_normal((2, 7, 5, 512)).astype(np.float32) * 3
    x[0, 0, 0] = 0                                             # zero vector: the 1e-12 clamp
    out = L2Normalization(gamma_init=20)(x)
    ss = np.maximum((x.astype(np.float64) ** 2).sum(-1, keepdims=True), 1e-12)
    np.testing.assert_allclose(out, x / np.sqrt(ss) * 20.0, rtol=2e-6, atol=1e-6)


def test_weights_roundtrip(tmp_path):
    from ssd_keras_b200.models.keras_ssd7 import build_model
    m = build_model((96, 96, 3), 5, scales=SC7)
    p = str(tmp_path / 'w.npz')
    m.save_weights(p)
    m2 = build_model((96, 96, 3), 5, scales=SC7, weights_seed=9)
    m2.load_weights(p, by_name=True)
    for k, v in m.get_weights().items():
        np.testing.assert_array_equal(v, m2.get_weights()[k])
    with pytest.raises(ValueError):
        m2.set_weights({'conv1/kernel': np.zeros((3, 3, 3, 32), np.float32)})
