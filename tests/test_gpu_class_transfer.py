"""GPU tests of weight_sampling_tutorial.ipynb end to end: an 80-class (COCO) SSD300 whose class heads are sub-sampled to 8
classes by ``subsample_classifier_weights`` must predict, on the same images, the source's class probabilities restricted to
the kept classes (softmax over a subset S is ``P[..., S] / sum(P[..., S])``), the same box offsets and the same anchors; the
transferred model decodes, fine-tunes with the tutorial's ``Adam`` + ``SSDLoss`` and round-trips through ``save`` /
``load_model``; a 21-class model up-sampled to 30 classes builds, loads and trains.

Bars are those of tests/test_gpu_model.py for a whole network: relative to the tensor's maximum, 1e-4 under 'bf16x3' and
5e-2 under 'bf16'; anchors and variances bit for bit.  The images are normalised by the preprocessing lambdas (mean, then
/64) so that the softmax is not saturated and a restricted softmax is well conditioned."""
import numpy as np
import pytest

from oracle import decoder as odec
from oracle import synth
from oracle.encoder import OracleEncoder
from oracle.model import vgg_weight_shapes
from sampling_cases import TUTORIAL_CLASSES, in_keras_order

pytestmark = pytest.mark.gpu

COCO_SCALES = [0.07, 0.15, 0.33, 0.51, 0.69, 0.87, 1.05]
PRE = dict(subtract_mean=[123, 117, 104], divide_by_stddev=[64, 64, 64], swap_channels=[2, 1, 0])
TOL = {'bf16x3': 1e-4, 'bf16': 5e-2}
B = 4


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


def _source_file(path, n_classes, seed):
    from ssd_keras_b200.misc_utils.hdf5_lite import write_keras_weights
    w = synth.synth_weights(seed, vgg_weight_shapes(300, n_classes), bias_scale=0.02)
    w['conv4_3_norm/gamma'] = np.full((512,), 20.0, np.float32)
    write_keras_weights(path, in_keras_order(w))
    return path


@pytest.fixture(scope='module')
def files(tmp_path_factory):
    from ssd_keras_b200.misc_utils.tensor_sampling_utils import SSD300_CLASSIFIER_NAMES, subsample_classifier_weights
    d = tmp_path_factory.mktemp('class_transfer')
    src = _source_file(str(d / 'coco_80.h5'), 80, 1)
    dst = str(d / 'coco_80_subsampled_8.h5')
    np.random.seed(0)
    subsample_classifier_weights(src, dst, SSD300_CLASSIFIER_NAMES, 81, TUTORIAL_CLASSES)
    return src, dst


def _model(n_classes, path, mode='training', precision='bf16x3'):
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    m = ssd_300((300, 300, 3), n_classes, mode=mode, scales=COCO_SCALES, precision=precision, **PRE)
    m.load_weights(path, by_name=True)
    return m


def _images():
    import torch
    return torch.from_numpy(synth.synth_images(0, B, 300, 300)).cuda()


@pytest.mark.parametrize('precision', ['bf16x3', 'bf16'])
def test_transferred_model_predicts_the_source_restricted_to_its_classes(files, precision):
    src, dst = files
    x = _images()
    p_src = _model(80, src, precision=precision).predict_device(x).cpu().numpy()
    p_dst = _model(8, dst, precision=precision).predict_device(x).cpu().numpy()
    assert p_src.shape == (B, 8732, 93) and p_dst.shape == (B, 8732, 21)
    kept = p_src[..., TUTORIAL_CLASSES].astype(np.float64)
    expect = kept / kept.sum(axis=-1, keepdims=True)
    e_cls = np.abs(p_dst[..., :9] - expect).max() / np.abs(expect).max()
    off_src, off_dst = p_src[..., 81:85].astype(np.float64), p_dst[..., 9:13]
    e_off = np.abs(off_dst - off_src).max() / np.abs(off_src).max()
    assert e_cls <= TOL[precision], 'class columns off by %.3e of their max (bound %.1e)' % (e_cls, TOL[precision])
    assert e_off <= TOL[precision], 'box offsets off by %.3e of their max (bound %.1e)' % (e_off, TOL[precision])
    np.testing.assert_array_equal(p_dst[..., 13:], p_src[..., 85:])


def test_transferred_inference_model_decodes_its_own_predictions(files):
    """mode='inference': the 8-class model's detections equal DecodeDetections (the layer oracle) of its own raw y_pred, as
    tests/test_gpu_model.py holds them: class ids and confidences bit for bit, coordinates at 1e-6 relative."""
    _, dst = files
    x = _images()
    m = _model(8, dst, mode='inference')
    y_pred = m.forward_device(x).cpu().numpy()
    out = m.predict(x.cpu().numpy())
    assert out.shape == (B, 200, 6)
    ref = odec.decode_layer(y_pred, 0.01, 0.45, 200, 400, True, 300, 300)
    np.testing.assert_array_equal(out[:, :, :2], ref[:, :, :2])
    np.testing.assert_allclose(out[:, :, 2:], ref[:, :, 2:], rtol=1e-6, atol=1e-4)


def _encoded_batch(m, seed):
    n = m.n_classes - 1
    enc = OracleEncoder(300, 300, n, m.predictor_sizes, scales=COCO_SCALES, aspect_ratios_per_layer=m.anchor_cfg['aspect_ratios_per_layer'],
                        steps=[8, 16, 32, 64, 100, 300], variances=[0.1, 0.1, 0.2, 0.2])
    assert np.array_equal(enc.anchors, m.anchors)
    return synth.synth_images(seed, B, 300, 300), enc(synth.synth_gt(seed + 50, B, 4, 300, 300, n)).astype(np.float32)


def _compile(m):
    from ssd_keras_b200.keras_loss_function.keras_ssd_loss import SSDLoss
    from ssd_keras_b200.optimizers import Adam
    ssd_loss = SSDLoss(neg_pos_ratio=3, alpha=1.0)
    m.compile(optimizer=Adam(lr=0.001, beta_1=0.9, beta_2=0.999, epsilon=1e-08, decay=0.0), loss=ssd_loss.compute_loss)
    return ssd_loss


def test_fine_tune_the_transferred_model_and_save_it(files, tmp_path):
    from ssd_keras_b200.models import load_model
    _, dst = files
    m = _model(8, dst)
    ssd_loss = _compile(m)
    x, y = _encoded_batch(m, 7)
    losses = [float(m.train_on_batch(x, y)) for _ in range(20)]
    assert np.all(np.isfinite(losses)), losses
    assert losses[-1] < losses[0], losses
    path = str(tmp_path / 'fine_tuned.h5')
    m.save(path)
    m2 = load_model(path, custom_objects={'compute_loss': ssd_loss.compute_loss})
    w, w2 = m.get_weights(), m2.get_weights()
    assert sorted(w) == sorted(w2)
    for k in w:
        assert w2[k].dtype == w[k].dtype and w2[k].tobytes() == w[k].tobytes(), k


def test_upsample_21_to_30_classes_builds_loads_and_trains(tmp_path):
    from ssd_keras_b200.misc_utils.hdf5_lite import read_keras_weights
    from ssd_keras_b200.misc_utils.tensor_sampling_utils import SSD300_CLASSIFIER_NAMES, subsample_classifier_weights
    src = _source_file(str(tmp_path / 'voc_20.h5'), 20, 2)
    dst = str(tmp_path / 'up_29.h5')
    np.random.seed(1)
    subsample_classifier_weights(src, dst, SSD300_CLASSIFIER_NAMES, 21, 30)
    assert read_keras_weights(dst)['fc7_mbox_conf/kernel'].shape == (3, 3, 1024, 6 * 30)
    m = _model(29, dst)
    _compile(m)
    x, y = _encoded_batch(m, 9)
    loss = float(m.train_on_batch(x, y))
    assert np.isfinite(loss)
