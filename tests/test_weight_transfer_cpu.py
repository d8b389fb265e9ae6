"""The class transfer of weight_sampling_tutorial.ipynb on files, without h5py: a reference-shaped SSD300 weights file (81
classes, layers in Keras' order, a layer this package does not use, chunked + gzip heads) through
``subsample_classifier_weights`` must come back with the source's layer order, ``weight_names`` and attributes, every tensor
but the twelve class-head ones byte for byte, and the class heads exactly as ``sample_tensors`` makes them under the same
seed.  Also the tutorial's sample chain: ``max_crop_patch`` / ``max_crop_ops`` against the REAL reference's
``RandomMaxCropFixedAR`` draws and, through the device's image and box oracles, its crop + ``Resize`` bit for bit
(tests/golden/ref_sampling_golden.npz)."""
import os

import numpy as np
import pytest

from oracle import boxops, imageops, synth
from oracle.model import vgg_weight_shapes
from sampling_cases import TUTORIAL_CLASSES, crop_cases, crop_images, crop_labels, in_keras_order, keras_layer_order_ssd300, sha
from ssd_keras_b200.misc_utils import hdf5_lite as h5
from ssd_keras_b200.misc_utils.tensor_sampling_utils import (SSD300_CLASSIFIER_NAMES, classifier_indices, sample_tensors,
                                                             subsample_classifier_arrays, subsample_classifier_weights)

HERE = os.path.dirname(os.path.abspath(__file__))
EXTRA = ('fc7', {'fc8/kernel': np.arange(160, dtype=np.float32).reshape(1, 1, 16, 10), 'fc8/bias': np.linspace(-1, 1, 10).astype(np.float32)})
HEADS = [s + t for s in ('conv4_3_norm', 'fc7', 'conv6_2', 'conv7_2', 'conv8_2', 'conv9_2') for t in ('_mbox_conf', '_mbox_loc')]


def _names(v):
    return [bytes(n).decode() for n in np.atleast_1d(v)]


@pytest.fixture(scope='module')
def source(tmp_path_factory):
    """A COCO-shaped SSD300 weights file (80 classes + background), in Keras' layer order, with an extra layer and chunked +
    gzip head datasets."""
    w = synth.synth_weights(3, vgg_weight_shapes(300, 80), bias_scale=0.1)
    w['conv4_3_norm/gamma'] = np.full(512, 20.0, np.float32)
    w = in_keras_order(w, EXTRA)
    p = str(tmp_path_factory.mktemp('transfer') / 'VGG_coco_SSD_300x300.h5')
    h5.write_keras_weights(p, w, chunked=[h + '/' + t for h in HEADS for t in ('kernel', 'bias')])
    return p, w


def _tutorial_loop(weights, seed, classes):
    np.random.seed(seed)
    out = {}
    for name in SSD300_CLASSIFIER_NAMES:
        k, b = weights[name + '/kernel'], weights[name + '/bias']
        out[name + '/kernel'], out[name + '/bias'] = sample_tensors([k, b], [k.shape[0], k.shape[1], k.shape[2],
                                                                             classifier_indices(k.shape[3], 81, classes)],
                                                                    axes=[[3]], init=['gaussian', 'zeros'], mean=0.0, stddev=0.005)
    return out, np.random.get_state()


@pytest.mark.parametrize('classes', [TUTORIAL_CLASSES, 9, 100], ids=['list', 'int', 'int_up'])
def test_subsample_classifier_weights_file(source, tmp_path, classes):
    src, w = source
    dst = str(tmp_path / 'subsampled.h5')
    np.random.seed(11)
    subsample_classifier_weights(src, dst, SSD300_CLASSIFIER_NAMES, 81, classes)
    state = np.random.get_state()
    expect, expect_state = _tutorial_loop(w, 11, classes)
    assert state[2:] == expect_state[2:] and np.array_equal(state[1], expect_state[1])

    a, b = h5.read_keras_file(src), h5.read_keras_file(dst)
    assert [l for l, _, _ in b.layers] == [l for l, _, _ in a.layers] == _names(b.attrs['layer_names'])
    assert _names(b.attrs['layer_names']) == keras_layer_order_ssd300()[:15] + ['fc8'] + keras_layer_order_ssd300()[15:]
    assert set(b.attrs) == set(a.attrs) == {'layer_names', 'backend', 'keras_version'}
    for k in a.attrs:
        assert b.attrs[k].tobytes() == a.attrs[k].tobytes(), k
    for (layer, ga, ia), (_, gb, ib) in zip(a.layers, b.layers):
        assert _names(gb['weight_names']) == _names(ga['weight_names']) == [n for n, _ in ib], layer
    got = h5.read_keras_weights(dst)
    assert list(got) == list(w)
    for k, v in w.items():
        if k in expect:
            assert got[k].dtype == expect[k].dtype and got[k].tobytes() == expect[k].tobytes(), k
        else:
            assert got[k].dtype == v.dtype and got[k].tobytes() == v.tobytes(), k           # trunk, box heads, the extra layer
    n_cls = 9 if classes != 100 else 100
    assert got['conv4_3_norm_mbox_conf/kernel'].shape == (3, 3, 512, 4 * n_cls)
    assert got['fc7_mbox_conf/bias'].dtype == (np.float32 if classes != 100 else np.float64)


def test_positional_read_maps_every_tensor_to_its_layer(source, tmp_path):
    """Keras' ``load_weights(by_name=False)`` walks ``layer_names`` and hands layer k the arrays of its ``weight_names``.  The
    dict the package reads has to list the layers in that order too: read -> modify -> write must not reorder them."""
    src, w = source
    dst = str(tmp_path / 'rewritten.h5')
    r = h5.read_keras_weights(src)
    h5.write_keras_weights(dst, subsample_classifier_arrays(r, SSD300_CLASSIFIER_NAMES, 81, TUTORIAL_CLASSES))
    for path in (src, dst):
        got = h5.read_keras_weights(path)
        positional = []
        for k in got:
            if not positional or positional[-1][0] != k.split('/')[0]:
                positional.append((k.split('/')[0], []))
            positional[-1][1].append(got[k])
        expected = [l for l in keras_layer_order_ssd300()]
        expected.insert(expected.index('fc7') + 1, 'fc8')
        assert [l for l, _ in positional] == expected, path
        for layer, arrays in positional:
            names = [k for k in w if k.split('/')[0] == layer]
            assert len(arrays) == len(names)
            for k, a in zip(names, arrays):
                if not k.startswith(tuple(SSD300_CLASSIFIER_NAMES)):
                    assert a.tobytes() == w[k].tobytes(), (path, k)


def test_in_memory_variant_equals_file_helper(source, tmp_path):
    src, w = source
    dst = str(tmp_path / 'd.h5')
    np.random.seed(5)
    subsample_classifier_weights(src, dst, SSD300_CLASSIFIER_NAMES, 81, 9)
    np.random.seed(5)
    mem = subsample_classifier_arrays(w, SSD300_CLASSIFIER_NAMES, 81, 9)
    got = h5.read_keras_weights(dst)
    assert list(mem) == list(got)
    for k in mem:
        assert mem[k].tobytes() == got[k].tobytes(), k
    for k in w:
        if not k.startswith(tuple(SSD300_CLASSIFIER_NAMES)):
            assert mem[k] is w[k]


def test_transferred_weights_load_into_an_8_class_model(source, tmp_path):
    """Host side only: the 8-class SSD300 takes the file (by name; the extra layer is skipped) and the dict; up-sampled float64
    heads are cast to float32 as every other weight."""
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    src, w = source
    dst = str(tmp_path / 'd.h5')
    subsample_classifier_weights(src, dst, SSD300_CLASSIFIER_NAMES, 81, TUTORIAL_CLASSES)
    m = ssd_300((300, 300, 3), 8, mode='inference', scales=[0.07, 0.15, 0.33, 0.51, 0.69, 0.87, 1.05])
    m.load_weights(dst, by_name=True)
    got = h5.read_keras_weights(dst)
    for k, v in m.get_weights().items():
        np.testing.assert_array_equal(v, got[k])
    big = str(tmp_path / 'up.h5')
    subsample_classifier_weights(dst, big, SSD300_CLASSIFIER_NAMES, 9, 12)
    assert h5.read_keras_weights(big)['conv9_2_mbox_conf/kernel'].dtype == np.float64
    m11 = ssd_300((300, 300, 3), 11, mode='training', scales=[0.07, 0.15, 0.33, 0.51, 0.69, 0.87, 1.05])
    m11.load_weights(big, by_name=True)
    assert m11.get_weights()['conv9_2_mbox_conf/kernel'].dtype == np.float32


def test_full_model_file_drops_training_state(tmp_path):
    w = {'conv1/kernel': np.ones((3, 3, 3, 4), np.float32), 'conv1/bias': np.zeros(4, np.float32),
         'head_mbox_conf/kernel': np.arange(3 * 3 * 4 * 6, dtype=np.float32).reshape(3, 3, 4, 6), 'head_mbox_conf/bias': np.arange(6, dtype=np.float32)}
    src = str(tmp_path / 'full.h5')
    h5.write_keras_weights(src, w, full_model=True, root_attrs={'model_config': b'{"class_name": "Model"}', 'training_config': b'{}'},
                           optimizer_weights=[('iterations:0', np.array(7, np.int64)), ('Adam/m/conv1:0', np.ones(4, np.float32))])
    kf = h5.read_keras_file(src)
    assert kf.full_model and [n for n, _ in kf.optimizer_weights] == ['iterations:0', 'Adam/m/conv1:0']
    same = str(tmp_path / 'same.h5')
    h5.write_keras_file(same, kf)
    again = h5.read_keras_file(same)
    assert set(again.root_attrs) == set(kf.root_attrs) and len(again.optimizer_weights) == 2
    dst = str(tmp_path / 'sub.h5')
    subsample_classifier_weights(src, dst, ['head_mbox_conf'], 3, [0, 2])
    out = h5.read_keras_file(dst)
    assert out.full_model and out.optimizer_weights == [] and '/optimizer_weights' not in ''.join(h5.read_datasets(dst))
    assert 'training_config' not in out.root_attrs and out.root_attrs['model_config'].tobytes() == kf.root_attrs['model_config'].tobytes()
    np.testing.assert_array_equal(h5.read_keras_weights(dst)['head_mbox_conf/bias'], [0, 2, 3, 5])
    with pytest.raises(ValueError, match='include_optimizer=False'):
        h5.write_keras_file(str(tmp_path / 'x.h5'), kf, replace={'head_mbox_conf/bias': np.zeros(4, np.float32)}, include_optimizer=True)
    with pytest.raises(ValueError, match='no such weights'):
        h5.write_keras_file(str(tmp_path / 'x.h5'), kf, replace={'nope/kernel': np.zeros(1, np.float32)})


def test_layers_without_weights_and_unlisted_datasets_survive(tmp_path):
    """Keras lists weightless layers (input, pooling) in ``layer_names`` with empty ``weight_names``; a rewrite keeps them, any
    other attribute of a layer group, and a dataset no ``weight_names`` lists."""
    layers = [('input_1', {'weight_names': np.zeros((0,), np.float64)}, []),
              ('conv_b', {'weight_names': np.array([b'conv_b/kernel:0', b'conv_b/bias:0']), 'note': np.array(b'x')},
               [('conv_b/kernel:0', np.full((1, 1, 2, 2), 2.0, np.float32)), ('conv_b/bias:0', np.ones(2, np.float32)),
                ('conv_b/unlisted:0', np.zeros(3, np.float16))]),
              ('conv_a', {'weight_names': np.array([b'conv_a/bias:0', b'conv_a/kernel:0'])},
               [('conv_a/bias:0', np.ones(2, np.float64)), ('conv_a/kernel:0', np.zeros((1, 1, 2, 2), np.float32))])]
    attrs = {'layer_names': np.array([b'input_1', b'conv_b', b'conv_a']), 'backend': np.array(b'tensorflow'), 'keras_version': np.array(b'2.1.4')}
    p = str(tmp_path / 'w.h5')
    h5.write_keras_file(p, h5.KerasFile(layers, attrs))
    kf = h5.read_keras_file(p)
    assert not kf.full_model and [l for l, _, _ in kf.layers] == ['input_1', 'conv_b', 'conv_a']
    for (l0, g0, i0), (l1, g1, i1) in zip(layers, kf.layers):
        assert set(g1) == set(g0) and all(g1[k].tobytes() == g0[k].tobytes() and g1[k].dtype == g0[k].dtype for k in g0), l0
        assert [n for n, _ in i1] == [n for n, _ in i0], l0
        assert all(a.dtype == b.dtype and a.tobytes() == b.tobytes() for (_, a), (_, b) in zip(i0, i1)), l0
    assert list(h5.read_keras_weights(p)) == ['conv_b/kernel', 'conv_b/bias', 'conv_b/unlisted', 'conv_a/bias', 'conv_a/kernel']


def test_big_endian_datasets_are_rewritten_little_endian(tmp_path):
    p = str(tmp_path / 'be.h5')
    be = np.arange(6, dtype='>f4').reshape(2, 3)
    h5.write_keras_weights(p, {'a/kernel': be})
    got = h5.read_keras_weights(p)['a/kernel']
    np.testing.assert_array_equal(got, be)


# ---- the tutorial's sample chain: ConvertTo3Channels -> RandomMaxCropFixedAR -> Resize ------------------------------------

@pytest.fixture(scope='module')
def g():
    with np.load(os.path.join(HERE, 'golden', 'ref_sampling_golden.npz')) as z:
        return {k: z[k] for k in z.files if k.startswith('crop/')}


def test_max_crop_draws_equal_reference(g):
    from ssd_keras_b200.eval_utils.dataset_predict import max_crop_patch
    images = crop_images()
    assert [sha(im) for im in images] == list(g['crop/image_sha'])
    for k, ((shape, ar, _, _), im) in enumerate(zip(crop_cases(), images)):
        np.random.seed(100 + k)
        assert max_crop_patch(im.shape[0], im.shape[1], ar) == tuple(int(v) for v in g['crop/patches'][k]), k
        assert np.random.randint(0, 2 ** 31 - 1) == int(g['crop/next_draw'][k]), k
        rs = np.random.RandomState(100 + k)
        assert max_crop_patch(im.shape[0], im.shape[1], ar, rs) == tuple(int(v) for v in g['crop/patches'][k]), k


def test_max_crop_ops_image_and_boxes_equal_reference_crop_and_resize(g):
    """The op lists assemble_images_device / assemble_batch_device run, through their oracles (oracle/imageops.py,
    oracle/boxops.py): the reference chain's image and boxes, bit for bit."""
    from ssd_keras_b200.data_generator import batch_assembly as ba
    from ssd_keras_b200.eval_utils.dataset_predict import max_crop_ops
    for k, ((shape, ar, oh, ow), im, lab) in enumerate(zip(crop_cases(), crop_images(), crop_labels())):
        np.random.seed(100 + k)
        ops = max_crop_ops(im.shape[0], im.shape[1], ar)
        ph, pw = int(ops[0][4]), int(ops[0][5])
        ops = ops + ba.resize_ops(ph, pw, oh, ow)
        ref = g['crop/out/%d' % k]
        got = imageops.apply_ops(im, ops)
        assert got.shape == ref.shape == (oh, ow, 3), k
        np.testing.assert_array_equal(got, ref, err_msg='case %d' % k)
        np.testing.assert_array_equal(boxops.apply_box_ops(lab, ops), g['crop/labels/%d' % k], err_msg='case %d' % k)


def test_max_crop_ops_with_retries_is_not_supported():
    from ssd_keras_b200.eval_utils.dataset_predict import max_crop_ops
    with pytest.raises(NotImplementedError):
        max_crop_ops(40, 60, 1.0, box_filter={'overlap_criterion': 'area'})
    with pytest.raises(NotImplementedError):
        max_crop_ops(40, 60, 1.0, image_validator=object())
