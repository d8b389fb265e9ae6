"""The device half of DataGenerator.generate: ``resize_interp`` in every cv2 mode bit for bit with tests/resize_reference.py
(alone, and after crops, pads, flips and the photometric pre-pass), generate() against the real reference's batches
(tests/golden/make_ssd_augmentation_golden.py), its encoded labels against the oracle encoder, the degenerate-box rules, a
refused op list, and fit_generator on an SSD300 fed by generate()."""
import os
import warnings

import numpy as np
import pytest

import augmentation_dataset as ds
import resize_reference as rr
from test_resize_interp_cpu import size_pairs

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_ssd_augmentation_golden.npz')
MODES = {0: 'nearest', 1: 'linear', 2: 'cubic', 3: 'area', 4: 'lanczos4'}


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()


@pytest.fixture(scope='module')
def ba():
    from ssd_keras_b200.data_generator import batch_assembly
    return batch_assembly


def _pre_ops(ba, rng, h, w):
    """Photometric ops, a pad, a crop and flips that end on an h x w canvas: -> (ops, canvas size before them)."""
    ph, pw = h + int(rng.integers(0, 5)), w + int(rng.integers(0, 5))
    ops = ba.photometric_ops(1, brightness=12.5, contrast=1.25, saturation=0.75, hue=-9.0)
    ops += [ba.crop_pad(-2, -3, ph, pw, background=(123, 117, 104)), ba.flip(pw, 'horizontal'),
            ba.crop_pad(ph - h, pw - w, h, w), ba.flip(h, 'vertical')]
    return ops, (ph - 2, pw - 3)


@pytest.mark.parametrize('mode', sorted(MODES), ids=[MODES[m] for m in sorted(MODES)])
def test_resize_interp_equals_reference(ba, mode):
    rng = np.random.default_rng(40 + mode)
    for h, w, oh, ow in size_pairs(mode, 150):
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        pre, (sh, sw) = _pre_ops(ba, rng, h, w)
        src = rng.integers(0, 256, (max(sh, 1), max(sw, 1), 4), dtype=np.uint8)
        lists = [[ba.resize_interp(h, w, oh, ow, mode)], pre + [ba.resize_interp(h, w, oh, ow, mode)]]
        x = ba.assemble_images_device([img, src], lists, oh, ow).cpu().numpy()
        for got, im, ops in zip(x, (img, src), lists):
            want = rr.apply_ops(im, ops)
            assert np.array_equal(got, want.astype(np.float32)), (MODES[mode], h, w, oh, ow, ops is lists[1])


def test_mixed_modes_in_one_batch(ba):
    """One launch, every mode and a plain crop, each image as its own list says."""
    rng = np.random.default_rng(9)
    images = [rng.integers(0, 256, (int(rng.integers(20, 90)), int(rng.integers(20, 90)), 3), dtype=np.uint8) for _ in range(7)]
    lists = [[ba.resize_interp(im.shape[0], im.shape[1], 48, 64, m % 5)] for m, im in enumerate(images[:6])]
    lists.append([ba.crop_pad(0, 0, 48, 64)])
    x = ba.assemble_images_device(images, lists, 48, 64).cpu().numpy()
    for got, im, ops in zip(x, images, lists):
        assert np.array_equal(got, rr.apply_ops(im, ops).astype(np.float32))


def test_resize_keeps_its_refusals_and_bad_lists_leave_out_untouched(ba):
    import torch
    img = np.zeros((10, 12, 3), np.uint8)
    out = torch.full((1, 5, 6, 3), -7.0, device='cuda')
    for ops in ([ba.resize(10, 12, 5, 6, interpolation_mode=2)], [ba.resize(10, 12, 5, 6, interpolation_mode=3)],
                [ba.resize_interp(10, 12, 5, 6, 2), ba.flip(6)], [ba.resize_interp(10, 11, 5, 6, 4)],
                [(25, 5 << 8, 10.0, 12.0, 5.0, 6.0)]):
        with pytest.raises(Exception):
            ba.assemble_images_device([img], [ops], 5, 6, out=out)
        torch.cuda.synchronize()
        assert bool((out == -7.0).all())


def test_box_half_is_resize(ba):
    from oracle import boxops as bo
    labels = [np.array([[1, 0, 0, 7, 9], [2, 3, 4, 4, 5], [3, 10, 2, 12, 10]], np.float64)]
    for drop in (True, False):
        gt, offs = ba.assemble_batch_device(labels, [[ba.resize_interp(10, 12, 7, 5, 3, drop_degenerate=drop)]])[:2]
        want = bo.apply_box_ops(labels[0], [ba.resize(10, 12, 7, 5, drop_degenerate=drop)])
        assert np.array_equal(gt.cpu().numpy()[:offs[-1].item()], want.astype(np.float32))


def _golden_generator():
    from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator
    g = np.load(GOLDEN)
    images, labels = ds.dataset()
    assert len(images) == int(g['n_images']) and ds.digest(images) == str(g['digest'])
    gen = DataGenerator(filenames=['%d' % i for i in range(len(images))], labels=labels)
    gen.images = images
    return g, gen


def _encoder_config(h, w):
    return dict(img_height=h, img_width=w, n_classes=20, predictor_sizes=[(15, 19), (8, 10), (4, 5), (2, 3)],
                scales=[0.1, 0.3, 0.5, 0.7, 0.9], aspect_ratios_global=[0.5, 1.0, 2.0], two_boxes_for_ar1=True, steps=None,
                offsets=None, clip_boxes=False, variances=[0.1, 0.1, 0.2, 0.2], matching_type='multi', pos_iou_threshold=0.5,
                neg_iou_limit=0.4, normalize_coords=True)


def test_generate_equals_the_reference():
    from oracle.encoder import OracleEncoder
    from ssd_keras_b200.data_generator.data_augmentation_chain_original_ssd import SSDDataAugmentation
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    g, gen = _golden_generator()
    h, w = (int(v) for v in g['out_hw'])
    cfg = _encoder_config(h, w)
    np.random.seed(int(g['seed']))
    it = gen.generate(batch_size=int(g['batch_size']), shuffle=True, transformations=[SSDDataAugmentation(h, w)],
                      label_encoder=SSDInputEncoder(**cfg), returns={'processed_images', 'encoded_labels', 'processed_labels', 'filenames'},
                      keep_images_without_gt=False)
    for k in range(int(g['n_batches'])):
        x, y_enc, labels, files = next(it)
        assert [int(f) for f in files] == g['b%d_files' % k].tolist()
        assert x.is_cuda and x.dtype.is_floating_point and y_enc.is_cuda
        assert np.array_equal(x.cpu().numpy(), g['b%d_x' % k].astype(np.float32)), k
        counts = g['b%d_counts' % k]
        assert [len(a) for a in labels] == counts.tolist()
        assert np.array_equal(np.concatenate(labels), g['b%d_labels' % k]), k
        ref = np.split(g['b%d_labels' % k], np.cumsum(counts)[:-1])
        y_ref = OracleEncoder(**cfg)(ref).astype(np.float32)
        y = y_enc.cpu().numpy()
        np.testing.assert_array_equal(y[:, :, :21] > 0.5, y_ref[:, :, :21] > 0.5)
        np.testing.assert_allclose(y, y_ref, rtol=1e-6, atol=1e-6)
        state = np.random.get_state()
        assert state[2] == int(g['b%d_pos' % k]) and np.array_equal(state[1], g['b%d_state' % k]), k


def test_degenerate_boxes_remove_and_warn():
    """Without a chain the processed boxes are the dataset's: 'remove' drops the degenerate ones and the images it empties,
    'warn' keeps them and warns."""
    from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator
    images = [np.full((8, 9, 3), i, np.uint8) for i in range(3)]
    labels = [np.array([[1, 2, 2, 2, 5]], np.float64), np.array([[1, 0, 0, 4, 4], [2, 3, 3, 3, 6]], np.float64),
              np.array([[1, 1, 1, 5, 5]], np.float64)]
    gen = DataGenerator(filenames=['a', 'b', 'c'], labels=labels)
    gen.images = images
    x, y, names = next(gen.generate(batch_size=3, shuffle=False, returns={'processed_images', 'processed_labels', 'filenames'}))
    assert names == ['b', 'c'] and tuple(x.shape) == (2, 8, 9, 3)
    assert [a.tolist() for a in y] == [[[1, 0, 0, 4, 4]], [[1, 1, 1, 5, 5]]]
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter('always')
        x, y, names = next(gen.generate(batch_size=3, shuffle=False, returns={'processed_images', 'processed_labels', 'filenames'},
                                        degenerate_box_handling='warn'))
    assert names == ['a', 'b', 'c'] and [len(a) for a in y] == [1, 2, 1]
    assert sum('degenerate' in str(r.message) for r in rec) == 2


def test_generate_from_image_files(tmp_path):
    """Files decoded with PIL on the thread pool give what the same arrays in memory give."""
    from PIL import Image
    from ssd_keras_b200.data_generator.data_augmentation_chain_original_ssd import SSDDataAugmentation
    from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator
    g, mem = _golden_generator()
    names = []
    for i, im in enumerate(mem.images):
        names.append(str(tmp_path / ('%d.png' % i)))
        Image.fromarray(im[:, :, 0] if im.ndim == 3 and im.shape[2] == 1 else im).save(names[-1])
    files = DataGenerator(filenames=names, labels=[l.copy() for l in mem.labels])
    outs = []
    for gen in (mem, files):
        np.random.seed(3)
        it = gen.generate(batch_size=4, transformations=[SSDDataAugmentation(60, 80)], returns={'processed_images'})
        outs.append([next(it)[0].cpu().numpy() for _ in range(4)])
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


def test_fit_generator_on_ssd300():
    from oracle import synth
    from oracle.model import SSD300_AR, vgg_weight_shapes
    from ssd_keras_b200.data_generator.data_augmentation_chain_original_ssd import SSDDataAugmentation
    from ssd_keras_b200.keras_loss_function.keras_ssd_loss import SSDLoss
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    from ssd_keras_b200.optimizers import SGD
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    g, gen = _golden_generator()
    scales = [0.1, 0.2, 0.37, 0.54, 0.71, 0.88, 1.05]
    model = ssd_300((300, 300, 3), 20, mode='training', scales=scales, subtract_mean=[123, 117, 104], swap_channels=[2, 1, 0])
    model.set_weights(synth.synth_weights(0, vgg_weight_shapes(300, 20), bias_scale=0.02))
    model.compile(optimizer=SGD(lr=1e-4, momentum=0.9), loss=SSDLoss(neg_pos_ratio=3, alpha=1.0).compute_loss)
    encoder = SSDInputEncoder(img_height=300, img_width=300, n_classes=20, predictor_sizes=model.predictor_sizes, scales=scales,
                              aspect_ratios_per_layer=SSD300_AR, two_boxes_for_ar1=True, steps=[8, 16, 32, 64, 100, 300],
                              offsets=[0.5] * 6, clip_boxes=False, variances=[0.1, 0.1, 0.2, 0.2], matching_type='multi',
                              pos_iou_threshold=0.5, neg_iou_limit=0.5, normalize_coords=True)
    np.random.seed(1)
    batches = gen.generate(batch_size=2, shuffle=True, transformations=[SSDDataAugmentation(300, 300)], label_encoder=encoder,
                           returns={'processed_images', 'encoded_labels'}, keep_images_without_gt=False)
    h = model.fit_generator(generator=batches, steps_per_epoch=2, epochs=1)
    assert len(h.history['loss']) == 1 and all(np.isfinite(v) for v in h.history['loss'])
