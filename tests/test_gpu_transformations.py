"""The transformation classes and histogram equalisation on the device: ``DataGenerator.generate`` with custom chains against
the real reference's batches (tests/golden/make_transformations_golden.py), bit for bit in the images, the processed labels and
the generator state, the encoded labels against the oracle encoder; and ``assemble_images_device`` with ``EQUALIZE_V`` against
tests/equalize_reference.py: mixed batches, several equalisations in one list, odd widths, a 1 x 1 image, an image above 2^24
pixels, and the refusals."""
import numpy as np
import pytest

import equalize_reference as er
import transformations_cases as tc
from test_transformations_cpu import chain_generator

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()


@pytest.fixture(scope='module')
def ba():
    from ssd_keras_b200.data_generator import batch_assembly
    return batch_assembly


def _encoder_config(h, w):
    return dict(img_height=h, img_width=w, n_classes=5, predictor_sizes=[(h // 4, w // 4), (h // 8, w // 8), (h // 16, w // 16)],
                scales=[0.1, 0.3, 0.6, 0.9], aspect_ratios_global=[0.5, 1.0, 2.0], two_boxes_for_ar1=True, steps=None, offsets=None,
                clip_boxes=False, variances=[1.0, 1.0, 1.0, 1.0], matching_type='multi', pos_iou_threshold=0.5, neg_iou_limit=0.3,
                normalize_coords=True)


@pytest.mark.parametrize('name', sorted(tc.CHAINS))
def test_generate_equals_the_reference(name):
    from oracle.encoder import OracleEncoder
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    g, gen, chain, n_batches = chain_generator(name)
    h, w = g[name + '_b0_x'].shape[1:3]
    cfg = _encoder_config(h, w)
    it = gen.generate(batch_size=tc.BATCH, shuffle=True, transformations=chain, label_encoder=SSDInputEncoder(**cfg),
                      returns={'processed_images', 'encoded_labels', 'processed_labels', 'filenames'}, keep_images_without_gt=False)
    for k in range(n_batches):
        p = '%s_b%d_' % (name, k)
        x, y_enc, labels, files = next(it)
        assert [int(f) for f in files] == g[p + 'files'].tolist(), p
        assert np.array_equal(x.cpu().numpy(), g[p + 'x'].astype(np.float32)), p
        counts = g[p + 'counts']
        assert [len(a) for a in labels] == counts.tolist(), p
        assert np.array_equal(np.concatenate(labels), g[p + 'labels']), p
        y_ref = OracleEncoder(**cfg)(np.split(g[p + 'labels'], np.cumsum(counts)[:-1])).astype(np.float32)
        y = y_enc.cpu().numpy()
        np.testing.assert_array_equal(y[:, :, :6] > 0.5, y_ref[:, :, :6] > 0.5)
        np.testing.assert_allclose(y, y_ref, rtol=1e-6, atol=1e-6)
        state = np.random.get_state()
        assert state[2] == int(g[p + 'pos']) and np.array_equal(state[1], g[p + 'state']), p


def _assemble(images, ops, oh, ow):
    from ssd_keras_b200.data_generator.batch_assembly import assemble_images_device
    return assemble_images_device(images, ops, oh, ow)


def _check(images, ops, oh, ow):
    got = _assemble(images, ops, oh, ow).cpu().numpy()
    for b, (im, o) in enumerate(zip(images, ops)):
        want = er.apply_ops(im, o).astype(np.float32)
        bad = np.argwhere(got[b] != want)
        assert len(bad) == 0, (b, len(bad), bad[:5].tolist(), o)


def _image(rng, h, w, c, lo=0, hi=256):
    return rng.integers(lo, hi, (h, w) if c == 0 else (h, w, c), dtype=np.uint8)


def test_mixed_batches_with_and_without_equalisation(ba):
    """Odd widths put the kernels' 4-pixel groups across rows and images; gray, RGBA and narrow value ranges; one image with
    equalisation and no other photometric op, one with photometric ops but none, one with no photometric op at all."""
    rng = np.random.default_rng(1)
    eq, hsv, rgb = ba.equalize_hist(), ba.convert_color('RGB', 'HSV'), ba.convert_color('HSV', 'RGB')
    f32, u8 = ba.convert_dtype('float32'), ba.convert_dtype('uint8')
    shapes = [(37, 53, 3), (41, 29, 0), (33, 67, 4), (45, 31, 1), (39, 47, 3), (35, 61, 3), (43, 57, 3)]
    photos = [[hsv, eq, rgb], [], [eq], [f32, ba.brightness(12.0), u8, hsv, eq, f32, ba.hue(5.0), u8, rgb],
              [hsv, f32, ba.saturation(1.2), u8, rgb], [ba.channel_swap((2, 1, 0)), eq], [hsv, eq, rgb]]
    images, ops = [], []
    for (h, w, c), ph in zip(shapes, photos):
        lo = int(rng.integers(0, 120))
        images.append(_image(rng, h, w, c, lo, lo + int(rng.integers(1, 136))))
        ops.append(ph + ([ba.flip(w)] if rng.random() < 0.5 else []) + [ba.resize(h, w, 30, 35)])
    _check(images, ops, 30, 35)
    _check(images[1:2], ops[1:2], 30, 35)                         # no photometric op at all


@pytest.mark.parametrize('n_eq', [2, 4])
def test_several_equalisations_in_one_list(ba, n_eq):
    rng = np.random.default_rng(n_eq)
    eq, hsv, rgb = ba.equalize_hist(), ba.convert_color('RGB', 'HSV'), ba.convert_color('HSV', 'RGB')
    f32, u8 = ba.convert_dtype('float32'), ba.convert_dtype('uint8')
    between = [[f32, ba.contrast(1.4), u8], [rgb, ba.channel_swap((1, 2, 0)), hsv], [], [f32, ba.brightness(-30.0), u8]]
    full = [hsv]
    for k in range(n_eq):
        full += [eq] + between[k]
    full.append(rgb)
    images = [_image(rng, 23, 19, 3, 40, 90), _image(rng, 17, 31, 0), _image(rng, 29, 13, 3)]
    ops = [full, [hsv, eq, rgb], full[:5] + [rgb]]                # images with different numbers of passes
    for im, o in zip(images, ops):
        _check([im], [o], im.shape[0], im.shape[1])
    same = [_image(rng, 21, 27, 3) for _ in range(3)]
    _check(same, ops, 21, 27)


def test_refusals_leave_the_output_alone(ba):
    import torch
    from ssd_keras_b200.data_generator.batch_assembly import assemble_images_device
    img = np.zeros((8, 9, 3), np.uint8)
    eq = ba.equalize_hist()
    out = torch.full((1, 8, 9, 3), -1.0, device='cuda')
    for ops, match in (([eq] * 5, 'more than 4 EQUALIZE_V'),
                       ([ba.convert_dtype('float32'), eq, ba.convert_dtype('uint8')], 'EQUALIZE_V needs a uint8 image'),
                       ([ba.flip(9), eq], 'photometric ops must come before')):
        with pytest.raises(ValueError, match=match):
            assemble_images_device([img], [ops], 8, 9, out=out)
        assert bool((out == -1).all())
    _check([img], [[eq] * 4], 8, 9)


def test_one_pixel_and_constant_images(ba):
    eq = ba.equalize_hist()
    _check([np.array([[[10, 20, 30]]], np.uint8)], [[eq]], 1, 1)
    _check([np.full((5, 7, 3), 77, np.uint8), np.array([[[0, 0, 5], [0, 0, 250]]], np.uint8)], [[eq], [eq, ba.resize(1, 2, 5, 7)]], 5, 7)


def test_an_image_above_2_24_pixels(ba):
    """The sums past 2^24 are rounded to float32 before the product, as cv2 does; 4099 x 4099 one-channel pixels."""
    rng = np.random.default_rng(9)
    n = 4099
    img = np.minimum(rng.geometric(0.02, (n, n)), 255).astype(np.uint8)
    assert img.size > 1 << 24
    got = _assemble([img], [[ba.equalize_hist()]], n, n)[0, :, :, 2].to(dtype=__import__('torch').uint8).cpu().numpy()
    assert np.array_equal(got, er.equalize_hist(img))
