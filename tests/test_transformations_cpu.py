"""The transformation classes added as planners (``Flip``, ``Translate``, ``Scale``, ``Rotate``, ``CropPad``, ``Crop``, ``Pad``,
``RandomPatchInf``, ``RandomMaxCropFixedAR``, ``RandomPadFixedAR``, ``ConvertColor``, ``ConvertDataType``, ``Brightness``,
``Contrast``, ``Saturation``, ``Hue``, ``ChannelSwap``, ``RandomChannelSwap``, ``HistogramEqualization``,
``RandomHistogramEqualization``) against the real reference (tests/golden/make_transformations_golden.py): each one alone and
custom chains through ``generate``'s host half, run through the oracle's ops, reproduce the reference's images, boxes and
``np.random`` state bit for bit.  Also ``cv2.equalizeHist`` against its NumPy restatement (tests/equalize_reference.py), the
constructors' errors and the refusals."""
import os
import sys

import numpy as np
import pytest

import chain_dataset as ds
import equalize_reference as er
import transformations_cases as tc
from ssd_keras_b200 import _ffi
from ssd_keras_b200.data_generator import batch_assembly as ba
from ssd_keras_b200.data_generator import object_detection_2d_geometric_ops as geo
from ssd_keras_b200.data_generator import object_detection_2d_image_boxes_validation_utils as valid
from ssd_keras_b200.data_generator import object_detection_2d_patch_sampling_ops as patch
from ssd_keras_b200.data_generator import object_detection_2d_photometric_ops as photo
from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_transformations_golden.npz')
REFERENCE = os.environ.get('SSD_REFERENCE_ROOT', '/root/reference')


class Modules:
    pass


MINE = Modules()
MINE.geo, MINE.patch, MINE.photo, MINE.valid = geo, patch, photo, valid


def plan_chain(chain, h, w, labels):
    ops = []
    for t in chain:
        o, h, w, labels = t.plan(h, w, labels)
        ops += o
    return ops, h, w, labels


@pytest.mark.parametrize('name', sorted(tc.SINGLES))
def test_each_class_alone_equals_the_reference(name):
    g = np.load(GOLDEN)
    images, labels = ds.variable_dataset('float')
    chain = [photo.ConvertTo3Channels()] + tc.SINGLES[name](MINE)
    np.random.seed(tc.SINGLE_SEED)
    for k in g['single_images'].tolist():
        p = 'single_%s_%d_' % (name, k)
        ops, h, w, host_labels = plan_chain(chain, images[k].shape[0], images[k].shape[1], labels[k].copy())
        x = er.apply_ops(images[k], ops)
        assert x.shape[:2] == (h, w) and np.array_equal(x, g[p + 'x']), p
        y = er.apply_box_ops(labels[k], ops)
        assert np.array_equal(y, g[p + 'labels']), (p, y, g[p + 'labels'])
        if host_labels is not None:                      # what a later validator would read
            assert np.array_equal(host_labels, g[p + 'labels']), p
        assert np.random.get_state()[2] == int(g[p + 'pos']), p
    assert np.array_equal(np.random.get_state()[1], g['single_%s_state' % name]), name


def _drop_degenerate(x, y, files):
    """The reference's ``degenerate_box_handling='remove'`` and the images it empties."""
    keep = [(a, b[(b[:, 3] > b[:, 1]) & (b[:, 4] > b[:, 2])], f) for a, b, f in zip(x, y, files)]
    keep = [t for t in keep if len(t[1])]
    return [t[0] for t in keep], [t[1] for t in keep], [t[2] for t in keep]


def chain_generator(name):
    g = np.load(GOLDEN)
    make, dataset, dtype, seed, n_batches = tc.CHAINS[name]
    images, labels = dataset(dtype)
    assert ds.digest(images, labels) == str(g[name + '_digest'])
    gen = DataGenerator(filenames=['%d' % i for i in range(len(images))], labels=labels)
    gen.images = images
    np.random.seed(seed)
    return g, gen, make(MINE), n_batches


@pytest.mark.parametrize('name', sorted(tc.CHAINS))
def test_custom_chains_reproduce_the_reference_batches(name):
    g, gen, chain, n_batches = chain_generator(name)
    for t in chain:
        t.labels_format = gen.labels_format
    batches = gen.plan_batches(tc.BATCH, True, chain, False)
    equalized = 0
    for k in range(n_batches):
        p = '%s_b%d_' % (name, k)
        b = next(batches)
        x = [er.apply_ops(b['images'][i], o) for i, o in zip(b['keep'], b['ops'])]
        y = [er.apply_box_ops(b['labels'][i], o) for i, o in zip(b['keep'], b['ops'])]
        x, y, files = _drop_degenerate(x, y, [int(b['filenames'][i]) for i in b['keep']])
        assert files == g[p + 'files'].tolist(), p
        assert np.array_equal(np.stack(x), g[p + 'x']), p
        assert [len(a) for a in y] == g[p + 'counts'].tolist(), p
        assert np.array_equal(np.concatenate(y), g[p + 'labels']), p
        state = np.random.get_state()
        assert state[2] == int(g[p + 'pos']) and np.array_equal(state[1], g[p + 'state']), p
        equalized += sum(o[0] == _ffi.BOXOP_EQUALIZE_V for ops in b['ops'] for o in ops)
    assert equalized > 0


def _check_equalize(cv2, a):
    np.testing.assert_array_equal(er.equalize_hist(a), cv2.equalizeHist(a), err_msg=str(a.shape))


def _tie():
    """(n, s) with (float)s * (255.f / n) exactly halfway between two integers in float32, if a search finds one."""
    for n in range(2, 4000):
        scale = np.float32(255.0) / np.float32(n)
        prod = np.arange(1, n + 1, dtype=np.float32) * scale
        hit = np.flatnonzero(prod - np.floor(prod) == np.float32(0.5))
        if len(hit):
            return n, int(hit[0]) + 1
    return None


def test_equalize_hist_equals_cv2():
    cv2 = pytest.importorskip('cv2')
    rng = np.random.default_rng(8)
    for _ in range(600):
        h, w = (int(v) for v in rng.integers(1, 81, 2))
        lo = int(rng.integers(0, 256))
        hi = int(rng.integers(lo, 256))
        _check_equalize(cv2, rng.integers(lo, hi + 1, (h, w)).astype(np.uint8))
    _check_equalize(cv2, np.array([[77]], np.uint8))                                   # one pixel
    _check_equalize(cv2, np.full((13, 9), 200, np.uint8))                             # constant
    _check_equalize(cv2, np.array([[3, 250, 3], [250, 3, 3]], np.uint8))              # two levels
    _check_equalize(cv2, rng.permutation(np.repeat(np.arange(256), 3)).astype(np.uint8).reshape(24, 32))   # every bin
    tie = _tie()
    assert tie is not None
    n, s = tie                                     # value 0 once (i0), s pixels at 1, n - s at 2: lut[1] = rint(s * scale)
    a = np.array([0] + [1] * s + [2] * (n - s), np.uint8).reshape(1, -1)
    _check_equalize(cv2, a)
    prod = np.float32(s) * (np.float32(255.0) / np.float32(n))
    assert prod - np.floor(prod) == 0.5 and er.equalize_hist(a)[0, 1] == np.rint(prod)


def test_equalize_hist_rounds_the_sum_above_2_24_pixels():
    """The int sum goes through float32: past 2^24 it is rounded, which the table shows."""
    cv2 = pytest.importorskip('cv2')
    n = (1 << 24) + 4099
    a = np.zeros(n, np.uint8)
    a[1:] = 1
    a[-4099:] = 2
    a[-3:] = 255
    _check_equalize(cv2, a.reshape(1, -1))


def test_the_record_and_the_planners():
    assert ba.equalize_hist() == (_ffi.BOXOP_EQUALIZE_V, 0, 0.0, 0.0, 0.0, 0.0) and _ffi.BOXOP_EQUALIZE_V == 26
    assert _ffi.BOXOP_EQUALIZE_V in _ffi.PHOTO_OPS
    header = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'include', 'ssdk.h')).read()
    assert 'SSDK_BOXOP_EQUALIZE_V = SSDK_BOXOP_RESIZE_INTERP + 1' in header and _ffi.BOXOP_RESIZE_INTERP + 1 == 26
    assert photo.HistogramEqualization().plan(5, 6, None) == ([ba.equalize_hist()], 5, 6, None)
    assert photo.ConvertColor('HSV', 'HSV').plan(5, 6, None)[0] == []
    assert photo.ConvertColor('HSV', 'RGB').plan(5, 6, None)[0] == [ba.convert_color('HSV', 'RGB')]
    np.random.seed(3)
    draws = [photo.RandomChannelSwap(0.5).plan(4, 4, None)[0] for _ in range(40)]
    np.random.seed(3)
    want = []
    for _ in range(40):
        want.append([ba.channel_swap(((0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0))[np.random.randint(5)])]
                    if np.random.uniform(0, 1) >= 0.5 else [])
    assert draws == want and any(draws) and not all(draws)


def test_constructors_raise_the_reference_errors():
    pcg = patch.PatchCoordinateGenerator()
    cases = [
        (ValueError, lambda: geo.Flip('diagonal')),
        (ValueError, lambda: geo.Translate(0.1, 0.1, box_filter=valid.ImageValidator())),
        (ValueError, lambda: geo.Scale(0)),
        (ValueError, lambda: geo.Scale(-1.0)),
        (ValueError, lambda: geo.Scale(1.2, box_filter=object())),
        (ValueError, lambda: geo.Rotate(45)),
        (ValueError, lambda: patch.CropPad(0, 0, 5, 5, box_filter=valid.ImageValidator())),
        (ValueError, lambda: patch.Crop(1, 1, 1, 1, box_filter=object())),
        (ValueError, lambda: patch.RandomPatchInf(None)),
        (ValueError, lambda: patch.RandomPatchInf(pcg, image_validator=valid.BoxFilter())),
        (ValueError, lambda: patch.RandomMaxCropFixedAR(1.0, image_validator=valid.BoxFilter())),
        (NotImplementedError, lambda: photo.ConvertColor('GRAY', 'RGB')),
        (NotImplementedError, lambda: photo.ConvertColor('RGB', 'LAB')),
        (ValueError, lambda: photo.ConvertDataType('float64')),
        (ValueError, lambda: photo.Contrast(0.0)),
        (ValueError, lambda: photo.Saturation(-0.5)),
        (ValueError, lambda: photo.Hue(181)),
        (ValueError, lambda: photo.Hue(-180.5)),
    ]
    for exc, make in cases:
        with pytest.raises(exc):
            make()


def test_refusals():
    with pytest.raises(NotImplementedError, match='GRAY'):
        photo.ConvertColor('RGB', 'GRAY').plan(4, 4, None)
    with pytest.raises(NotImplementedError, match='BoundGenerator'):
        patch.RandomPatchInf(patch.PatchCoordinateGenerator(), bound_generator=object())
    with pytest.raises(ValueError, match="doesn't overlap"):
        patch.CropPad(9, 0, 4, 4).plan(8, 8, None)
    for planner in (geo.Flip(), geo.Translate(0.1, 0.1), geo.Scale(1.1), geo.Rotate(90), patch.CropPad(0, 0, 2, 2), patch.Crop(0, 0, 0, 0),
                    patch.Pad(1, 1, 1, 1), patch.RandomPatchInf(patch.PatchCoordinateGenerator()), patch.RandomMaxCropFixedAR(1.0),
                    patch.RandomPadFixedAR(1.0), photo.ConvertColor(), photo.ConvertDataType(), photo.Brightness(1), photo.Contrast(1.1),
                    photo.Saturation(1.1), photo.Hue(1), photo.ChannelSwap((0, 2, 1)), photo.RandomChannelSwap(),
                    photo.HistogramEqualization(), photo.RandomHistogramEqualization()):
        with pytest.raises(TypeError, match='generate'):
            planner(np.zeros((4, 4, 3), np.uint8), np.zeros((0, 5)))


def test_a_photometric_op_after_the_geometry_is_refused_when_planned():
    images = [np.zeros((10, 12, 3), np.uint8)] * 2
    gen = DataGenerator(filenames=['0', '1'], labels=[np.array([[1, 1, 1, 8, 8]])] * 2)
    gen.images = images
    chain = [geo.Flip(), photo.ConvertColor('RGB', 'HSV'), photo.HistogramEqualization(), photo.ConvertColor('HSV', 'RGB')]
    with pytest.raises(ValueError, match='ConvertColor.*comes after.*Flip'):
        next(gen.plan_batches(2, False, chain, False))
    next(gen.plan_batches(2, False, chain[1:] + chain[:1], False))


reference = pytest.mark.skipif(not os.path.isdir(os.path.join(REFERENCE, 'data_generator')), reason='the reference tree is not present')


@reference
def test_constructor_errors_match_the_reference_classes():
    pytest.importorskip('cv2')
    sys.path.insert(0, REFERENCE)
    try:
        from data_generator import object_detection_2d_geometric_ops as rg
        from data_generator import object_detection_2d_image_boxes_validation_utils as rv
        from data_generator import object_detection_2d_patch_sampling_ops as rp
        from data_generator import object_detection_2d_photometric_ops as rph
    finally:
        sys.path.remove(REFERENCE)
    cases = [('geo', 'Flip', ('diagonal',)), ('geo', 'Scale', (0,)), ('geo', 'Rotate', (45,)), ('photo', 'ConvertColor', ('GRAY', 'RGB')),
             ('photo', 'ConvertDataType', ('float64',)), ('photo', 'Contrast', (0.0,)), ('photo', 'Saturation', (-1,)), ('photo', 'Hue', (200,)),
             ('patch', 'RandomPatchInf', (None,))]
    theirs = {'geo': rg, 'photo': rph, 'patch': rp}
    ours = {'geo': geo, 'photo': photo, 'patch': patch}
    for mod, cls, args in cases:
        errors = []
        for m in (theirs, ours):
            try:
                getattr(m[mod], cls)(*args)
                errors.append(None)
            except Exception as e:                                                   # noqa: BLE001
                errors.append((type(e), str(e)))
        assert errors[0] == errors[1], (cls, errors)
    for make in (lambda m, v: m.Translate(0.1, 0.1, box_filter=v.ImageValidator()), lambda m, v: m.Scale(1.5, box_filter=v.ImageValidator())):
        errors = []
        for m, v in ((rg, rv), (geo, valid)):
            with pytest.raises(ValueError) as e:
                make(m, v)
            errors.append(str(e.value))
        assert errors[0] == errors[1]
