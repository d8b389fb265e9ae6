"""The SSD7, variable-input-size and satellite chains' planners and ``parse_csv`` against the real reference
(tests/golden/make_augmentation_chains_golden.py): the shuffle, the batch slices, the images dropped for having no boxes and
every draw of the chains, run through the oracle's image and box ops, reproduce the reference's batches bit for bit and leave
both ``np.random`` and Python's ``random`` where the reference left them.  Also the constructors' errors, the refusals, and a
seeded fuzz of the host box tracking against the reference's classes where its tree exists."""
import os
import random
import sys

import numpy as np
import pytest

import chain_dataset as ds
import resize_reference as rr
from ssd_keras_b200 import _ffi
from ssd_keras_b200.data_generator import batch_assembly as ba
from ssd_keras_b200.data_generator.data_augmentation_chain_constant_input_size import DataAugmentationConstantInputSize
from ssd_keras_b200.data_generator.data_augmentation_chain_satellite import DataAugmentationSatellite
from ssd_keras_b200.data_generator.data_augmentation_chain_variable_input_size import DataAugmentationVariableInputSize
from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator
from ssd_keras_b200.data_generator.object_detection_2d_geometric_ops import RandomRotate, RandomScale, RandomTranslate
from ssd_keras_b200.data_generator.object_detection_2d_image_boxes_validation_utils import BoxFilter, ImageValidator
from ssd_keras_b200.data_generator.object_detection_2d_patch_sampling_ops import PatchCoordinateGenerator, RandomPatch
from ssd_keras_b200.data_generator.object_detection_2d_photometric_ops import (RandomBrightness, RandomContrast, RandomHue,
                                                                               RandomSaturation)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_augmentation_chains_golden.npz')
REFERENCE = os.environ.get('SSD_REFERENCE_ROOT', '/root/reference')
SSD7_ARGS = dict(random_brightness=(-48, 48, 0.5), random_contrast=(0.5, 1.8, 0.5), random_saturation=(0.5, 1.8, 0.5),
                 random_hue=(18, 0.5), random_flip=0.5, random_translate=((0.03, 0.5), (0.03, 0.5), 0.5), random_scale=(0.5, 2.0, 0.5),
                 n_trials_max=3, clip_boxes=True, overlap_criterion='area', bounds_box_filter=(0.3, 1.0), bounds_validator=(0.5, 1.0),
                 n_boxes_min=1, background=(0, 0, 0))
# name: (dataset, labels dtype, chain, keep_images_without_gt), as in the golden generator
RUNS = {
    'ssd7_int': (ds.ssd7_dataset, 'int', lambda: DataAugmentationConstantInputSize(**SSD7_ARGS), False),
    'ssd7_float': (ds.ssd7_dataset, 'float', lambda: DataAugmentationConstantInputSize(**dict(SSD7_ARGS, background=(123, 117, 104))), True),
    'variable': (ds.variable_dataset, 'int', lambda: DataAugmentationVariableInputSize(48, 64), False),
    'satellite': (ds.variable_dataset, 'float', lambda: DataAugmentationSatellite(48, 64, background=(200, 100, 50)), True),
}


def golden_generator(name):
    g = np.load(GOLDEN)
    dataset, dtype, chain, keep = RUNS[name]
    images, labels = dataset(dtype)
    assert ds.digest(images, labels) == str(g[name + '_digest'])
    gen = DataGenerator(filenames=['%d' % i for i in range(len(images))], labels=labels)
    gen.images = images
    return g, gen, chain, keep


def seed(g, name):
    np.random.seed(int(g[name + '_seed']))
    random.seed(int(g[name + '_seed']))


def assert_states(g, p):
    state = np.random.get_state()
    assert state[2] == int(g[p + 'pos']) and np.array_equal(state[1], g[p + 'state']), p
    assert np.array_equal(np.array(random.getstate()[1], np.int64), g[p + 'pystate']), p


def _features(ops):
    """What an op list exercises: sequence 2 of SSD7, zoom in / out, rotations, pads, vertical flips, translations."""
    f = set()
    codes = [o[0] for o in ops]
    if codes.count(_ffi.BOXOP_TO_FLOAT32) == 3:
        f.add('sequence2')
    for o in ops:
        if o[0] == _ffi.BOXOP_SCALE:
            f.add('zoom_in' if o[2] > 1 else 'zoom_out')
        elif o[0] == _ffi.BOXOP_ROTATE:
            f.add('rotate%d' % o[2])
        elif o[0] == _ffi.BOXOP_CROP_PAD and o[2] < 0 or o[0] == _ffi.BOXOP_CROP_PAD and o[3] < 0:
            f.add('pad')
        elif o[0] == _ffi.BOXOP_FLIP_V:
            f.add('flip_v')
        elif o[0] == _ffi.BOXOP_TRANSLATE:
            f.add('translate')
    return f


WANT = {'ssd7_int': {'sequence2', 'zoom_in', 'zoom_out', 'translate'}, 'ssd7_float': {'sequence2', 'zoom_in', 'zoom_out', 'translate'},
        'variable': {'pad'}, 'satellite': {'rotate90', 'rotate180', 'rotate270', 'pad', 'flip_v'}}


@pytest.mark.parametrize('name', sorted(RUNS))
def test_planners_reproduce_the_reference_batches(name):
    g, gen, chain, keep = golden_generator(name)
    seed(g, name)
    batches = gen.plan_batches(int(g['batch_size']), True, [chain()], keep)
    seen = set()
    for k in range(int(g[name + '_n_batches'])):
        p = '%s_b%d_' % (name, k)
        b = next(batches)
        assert [int(b['filenames'][i]) for i in b['keep']] == g[p + 'files'].tolist(), p
        x = [rr.apply_ops(b['images'][i], o) for i, o in zip(b['keep'], b['ops'])]
        y = [rr.apply_box_ops(b['labels'][i], o) for i, o in zip(b['keep'], b['ops'])]
        assert all(np.all(a[:, 3] > a[:, 1]) and np.all(a[:, 4] > a[:, 2]) for a in y)      # nothing for the degenerate check
        assert tuple(b['out_hw']) == g[p + 'x'].shape[1:3]
        assert np.array_equal(np.stack(x), g[p + 'x']), p
        assert [len(a) for a in y] == g[p + 'counts'].tolist(), p
        assert np.array_equal(np.concatenate(y), g[p + 'labels']), p
        assert_states(g, p)
        for ops in b['ops']:
            seen |= _features(ops)
    assert WANT[name] <= seen, WANT[name] - seen


def test_satellite_pads_black_whatever_the_background():
    np.random.seed(2)
    random.seed(2)
    chain = DataAugmentationSatellite(40, 40, background=(200, 100, 50), min_scale=1.5, max_scale=2.0)
    for _ in range(20):
        ops = chain.plan(30, 50, np.array([[1, 10, 5, 30, 25]]))[0]
        assert all(o[1] >> 8 == 0 for o in ops if o[0] == _ffi.BOXOP_CROP_PAD)


def test_parse_csv_equals_the_reference(tmp_path):
    g = np.load(GOLDEN)
    path = tmp_path / 'labels.csv'
    path.write_text(ds.csv_text())
    gen = DataGenerator()
    np.random.seed(int(g['csv_seed']))
    images, filenames, labels, image_ids = gen.parse_csv('images', str(path), ds.CSV_INPUT_FORMAT, include_classes=ds.CSV_INCLUDE,
                                                         random_sample=ds.CSV_SAMPLE, ret=True, verbose=False)
    assert images is None
    assert [os.path.relpath(f, 'images') for f in filenames] == g['csv_filenames'].tolist()
    assert image_ids == g['csv_image_ids'].tolist()
    assert [len(a) for a in labels] == g['csv_counts'].tolist()
    assert all(a.dtype == np.dtype(str(g['csv_dtype'])) for a in labels)
    assert np.array_equal(np.concatenate(labels), g['csv_labels'])
    state = np.random.get_state()
    assert state[2] == int(g['csv_pos']) and np.array_equal(state[1], g['csv_state'])
    assert gen.get_dataset_size() == len(filenames) and gen.dataset_indices.tolist() == list(range(len(filenames)))


def test_parse_csv_everything_and_into_memory(tmp_path):
    from PIL import Image
    (tmp_path / 'img').mkdir()
    for name, shape in (('b.1.png', (6, 9, 3)), ('a.png', (5, 7))):
        Image.fromarray(np.full(shape, 40, np.uint8)).save(str(tmp_path / 'img' / name))
    (tmp_path / 'l.csv').write_text('frame,xmin,xmax,ymin,ymax,class_id\nb.1.png,1,4,2,5,3\na.png, 0 ,3,1,4,1\nb.1.png,0,2,0,2,1\n')
    gen = DataGenerator(load_images_into_memory=True)
    state = np.random.get_state()[1].copy()
    images, filenames, labels, ids = gen.parse_csv(str(tmp_path / 'img'), str(tmp_path / 'l.csv'),
                                                   ['image_name', 'xmin', 'xmax', 'ymin', 'ymax', 'class_id'], ret=True)
    assert np.array_equal(np.random.get_state()[1], state)                       # no draw without random_sample
    assert ids == ['a', 'b'] and [os.path.basename(f) for f in filenames] == ['a.png', 'b.1.png']
    assert [a.tolist() for a in labels] == [[[1, 0, 1, 3, 4]], [[1, 0, 0, 2, 2], [3, 1, 2, 4, 5]]]
    assert [im.shape for im in images] == [(5, 7), (6, 9, 3)]
    with pytest.raises(ValueError):
        gen.parse_csv(str(tmp_path), None, ['image_name'])


def test_constructors_raise_the_reference_errors():
    pcg = PatchCoordinateGenerator()
    cases = [
        (ValueError, lambda: DataAugmentationConstantInputSize(random_scale=(1.0, 2.0, 0.5))),
        (ValueError, lambda: DataAugmentationConstantInputSize(random_scale=(0.5, 1.0, 0.5))),
        (ValueError, lambda: RandomTranslate(dy_minmax=(0.3, 0.1))),
        (ValueError, lambda: RandomTranslate(dx_minmax=(0.3, 0.1))),
        (ValueError, lambda: RandomTranslate(dy_minmax=(-0.1, 0.1))),
        (ValueError, lambda: RandomTranslate(image_validator=object())),
        (ValueError, lambda: RandomTranslate(box_filter=dict(check_overlap=False))),
        (ValueError, lambda: RandomScale(min_factor=0)),
        (ValueError, lambda: RandomScale(min_factor=2, max_factor=1)),
        (ValueError, lambda: RandomScale(image_validator=BoxFilter())),
        (ValueError, lambda: RandomRotate(angles=[90, 45])),
        (ValueError, lambda: RandomBrightness(10, 10)),
        (ValueError, lambda: RandomContrast(1.5, 0.5)),
        (ValueError, lambda: RandomSaturation(2.0, 2.0)),
        (ValueError, lambda: RandomHue(181)),
        (ValueError, lambda: RandomHue(-1)),
        (ValueError, lambda: PatchCoordinateGenerator(must_match='ar')),
        (ValueError, lambda: PatchCoordinateGenerator(min_scale=1.0, max_scale=1.0)),
        (ValueError, lambda: PatchCoordinateGenerator(min_aspect_ratio=2.0, max_aspect_ratio=1.0)),
        (ValueError, lambda: PatchCoordinateGenerator(scale_uniformly=True, patch_height=10)),
        (ValueError, lambda: RandomPatch(patch_coord_generator=None)),
        (ValueError, lambda: RandomPatch(pcg, image_validator=BoxFilter())),
        (ValueError, lambda: RandomPatch(pcg, box_filter=ImageValidator())),
        (ValueError, lambda: BoxFilter(overlap_bounds=(0.9, 0.1))),
        (ValueError, lambda: BoxFilter(overlap_bounds=0.5)),
        (ValueError, lambda: BoxFilter(overlap_criterion='centre')),
        (ValueError, lambda: ImageValidator(n_boxes_min=0)),
        (ValueError, lambda: ImageValidator(n_boxes_min='some')),
    ]
    for exc, make in cases:
        with pytest.raises(exc):
            make()


def test_unsupported_options_are_refused():
    with pytest.raises(NotImplementedError):
        BoxFilter(overlap_bounds=lambda: (0.1, 1.0))
    never = ImageValidator(overlap_criterion='area', bounds=(1.0, 1.0), n_boxes_min='all')
    patch = RandomPatch(PatchCoordinateGenerator(min_scale=0.2, max_scale=0.3), image_validator=never, can_fail=True)
    np.random.seed(0)
    with pytest.raises(NotImplementedError, match='can_fail'):
        patch.plan(50, 50, np.array([[1, 0, 0, 50, 50]]))
    for chain in (DataAugmentationVariableInputSize(30, 30), DataAugmentationSatellite(30, 30)):
        with pytest.raises(AttributeError, match='sequence1'):
            chain.plan(20, 20, None)
    for planner in (DataAugmentationConstantInputSize(), DataAugmentationVariableInputSize(3, 3), DataAugmentationSatellite(3, 3),
                    RandomTranslate(), RandomScale(), RandomRotate(), RandomPatch(PatchCoordinateGenerator()), RandomHue()):
        with pytest.raises(TypeError, match='generate'):
            planner(np.zeros((4, 4, 3), np.uint8), np.zeros((0, 5)))


def test_box_filter_ops_take_a_box_filter():
    spec = dict(check_overlap=True, check_min_area=True, check_degenerate=False, overlap_criterion='iou', overlap_bounds=(0.2, 0.9),
                min_area=9, border_pixels='include')
    assert ba.box_filter_ops(BoxFilter(**spec), 30, 40) == ba.box_filter_ops(spec, 30, 40)
    assert ba.box_filter_ops(BoxFilter(check_overlap=False, check_min_area=False, check_degenerate=False), 3, 4) == []


def test_the_constant_chain_plans_without_labels():
    np.random.seed(4)
    ops, h, w, labels = DataAugmentationConstantInputSize().plan(60, 96, None)
    assert (h, w, labels) == (60, 96, None) and ops[0][0] == _ffi.BOXOP_TO_FLOAT32


reference = pytest.mark.skipif(not os.path.isdir(os.path.join(REFERENCE, 'data_generator')), reason='the reference tree is not present')


@reference
def test_fuzz_planners_against_the_reference():
    """Each planner and the reference's class, from the same seeds, on random images and int / float labels: the same labels
    after the op (what a later validator reads), the same image size and the same generator states."""
    cv2 = pytest.importorskip('cv2')
    sys.path.insert(0, REFERENCE)
    np.int, np.float = int, float
    try:
        from data_generator import object_detection_2d_geometric_ops as rg
        from data_generator import object_detection_2d_image_boxes_validation_utils as rv
        from data_generator import object_detection_2d_patch_sampling_ops as rp
    finally:
        sys.path.remove(REFERENCE)
    cv2.ipp.setUseIPP(False)
    rng = np.random.default_rng(77)

    def pair(k):
        crit = ['area', 'center_point', 'iou'][k % 3]
        bf = dict(check_overlap=True, check_min_area=k % 2 == 0, check_degenerate=True, overlap_criterion=crit, overlap_bounds=(0.3, 1.0),
                  min_area=16)
        iv = dict(overlap_criterion=crit, bounds=(0.5, 1.0), n_boxes_min=1 + k % 2)
        mine_f, ref_f, mine_v, ref_v = BoxFilter(**bf), rv.BoxFilter(**bf), ImageValidator(**iv), rv.ImageValidator(**iv)
        kw = dict(prob=0.8, clip_boxes=k % 4 != 1, n_trials_max=k % 4)
        if k % 4 == 0:
            return (RandomTranslate(box_filter=mine_f, image_validator=mine_v, **kw),
                    rg.RandomTranslate(box_filter=ref_f, image_validator=ref_v, **kw))
        if k % 4 == 1:
            return (RandomScale(0.4, 1.8, box_filter=mine_f, image_validator=mine_v, **kw),
                    rg.RandomScale(0.4, 1.8, box_filter=ref_f, image_validator=ref_v, **kw))
        if k % 4 == 2:
            return RandomRotate(prob=0.8), rg.RandomRotate(prob=0.8)
        mm = ['h_w', 'h_ar', 'w_ar'][k % 3]
        pg = dict(must_match=mm, min_scale=0.3, max_scale=1.7, scale_uniformly=k % 5 == 0 and mm == 'h_w')
        return (RandomPatch(PatchCoordinateGenerator(**pg), box_filter=mine_f, image_validator=mine_v, **kw),
                rg_patch(rp, pg, ref_f, ref_v, kw))

    for k in range(240):
        h, w = int(rng.integers(8, 60)), int(rng.integers(8, 60))
        n = int(rng.integers(0, 5))
        x0, y0 = rng.integers(-10, w, n), rng.integers(-10, h, n)
        labels = np.stack([rng.integers(1, 4, n), x0, y0, x0 + rng.integers(0, 40, n), y0 + rng.integers(0, 40, n)], axis=1).astype(np.int64)
        if k % 2:
            labels = labels + 0.5 * rng.integers(0, 2, labels.shape)
        mine, ref = pair(k)
        np.random.seed(k)
        random.seed(k)
        _, mh, mw, mlab = mine.plan(h, w, labels)
        ms, mp = np.random.get_state(), random.getstate()
        np.random.seed(k)
        random.seed(k)
        image, rlab = ref(np.zeros((h, w, 3), np.uint8), labels)
        assert (mh, mw) == image.shape[:2], k
        assert mlab.dtype == rlab.dtype and np.array_equal(mlab, rlab), (k, mlab, rlab)
        assert np.array_equal(ms[1], np.random.get_state()[1]) and ms[2] == np.random.get_state()[2] and mp == random.getstate(), k


def rg_patch(rp, pg, ref_f, ref_v, kw):
    return rp.RandomPatch(rp.PatchCoordinateGenerator(**pg), box_filter=ref_f, image_validator=ref_v, **kw)
