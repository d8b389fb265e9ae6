"""DataGenerator's host half against the real reference (tests/golden/make_ssd_augmentation_golden.py): the shuffle, the
batch slices, the images dropped for having no boxes and the draws of SSDDataAugmentation's planners, run through the
oracle's image and box ops (tests/resize_reference.py for the resize modes), reproduce the reference's batches bit for bit and
leave ``np.random`` where the reference left it.  Also the shuffle against sklearn's, and the refusals."""
import os

import numpy as np
import pytest

import augmentation_dataset as ds
import resize_reference as rr
from ssd_keras_b200.data_generator import batch_assembly as ba
from ssd_keras_b200.data_generator.data_augmentation_chain_original_ssd import (SSDDataAugmentation, SSDExpand,
                                                                                SSDPhotometricDistortions, SSDRandomCrop)
from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator, DatasetError, shuffle_together
from ssd_keras_b200.data_generator.object_detection_2d_geometric_ops import RandomFlip, Resize, ResizeRandomInterp
from ssd_keras_b200.data_generator.object_detection_2d_photometric_ops import ConvertTo3Channels

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_ssd_augmentation_golden.npz')


def golden_dataset():
    g = np.load(GOLDEN)
    images, labels = ds.dataset()
    assert len(images) == int(g['n_images']) and ds.digest(images) == str(g['digest'])
    gen = DataGenerator(filenames=['%d' % i for i in range(len(images))], labels=labels)
    gen.images = images
    return g, gen


def test_planners_reproduce_the_reference_batches():
    g, gen = golden_dataset()
    out_h, out_w = (int(v) for v in g['out_hw'])
    np.random.seed(int(g['seed']))
    batches = gen.plan_batches(int(g['batch_size']), True, [SSDDataAugmentation(out_h, out_w)], False)
    modes = set()
    for k in range(int(g['n_batches'])):
        b = next(batches)
        assert [int(b['filenames'][i]) for i in b['keep']] == g['b%d_files' % k].tolist(), k
        assert b['out_hw'] == (out_h, out_w)
        x = [rr.apply_ops(b['images'][i], o) for i, o in zip(b['keep'], b['ops'])]
        y = [rr.apply_box_ops(b['labels'][i], o) for i, o in zip(b['keep'], b['ops'])]
        assert np.array_equal(np.stack(x), g['b%d_x' % k]), k
        assert [len(a) for a in y] == g['b%d_counts' % k].tolist(), k
        assert np.array_equal(np.concatenate(y), g['b%d_labels' % k]), k
        state = np.random.get_state()
        assert state[2] == int(g['b%d_pos' % k]) and np.array_equal(state[1], g['b%d_state' % k]), k
        modes |= {(o[1] >> 8) & 255 for ops in b['ops'] for o in ops if o[0] == rr.OP_RESIZE_INTERP}
    assert modes == {0, 1, 2, 3, 4}


def test_shuffle_equals_sklearn():
    sk = pytest.importorskip('sklearn.utils')
    rng = np.random.default_rng(5)
    for n in (1, 2, 7, 50):
        idx = np.arange(n, dtype=np.int32)
        names = ['f%d' % i for i in range(n)]
        labels = [rng.integers(0, 9, (int(rng.integers(0, 4)), 5)) for _ in range(n)]
        np.random.seed(n)
        want = sk.shuffle(idx.copy(), list(names), list(labels))
        want_state = np.random.get_state()[1:3]
        np.random.seed(n)
        got = [idx.copy(), list(names), list(labels)]
        shuffle_together(got)
        assert np.array_equal(got[0], want[0]) and got[1] == want[1]
        assert all(a is b for a, b in zip(got[2], want[2]))
        s = np.random.get_state()
        assert np.array_equal(s[1], want_state[0]) and s[2] == want_state[1]


def test_planners_build_the_records():
    np.random.seed(0)
    ops, h, w, _ = Resize(30, 40, interpolation_mode=2).plan(10, 20, None)
    assert ops == [ba.resize_interp(10, 20, 30, 40, 2, drop_degenerate=False)] and (h, w) == (30, 40)
    assert ConvertTo3Channels().plan(5, 6, None) == ([], 5, 6, None)
    for cls in (SSDDataAugmentation, SSDPhotometricDistortions, SSDExpand, SSDRandomCrop, RandomFlip, ConvertTo3Channels):
        with pytest.raises(TypeError, match='generate'):
            cls()(np.zeros((4, 4, 3), np.uint8), np.zeros((0, 5)))
    with pytest.raises(TypeError, match='generate'):
        ResizeRandomInterp(4, 4)(np.zeros((4, 4, 3), np.uint8))


def test_refusals(tmp_path):
    g, gen = golden_dataset()
    with pytest.raises(NotImplementedError):
        DataGenerator(hdf5_dataset_path=str(tmp_path / 'x.h5'))
    for returns in ({'processed_images', 'matched_anchors'}, {'processed_images', 'inverse_transform'}):
        with pytest.raises(NotImplementedError):
            next(gen.generate(batch_size=2, returns=returns))
    with pytest.raises(NotImplementedError, match='transformation'):
        next(gen.generate(batch_size=2, transformations=[lambda image, labels: (image, labels)]))
    with pytest.raises(DatasetError):
        next(DataGenerator().generate(batch_size=2))
    with pytest.raises(ValueError):
        ba.resize_interp(4, 4, 2, 2, 5)


def test_dataset_accessors(tmp_path):
    from PIL import Image
    names = []
    for i, shape in enumerate([(5, 7, 3), (6, 4)]):
        Image.fromarray(np.full(shape, 10 * i, np.uint8)).save(str(tmp_path / ('%d.png' % i)))
        names.append('%d.png' % i)
    (tmp_path / 'list.txt').write_text('\n'.join(names) + '\n')
    gen = DataGenerator(load_images_into_memory=True, filenames=str(tmp_path / 'list.txt'), images_dir=str(tmp_path),
                        labels=[np.zeros((0, 5))] * 2, image_ids=['a', 'b'])
    assert gen.get_dataset_size() == 2 and gen.get_dataset()[2] == ['a', 'b']
    assert [im.shape for im in gen.images] == [(5, 7, 3), (6, 4)]
