"""``DataGenerator.parse_xml``, ``parse_json`` and ``save_dataset`` against the real reference
(tests/golden/make_dataset_parsers_golden.py) on the VOC / COCO shaped dataset of tests/voc_dataset.py: every recorded option
set gives the reference's values with the reference's Python types and sets the same attributes; malformed inputs raise the
reference's exception types; a saved dataset reads back through the constructor; and ``plan_batches`` over a parsed dataset,
run through the oracle's image and box ops, reproduces the reference's ``generate()`` and its ``np.random`` state."""
import json
import os
import pickle

import numpy as np
import pytest

import resize_reference as rr
import voc_dataset as ds
from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator
from ssd_keras_b200.data_generator.object_detection_2d_geometric_ops import Resize
from ssd_keras_b200.data_generator.object_detection_2d_photometric_ops import ConvertTo3Channels

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_dataset_parsers_golden.json')
@pytest.fixture(scope='module')
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.fixture(scope='module')
def root(tmp_path_factory, golden):
    """The dataset the golden was recorded from, rebuilt and checked by its digest."""
    path = str(tmp_path_factory.mktemp('voc') / 'data') + os.sep
    ds.write(path)
    assert ds.digest(path) == golden['digest']
    return path


def assert_same(got, want, where):
    """Equal values of the same Python types: lists are lists, ints ints, floats floats, bools bools."""
    if isinstance(want, list):
        assert type(got) is list, (where, type(got))
        assert len(got) == len(want), where
        for k, (a, b) in enumerate(zip(got, want)):
            assert_same(a, b, '%s[%d]' % (where, k))
    else:
        assert type(got) is type(want) and got == want, (where, got, want)


def parse(root, kind, name):
    ctor, calls = (ds.xml_runs if kind == 'xml' else ds.json_runs)(root)[name]
    gen = DataGenerator(**ctor)
    for call in calls:
        ret = getattr(gen, 'parse_' + kind)(ret=True, verbose=False, **call)
    return gen, ret


def assert_record(root, gen, ret, want, names):
    got = ds.record(root, gen, ret, names)
    assert sorted(got) == sorted(want)
    for k in want:
        assert_same(got[k], want[k], k)
    order = ('images', 'filenames', 'labels', 'image_ids', 'eval_neutral')
    assert type(ret) is tuple and all(r is getattr(gen, n) for r, n in zip(ret, order))


@pytest.mark.parametrize('name', list(ds.xml_runs('')))
def test_parse_xml_equals_the_reference(root, golden, name):
    gen, ret = parse(root, 'xml', name)
    assert_record(root, gen, ret, golden['xml'][name], ds.XML_ATTRS)


@pytest.mark.parametrize('name', list(ds.json_runs('')))
def test_parse_json_equals_the_reference(root, golden, name):
    gen, ret = parse(root, 'json', name)
    assert_record(root, gen, ret, golden['json'][name], ds.JSON_ATTRS)


def test_images_in_memory_are_the_pil_decode(root):
    from ssd_keras_b200.eval_utils.dataset_predict import load_image
    for kind in ('xml', 'json'):
        gen, ret = parse(root, kind, 'memory')
        assert len(gen.images) == len(gen.filenames)
        for a, f in zip(gen.images, gen.filenames):
            b = load_image(f)
            assert a.dtype == np.uint8 and a.shape == b.shape and np.array_equal(a, b)
        assert any(a.ndim == 2 for a in gen.images)                 # the gray image stays 2-D, as PIL gives it


def test_parse_json_leaves_eval_neutral_alone(root, golden):
    gen = DataGenerator()
    gen.parse_xml(**ds.xml_runs(root)['test'][1][0], verbose=False)
    neutral = gen.eval_neutral
    val_dir, val = ds.coco_paths(root, 'val')
    ret = gen.parse_json(images_dirs=[val_dir], annotations_filenames=[val], ground_truth_available=False, ret=True, verbose=False)
    assert gen.eval_neutral is neutral and gen.labels is None
    assert_record(root, gen, ret, golden['xml_then_json'], ds.JSON_ATTRS)


def test_a_new_parse_erases_the_previous_one(root):
    gen, _ = parse(root, 'json', 'two_files')
    gen.parse_xml(**ds.xml_runs(root)['test'][1][0], verbose=False)
    assert gen.dataset_size == len(gen.filenames) == len(gen.labels) == len(gen.image_ids) == len(gen.eval_neutral) == 10
    assert all(isinstance(i, str) for i in gen.image_ids)
    gen.parse_json(**ds.json_runs(root)['gt'][1][0], verbose=False)
    assert gen.dataset_size == len(gen.filenames) == len(gen.labels) == 8 and len(gen.eval_neutral) == 10
    assert all(isinstance(i, int) for i in gen.image_ids)


@pytest.mark.parametrize('name', list(ds.ERROR_CASES))
def test_malformed_inputs_raise_the_reference_exceptions(tmp_path, golden, name):
    kind, kwargs = ds.write_error_case(str(tmp_path), name)
    want = golden['errors'][name]
    assert want in ('ValueError', 'FileNotFoundError', 'AttributeError', 'KeyError')
    with pytest.raises(Exception) as e:
        getattr(DataGenerator(), 'parse_' + kind)(verbose=False, **kwargs)
    assert type(e.value).__name__ == want


@pytest.mark.parametrize('kind,name', [('xml', 'merged'), ('xml', 'no_annotations'), ('json', 'two_files')])
def test_save_dataset_reads_back_through_the_constructor(root, tmp_path, kind, name):
    gen, _ = parse(root, kind, name)
    paths = {k: str(tmp_path / (k + '.pkl')) for k in ('filenames', 'labels', 'image_ids', 'eval_neutral')}
    gen.save_dataset(filenames_path=paths['filenames'], labels_path=paths['labels'], image_ids_path=paths['image_ids'],
                     eval_neutral_path=paths['eval_neutral'])
    back = DataGenerator(filenames=paths['filenames'], filenames_type='pickle', labels=paths['labels'], image_ids=paths['image_ids'],
                         eval_neutral=paths['eval_neutral'])
    assert back.get_dataset_size() == gen.get_dataset_size()
    assert np.array_equal(back.dataset_indices, gen.dataset_indices) and back.dataset_indices.dtype == np.int32
    for got, want, n in zip(back.get_dataset(), gen.get_dataset(), ('filenames', 'labels', 'image_ids', 'eval_neutral')):
        if want is None:
            assert got is None, n
        else:
            assert_same(got, want, n)


def test_save_dataset_writes_only_the_paths_given(root, tmp_path, monkeypatch):
    gen, _ = parse(root, 'xml', 'test')
    monkeypatch.chdir(tmp_path)
    gen.save_dataset()
    assert os.listdir(str(tmp_path)) == ['filenames.pkl']
    with open(str(tmp_path / 'filenames.pkl'), 'rb') as f:
        assert pickle.load(f) == gen.filenames


def test_plan_batches_reproduce_the_reference_generate(root, golden):
    """The training notebook's validation chain over a parsed VOC test list: the shuffle, the image without boxes dropped, the
    ids, flags and file names of each batch, and the images and boxes through the oracle, bit for bit."""
    g = golden['generate']
    gen, _ = parse(root, 'xml', 'test')
    np.random.seed(g['seed'])
    batches = gen.plan_batches(g['batch_size'], True, [ConvertTo3Channels(), Resize(300, 300)], False)
    for k, want in enumerate(g['batches']):
        b = next(batches)
        keep = b['keep']
        x = [rr.apply_ops(b['images'][i], o) for i, o in zip(keep, b['ops'])]
        y = [rr.apply_box_ops(b['labels'][i], o) for i, o in zip(keep, b['ops'])]
        assert [ds.image_digest(a) for a in x] == want['x'] and [len(x)] + list(x[0].shape) == want['x_shape'], k
        assert_same([a.astype(np.float64).tolist() for a in y], want['labels'], 'labels')
        assert_same(ds.rel(root, [b['filenames'][i] for i in keep]), want['filenames'], 'filenames')
        assert_same([b['image_ids'][i] for i in keep], want['image_ids'], 'image_ids')
        assert_same([b['eval_neutral'][i] for i in keep], want['eval_neutral'], 'eval_neutral')
        assert_same([b['labels'][i].tolist() for i in keep], want['original_labels'], 'original_labels')
        state = np.random.get_state()
        assert ds.image_digest(state[1]) == want['state_digest'] and state[2] == want['pos'], k
