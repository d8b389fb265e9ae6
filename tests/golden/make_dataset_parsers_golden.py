#!/usr/bin/env python
"""Goldens of the REAL reference's ``DataGenerator.parse_xml``, ``parse_json`` and one ``generate()`` over a parsed dataset
(data_generator/object_detection_2d_data_generator.py), on the dataset tests/voc_dataset.py rebuilds from a seed.

- ``xml``: ``parse_xml`` over an option matrix (one image set; 2007 + 2012 merged; ``include_classes``; ``exclude_truncated``;
  ``exclude_difficult``; both with ``include_classes``; no annotations; a custom ``labels_output_format``; images loaded into
  memory) and two re-parses on one generator.  Each run calls with ``ret=True`` and records the returned tuple and the
  attributes the parser sets, paths relative to the dataset root and images as a digest of the decoded arrays.
- ``json``: ``parse_json`` with and without ground truth, ``include_classes``, two annotations files, a custom format, images in
  memory, and a ``parse_json`` after a ``parse_xml`` (it leaves ``eval_neutral`` alone).
- ``errors``: the exception type each malformed input raises (``voc_dataset.ERROR_CASES``).
- ``generate``: ``parse_xml`` of the 2007 test list, then ``np.random.seed(GENERATE_SEED)`` and ``generate()`` with
  ``ConvertTo3Channels`` then ``Resize(300, 300)`` (the training notebook's validation chain), batches of 4 with shuffling so
  that a pass wraps, returning the processed images (digests), processed labels, file names, ids, evaluation-neutral flags and
  original labels, and ``np.random``'s state after each batch.

The reference reads VOC annotations with BeautifulSoup's ``'xml'`` parser (lxml), neither of which is installed here.  A small
stand-in for ``bs4`` is put into ``sys.modules`` first, as tf_shim.py does for TensorFlow: ``BeautifulSoup(f, 'xml')`` parses
with ``xml.etree.ElementTree``; ``tag.<name>`` and ``find(name)`` give the first descendant of that name in document order,
``find(name, recursive=False)`` the first direct child, ``find_all(name)`` every descendant, and ``.text`` the text of all
descendants.  So these goldens pin the reference's own logic -- its order of lookups, filters and exclusions, its quirks and
the exception types its code raises -- but not BeautifulSoup itself; that the stand-in agrees with BeautifulSoup on these
files is not checked here (it cannot be without bs4 and lxml).  Only well-formed XML is covered.

cv2 runs with IPP off.  Needs the reference tree, cv2, PIL, sklearn and tqdm; run once, the .json is data."""
import json
import os
import sys
import tempfile
import types
import xml.etree.ElementTree as ET

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import voc_dataset as ds  # noqa: E402


class _Tag:
    """The part of a bs4 ``Tag`` the reference's ``parse_xml`` uses, over an ElementTree element."""

    def __init__(self, element):
        self._e = element

    def find(self, name, recursive=True):
        e = self._e.find(name) if not recursive else next((d for d in self._e.iter(name) if d is not self._e), None)
        return None if e is None else _Tag(e)

    def find_all(self, name):
        return [_Tag(d) for d in self._e.iter(name) if d is not self._e]

    def __getattr__(self, name):
        if name.startswith('_'):
            raise AttributeError(name)
        return self.find(name)

    @property
    def text(self):
        return ''.join(self._e.itertext())


def _beautiful_soup(markup, features):
    assert features == 'xml'
    document = ET.Element('[document]')
    document.append(ET.fromstring(markup.read() if hasattr(markup, 'read') else markup))
    return _Tag(document)


sys.modules['bs4'] = types.SimpleNamespace(BeautifulSoup=_beautiful_soup)
sys.path.insert(0, os.environ.get('SSD_REFERENCE_ROOT', '/root/reference'))

import cv2  # noqa: E402

from data_generator.object_detection_2d_data_generator import DataGenerator  # noqa: E402
from data_generator.object_detection_2d_geometric_ops import Resize  # noqa: E402
from data_generator.object_detection_2d_photometric_ops import ConvertTo3Channels  # noqa: E402

GENERATE_SEED, GENERATE_BATCH, GENERATE_BATCHES = 23, 4, 4


def parse(root, kind, runs):
    out = {}
    for name, (ctor, calls) in runs.items():
        gen = DataGenerator(**ctor)
        for call in calls:
            ret = getattr(gen, 'parse_' + kind)(ret=True, verbose=False, **call)
        out[name] = ds.record(root, gen, ret, ds.XML_ATTRS if kind == 'xml' else ds.JSON_ATTRS)
        print(kind, name, gen.dataset_size, 'images')
    return out


def xml_then_json(root):
    gen = DataGenerator()
    im07, an07, sets07 = ds.voc_dirs(root, 'VOC2007')
    gen.parse_xml(images_dirs=[im07], image_set_filenames=[os.path.join(sets07, 'test.txt')], annotations_dirs=[an07], verbose=False)
    val_dir, val = ds.coco_paths(root, 'val')
    ret = gen.parse_json(images_dirs=[val_dir], annotations_filenames=[val], ground_truth_available=False, ret=True, verbose=False)
    return ds.record(root, gen, ret, ds.JSON_ATTRS)


def errors():
    out = {}
    for name in ds.ERROR_CASES:
        with tempfile.TemporaryDirectory() as tmp:
            kind, kwargs = ds.write_error_case(tmp, name)
            try:
                getattr(DataGenerator(), 'parse_' + kind)(verbose=False, **kwargs)
                out[name] = None
            except Exception as e:                   # the type is what is recorded
                out[name] = type(e).__name__
        print('error', name, out[name])
    return out


def generate(root):
    im07, an07, sets07 = ds.voc_dirs(root, 'VOC2007')
    gen = DataGenerator()
    gen.parse_xml(images_dirs=[im07], image_set_filenames=[os.path.join(sets07, 'test.txt')], annotations_dirs=[an07], verbose=False)
    np.random.seed(GENERATE_SEED)
    it = gen.generate(batch_size=GENERATE_BATCH, shuffle=True, transformations=[ConvertTo3Channels(), Resize(300, 300)], label_encoder=None,
                      returns={'processed_images', 'processed_labels', 'filenames', 'image_ids', 'evaluation-neutral', 'original_labels'},
                      keep_images_without_gt=False)
    batches = []
    for k in range(GENERATE_BATCHES):
        x, y, files, ids, neutral, original = next(it)
        state = np.random.get_state()
        batches.append({'x': [ds.image_digest(np.asarray(a, np.uint8)) for a in x], 'x_shape': list(np.asarray(x).shape),
                        'labels': [np.asarray(a, np.float64).tolist() for a in y], 'filenames': ds.rel(root, files), 'image_ids': ids,
                        'eval_neutral': neutral, 'original_labels': original, 'state_digest': ds.image_digest(state[1]), 'pos': int(state[2])})
        print('generate batch', k, ids)
    return {'seed': GENERATE_SEED, 'batch_size': GENERATE_BATCH, 'batches': batches}


def main():
    cv2.ipp.setUseIPP(False)
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, 'data') + os.sep
        ds.write(root)
        out = {'digest': ds.digest(root), 'xml': parse(root, 'xml', ds.xml_runs(root)), 'json': parse(root, 'json', ds.json_runs(root)),
               'xml_then_json': xml_then_json(root), 'errors': errors(), 'generate': generate(root)}
    with open(os.path.join(HERE, 'ref_dataset_parsers_golden.json'), 'w') as f:
        json.dump(out, f, indent=None, separators=(',', ':'))
        f.write('\n')


if __name__ == '__main__':
    main()
