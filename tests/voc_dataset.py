"""A small Pascal VOC / MS COCO shaped dataset, rebuilt from a seed with NumPy and PIL, for the parsers of ``DataGenerator``
(tests/golden/make_dataset_parsers_golden.py) and the notebook tests on the device.

``write(root)`` writes:

- ``VOCdevkit/VOC2007`` and ``VOCdevkit/VOC2012``, each with ``JPEGImages/``, ``Annotations/`` and ``ImageSets/Main/`` (2007:
  ``trainval.txt`` and ``test.txt``; 2012: ``trainval.txt``).  The annotations have several objects each, ``difficult`` and
  ``truncated`` set, person objects with ``<part>`` children that have their own ``name`` and ``bndbox`` (some placed before
  the object's own ``bndbox``), numbers padded with whitespace, a ``folder`` nested in an earlier element, a ``pose`` split
  by a child element, an image without objects and one whose objects are all cats (excluded by ``VOC_INCLUDE``);
- ``coco/val`` with ``coco/annotations/instances_val.json`` (non-consecutive category ids out of order, float and int boxes,
  an image without annotations) and ``coco/extra`` with ``instances_extra.json``, whose category list differs from the first
  file's and has a category the first file lacks.

Every image file is PNG content under a ``.jpg`` name (PIL picks the format from the header), so decoding it depends on no
JPEG library.  ``digest(root)`` hashes the decoded images and the annotation files: a test checks with it that the tree is
the one the golden was recorded from."""
import hashlib
import json
import os

import numpy as np

SEED = 20261020
VOC_CLASSES = ['background', 'aeroplane', 'bicycle', 'bird', 'boat', 'bottle', 'bus', 'car', 'cat', 'chair', 'cow', 'diningtable',
               'dog', 'horse', 'motorbike', 'person', 'pottedplant', 'sheep', 'sofa', 'train', 'tvmonitor']
VOC_SIZES = [(375, 500), (500, 375), (333, 500), (500, 333), (281, 500), (366, 500), (500, 400), (338, 500)]
VOC_INCLUDE = [7, 12, 15]                     # car, dog, person
N_2007, N_2012 = 16, 6
TEST_2007 = [3, 11, 0, 7, 14, 5, 9, 15, 2, 12]  # indices into the 2007 ids, in the order of test.txt; the rest is trainval
EMPTY_2007, CATS_ONLY_2007 = 9, 2              # an image without objects and one with cats only (both in test.txt)
GRAY_2007 = 5                                  # a single-channel image
COCO_CATS = [(1, 'person'), (3, 'car'), (90, 'toothbrush'), (18, 'dog'), (44, 'bottle')]
COCO_EXTRA_CATS = [(3, 'car'), (7, 'train'), (1, 'person')]
COCO_SIZES = [(480, 640), (427, 640), (640, 480), (375, 500), (640, 427), (512, 512), (333, 500), (424, 640)]
COCO_INCLUDE = [1, 3, 90]


def voc_ids():
    return ['%06d' % (i + 1) for i in range(N_2007)], ['2008_%06d' % (2 * i + 3) for i in range(N_2012)]


def _image(rng, h, w, gray=False):
    """16 x 16 blocks of random colour over a smooth ramp (small PNGs)."""
    base = rng.integers(0, 200, (h // 16 + 1, w // 16 + 1, 1 if gray else 3), dtype=np.int64)
    img = np.repeat(np.repeat(base, 16, 0), 16, 1)[:h, :w]
    img = img + ((np.arange(h)[:, None] + np.arange(w)[None, :]) * 55 // (h + w))[:, :, None]
    img = img.astype(np.uint8)
    return img[:, :, 0] if gray else img


def _save(img, path):
    from PIL import Image
    os.makedirs(os.path.dirname(path), exist_ok=True)
    Image.fromarray(img).save(path, format='PNG')


def _num(rng, v):
    """A coordinate or flag, sometimes padded with whitespace."""
    return ['%d' % v, ' %d ' % v, '\n\t\t\t%d\n\t\t' % v][int(rng.integers(3))]


def _bndbox(rng, h, w, indent):
    x0, y0 = int(rng.integers(1, w - 40)), int(rng.integers(1, h - 40))
    x1, y1 = int(rng.integers(x0 + 20, w + 1)), int(rng.integers(y0 + 20, h + 1))
    t = indent + '\t'
    return (indent + '<bndbox>\n' + ''.join('%s<%s>%s</%s>\n' % (t, k, _num(rng, v), k) for k, v in
                                             (('xmin', x0), ('ymin', y0), ('xmax', x1), ('ymax', y1))) + indent + '</bndbox>\n')


def _object(rng, h, w, name):
    pose = ['Left', 'Right', 'Frontal', 'Unspecified'][int(rng.integers(4))]
    if rng.integers(4) == 0:
        pose = pose[:2] + '<i>' + pose[2:4] + '</i>' + pose[4:]   # its text is that of all descendants
    trunc, diff = int(rng.integers(3) == 0), int(rng.integers(4) == 0)
    parts = ''
    if name == 'person':
        for part in ('head', 'hand', 'foot')[:int(rng.integers(1, 4))]:
            parts += '\t\t<part>\n\t\t\t<name>%s</name>\n%s\t\t</part>\n' % (part, _bndbox(rng, h, w, '\t\t\t'))
    box = _bndbox(rng, h, w, '\t\t')
    early = name == 'person' and rng.integers(2) == 0
    return ('\t<object>\n\t\t<name>%s</name>\n\t\t<pose>%s</pose>\n\t\t<truncated>%s</truncated>\n\t\t<difficult>%s</difficult>\n'
            % (name, pose, _num(rng, trunc), _num(rng, diff)) + (parts + box if early else box + parts) + '\t</object>\n')


def _xml(rng, folder, image_id, h, w, names, nested_folder=False):
    head = '\t<owner>\n\t\t<folder>owners</folder>\n\t</owner>\n' if nested_folder else ''
    return ('<annotation>\n%s\t<folder>%s</folder>\n\t<filename>%s.jpg</filename>\n\t<size>\n\t\t<width>%d</width>\n'
            '\t\t<height>%d</height>\n\t\t<depth>3</depth>\n\t</size>\n\t<segmented>0</segmented>\n%s</annotation>\n'
            % (head, folder, image_id, w, h, ''.join(_object(rng, h, w, n) for n in names)))


def _voc_year(rng, root, year, ids, sets, special=None):
    base = os.path.join(root, 'VOCdevkit', year)
    os.makedirs(os.path.join(base, 'Annotations'), exist_ok=True)
    os.makedirs(os.path.join(base, 'ImageSets', 'Main'), exist_ok=True)
    for i, image_id in enumerate(ids):
        h, w = VOC_SIZES[int(rng.integers(len(VOC_SIZES)))]
        _save(_image(rng, h, w, gray=special is not None and i == GRAY_2007), os.path.join(base, 'JPEGImages', image_id + '.jpg'))
        if special is not None and i == EMPTY_2007:
            names = []
        elif special is not None and i == CATS_ONLY_2007:
            names = ['cat', 'cat']
        else:
            names = [VOC_CLASSES[int(c)] for c in rng.integers(1, 21, int(rng.integers(1, 6)))]
            names += ['person'] if i % 3 == 0 else []
        with open(os.path.join(base, 'Annotations', image_id + '.xml'), 'w') as f:
            f.write(_xml(rng, year, image_id, h, w, names, nested_folder=i % 4 == 1))
    for name, members in sets.items():
        with open(os.path.join(base, 'ImageSets', 'Main', name + '.txt'), 'w') as f:
            f.write(''.join(ids[i] + (' \n' if k % 3 == 1 else '\n') for k, i in enumerate(members)))


def _coco_file(rng, root, split, cats, ids, n_ann, empty):
    images, anns = [], []
    for k, image_id in enumerate(ids):
        h, w = COCO_SIZES[k % len(COCO_SIZES)]
        name = '%012d.jpg' % image_id
        _save(_image(rng, h, w, gray=k == 3), os.path.join(root, 'coco', split, name))
        images.append({'license': 1, 'file_name': name, 'height': h, 'width': w, 'id': image_id})
        for _ in range(0 if k == empty else n_ann):
            bw, bh = float(rng.uniform(8, w / 2)), float(rng.uniform(8, h / 2))
            box = [round(float(rng.uniform(0, w - bw)), 2), round(float(rng.uniform(0, h - bh)), 2), round(bw, 2), round(bh, 2)]
            if rng.integers(5) == 0:
                box = [int(v) for v in box]                      # int boxes stay int
            anns.append({'segmentation': [], 'area': round(box[2] * box[3], 3), 'iscrowd': 0, 'image_id': image_id, 'bbox': box,
                         'category_id': cats[int(rng.integers(len(cats)))][0], 'id': 900000 + len(anns) + 1000 * len(ids)})
    doc = {'info': {'description': 'synthetic'}, 'licenses': [{'id': 1, 'name': 'none'}], 'images': images, 'annotations': anns,
           'categories': [{'supercategory': 'thing', 'id': c, 'name': n} for c, n in cats]}
    path = os.path.join(root, 'coco', 'annotations', 'instances_%s.json' % split)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, 'w') as f:
        json.dump(doc, f)


def write(root):
    """Writes the dataset under ``root`` (see the module's docstring)."""
    rng = np.random.default_rng(SEED)
    ids07, ids12 = voc_ids()
    test = TEST_2007
    trainval = [i for i in range(N_2007) if i not in test]
    _voc_year(rng, root, 'VOC2007', ids07, {'trainval': trainval, 'test': test}, special=True)
    _voc_year(rng, root, 'VOC2012', ids12, {'trainval': [4, 0, 2, 1, 5, 3]})
    _coco_file(rng, root, 'val', COCO_CATS, [139, 285, 632, 724, 776, 1000, 1268, 1296], 4, empty=5)
    _coco_file(rng, root, 'extra', COCO_EXTRA_CATS, [397133, 37777, 252219, 87038], 3, empty=None)


def voc_dirs(root, year):
    base = os.path.join(root, 'VOCdevkit', year)
    return os.path.join(base, 'JPEGImages'), os.path.join(base, 'Annotations'), os.path.join(base, 'ImageSets', 'Main')


def coco_paths(root, split):
    return os.path.join(root, 'coco', split), os.path.join(root, 'coco', 'annotations', 'instances_%s.json' % split)


def digest(root):
    from PIL import Image
    h = hashlib.sha256()
    for d, _, files in sorted(os.walk(root)):
        for name in sorted(files):
            path = os.path.join(d, name)
            h.update(os.path.relpath(path, root).encode())
            if name.endswith('.jpg'):
                with Image.open(path) as im:
                    a = np.array(im, dtype=np.uint8)
                h.update(str(a.shape).encode())
                h.update(a.tobytes())
            else:
                with open(path, 'rb') as f:
                    h.update(f.read())
    return h.hexdigest()


XML_ATTRS = ['filenames', 'image_ids', 'labels', 'eval_neutral', 'images_dirs', 'annotations_dirs', 'image_set_filenames', 'classes',
             'include_classes']
JSON_ATTRS = ['filenames', 'image_ids', 'labels', 'eval_neutral', 'images_dirs', 'annotations_filenames', 'include_classes',
              'cats_to_names', 'classes_to_names', 'cats_to_classes', 'classes_to_cats']


def image_digest(a):
    return hashlib.sha256(str(a.shape).encode() + np.ascontiguousarray(a).tobytes()).hexdigest()


def rel(root, v):
    """Paths relative to the dataset root, everything else as it is."""
    if isinstance(v, str) and v.startswith(root):
        return os.path.relpath(v, root)
    if isinstance(v, (list, tuple)):
        return [rel(root, x) for x in v]
    return v


def record(root, gen, ret, names):
    """What the golden records of a parse: the returned tuple and the attributes ``names``, paths relative to ``root`` and
    images as digests."""
    out = {'ret': None if ret is None else [len(ret)] + [rel(root, r) for r in ret[1:]],
           'images': None if gen.images is None else [image_digest(a) for a in gen.images],
           'dataset_size': gen.dataset_size, 'dataset_indices': gen.dataset_indices.tolist(),
           'dataset_indices_dtype': str(gen.dataset_indices.dtype)}
    for n in names:
        v = getattr(gen, n)
        out[n] = [[k, x] for k, x in v.items()] if isinstance(v, dict) else rel(root, v)
    return out


def xml_runs(root):
    """The recorded ``parse_xml`` runs: name -> (constructor kwargs, [parse_xml kwargs, ...]); the last call is recorded."""
    im07, an07, sets07 = voc_dirs(root, 'VOC2007')
    im12, an12, sets12 = voc_dirs(root, 'VOC2012')
    test = dict(images_dirs=[im07], image_set_filenames=[os.path.join(sets07, 'test.txt')], annotations_dirs=[an07])
    merged = dict(images_dirs=[im07, im12], image_set_filenames=[os.path.join(sets07, 'trainval.txt'), os.path.join(sets12, 'trainval.txt')],
                  annotations_dirs=[an07, an12])
    return {
        'test': ({}, [test]),
        'merged': ({}, [merged]),
        'include': ({}, [dict(test, include_classes=VOC_INCLUDE)]),
        'truncated': ({}, [dict(merged, exclude_truncated=True)]),
        'difficult': ({}, [dict(merged, exclude_difficult=True)]),
        'include_both': ({}, [dict(test, include_classes=VOC_INCLUDE, exclude_truncated=True, exclude_difficult=True)]),
        'no_annotations': ({}, [dict(merged, annotations_dirs=[])]),
        'format': (dict(labels_output_format=('ymin', 'folder', 'xmin', 'ymax', 'class_id', 'xmax', 'pose', 'truncated')), [test]),
        'memory': (dict(load_images_into_memory=True), [dict(test, include_classes=VOC_INCLUDE)]),
        'reparse': ({}, [merged, dict(test, annotations_dirs=[])]),
    }


def json_runs(root):
    """The recorded ``parse_json`` runs, as ``xml_runs``."""
    val_dir, val = coco_paths(root, 'val')
    extra_dir, extra = coco_paths(root, 'extra')
    one = dict(images_dirs=[val_dir], annotations_filenames=[val])
    two = dict(images_dirs=[val_dir, extra_dir], annotations_filenames=[val, extra])
    return {
        'gt': ({}, [dict(one, ground_truth_available=True)]),
        'no_gt': ({}, [one]),
        'include': ({}, [dict(one, ground_truth_available=True, include_classes=COCO_INCLUDE)]),
        'two_files': ({}, [dict(two, ground_truth_available=True, include_classes=COCO_INCLUDE)]),
        'two_files_no_gt': ({}, [two]),
        'format': (dict(labels_output_format=('xmin', 'image_id', 'ymin', 'xmax', 'ymax', 'class_id')), [dict(one, ground_truth_available=True)]),
        'memory': (dict(load_images_into_memory=True), [dict(one, ground_truth_available=True)]),
    }


# Malformed inputs: name -> the change to a one-image dataset.  XML: the object has a person ``<part>`` with its own ``name``
# and ``bndbox`` before its own tags, so that only a direct-child lookup misses a removed tag.
_ERROR_XML = ('<annotation>\n\t<folder>VOC2007</folder>\n\t<object>\n\t\t<part>\n\t\t\t<name>head</name>\n\t\t\t<bndbox><xmin>1</xmin>'
              '<ymin>2</ymin><xmax>3</xmax><ymax>4</ymax></bndbox>\n\t\t</part>\n\t\t<name>person</name>\n\t\t<pose>Left</pose>\n'
              '\t\t<truncated>0</truncated>\n\t\t<difficult>0</difficult>\n\t\t<bndbox>\n\t\t\t<xmin>48</xmin>\n\t\t\t<ymin>40</ymin>\n'
              '\t\t\t<xmax>195</xmax>\n\t\t\t<ymax>371</ymax>\n\t\t</bndbox>\n\t</object>\n</annotation>\n')
ERROR_CASES = {
    'unknown_class': ('xml', ('<name>person</name>', '<name>unicorn</name>')),
    'padded_class_name': ('xml', ('<name>person</name>', '<name> person</name>')),
    'float_coordinate': ('xml', ('<xmin>48</xmin>', '<xmin>48.5</xmin>')),
    'text_flag': ('xml', ('<difficult>0</difficult>', '<difficult>no</difficult>')),
    'missing_file': ('xml', None),
    'no_folder': ('xml', ('<folder>VOC2007</folder>', '')),
    'no_name': ('xml', ('<name>person</name>', '')),
    'no_pose': ('xml', ('<pose>Left</pose>', '')),
    'no_truncated': ('xml', ('<truncated>0</truncated>', '')),
    'no_difficult': ('xml', ('<difficult>0</difficult>', '')),
    'no_bndbox': ('xml', ('<bndbox>\n\t\t\t<xmin>48</xmin>\n\t\t\t<ymin>40</ymin>\n\t\t\t<xmax>195</xmax>\n\t\t\t<ymax>371</ymax>\n\t\t</bndbox>', '')),
    'no_ymax': ('xml', ('<ymax>371</ymax>', '')),
    'json_unknown_category': ('json', 'category_id'),
    'json_no_file_name': ('json', 'file_name'),
    'json_no_bbox': ('json', 'bbox'),
    'json_no_categories': ('json', 'categories'),
    'json_no_image_id': ('json', 'image_id'),
}


def write_error_case(root, name):
    """Writes the malformed dataset ``name`` under ``root`` -> (``'xml'`` or ``'json'``, the parser's keyword arguments)."""
    kind, change = ERROR_CASES[name]
    if kind == 'xml':
        for d in ('JPEGImages', 'Annotations'):
            os.makedirs(os.path.join(root, d), exist_ok=True)
        with open(os.path.join(root, 'set.txt'), 'w') as f:
            f.write('000001\n' if change is not None else 'nofile\n')
        if change is not None:
            assert change[0] in _ERROR_XML
            with open(os.path.join(root, 'Annotations', '000001.xml'), 'w') as f:
                f.write(_ERROR_XML.replace(change[0], change[1], 1))
        return kind, dict(images_dirs=[os.path.join(root, 'JPEGImages')], image_set_filenames=[os.path.join(root, 'set.txt')],
                          annotations_dirs=[os.path.join(root, 'Annotations')])
    doc = {'images': [{'file_name': 'a.jpg', 'id': 1}],
           'annotations': [{'image_id': 1, 'bbox': [1.5, 2, 30, 40.25], 'category_id': 3}],
           'categories': [{'id': 3, 'name': 'car'}]}
    if change == 'category_id':
        doc['annotations'][0]['category_id'] = 7
    elif change == 'categories':
        del doc['categories']
    elif change == 'file_name':
        del doc['images'][0]['file_name']
    else:
        del doc['annotations'][0][change]
    with open(os.path.join(root, 'instances.json'), 'w') as f:
        json.dump(doc, f)
    return kind, dict(images_dirs=[root], annotations_filenames=[os.path.join(root, 'instances.json')], ground_truth_available=True)
