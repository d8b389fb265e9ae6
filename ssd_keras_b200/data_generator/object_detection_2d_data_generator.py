"""``DataGenerator`` (the reference's object_detection_2d_data_generator.py): a dataset of images and labels, and ``generate()``,
which yields training batches assembled on the device.

``parse_csv`` (a CSV of boxes), ``parse_xml`` (Pascal VOC annotations) and ``parse_json`` (MS COCO annotations) read a dataset as
the reference's do, with the same attributes and return values; ``save_dataset`` pickles the parsed lists for the constructor.

Per batch, the host does what only the host can: the shuffle (``sklearn.utils.shuffle``'s permutation, drawn from the global
``np.random``), the batch slice, dropping images without boxes, and the random draws of the augmentation planners (the
``data_augmentation_chain_*`` modules and their parts), which turn each image into one op list.  Images are decoded with PIL on a small
thread pool ahead of the batch that needs them (or taken from memory).  The device then runs one assembly per batch:
``ssdk_assemble_images`` for the pixels, ``ssdk_assemble_batch`` for the boxes and the encoder on its output
(``batch_assembly.assemble_training_batch``), so ``'processed_images'`` and ``'encoded_labels'`` are the float32 CUDA tensors
``train_on_batch`` takes.

The reference checks the processed boxes for degenerate ones after the chain.  When every op list of a batch ends in a
degenerate-box filter (``Resize`` with one, as in ``SSDDataAugmentation`` and the variable-input-size and satellite chains), no
box can be degenerate and nothing is checked; otherwise (the SSD7 chain's lists end in a flip, or in the clip of a translation
or zoom) the processed boxes are read back once and the reference's ``'remove'`` / ``'warn'`` rules are applied to them.
That read-back, and the one of ``'processed_labels'``, run on a side stream of their own: they wait for the box work they
need, not for a training step or prediction still running on the caller's stream, so ``fit_generator`` can plan and assemble
the next batch while the device trains on the current one.

Not covered: HDF5 datasets, ``'matched_anchors'`` and ``'inverse_transform'`` returns, and
transformations other than the planners of this package."""
import csv
import json
import os
import pickle
import warnings
import xml.etree.ElementTree as ET
from collections import defaultdict
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import batch_assembly as ba
from .. import _ffi
from ..eval_utils.dataset_predict import load_image
from .object_detection_2d_geometric_ops import DevicePlanner

_DECODE_THREADS = 8
_DECODE_AHEAD = 2                      # batches decoded ahead of the one being assembled


class DegenerateBatchError(Exception):
    """An error indicating that an empty batch was produced."""


class DatasetError(Exception):
    """An error indicating that something is wrong with the dataset."""


def _load_list(value, name):
    if value is None or isinstance(value, (list, tuple)):
        return value
    if isinstance(value, str):
        with open(value, 'rb') as f:
            return pickle.load(f)
    raise ValueError('`%s` must be either a Python list/tuple or a string representing the path to a pickled file containing a '
                     'list/tuple. The value you passed is neither of the two.' % name)


def _text(element):
    """BeautifulSoup's ``.text``: the text of the element and all its descendants.  A tag that was not found (``None``) raises
    ``AttributeError``, as the reference's ``.text`` on BeautifulSoup's ``None`` does."""
    if element is None:
        raise AttributeError("'NoneType' object has no attribute 'text'")
    return ''.join(element.itertext())


def shuffle_together(objects):
    """``sklearn.utils.shuffle(*objects)`` written back in place: one permutation from the global ``np.random``
    (``np.random.shuffle(np.arange(n))``) applied to every list / array."""
    perm = np.arange(len(objects[0]))
    np.random.shuffle(perm)
    for o in objects:
        o[:] = [o[i] for i in perm] if isinstance(o, list) else o[perm]


def _has_degenerate(labels, fmt):
    return bool(np.any(labels[:, fmt['xmax']] - labels[:, fmt['xmin']] <= 0) or np.any(labels[:, fmt['ymax']] - labels[:, fmt['ymin']] <= 0))


def _ends_degenerate_free(ops):
    """Whether the list leaves no degenerate box: its last op that moves or filters boxes is a degenerate-box filter (an
    overlap test or a photometric op after it changes no box)."""
    for code, flags in ((o[0], o[1]) for o in reversed(ops)):
        if code in (_ffi.BOXOP_RESIZE, _ffi.BOXOP_RESIZE_INTERP, _ffi.BOXOP_FILTER):
            return bool(flags & 1)
        if code != _ffi.BOXOP_OVERLAP and code not in _ffi.PHOTO_OPS:
            return False
    return False


_GEOMETRIC_OPS = frozenset(range(_ffi.BOXOP_CROP_PAD, _ffi.BOXOP_ROTATE + 1)) - {_ffi.BOXOP_FILTER} | {_ffi.BOXOP_RESIZE_INTERP}


def _check_photometric_prefix(ops, transformations, owners):
    """The device runs an image's photometric ops before its geometry: refuse a list where one follows an op that changes the
    image geometry, naming both transformations."""
    first_geometric = None
    for o, k in zip(ops, owners):
        if o[0] in _GEOMETRIC_OPS and first_geometric is None:
            first_geometric = k
        elif o[0] in _ffi.PHOTO_OPS and first_geometric is not None:
            raise ValueError('the photometric transformation %r comes after %r, which changes the image geometry; the device runs '
                             'the photometric ops of an image first, so they must come before every crop, pad, flip, resize, '
                             'translation, scale and rotation' % (transformations[k], transformations[first_geometric]))


def _read_boxes(labels, ops, side):
    """The boxes of ``labels`` after ``ops``, read back to the host: float32 ``(N, 5)`` rows and ``(B+1,)`` offsets.  The work
    runs on ``side``, a stream held in a list that the first call fills: it starts once the previous box assembly has
    finished (``ssdk_assemble_batch`` orders its calls) and the host waits for nothing else on the device."""
    import torch
    if not side:
        side.append(torch.cuda.Stream())
    with torch.cuda.stream(side[0]):
        gt, offs = ba.assemble_batch_device(labels, ops)[:2]
        return gt.cpu().numpy(), offs.cpu().numpy()


class DataGenerator:
    """A dataset of images (files, or arrays in memory) with their labels, image ids and evaluation-neutral flags."""

    def __init__(self, load_images_into_memory=False, hdf5_dataset_path=None, filenames=None, filenames_type='text', images_dir=None,
                 labels=None, image_ids=None, eval_neutral=None, labels_output_format=('class_id', 'xmin', 'ymin', 'xmax', 'ymax'),
                 verbose=True):
        if hdf5_dataset_path is not None:
            raise NotImplementedError('HDF5 datasets are not supported; pass `filenames` (and `labels`)')
        self.labels_output_format = labels_output_format
        self.labels_format = {k: labels_output_format.index(k) for k in ('class_id', 'xmin', 'ymin', 'xmax', 'ymax')}
        self.dataset_size = 0
        self.load_images_into_memory = load_images_into_memory
        self.images = None
        self.hdf5_dataset = None
        self.filenames = None
        if filenames is not None:
            if isinstance(filenames, (list, tuple)):
                self.filenames = list(filenames)
            elif isinstance(filenames, str):
                if filenames_type == 'pickle':
                    with open(filenames, 'rb') as f:
                        self.filenames = pickle.load(f)
                elif filenames_type == 'text':
                    with open(filenames) as f:
                        self.filenames = [os.path.join(images_dir, line.strip()) for line in f]
                else:
                    raise ValueError("`filenames_type` can be either 'text' or 'pickle'.")
            else:
                raise ValueError('`filenames` must be either a Python list/tuple or a string representing a filepath (to a pickled '
                                 'or text file). The value you passed is neither of the two.')
            self._index_dataset()
        self.labels = _load_list(labels, 'labels')
        self.image_ids = _load_list(image_ids, 'image_ids')
        self.eval_neutral = _load_list(eval_neutral, 'eval_neutral')

    def parse_csv(self, images_dir, labels_filename, input_format, include_classes='all', random_sample=False, ret=False, verbose=True):
        """The reference's ``parse_csv``: one box per CSV row (after a header), its first six columns named by ``input_format``
        (``'image_name'``, ``'class_id'``, ``'xmin'``, ``'xmax'``, ``'ymin'``, ``'ymax'``).  Rows of ``include_classes`` are sorted
        (by file name, then by the label values), grouped by file into int64 label arrays in ``labels_output_format`` order, and
        the image id is the file name up to its first dot.  ``random_sample``: each image is kept if ``np.random.uniform(0, 1)
        >= 1 - random_sample``, one draw per image in file order.  With ``ret``, returns ``(images, filenames, labels,
        image_ids)``."""
        self.images_dir = images_dir
        self.labels_filename = labels_filename
        self.input_format = input_format
        self.include_classes = include_classes
        if self.labels_filename is None or self.input_format is None:
            raise ValueError("`labels_filename` and/or `input_format` have not been set yet. You need to pass them as arguments.")
        self.filenames = []
        self.image_ids = []
        self.labels = []
        data = []
        with open(self.labels_filename, newline='') as csvfile:
            csvread = csv.reader(csvfile, delimiter=',')
            next(csvread)
            for row in csvread:
                if self.include_classes == 'all' or int(row[self.input_format.index('class_id')].strip()) in self.include_classes:
                    box = [row[self.input_format.index('image_name')].strip()]
                    for element in self.labels_output_format:
                        box.append(int(row[self.input_format.index(element)].strip()))
                    data.append(box)
        data = sorted(data)
        groups = []                                          # (file name, its boxes) in sorted order
        for box in data:
            if not groups or box[0] != groups[-1][0]:
                groups.append((box[0], []))
            groups[-1][1].append(box[1:])
        if not groups:
            raise IndexError('list index out of range')      # the reference reads data[0]
        for current_file, current_labels in groups:
            if random_sample and not np.random.uniform(0, 1) >= (1 - random_sample):
                continue
            self.labels.append(np.stack(current_labels, axis=0))
            self.filenames.append(os.path.join(self.images_dir, current_file))
            self.image_ids.append(current_file.split('.')[0])
        self._index_dataset()
        if ret:
            return self.images, self.filenames, self.labels, self.image_ids

    def parse_xml(self, images_dirs, image_set_filenames, annotations_dirs=[],
                  classes=['background', 'aeroplane', 'bicycle', 'bird', 'boat', 'bottle', 'bus', 'car', 'cat', 'chair', 'cow',
                           'diningtable', 'dog', 'horse', 'motorbike', 'person', 'pottedplant', 'sheep', 'sofa', 'train', 'tvmonitor'],
                  include_classes='all', exclude_truncated=False, exclude_difficult=False, ret=False, verbose=True):
        """The reference's Pascal VOC parser.  Per image directory, the ids are the stripped lines of its image-set file (strings)
        and the file names ``<id>.jpg``; without ``annotations_dirs``, ``labels`` and ``eval_neutral`` are ``None``.  Otherwise
        each ``<id>.xml`` gives one box per ``object`` element in document order: ``[class_id, xmin, ymin, xmax, ymax]`` as Python
        ints in ``labels_output_format`` order (class ids index ``classes``), and its ``difficult`` flag as a bool in
        ``eval_neutral``.  ``include_classes`` is tested on the class id before ``exclude_truncated`` and ``exclude_difficult``.

        The reference reads the files with BeautifulSoup; here ``xml.etree.ElementTree`` does its lookups: the first ``folder``
        of the document, an object's direct ``name`` / ``pose`` / ``truncated`` / ``difficult`` / ``bndbox`` children (so the
        ``<part>`` children of VOC person objects never match), the first ``xmin`` ... under ``bndbox``, and an element's text
        as that of all its descendants.  A missing tag raises ``AttributeError``, an unknown class name or a non-integer
        number ``ValueError``.  With ``ret``, returns ``(images, filenames, labels, image_ids, eval_neutral)``."""
        self.images_dirs = images_dirs
        self.annotations_dirs = annotations_dirs
        self.image_set_filenames = image_set_filenames
        self.classes = classes
        self.include_classes = include_classes
        self.filenames = []
        self.image_ids = []
        self.labels = []
        self.eval_neutral = []
        if not annotations_dirs:
            self.labels = None
            self.eval_neutral = None
            annotations_dirs = [None] * len(images_dirs)
        for images_dir, image_set_filename, annotations_dir in zip(images_dirs, image_set_filenames, annotations_dirs):
            with open(image_set_filename) as f:
                image_ids = [line.strip() for line in f]
            self.image_ids += image_ids
            for image_id in image_ids:
                filename = image_id + '.jpg'
                self.filenames.append(os.path.join(images_dir, filename))
                if annotations_dir is None:
                    continue
                root = ET.parse(os.path.join(annotations_dir, image_id + '.xml')).getroot()
                folder = _text(next(root.iter('folder'), None))
                boxes, eval_neutr = [], []
                for obj in root.iter('object'):
                    class_name = _text(obj.find('name'))
                    class_id = self.classes.index(class_name)
                    if self.include_classes != 'all' and class_id not in self.include_classes:
                        continue
                    pose = _text(obj.find('pose'))
                    truncated = int(_text(obj.find('truncated')))
                    if exclude_truncated and truncated == 1:
                        continue
                    difficult = int(_text(obj.find('difficult')))
                    if exclude_difficult and difficult == 1:
                        continue
                    bndbox = obj.find('bndbox')
                    xmin, ymin, xmax, ymax = (int(_text(bndbox.find('.//' + k))) for k in ('xmin', 'ymin', 'xmax', 'ymax'))
                    item = {'folder': folder, 'image_name': filename, 'image_id': image_id, 'class_name': class_name,
                            'class_id': class_id, 'pose': pose, 'truncated': truncated, 'difficult': difficult,
                            'xmin': xmin, 'ymin': ymin, 'xmax': xmax, 'ymax': ymax}
                    boxes.append([item[k] for k in self.labels_output_format])
                    eval_neutr.append(bool(difficult))
                self.labels.append(boxes)
                self.eval_neutral.append(eval_neutr)
        self._index_dataset()
        if ret:
            return self.images, self.filenames, self.labels, self.image_ids, self.eval_neutral

    def parse_json(self, images_dirs, annotations_filenames, ground_truth_available=False, include_classes='all', ret=False,
                   verbose=True):
        """The reference's MS COCO parser.  The class maps come from the first annotations file's ``categories``, in its order:
        ``cats_to_names`` (COCO id -> name), ``classes_to_names`` (``'background'`` then the names), ``cats_to_classes`` (COCO id
        -> consecutive id from 1) and ``classes_to_cats``.  Per file, its ``images`` give the file names and the image ids
        (the JSON ints).  With ``ground_truth_available``, each image's ``annotations`` whose original category id is in
        ``include_classes`` give the boxes ``[class_id, x, y, x + w, y + h]`` in ``labels_output_format`` order, the JSON's
        numbers as they are; otherwise ``labels`` is ``None``.  ``eval_neutral`` is left as it is.  With ``ret``, returns
        ``(images, filenames, labels, image_ids)``."""
        self.images_dirs = images_dirs
        self.annotations_filenames = annotations_filenames
        self.include_classes = include_classes
        self.filenames = []
        self.image_ids = []
        self.labels = [] if ground_truth_available else None
        with open(annotations_filenames[0]) as f:
            categories = json.load(f)['categories']
        self.cats_to_names = {}
        self.classes_to_names = ['background']
        self.cats_to_classes = {}
        self.classes_to_cats = {}
        for i, cat in enumerate(categories):
            self.cats_to_names[cat['id']] = cat['name']
            self.classes_to_names.append(cat['name'])
            self.cats_to_classes[cat['id']] = i + 1
            self.classes_to_cats[i + 1] = cat['id']
        for images_dir, annotations_filename in zip(self.images_dirs, self.annotations_filenames):
            with open(annotations_filename) as f:
                annotations = json.load(f)
            if ground_truth_available:
                image_ids_to_annotations = defaultdict(list)
                for annotation in annotations['annotations']:
                    image_ids_to_annotations[annotation['image_id']].append(annotation)
            for img in annotations['images']:
                self.filenames.append(os.path.join(images_dir, img['file_name']))
                self.image_ids.append(img['id'])
                if not ground_truth_available:
                    continue
                boxes = []
                for annotation in image_ids_to_annotations[img['id']]:
                    cat_id = annotation['category_id']
                    if self.include_classes != 'all' and cat_id not in self.include_classes:
                        continue
                    class_id = self.cats_to_classes[cat_id]
                    xmin, ymin, width, height = (annotation['bbox'][k] for k in range(4))
                    item = {'image_name': img['file_name'], 'image_id': img['id'], 'class_id': class_id,
                            'xmin': xmin, 'ymin': ymin, 'xmax': xmin + width, 'ymax': ymin + height}
                    boxes.append([item[k] for k in self.labels_output_format])
                self.labels.append(boxes)
        self._index_dataset()
        if ret:
            return self.images, self.filenames, self.labels, self.image_ids

    def _index_dataset(self):
        """What every way of loading a dataset ends with: its size and indices, and its images decoded into memory when
        ``load_images_into_memory`` is set."""
        self.dataset_size = len(self.filenames)
        self.dataset_indices = np.arange(self.dataset_size, dtype=np.int32)
        if self.load_images_into_memory:
            with ThreadPoolExecutor(_DECODE_THREADS) as pool:
                self.images = list(pool.map(load_image, self.filenames))

    def save_dataset(self, filenames_path='filenames.pkl', labels_path=None, image_ids_path=None, eval_neutral_path=None):
        """Pickles ``filenames`` and, for each path given, ``labels``, ``image_ids`` and ``eval_neutral``, so that a slow parse
        is done once: the constructor reads the files back (``filenames_type='pickle'``, ``labels=``, ``image_ids=``,
        ``eval_neutral=``)."""
        with open(filenames_path, 'wb') as f:
            pickle.dump(self.filenames, f)
        for path, value in ((labels_path, self.labels), (image_ids_path, self.image_ids), (eval_neutral_path, self.eval_neutral)):
            if path is not None:
                with open(path, 'wb') as f:
                    pickle.dump(value, f)

    def get_dataset(self):
        return self.filenames, self.labels, self.image_ids, self.eval_neutral

    def get_dataset_size(self):
        return self.dataset_size

    def generate(self, batch_size=32, shuffle=True, transformations=[], label_encoder=None, returns={'processed_images', 'encoded_labels'},
                 keep_images_without_gt=False, degenerate_box_handling='remove'):
        """Yields batches indefinitely, as the reference's ``generate`` (same arguments and return order), from a device assembly
        of each batch.  ``transformations``: planners of this package (the three training chains, ``SSDDataAugmentation`` and
        the classes of the op modules: ``object_detection_2d_geometric_ops``, ``_patch_sampling_ops`` and ``_photometric_ops``),
        in any order that puts the photometric ops of an image before its first crop, pad, flip, resize, translation, scale or
        rotation (``ValueError`` otherwise); after them every image of a batch must have one size.
        ``'processed_images'`` is a float32 CUDA tensor ``(B, H, W, 3)``; ``'encoded_labels'`` the float32 CUDA ``y_true``;
        ``'processed_labels'`` a list of float64 arrays read back from the device."""
        if self.dataset_size == 0:
            raise DatasetError('Cannot generate batches because you did not load a dataset.')
        for r in ('matched_anchors', 'inverse_transform'):
            if r in returns:
                raise NotImplementedError("the '%s' return is not supported" % r)
        for t in transformations:
            if not isinstance(t, DevicePlanner):
                raise NotImplementedError('transformation %r is not one the device generator knows; use the planners of '
                                          'ssd_keras_b200.data_generator' % (t,))
        if self.labels is not None and self.labels_format != {'class_id': 0, 'xmin': 1, 'ymin': 2, 'xmax': 3, 'ymax': 4}:
            raise NotImplementedError("the device generator takes labels as ('class_id', 'xmin', 'ymin', 'xmax', 'ymax')")
        if degenerate_box_handling not in ('remove', 'warn'):
            raise ValueError("`degenerate_box_handling` must be either 'remove' or 'warn'")
        if self.labels is None:
            if any(r in returns for r in ('encoded_labels', 'processed_labels', 'original_labels')):
                warnings.warn('Since no labels were given, none of the label returns are possible; they will be `None`.')
        elif label_encoder is None and 'encoded_labels' in returns:
            warnings.warn("Since no label encoder was given, 'encoded_labels' is not possible; it will be `None`.")
        for t in transformations:
            t.labels_format = self.labels_format
        side = []                              # the stream of the box read-backs, made by the first one
        with ThreadPoolExecutor(_DECODE_THREADS) as pool:
            for batch in self.plan_batches(batch_size, shuffle, transformations, keep_images_without_gt, pool):
                batch_X, batch_y, keep, ops, out_hw = (batch[k] for k in ('images', 'labels', 'keep', 'ops', 'out_hw'))
                batch_filenames, batch_image_ids, batch_eval_neutral = batch['filenames'], batch['image_ids'], batch['eval_neutral']
                batch_original_images = [np.copy(x) for x in batch_X] if 'original_images' in returns else None
                batch_original_labels = [np.copy(y) for y in batch_y] if 'original_labels' in returns and batch_y is not None else None
                if batch_y is not None and keep and not all(_ends_degenerate_free(o) for o in ops):
                    keep, ops = self._degenerate_check(batch_X, batch_y, keep, ops, degenerate_box_handling, keep_images_without_gt, side)
                if not keep:
                    raise DegenerateBatchError('You produced an empty batch.')

                def pick(lst):
                    return None if lst is None else [lst[i] for i in keep]
                X_in, y_in = [batch_X[i] for i in keep], pick(batch_y)
                if batch_y is not None and label_encoder is not None:
                    X, y_enc = ba.assemble_training_batch(label_encoder, X_in, y_in, ops, out_hw[0], out_hw[1])
                else:
                    X, y_enc = ba.assemble_images_device(X_in, ops, out_hw[0], out_hw[1]), None
                processed = None
                if 'processed_labels' in returns and batch_y is not None:
                    gt, offs = _read_boxes(y_in, ops, side)
                    processed = [gt[offs[b]:offs[b + 1]].astype(np.float64) for b in range(len(keep))]
                ret = []
                if 'processed_images' in returns: ret.append(X)
                if 'encoded_labels' in returns: ret.append(y_enc)
                if 'processed_labels' in returns: ret.append(processed)
                if 'filenames' in returns: ret.append(pick(batch_filenames))
                if 'image_ids' in returns: ret.append(pick(batch_image_ids))
                if 'evaluation-neutral' in returns: ret.append(pick(batch_eval_neutral))
                if 'original_images' in returns: ret.append(pick(batch_original_images))
                if 'original_labels' in returns: ret.append(pick(batch_original_labels))
                yield ret

    def plan_batches(self, batch_size, shuffle, transformations, keep_images_without_gt, pool=None):
        """The host half of ``generate``: shuffles, slices, drops the images without boxes and draws every kept image's op
        list, in the reference's ``np.random`` order.  Yields dicts with the batch's ``images``, ``labels`` (arrays),
        ``filenames``, ``image_ids``, ``eval_neutral``, the indices ``keep`` of the images that go on, their ``ops`` and the
        common output size ``out_hw``."""
        if shuffle:
            self._shuffle()
        current = 0
        ahead = {}
        while True:
            if current >= self.dataset_size:
                current = 0
                if shuffle:
                    ahead.clear()
                    self._shuffle()
            for k in range(_DECODE_AHEAD + 1 if pool is not None else 1):
                lo = current + k * batch_size
                if lo < self.dataset_size and lo not in ahead:
                    ahead[lo] = self._fetch(pool, lo, batch_size)
            batch_X = [a.result() if hasattr(a, 'result') else a for a in ahead.pop(current)]
            sl = slice(current, current + batch_size)
            batch_y = [np.array(y) for y in self.labels[sl]] if self.labels is not None else None
            current += batch_size
            keep, ops, out_hw = [], [], None
            for i, x in enumerate(batch_X):
                labels = batch_y[i] if batch_y is not None else None
                if labels is not None and labels.size == 0 and not keep_images_without_gt:
                    continue                                       # no draws for an image without boxes
                o, owners, h, w = [], [], x.shape[0], x.shape[1]
                for k, t in enumerate(transformations):
                    o_t, h, w, labels = t.plan(h, w, labels)
                    o += o_t
                    owners += [k] * len(o_t)
                _check_photometric_prefix(o, transformations, owners)
                if out_hw is None:
                    out_hw = (h, w)
                elif out_hw != (h, w):
                    raise DegenerateBatchError('You produced an empty batch. This might be because the images in the batch vary in '
                                               'their size and/or number of channels. Note that after all transformations (if any '
                                               'were given) have been applied to all images in the batch, all images must be '
                                               'homogenous in size along all axes.')
                keep.append(i)
                ops.append(o)
            yield dict(images=batch_X, labels=batch_y, keep=keep, ops=ops, out_hw=out_hw,
                       filenames=list(self.filenames[sl]) if self.filenames is not None else None,
                       image_ids=list(self.image_ids[sl]) if self.image_ids is not None else None,
                       eval_neutral=list(self.eval_neutral[sl]) if self.eval_neutral is not None else None)

    def _shuffle(self):
        objects = [self.dataset_indices]
        for o in (self.filenames, self.labels, self.image_ids, self.eval_neutral):
            if o is not None:
                objects.append(o)
        shuffle_together(objects)

    def _fetch(self, pool, lo, batch_size):
        idx = self.dataset_indices[lo:lo + batch_size]
        if self.images is not None:
            return [self.images[i] for i in idx]
        names = self.filenames[lo:lo + batch_size]
        return [pool.submit(load_image, f) for f in names] if pool is not None else [load_image(f) for f in names]

    def _degenerate_check(self, batch_X, batch_y, keep, ops, handling, keep_images_without_gt, side):
        """The reference's check on the processed boxes (one read-back, see ``_read_boxes``): 'warn' warns, 'remove' filters the
        degenerate boxes and drops the images it empties (unless ``keep_images_without_gt``); the filter joins the image's op
        list."""
        gt, offs = _read_boxes([batch_y[i] for i in keep], ops, side)
        new_keep, new_ops = [], []
        for b, (i, o) in enumerate(zip(keep, ops)):
            labels = gt[offs[b]:offs[b + 1]]
            if _has_degenerate(labels, {'xmin': 1, 'ymin': 2, 'xmax': 3, 'ymax': 4}):
                if handling == 'warn':
                    warnings.warn('Detected degenerate ground truth bounding boxes for batch item {} with bounding boxes {}, i.e. '
                                  'bounding boxes where xmax <= xmin and/or ymax <= ymin.'.format(i, labels))
                else:
                    o = o + [ba.box_filter(check_degenerate=True)]
                    survivors = (labels[:, 3] > labels[:, 1]) & (labels[:, 4] > labels[:, 2])
                    if not survivors.any() and not keep_images_without_gt:
                        continue
            new_keep.append(i)
            new_ops.append(o)
        return new_keep, new_ops
