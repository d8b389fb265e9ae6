"""The geometric ops as planners for ``DataGenerator.generate``: ``Resize``, ``ResizeRandomInterp``, ``Flip``, ``RandomFlip``,
``Translate``, ``RandomTranslate``, ``Scale``, ``RandomScale``, ``Rotate`` and ``RandomRotate`` (the reference's
object_detection_2d_geometric_ops.py), each random one built on its deterministic one, as there.  Each one draws what the
reference draws, from the global ``np.random`` in the same order (``RandomRotate``'s angle from Python's ``random``, as there),
and returns the op records of ``batch_assembly`` that the device runs for it.

A planner's ``plan(img_height, img_width, labels)`` returns ``(ops, img_height, img_width, labels)``: the records, the image
size after them, and the host's copy of the labels where a later draw still depends on them (``None`` once the boxes are the
device's alone).  Translate, Scale, Rotate and Flip carry the labels exactly as the reference leaves them, in the labels' own
dtype: a later ``ImageValidator`` (zoom in after a translation, a patch after a rotation) reads them.  Scale and Rotate move
each corner as ``(m0*x + m1*y) + m2``, every step rounded, then ``np.round`` and ``astype(int)``: the arithmetic of the
device's box ops and of the reference's ``np.dot`` with NumPy's OpenBLAS."""
import math
import random

import numpy as np

from . import batch_assembly as ba
from .object_detection_2d_image_boxes_validation_utils import BoxFilter, ImageValidator

DEFAULT_LABELS_FORMAT = {'class_id': 0, 'xmin': 1, 'ymin': 2, 'xmax': 3, 'ymax': 4}


def box_columns(fmt):
    return fmt['xmin'], fmt['ymin'], fmt['xmax'], fmt['ymax']


def check_box_filter(box_filter):
    """The reference's check on a ``box_filter`` argument (``Translate``, ``Scale``, ``CropPad``)."""
    if not (isinstance(box_filter, BoxFilter) or box_filter is None):
        raise ValueError("`box_filter` must be either `None` or a `BoxFilter` object.")


def check_image_validator(image_validator):
    if not (isinstance(image_validator, ImageValidator) or image_validator is None):
        raise ValueError("`image_validator` must be either `None` or an `ImageValidator` object.")


def filter_and_clip(labels, box_filter, clip_boxes, img_height, img_width, fmt):
    """The tail of ``Translate`` / ``Scale`` / ``CropPad.__call__`` on labels already in the new image's coordinates."""
    xmin, ymin, xmax, ymax = box_columns(fmt)
    if box_filter is not None:
        box_filter.labels_format = fmt
        labels = box_filter(labels=labels, image_height=img_height, image_width=img_width)
    if clip_boxes:
        labels[:, [ymin, ymax]] = np.clip(labels[:, [ymin, ymax]], a_min=0, a_max=img_height - 1)
        labels[:, [xmin, xmax]] = np.clip(labels[:, [xmin, xmax]], a_min=0, a_max=img_width - 1)
    return labels


def rotation_matrix_2d(center_x, center_y, angle, scale):
    """``cv2.getRotationMatrix2D((center_x, center_y), angle, scale)``: the centre is a ``Point2f``."""
    cx, cy = float(np.float32(center_x)), float(np.float32(center_y))
    a = float(angle) * (math.pi / 180)
    alpha, beta = math.cos(a) * scale, math.sin(a) * scale
    return ((alpha, beta, (1 - alpha) * cx - beta * cy), (-beta, alpha, beta * cx + (1 - alpha) * cy))


def rotate_geometry(img_height, img_width, angle):
    """``Rotate.__call__``'s matrix and output size."""
    (m0, m1, m2), (m3, m4, m5) = rotation_matrix_2d(img_width / 2, img_height / 2, angle, 1)
    cos_angle, sin_angle = abs(m0), abs(m1)
    img_width_new = int(img_height * sin_angle + img_width * cos_angle)
    img_height_new = int(img_height * cos_angle + img_width * sin_angle)
    m5 += (img_height_new - img_height) / 2
    m2 += (img_width_new - img_width) / 2
    return ((m0, m1, m2), (m3, m4, m5)), img_height_new, img_width_new


def move_corners(labels, M, fmt):
    """Both corners of every box through the 2 x 3 matrix ``M``, then ``np.round(...).astype(int)``, into a copy of ``labels``."""
    xmin, ymin, xmax, ymax = box_columns(fmt)
    (m0, m1, m2), (m3, m4, m5) = M
    out = np.copy(labels)
    for cx, cy in ((xmin, ymin), (xmax, ymax)):
        x, y = labels[:, cx].astype(np.float64), labels[:, cy].astype(np.float64)
        out[:, cx] = np.round((m0 * x + m1 * y) + m2).astype(int)
        out[:, cy] = np.round((m3 * x + m4 * y) + m5).astype(int)
    return out


class DevicePlanner:
    """Base of the planners: they describe work for the device and do not transform a NumPy image themselves."""

    def __call__(self, *args, **kwargs):
        raise TypeError('%s runs on the device: pass it to DataGenerator.generate(transformations=[...]) instead of calling it '
                        'on an image' % type(self).__name__)

    def plan(self, img_height, img_width, labels):
        raise NotImplementedError


class Resize(DevicePlanner):
    """``Resize(height, width, interpolation_mode, box_filter)``: the image to ``height x width`` with the cv2 code, the boxes
    scaled and rounded, then ``box_filter`` against the new size."""

    def __init__(self, height, width, interpolation_mode=1, box_filter=None, labels_format=DEFAULT_LABELS_FORMAT):
        self.out_height = height
        self.out_width = width
        self.interpolation_mode = interpolation_mode
        self.box_filter = box_filter
        self.labels_format = labels_format

    def plan(self, img_height, img_width, labels):
        ops = ([ba.resize_interp(img_height, img_width, self.out_height, self.out_width, self.interpolation_mode,
                                 drop_degenerate=False)] + ba.box_filter_ops(self.box_filter, self.out_height, self.out_width))
        return ops, self.out_height, self.out_width, None


class ResizeRandomInterp(DevicePlanner):
    """``Resize`` with the mode drawn by ``np.random.choice(interpolation_modes)``."""

    def __init__(self, height, width, interpolation_modes=(0, 1, 2, 3, 4), box_filter=None, labels_format=DEFAULT_LABELS_FORMAT):
        if not isinstance(interpolation_modes, (list, tuple)):
            raise ValueError('`interpolation_mode` must be a list or tuple.')
        self.height = height
        self.width = width
        self.interpolation_modes = interpolation_modes
        self.box_filter = box_filter
        self.labels_format = labels_format
        self.resize = Resize(height=height, width=width, box_filter=box_filter, labels_format=labels_format)

    def plan(self, img_height, img_width, labels):
        self.resize.interpolation_mode = np.random.choice(self.interpolation_modes)
        return self.resize.plan(img_height, img_width, labels)


class Flip(DevicePlanner):
    """``Flip(dim)``: the image mirrored horizontally or vertically, the boxes with it."""

    def __init__(self, dim='horizontal', labels_format=DEFAULT_LABELS_FORMAT):
        if dim not in {'horizontal', 'vertical'}:
            raise ValueError("`dim` can be one of 'horizontal' and 'vertical'.")
        self.dim = dim
        self.labels_format = labels_format

    def plan(self, img_height, img_width, labels):
        xmin, ymin, xmax, ymax = box_columns(self.labels_format)
        size = img_width if self.dim == 'horizontal' else img_height
        if labels is not None:
            labels = np.copy(labels)
            if self.dim == 'horizontal':
                labels[:, [xmin, xmax]] = img_width - labels[:, [xmax, xmin]]
            else:
                labels[:, [ymin, ymax]] = img_height - labels[:, [ymax, ymin]]
        return [ba.flip(size, self.dim)], img_height, img_width, labels


class RandomFlip(DevicePlanner):
    """``RandomFlip(dim, prob)``: ``Flip`` when ``np.random.uniform(0, 1) >= 1 - prob``."""

    def __init__(self, dim='horizontal', prob=0.5, labels_format=DEFAULT_LABELS_FORMAT):
        if dim not in {'horizontal', 'vertical'}:
            raise ValueError("`dim` can be one of 'horizontal' and 'vertical'.")
        self.dim = dim
        self.prob = prob
        self.labels_format = labels_format
        self.flip = Flip(dim=dim, labels_format=labels_format)

    def plan(self, img_height, img_width, labels):
        p = np.random.uniform(0, 1)
        if p >= (1.0 - self.prob):
            self.flip.labels_format = self.labels_format
            return self.flip.plan(img_height, img_width, labels)
        return [], img_height, img_width, labels


class Translate(DevicePlanner):
    """``Translate(dy, dx, clip_boxes, box_filter, background)``: a shift by ``int(round(h * dy))`` rows and
    ``int(round(w * dx))`` columns, then ``box_filter`` against the image and the clip."""

    def __init__(self, dy, dx, clip_boxes=True, box_filter=None, background=(0, 0, 0), labels_format=DEFAULT_LABELS_FORMAT):
        check_box_filter(box_filter)
        self.dy_rel = dy
        self.dx_rel = dx
        self.clip_boxes = clip_boxes
        self.box_filter = box_filter
        self.background = background
        self.labels_format = labels_format

    def plan(self, img_height, img_width, labels):
        ops = ba.translate_ops(img_height, img_width, self.dy_rel, self.dx_rel, self.box_filter, self.clip_boxes, self.background)
        if labels is not None:
            xmin, ymin, xmax, ymax = box_columns(self.labels_format)
            labels = np.copy(labels)
            labels[:, [xmin, xmax]] += int(round(img_width * self.dx_rel))
            labels[:, [ymin, ymax]] += int(round(img_height * self.dy_rel))
            labels = filter_and_clip(labels, self.box_filter, self.clip_boxes, img_height, img_width, self.labels_format)
        return ops, img_height, img_width, labels


class RandomTranslate(DevicePlanner):
    """``RandomTranslate``: with probability ``prob``, up to ``max(1, n_trials_max)`` shifts by a random fraction of the image
    size in a random direction until ``image_validator`` accepts the shifted boxes (before any filter or clip); the first
    accepted shift runs as ``Translate`` with ``box_filter``, ``clip_boxes`` and ``background``.  If every trial fails, the
    image is left unchanged."""

    def __init__(self, dy_minmax=(0.03, 0.3), dx_minmax=(0.03, 0.3), prob=0.5, clip_boxes=True, box_filter=None, image_validator=None,
                 n_trials_max=3, background=(0, 0, 0), labels_format=DEFAULT_LABELS_FORMAT):
        if dy_minmax[0] > dy_minmax[1]:
            raise ValueError("It must be `dy_minmax[0] <= dy_minmax[1]`.")
        if dx_minmax[0] > dx_minmax[1]:
            raise ValueError("It must be `dx_minmax[0] <= dx_minmax[1]`.")
        if dy_minmax[0] < 0 or dx_minmax[0] < 0:
            raise ValueError("It must be `dy_minmax[0] >= 0` and `dx_minmax[0] >= 0`.")
        check_image_validator(image_validator)
        self.dy_minmax = dy_minmax
        self.dx_minmax = dx_minmax
        self.prob = prob
        self.clip_boxes = clip_boxes
        self.box_filter = box_filter
        self.image_validator = image_validator
        self.n_trials_max = n_trials_max
        self.background = background
        self.labels_format = labels_format
        self.translate = Translate(dy=0, dx=0, clip_boxes=clip_boxes, box_filter=box_filter, background=background,
                                   labels_format=labels_format)

    def _translate(self, img_height, img_width, dy, dx, labels):
        self.translate.dy_rel, self.translate.dx_rel = dy, dx
        self.translate.labels_format = self.labels_format
        return self.translate.plan(img_height, img_width, labels)

    def plan(self, img_height, img_width, labels):
        if not np.random.uniform(0, 1) >= (1.0 - self.prob):
            return [], img_height, img_width, labels
        xmin, ymin, xmax, ymax = box_columns(self.labels_format)
        if self.image_validator is not None:
            self.image_validator.labels_format = self.labels_format
        for _ in range(max(1, self.n_trials_max)):
            dy_abs = np.random.uniform(self.dy_minmax[0], self.dy_minmax[1])
            dx_abs = np.random.uniform(self.dx_minmax[0], self.dx_minmax[1])
            dy = np.random.choice([-dy_abs, dy_abs])
            dx = np.random.choice([-dx_abs, dx_abs])
            if labels is None or self.image_validator is None:
                return self._translate(img_height, img_width, dy, dx, labels)
            new_labels = np.copy(labels)
            new_labels[:, [ymin, ymax]] += int(round(img_height * dy))
            new_labels[:, [xmin, xmax]] += int(round(img_width * dx))
            if self.image_validator(labels=new_labels, image_height=img_height, image_width=img_width):
                return self._translate(img_height, img_width, dy, dx, labels)
        return [], img_height, img_width, labels


class Scale(DevicePlanner):
    """``Scale(factor, clip_boxes, box_filter, background)``: a zoom by ``factor`` about the image centre, same output size,
    then ``box_filter`` against the image and the clip."""

    def __init__(self, factor, clip_boxes=True, box_filter=None, background=(0, 0, 0), labels_format=DEFAULT_LABELS_FORMAT):
        if factor <= 0:
            raise ValueError("It must be `factor > 0`.")
        check_box_filter(box_filter)
        self.factor = factor
        self.clip_boxes = clip_boxes
        self.box_filter = box_filter
        self.background = background
        self.labels_format = labels_format

    def plan(self, img_height, img_width, labels):
        ops = ba.scale_ops(img_height, img_width, self.factor, self.box_filter, self.clip_boxes, self.background)
        if labels is not None:
            M = rotation_matrix_2d(img_width / 2, img_height / 2, 0, self.factor)
            labels = filter_and_clip(move_corners(labels, M, self.labels_format), self.box_filter, self.clip_boxes, img_height,
                                     img_width, self.labels_format)
        return ops, img_height, img_width, labels


class RandomScale(DevicePlanner):
    """``RandomScale``: with probability ``prob``, up to ``max(1, n_trials_max)`` zoom factors in ``[min_factor, max_factor]``
    about the image centre until ``image_validator`` accepts the scaled boxes; the first accepted factor runs as ``Scale``.  If
    every trial fails, the image is left unchanged."""

    def __init__(self, min_factor=0.5, max_factor=1.5, prob=0.5, clip_boxes=True, box_filter=None, image_validator=None, n_trials_max=3,
                 background=(0, 0, 0), labels_format=DEFAULT_LABELS_FORMAT):
        if not (0 < min_factor <= max_factor):
            raise ValueError("It must be `0 < min_factor <= max_factor`.")
        check_image_validator(image_validator)
        self.min_factor = min_factor
        self.max_factor = max_factor
        self.prob = prob
        self.clip_boxes = clip_boxes
        self.box_filter = box_filter
        self.image_validator = image_validator
        self.n_trials_max = n_trials_max
        self.background = background
        self.labels_format = labels_format
        self.scale = Scale(factor=1.0, clip_boxes=clip_boxes, box_filter=box_filter, background=background, labels_format=labels_format)

    def _scale(self, img_height, img_width, factor, labels):
        self.scale.factor = factor
        self.scale.labels_format = self.labels_format
        return self.scale.plan(img_height, img_width, labels)

    def plan(self, img_height, img_width, labels):
        if not np.random.uniform(0, 1) >= (1.0 - self.prob):
            return [], img_height, img_width, labels
        if self.image_validator is not None:
            self.image_validator.labels_format = self.labels_format
        for _ in range(max(1, self.n_trials_max)):
            factor = np.random.uniform(self.min_factor, self.max_factor)
            if labels is None or self.image_validator is None:
                return self._scale(img_height, img_width, factor, labels)
            new_labels = move_corners(labels, rotation_matrix_2d(img_width / 2, img_height / 2, 0, factor), self.labels_format)
            if self.image_validator(labels=new_labels, image_height=img_height, image_width=img_width):
                return self._scale(img_height, img_width, factor, labels)
        return [], img_height, img_width, labels


class Rotate(DevicePlanner):
    """``Rotate(angle)``: counter-clockwise by 90, 180 or 270 degrees; the output is w x h for 90 and 270."""

    def __init__(self, angle, labels_format=DEFAULT_LABELS_FORMAT):
        if angle not in {90, 180, 270}:
            raise ValueError("`angle` must be in the set {90, 180, 270}.")
        self.angle = angle
        self.labels_format = labels_format

    def plan(self, img_height, img_width, labels):
        M, h_new, w_new = rotate_geometry(img_height, img_width, self.angle)
        if labels is not None:
            xmin, ymin, xmax, ymax = box_columns(self.labels_format)
            labels = move_corners(labels, M, self.labels_format)
            if self.angle in (90, 180):
                labels[:, [ymax, ymin]] = labels[:, [ymin, ymax]]
            if self.angle in (180, 270):
                labels[:, [xmax, xmin]] = labels[:, [xmin, xmax]]
        return ba.rotate_ops(img_height, img_width, self.angle), h_new, w_new, labels


class RandomRotate(DevicePlanner):
    """``RandomRotate``: with probability ``prob`` (``np.random``), ``Rotate`` by an angle drawn with Python's
    ``random.choice(angles)``."""

    def __init__(self, angles=(90, 180, 270), prob=0.5, labels_format=DEFAULT_LABELS_FORMAT):
        for angle in angles:
            if angle not in {90, 180, 270}:
                raise ValueError("`angles` can only contain the values 90, 180, and 270.")
        self.angles = list(angles)
        self.prob = prob
        self.labels_format = labels_format
        self.rotate = Rotate(angle=90, labels_format=labels_format)

    def plan(self, img_height, img_width, labels):
        if not np.random.uniform(0, 1) >= (1.0 - self.prob):
            return [], img_height, img_width, labels
        self.rotate.angle = random.choice(self.angles)
        self.rotate.labels_format = self.labels_format
        return self.rotate.plan(img_height, img_width, labels)
