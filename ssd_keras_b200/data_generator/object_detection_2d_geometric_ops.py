"""The geometric ops of the original SSD chain as planners for ``DataGenerator.generate``: ``Resize``, ``ResizeRandomInterp``
and ``RandomFlip`` (the reference's object_detection_2d_geometric_ops.py).  Each one draws what the reference draws, from the
global ``np.random`` in the same order, and returns the op records of ``batch_assembly`` that the device runs for it.

A planner's ``plan(img_height, img_width, labels)`` returns ``(ops, img_height, img_width, labels)``: the records, the image
size after them, and the host's copy of the labels where a later draw still depends on them (``None`` once the boxes are the
device's alone)."""
import numpy as np

from . import batch_assembly as ba

DEFAULT_LABELS_FORMAT = {'class_id': 0, 'xmin': 1, 'ymin': 2, 'xmax': 3, 'ymax': 4}


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


class RandomFlip(DevicePlanner):
    """``RandomFlip(dim, prob)``: flips when ``np.random.uniform(0, 1) >= 1 - prob``."""

    def __init__(self, dim='horizontal', prob=0.5, labels_format=DEFAULT_LABELS_FORMAT):
        if dim not in {'horizontal', 'vertical'}:
            raise ValueError("`dim` can be one of 'horizontal' and 'vertical'.")
        self.dim = dim
        self.prob = prob
        self.labels_format = labels_format

    def plan(self, img_height, img_width, labels):
        p = np.random.uniform(0, 1)
        if p >= (1.0 - self.prob):
            size = img_width if self.dim == 'horizontal' else img_height
            return [ba.flip(size, self.dim)], img_height, img_width, None
        return [], img_height, img_width, labels
