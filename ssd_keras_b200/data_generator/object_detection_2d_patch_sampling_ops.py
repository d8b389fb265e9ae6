"""``PatchCoordinateGenerator`` and ``RandomPatch`` (the reference's object_detection_2d_patch_sampling_ops.py) as planners for
``DataGenerator.generate``: the patch is drawn on the host from the global ``np.random`` in the reference's order, and the
crop or pad runs on the device as one ``CROP_PAD`` record with its box filter and clip (``batch_assembly.crop_pad_ops``).

``RandomPatch(can_fail=True)``: when no patch passes the validator, the reference returns ``None`` for the image, and its
``generate()`` then fails on the missing labels.  There is nothing faithful to do with such an image, so the planner raises
``NotImplementedError`` in that case; a search that succeeds, and ``can_fail=False``, work as in the reference."""
import numpy as np

from . import batch_assembly as ba
from .object_detection_2d_geometric_ops import (DEFAULT_LABELS_FORMAT, DevicePlanner, box_columns, check_box_filter,
                                               check_image_validator, filter_and_clip)


class PatchCoordinateGenerator:
    """Random patch coordinates ``(ymin, xmin, height, width)``: two of height, width and aspect ratio drawn (``must_match``),
    the third derived, then the position so that the patch overlaps the image as much as it can.  Called with the image size
    set in ``img_height`` / ``img_width``, as ``RandomPatch`` does."""

    def __init__(self, img_height=None, img_width=None, must_match='h_w', min_scale=0.3, max_scale=1.0, scale_uniformly=False,
                 min_aspect_ratio=0.5, max_aspect_ratio=2.0, patch_ymin=None, patch_xmin=None, patch_height=None, patch_width=None,
                 patch_aspect_ratio=None):
        if must_match not in {'h_w', 'h_ar', 'w_ar'}:
            raise ValueError("`must_match` must be either of 'h_w', 'h_ar' and 'w_ar'.")
        if min_scale >= max_scale:
            raise ValueError("It must be `min_scale < max_scale`.")
        if min_aspect_ratio >= max_aspect_ratio:
            raise ValueError("It must be `min_aspect_ratio < max_aspect_ratio`.")
        if scale_uniformly and not ((patch_height is None) and (patch_width is None)):
            raise ValueError("If `scale_uniformly == True`, `patch_height` and `patch_width` must both be `None`.")
        self.img_height = img_height
        self.img_width = img_width
        self.must_match = must_match
        self.min_scale = min_scale
        self.max_scale = max_scale
        self.scale_uniformly = scale_uniformly
        self.min_aspect_ratio = min_aspect_ratio
        self.max_aspect_ratio = max_aspect_ratio
        self.patch_ymin = patch_ymin
        self.patch_xmin = patch_xmin
        self.patch_height = patch_height
        self.patch_width = patch_width
        self.patch_aspect_ratio = patch_aspect_ratio

    def _side(self, fixed, img_size):
        return int(np.random.uniform(self.min_scale, self.max_scale) * img_size) if fixed is None else fixed

    def _aspect_ratio(self):
        if self.patch_aspect_ratio is None:
            return np.random.uniform(self.min_aspect_ratio, self.max_aspect_ratio)
        return self.patch_aspect_ratio

    @staticmethod
    def _origin(fixed, img_size, patch_size):
        if fixed is not None:
            return fixed
        room = img_size - patch_size
        return np.random.randint(0, room + 1) if room >= 0 else np.random.randint(room, 1)

    def __call__(self):
        if self.must_match == 'h_w':
            if not self.scale_uniformly:
                patch_height = self._side(self.patch_height, self.img_height)
                patch_width = self._side(self.patch_width, self.img_width)
            else:
                scaling_factor = np.random.uniform(self.min_scale, self.max_scale)
                patch_height = int(scaling_factor * self.img_height)
                patch_width = int(scaling_factor * self.img_width)
        elif self.must_match == 'h_ar':
            patch_height = self._side(self.patch_height, self.img_height)
            patch_width = int(patch_height * self._aspect_ratio())
        else:
            patch_width = self._side(self.patch_width, self.img_width)
            patch_height = int(patch_width / self._aspect_ratio())
        patch_ymin = self._origin(self.patch_ymin, self.img_height, patch_height)
        patch_xmin = self._origin(self.patch_xmin, self.img_width, patch_width)
        return (patch_ymin, patch_xmin, patch_height, patch_width)


class RandomPatch(DevicePlanner):
    """``RandomPatch``: with probability ``prob``, up to ``max(1, n_trials_max)`` patches from ``patch_coord_generator`` until
    ``image_validator`` accepts the boxes in the patch's coordinates; the first accepted patch is cropped and / or padded with
    ``background``, its boxes filtered by ``box_filter`` against the patch and clipped.  If every trial fails, the image is left
    unchanged (``can_fail=False``) or ``NotImplementedError`` is raised (``can_fail=True``, see the module docstring)."""

    def __init__(self, patch_coord_generator, box_filter=None, image_validator=None, n_trials_max=3, clip_boxes=True, prob=1.0,
                 background=(0, 0, 0), can_fail=False, labels_format=DEFAULT_LABELS_FORMAT):
        if not isinstance(patch_coord_generator, PatchCoordinateGenerator):
            raise ValueError("`patch_coord_generator` must be an instance of `PatchCoordinateGenerator`.")
        check_image_validator(image_validator)
        check_box_filter(box_filter)
        self.patch_coord_generator = patch_coord_generator
        self.box_filter = box_filter
        self.image_validator = image_validator
        self.n_trials_max = n_trials_max
        self.clip_boxes = clip_boxes
        self.prob = prob
        self.background = background
        self.can_fail = can_fail
        self.labels_format = labels_format

    def _patch(self, patch_ymin, patch_xmin, patch_height, patch_width, labels):
        ops = ba.crop_pad_ops(patch_ymin, patch_xmin, patch_height, patch_width, self.box_filter, self.clip_boxes, self.background)
        if labels is not None:
            xmin, ymin, xmax, ymax = box_columns(self.labels_format)
            labels = np.copy(labels)
            labels[:, [ymin, ymax]] -= patch_ymin
            labels[:, [xmin, xmax]] -= patch_xmin
            labels = filter_and_clip(labels, self.box_filter, self.clip_boxes, patch_height, patch_width, self.labels_format)
        return ops, patch_height, patch_width, labels

    def plan(self, img_height, img_width, labels):
        if not np.random.uniform(0, 1) >= (1.0 - self.prob):
            return [], img_height, img_width, labels
        self.patch_coord_generator.img_height = img_height
        self.patch_coord_generator.img_width = img_width
        xmin, ymin, xmax, ymax = box_columns(self.labels_format)
        if self.image_validator is not None:
            self.image_validator.labels_format = self.labels_format
        for _ in range(max(1, self.n_trials_max)):
            patch_ymin, patch_xmin, patch_height, patch_width = self.patch_coord_generator()
            if labels is None or self.image_validator is None:
                return self._patch(patch_ymin, patch_xmin, patch_height, patch_width, labels)
            new_labels = np.copy(labels)
            new_labels[:, [ymin, ymax]] -= patch_ymin
            new_labels[:, [xmin, xmax]] -= patch_xmin
            if self.image_validator(labels=new_labels, image_height=patch_height, image_width=patch_width):
                return self._patch(patch_ymin, patch_xmin, patch_height, patch_width, labels)
        if self.can_fail:
            raise NotImplementedError('RandomPatch(can_fail=True) found no valid patch; dropping the image from its batch is not '
                                      'supported (use can_fail=False to keep the image unchanged)')
        return [], img_height, img_width, labels
