"""``PatchCoordinateGenerator``, ``CropPad``, ``Crop``, ``Pad``, ``RandomPatch``, ``RandomPatchInf``, ``RandomMaxCropFixedAR`` and
``RandomPadFixedAR`` (the reference's object_detection_2d_patch_sampling_ops.py) as planners for ``DataGenerator.generate``:
the patch is drawn on the host from the global ``np.random`` in the reference's order, and the crop or pad runs on the device
as one ``CROP_PAD`` record with its box filter and clip (``batch_assembly.crop_pad_ops``).  The random ones end in ``CropPad``,
and the two fixed-aspect-ratio ones are ``RandomPatch`` with a ``PatchCoordinateGenerator`` of fixed size, as there.

``RandomPatch(can_fail=True)``: when no patch passes the validator, the reference returns ``None`` for the image, and its
``generate()`` then fails on the missing labels.  There is nothing faithful to do with such an image, so the planner raises
``NotImplementedError`` in that case; a search that succeeds, and ``can_fail=False``, work as in the reference."""
import numpy as np

from . import batch_assembly as ba
from .object_detection_2d_geometric_ops import (DEFAULT_LABELS_FORMAT, DevicePlanner, box_columns, check_box_filter,
                                               check_image_validator, filter_and_clip)


def _sample(crop_pad, labels_format, img_height, img_width, patch, labels):
    """The random patch ops' last step: their ``CropPad`` with the patch ``(ymin, xmin, height, width)`` they drew."""
    crop_pad.patch_ymin, crop_pad.patch_xmin, crop_pad.patch_height, crop_pad.patch_width = patch
    crop_pad.labels_format = labels_format
    return crop_pad.plan(img_height, img_width, labels)


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


class CropPad(DevicePlanner):
    """``CropPad(patch_ymin, patch_xmin, patch_height, patch_width, clip_boxes, box_filter, background)``: the patch, which may
    reach outside the image (padded with ``background``), its boxes filtered by ``box_filter`` against the patch and clipped.
    Like the reference, a patch whose origin lies below or right of the image raises ``ValueError`` when planned."""

    def __init__(self, patch_ymin, patch_xmin, patch_height, patch_width, clip_boxes=True, box_filter=None, background=(0, 0, 0),
                 labels_format=DEFAULT_LABELS_FORMAT):
        check_box_filter(box_filter)
        self.patch_height = patch_height
        self.patch_width = patch_width
        self.patch_ymin = patch_ymin
        self.patch_xmin = patch_xmin
        self.clip_boxes = clip_boxes
        self.box_filter = box_filter
        self.background = background
        self.labels_format = labels_format

    def plan(self, img_height, img_width, labels):
        if (self.patch_ymin > img_height) or (self.patch_xmin > img_width):
            raise ValueError("The given patch doesn't overlap with the input image.")
        ops = ba.crop_pad_ops(self.patch_ymin, self.patch_xmin, self.patch_height, self.patch_width, self.box_filter, self.clip_boxes,
                              self.background)
        if labels is not None:
            xmin, ymin, xmax, ymax = box_columns(self.labels_format)
            labels = np.copy(labels)
            labels[:, [ymin, ymax]] -= self.patch_ymin
            labels[:, [xmin, xmax]] -= self.patch_xmin
            labels = filter_and_clip(labels, self.box_filter, self.clip_boxes, self.patch_height, self.patch_width, self.labels_format)
        return ops, self.patch_height, self.patch_width, labels


class Crop(DevicePlanner):
    """``Crop(crop_top, crop_bottom, crop_left, crop_right, clip_boxes, box_filter)``: ``CropPad`` of the image less the given
    borders."""

    def __init__(self, crop_top, crop_bottom, crop_left, crop_right, clip_boxes=True, box_filter=None, labels_format=DEFAULT_LABELS_FORMAT):
        self.crop_top = crop_top
        self.crop_bottom = crop_bottom
        self.crop_left = crop_left
        self.crop_right = crop_right
        self.clip_boxes = clip_boxes
        self.box_filter = box_filter
        self.labels_format = labels_format
        self.crop = CropPad(patch_ymin=crop_top, patch_xmin=crop_left, patch_height=None, patch_width=None, clip_boxes=clip_boxes,
                            box_filter=box_filter, labels_format=labels_format)

    def plan(self, img_height, img_width, labels):
        self.crop.patch_height = img_height - self.crop_top - self.crop_bottom
        self.crop.patch_width = img_width - self.crop_left - self.crop_right
        self.crop.labels_format = self.labels_format
        return self.crop.plan(img_height, img_width, labels)


class Pad(DevicePlanner):
    """``Pad(pad_top, pad_bottom, pad_left, pad_right, background)``: ``CropPad`` of the image with the given borders added,
    boxes neither filtered nor clipped."""

    def __init__(self, pad_top, pad_bottom, pad_left, pad_right, background=(0, 0, 0), labels_format=DEFAULT_LABELS_FORMAT):
        self.pad_top = pad_top
        self.pad_bottom = pad_bottom
        self.pad_left = pad_left
        self.pad_right = pad_right
        self.background = background
        self.labels_format = labels_format
        self.pad = CropPad(patch_ymin=-pad_top, patch_xmin=-pad_left, patch_height=None, patch_width=None, clip_boxes=False,
                           box_filter=None, background=background, labels_format=labels_format)

    def plan(self, img_height, img_width, labels):
        self.pad.patch_height = img_height + self.pad_top + self.pad_bottom
        self.pad.patch_width = img_width + self.pad_left + self.pad_right
        self.pad.labels_format = self.labels_format
        return self.pad.plan(img_height, img_width, labels)


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
        self.sample_patch = CropPad(patch_ymin=None, patch_xmin=None, patch_height=None, patch_width=None, clip_boxes=clip_boxes,
                                    box_filter=box_filter, background=background, labels_format=labels_format)


    def plan(self, img_height, img_width, labels):
        if not np.random.uniform(0, 1) >= (1.0 - self.prob):
            return [], img_height, img_width, labels
        self.patch_coord_generator.img_height = img_height
        self.patch_coord_generator.img_width = img_width
        xmin, ymin, xmax, ymax = box_columns(self.labels_format)
        if self.image_validator is not None:
            self.image_validator.labels_format = self.labels_format
        for _ in range(max(1, self.n_trials_max)):
            patch = patch_ymin, patch_xmin, patch_height, patch_width = self.patch_coord_generator()
            if labels is None or self.image_validator is None:
                return _sample(self.sample_patch, self.labels_format, img_height, img_width, patch, labels)
            new_labels = np.copy(labels)
            new_labels[:, [ymin, ymax]] -= patch_ymin
            new_labels[:, [xmin, xmax]] -= patch_xmin
            if self.image_validator(labels=new_labels, image_height=patch_height, image_width=patch_width):
                return _sample(self.sample_patch, self.labels_format, img_height, img_width, patch, labels)
        if self.can_fail:
            raise NotImplementedError('RandomPatch(can_fail=True) found no valid patch; dropping the image from its batch is not '
                                      'supported (use can_fail=False to keep the image unchanged)')
        return [], img_height, img_width, labels


class RandomPatchInf(DevicePlanner):
    """``RandomPatchInf``: until it returns, draws ``uniform(0, 1)`` against ``prob`` (a miss leaves the image unchanged), then
    up to ``max(1, n_trials_max)`` patches; a patch whose aspect ratio lies outside the generator's
    ``[min_aspect_ratio, max_aspect_ratio]`` is skipped, the first that ``image_validator`` accepts is sampled as ``RandomPatch``
    does.  Random validator bounds (``bound_generator``) are not supported."""

    def __init__(self, patch_coord_generator, box_filter=None, image_validator=None, bound_generator=None, n_trials_max=50,
                 clip_boxes=True, prob=0.857, background=(0, 0, 0), labels_format=DEFAULT_LABELS_FORMAT):
        if not isinstance(patch_coord_generator, PatchCoordinateGenerator):
            raise ValueError("`patch_coord_generator` must be an instance of `PatchCoordinateGenerator`.")
        check_image_validator(image_validator)
        if bound_generator is not None:
            raise NotImplementedError('random validator bounds (`BoundGenerator`) are not supported; pass `bound_generator=None`')
        self.patch_coord_generator = patch_coord_generator
        self.box_filter = box_filter
        self.image_validator = image_validator
        self.bound_generator = bound_generator
        self.n_trials_max = n_trials_max
        self.clip_boxes = clip_boxes
        self.prob = prob
        self.background = background
        self.labels_format = labels_format
        self.sample_patch = CropPad(patch_ymin=None, patch_xmin=None, patch_height=None, patch_width=None, clip_boxes=clip_boxes,
                                    box_filter=box_filter, background=background, labels_format=labels_format)

    def plan(self, img_height, img_width, labels):
        pcg = self.patch_coord_generator
        pcg.img_height = img_height
        pcg.img_width = img_width
        xmin, ymin, xmax, ymax = box_columns(self.labels_format)
        if self.image_validator is not None:
            self.image_validator.labels_format = self.labels_format
        while True:
            if not np.random.uniform(0, 1) >= (1.0 - self.prob):
                return [], img_height, img_width, labels
            for _ in range(max(1, self.n_trials_max)):
                patch = patch_ymin, patch_xmin, patch_height, patch_width = pcg()
                if not (pcg.min_aspect_ratio <= patch_width / patch_height <= pcg.max_aspect_ratio):
                    continue
                if labels is None or self.image_validator is None:
                    return _sample(self.sample_patch, self.labels_format, img_height, img_width, patch, labels)
                new_labels = np.copy(labels)
                new_labels[:, [ymin, ymax]] -= patch_ymin
                new_labels[:, [xmin, xmax]] -= patch_xmin
                if self.image_validator(labels=new_labels, image_height=patch_height, image_width=patch_width):
                    return _sample(self.sample_patch, self.labels_format, img_height, img_width, patch, labels)


class RandomMaxCropFixedAR(DevicePlanner):
    """``RandomMaxCropFixedAR(patch_aspect_ratio, ...)``: the largest patch of the given aspect ratio (``round``ed sides) at a
    random position: ``RandomPatch`` with a fixed-size ``PatchCoordinateGenerator(must_match='h_w')``, ``prob=1``,
    ``can_fail=False``."""

    def __init__(self, patch_aspect_ratio, box_filter=None, image_validator=None, n_trials_max=3, clip_boxes=True,
                 labels_format=DEFAULT_LABELS_FORMAT):
        self.patch_aspect_ratio = patch_aspect_ratio
        self.box_filter = box_filter
        self.image_validator = image_validator
        self.n_trials_max = n_trials_max
        self.clip_boxes = clip_boxes
        self.labels_format = labels_format
        self.random_patch = RandomPatch(patch_coord_generator=PatchCoordinateGenerator(), box_filter=box_filter,
                                        image_validator=image_validator, n_trials_max=n_trials_max, clip_boxes=clip_boxes, prob=1.0,
                                        can_fail=False, labels_format=labels_format)

    def plan(self, img_height, img_width, labels):
        if img_width / img_height < self.patch_aspect_ratio:
            patch_width = img_width
            patch_height = int(round(patch_width / self.patch_aspect_ratio))
        else:
            patch_height = img_height
            patch_width = int(round(patch_height * self.patch_aspect_ratio))
        self.random_patch.patch_coord_generator = PatchCoordinateGenerator(img_height=img_height, img_width=img_width, must_match='h_w',
                                                                           patch_height=patch_height, patch_width=patch_width)
        self.random_patch.labels_format = self.labels_format
        return self.random_patch.plan(img_height, img_width, labels)


class RandomPadFixedAR(DevicePlanner):
    """``RandomPadFixedAR(patch_aspect_ratio, background)``: the smallest patch of the given aspect ratio around the longer side
    of the image at a random position: ``RandomPatch`` with a fixed-size ``PatchCoordinateGenerator(must_match='h_w')``, no
    filter or clip, one trial."""

    def __init__(self, patch_aspect_ratio, background=(0, 0, 0), labels_format=DEFAULT_LABELS_FORMAT):
        self.patch_aspect_ratio = patch_aspect_ratio
        self.background = background
        self.labels_format = labels_format
        self.random_patch = RandomPatch(patch_coord_generator=PatchCoordinateGenerator(), box_filter=None, image_validator=None,
                                        n_trials_max=1, clip_boxes=False, background=background, prob=1.0, labels_format=labels_format)

    def plan(self, img_height, img_width, labels):
        if img_width < img_height:
            patch_height = img_height
            patch_width = int(round(patch_height * self.patch_aspect_ratio))
        else:
            patch_width = img_width
            patch_height = int(round(patch_width / self.patch_aspect_ratio))
        self.random_patch.patch_coord_generator = PatchCoordinateGenerator(img_height=img_height, img_width=img_width, must_match='h_w',
                                                                           patch_height=patch_height, patch_width=patch_width)
        self.random_patch.labels_format = self.labels_format
        return self.random_patch.plan(img_height, img_width, labels)
