"""The original SSD training augmentation chain (the reference's data_augmentation_chain_original_ssd.py) as planners for
``DataGenerator.generate``: each object draws its random decisions from the global ``np.random``, in the number and order the
reference draws them, and returns the per-image op list that ``assemble_images_device`` / ``assemble_batch_device`` run.

The one decision that depends on the boxes is ``SSDRandomCrop``'s: ``RandomPatchInf`` retries patches until ``ImageValidator``
accepts one, so the number of draws an image consumes depends on its boxes.  The host therefore carries the labels through the
expansion (a shift) and evaluates the validator ('iou' against the patch, at least one box strictly above the drawn lower bound,
``border_pixels='half'``) in float64 NumPy, in the reference's expression order.  Everything else that happens to the boxes (the
crop's center-point filter and clip, the flip, the resize and its degenerate filter) and every pixel stays on the device."""
import numpy as np

from . import batch_assembly as ba
from .object_detection_2d_geometric_ops import DEFAULT_LABELS_FORMAT, DevicePlanner, RandomFlip, ResizeRandomInterp
from .object_detection_2d_image_boxes_validation_utils import iou_with_image

_DEGENERATE_ONLY = dict(check_overlap=False, check_min_area=False, check_degenerate=True)


def _expand_draws(img_height, img_width, min_scale, max_scale):
    """``PatchCoordinateGenerator(must_match='h_w', scale_uniformly=True)()``: one scale, then the two origins."""
    scaling_factor = np.random.uniform(min_scale, max_scale)
    patch_height = int(scaling_factor * img_height)
    patch_width = int(scaling_factor * img_width)
    return _origin(img_height, img_width, patch_height, patch_width)


def _crop_draws(img_height, img_width, min_scale, max_scale):
    """``PatchCoordinateGenerator(must_match='h_w', scale_uniformly=False)()``: height, width, then the two origins."""
    patch_height = int(np.random.uniform(min_scale, max_scale) * img_height)
    patch_width = int(np.random.uniform(min_scale, max_scale) * img_width)
    return _origin(img_height, img_width, patch_height, patch_width)


def _origin(img_height, img_width, patch_height, patch_width):
    y_range = img_height - patch_height
    patch_ymin = np.random.randint(0, y_range + 1) if y_range >= 0 else np.random.randint(y_range, 1)
    x_range = img_width - patch_width
    patch_xmin = np.random.randint(0, x_range + 1) if x_range >= 0 else np.random.randint(x_range, 1)
    return patch_ymin, patch_xmin, patch_height, patch_width


class SSDPhotometricDistortions(DevicePlanner):
    """Brightness, contrast, saturation and hue with probability 0.5 each in one of two orders, ``np.random.choice(2)``
    picking the order; ``RandomChannelSwap(prob=0.0)`` still draws its ``uniform``."""

    def plan(self, img_height, img_width, labels):
        sequence = 1 if np.random.choice(2) else 2

        def draw(lower, upper):                                # Random*: uniform against prob, then the parameter
            return np.random.uniform(lower, upper) if np.random.uniform(0, 1) >= 0.5 else None

        brightness = draw(-32, 32)
        contrast = draw(0.5, 1.5) if sequence == 1 else None
        saturation = draw(0.5, 1.5)
        hue = draw(-18, 18)
        if sequence == 2:
            contrast = draw(0.5, 1.5)
        np.random.uniform(0, 1)                                # RandomChannelSwap(prob=0.0): never swaps
        ops = ba.photometric_ops(sequence, brightness=brightness, contrast=contrast, saturation=saturation, hue=hue)
        return ops, img_height, img_width, labels


class SSDExpand(DevicePlanner):
    """``RandomPatch`` with probability 0.5: a canvas 1 to 4 times the image's size filled with ``background``, the image at
    a random place; boxes shifted, neither filtered nor clipped."""

    def __init__(self, background=(123, 117, 104), labels_format=DEFAULT_LABELS_FORMAT):
        self.background = background
        self.labels_format = labels_format

    def plan(self, img_height, img_width, labels):
        if not np.random.uniform(0, 1) >= (1.0 - 0.5):
            return [], img_height, img_width, labels
        patch_ymin, patch_xmin, patch_height, patch_width = _expand_draws(img_height, img_width, 1.0, 4.0)
        ops = ba.crop_pad_ops(patch_ymin, patch_xmin, patch_height, patch_width, clip_boxes=False, background=self.background)
        if labels is not None:
            fmt = self.labels_format
            labels = np.copy(labels)
            labels[:, [fmt['ymin'], fmt['ymax']]] -= patch_ymin
            labels[:, [fmt['xmin'], fmt['xmax']]] -= patch_xmin
        return ops, patch_height, patch_width, labels


class SSDRandomCrop(DevicePlanner):
    """``RandomPatchInf`` with probability 0.857 per round: a minimum IoU drawn from {none, 0.1, 0.3, 0.5, 0.7, 0.9}, then up
    to 50 patches of 0.3 to 1 times the image's sides with aspect ratio in [0.5, 2] until one overlaps a box by more than it;
    a round that finds none starts over.  The boxes whose centers lie in the patch are kept and clipped to it."""

    SAMPLE_SPACE = ((0.0, 1.0), (0.1, 1.0), (0.3, 1.0), (0.5, 1.0), (0.7, 1.0), (0.9, 1.0))

    def __init__(self, labels_format=DEFAULT_LABELS_FORMAT):
        self.labels_format = labels_format

    def _valid(self, labels, patch_ymin, patch_xmin, patch_height, patch_width, lower, upper):
        fmt = self.labels_format
        new_labels = np.copy(labels)
        new_labels[:, [fmt['ymin'], fmt['ymax']]] -= patch_ymin
        new_labels[:, [fmt['xmin'], fmt['xmax']]] -= patch_xmin
        ious = iou_with_image(new_labels[:, [fmt['xmin'], fmt['ymin'], fmt['xmax'], fmt['ymax']]], patch_height, patch_width)
        return np.count_nonzero((ious > lower) * (ious <= upper)) >= 1

    def plan(self, img_height, img_width, labels):
        n_bounds = len(self.SAMPLE_SPACE)
        while True:
            if not np.random.uniform(0, 1) >= (1.0 - 0.857):
                return [], img_height, img_width, labels
            lower, upper = self.SAMPLE_SPACE[np.random.choice(n_bounds, p=[1.0 / n_bounds] * n_bounds)]
            for _ in range(50):
                patch = _crop_draws(img_height, img_width, 0.3, 1.0)
                aspect_ratio = patch[3] / patch[2]
                if not (0.5 <= aspect_ratio <= 2.0):
                    continue
                if labels is None or self._valid(labels, *patch, lower, upper):
                    ops = ba.crop_pad_ops(*patch, box_filter=dict(check_overlap=True, check_min_area=False, check_degenerate=False,
                                                                  overlap_criterion='center_point'), clip_boxes=True)
                    return ops, patch[2], patch[3], None


class SSDDataAugmentation(DevicePlanner):
    """Photometric distortions, expand, random crop, random horizontal flip, then a resize to ``img_height x img_width`` with
    a random interpolation mode and the degenerate-box filter."""

    def __init__(self, img_height=300, img_width=300, background=(123, 117, 104), labels_format=DEFAULT_LABELS_FORMAT):
        self.labels_format = labels_format
        self.photometric_distortions = SSDPhotometricDistortions()
        self.expand = SSDExpand(background=background, labels_format=labels_format)
        self.random_crop = SSDRandomCrop(labels_format=labels_format)
        self.random_flip = RandomFlip(dim='horizontal', prob=0.5, labels_format=labels_format)
        self.resize = ResizeRandomInterp(height=img_height, width=img_width, interpolation_modes=[0, 1, 2, 3, 4],
                                         box_filter=_DEGENERATE_ONLY, labels_format=labels_format)
        self.sequence = [self.photometric_distortions, self.expand, self.random_crop, self.random_flip, self.resize]

    def plan(self, img_height, img_width, labels):
        for transform in self.sequence:
            transform.labels_format = self.labels_format
        ops = []
        for transform in self.sequence:
            o, img_height, img_width, labels = transform.plan(img_height, img_width, labels)
            ops += o
        return ops, img_height, img_width, labels
