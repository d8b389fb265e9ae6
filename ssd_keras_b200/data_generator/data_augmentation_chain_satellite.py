"""``DataAugmentationSatellite`` (the reference's data_augmentation_chain_satellite.py), for images in bird's eye view, as a
planner for ``DataGenerator.generate``: brightness, contrast, saturation, hue, a horizontal and a vertical flip, a rotation by
90, 180 or 270 degrees, a ``RandomPatch`` that the ``ImageValidator`` accepts, then ``Resize`` with the degenerate /
minimum-area ``BoxFilter``.  The flips and the rotation move the labels the patch's validator reads, so the host carries them.

The rotation's border and the patch's pads are both black, as in the reference (which does not hand ``background`` to the
patch), so each list has one background colour.  Images without labels fail as in the reference (``AttributeError``)."""
from .data_augmentation_chain_variable_input_size import init_patch_chain, plan_patch_chain
from .object_detection_2d_geometric_ops import DEFAULT_LABELS_FORMAT, DevicePlanner, RandomFlip, RandomRotate


class DataAugmentationSatellite(DevicePlanner):
    """The satellite chain; the arguments are the reference's."""

    def __init__(self, resize_height, resize_width, random_brightness=(-48, 48, 0.5), random_contrast=(0.5, 1.8, 0.5),
                 random_saturation=(0.5, 1.8, 0.5), random_hue=(18, 0.5), random_flip=0.5, random_rotate=([90, 180, 270], 0.5),
                 min_scale=0.3, max_scale=2.0, min_aspect_ratio=0.8, max_aspect_ratio=1.25, n_trials_max=3, clip_boxes=True,
                 overlap_criterion='area', bounds_box_filter=(0.3, 1.0), bounds_validator=(0.5, 1.0), n_boxes_min=1, background=(0, 0, 0),
                 labels_format=DEFAULT_LABELS_FORMAT):
        init_patch_chain(self, resize_height, resize_width, random_brightness, random_contrast, random_saturation, random_hue,
                         random_flip, min_scale, max_scale, min_aspect_ratio, max_aspect_ratio, n_trials_max, clip_boxes,
                         overlap_criterion, bounds_box_filter, bounds_validator, n_boxes_min, background, labels_format)
        self.random_horizontal_flip = RandomFlip(dim='horizontal', prob=random_flip, labels_format=labels_format)
        self.random_vertical_flip = RandomFlip(dim='vertical', prob=random_flip, labels_format=labels_format)
        self.random_rotate = RandomRotate(angles=random_rotate[0], prob=random_rotate[1], labels_format=labels_format)
        self.geometric = [self.random_horizontal_flip, self.random_vertical_flip, self.random_rotate, self.random_patch, self.resize]

    def plan(self, img_height, img_width, labels):
        return plan_patch_chain(self, img_height, img_width, labels)
