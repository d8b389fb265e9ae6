"""``DataAugmentationConstantInputSize`` (the reference's data_augmentation_chain_constant_input_size.py), the SSD7 training
chain, as a planner for ``DataGenerator.generate``.  ``np.random.choice(2)`` picks one of two sequences:

1. brightness, contrast, saturation, hue, then translate, zoom in (``RandomScale`` with factors in ``[1, max]``), flip;
2. brightness, saturation, hue, contrast, then zoom out (factors in ``[min, 1]``), translate, flip.

The translation and the zoom retry until ``ImageValidator`` accepts the moved boxes, so the host carries the labels through
the first of them into the second.  The image keeps its size, and the whole sequence is one op list on the device."""
import numpy as np

from .object_detection_2d_geometric_ops import DEFAULT_LABELS_FORMAT, DevicePlanner, RandomFlip, RandomScale, RandomTranslate
from .object_detection_2d_image_boxes_validation_utils import BoxFilter, ImageValidator
from .object_detection_2d_photometric_ops import (RandomBrightness, RandomContrast, RandomHue, RandomSaturation,
                                                  photometric_draws)


class DataAugmentationConstantInputSize(DevicePlanner):
    """The chain for constant-size images; the arguments are the reference's."""

    def __init__(self, random_brightness=(-48, 48, 0.5), random_contrast=(0.5, 1.8, 0.5), random_saturation=(0.5, 1.8, 0.5),
                 random_hue=(18, 0.5), random_flip=0.5, random_translate=((0.03, 0.5), (0.03, 0.5), 0.5), random_scale=(0.5, 2.0, 0.5),
                 n_trials_max=3, clip_boxes=True, overlap_criterion='area', bounds_box_filter=(0.3, 1.0), bounds_validator=(0.5, 1.0),
                 n_boxes_min=1, background=(0, 0, 0), labels_format=DEFAULT_LABELS_FORMAT):
        if (random_scale[0] >= 1) or (random_scale[1] <= 1):
            raise ValueError("This sequence of transformations only makes sense if the minimum scaling factor is <1 and the maximum "
                             "scaling factor is >1.")
        self.n_trials_max = n_trials_max
        self.clip_boxes = clip_boxes
        self.overlap_criterion = overlap_criterion
        self.bounds_box_filter = bounds_box_filter
        self.bounds_validator = bounds_validator
        self.n_boxes_min = n_boxes_min
        self.background = background
        self.labels_format = labels_format
        self.box_filter = BoxFilter(check_overlap=True, check_min_area=True, check_degenerate=True, overlap_criterion=overlap_criterion,
                                    overlap_bounds=bounds_box_filter, min_area=16, labels_format=labels_format)
        self.image_validator = ImageValidator(overlap_criterion=overlap_criterion, bounds=bounds_validator, n_boxes_min=n_boxes_min,
                                              labels_format=labels_format)
        self.random_brightness = RandomBrightness(lower=random_brightness[0], upper=random_brightness[1], prob=random_brightness[2])
        self.random_contrast = RandomContrast(lower=random_contrast[0], upper=random_contrast[1], prob=random_contrast[2])
        self.random_saturation = RandomSaturation(lower=random_saturation[0], upper=random_saturation[1], prob=random_saturation[2])
        self.random_hue = RandomHue(max_delta=random_hue[0], prob=random_hue[1])
        self.random_flip = RandomFlip(dim='horizontal', prob=random_flip, labels_format=labels_format)
        geometric = dict(clip_boxes=clip_boxes, box_filter=self.box_filter, image_validator=self.image_validator,
                         n_trials_max=n_trials_max, background=background, labels_format=labels_format)
        self.random_translate = RandomTranslate(dy_minmax=random_translate[0], dx_minmax=random_translate[1], prob=random_translate[2],
                                                **geometric)
        self.random_zoom_in = RandomScale(min_factor=1.0, max_factor=random_scale[1], prob=random_scale[2], **geometric)
        self.random_zoom_out = RandomScale(min_factor=random_scale[0], max_factor=1.0, prob=random_scale[2], **geometric)
        self.sequence1 = [self.random_translate, self.random_zoom_in, self.random_flip]
        self.sequence2 = [self.random_zoom_out, self.random_translate, self.random_flip]

    def plan(self, img_height, img_width, labels):
        for transform in (self.random_translate, self.random_zoom_in, self.random_zoom_out, self.random_flip):
            transform.labels_format = self.labels_format
        sequence = 1 if np.random.choice(2) else 2
        ops = photometric_draws(self.random_brightness, self.random_contrast, self.random_saturation, self.random_hue, sequence)
        first, second, flip = self.sequence1 if sequence == 1 else self.sequence2
        for transform in (first, second):
            o, img_height, img_width, labels = transform.plan(img_height, img_width, labels)
            ops += o
        o, img_height, img_width, _ = flip.plan(img_height, img_width, None)      # no later draw reads the labels
        return ops + o, img_height, img_width, None
