"""``DataAugmentationVariableInputSize`` (the reference's data_augmentation_chain_variable_input_size.py) as a planner for
``DataGenerator.generate``: brightness, contrast, saturation, hue, a ``RandomPatch`` of random width and aspect ratio that the
``ImageValidator`` accepts, a horizontal flip, then ``Resize`` with the degenerate / minimum-area ``BoxFilter``.

Images without labels: the reference's ``__call__`` runs ``self.sequence1``, which this chain does not have, and fails with an
``AttributeError``; so does this planner."""
from .object_detection_2d_geometric_ops import DEFAULT_LABELS_FORMAT, DevicePlanner, RandomFlip, Resize
from .object_detection_2d_image_boxes_validation_utils import BoxFilter, ImageValidator
from .object_detection_2d_patch_sampling_ops import PatchCoordinateGenerator, RandomPatch
from .object_detection_2d_photometric_ops import (RandomBrightness, RandomContrast, RandomHue, RandomSaturation,
                                                  photometric_draws)


class DataAugmentationVariableInputSize(DevicePlanner):
    """The chain for images of any size, resized to ``resize_height x resize_width``; the arguments are the reference's."""

    def __init__(self, resize_height, resize_width, random_brightness=(-48, 48, 0.5), random_contrast=(0.5, 1.8, 0.5),
                 random_saturation=(0.5, 1.8, 0.5), random_hue=(18, 0.5), random_flip=0.5, min_scale=0.3, max_scale=2.0,
                 min_aspect_ratio=0.5, max_aspect_ratio=2.0, n_trials_max=3, clip_boxes=True, overlap_criterion='area',
                 bounds_box_filter=(0.3, 1.0), bounds_validator=(0.5, 1.0), n_boxes_min=1, background=(0, 0, 0),
                 labels_format=DEFAULT_LABELS_FORMAT):
        init_patch_chain(self, resize_height, resize_width, random_brightness, random_contrast, random_saturation, random_hue,
                         random_flip, min_scale, max_scale, min_aspect_ratio, max_aspect_ratio, n_trials_max, clip_boxes,
                         overlap_criterion, bounds_box_filter, bounds_validator, n_boxes_min, background, labels_format)
        self.random_flip = RandomFlip(dim='horizontal', prob=random_flip, labels_format=labels_format)
        self.geometric = [self.random_patch, self.random_flip, self.resize]

    def plan(self, img_height, img_width, labels):
        return plan_patch_chain(self, img_height, img_width, labels)


def init_patch_chain(chain, resize_height, resize_width, random_brightness, random_contrast, random_saturation, random_hue, random_flip,
                     min_scale, max_scale, min_aspect_ratio, max_aspect_ratio, n_trials_max, clip_boxes, overlap_criterion,
                     bounds_box_filter, bounds_validator, n_boxes_min, background, labels_format):
    """The parts the variable-input-size and satellite chains share, built as the reference builds them.  ``background`` is
    kept but, as in the reference, not handed to ``RandomPatch``: its pads are black."""
    chain.n_trials_max = n_trials_max
    chain.clip_boxes = clip_boxes
    chain.overlap_criterion = overlap_criterion
    chain.bounds_box_filter = bounds_box_filter
    chain.bounds_validator = bounds_validator
    chain.n_boxes_min = n_boxes_min
    chain.background = background
    chain.labels_format = labels_format
    chain.box_filter_patch = BoxFilter(check_overlap=True, check_min_area=False, check_degenerate=False,
                                       overlap_criterion=overlap_criterion, overlap_bounds=bounds_box_filter, labels_format=labels_format)
    chain.box_filter_resize = BoxFilter(check_overlap=False, check_min_area=True, check_degenerate=True, min_area=16,
                                        labels_format=labels_format)
    chain.image_validator = ImageValidator(overlap_criterion=overlap_criterion, bounds=bounds_validator, n_boxes_min=n_boxes_min,
                                           labels_format=labels_format)
    chain.resize = Resize(height=resize_height, width=resize_width, box_filter=chain.box_filter_resize, labels_format=labels_format)
    chain.random_brightness = RandomBrightness(lower=random_brightness[0], upper=random_brightness[1], prob=random_brightness[2])
    chain.random_contrast = RandomContrast(lower=random_contrast[0], upper=random_contrast[1], prob=random_contrast[2])
    chain.random_saturation = RandomSaturation(lower=random_saturation[0], upper=random_saturation[1], prob=random_saturation[2])
    chain.random_hue = RandomHue(max_delta=random_hue[0], prob=random_hue[1])
    chain.patch_coord_generator = PatchCoordinateGenerator(must_match='w_ar', min_scale=min_scale, max_scale=max_scale,
                                                           scale_uniformly=False, min_aspect_ratio=min_aspect_ratio,
                                                           max_aspect_ratio=max_aspect_ratio)
    chain.random_patch = RandomPatch(patch_coord_generator=chain.patch_coord_generator, box_filter=chain.box_filter_patch,
                                     image_validator=chain.image_validator, n_trials_max=n_trials_max, clip_boxes=clip_boxes, prob=1.0,
                                     can_fail=False, labels_format=labels_format)


def plan_patch_chain(chain, img_height, img_width, labels):
    """Photometric sequence 1, then ``chain.geometric`` in order."""
    if labels is None:                              # the reference's __call__ runs the missing self.sequence1 here
        raise AttributeError("'%s' object has no attribute 'sequence1' (the chain needs labels)" % type(chain).__name__)
    for transform in chain.geometric:
        transform.labels_format = chain.labels_format
    ops = photometric_draws(chain.random_brightness, chain.random_contrast, chain.random_saturation, chain.random_hue, 1)
    for transform in chain.geometric:
        o, img_height, img_width, labels = transform.plan(img_height, img_width, labels)
        ops += o
    return ops, img_height, img_width, None
