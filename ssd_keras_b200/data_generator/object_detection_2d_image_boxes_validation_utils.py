"""``BoxFilter`` and ``ImageValidator`` (the reference's object_detection_2d_image_boxes_validation_utils.py) for the planners of
``DataGenerator.generate``.  They have two uses:

- on the host, a planner that retries (``RandomTranslate``, ``RandomScale``, ``RandomPatch``) asks ``ImageValidator`` about the
  moved boxes, and carries the labels through an accepted op's ``BoxFilter``, so that later draws see the boxes the reference
  sees.  Both evaluate the reference's expressions in its order, in the labels' own dtype (int64 from ``parse_csv``, or float);
- on the device, a ``BoxFilter`` is the spec of ``batch_assembly.box_filter_ops``.

Fixed bounds only: the reference's ``BoundGenerator`` (random bounds) is not supported."""
import numpy as np

DEFAULT_LABELS_FORMAT = {'class_id': 0, 'xmin': 1, 'ymin': 2, 'xmax': 3, 'ymax': 4}
_BORDER_D = {'half': 0, 'include': 1, 'exclude': -1}


def iou_with_image(boxes, image_height, image_width, border_pixels='half'):
    """``bounding_box_utils.iou(np.array([0, 0, w, h]), boxes, coords='corners', mode='element-wise', border_pixels)`` on the
    host, in the boxes' dtype: ``boxes`` is ``(k, 4)`` ``[xmin, ymin, xmax, ymax]``.  As there, the intersection ignores
    ``border_pixels`` and the areas do not."""
    image = np.array([[0, 0, image_width, image_height]])
    min_xy = np.maximum(image[:, [0, 1]], boxes[:, [0, 1]])
    max_xy = np.minimum(image[:, [2, 3]], boxes[:, [2, 3]])
    side_lengths = np.maximum(0, max_xy - min_xy)
    intersection = side_lengths[:, 0] * side_lengths[:, 1]
    d = _BORDER_D[border_pixels]
    image_area = (image[:, 2] - image[:, 0] + d) * (image[:, 3] - image[:, 1] + d)
    box_areas = (boxes[:, 2] - boxes[:, 0] + d) * (boxes[:, 3] - boxes[:, 1] + d)
    return intersection / (image_area + box_areas - intersection)


class BoxFilter:
    """Keeps the boxes that are non-degenerate, at least ``min_area`` large and overlap the image by ``overlap_bounds`` under
    ``overlap_criterion`` (each test as enabled)."""

    def __init__(self, check_overlap=True, check_min_area=True, check_degenerate=True, overlap_criterion='center_point',
                 overlap_bounds=(0.3, 1.0), min_area=16, labels_format=DEFAULT_LABELS_FORMAT, border_pixels='half'):
        if callable(overlap_bounds):
            raise NotImplementedError('random bounds (`BoundGenerator`) are not supported; pass a 2-tuple of scalars')
        if not isinstance(overlap_bounds, (list, tuple)):
            raise ValueError('`overlap_bounds` must be either a 2-tuple of scalars or a `BoundGenerator` object.')
        if overlap_bounds[0] > overlap_bounds[1]:
            raise ValueError('The lower bound must not be greater than the upper bound.')
        if overlap_criterion not in {'iou', 'area', 'center_point'}:
            raise ValueError("`overlap_criterion` must be one of 'iou', 'area', or 'center_point'.")
        self.overlap_criterion = overlap_criterion
        self.overlap_bounds = overlap_bounds
        self.min_area = min_area
        self.check_overlap = check_overlap
        self.check_min_area = check_min_area
        self.check_degenerate = check_degenerate
        self.labels_format = labels_format
        self.border_pixels = border_pixels

    def __call__(self, labels, image_height=None, image_width=None):
        """-> the rows of ``labels`` that pass, as the reference computes them (a copy, same dtype)."""
        labels = np.copy(labels)
        xmin, ymin, xmax, ymax = (self.labels_format[k] for k in ('xmin', 'ymin', 'xmax', 'ymax'))
        requirements_met = np.ones(shape=labels.shape[0], dtype=bool)
        if self.check_degenerate:
            requirements_met *= (labels[:, xmax] > labels[:, xmin]) * (labels[:, ymax] > labels[:, ymin])
        if self.check_min_area:
            requirements_met *= (labels[:, xmax] - labels[:, xmin]) * (labels[:, ymax] - labels[:, ymin]) >= self.min_area
        if self.check_overlap:
            lower, upper = self.overlap_bounds
            if self.overlap_criterion == 'iou':
                image_boxes_iou = iou_with_image(labels[:, [xmin, ymin, xmax, ymax]], image_height, image_width, self.border_pixels)
                requirements_met *= (image_boxes_iou > lower) * (image_boxes_iou <= upper)
            elif self.overlap_criterion == 'area':
                d = _BORDER_D[self.border_pixels]
                box_areas = (labels[:, xmax] - labels[:, xmin] + d) * (labels[:, ymax] - labels[:, ymin] + d)
                clipped_boxes = np.copy(labels)
                clipped_boxes[:, [ymin, ymax]] = np.clip(labels[:, [ymin, ymax]], a_min=0, a_max=image_height - 1)
                clipped_boxes[:, [xmin, xmax]] = np.clip(labels[:, [xmin, xmax]], a_min=0, a_max=image_width - 1)
                intersection_areas = ((clipped_boxes[:, xmax] - clipped_boxes[:, xmin] + d)
                                      * (clipped_boxes[:, ymax] - clipped_boxes[:, ymin] + d))
                if lower == 0.0:
                    mask_lower = intersection_areas > lower * box_areas
                else:
                    mask_lower = intersection_areas >= lower * box_areas
                requirements_met *= mask_lower * (intersection_areas <= upper * box_areas)
            else:
                cy = (labels[:, ymin] + labels[:, ymax]) / 2
                cx = (labels[:, xmin] + labels[:, xmax]) / 2
                requirements_met *= (cy >= 0.0) * (cy <= image_height - 1) * (cx >= 0.0) * (cx <= image_width - 1)
        return labels[requirements_met]


class ImageValidator:
    """An image is valid if at least ``n_boxes_min`` boxes (or ``'all'``) meet ``overlap_criterion`` within ``bounds``."""

    def __init__(self, overlap_criterion='center_point', bounds=(0.3, 1.0), n_boxes_min=1, labels_format=DEFAULT_LABELS_FORMAT,
                 border_pixels='half'):
        if not ((isinstance(n_boxes_min, int) and n_boxes_min > 0) or n_boxes_min == 'all'):
            raise ValueError("`n_boxes_min` must be a positive integer or 'all'.")
        self.overlap_criterion = overlap_criterion
        self.bounds = bounds
        self.n_boxes_min = n_boxes_min
        self.labels_format = labels_format
        self.border_pixels = border_pixels
        self.box_filter = BoxFilter(check_overlap=True, check_min_area=False, check_degenerate=False,
                                    overlap_criterion=self.overlap_criterion, overlap_bounds=self.bounds,
                                    labels_format=self.labels_format, border_pixels=self.border_pixels)

    def __call__(self, labels, image_height, image_width):
        self.box_filter.overlap_bounds = self.bounds
        self.box_filter.labels_format = self.labels_format
        valid_labels = self.box_filter(labels=labels, image_height=image_height, image_width=image_width)
        if isinstance(self.n_boxes_min, int):
            return len(valid_labels) >= self.n_boxes_min
        return len(valid_labels) == len(labels)
