"""NumPy restatement of the box half of the per-image op lists (``ssdk_assemble_batch``'s ``box_ops_kernel``), float64.

Each op is the label arithmetic of one reference class (paths relative to the reference root), in its order of operations:
  - ``CROP_PAD``  ``CropPad.__call__`` (data_generator/object_detection_2d_patch_sampling_ops.py:322-345): shift to the patch,
    optional 'center_point' filter, optional clip;
  - ``FLIP_H`` / ``FLIP_V``  ``Flip`` (data_generator/object_detection_2d_geometric_ops.py:171-195);
  - ``RESIZE``  ``Resize`` (:88-100): ``np.round(labels * (out / in))`` and the degenerate filter;
  - ``FILTER``  ``BoxFilter``'s degenerate and minimum-area tests (object_detection_2d_image_boxes_validation_utils.py:176-184);
  - ``TRANSLATE``  ``Translate`` (:276-317): ``+= dx_abs / dy_abs``;
  - ``SCALE`` / ``ROTATE``  ``Scale`` (:487-532) / ``Rotate`` (:681-737): both corners through ``np.dot(M, [x, y, 1])`` and
    ``np.round``, then ``Rotate``'s ymin / ymax and xmin / xmax swaps;
  - ``OVERLAP``  ``BoxFilter``'s overlap test (:186-230): 'center_point', 'area' (with the ``lower == 0`` -> ``>`` rule) or
    'iou' (``bounding_box_utils.iou``, whose intersection ignores ``border_pixels``: oracle/boxes.py);
  - ``CLIP``  the ``clip_boxes`` step of ``Translate`` / ``Scale`` / ``CropPad``.

``np.dot(M, corners)`` goes through BLAS.  With numpy's OpenBLAS 0.3.30 (Haswell kernels) the product is evaluated as
``(m0*x + m1*y) + m2`` with every product and sum rounded once: no fused multiply-add reaches the result, for one box or many.
For ``Scale``, ``m1*y`` (or ``m0*x``) is an exact zero, so a corner is ``round(f*x) + m2``, and when that sum cancels to an exact
``k + 0.5`` the half-even rounding of ``np.round`` sees the tie that a fused ``f*x + m2`` would not (tests/golden/
make_warp_golden.py holds such a corner, computed by the reference itself).  Rows are ``[class_id, xmin, ymin, xmax, ymax]``."""
import numpy as np

from . import boxes as _boxes
from . import warpops as _io

CRITERIA = ('center_point', 'area', 'iou')
BORDERS = ('half', 'include', 'exclude')


def _corners(M, lab):
    """Both corners of every box through M, as ``np.dot`` computes them, then ``np.round(...).astype(int)`` stored back into
    the float64 labels: a corner that rounds to -0 becomes +0 (``+ 0.0``).  A NaN or infinite corner has no integer, so its
    ``astype(int)`` is platform-defined; those keep the rounded float here."""
    x0, y0, x1, y1 = lab[:, 1], lab[:, 2], lab[:, 3], lab[:, 4]
    nx0 = (M[0, 0] * x0 + M[0, 1] * y0) + M[0, 2]
    ny0 = (M[1, 0] * x0 + M[1, 1] * y0) + M[1, 2]
    nx1 = (M[0, 0] * x1 + M[0, 1] * y1) + M[0, 2]
    ny1 = (M[1, 0] * x1 + M[1, 1] * y1) + M[1, 2]
    return np.round(nx0) + 0.0, np.round(ny0) + 0.0, np.round(nx1) + 0.0, np.round(ny1) + 0.0


def overlap_mask(lab, h, w, criterion, lower, upper, border_pixels='half'):
    """``BoxFilter``'s overlap test against an h x w image -> boolean mask."""
    x0, y0, x1, y1 = lab[:, 1], lab[:, 2], lab[:, 3], lab[:, 4]
    if criterion == 'center_point':
        cy, cx = (y0 + y1) / 2, (x0 + x1) / 2
        return (cy >= 0.0) & (cy <= h - 1) & (cx >= 0.0) & (cx <= w - 1)
    d = _boxes._BORDER_D[border_pixels]
    if criterion == 'iou':
        v = _boxes.iou(np.array([0, 0, w, h]), lab[:, 1:5], coords='corners', mode='element-wise', border_pixels=border_pixels)
        v = np.asarray(v).reshape(-1)
        return (v > lower) & (v <= upper)
    area = (x1 - x0 + d) * (y1 - y0 + d)
    inter = (np.clip(x1, 0, w - 1) - np.clip(x0, 0, w - 1) + d) * (np.clip(y1, 0, h - 1) - np.clip(y0, 0, h - 1) + d)
    lo = inter > lower * area if lower == 0.0 else inter >= lower * area
    return lo & (inter <= upper * area)


def apply_box_ops(labels, ops):
    """One image's label array through an op list -> float64 (k, 5), the surviving rows in their order."""
    lab = np.array(labels, dtype=np.float64).reshape(-1, 5)
    for o in ops:
        op, flags = int(o[0]), int(o[1]) & 0xFFFFFFFF
        a0, a1, a2, a3 = (float(v) for v in o[2:6])
        if op == _io.OP_END:
            break
        keep = None
        if op == _io.OP_CROP_PAD:
            lab[:, [2, 4]] -= a0
            lab[:, [1, 3]] -= a1
            if flags & 1:
                keep = overlap_mask(lab, a2, a3, 'center_point', 0, 1)
            if flags & 2:
                lab[:, [2, 4]] = np.clip(lab[:, [2, 4]], 0, a2 - 1)
                lab[:, [1, 3]] = np.clip(lab[:, [1, 3]], 0, a3 - 1)
        elif op == _io.OP_FLIP_H:
            lab[:, [1, 3]] = a0 - lab[:, [3, 1]]
        elif op == _io.OP_FLIP_V:
            lab[:, [2, 4]] = a0 - lab[:, [4, 2]]
        elif op == _io.OP_RESIZE:
            lab[:, [2, 4]] = np.round(lab[:, [2, 4]] * (a2 / a0))
            lab[:, [1, 3]] = np.round(lab[:, [1, 3]] * (a3 / a1))
            if flags & 1:
                keep = (lab[:, 3] > lab[:, 1]) & (lab[:, 4] > lab[:, 2])
        elif op == _io.OP_FILTER:
            keep = np.ones(lab.shape[0], bool)
            if flags & 1:
                keep &= (lab[:, 3] > lab[:, 1]) & (lab[:, 4] > lab[:, 2])
            if flags & 2:
                keep &= (lab[:, 3] - lab[:, 1]) * (lab[:, 4] - lab[:, 2]) >= a0
        elif op == _io.OP_TRANSLATE:
            lab[:, [1, 3]] += a1
            lab[:, [2, 4]] += a0
        elif op == _io.OP_SCALE:
            M = _io.rotation_matrix_2d((a2 / 2, a1 / 2), 0, a0)
            lab[:, 1], lab[:, 2], lab[:, 3], lab[:, 4] = _corners(M, lab)
        elif op == _io.OP_ROTATE and a0 in (90.0, 180.0, 270.0):    # other angles leave the boxes alone, as in ssdk.h
            angle = int(a0)
            M, _, _ = _io.rotate_geometry(int(a1), int(a2), angle)
            lab[:, 1], lab[:, 2], lab[:, 3], lab[:, 4] = _corners(M, lab)
            if angle in (90, 180):
                lab[:, [4, 2]] = lab[:, [2, 4]]
            if angle in (180, 270):
                lab[:, [3, 1]] = lab[:, [1, 3]]
        elif op == _io.OP_OVERLAP:
            keep = overlap_mask(lab, a2, a3, CRITERIA[flags & 3], a0, a1, BORDERS[(flags >> 2) & 3])
        elif op == _io.OP_CLIP:
            lab[:, [2, 4]] = np.clip(lab[:, [2, 4]], 0, a0 - 1)
            lab[:, [1, 3]] = np.clip(lab[:, [1, 3]], 0, a1 - 1)
        if keep is not None:
            lab = lab[keep]
    return lab
