"""NumPy restatement of the image half of ``Translate`` / ``Scale`` / ``Rotate`` (paths relative to the reference root:
data_generator/object_detection_2d_geometric_ops.py:233-317, :449-532, :659-737), i.e. uint8 ``cv2.warpAffine`` with
``INTER_LINEAR`` and ``BORDER_CONSTANT``, with no cv2 dependency at run time, and ``apply_ops`` over the whole op list: the
crop / pad / flip / resize of oracle/imageops.py plus the new ops.

The warp follows the fixed-point scheme of OpenCV's ``modules/imgproc/src/imgwarp.cpp``:
  * the matrix ``M`` (``getRotationMatrix2D``: ``alpha = cos(a)*s``, ``beta = sin(a)*s`` with ``a = angle * (pi/180)``, the
    centre as float32) is inverted in float64 as ``invertAffineTransform`` does;
  * ``adelta[x] = rint(m0*x*1024)``, ``bdelta[x] = rint(m3*x*1024)``, ``X0 = rint((m1*y + m2)*1024) + 16``, likewise ``Y0``;
    ``X = (X0 + adelta[x]) >> 5``: source column ``X >> 5`` (saturated to int16), fraction ``X & 31``;
  * weights ``(32-fy)(32-fx)*32``, ``(32-fy)*fx*32``, ``fy*(32-fx)*32``, ``fy*fx*32`` (exact: they sum to 2^15), result
    ``(sum + 2^14) >> 15``; a tap outside the source reads the border colour.
``Translate`` passes a float32 integer matrix, so every sample has fraction 0: an integer shift with background.  ``Rotate``
by 90 / 180 / 270 degrees has ``cos`` of about 6e-17, which the fixed point rounds away: a signed axis permutation plus, where
the inverse map lands one pixel outside the source, a black line.  Bit-exact to OpenCV 4.13 (tests/test_warp_ops_cpu.py).

Op tuples are those of ``ssd_keras_b200.data_generator.batch_assembly``; ``TRANSLATE`` and ``SCALE`` keep the background R, G,
B in flag bits 8-31 like ``CROP_PAD``.  ``OVERLAP`` and ``CLIP``, like ``FILTER``, move boxes only."""
import math

import numpy as np

from .imageops import (INTER_LINEAR, INTER_NEAREST, OP_CROP_PAD, OP_END, OP_FILTER, OP_FLIP_H, OP_FLIP_V, OP_RESIZE,  # noqa: F401
                       background_of, crop_pad, flip, interpolation_of, resize, to3)

OP_TRANSLATE, OP_SCALE, OP_ROTATE, OP_OVERLAP, OP_CLIP = range(6, 11)


def rotation_matrix_2d(center, angle, scale):
    """``cv2.getRotationMatrix2D``: the centre is a ``Point2f``, the angle goes to radians as ``angle * (CV_PI/180)``."""
    cx, cy = float(np.float32(center[0])), float(np.float32(center[1]))
    a = float(angle) * (math.pi / 180)
    alpha, beta = math.cos(a) * scale, math.sin(a) * scale
    return np.array([[alpha, beta, (1 - alpha) * cx - beta * cy], [-beta, alpha, beta * cx + (1 - alpha) * cy]], np.float64)


def invert_affine(M):
    """``cv2.invertAffineTransform`` (and warpAffine's own inversion of a forward matrix), float64."""
    m = [float(v) for v in np.asarray(M, np.float64).reshape(6)]
    D = m[0] * m[4] - m[1] * m[3]
    D = 1.0 / D if D != 0 else 0.0
    a11, a22 = m[4] * D, m[0] * D
    m[0], m[1], m[3], m[4] = a11, m[1] * -D, m[3] * -D, a22
    b1 = -m[0] * m[2] - m[1] * m[5]
    b2 = -m[3] * m[2] - m[4] * m[5]
    m[2], m[5] = b1, b2
    return np.array(m, np.float64).reshape(2, 3)


def _sat_int(v):
    """saturate_cast<int>(double): round half to even, saturated to int32."""
    return np.clip(np.rint(v), -2 ** 31, 2 ** 31 - 1).astype(np.int64)


def warp_map(M, out_h, out_w):
    """cv2.warpAffine's fixed-point inverse map for INTER_LINEAR -> (sy, sx, fy, fx), each (out_h, out_w) int64."""
    m = invert_affine(M)
    x = np.arange(out_w, dtype=np.float64)
    y = np.arange(out_h, dtype=np.float64)
    adelta = _sat_int(m[0, 0] * x * 1024.0)
    bdelta = _sat_int(m[1, 0] * x * 1024.0)
    X0 = _sat_int((m[0, 1] * y + m[0, 2]) * 1024.0) + 16
    Y0 = _sat_int((m[1, 1] * y + m[1, 2]) * 1024.0) + 16
    X = (X0[:, None] + adelta[None, :]) >> 5
    Y = (Y0[:, None] + bdelta[None, :]) >> 5
    return np.clip(Y >> 5, -32768, 32767), np.clip(X >> 5, -32768, 32767), Y & 31, X & 31


def warp_affine(img, M, out_h, out_w, border=(0, 0, 0)):
    """uint8 ``cv2.warpAffine(img, M, (out_w, out_h), flags=INTER_LINEAR, borderMode=BORDER_CONSTANT, borderValue=border)``
    for (h,w,3) images."""
    h, w = img.shape[:2]
    sy, sx, fy, fx = warp_map(M, out_h, out_w)
    S = img.astype(np.int64)
    cval = np.asarray(border, np.int64)

    def tap(r, c):
        inside = (r >= 0) & (r < h) & (c >= 0) & (c < w)
        v = S[np.clip(r, 0, h - 1), np.clip(c, 0, w - 1)]
        return np.where(inside[..., None], v, cval)
    acc = (tap(sy, sx) * ((32 - fy) * (32 - fx) * 32)[..., None] + tap(sy, sx + 1) * ((32 - fy) * fx * 32)[..., None]
           + tap(sy + 1, sx) * (fy * (32 - fx) * 32)[..., None] + tap(sy + 1, sx + 1) * (fy * fx * 32)[..., None])
    v = (acc + (1 << 14)) >> 15
    outside = (sx >= w) | (sx + 1 < 0) | (sy >= h) | (sy + 1 < 0)
    v = np.where(outside[..., None], cval, v)
    return np.clip(v, 0, 255).astype(np.uint8)


def translate_matrix(dy_abs, dx_abs):
    """``Translate``'s matrix: float32, integer shifts."""
    return np.float32([[1, 0, dx_abs], [0, 1, dy_abs]]).astype(np.float64)


def rotate_geometry(h, w, angle):
    """``Rotate.__call__``'s matrix and output size: getRotationMatrix2D about the centre, then shifted to the new bounds."""
    M = rotation_matrix_2d((w / 2, h / 2), angle, 1)
    cos_a, sin_a = abs(M[0, 0]), abs(M[0, 1])
    w_new = int(h * sin_a + w * cos_a)
    h_new = int(h * cos_a + w * sin_a)
    M[1, 2] += (h_new - h) / 2
    M[0, 2] += (w_new - w) / 2
    return M, h_new, w_new


def translate(img, dy_abs, dx_abs, background=(0, 0, 0)):
    h, w = img.shape[:2]
    return warp_affine(img, translate_matrix(dy_abs, dx_abs), h, w, background)


def scale(img, factor, background=(0, 0, 0)):
    h, w = img.shape[:2]
    return warp_affine(img, rotation_matrix_2d((w / 2, h / 2), 0, factor), h, w, background)


def rotate(img, angle):
    h, w = img.shape[:2]
    M, h_new, w_new = rotate_geometry(h, w, angle)
    return warp_affine(img, M, h_new, w_new)


def apply_ops(img, ops):
    """One image through a list of op tuples -> (h,w,3) uint8, the composition the device evaluates."""
    img = to3(img)
    for o in ops:
        op, flags = int(o[0]), int(o[1])
        if op == OP_END:
            break
        if op == OP_CROP_PAD:
            img = crop_pad(img, int(o[2]), int(o[3]), int(o[4]), int(o[5]), background_of(flags))
        elif op == OP_FLIP_H:
            img = flip(img, 'horizontal')
        elif op == OP_FLIP_V:
            img = flip(img, 'vertical')
        elif op == OP_RESIZE:
            img = resize(img, int(o[4]), int(o[5]), interpolation_of(flags))
        elif op == OP_TRANSLATE:
            img = translate(img, int(o[2]), int(o[3]), background_of(flags))
        elif op == OP_SCALE:
            img = scale(img, float(o[2]), background_of(flags))
        elif op == OP_ROTATE:
            img = rotate(img, int(o[2]))
    return img
