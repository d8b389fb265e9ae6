"""``HistogramEqualization`` restated in NumPy without cv2: ``cv2.equalizeHist`` as OpenCV 4.13 computes it, and the op lists'
image half with ``EQUALIZE_V`` among the photometric ops.  What ``equalize_hist_kernel`` / ``equalize_lut_kernel`` and the
passes of ``photometric_kernel`` (csrc/batch.cu) must reproduce bit for bit; pinned to cv2 by tests/test_transformations_cpu.py.

OpenCV's table (histogram.cpp, ``equalizeHist``): ``i0`` is the first non-empty bin of the 256-bin histogram; if it holds every
pixel, the result is ``i0`` everywhere.  Otherwise ``scale = 255.f / (total - hist[i0])`` in float32, ``lut[i0] = 0`` and, for
``i > i0``, ``sum += hist[i]; lut[i] = saturate_cast<uchar>(sum * scale)``: the int sum converted to float32 (rounded, which
matters above 2^24 pixels), the float32 product, then rounded half to even."""
import numpy as np

from oracle import photoops as po

import resize_reference as rr

EQUALIZE_V = 26
PHOTO_CODES = po.PHOTO_CODES | {EQUALIZE_V}


def equalize_hist(channel):
    """uint8 ``cv2.equalizeHist`` of a 2-D uint8 array."""
    channel = np.asarray(channel)
    assert channel.dtype == np.uint8 and channel.ndim == 2
    hist = np.bincount(channel.ravel(), minlength=256).astype(np.int64)
    i0 = int(np.flatnonzero(hist)[0])
    total = channel.size
    if hist[i0] == total:
        return np.full_like(channel, i0)
    scale = np.float32(255.0) / np.float32(total - hist[i0])
    lut = np.zeros(256, np.uint8)
    sums = np.cumsum(hist[i0 + 1:]).astype(np.float32)
    lut[i0 + 1:] = np.clip(np.rint(sums * scale), 0, 255).astype(np.uint8)
    return lut[channel]


def apply_photo(image, ops):
    """``ConvertTo3Channels`` and the photometric ops of ``ops``, ``EQUALIZE_V`` included -> uint8 ``(h, w, 3)``."""
    x = po.to_3_channels(np.asarray(image))
    for o in ops:
        code = int(o[0])
        if code == EQUALIZE_V:
            assert x.dtype == np.uint8, 'cv2.equalizeHist takes 8-bit images only'
            x = x.copy()
            x[:, :, 2] = equalize_hist(np.ascontiguousarray(x[:, :, 2]))
        elif code in po.PHOTO_CODES:
            x = po.apply_op(x, o)
    assert x.dtype == np.uint8, 'the photometric ops must end in the uint8 state'
    return np.ascontiguousarray(x)


def apply_ops(image, ops):
    """The whole image half of an op list: the photometric prefix, then the geometric ops (``resize_reference.apply_ops``)."""
    rest = [o for o in ops if int(o[0]) not in PHOTO_CODES]
    return rr.apply_ops(apply_photo(image, ops), rest)


def apply_box_ops(labels, ops):
    return rr.apply_box_ops(labels, [o for o in ops if int(o[0]) != EQUALIZE_V])
