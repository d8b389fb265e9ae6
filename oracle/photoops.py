"""The photometric ops of the reference's training chains (``object_detection_2d_photometric_ops.py``), restated operation for
operation and dtype for dtype in NumPy, without cv2: what ``photometric_kernel`` (csrc/batch.cu) must reproduce bit for bit.
Pinned to the reference's own classes and to cv2 4.13 by ``tests/test_photo_ops_cpu.py``.

The parameters are values, not distributions: ``delta`` / ``factor`` are Python floats, so NumPy rounds them to float32 and
every intermediate stays float32 (``Brightness.__call__`` etc. on a float32 image).

The two uint8 ``cv2.cvtColor`` conversions as OpenCV 4.13's x86-64 wheel computes them on a CPU with AVX2 (its dispatched
path; found by exhaustive comparison over all 256^3 inputs, see DESIGN.md section 1):

- RGB -> HSV is integer code, the same for every pixel.
- HSV -> RGB is float32: ``s = S * (1/255)``, ``v = V * (1/255)``, ``h = H * (6/180)``, sector = trunc(h) mod 6, ``f = h - trunc(h)``,
  ``tab = {v, v * (1 - s), v * fma(-s, f, 1), v * fma(-s, 1 - f, 1)}`` -- the two inner ``1 - s * x`` are fused multiply-adds,
  everything else is rounded step by step -- then ``* 255``.  The last step depends on where the pixel lies in its row: the
  vector loop takes 32 pixels at a time and TRUNCATES, the scalar loop that finishes the row (columns
  ``>= width // 32 * 32``) ROUNDS half to even.  ``hsv2rgb`` therefore needs the image, not the pixel."""
import numpy as np

# ssdk_box_op_kind, photometric codes (include/ssdk.h)
TO_FLOAT32, TO_UINT8, BRIGHTNESS, CONTRAST, SATURATION, HUE, RGB2HSV, HSV2RGB, CHANNEL_SWAP = range(16, 25)
PHOTO_CODES = frozenset(range(16, 25))
HSV2RGB_VECTOR_PIXELS = 32

f32 = np.float32
_I = np.arange(1, 256, dtype=np.float64)
SDIV = np.concatenate([[0], np.rint((255 << 12) / _I)]).astype(np.int64)
HDIV = np.concatenate([[0], np.rint((180 << 12) / (6 * _I))]).astype(np.int64)


def to_3_channels(image):
    """``ConvertTo3Channels``."""
    if image.ndim == 2:
        return np.stack([image] * 3, axis=-1)
    if image.shape[2] == 1:
        return np.concatenate([image] * 3, axis=-1)
    return image[:, :, :3]


def fma32(a, b, c):
    """float32 fused multiply-add, exactly: the float32 product is exact in float64; the float64 sum is rounded to odd before
    the final rounding to float32, which removes the double rounding."""
    p = a.astype(np.float64) * b.astype(np.float64)
    c = c.astype(np.float64)
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)                  # TwoSum: p + c = s + err exactly
    bits = s.view(np.int64).copy()
    odd = (bits & 1) == 1
    fix = (err != 0) & ~odd                          # inexact and even: move one ulp towards the true sum
    up = fix & ((err > 0) == (s > 0))
    bits[up] += 1
    bits[fix & ~up] -= 1
    return bits.view(np.float64).astype(f32)


def rgb2hsv(image):
    """uint8 ``cv2.cvtColor(COLOR_RGB2HSV)`` (H in 0..179)."""
    r, g, b = (image[..., k].astype(np.int64) for k in range(3))
    v = np.maximum(np.maximum(r, g), b)
    d = v - np.minimum(np.minimum(r, g), b)
    s = (d * SDIV[v] + (1 << 11)) >> 12
    h = np.where(v == r, g - b, np.where(v == g, b - r + 2 * d, r - g + 4 * d))
    h = (h * HDIV[d] + (1 << 11)) >> 12
    h = h + np.where(h < 0, 180, 0)
    return np.stack([h, s, v], axis=-1).astype(np.uint8)


def hsv2rgb(image):
    """uint8 ``cv2.cvtColor(COLOR_HSV2RGB)`` of an ``(h, w, 3)`` image, any H in 0..255 (see the module docstring)."""
    H, S, V = (image[..., k].astype(f32) for k in range(3))
    s, v = S * f32(1.0 / 255.0), V * f32(1.0 / 255.0)
    h = H * f32(6.0 / 180.0)
    ps = np.trunc(h)
    f = h - ps
    sector = ps.astype(np.int64) % 6
    one = np.ones_like(v)
    tab = [v, v * (one - s), v * fma32(-s, f, one), v * fma32(-s, one - f, one)]
    pick = np.array([[0, 3, 1], [2, 0, 1], [1, 0, 3], [1, 2, 0], [3, 1, 0], [0, 1, 2]])      # sector -> tab index of R, G, B
    out = np.empty(image.shape, np.uint8)
    tail = np.broadcast_to(np.arange(image.shape[1]) >= image.shape[1] // HSV2RGB_VECTOR_PIXELS * HSV2RGB_VECTOR_PIXELS, v.shape)
    for k in range(3):
        x = np.choose(pick[sector, k], tab) * f32(255.0)
        out[..., k] = np.clip(np.where(tail, np.rint(x), np.trunc(x)), 0, 255).astype(np.uint8)
    return out


def apply_op(image, o):
    """One photometric op tuple ``(code, flags, a0, a1, a2, a3)`` on an ``(h, w, 3)`` image, as the reference class does it."""
    code, a0 = int(o[0]), o[2]
    if code == TO_FLOAT32:
        return image.astype(f32)
    if code == TO_UINT8:
        return np.round(image, decimals=0).astype(np.uint8)
    if code == BRIGHTNESS:
        return np.clip(image + float(a0), 0, 255)
    if code == CONTRAST:
        return np.clip(127.5 + float(a0) * (image - 127.5), 0, 255)
    if code == SATURATION:
        image = image.copy()
        image[:, :, 1] = np.clip(image[:, :, 1] * float(a0), 0, 255)
        return image
    if code == HUE:
        image = image.copy()
        image[:, :, 0] = (image[:, :, 0] + float(a0)) % 180.0
        return image
    if code == RGB2HSV:
        return rgb2hsv(image)
    if code == HSV2RGB:
        return hsv2rgb(image)
    if code == CHANNEL_SWAP:
        return image[:, :, [int(o[2]), int(o[3]), int(o[4])]]
    raise ValueError('not a photometric op: %r' % (o,))


def split_ops(ops):
    """An op list -> (its photometric ops, the rest in order)."""
    return [o for o in ops if int(o[0]) in PHOTO_CODES], [o for o in ops if int(o[0]) not in PHOTO_CODES]


def apply_ops(image, ops):
    """``ConvertTo3Channels`` and the photometric ops of ``ops`` (others are ignored) -> uint8 ``(h, w, 3)``."""
    x = to_3_channels(np.asarray(image))
    for o in split_ops(ops)[0]:
        x = apply_op(x, o)
    assert x.dtype == np.uint8, 'the photometric ops must end in the uint8 state'
    return np.ascontiguousarray(x)
