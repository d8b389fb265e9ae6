"""NumPy restatement of the image half of the reference's geometric augmentation ops, and of the uint8 ``cv2.resize`` they
call, with no cv2 dependency at run time.

What is restated (reference paths relative to the reference root):
  - ``ConvertTo3Channels`` (data_generator/object_detection_2d_photometric_ops.py:88-108): gray is replicated, RGBA drops
    alpha.  The device assembles 3-channel images, so this conversion is applied first, as both reference chains do.
  - the image half of ``CropPad`` (data_generator/object_detection_2d_patch_sampling_ops.py:266-313): a canvas of the patch
    size filled with the background colour, the overlapping part of the input copied in.
  - ``Flip`` (data_generator/object_detection_2d_geometric_ops.py:171-195): ``image[:, ::-1]`` / ``image[::-1]``.
  - ``Resize`` (:61-100), i.e. ``cv2.resize`` on uint8 images, for ``INTER_NEAREST`` (0) and ``INTER_LINEAR`` (1), in the
    scheme of OpenCV's source (``modules/imgproc/src/resize.cpp``):
      * equal sizes: a copy;
      * ``INTER_NEAREST``: ``sx = min(floor(dx * (1.0 / (out/in))), in-1)``, the scale in float64;
      * ``INTER_LINEAR`` with an exact 2x downscale in both axes: ``INTER_AREA``'s fast path, ``(a+b+c+d+2) >> 2``;
      * ``INTER_LINEAR`` otherwise: ``fx = float32((dx+0.5)*scale - 0.5)``, ``sx = floor(fx)``, ``fx -= sx`` (float32);
        columns with ``sx < 0`` or ``sx >= in-1`` take ``sx`` clamped and ``fx = 0``; rows keep ``fy`` and clamp the two
        source rows.  Coefficients are 11-bit fixed point, ``rint((1-f)*2048)`` and ``rint(f*2048)``.  The horizontal pass
        sums into int; the vertical pass is ``(((b0*(S0>>4))>>16) + ((b1*(S1>>4))>>16) + 2) >> 2`` (OpenCV's SIMD rule).
    The two axes are not treated alike at the borders: a column past either edge takes the edge pixel with weight 2048, but
    a row past either edge keeps its fraction and reads the edge row twice, which rounds differently in the vertical pass.
    With that asymmetry the restatement is bit-exact to uint8 ``cv2.resize`` of OpenCV 4.13 in both modes, on every size
    pair tested, one axis or both (tests/test_image_ops_cpu.py, DESIGN.md section 1).

Op lists are the tuples of ``ssd_keras_b200.data_generator.batch_assembly`` (``(op, flags, a0, a1, a2, a3)``); the image
fields live in flag bits the box kernel never reads: ``CROP_PAD`` bits 8-31 = background R, G, B; ``RESIZE`` bits 8-15 = the
cv2 interpolation code."""
import numpy as np

OP_END, OP_CROP_PAD, OP_FLIP_H, OP_FLIP_V, OP_RESIZE, OP_FILTER = range(6)
INTER_NEAREST, INTER_LINEAR = 0, 1


def to3(img):
    """``ConvertTo3Channels``: (h,w) / (h,w,1) / (h,w,3) / (h,w,4) uint8 -> (h,w,3) uint8."""
    img = np.asarray(img, dtype=np.uint8)
    if img.ndim == 2:
        return np.stack([img] * 3, axis=-1)
    if img.shape[2] == 1:
        return np.concatenate([img] * 3, axis=-1)
    if img.shape[2] == 4:
        return img[:, :, :3].copy()
    if img.shape[2] == 3:
        return img.copy()
    raise ValueError('images must have 1, 3 or 4 channels')


def crop_pad(img, py, px, ph, pw, background=(0, 0, 0)):
    """Image half of ``CropPad``: canvas pixel (r, c) shows input pixel (r+py, c+px) where that exists, else the background."""
    H, W = img.shape[:2]
    if py > H or px > W:
        raise ValueError("The given patch doesn't overlap with the input image.")
    canvas = np.empty((ph, pw, 3), np.uint8)
    canvas[:, :] = np.asarray(background, np.uint8)
    r0, r1 = max(0, -py), min(ph, H - py)
    c0, c1 = max(0, -px), min(pw, W - px)
    if r1 > r0 and c1 > c0:
        canvas[r0:r1, c0:c1] = img[r0 + py:r1 + py, c0 + px:c1 + px]
    return canvas


def flip(img, dim='horizontal'):
    return (img[:, ::-1] if dim == 'horizontal' else img[::-1]).copy()


def _nearest_index(n_in, n_out):
    ifx = 1.0 / (np.float64(n_out) / np.float64(n_in))
    return np.minimum(np.floor(np.arange(n_out, dtype=np.float64) * ifx).astype(np.int64), n_in - 1)


def _linear_coords(n_in, n_out):
    """-> (s, f) per output index: first source index (unclamped) and the float32 fraction, cv2's float arithmetic."""
    scale = 1.0 / (np.float64(n_out) / np.float64(n_in))
    f = ((np.arange(n_out, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    return s, f


def _coef(f):
    """saturate_cast<short>((1-f)*2048), saturate_cast<short>(f*2048): round half to even."""
    one = np.float32(1.0)
    c0 = np.rint((one - f).astype(np.float32) * np.float32(2048)).astype(np.int64)
    c1 = np.rint(f * np.float32(2048)).astype(np.int64)
    return c0, c1


def linear_tables(n_in, n_out, axis):
    """Taps and 11-bit coefficients of one axis: axis 'x' clamps the column and zeroes the fraction at the borders; axis 'y'
    keeps the fraction and clamps the two rows (resizeGeneric_)."""
    s, f = _linear_coords(n_in, n_out)
    if axis == 'x':
        lo = s < 0
        s = np.where(lo, 0, s); f = np.where(lo, np.float32(0), f).astype(np.float32)
        hi = s >= n_in - 1
        s = np.where(hi, n_in - 1, s); f = np.where(hi, np.float32(0), f).astype(np.float32)
        t0, t1 = s, np.minimum(s + 1, n_in - 1)
    else:
        t0, t1 = np.clip(s, 0, n_in - 1), np.clip(s + 1, 0, n_in - 1)
    c0, c1 = _coef(f)
    return t0, t1, c0, c1


def resize(img, out_h, out_w, interpolation=INTER_LINEAR):
    """uint8 ``cv2.resize(img, (out_w, out_h), interpolation)`` for (h,w,3) images, modes 0 and 1."""
    h, w = img.shape[:2]
    if (h, w) == (out_h, out_w):
        return img.copy()
    if interpolation == INTER_NEAREST:
        return img[_nearest_index(h, out_h)][:, _nearest_index(w, out_w)].copy()
    if interpolation != INTER_LINEAR:
        raise ValueError('unsupported interpolation mode %r' % (interpolation,))
    S = img.astype(np.int64)
    if h == 2 * out_h and w == 2 * out_w:
        return ((S[0::2, 0::2] + S[0::2, 1::2] + S[1::2, 0::2] + S[1::2, 1::2] + 2) >> 2).astype(np.uint8)
    x0, x1, a0, a1 = linear_tables(w, out_w, 'x')
    y0, y1, b0, b1 = linear_tables(h, out_h, 'y')
    D = S[:, x0] * a0[None, :, None] + S[:, x1] * a1[None, :, None]              # horizontal pass, int
    v = (((b0[:, None, None] * (D[y0] >> 4)) >> 16) + ((b1[:, None, None] * (D[y1] >> 4)) >> 16) + 2) >> 2
    return np.clip(v, 0, 255).astype(np.uint8)


def background_of(flags):
    f = int(flags) & 0xFFFFFFFF
    return ((f >> 8) & 255, (f >> 16) & 255, (f >> 24) & 255)


def interpolation_of(flags):
    return (int(flags) >> 8) & 255


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
    return img
