"""Batch assembly for the encoder on the device (SURVEY.md section 8f(3)).

In the reference, ``DataGenerator.generate`` (``data_generator/object_detection_2d_data_generator.py:830``) runs the augmentation
chain per image on the host -- image ops and, for every geometric op, the matching arithmetic on the label array -- filters
degenerate boxes (``:1095-1112``) and hands the list of label arrays to ``SSDInputEncoder.__call__`` (``:1146-1151``).
Here the label half runs on the GPU: ``assemble_batch_device`` uploads the ragged labels once (one pinned copy), applies a
per-image list of box operations (``ssdk_assemble_batch``: the label arithmetic of the reference's ``CropPad`` / ``Flip`` /
``Resize`` / ``BoxFilter``, with the parameters the caller's random augmentation logic picked) and leaves the packed
``(sum G_i, 5)`` rows + ``(B+1,)`` offsets on the device, which ``SSDInputEncoder.encode_device_offsets`` consumes without a
host round trip.

The image half of the same op lists runs on the device too (``assemble_images_device``, ``ssdk_assemble_images``), so that
one list moves the boxes and produces the image batch; ``assemble_training_batch`` returns both, ready for
``SSDTrainer.train_on_batch``.  Per image, in list order:

- ``ConvertTo3Channels`` first (gray is replicated, RGBA drops alpha), as both reference chains do;
- ``crop_pad(..., background=(r, g, b))``: the image half of ``CropPad`` (``patch_sampling_ops.py:266-313``); ``SSDExpand``
  pads with ``(123, 117, 104)``;
- ``flip(width_or_height, dim)``: ``Flip``;
- ``resize(..., interpolation_mode=1)``: uint8 ``cv2.resize`` with ``INTER_NEAREST`` (0) or ``INTER_LINEAR`` (1), bit-exact
  to OpenCV 4.13 (``oracle/imageops.py`` restates it); nothing that changes the image may follow it;
- ``resize_interp(..., interpolation_mode)``: the same step with every mode ``ResizeRandomInterp`` draws, ``INTER_CUBIC`` (2),
  ``INTER_AREA`` (3) and ``INTER_LANCZOS4`` (4) too, bit-exact to OpenCV 4.13's own resize code (``tests/resize_reference.py``
  restates the three); its boxes are ``resize``'s;
- ``translate`` / ``scale`` / ``rotate``: ``Translate`` / ``Scale`` / ``Rotate`` (``geometric_ops.py:233-737``), uint8
  ``cv2.warpAffine`` with ``INTER_LINEAR`` and ``BORDER_CONSTANT``, bit-exact to OpenCV 4.13.  ``translate`` and ``rotate``
  (90 / 180 / 270) are exact integer maps; ``scale`` is a bilinear warp.  A list holds at most one resampling step
  (``resize`` or ``scale``); crops, pads, flips, translations and rotations may come before it, and after a ``scale`` too.
  One background colour per list: pads, translations and scales that bring in background must agree, and a rotation's
  border is black;
- ``box_filter``, ``overlap_filter``, ``clip``: boxes only;
- the photometric ops (``convert_dtype``, ``brightness``, ``contrast``, ``saturation``, ``hue``, ``convert_color``,
  ``channel_swap``, ``equalize_hist``; ``object_detection_2d_photometric_ops.py``) come before every geometric op, as in all
  three training chains, and run as a uint8 pre-pass on the device, bit-exact to NumPy and to OpenCV 4.13's uint8
  ``cv2.cvtColor`` on a CPU with AVX2 (``oracle/photoops.py`` restates them) and ``cv2.equalizeHist``
  (``tests/equalize_reference.py``).  ``photometric_ops`` returns ``SSDPhotometricDistortions``' two sequences.

``translate_ops`` / ``scale_ops`` / ``rotate_ops`` / ``crop_pad_ops`` / ``resize_ops`` / ``box_filter_ops`` return the whole op
sequence one call of the reference class runs, box filter and clipping included, so the geometric halves of
``DataAugmentationConstantInputSize`` (SSD7: translate -> zoom in -> flip, or zoom out -> translate -> flip) and
``DataAugmentationSatellite`` (flips -> rotate -> patch -> resize) are one op list per image.

Not covered: ``Gamma`` (the reference's raises), conversion to GRAY, a second resampling step, JPEG decoding.  The random decisions of a chain (which patch, flip or not, which factor, which photometric op with which delta) are
the caller's: the planners of ``data_augmentation_chain_original_ssd``, ``_constant_input_size`` (SSD7), ``_variable_input_size``
and ``_satellite`` draw them in the reference's order, and ``DataGenerator.generate`` runs them."""
import ctypes as C

import numpy as np

from .. import _ffi


def _int32(v):
    """An unsigned 32-bit flag word as the C struct's signed ``int``."""
    return v - (1 << 32) if v >= (1 << 31) else v


def crop_pad(patch_ymin, patch_xmin, patch_height, patch_width, center_point_filter=False, clip_boxes=True, background=(0, 0, 0)):
    """``CropPad`` (patch_sampling_ops.py:266-330).  ``SSDExpand``: negative origin, no filter, no clip, ``background=(123, 117,
    104)``; ``SSDRandomCrop``: ``center_point_filter=True, clip_boxes=True``.  ``background`` (R, G, B) goes to flag bits 8-31."""
    bg = tuple(int(v) for v in background)
    if len(bg) != 3 or any(v < 0 or v > 255 for v in bg):
        raise ValueError('`background` must be three integers in [0, 255]')
    flags = (1 if center_point_filter else 0) | (2 if clip_boxes else 0) | (bg[0] << 8) | (bg[1] << 16) | (bg[2] << 24)
    return (_ffi.BOXOP_CROP_PAD, _int32(flags), float(patch_ymin), float(patch_xmin), float(patch_height), float(patch_width))


def flip(img_size, dim='horizontal'):
    """``Flip`` (geometric_ops.py:186,194): ``img_size`` is the image width (horizontal) or height (vertical)."""
    if dim not in ('horizontal', 'vertical'):
        raise ValueError("`dim` can be one of 'horizontal' and 'vertical'.")
    return (_ffi.BOXOP_FLIP_H if dim == 'horizontal' else _ffi.BOXOP_FLIP_V, 0, float(img_size), 0.0, 0.0, 0.0)


def resize(in_height, in_width, out_height, out_width, drop_degenerate=True, interpolation_mode=_ffi.INTER_LINEAR):
    """``Resize`` (geometric_ops.py:61-100) with its degenerate-box ``BoxFilter``.  ``interpolation_mode`` is the cv2 code
    (``Resize``'s default ``cv2.INTER_LINEAR`` = 1; the images support 0 and 1), kept in flag bits 8-15."""
    mode = int(interpolation_mode)
    if not 0 <= mode <= 255:
        raise ValueError('`interpolation_mode` must be a cv2 interpolation code')
    return (_ffi.BOXOP_RESIZE, (1 if drop_degenerate else 0) | (mode << 8), float(in_height), float(in_width), float(out_height),
            float(out_width))


def resize_interp(in_height, in_width, out_height, out_width, interpolation_mode, drop_degenerate=True):
    """``Resize`` with any of the five cv2 codes ``ResizeRandomInterp`` draws from: ``INTER_NEAREST`` (0), ``INTER_LINEAR`` (1),
    ``INTER_CUBIC`` (2), ``INTER_AREA`` (3), ``INTER_LANCZOS4`` (4).  The boxes are ``resize``'s."""
    mode = int(interpolation_mode)
    if not 0 <= mode <= 4:
        raise ValueError('`interpolation_mode` must be one of the cv2 codes 0-4')
    return (_ffi.BOXOP_RESIZE_INTERP, (1 if drop_degenerate else 0) | (mode << 8), float(in_height), float(in_width),
            float(out_height), float(out_width))


def box_filter(check_degenerate=True, min_area=None):
    """``BoxFilter`` without the overlap test (validation_utils.py:155-165); also ``degenerate_box_handling='remove'``."""
    return (_ffi.BOXOP_FILTER, (1 if check_degenerate else 0) | (2 if min_area is not None else 0), float(min_area or 0.0), 0.0, 0.0, 0.0)


def _colour(background):
    bg = tuple(int(v) for v in background)
    if len(bg) != 3 or any(v < 0 or v > 255 for v in bg):
        raise ValueError('`background` must be three integers in [0, 255]')
    return (bg[0] << 8) | (bg[1] << 16) | (bg[2] << 24)


def translate(img_height, img_width, dy, dx, background=(0, 0, 0)):
    """``Translate`` (geometric_ops.py:276-304): ``dy`` / ``dx`` are fractions of the image height / width; the shifts are
    ``int(round(h*dy))`` / ``int(round(w*dx))`` as there.  ``background`` (R, G, B) goes to flag bits 8-31."""
    h, w = int(img_height), int(img_width)
    return (_ffi.BOXOP_TRANSLATE, _int32(_colour(background)), float(int(round(h * dy))), float(int(round(w * dx))), float(h), float(w))


def scale(img_height, img_width, factor, background=(0, 0, 0)):
    """``Scale`` (geometric_ops.py:487-519): zoom by ``factor`` about the image centre, same output size."""
    if not factor > 0:
        raise ValueError('It must be `factor > 0`.')
    return (_ffi.BOXOP_SCALE, _int32(_colour(background)), float(factor), float(img_height), float(img_width), 0.0)


def rotate(img_height, img_width, angle):
    """``Rotate`` (geometric_ops.py:681-737): counter-clockwise by 90, 180 or 270 degrees; the output is w x h for 90 / 270."""
    if angle not in {90, 180, 270}:
        raise ValueError('`angle` must be in the set {90, 180, 270}.')
    return (_ffi.BOXOP_ROTATE, 0, float(angle), float(img_height), float(img_width), 0.0)


_CRITERIA = {'center_point': 0, 'area': 1, 'iou': 2}
_BORDERS = {'half': 0, 'include': 1, 'exclude': 2}


def overlap_filter(img_height, img_width, overlap_criterion='center_point', overlap_bounds=(0.3, 1.0), border_pixels='half'):
    """``BoxFilter``'s overlap test (validation_utils.py:186-230) against an ``img_height x img_width`` image."""
    if overlap_criterion not in _CRITERIA:
        raise ValueError("`overlap_criterion` must be one of 'iou', 'area', or 'center_point'.")
    if border_pixels not in _BORDERS:
        raise ValueError("`border_pixels` must be one of 'half', 'include', or 'exclude'.")
    lower, upper = (float(v) for v in overlap_bounds)
    if lower > upper:
        raise ValueError('The lower bound must not be greater than the upper bound.')
    return (_ffi.BOXOP_OVERLAP, _CRITERIA[overlap_criterion] | (_BORDERS[border_pixels] << 2), lower, upper, float(img_height),
            float(img_width))


def clip(img_height, img_width):
    """``clip_boxes``: boxes clipped to ``[0, h-1] x [0, w-1]``."""
    return (_ffi.BOXOP_CLIP, 0, float(img_height), float(img_width), 0.0, 0.0)


def convert_dtype(to='uint8'):
    """``ConvertDataType`` (photometric_ops.py:62-86): ``astype(float32)``, or ``np.round`` and ``astype(uint8)``."""
    if to not in ('uint8', 'float32'):
        raise ValueError("`to` can be either of 'uint8' or 'float32'.")
    return (_ffi.BOXOP_TO_UINT8 if to == 'uint8' else _ffi.BOXOP_TO_FLOAT32, 0, 0.0, 0.0, 0.0, 0.0)


def brightness(delta):
    """``Brightness`` (:225-246) on a float32 image; ``delta`` is rounded to float32, as NumPy does with a Python float."""
    return (_ffi.BOXOP_BRIGHTNESS, 0, float(delta), 0.0, 0.0, 0.0)


def contrast(factor):
    """``Contrast`` (:281-304) on a float32 image."""
    if factor <= 0.0:
        raise ValueError('It must be `factor > 0`.')
    return (_ffi.BOXOP_CONTRAST, 0, float(factor), 0.0, 0.0, 0.0)


def saturation(factor):
    """``Saturation`` (:166-189) on a float32 HSV image."""
    if factor <= 0.0:
        raise ValueError('It must be `factor > 0`.')
    return (_ffi.BOXOP_SATURATION, 0, float(factor), 0.0, 0.0, 0.0)


def hue(delta):
    """``Hue`` (:110-133) on a float32 HSV image (H in [0, 180])."""
    if not (-180 <= delta <= 180):
        raise ValueError('`delta` must be in the closed interval `[-180, 180]`.')
    return (_ffi.BOXOP_HUE, 0, float(delta), 0.0, 0.0, 0.0)


def convert_color(current='RGB', to='HSV'):
    """``ConvertColor`` (:23-60) between RGB and HSV on a uint8 image; the GRAY targets are not supported."""
    if not ((current == 'RGB' and to == 'HSV') or (current == 'HSV' and to == 'RGB')):
        raise NotImplementedError
    return (_ffi.BOXOP_RGB2HSV if to == 'HSV' else _ffi.BOXOP_HSV2RGB, 0, 0.0, 0.0, 0.0, 0.0)


def channel_swap(order):
    """``ChannelSwap`` (:438-455): ``image[:, :, order]``."""
    order = tuple(int(v) for v in order)
    if sorted(order) != [0, 1, 2]:
        raise ValueError('`order` must be a permutation of (0, 1, 2)')
    return (_ffi.BOXOP_CHANNEL_SWAP, 0, float(order[0]), float(order[1]), float(order[2]), 0.0)


def equalize_hist():
    """``HistogramEqualization`` (photometric_ops.py:397-411): ``image[:, :, 2] = cv2.equalizeHist(image[:, :, 2])`` on a uint8
    image (HSV in the reference's intent; nothing checks it), OpenCV 4.13's table bit for bit."""
    return (_ffi.BOXOP_EQUALIZE_V, 0, 0.0, 0.0, 0.0, 0.0)


def photometric_ops(sequence, brightness=None, contrast=None, saturation=None, hue=None, channel_swap=None):
    """The op list of ``SSDPhotometricDistortions.sequence1`` / ``sequence2`` (data_augmentation_chain_original_ssd.py:165-191;
    also the photometric part of ``DataAugmentationConstantInputSize``'s sequences) for ``sequence`` 1 or 2, with the values the
    caller drew; an op whose argument is ``None`` (its draw skipped it) is left out, the conversions stay as the reference
    keeps them.  Prepend it to the geometric ops of the image."""
    if sequence not in (1, 2):
        raise ValueError('`sequence` must be 1 or 2')
    g = globals()
    f32, u8 = convert_dtype('float32'), convert_dtype('uint8')
    b = [g['brightness'](brightness)] if brightness is not None else []
    c = [g['contrast'](contrast)] if contrast is not None else []
    hsv = ([convert_color('RGB', 'HSV'), f32] + ([g['saturation'](saturation)] if saturation is not None else [])
           + ([g['hue'](hue)] if hue is not None else []) + [u8, convert_color('HSV', 'RGB')])
    swap = [g['channel_swap'](channel_swap)] if channel_swap is not None else []
    if sequence == 1:
        return [f32] + b + c + [u8] + hsv + swap
    return [f32] + b + [u8] + hsv + [f32] + c + [u8] + swap


_BOX_FILTER_DEFAULTS = dict(check_overlap=True, check_min_area=True, check_degenerate=True, overlap_criterion='center_point',
                            overlap_bounds=(0.3, 1.0), min_area=16, border_pixels='half')


def box_filter_ops(spec, img_height, img_width):
    """The ops of one ``BoxFilter.__call__`` (validation_utils.py:147-232) against an ``img_height x img_width`` image: the
    degenerate / minimum-area test, then the overlap test (all three are ANDed there, so the order does not matter).  ``spec``
    is a ``BoxFilter`` (``object_detection_2d_image_boxes_validation_utils``, or the reference's), a dict of ``BoxFilter``'s
    keyword arguments (its defaults fill the rest) or any object with those attributes; ``None`` gives no ops.  Fixed bounds
    only (no ``BoundGenerator``)."""
    if spec is None:
        return []
    if isinstance(spec, dict):
        unknown = set(spec) - set(_BOX_FILTER_DEFAULTS) - {'labels_format'}
        if unknown:
            raise ValueError('unknown BoxFilter arguments %s' % sorted(unknown))
        get = lambda k: spec.get(k, _BOX_FILTER_DEFAULTS[k])          # noqa: E731
    else:
        get = lambda k: getattr(spec, k, _BOX_FILTER_DEFAULTS[k])      # noqa: E731
    if not isinstance(get('overlap_bounds'), (list, tuple)):
        raise ValueError('only fixed `overlap_bounds` (a 2-tuple) are supported')
    ops = []
    if get('check_degenerate') or get('check_min_area'):
        ops.append(box_filter(check_degenerate=bool(get('check_degenerate')), min_area=get('min_area') if get('check_min_area') else None))
    if get('check_overlap'):
        ops.append(overlap_filter(img_height, img_width, get('overlap_criterion'), get('overlap_bounds'), get('border_pixels')))
    return ops


def translate_ops(img_height, img_width, dy, dx, box_filter=None, clip_boxes=True, background=(0, 0, 0)):
    """What ``Translate(dy, dx, clip_boxes, box_filter, background)(image, labels)`` runs: the shift, its box filter against
    the image, then the clip."""
    return ([translate(img_height, img_width, dy, dx, background)] + box_filter_ops(box_filter, img_height, img_width)
            + ([clip(img_height, img_width)] if clip_boxes else []))


def scale_ops(img_height, img_width, factor, box_filter=None, clip_boxes=True, background=(0, 0, 0)):
    """What ``Scale(factor, clip_boxes, box_filter, background)(image, labels)`` runs."""
    return ([scale(img_height, img_width, factor, background)] + box_filter_ops(box_filter, img_height, img_width)
            + ([clip(img_height, img_width)] if clip_boxes else []))


def rotate_ops(img_height, img_width, angle):
    """What ``Rotate(angle)(image, labels)`` runs: the rotation alone (it neither filters nor clips)."""
    return [rotate(img_height, img_width, angle)]


def crop_pad_ops(patch_ymin, patch_xmin, patch_height, patch_width, box_filter=None, clip_boxes=True, background=(0, 0, 0)):
    """What ``CropPad(..., clip_boxes, box_filter, background)(image, labels)`` runs, for any ``BoxFilter`` (``RandomPatch``
    with the satellite chain's 'area' filter, for instance): the patch, its box filter against the patch, then the clip."""
    return ([crop_pad(patch_ymin, patch_xmin, patch_height, patch_width, clip_boxes=False, background=background)]
            + box_filter_ops(box_filter, patch_height, patch_width) + ([clip(patch_height, patch_width)] if clip_boxes else []))


def resize_ops(in_height, in_width, out_height, out_width, box_filter=None, interpolation_mode=_ffi.INTER_LINEAR):
    """What ``Resize(out_height, out_width, interpolation_mode, box_filter)(image, labels)`` runs."""
    return ([resize(in_height, in_width, out_height, out_width, drop_degenerate=False, interpolation_mode=interpolation_mode)]
            + box_filter_ops(box_filter, out_height, out_width))


def _pack_ops(ops_per_image, B):
    """B op lists -> (ctypes ``BoxOp`` array [B*max_ops] or None, max_ops); shorter lists end with zeroed (END) records."""
    max_ops = max([len(o) for o in ops_per_image] + [0]) if ops_per_image else 0
    if not max_ops:
        return None, 0
    if len(ops_per_image) != B:
        raise ValueError('ops_per_image must have one list per batch item')
    arr = (_ffi.BoxOp * (B * max_ops))()
    for b, lst in enumerate(ops_per_image):
        for i, o in enumerate(lst):
            e = arr[b * max_ops + i]
            e.op, e.flags, e.a0, e.a1, e.a2, e.a3 = o
    return arr, max_ops


def assemble_batch_device(labels_list, ops_per_image=None):
    """``labels_list``: B arrays ``(k_i, 5)`` ``[class_id, xmin, ymin, xmax, ymax]`` (any numeric dtype, possibly empty).
    ``ops_per_image``: optional list of B lists of operations built with ``crop_pad`` / ``flip`` / ``resize`` / ``box_filter``.
    Returns ``(gt_dev (N,5) float32, offsets_dev (B+1,) int32, stats_dev int32[2] = (boxes left, largest image), total_upper,
    max_upper)`` -- CUDA tensors; the two upper bounds are host integers (box counts before filtering)."""
    import torch
    rows, offs = [], [0]
    for g in labels_list:
        g = np.asarray(g.detach().cpu().numpy() if hasattr(g, 'detach') else g, dtype=np.float64).reshape(-1, 5) if np.size(g) else np.zeros((0, 5), np.float64)
        rows.append(g)
        offs.append(offs[-1] + g.shape[0])
    B = len(rows)
    total = offs[-1]
    max_g = max([r.shape[0] for r in rows] + [0])
    flat = np.concatenate(rows, axis=0) if total else np.zeros((1, 5), np.float64)      # float64 like the reference's label arrays
    gt_in = torch.from_numpy(np.ascontiguousarray(flat)).pin_memory().cuda(non_blocking=True)
    offs_in = torch.from_numpy(np.asarray(offs, dtype=np.int32)).pin_memory().cuda(non_blocking=True)
    arr, max_ops = _pack_ops(ops_per_image, B)
    ops_dev = None
    if max_ops:
        host = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8)
        ops_dev = host.pin_memory().cuda(non_blocking=True)
    gt_out = torch.empty((max(total, 1), 5), dtype=torch.float32, device='cuda')
    offs_out = torch.empty((B + 1,), dtype=torch.int32, device='cuda')
    stats = torch.empty((2,), dtype=torch.int32, device='cuda')
    _ffi.check(_ffi.lib().ssdk_assemble_batch(_ffi.context(), _ffi.dptr(gt_in), 1, _ffi.dptr(offs_in), B, int(total), _ffi.dptr(ops_dev),
                                              int(max_ops), _ffi.dptr(gt_out), _ffi.dptr(offs_out), _ffi.dptr(stats), _ffi.stream_ptr()))
    return gt_out, offs_out, stats, int(total), int(max_g)


def encode_batch_device(encoder, labels_list, ops_per_image=None, out=None):
    """``label_encoder(batch_y)`` of the reference's generator (:1146-1151) without leaving the device: box operations, packing
    and ``SSDInputEncoder`` -> float32 CUDA tensor ``(B, P, C+12)``."""
    gt, offs, _, total, max_g = assemble_batch_device(labels_list, ops_per_image)
    return encoder.encode_device_offsets(gt, offs, total, max_g, out=out)


def assemble_images_device(images_list, ops_per_image, out_height, out_width, out=None):
    """The image half of the op lists on the device (``ssdk_assemble_images``).  ``images_list``: B uint8 arrays or CPU tensors,
    ``(h,w)``, ``(h,w,1)``, ``(h,w,3)`` or ``(h,w,4)``, of any size; ``ops_per_image``: B op lists (or None: every image must
    already be ``out_height x out_width``).  The images are packed into one pinned buffer and uploaded with one asynchronous
    copy; one kernel launch.  Returns the float32 CUDA tensor ``(B, out_height, out_width, 3)`` of [0,255] integers (``out``
    if given), what ``SSDTrainer.train_on_batch`` / ``predict_device`` take.  A bad op list raises ``ValueError`` before
    anything is written."""
    import torch
    B = len(images_list)
    if B == 0:
        raise ValueError('images_list is empty')
    arrays, hwc, offs = [], np.zeros((B, 3), np.int32), np.zeros((B + 1,), np.int64)
    for b, im in enumerate(images_list):
        a = np.asarray(im.detach().cpu().numpy() if hasattr(im, 'detach') else im)
        if a.dtype != np.uint8 or a.ndim not in (2, 3):
            raise ValueError('image %d: expected a uint8 array (h,w) or (h,w,c), got %s %s' % (b, a.dtype, a.shape))
        hwc[b] = (a.shape[0], a.shape[1], 1 if a.ndim == 2 else a.shape[2])
        arrays.append(a)
        offs[b + 1] = offs[b] + a.size
    oh, ow = int(out_height), int(out_width)
    if out is not None:
        if tuple(out.shape) != (B, oh, ow, 3) or out.dtype != torch.float32 or not out.is_cuda or not out.is_contiguous():
            raise ValueError('`out` must be a contiguous float32 CUDA tensor of shape %s' % ((B, oh, ow, 3),))
    arr, max_ops = _pack_ops(ops_per_image, B)
    host = torch.empty((max(int(offs[-1]), 1),), dtype=torch.uint8, pin_memory=True)
    flat = host.numpy()
    for b, a in enumerate(arrays):
        flat[offs[b]:offs[b + 1]] = a.reshape(-1)
    src = host.to('cuda', non_blocking=True)
    x = out if out is not None else torch.empty((B, oh, ow, 3), dtype=torch.float32, device='cuda')
    _ffi.check(_ffi.lib().ssdk_assemble_images(_ffi.context(), _ffi.dptr(src), _ffi.np_ptr(offs, C.c_longlong), _ffi.np_ptr(hwc, C.c_int),
                                               B, arr, int(max_ops), oh, ow, _ffi.dptr(x), _ffi.stream_ptr()))
    return x


def assemble_training_batch(encoder, images_list, labels_list, ops_per_image, out_height, out_width, x_out=None, y_out=None):
    """One training batch from raw images and labels, driven by ONE op list per image: the images through
    ``ssdk_assemble_images``, the boxes through ``ssdk_assemble_batch`` and ``encoder.encode_device_offsets``.  Returns
    ``(x (B,H,W,3) float32, y_true (B,P,C+12) float32)``, CUDA tensors ready for ``SSDTrainer.train_on_batch`` /
    ``model.train_on_batch``.  Everything is enqueued asynchronously: the host does not wait for the device."""
    x = assemble_images_device(images_list, ops_per_image, out_height, out_width, out=x_out)
    y = encode_batch_device(encoder, labels_list, ops_per_image, out=y_out)
    return x, y
