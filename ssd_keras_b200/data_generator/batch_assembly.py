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
  to OpenCV 4.13 (``oracle/imageops.py`` restates it); at most one, as the last op that changes the image;
- ``box_filter``: boxes only.

Not covered: photometric distortions, other interpolation modes (``INTER_CUBIC``, ``INTER_LANCZOS4``, ``INTER_AREA`` apart from
cv2's own exact-2x linear path), ``Translate`` / ``Scale`` / ``Rotate`` (``cv2.warpAffine``), the random patch samplers, JPEG
decoding.  The random decisions of a chain (which patch, flip or not, which interpolation) stay with the caller, as for the
boxes."""
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


def box_filter(check_degenerate=True, min_area=None):
    """``BoxFilter`` without the overlap test (validation_utils.py:155-165); also ``degenerate_box_handling='remove'``."""
    return (_ffi.BOXOP_FILTER, (1 if check_degenerate else 0) | (2 if min_area is not None else 0), float(min_area or 0.0), 0.0, 0.0, 0.0)


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
