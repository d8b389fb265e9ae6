"""Predictions over a dataset of images of any size, on the device: the loop behind ``Evaluator.predict_on_dataset`` (reference
``eval_utils/average_precision_evaluator.py:258-424``) and ``coco_utils.predict_all_to_json`` (``coco_utils.py:62-200``).

The reference's generator runs ``ConvertTo3Channels`` and ``Resize`` (mode 'resize') or ``ConvertTo3Channels``,
``RandomPadFixedAR`` and ``Resize`` (mode 'pad') on every image, predicts, and maps every detection back to the original image
through the inverters of those transforms (``apply_inverse_transforms``).  Here, per batch:

- the images come from ``data_generator.images`` (uint8 arrays of any size and channel count) or are decoded from
  ``data_generator.filenames`` with PIL as the reference's generator does (``object_detection_2d_data_generator.py:1014-1018``),
  on a small thread pool a bounded number of batches ahead of the device;
- each image gets an op list (``batch_assembly.resize`` and, in 'pad' mode, a ``crop_pad`` with the patch ``RandomPadFixedAR``
  draws from ``np.random`` in the reference's order) and four inverter parameters;
- the inverter parameters and the image bytes go to the device with one copy out of a ring of pinned buffers owned by the
  loop; one ``ssdk_assemble_images`` launch makes the batch; ``model.predict_device`` and, for 'training'-mode models,
  ``decode_device`` (``decode_detections``' semantics) decode it; one ``ssdk_eval_collect`` launch keeps the detections, applies
  the inverters with the reference's arithmetic and appends them to device arrays.

The host waits for the device only before it refills a pinned buffer; the results stay on the device (``DeviceDetections``)."""
import ctypes as C
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from .. import _ffi
from ..data_generator import batch_assembly as ba

_PIN_SLOTS = 3
_DECODE_THREADS = 4
_DECODE_AHEAD = 2          # batches decoded ahead of the one being assembled


def load_image(filename):
    """What the reference's generator does with a filename: ``np.array(Image.open(f), dtype=np.uint8)``."""
    from PIL import Image
    with Image.open(filename) as image:
        return np.array(image, dtype=np.uint8)


def _random_patch(img_h, img_w, ph, pw, random):
    """``RandomPatch``'s draws for a ``ph x pw`` patch (patch_sampling_ops.py:506, :180-193): one ``uniform(0, 1)``, then the
    ``randint`` for y and for x, all three also when a range is 0.  Returns ``(patch_ymin, patch_xmin, ph, pw)``."""
    random.uniform(0, 1)
    y_range = img_h - ph
    py = random.randint(0, y_range + 1) if y_range >= 0 else random.randint(y_range, 1)
    x_range = img_w - pw
    px = random.randint(0, x_range + 1) if x_range >= 0 else random.randint(x_range, 1)
    return py, px, ph, pw


def pad_patch(img_h, img_w, img_height, img_width, random=np.random):
    """``RandomPadFixedAR(patch_aspect_ratio=img_width/img_height)`` on an ``img_h x img_w`` image (patch_sampling_ops.py:859-881,
    :180-193, :508): the patch size, then one ``uniform(0, 1)`` and the ``randint`` draws for y and x, all three also when a range
    is 0.  Returns ``(patch_ymin, patch_xmin, patch_height, patch_width)``.  With a non-square target an image whose aspect ratio
    lies between 1 and the target's gets a positive range: the patch crops it, as in the reference."""
    ar = img_width / img_height
    if img_w < img_h:
        ph = img_h
        pw = int(round(ph * ar))
    else:
        pw = img_w
        ph = int(round(pw / ar))
    return _random_patch(img_h, img_w, ph, pw, random)


def max_crop_patch(img_h, img_w, patch_aspect_ratio, random=np.random):
    """``RandomMaxCropFixedAR(patch_aspect_ratio)`` on an ``img_h x img_w`` image (patch_sampling_ops.py:796-821, :117-193,
    :506), the patch of ``weight_sampling_tutorial.ipynb``'s sample chain: the largest patch of that aspect ratio, then
    ``RandomPatch``'s ``uniform(0, 1)`` and the ``randint`` draws for y and x, all three also when a range is 0.  Returns
    ``(patch_ymin, patch_xmin, patch_height, patch_width)``."""
    if img_w / img_h < patch_aspect_ratio:
        pw = img_w
        ph = int(round(pw / patch_aspect_ratio))
    else:
        ph = img_h
        pw = int(round(ph * patch_aspect_ratio))
    return _random_patch(img_h, img_w, ph, pw, random)


def max_crop_ops(img_h, img_w, patch_aspect_ratio, box_filter=None, image_validator=None, clip_boxes=True, random=np.random):
    """The op list of one ``RandomMaxCropFixedAR(patch_aspect_ratio, clip_boxes=clip_boxes)`` call with ``max_crop_patch``'s
    draw: the ``crop_pad`` of the patch and, with ``clip_boxes``, the clip to it.  Follow it with ``batch_assembly.resize_ops``
    and give the lists to ``assemble_images_device`` / ``assemble_training_batch``: the tutorial's ``ConvertTo3Channels ->
    RandomMaxCropFixedAR -> Resize``.  Without a ``box_filter`` or ``image_validator`` the first patch is the one the reference
    keeps; with one of them it may retry, and those draws stay with the caller (``NotImplementedError``)."""
    if box_filter is not None or image_validator is not None:
        raise NotImplementedError('RandomMaxCropFixedAR with a box_filter or image_validator: draw the patches and build the '
                                  'ops with batch_assembly.crop_pad_ops')
    py, px, ph, pw = max_crop_patch(img_h, img_w, patch_aspect_ratio, random)
    return ba.crop_pad_ops(py, px, ph, pw, clip_boxes=clip_boxes)


def image_plan(img_h, img_w, img_height, img_width, mode, random=np.random):
    """The op list of one image and its inverter parameters ``(ratio_y, ratio_x, offset_y, offset_x)`` (Resize's inverter scales
    by canvas / output size, CropPad's adds the patch origin)."""
    if mode == 'resize':
        return [ba.resize(img_h, img_w, img_height, img_width, drop_degenerate=False)], (img_h / img_height, img_w / img_width, 0.0, 0.0)
    py, px, ph, pw = pad_patch(img_h, img_w, img_height, img_width, random)
    return ([ba.crop_pad(py, px, ph, pw, clip_boxes=False, background=(0, 0, 0)),
             ba.resize(ph, pw, img_height, img_width, drop_degenerate=False)], (ph / img_height, pw / img_width, float(py), float(px)))


class DeviceDetections:
    """The detections of a dataset on the device, in the reference's collection order (image, then row): ``image`` (index into
    the dataset), ``cls``, ``conf`` and ``box`` (xmin, ymin, xmax, ymax), the last two float64 holding values of ``dtype``
    (float32 for the layer path, float64 for ``decode_detections``)."""

    def __init__(self, image, cls, conf, box, count, dtype, image_ids):
        self._image, self._cls, self._conf, self._box, self._count = image, cls, conf, box, count
        self.dtype = dtype
        self.image_ids = image_ids
        self._n = None

    def __len__(self):
        if self._n is None:
            self._n = int(self._count.item())
            if self._n > self._image.numel():
                raise RuntimeError('ssdk_eval_collect: %d detections for %d slots' % (self._n, self._image.numel()))
        return self._n

    def device(self):
        """``(image int32, cls int32, conf float64, box (n,4) float64)`` CUDA tensors."""
        n = len(self)
        return self._image[:n], self._cls[:n], self._conf[:n], self._box[:n]

    def host(self):
        """The same as ndarrays, ``conf`` and ``box`` in ``dtype``."""
        img, cls, conf, box = (t.cpu().numpy() for t in self.device())
        return img, cls, conf.astype(self.dtype), box.astype(self.dtype)

    def per_class(self, n_classes):
        """The reference's ``prediction_results``: per class a list of ``(image_id, conf, xmin, ymin, xmax, ymax)`` tuples with
        NumPy scalars of ``dtype``, in collection order."""
        img, cls, conf, box = self.host()
        ids = np.empty(len(self.image_ids), dtype=object)
        ids[:] = list(self.image_ids)
        results = [list() for _ in range(n_classes + 1)]
        for c in np.unique(cls):
            sel = np.flatnonzero(cls == c)
            results[int(c)].extend(zip(ids[img[sel]], conf[sel], box[sel, 0], box[sel, 1], box[sel, 2], box[sel, 3]))
        return results


class _PinnedRing:
    """Pinned host buffers (with their device twins) reused round-robin; a buffer is refilled only after the copy out of it has
    run (its event), so the host waits for the device only here."""

    def __init__(self, n=_PIN_SLOTS):
        self.slots = [None] * n
        self.next = 0

    def take(self, nbytes):
        import torch
        k = self.next
        self.next = (k + 1) % len(self.slots)
        s = self.slots[k]
        if s is not None:
            s[2].synchronize()
        if s is None or s[0].numel() < nbytes:
            size = max(int(nbytes * 1.25), 1 << 20)
            s = [torch.empty((size,), dtype=torch.uint8, pin_memory=True), torch.empty((size,), dtype=torch.uint8, device='cuda'),
                 torch.cuda.Event()]
            self.slots[k] = s
        return s


def _image_source(data_generator, pool):
    """(number of images, function i -> future-or-array of image i)."""
    images = getattr(data_generator, 'images', None)
    if images is not None:
        return len(images), lambda i: images[i]
    filenames = getattr(data_generator, 'filenames', None)
    if filenames is None:
        raise ValueError('`data_generator` has neither `images` nor `filenames`.')
    return len(filenames), lambda i: pool.submit(load_image, filenames[i])


def predict_dataset(model, data_generator, img_height, img_width, batch_size, mode='resize', model_mode='inference',
                    decode_kwargs=None, round_confidences=False, pred_format=None, gt_format=None, random=np.random):
    """Predict over the whole dataset; returns ``DeviceDetections``.  ``model`` needs ``predict_device`` (float32 CUDA batch
    ``(B, img_height, img_width, 3)`` -> decoded rows ``(B, k, 6)`` in 'inference' mode, raw ``(B, P, C+12)`` in 'training'
    mode, then decoded here with ``decode_kwargs``: ``confidence_thresh``, ``iou_threshold``, ``top_k``, ``input_coords``,
    ``normalize_coords``, ``border_pixels``)."""
    import torch
    from ..ssd_encoder_decoder.ssd_output_decoder import decode_device, PER_CLASS
    if mode not in ('resize', 'pad'):
        raise ValueError("`data_generator_mode` can be either of 'resize' or 'pad', but received '{}'.".format(mode))
    if model_mode not in ('inference', 'training'):
        raise ValueError("`model_mode` can be either 'training' or 'inference', but received '{}'.".format(model_mode))
    pred_format = pred_format or {'class_id': 0, 'conf': 1, 'xmin': 2, 'ymin': 3, 'xmax': 4, 'ymax': 5}
    gt_format = gt_format or {'class_id': 0, 'xmin': 1, 'ymin': 2, 'xmax': 3, 'ymax': 4}
    cols = np.array([pred_format[k] for k in ('class_id', 'conf', 'xmin', 'ymin', 'xmax', 'ymax')]
                    + [gt_format[k] + 1 for k in ('ymin', 'ymax', 'xmin', 'xmax')], dtype=np.int32)
    training = model_mode == 'training'
    f64 = 1 if training else 0
    H, W, bs = int(img_height), int(img_width), int(batch_size)
    ring = _PinnedRing()
    ctx = _ffi.context()
    lib = _ffi.lib()
    out = None
    count = torch.zeros((1,), dtype=torch.int32, device='cuda')
    with ThreadPoolExecutor(_DECODE_THREADS) as pool:
        n_images, get = _image_source(data_generator, pool)
        if data_generator.image_ids is None:                  # pseudo image ids, as the reference makes them (:348-349)
            data_generator.image_ids = list(range(n_images))
        ahead = {}

        def fetch(lo):
            if lo < n_images and lo not in ahead:
                ahead[lo] = [get(i) for i in range(lo, min(lo + bs, n_images))]

        for lo in range(0, n_images, bs):
            for k in range(_DECODE_AHEAD + 1):
                fetch(lo + k * bs)
            arrays = []
            for a in ahead.pop(lo):
                a = a.result() if hasattr(a, 'result') else a
                a = np.asarray(a.detach().cpu().numpy() if hasattr(a, 'detach') else a)
                if a.dtype != np.uint8 or a.ndim not in (2, 3):
                    raise ValueError('image %d: expected a uint8 array (h,w) or (h,w,c), got %s %s' % (lo + len(arrays), a.dtype, a.shape))
                arrays.append(a)
            B = len(arrays)
            ops, inv = [], np.empty((B, 4), dtype=np.float64)
            for b, a in enumerate(arrays):
                o, inv[b] = image_plan(a.shape[0], a.shape[1], H, W, mode, random)
                ops.append(o)
            # one pinned buffer: the inverter parameters, then the image bytes
            head = inv.nbytes
            offs = np.zeros((B + 1,), np.int64)
            hwc = np.zeros((B, 3), np.int32)
            for b, a in enumerate(arrays):
                hwc[b] = (a.shape[0], a.shape[1], 1 if a.ndim == 2 else a.shape[2])
                offs[b + 1] = offs[b] + a.size
            host, dev, done = ring.take(head + int(offs[-1]))
            flat = host.numpy()
            flat[:head] = inv.reshape(-1).view(np.uint8)
            for b, a in enumerate(arrays):
                flat[head + offs[b]:head + offs[b + 1]] = a.reshape(-1)
            dev[:head + int(offs[-1])].copy_(host[:head + int(offs[-1])], non_blocking=True)
            done.record()
            arr, max_ops = ba._pack_ops(ops, B)
            x = torch.empty((B, H, W, 3), dtype=torch.float32, device='cuda')
            _ffi.check(lib.ssdk_assemble_images(ctx, C.c_void_p(dev.data_ptr() + head), _ffi.np_ptr(offs, C.c_longlong),
                                                _ffi.np_ptr(hwc, C.c_int), B, arr, int(max_ops), H, W, _ffi.dptr(x), _ffi.stream_ptr()))
            y = model.predict_device(x)
            counts = None
            if training:
                d = decode_kwargs or {}
                y, counts = decode_device(y, PER_CLASS, False, d.get('confidence_thresh', 0.01), d.get('iou_threshold', 0.45),
                                          d.get('top_k', 200), 0, d.get('input_coords', 'centroids'), d.get('normalize_coords', True),
                                          H, W, d.get('border_pixels', 'half'))
            y = y.to(torch.float32).contiguous()
            if y.dim() != 3 or y.shape[0] != B or y.shape[2] != 6:
                raise ValueError('the decoded predictions must have the shape (%d, k, 6), got %s' % (B, tuple(y.shape)))
            max_out = int(y.shape[1])
            if out is None:
                cap = n_images * max_out
                out = (torch.empty((cap,), dtype=torch.int32, device='cuda'), torch.empty((cap,), dtype=torch.int32, device='cuda'),
                       torch.empty((cap,), dtype=torch.float64, device='cuda'), torch.empty((cap, 4), dtype=torch.float64, device='cuda'))
            elif n_images * max_out > out[0].numel():
                raise ValueError('the decoded predictions of one batch have %d rows, the first batch had fewer' % max_out)
            _ffi.check(lib.ssdk_eval_collect(ctx, _ffi.dptr(y), B, max_out, _ffi.dptr(counts),
                                             C.c_void_p(dev.data_ptr()), _ffi.np_ptr(cols, C.c_int), f64, 1 if mode == 'pad' else 0,
                                             int(round_confidences) if round_confidences else 0, lo, int(out[0].numel()), _ffi.dptr(count),
                                             *(_ffi.dptr(t) for t in out), _ffi.stream_ptr()))
    if out is None:
        out = tuple(torch.empty((0,) + s, dtype=t, device='cuda') for s, t in (((), torch.int32), ((), torch.int32), ((), torch.float64),
                                                                                ((4,), torch.float64)))
    return DeviceDetections(*out, count, np.float64 if training else np.float32, list(data_generator.image_ids))
