"""``SSDInputEncoder`` on H100: same constructor / call surface as the reference class
(``ssd_encoder_decoder/ssd_input_encoder.py:36-57, 277``), computed by the CUDA kernels in
``csrc/encode.cu`` through ``ssdk_encode``.  Host side is argument validation and packing only.
"""
import ctypes as C

import numpy as np

from .. import _ffi


class DegenerateBoxError(Exception):
    """Raised for ground-truth boxes with xmax <= xmin or ymax <= ymin (reference :333-336, :613)."""
    pass


class SSDInputEncoder:

    def __init__(self, img_height, img_width, n_classes, predictor_sizes, min_scale=0.1, max_scale=0.9, scales=None,
                 aspect_ratios_global=[0.5, 1.0, 2.0], aspect_ratios_per_layer=None, two_boxes_for_ar1=True,
                 steps=None, offsets=None, clip_boxes=False, variances=[0.1, 0.1, 0.2, 0.2], matching_type='multi',
                 pos_iou_threshold=0.5, neg_iou_limit=0.3, border_pixels='half', coords='centroids',
                 normalize_coords=True, background_id=0):
        predictor_sizes = np.array(predictor_sizes)
        if predictor_sizes.ndim == 1:
            predictor_sizes = np.expand_dims(predictor_sizes, axis=0)
        n_layers = predictor_sizes.shape[0]
        # the reference's argument checks (:142-180), same conditions and exception types
        if (min_scale is None or max_scale is None) and scales is None:
            raise ValueError("Either `min_scale` and `max_scale` or `scales` need to be specified.")
        if scales:
            if len(scales) != n_layers + 1:
                raise ValueError("It must be either scales is None or len(scales) == len(predictor_sizes)+1, but "
                                 "len(scales) == {} and len(predictor_sizes)+1 == {}".format(len(scales), n_layers + 1))
            scales = np.array(scales)
            if np.any(scales <= 0):
                raise ValueError("All values in `scales` must be greater than 0, but the passed list of scales is {}".format(scales))
        elif not 0 < min_scale <= max_scale:
            raise ValueError("It must be 0 < min_scale <= max_scale, but it is min_scale = {} and max_scale = {}".format(min_scale, max_scale))
        if aspect_ratios_per_layer is not None:
            if len(aspect_ratios_per_layer) != n_layers:
                raise ValueError("It must be either aspect_ratios_per_layer is None or len(aspect_ratios_per_layer) == "
                                 "len(predictor_sizes), but len(aspect_ratios_per_layer) == {} and len(predictor_sizes) == {}"
                                 .format(len(aspect_ratios_per_layer), n_layers))
            for ar in aspect_ratios_per_layer:
                if np.any(np.array(ar) <= 0):
                    raise ValueError("All aspect ratios must be greater than zero.")
        else:
            if aspect_ratios_global is None:
                raise ValueError("At least one of `aspect_ratios_global` and `aspect_ratios_per_layer` must not be `None`.")
            if np.any(np.array(aspect_ratios_global) <= 0):
                raise ValueError("All aspect ratios must be greater than zero.")
        if len(variances) != 4:
            raise ValueError("4 variance values must be pased, but {} values were received.".format(len(variances)))
        variances = np.array(variances)
        if np.any(variances <= 0):
            raise ValueError("All variances must be >0, but the variances given are {}".format(variances))
        if coords not in ('minmax', 'centroids', 'corners'):
            raise ValueError("Unexpected value for `coords`. Supported values are 'minmax', 'corners' and 'centroids'.")
        if steps is not None and len(steps) != n_layers:
            raise ValueError("You must provide at least one step value per predictor layer.")
        if offsets is not None and len(offsets) != n_layers:
            raise ValueError("You must provide at least one offset value per predictor layer.")
        if border_pixels not in _ffi.BORDER_D:
            raise ValueError("`border_pixels` must be one of 'half', 'include', 'exclude'.")

        self.img_height, self.img_width = img_height, img_width
        self.n_classes = n_classes + 1
        self.predictor_sizes = predictor_sizes
        self.min_scale, self.max_scale = min_scale, max_scale
        self.scales = np.linspace(min_scale, max_scale, n_layers + 1) if scales is None else scales
        self.aspect_ratios = ([aspect_ratios_global] * n_layers) if aspect_ratios_per_layer is None else aspect_ratios_per_layer
        self.two_boxes_for_ar1 = two_boxes_for_ar1
        self.steps = steps if steps is not None else [None] * n_layers
        self.offsets = offsets if offsets is not None else [None] * n_layers
        self.clip_boxes = clip_boxes
        self.variances = variances
        self.matching_type = matching_type
        self.pos_iou_threshold = pos_iou_threshold
        self.neg_iou_limit = neg_iou_limit
        self.border_pixels = border_pixels
        self.coords = coords
        self.normalize_coords = normalize_coords
        self.background_id = background_id

        a64, a32, nb = _ffi.generate_anchors(img_height, img_width, predictor_sizes, self.scales, self.aspect_ratios,
                                             two_boxes_for_ar1, self.steps, self.offsets, clip_boxes, coords, normalize_coords)
        self.anchors = a64                    # (P,4) float64, model order
        self.anchors_f32 = a32
        if aspect_ratios_per_layer is not None:
            self.n_boxes = nb
        else:
            self.n_boxes = nb[0]
        self.boxes_list = []
        o = 0
        for (h, w), b in zip(predictor_sizes, nb):
            self.boxes_list.append(a64[o:o + h * w * b].reshape(h, w, b, 4))
            o += h * w * b
        self._n_boxes_per_layer = list(nb)
        self._diagnostics()
        self._handle = None
        self._status = None

    def generate_anchor_boxes_for_layer(self, feature_map_size, aspect_ratios, this_scale, next_scale, this_steps=None,
                                        this_offsets=None, diagnostics=False):
        """Reference :420-548: the anchors of ONE predictor layer as a (feature_map_height, feature_map_width, n_boxes, 4) float64
        array in this encoder's ``coords`` / ``normalize_coords`` / ``clip_boxes`` convention (same host routine as ``__init__``,
        ``ssdk_anchors_generate``).  With ``diagnostics`` also returns (centres, wh_list, step, offset) like the reference."""
        fh, fw = int(feature_map_size[0]), int(feature_map_size[1])
        a64, _, nb = _ffi.generate_anchors(self.img_height, self.img_width, [(fh, fw)], [this_scale, next_scale], [aspect_ratios],
                                           self.two_boxes_for_ar1, [this_steps], [this_offsets], self.clip_boxes, self.coords,
                                           self.normalize_coords)
        boxes = a64.reshape(fh, fw, nb[0], 4)
        if not diagnostics:
            return boxes
        size = min(self.img_height, self.img_width)
        wh = []
        for ar in aspect_ratios:
            if ar == 1:
                wh.append((this_scale * size,) * 2)
                if self.two_boxes_for_ar1:
                    wh.append((np.sqrt(this_scale * next_scale) * size,) * 2)
            else:
                wh.append((this_scale * size * np.sqrt(ar), this_scale * size / np.sqrt(ar)))
        st_h, st_w = _ffi._pair_or_nan(this_steps)
        if np.isnan(st_h):
            st_h, st_w = self.img_height / fh, self.img_width / fw
        of_h, of_w = _ffi._pair_or_nan(this_offsets)
        if np.isnan(of_h):
            of_h = of_w = 0.5
        cy = np.linspace(of_h * st_h, (of_h + fh - 1) * st_h, fh)
        cx = np.linspace(of_w * st_w, (of_w + fw - 1) * st_w, fw)
        return boxes, (cy, cx), np.array(wh), (st_h, st_w), (of_h, of_w)

    def _diagnostics(self):
        """wh / steps / offsets / centres per layer, the ``*_diag`` attributes of the reference (:254-275)."""
        self.wh_list_diag, self.steps_diag, self.offsets_diag, self.centers_diag = [], [], [], []
        size = min(self.img_height, self.img_width)
        for i, (fh, fw) in enumerate(self.predictor_sizes):
            wh = []
            for ar in self.aspect_ratios[i]:
                if ar == 1:
                    wh.append((self.scales[i] * size,) * 2)
                    if self.two_boxes_for_ar1:
                        wh.append((np.sqrt(self.scales[i] * self.scales[i + 1]) * size,) * 2)
                else:
                    wh.append((self.scales[i] * size * np.sqrt(ar), self.scales[i] * size / np.sqrt(ar)))
            st_h, st_w = _ffi._pair_or_nan(self.steps[i])
            if np.isnan(st_h):
                st_h, st_w = self.img_height / fh, self.img_width / fw
            of_h, of_w = _ffi._pair_or_nan(self.offsets[i])
            if np.isnan(of_h):
                of_h = of_w = 0.5
            cy = np.linspace(of_h * st_h, (of_h + fh - 1) * st_h, fh)
            cx = np.linspace(of_w * st_w, (of_w + fw - 1) * st_w, fw)
            self.wh_list_diag.append(np.array(wh)); self.steps_diag.append((st_h, st_w))
            self.offsets_diag.append((of_h, of_w)); self.centers_diag.append((cy, cx))

    # -----------------------------------------------------------------------------------------
    def _encoder(self):
        if self._handle is None:
            ps = np.ascontiguousarray(np.asarray(self.predictor_sizes, dtype=np.int32).reshape(-1, 2))
            fm_h = np.ascontiguousarray(ps[:, 0]); fm_w = np.ascontiguousarray(ps[:, 1])
            nb = np.ascontiguousarray(np.asarray(self._n_boxes_per_layer, dtype=np.int32))
            self._geom = (fm_h, fm_w, nb)                     # read during ssdk_encoder_create only
            cfg = _ffi.EncodeCfg(int(self.img_height), int(self.img_width), int(self.n_classes), int(self.anchors.shape[0]),
                                 int(self.background_id), _ffi.COORDS[self.coords], 1 if self.matching_type == 'multi' else 0,
                                 float(self.pos_iou_threshold), float(self.neg_iou_limit), _ffi.BORDER_D[self.border_pixels],
                                 int(bool(self.normalize_coords)), (C.c_double * 4)(*[float(v) for v in self.variances]),
                                 int(ps.shape[0]), _ffi.np_ptr(fm_h, C.c_int), _ffi.np_ptr(fm_w, C.c_int), _ffi.np_ptr(nb, C.c_int))
            h = C.c_void_p()
            anc = np.ascontiguousarray(self.anchors)
            _ffi.check(_ffi.lib().ssdk_encoder_create(_ffi.context(), C.byref(cfg), _ffi.np_ptr(anc, C.c_double), C.byref(h)))
            self._handle = h
        return self._handle

    def __del__(self):
        try:
            if getattr(self, '_handle', None) is not None:
                _ffi.lib().ssdk_encoder_destroy(self._handle)
        except Exception:
            pass

    @property
    def last_status(self):
        """int32 CUDA tensor (1,): 0, or the 1-based index of a batch item with a degenerate box seen by ``encode_device``
        since the flag was last read (the kernel raises it with an atomic; reading synchronises and clears it)."""
        import torch
        if self._status is None:
            return torch.zeros((1,), dtype=torch.int32, device='cuda')
        out = self._status.clone()
        if int(out.item()) != 0:
            self._status.zero_()
        return out

    def encode_device(self, gt_boxes_dev, gt_offsets, return_matches=False, out=None):
        """Hot path: ``gt_boxes_dev`` float32 (or float64) CUDA tensor (sum G_i, 5), ``gt_offsets`` host int32 (B+1,), or an
        int32 CUDA tensor together with ``(total_g, max_g)`` -- see ``encode_device_offsets``.  Returns the float32 CUDA tensor
        (B,P,C+12) (``out`` if given) and, optionally, the int32 match tensor (B,P).  ONE kernel launch, asynchronous;
        degenerate boxes are reported through ``self.last_status``."""
        import torch
        offs = np.ascontiguousarray(np.asarray(gt_offsets, dtype=np.int32))
        B = offs.shape[0] - 1
        P, W = self.anchors.shape[0], self.n_classes + 12
        dev = gt_boxes_dev.device if gt_boxes_dev is not None else torch.device('cuda')
        y = out if out is not None else torch.empty((B, P, W), dtype=torch.float32, device=dev)
        if tuple(y.shape) != (B, P, W) or y.dtype != torch.float32 or not y.is_contiguous():
            raise ValueError('`out` must be a contiguous float32 tensor of shape %s' % ((B, P, W),))
        match = torch.empty((B, P), dtype=torch.int32, device=dev) if return_matches else None
        if self._status is None:
            self._status = torch.zeros((1,), dtype=torch.int32, device=dev)
        f64 = gt_boxes_dev is not None and gt_boxes_dev.dtype == torch.float64
        _ffi.check(_ffi.lib().ssdk_encode(self._encoder(), _ffi.dptr(gt_boxes_dev), int(f64), _ffi.np_ptr(offs, C.c_int), None,
                                          B, 0, 0, _ffi.dptr(y), _ffi.dptr(match), _ffi.dptr(self._status), _ffi.stream_ptr()))
        return (y, match) if return_matches else y

    def encode_device_offsets(self, gt_boxes_dev, gt_offsets_dev, total_g, max_g, out=None):
        """Like ``encode_device`` for a batch that was assembled on the device (``data_generator.assemble_batch_device``):
        the row offsets are an int32 CUDA tensor (B+1,), nothing is read from the host.  The rows must be float32."""
        import torch
        B = gt_offsets_dev.shape[0] - 1
        P, W = self.anchors.shape[0], self.n_classes + 12
        y = out if out is not None else torch.empty((B, P, W), dtype=torch.float32, device=gt_offsets_dev.device)
        if self._status is None:
            self._status = torch.zeros((1,), dtype=torch.int32, device=gt_offsets_dev.device)
        f64 = gt_boxes_dev is not None and gt_boxes_dev.dtype == torch.float64
        _ffi.check(_ffi.lib().ssdk_encode(self._encoder(), _ffi.dptr(gt_boxes_dev), int(f64), None, _ffi.dptr(gt_offsets_dev), B,
                                          int(total_g), int(max_g), _ffi.dptr(y), _ffi.dptr(None), _ffi.dptr(self._status),
                                          _ffi.stream_ptr()))
        return y

    def __call__(self, ground_truth_labels, diagnostics=False):
        """Reference call (:277): list of ``(k_i, 5)`` arrays -> ``(B, P, C+12)`` float64 ndarray.  The labels go to the
        device as float64, which is what the reference computes on (:330)."""
        import torch
        rows, offs = [], [0]
        for i, g in enumerate(ground_truth_labels):
            g = np.asarray(g.detach().cpu().numpy() if hasattr(g, 'detach') else g)
            if g.size == 0:
                offs.append(offs[-1])
                continue
            lab = g.astype(np.float64).reshape(-1, 5)
            if np.any(lab[:, 3] - lab[:, 1] <= 0) or np.any(lab[:, 4] - lab[:, 2] <= 0):
                raise DegenerateBoxError("SSDInputEncoder detected degenerate ground truth bounding boxes for batch item {} with "
                                         "bounding boxes {}, i.e. bounding boxes where xmax <= xmin and/or ymax <= ymin. "
                                         "Degenerate ground truth bounding boxes will lead to NaN errors during the training."
                                         .format(i, lab))
            cls = lab[:, 0].astype(np.int64)                   # class_vectors[labels[:, class_id].astype(np.int)] (:349)
            if np.any(cls >= self.n_classes) or np.any(cls < -self.n_classes):
                bad = cls[(cls >= self.n_classes) | (cls < -self.n_classes)][0]
                raise IndexError("index {} is out of bounds for axis 0 with size {}".format(int(bad), self.n_classes))
            lab = lab.copy()
            lab[:, 0] = np.where(cls < 0, cls + self.n_classes, cls)   # NumPy's negative indices wrap around
            rows.append(lab)
            offs.append(offs[-1] + lab.shape[0])
        gt_dev = None
        if rows:
            host = torch.from_numpy(np.ascontiguousarray(np.concatenate(rows, axis=0))).pin_memory()
            gt_dev = host.cuda(non_blocking=True)
        y = self.encode_device(gt_dev, np.array(offs, dtype=np.int32)).cpu().numpy().astype(np.float64)
        if diagnostics:
            y2 = np.copy(y)
            y2[:, :, -12:-8] = 0
            return y, y2
        return y

    def generate_encoding_template(self, batch_size, diagnostics=False):
        """:550-611, host-side (cheap; the hot path never materialises it)."""
        P = self.anchors.shape[0]
        row = np.concatenate([np.zeros((P, self.n_classes)), self.anchors, self.anchors,
                              np.broadcast_to(np.asarray(self.variances, dtype=np.float64), (P, 4))], axis=1)
        t = np.tile(row[None], (batch_size, 1, 1))
        if diagnostics:
            return t, self.centers_diag, self.wh_list_diag, self.steps_diag, self.offsets_diag
        return t
