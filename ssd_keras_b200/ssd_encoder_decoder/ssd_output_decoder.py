"""``decode_detections`` / ``decode_detections_fast`` on H100 (reference
``ssd_encoder_decoder/ssd_output_decoder.py:111-333``), computed by ``csrc/decode.cu`` through ``ssdk_decode``.
"""
import ctypes as C

import numpy as np

from .. import _ffi

PER_CLASS, FAST = 0, 1


def decode_device(y_pred, mode, layer_semantics, confidence_thresh, iou_threshold, top_k, nms_max_output_size,
                  input_coords, normalize_coords, img_height, img_width, border_pixels='half', return_index=False):
    """Device-to-device decode.  ``y_pred``: float32 CUDA tensor (B,P,C+12).
    Returns (out (B,max_out,6) float32, counts (B,) int32[, prior index (B,max_out) int32])."""
    import torch
    if input_coords not in _ffi.COORDS:
        raise ValueError("Unexpected value for `input_coords`. Supported input coordinate formats are 'minmax', 'corners' and 'centroids'.")
    B, P, W = y_pred.shape
    Ctot = W - 12
    if layer_semantics:
        max_out = int(top_k)
        k = int(top_k)
    elif top_k == 'all' or top_k is None:
        k = 0
        max_out = P * (Ctot - 1) if mode == PER_CLASS else P
    else:
        k = int(top_k)
        max_out = k
    cfg = _ffi.DecodeCfg(mode, 1 if layer_semantics else 0, Ctot, P, float(confidence_thresh),
                         float(iou_threshold) if iou_threshold else 0.0, k, int(nms_max_output_size),
                         _ffi.COORDS[input_coords], int(bool(normalize_coords)),
                         int(img_height) if img_height is not None else 0, int(img_width) if img_width is not None else 0,
                         _ffi.BORDER_D[border_pixels], max_out)
    y_pred = y_pred.contiguous()
    out = torch.empty((B, max_out, 6), dtype=torch.float32, device=y_pred.device)
    counts = torch.empty((B,), dtype=torch.int32, device=y_pred.device)
    index = torch.empty((B, max_out), dtype=torch.int32, device=y_pred.device) if return_index else None
    _ffi.check(_ffi.lib().ssdk_decode(_ffi.context(y_pred.device.index), C.byref(cfg), _ffi.dptr(y_pred), B, _ffi.dptr(out),
                                      _ffi.dptr(counts), _ffi.dptr(index), _ffi.stream_ptr()))
    return (out, counts, index) if return_index else (out, counts)


def _to_device(y_pred):
    import torch
    if isinstance(y_pred, np.ndarray):
        t = torch.from_numpy(np.ascontiguousarray(y_pred, dtype=np.float32))
        return t.pin_memory().cuda(non_blocking=True)
    return y_pred.to(dtype=torch.float32, device='cuda')


def _check_norm(normalize_coords, img_height, img_width):
    if normalize_coords and ((img_height is None) or (img_width is None)):
        raise ValueError("If relative box coordinates are supposed to be converted to absolute coordinates, the decoder needs "
                         "the image size in order to decode the predictions, but `img_height == {}` and `img_width == {}`"
                         .format(img_height, img_width))


def _check_coords(input_coords, message):
    if input_coords not in ('centroids', 'minmax', 'corners'):
        raise ValueError(message)


def _ragged(out, counts):
    out = out.cpu().numpy().astype(np.float64)
    counts = counts.cpu().numpy()
    return [out[i, :counts[i]] if counts[i] > 0 else np.array([]) for i in range(out.shape[0])]


def decode_detections(y_pred, confidence_thresh=0.01, iou_threshold=0.45, top_k=200, input_coords='centroids',
                      normalize_coords=True, img_height=None, img_width=None, border_pixels='half'):
    """Reference :111-226.  Returns a list of ``(k_i, 6)`` float64 arrays ``[class, conf, xmin, ymin, xmax, ymax]``.
    When more than ``top_k`` boxes survive, the reference keeps an unordered top-k set (``argpartition``);
    here that set comes back sorted by confidence."""
    _check_norm(normalize_coords, img_height, img_width)
    _check_coords(input_coords, "Unexpected value for `input_coords`. Supported input coordinate formats are 'minmax', 'corners' "
                                "and 'centroids'.")                                                   # reference :192
    out, counts = decode_device(_to_device(y_pred), PER_CLASS, False, confidence_thresh, iou_threshold, top_k, 0,
                                input_coords, normalize_coords, img_height, img_width, border_pixels)
    return _ragged(out, counts)


def decode_detections_fast(y_pred, confidence_thresh=0.5, iou_threshold=0.45, top_k='all', input_coords='centroids',
                           normalize_coords=True, img_height=None, img_width=None, border_pixels='half'):
    """Reference :228-333 (class = argmax, one NMS over all classes, ``>=`` confidence test)."""
    _check_norm(normalize_coords, img_height, img_width)
    _check_coords(input_coords, "Unexpected value for `coords`. Supported values are 'minmax', 'corners' and 'centroids'.")  # :314
    out, counts = decode_device(_to_device(y_pred), FAST, False, confidence_thresh, iou_threshold, top_k, 0,
                                input_coords, normalize_coords, img_height, img_width, border_pixels)
    res = _ragged(out, counts)
    return [r if r.size else np.zeros((0, 6)) for r in res]


def nms_device(boxes, scores, confidence_thresh=0.01, iou_threshold=0.45, nms_max_output_size=400, top_k=200,
               return_index=False):
    """Single-class greedy NMS + top-k on CUDA tensors: boxes (B,n,4) corners, scores (B,n)."""
    import torch
    B, n = scores.shape
    out = torch.empty((B, top_k, 6), dtype=torch.float32, device=scores.device)
    counts = torch.empty((B,), dtype=torch.int32, device=scores.device)
    index = torch.empty((B, top_k), dtype=torch.int32, device=scores.device) if return_index else None
    _ffi.check(_ffi.lib().ssdk_nms(_ffi.context(scores.device.index), _ffi.dptr(boxes.contiguous()), _ffi.dptr(scores.contiguous()),
                                   B, n, float(confidence_thresh), float(iou_threshold), int(nms_max_output_size), int(top_k),
                                   _ffi.dptr(out), _ffi.dptr(counts), _ffi.dptr(index), _ffi.stream_ptr()))
    return (out, counts, index) if return_index else (out, counts)


# ---------------------------------------------------------------------------------------------
# debug / stand-alone utilities of the reference module (:27-75, :342-530)
# ---------------------------------------------------------------------------------------------
def decode_detections_debug(y_pred, confidence_thresh=0.01, iou_threshold=0.45, top_k=200, input_coords='centroids',
                            normalize_coords=True, img_height=None, img_width=None, variance_encoded_in_target=False,
                            border_pixels='half'):
    """Reference :342-455: ``decode_detections`` with the index of the prior that made each detection prepended,
    rows ``[box_id, class_id, confidence, xmin, ymin, xmax, ymax]``.  Same kernels as ``decode_detections`` -- the
    prior index is carried through the NMS and top-k stages (``out_index`` of ``ssdk_decode``)."""
    _check_norm(normalize_coords, img_height, img_width)
    _check_coords(input_coords, "Unexpected value for `input_coords`. Supported input coordinate formats are 'minmax', 'corners' "
                                "and 'centroids'.")
    y = _to_device(y_pred)
    if variance_encoded_in_target and input_coords == 'centroids':
        # :404-406: the offsets are used without the variances == the usual formula with variances of exactly 1
        y = y.clone()
        y[:, :, -4:] = 1.0
    out, counts, index = decode_device(y, PER_CLASS, False, confidence_thresh, iou_threshold, top_k, 0, input_coords,
                                       normalize_coords, img_height, img_width, border_pixels, return_index=True)
    out = out.cpu().numpy().astype(np.float64)
    counts = counts.cpu().numpy()
    index = index.cpu().numpy()
    res = []
    for i in range(out.shape[0]):
        k = int(counts[i])
        res.append(np.concatenate([index[i, :k, None].astype(np.float64), out[i, :k]], axis=1) if k > 0 else np.zeros((0, 7)))
    return res


def get_num_boxes_per_pred_layer(predictor_sizes, aspect_ratios, two_boxes_for_ar1):
    """Reference :488-501 (note: like the reference, one extra box per cell whenever ``two_boxes_for_ar1`` is set)."""
    out = []
    for i in range(len(predictor_sizes)):
        n = len(aspect_ratios[i]) + (1 if two_boxes_for_ar1 else 0)
        out.append(predictor_sizes[i][0] * predictor_sizes[i][1] * n)
    return out


def get_pred_layers(y_pred_decoded, num_boxes_per_pred_layer):
    """Reference :503-530: for predictions decoded with ``decode_detections_debug``, the index of the predictor layer that
    made each of them."""
    cum = np.cumsum(num_boxes_per_pred_layer)
    res = []
    for batch_item in y_pred_decoded:
        ids = np.asarray(batch_item, dtype=np.float64).reshape(-1, 7)[:, 0] if np.size(batch_item) else np.zeros((0,))
        if np.any(ids < 0) or np.any(ids >= cum[-1]):
            raise ValueError("Box index is out of bounds of the possible indices as given by the values in `num_boxes_per_pred_layer`.")
        res.append([int(v) for v in np.searchsorted(cum, ids, side='right')])
    return res


def greedy_nms(y_pred_decoded, iou_threshold=0.45, coords='corners', border_pixels='half'):
    """Reference :27-75: greedy NMS over already decoded predictions, one ``(k, 6)`` array ``[class_id, score, 4 coordinates]``
    per batch item; the score column decides, class ids are ignored, boxes with IoU <= ``iou_threshold`` to every kept
    box survive.  Host loop like the reference, the element-wise IoU of every round is ``ssdk_iou`` (float64, the
    reference's arithmetic incl. the border_pixels quirk); a utility, not part of the decode hot path."""
    from ..bounding_box_utils.bounding_box_utils import iou
    res = []
    for batch_item in y_pred_decoded:
        boxes_left = np.array(batch_item, dtype=np.float64, copy=True).reshape(-1, np.shape(batch_item)[-1] if np.ndim(batch_item) > 1 else 6)
        maxima = []
        while boxes_left.shape[0] > 0:
            m = int(np.argmax(boxes_left[:, 1]))
            box = boxes_left[m].copy()
            maxima.append(box)
            boxes_left = np.delete(boxes_left, m, axis=0)
            if boxes_left.shape[0] == 0:
                break
            sim = iou(boxes_left[:, 2:], box[2:], coords=coords, mode='element-wise', border_pixels=border_pixels)
            boxes_left = boxes_left[sim <= iou_threshold]
        res.append(np.array(maxima))
    return res
