"""Prediction decoders (oracle).

NumPy API (pinned against the real reference by make_golden.py):
  * ``decode_detections``       ssd_encoder_decoder/ssd_output_decoder.py:111-226 (+ ``_greedy_nms`` :77-92)
  * ``decode_detections_fast``  :228-333 (+ ``_greedy_nms2`` :94-109)
  * ``greedy_nms``              :27-75

Keras-layer semantics (TensorFlow 1.x is not installable here; pinned against the reference's own layer source run over
a NumPy stand-in for the TF primitives -- tests/golden/make_tf_golden.py, tests/test_oracle_tf_shim_golden.py: classes,
confidences, row order and padding exact):
  * ``decode_layer``       keras_layers/keras_layer_DecodeDetections.py:109-265
  * ``decode_layer_fast``  keras_layers/keras_layer_DecodeDetectionsFast.py:111-248
  They restate float32 arithmetic plus the published behaviour of
  ``tf.image.non_max_suppression`` (greedy, descending score, suppress iff IoU > thr,
  IoU of a non-positive-area box = 0, stops at max_output_size; ties -> lower index,
  the rule TF adopted explicitly in later releases) and ``tf.nn.top_k`` (ties -> lower index).
  Cross-pinned (tests/test_oracle_layer_vs_reference_cpu.py): on the golden y_pred tensors they return the same detections
  as the real reference's NumPy twins above; what stays unpinned is TensorFlow-specific behaviour the twins do not share
  (the nms_max_output_size cap, tie order, NaN handling, float32 rounding at the thresholds).
"""
import numpy as np

from .boxes import convert_coordinates, iou


# --------------------------------------------------------------------------------------
# NumPy API
# --------------------------------------------------------------------------------------

def _nms_rows(rows, score_col, box_col, iou_threshold, coords, border_pixels):
    """_greedy_nms / _greedy_nms2 (:77-109): pick first argmax, drop everything with
    IoU > thr (``similarities <= iou_threshold`` keeps; NaN is dropped)."""
    left = np.copy(rows)
    keep = []
    while left.shape[0] > 0:
        m = int(np.argmax(left[:, score_col]))
        best = np.copy(left[m])
        keep.append(best)
        left = np.delete(left, m, axis=0)
        if left.shape[0] == 0:
            break
        sim = iou(left[:, box_col:], best[box_col:], coords=coords, mode='element-wise',
                  border_pixels=border_pixels)
        left = left[sim <= iou_threshold]
    return np.array(keep)


def greedy_nms(y_pred_decoded, iou_threshold=0.45, coords='corners', border_pixels='half'):
    """ssd_output_decoder.py:27-75; rows are [class, score, 4 coords]."""
    return [_nms_rows(item, 1, 2, iou_threshold, coords, border_pixels) for item in y_pred_decoded]


def exp_cr(x):
    """float32 ``exp`` rounded once from float64 -- what the CUDA decoder computes (``exp_cr`` in csrc/decode.cu).  NumPy's own
    float32 ``np.exp`` may differ from it by an ulp or two; pass this as ``exp=`` to hold the kernels to the bit."""
    x = np.asarray(x)
    with np.errstate(over='ignore'):
        return np.exp(x.astype(np.float64)).astype(x.dtype)


def _decode_boxes_inplace(dst, y_pred, input_coords, cols, exp=np.exp):
    """Shared arithmetic of :174-190 / :296-312; ``cols`` = the four destination columns."""
    c0, c1, c2, c3 = cols
    if input_coords == 'centroids':
        dst[:, :, [c2, c3]] = exp(dst[:, :, [c2, c3]] * y_pred[:, :, [-2, -1]])
        dst[:, :, [c2, c3]] *= y_pred[:, :, [-6, -5]]
        dst[:, :, [c0, c1]] *= y_pred[:, :, [-4, -3]] * y_pred[:, :, [-6, -5]]
        dst[:, :, [c0, c1]] += y_pred[:, :, [-8, -7]]
        return convert_coordinates(dst, start_index=-4, conversion='centroids2corners')
    if input_coords == 'minmax':
        dst[:, :, c0:] *= y_pred[:, :, -4:]
        dst[:, :, [c0, c1]] *= (y_pred[:, :, -7] - y_pred[:, :, -8])[..., None]
        dst[:, :, [c2, c3]] *= (y_pred[:, :, -5] - y_pred[:, :, -6])[..., None]
        dst[:, :, c0:] += y_pred[:, :, -8:-4]
        return convert_coordinates(dst, start_index=-4, conversion='minmax2corners')
    if input_coords == 'corners':
        dst[:, :, c0:] *= y_pred[:, :, -4:]
        dst[:, :, [c0, c2]] *= (y_pred[:, :, -6] - y_pred[:, :, -8])[..., None]
        dst[:, :, [c1, c3]] *= (y_pred[:, :, -5] - y_pred[:, :, -7])[..., None]
        dst[:, :, c0:] += y_pred[:, :, -8:-4]
        return dst
    raise ValueError("Unexpected value for `input_coords`. Supported input coordinate formats are "
                     "'minmax', 'corners' and 'centroids'.")


def decode_detections(y_pred, confidence_thresh=0.01, iou_threshold=0.45, top_k=200, input_coords='centroids',
                      normalize_coords=True, img_height=None, img_width=None, border_pixels='half', exp=np.exp,
                      return_index=False):
    """ssd_output_decoder.py:111-226.  ``return_index`` also returns, per image, the prior index of every row."""
    if normalize_coords and (img_height is None or img_width is None):
        raise ValueError("If relative box coordinates are supposed to be converted to absolute coordinates, the "
                         "decoder needs the image size in order to decode the predictions, but `img_height == {}` "
                         "and `img_width == {}`".format(img_height, img_width))
    y_pred = np.asarray(y_pred)
    raw = np.copy(y_pred[:, :, :-8])                                          # :172
    n_cols = raw.shape[2]
    raw = _decode_boxes_inplace(raw, y_pred, input_coords, (n_cols - 4, n_cols - 3, n_cols - 2, n_cols - 1), exp)
    if normalize_coords:                                                      # :196-198
        raw[:, :, [-4, -2]] *= img_width
        raw[:, :, [-3, -1]] *= img_height
    n_classes = raw.shape[-1] - 4
    out, out_idx = [], []
    for item in raw:                                                          # :205
        per_class, per_idx = [], []
        prior = np.arange(item.shape[0]).astype(item.dtype)[:, None]          # carried along in front of the score
        for cid in range(1, n_classes):                                       # :207
            rows = np.concatenate([prior, item[:, [cid, -4, -3, -2, -1]]], axis=1)
            rows = rows[rows[:, 1] > confidence_thresh]                       # :209 (strict)
            if rows.shape[0] > 0:
                kept = _nms_rows(rows, 1, 2, iou_threshold, 'corners', border_pixels)
                block = np.zeros((kept.shape[0], 6))
                block[:, 0] = cid
                block[:, 1:] = kept[:, 1:]
                per_class.append(block)
                per_idx.append(kept[:, 0].astype(np.int64))
        if per_class:
            pred = np.concatenate(per_class, axis=0)
            pidx = np.concatenate(per_idx)
            if top_k != 'all' and pred.shape[0] > top_k:                      # :219-221 (unordered)
                sel = np.argpartition(pred[:, 1], kth=pred.shape[0] - top_k, axis=0)[pred.shape[0] - top_k:]
                pred, pidx = pred[sel], pidx[sel]
        else:
            pred = np.array(per_class)                                        # :223 -> shape (0,)
            pidx = np.zeros((0,), np.int64)
        out.append(pred)
        out_idx.append(pidx)
    return (out, out_idx) if return_index else out


def decode_detections_fast(y_pred, confidence_thresh=0.5, iou_threshold=0.45, top_k='all',
                           input_coords='centroids', normalize_coords=True, img_height=None, img_width=None,
                           border_pixels='half', exp=np.exp, return_index=False):
    """ssd_output_decoder.py:228-333.  ``return_index`` also returns, per image, the prior index of every row."""
    if normalize_coords and (img_height is None or img_width is None):
        raise ValueError("If relative box coordinates are supposed to be converted to absolute coordinates, the "
                         "decoder needs the image size in order to decode the predictions, but `img_height == {}` "
                         "and `img_width == {}`".format(img_height, img_width))
    y_pred = np.asarray(y_pred)
    conv = np.copy(y_pred[:, :, -14:-8])                                      # :291
    conv[:, :, 0] = np.argmax(y_pred[:, :, :-12], axis=-1)                    # :292
    conv[:, :, 1] = np.amax(y_pred[:, :, :-12], axis=-1)                      # :293
    conv = _decode_boxes_inplace(conv, y_pred, input_coords, (2, 3, 4, 5), exp)
    if normalize_coords:                                                      # :317-319
        conv[:, :, [2, 4]] *= img_width
        conv[:, :, [3, 5]] *= img_height
    out, out_idx = [], []
    for item in conv:
        prior = np.arange(item.shape[0])
        keep = np.nonzero(item[:, 0])[0]                                      # :324
        boxes, prior = item[keep], prior[keep]
        keep = boxes[:, 1] >= confidence_thresh                               # :325 (non-strict)
        boxes, prior = boxes[keep], prior[keep]
        if iou_threshold:                                                     # :326
            # the prior index rides in the class column, which the NMS does not read (the class comes back below)
            rows = np.concatenate([prior.astype(boxes.dtype)[:, None], boxes[:, 1:]], axis=1)
            kept = _nms_rows(rows, 1, 2, iou_threshold, 'corners', border_pixels)
            if kept.size:
                prior = kept[:, 0].astype(np.int64)
                boxes = item[prior]
            else:
                boxes, prior = kept, prior[:0]
        if top_k != 'all' and boxes.shape[0] > top_k:                         # :328-330
            sel = np.argpartition(boxes[:, 1], kth=boxes.shape[0] - top_k, axis=0)[boxes.shape[0] - top_k:]
            boxes, prior = boxes[sel], prior[sel]
        out.append(boxes)
        out_idx.append(prior)
    return (out, out_idx) if return_index else out


# --------------------------------------------------------------------------------------
# Keras-layer semantics (float32)
# --------------------------------------------------------------------------------------

def _smin(a, b):
    """std::min<float>(a, b) == (b < a) ? b : a -- NaN handling depends on the argument order, as in the TF kernel."""
    return np.where(b < a, b, a)


def _smax(a, b):
    """std::max<float>(a, b) == (a < b) ? b : a."""
    return np.where(a < b, b, a)


def _tf_iou(bi, bj):
    """IoU as tf.image.non_max_suppression computes it (float32), bi = candidate, bj = already selected box.
    Boxes are (ymin,xmin,ymax,xmax) in TF; here (x0,y0,x1,y1) with the same per-axis argument order."""
    f = np.float32
    with np.errstate(all='ignore'):
        bi = np.asarray(bi, f); bj = np.asarray(bj, f)
        x0i, x1i = _smin(bi[0], bi[2]), _smax(bi[0], bi[2]); y0i, y1i = _smin(bi[1], bi[3]), _smax(bi[1], bi[3])
        x0j, x1j = _smin(bj[0], bj[2]), _smax(bj[0], bj[2]); y0j, y1j = _smin(bj[1], bj[3]), _smax(bj[1], bj[3])
        ai = f(f(y1i - y0i) * f(x1i - x0i))
        aj = f(f(y1j - y0j) * f(x1j - x0j))
        if ai <= 0 or aj <= 0:
            return f(0.0)
        ih = _smax(f(_smin(y1i, y1j) - _smax(y0i, y0j)), f(0.0))
        iw = _smax(f(_smin(x1i, x1j) - _smax(x0i, x0j)), f(0.0))
        inter = f(ih * iw)
        return f(inter / f(f(ai + aj) - inter))


def tf_nms(boxes, scores, max_output_size, iou_threshold):
    """tf.image.non_max_suppression restated: returns selected indices in selection order."""
    order = sorted(range(len(scores)), key=lambda i: (-float(scores[i]), i))
    selected = []
    thr = np.float32(iou_threshold)
    for i in order:
        if len(selected) >= max_output_size:
            break
        ok = True
        for j in reversed(selected):
            if _tf_iou(boxes[i], boxes[j]) > thr:
                ok = False
                break
        if ok:
            selected.append(i)
    return selected


def tf_nms_fast(boxes, scores, max_output_size, iou_threshold):
    """Vectorised equivalent of ``tf_nms`` (same float32 formula and min/max argument order) for larger inputs."""
    f = np.float32
    boxes = np.asarray(boxes, dtype=f)
    scores = np.asarray(scores, dtype=f)
    n = len(scores)
    order = np.lexsort((np.arange(n), -scores.astype(np.float64)))
    with np.errstate(all='ignore'):
        x0 = _smin(boxes[:, 0], boxes[:, 2]); x1 = _smax(boxes[:, 0], boxes[:, 2])
        y0 = _smin(boxes[:, 1], boxes[:, 3]); y1 = _smax(boxes[:, 1], boxes[:, 3])
        area = ((y1 - y0).astype(f) * (x1 - x0).astype(f)).astype(f)
        alive = np.ones(n, dtype=bool)
        selected = []
        thr = f(iou_threshold)
        for r, i in enumerate(order):          # i is the SELECTED box (j in TF); the remaining ones are candidates
            if not alive[i]:
                continue
            selected.append(int(i))
            if len(selected) >= max_output_size:
                break
            rest = order[r + 1:]
            rest = rest[alive[rest]]
            if rest.size == 0:
                continue
            ih = _smax((_smin(y1[rest], y1[i]) - _smax(y0[rest], y0[i])).astype(f), f(0))
            iw = _smax((_smin(x1[rest], x1[i]) - _smax(x0[rest], x0[i])).astype(f), f(0))
            inter = (ih * iw).astype(f)
            v = (inter / ((area[rest] + area[i]).astype(f) - inter).astype(f)).astype(f)
            v = np.where((area[rest] <= 0) | (area[i] <= 0), f(0), v)
            alive[rest[v > thr]] = False
    return selected


def tf_nms_c(boxes, scores, max_output_size, iou_threshold):
    """``tf_nms`` through the C restatement oracle/tf_nms.c (compiled by oracle/cbuild.py); falls back to ``tf_nms_fast`` where no
    compiler exists.  Bit-identical to both (tests/test_oracle_c_nms_cpu.py); what bench.py's CPU arm times."""
    import ctypes as C
    from .cbuild import tf_nms_lib
    try:
        lib = tf_nms_lib()
    except (OSError, RuntimeError):
        lib = None
    if lib is None:
        return tf_nms_fast(boxes, scores, max_output_size, iou_threshold)
    b = np.ascontiguousarray(boxes, dtype=np.float32).reshape(-1, 4)
    sc = np.ascontiguousarray(scores, dtype=np.float32).reshape(-1)
    out = np.empty(max(int(max_output_size), 1), np.int32)
    k = lib.tf_nms_f32(b.ctypes.data_as(C.POINTER(C.c_float)), sc.ctypes.data_as(C.POINTER(C.c_float)), int(sc.shape[0]),
                       int(max_output_size), C.c_float(np.float32(iou_threshold)), out.ctypes.data_as(C.POINTER(C.c_int)))
    if k < 0:
        raise MemoryError('tf_nms_f32')
    return [int(v) for v in out[:k]]


def _layer_boxes(y_pred, normalize_coords, img_height, img_width, exp=np.exp):
    """keras_layer_DecodeDetections.py:124-146 in float32."""
    f = np.float32
    y = np.asarray(y_pred, dtype=f)
    cx = (y[..., -12] * y[..., -4] * y[..., -6] + y[..., -8]).astype(f)
    cy = (y[..., -11] * y[..., -3] * y[..., -5] + y[..., -7]).astype(f)
    w = (exp(y[..., -10] * y[..., -2]).astype(f) * y[..., -6]).astype(f)
    h = (exp(y[..., -9] * y[..., -1]).astype(f) * y[..., -5]).astype(f)
    xmin = (cx - f(0.5) * w).astype(f); ymin = (cy - f(0.5) * h).astype(f)
    xmax = (cx + f(0.5) * w).astype(f); ymax = (cy + f(0.5) * h).astype(f)
    if normalize_coords:
        xmin = (xmin * f(img_width)).astype(f); xmax = (xmax * f(img_width)).astype(f)
        ymin = (ymin * f(img_height)).astype(f); ymax = (ymax * f(img_height)).astype(f)
    return np.stack([xmin, ymin, xmax, ymax], axis=-1)


def _topk_pad(rows, top_k):
    """:238-251: pad with zero rows to >= top_k, then top_k by confidence, sorted desc, ties -> lower row."""
    rows = np.asarray(rows, dtype=np.float32).reshape(-1, 6)
    if rows.shape[0] < top_k:
        rows = np.concatenate([rows, np.zeros((top_k - rows.shape[0], 6), np.float32)], axis=0)
    order = np.lexsort((np.arange(rows.shape[0]), -rows[:, 1].astype(np.float64)))[:top_k]
    return rows[order]


def decode_layer(y_pred, confidence_thresh=0.01, iou_threshold=0.45, top_k=200, nms_max_output_size=400,
                 normalize_coords=True, img_height=None, img_width=None, return_indices=False, nms=None, exp=np.exp):
    """DecodeDetections.call, keras_layer_DecodeDetections.py:109-265 -> (B, top_k, 6) float32.

    ``return_indices`` also returns, per image, the prior index of every output row (-1 for padding)."""
    f = np.float32
    y = np.asarray(y_pred, dtype=f)
    boxes = _layer_boxes(y, normalize_coords, img_height, img_width, exp)
    B, P = y.shape[0], y.shape[1]
    n_classes = y.shape[2] - 12
    out = np.zeros((B, top_k, 6), f)
    out_idx = np.full((B, top_k), -1, np.int64)
    for b in range(B):
        rows, ridx = [], []
        for c in range(1, n_classes):                                          # :219, class-major
            conf = y[b, :, c]
            m = np.nonzero(conf > f(confidence_thresh))[0]                     # :180 strict
            blk = np.zeros((nms_max_output_size, 6), f)                        # :211-214 pad to 400 rows
            bidx = np.full(nms_max_output_size, -1, np.int64)
            if m.size:
                sel = (nms or tf_nms_fast)(boxes[b, m], conf[m], nms_max_output_size, iou_threshold)
                k = len(sel)
                blk[:k, 0] = c
                blk[:k, 1] = conf[m][sel]
                blk[:k, 2:] = boxes[b, m][sel]
                bidx[:k] = m[sel]
            rows.append(blk); ridx.append(bidx)
        rows = np.concatenate(rows, axis=0); ridx = np.concatenate(ridx)
        if rows.shape[0] < top_k:
            pad = top_k - rows.shape[0]
            rows = np.concatenate([rows, np.zeros((pad, 6), f)]); ridx = np.concatenate([ridx, np.full(pad, -1)])
        order = np.lexsort((np.arange(rows.shape[0]), -rows[:, 1].astype(np.float64)))[:top_k]
        out[b] = rows[order]; out_idx[b] = ridx[order]
    return (out, out_idx) if return_indices else out


def decode_layer_fast(y_pred, confidence_thresh=0.01, iou_threshold=0.45, top_k=200, nms_max_output_size=400,
                      normalize_coords=True, img_height=None, img_width=None, return_indices=False, nms=None, exp=np.exp):
    """DecodeDetectionsFast.call, keras_layer_DecodeDetectionsFast.py:111-248 -> (B, top_k, 6) float32."""
    f = np.float32
    y = np.asarray(y_pred, dtype=f)
    boxes = _layer_boxes(y, normalize_coords, img_height, img_width, exp)
    cls = np.argmax(y[..., :-12], axis=-1)                                     # :126 (first index on ties)
    conf = np.max(y[..., :-12], axis=-1)                                       # :128
    B = y.shape[0]
    out = np.zeros((B, top_k, 6), f)
    out_idx = np.full((B, top_k), -1, np.int64)
    for b in range(B):
        m = np.nonzero((cls[b] != 0) & (conf[b] > f(confidence_thresh)))[0]    # :174,:180 (strict)
        rows = np.zeros((0, 6), f); ridx = np.zeros((0,), np.int64)
        if m.size:
            sel = (nms or tf_nms_fast)(boxes[b, m], conf[b, m], nms_max_output_size, iou_threshold)
            rows = np.zeros((len(sel), 6), f)
            rows[:, 0] = cls[b, m][sel]; rows[:, 1] = conf[b, m][sel]; rows[:, 2:] = boxes[b, m][sel]
            ridx = m[sel]
        if rows.shape[0] < top_k:
            pad = top_k - rows.shape[0]
            rows = np.concatenate([rows, np.zeros((pad, 6), f)]); ridx = np.concatenate([ridx, np.full(pad, -1)])
        order = np.lexsort((np.arange(rows.shape[0]), -rows[:, 1].astype(np.float64)))[:top_k]
        out[b] = rows[order]; out_idx[b] = ridx[order]
    return (out, out_idx) if return_indices else out
