"""``Evaluator`` on H100 (reference ``eval_utils/average_precision_evaluator.py:36-905``): Pascal-VOC average precision.

The expensive step of the reference is ``match_predictions`` (:538-736): for every class, a Python loop over all predictions in
descending confidence with an element-wise ``iou`` against the ground truth of the prediction's image.  Here it is two stable
key sorts plus ``ssdk_eval_match`` (one warp per (class, image) pair, float64 IoU with the reference's arithmetic) and
``ssdk_eval_cumsum``; precision / recall / AP (:738-905) are the reference's NumPy expressions on the cumulative counts.

What the class needs from ``data_generator`` is what the reference reads from its ``DataGenerator``: ``labels`` (list of
``(k_i, 5)`` arrays), ``image_ids`` and optionally ``eval_neutral``; for ``predict_on_dataset`` additionally ``images`` (a
sequence of HxWx3 arrays already at the model's input size -- dataset parsing and resizing belong to the out-of-scope
``data_generator`` package).

Note on a reference quirk: with ``verbose=False`` the reference iterates ``range(len(predictions.shape))`` (:641), i.e. it
matches only the first prediction of every class.  This implementation always matches all of them (the ``verbose=True``
behaviour)."""
import ctypes as C

import numpy as np

from .. import _ffi


class Evaluator:

    def __init__(self, model, n_classes, data_generator, model_mode='inference',
                 pred_format={'class_id': 0, 'conf': 1, 'xmin': 2, 'ymin': 3, 'xmax': 4, 'ymax': 5},
                 gt_format={'class_id': 0, 'xmin': 1, 'ymin': 2, 'xmax': 3, 'ymax': 4}):
        if model_mode not in ('inference', 'training'):
            raise ValueError("`model_mode` can be either 'training' or 'inference', but received '{}'.".format(model_mode))
        self.model = model
        self.data_generator = data_generator
        self.n_classes = n_classes
        self.model_mode = model_mode
        self.pred_format = pred_format
        self.gt_format = gt_format
        self.prediction_results = None
        self.num_gt_per_class = None
        self.true_positives = None
        self.false_positives = None
        self.cumulative_true_positives = None
        self.cumulative_false_positives = None
        self.cumulative_precisions = None
        self.cumulative_recalls = None
        self.average_precisions = None
        self.mean_average_precision = None

    def __call__(self, img_height, img_width, batch_size, data_generator_mode='resize', round_confidences=False,
                 matching_iou_threshold=0.5, border_pixels='include', sorting_algorithm='quicksort', average_precision_mode='sample',
                 num_recall_points=11, ignore_neutral_boxes=True, return_precisions=False, return_recalls=False,
                 return_average_precisions=False, verbose=True, decoding_confidence_thresh=0.01, decoding_iou_threshold=0.45,
                 decoding_top_k=200, decoding_pred_coords='centroids', decoding_normalize_coords=True):
        """Reference :94-256: predict, match, precision / recall, average precisions, mAP."""
        self.predict_on_dataset(img_height=img_height, img_width=img_width, batch_size=batch_size,
                                data_generator_mode=data_generator_mode, decoding_confidence_thresh=decoding_confidence_thresh,
                                decoding_iou_threshold=decoding_iou_threshold, decoding_top_k=decoding_top_k,
                                decoding_pred_coords=decoding_pred_coords, decoding_normalize_coords=decoding_normalize_coords,
                                decoding_border_pixels=border_pixels, round_confidences=round_confidences, verbose=verbose, ret=False)
        self.get_num_gt_per_class(ignore_neutral_boxes=ignore_neutral_boxes, verbose=False, ret=False)
        self.match_predictions(ignore_neutral_boxes=ignore_neutral_boxes, matching_iou_threshold=matching_iou_threshold,
                               border_pixels=border_pixels, sorting_algorithm=sorting_algorithm, verbose=verbose, ret=False)
        self.compute_precision_recall(verbose=verbose, ret=False)
        self.compute_average_precisions(mode=average_precision_mode, num_recall_points=num_recall_points, verbose=verbose, ret=False)
        mean_average_precision = self.compute_mean_average_precision(ret=True)
        if return_precisions or return_recalls or return_average_precisions:
            ret = [mean_average_precision]
            if return_average_precisions:
                ret.append(self.average_precisions)
            if return_precisions:
                ret.append(self.cumulative_precisions)
            if return_recalls:
                ret.append(self.cumulative_recalls)
            return ret
        return mean_average_precision

    # -- predictions ----------------------------------------------------------------------------
    def predict_on_dataset(self, img_height, img_width, batch_size, data_generator_mode='resize', decoding_confidence_thresh=0.01,
                           decoding_iou_threshold=0.45, decoding_top_k=200, decoding_pred_coords='centroids',
                           decoding_normalize_coords=True, decoding_border_pixels='include', round_confidences=False, verbose=True,
                           ret=False):
        """Reference :258-448 for images that already have the model's input size (``data_generator.images``): forward pass,
        decoding (the model's own decoder in 'inference' mode, ``decode_detections`` in 'training' mode), results per class as
        ``(image_id, confidence, xmin, ymin, xmax, ymax)`` tuples."""
        from ..ssd_encoder_decoder.ssd_output_decoder import decode_detections
        images = getattr(self.data_generator, 'images', None)
        if images is None:
            raise ValueError("`data_generator.images` is needed to predict: a sequence of images at the model's input size.")
        ids = list(self.data_generator.image_ids)
        results = [list() for _ in range(self.n_classes + 1)]
        cid, conf = self.pred_format['class_id'], self.pred_format['conf']
        xs = [self.pred_format[k] for k in ('xmin', 'ymin', 'xmax', 'ymax')]
        for lo in range(0, len(images), batch_size):
            batch = np.asarray(images[lo:lo + batch_size], dtype=np.float32)
            if batch.shape[1] != img_height or batch.shape[2] != img_width:
                raise ValueError('images must already have the size (%d, %d)' % (img_height, img_width))
            y = self.model.predict(batch)
            if self.model_mode == 'inference':
                dets = [y[k][y[k, :, 0] != 0] for k in range(y.shape[0])]       # drop the zero padding (reference :388-396)
            else:
                dets = decode_detections(y, confidence_thresh=decoding_confidence_thresh, iou_threshold=decoding_iou_threshold,
                                         top_k=decoding_top_k, input_coords=decoding_pred_coords,
                                         normalize_coords=decoding_normalize_coords, img_height=img_height, img_width=img_width,
                                         border_pixels=decoding_border_pixels)
            for k, d in enumerate(dets):
                image_id = ids[lo + k]
                for box in np.asarray(d).reshape(-1, 6):
                    c = float(box[conf])
                    if round_confidences:
                        c = round(c, round_confidences)
                    results[int(box[cid])].append((image_id, c, round(float(box[xs[0]]), 1), round(float(box[xs[1]]), 1),
                                                   round(float(box[xs[2]]), 1), round(float(box[xs[3]]), 1)))
        self.prediction_results = results
        if ret:
            return results

    def get_num_gt_per_class(self, ignore_neutral_boxes=True, verbose=False, ret=False):
        """Reference :490-536."""
        if self.data_generator.labels is None:
            raise ValueError("Computing the number of ground truth boxes per class not possible, no ground truth given.")
        num = np.zeros(shape=(self.n_classes + 1), dtype=int)
        ci = self.gt_format['class_id']
        neutral = getattr(self.data_generator, 'eval_neutral', None)
        for i, boxes in enumerate(self.data_generator.labels):
            boxes = np.asarray(boxes)
            if boxes.size == 0:
                continue
            cls = boxes[:, ci].astype(int)
            if ignore_neutral_boxes and neutral is not None:
                cls = cls[~np.asarray(neutral[i], dtype=bool)]
            np.add.at(num, cls, 1)
        self.num_gt_per_class = num
        if ret:
            return num

    # -- matching (GPU) ---------------------------------------------------------------------------
    def match_predictions(self, ignore_neutral_boxes=True, matching_iou_threshold=0.5, border_pixels='include',
                          sorting_algorithm='quicksort', verbose=True, ret=False):
        """Reference :538-736.  Equal confidences keep their input order (the reference's 'mergesort' option; its default
        'quicksort' leaves the order of ties unspecified)."""
        import torch
        if self.data_generator.labels is None:
            raise ValueError("Matching predictions to ground truth boxes not possible, no ground truth given.")
        if self.prediction_results is None:
            raise ValueError("There are no prediction results. You must run `predict_on_dataset()` before calling this method.")
        if border_pixels not in _ffi.BORDER_D:
            raise ValueError("`border_pixels` must be one of 'half', 'include', 'exclude'.")
        nC = self.n_classes
        id_index = {str(i): k for k, i in enumerate(self.data_generator.image_ids)}
        # ground truth -> packed float64 rows in the column order (class, xmin, ymin, xmax, ymax)
        cols = [self.gt_format[k] for k in ('class_id', 'xmin', 'ymin', 'xmax', 'ymax')]
        rows, offs = [], [0]
        for lab in self.data_generator.labels:
            lab = np.asarray(lab, dtype=np.float64)
            lab = lab.reshape(-1, lab.shape[-1])[:, cols] if lab.size else np.zeros((0, 5))
            rows.append(lab); offs.append(offs[-1] + lab.shape[0])
        gt = np.concatenate(rows, axis=0) if offs[-1] else np.zeros((1, 5))
        neutral = getattr(self.data_generator, 'eval_neutral', None)
        use_neutral = ignore_neutral_boxes and neutral is not None
        # predictions -> flat arrays, class-major, input order inside a class
        counts = [len(self.prediction_results[c]) for c in range(nC + 1)]
        counts[0] = 0
        n = int(sum(counts))
        tp_all = [[]] + [np.zeros(counts[c], dtype=int) for c in range(1, nC + 1)]
        fp_all = [[]] + [np.zeros(counts[c], dtype=int) for c in range(1, nC + 1)]
        ctp_all = [[]] + [np.zeros(counts[c], dtype=int) for c in range(1, nC + 1)]
        cfp_all = [[]] + [np.zeros(counts[c], dtype=int) for c in range(1, nC + 1)]
        if n:
            img = np.empty(n, np.int32); cls = np.empty(n, np.int32); conf = np.empty(n, np.float32); box = np.empty((n, 4), np.float32)
            o = 0
            for c in range(1, nC + 1):
                for p in self.prediction_results[c]:
                    img[o] = id_index[str(p[0])]; cls[o] = c; conf[o] = p[1]; box[o] = p[2:6]
                    o += 1
            dev = 'cuda'
            t_img, t_cls = torch.from_numpy(img).to(dev), torch.from_numpy(cls).to(dev)
            t_conf, t_box = torch.from_numpy(conf).to(dev), torch.from_numpy(box).to(dev)
            # order 1: (class, confidence desc), stable: two stable sorts, least significant key first
            ord_conf = torch.sort(-t_conf, stable=True).indices                 # by confidence desc (ties keep the input order)
            ord1 = ord_conf[torch.sort(t_cls[ord_conf].long(), stable=True).indices]     # then by class (stable): (class, conf desc)
            rank = torch.empty(n, dtype=torch.int32, device=dev)
            rank[ord1] = torch.arange(n, dtype=torch.int32, device=dev)
            # order 2: (class, image, confidence desc): a stable sort of order 1 by image inside each class
            key2 = t_cls[ord1].long() * (len(id_index) + 1) + t_img[ord1].long()
            ord2 = ord1[torch.sort(key2, stable=True).indices]
            k2 = t_cls[ord2].long() * (len(id_index) + 1) + t_img[ord2].long()
            start = torch.ones(n, dtype=torch.bool, device=dev)
            start[1:] = k2[1:] != k2[:-1]
            seg = torch.cat([torch.nonzero(start).flatten().int(), torch.tensor([n], dtype=torch.int32, device=dev)]).contiguous()
            n_seg = int(seg.numel()) - 1
            p_img, p_cls = t_img[ord2].contiguous(), t_cls[ord2].contiguous()
            p_box, p_rank = t_box[ord2].contiguous(), rank[ord2].contiguous()
            d_gt = torch.from_numpy(np.ascontiguousarray(gt)).to(dev)
            d_off = torch.from_numpy(np.asarray(offs, dtype=np.int32)).to(dev)
            d_neutral = None
            if use_neutral:
                flat = np.concatenate([np.asarray(e, dtype=np.uint8).reshape(-1) for e in neutral]) if offs[-1] else np.zeros(1, np.uint8)
                d_neutral = torch.from_numpy(np.ascontiguousarray(flat)).to(dev)
            matched = torch.zeros(max(offs[-1], 1), dtype=torch.uint8, device=dev)
            tp = torch.zeros(n, dtype=torch.int32, device=dev); fp = torch.zeros(n, dtype=torch.int32, device=dev)
            ctp = torch.empty_like(tp); cfp = torch.empty_like(fp)
            ctx = _ffi.context()
            _ffi.check(_ffi.lib().ssdk_eval_match(ctx, n, _ffi.dptr(seg), n_seg, _ffi.dptr(p_img), _ffi.dptr(p_cls), _ffi.dptr(p_box),
                                                  _ffi.dptr(p_rank), _ffi.dptr(d_gt), _ffi.dptr(d_off), _ffi.dptr(d_neutral), _ffi.dptr(matched),
                                                  float(matching_iou_threshold), _ffi.BORDER_D[border_pixels], _ffi.dptr(tp), _ffi.dptr(fp),
                                                  _ffi.stream_ptr()))
            coff = torch.from_numpy(np.concatenate([[0], np.cumsum(counts[1:])]).astype(np.int32)).to(dev)
            _ffi.check(_ffi.lib().ssdk_eval_cumsum(ctx, _ffi.dptr(tp), _ffi.dptr(fp), _ffi.dptr(coff), nC, _ffi.dptr(ctp), _ffi.dptr(cfp),
                                                   _ffi.stream_ptr()))
            tp, fp, ctp, cfp = tp.cpu().numpy(), fp.cpu().numpy(), ctp.cpu().numpy(), cfp.cpu().numpy()
            o = 0
            for c in range(1, nC + 1):
                k = counts[c]
                tp_all[c], fp_all[c] = tp[o:o + k].astype(int), fp[o:o + k].astype(int)
                ctp_all[c], cfp_all[c] = ctp[o:o + k].astype(int), cfp[o:o + k].astype(int)
                o += k
        self.true_positives, self.false_positives = tp_all, fp_all
        self.cumulative_true_positives, self.cumulative_false_positives = ctp_all, cfp_all
        if ret:
            return tp_all, fp_all, ctp_all, cfp_all

    # -- precision / recall / AP: the reference's NumPy expressions (:738-905) -----------------------------
    def compute_precision_recall(self, verbose=True, ret=False):
        if (self.cumulative_true_positives is None) or (self.cumulative_false_positives is None):
            raise ValueError("True and false positives not available. You must run `match_predictions()` before you call this method.")
        if self.num_gt_per_class is None:
            raise ValueError("Number of ground truth boxes per class not available. You must run `get_num_gt_per_class()` before you call this method.")
        precisions, recalls = [[]], [[]]
        for c in range(1, self.n_classes + 1):
            tp = self.cumulative_true_positives[c]
            fp = self.cumulative_false_positives[c]
            with np.errstate(divide='ignore', invalid='ignore'):
                precisions.append(np.where(tp + fp > 0, tp / (tp + fp), 0))
                recalls.append(tp / self.num_gt_per_class[c])
        self.cumulative_precisions, self.cumulative_recalls = precisions, recalls
        if ret:
            return precisions, recalls

    def compute_average_precisions(self, mode='sample', num_recall_points=11, verbose=True, ret=False):
        if (self.cumulative_precisions is None) or (self.cumulative_recalls is None):
            raise ValueError("Precisions and recalls not available. You must run `compute_precision_recall()` before you call this method.")
        if mode not in {'sample', 'integrate'}:
            raise ValueError("`mode` can be either 'sample' or 'integrate', but received '{}'".format(mode))
        aps = [0.0]
        for c in range(1, self.n_classes + 1):
            prec, rec = self.cumulative_precisions[c], self.cumulative_recalls[c]
            ap = 0.0
            if mode == 'sample':
                for t in np.linspace(start=0, stop=1, num=num_recall_points, endpoint=True):
                    sel = prec[rec >= t]
                    ap += 0.0 if sel.size == 0 else np.amax(sel)
                ap /= num_recall_points
            else:
                ur, ui, _ = np.unique(rec, return_index=True, return_counts=True)
                mp = np.zeros_like(ur); dr = np.zeros_like(ur)
                for i in range(len(ur) - 2, -1, -1):
                    mp[i] = np.maximum(np.amax(prec[ui[i]:ui[i + 1]]), mp[i + 1])
                    dr[i] = ur[i + 1] - ur[i]
                ap = np.sum(mp * dr)
            aps.append(ap)
        self.average_precisions = aps
        if ret:
            return aps

    def compute_mean_average_precision(self, ret=True):
        if self.average_precisions is None:
            raise ValueError("Average precisions not available. You must run `compute_average_precisions()` before you call this method.")
        self.mean_average_precision = np.average(self.average_precisions[1:])
        if ret:
            return self.mean_average_precision
