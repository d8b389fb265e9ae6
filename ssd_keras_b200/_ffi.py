"""ctypes binding of libssdk.so (include/ssdk.h).  PyTorch is used only for device memory and streams."""
import ctypes as C
import os
import threading

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, '_lib', 'libssdk.so')

SSDK_OK = 0
SSDK_ERR_INVALID = -1
SSDK_ERR_CUDA = -2
SSDK_ERR_UNSUPPORTED = -3
SSDK_ERR_NOMEM = -4
SSDK_ERR_DEGENERATE = -5

COORDS = {'centroids': 0, 'corners': 1, 'minmax': 2}
BORDER_D = {'half': 0, 'include': 1, 'exclude': -1}

c_int_p = C.POINTER(C.c_int)
c_float_p = C.POINTER(C.c_float)
c_double_p = C.POINTER(C.c_double)


# The structs of include/ssdk.h, each named after the C struct without its ssdk_ prefix (BoxOp = ssdk_box_op).
class AnchorCfg(C.Structure):
    _fields_ = [('img_height', C.c_int), ('img_width', C.c_int), ('n_layers', C.c_int),
                ('fm_height', c_int_p), ('fm_width', c_int_p), ('scales', c_double_p),
                ('n_aspect_ratios', c_int_p), ('aspect_ratios', c_double_p), ('two_boxes_for_ar1', C.c_int),
                ('steps_h', c_double_p), ('steps_w', c_double_p), ('offsets_h', c_double_p), ('offsets_w', c_double_p),
                ('clip_boxes', C.c_int), ('coords', C.c_int), ('normalize_coords', C.c_int)]


class EncodeCfg(C.Structure):
    _fields_ = [('img_height', C.c_int), ('img_width', C.c_int), ('n_classes_total', C.c_int), ('P', C.c_int),
                ('background_id', C.c_int), ('coords', C.c_int), ('matching_multi', C.c_int),
                ('pos_iou_threshold', C.c_double), ('neg_iou_limit', C.c_double), ('border_d', C.c_int),
                ('normalize_coords', C.c_int), ('variances', C.c_double * 4),
                ('n_layers', C.c_int), ('fm_height', c_int_p), ('fm_width', c_int_p), ('n_boxes', c_int_p)]


class DecodeCfg(C.Structure):
    _fields_ = [('mode', C.c_int), ('layer_semantics', C.c_int), ('n_classes_total', C.c_int), ('P', C.c_int),
                ('confidence_thresh', C.c_double), ('iou_threshold', C.c_double), ('top_k', C.c_int),
                ('nms_max_output', C.c_int), ('coords', C.c_int), ('normalize_coords', C.c_int),
                ('img_height', C.c_int), ('img_width', C.c_int), ('border_d', C.c_int), ('max_out', C.c_int)]


class BoxOp(C.Structure):
    _fields_ = [('op', C.c_int), ('flags', C.c_int), ('a0', C.c_double), ('a1', C.c_double), ('a2', C.c_double), ('a3', C.c_double)]


BOXOP_END, BOXOP_CROP_PAD, BOXOP_FLIP_H, BOXOP_FLIP_V, BOXOP_RESIZE, BOXOP_FILTER = range(6)
BOXOP_TRANSLATE, BOXOP_SCALE, BOXOP_ROTATE, BOXOP_OVERLAP, BOXOP_CLIP = range(6, 11)
(BOXOP_TO_FLOAT32, BOXOP_TO_UINT8, BOXOP_BRIGHTNESS, BOXOP_CONTRAST, BOXOP_SATURATION, BOXOP_HUE, BOXOP_RGB2HSV, BOXOP_HSV2RGB,
 BOXOP_CHANNEL_SWAP) = range(16, 25)         # photometric ops: images only (ssdk_assemble_images)
BOXOP_RESIZE_INTERP = 25                    # RESIZE with all five cv2 modes (the boxes as RESIZE)
BOXOP_EQUALIZE_V = 26                       # photometric: cv2.equalizeHist of channel 2 (images only)
PHOTO_OPS = frozenset(range(BOXOP_TO_FLOAT32, BOXOP_CHANNEL_SWAP + 1)) | {BOXOP_EQUALIZE_V}
INTER_NEAREST, INTER_LINEAR, INTER_CUBIC, INTER_AREA, INTER_LANCZOS4 = range(5)   # cv2's codes, in flag bits 8-15


class LossWsLayout(C.Structure):
    _fields_ = [('bytes', C.c_longlong), ('counts_offset', C.c_longlong), ('counts_n', C.c_longlong), ('hist1_offset', C.c_longlong),
                ('hist2_offset', C.c_longlong), ('hist_n', C.c_longlong), ('ties_offset', C.c_longlong)]


class LossPlan(C.Structure):
    _fields_ = [('stages', C.c_int), ('bulk_ok', C.c_int), ('grid', C.c_int), ('smem_bytes', C.c_longlong)]


def loss_plan(y_true, y_pred, n_classes_total, want_grad, cooperative=True):
    """The launch the loss would make for these (B, P, C+12) device tensors, as a dict (ssdk_ssd_loss_plan); raises what the
    launch would raise."""
    B, P = y_pred.shape[0], y_pred.shape[1]
    p = LossPlan()
    check(lib().ssdk_ssd_loss_plan(context(y_pred.device.index), dptr(y_true), dptr(y_pred), B, P, int(n_classes_total),
                                   int(bool(want_grad)), int(bool(cooperative)), C.byref(p)))
    return {n: getattr(p, n) for n, _ in LossPlan._fields_}


def loss_box_losses(B, P, ws=None, device=None):
    """(cls, negl), (B, P) float32 device tensors: the per-box losses the loss kernel's first phase stored, in the context's own
    workspace (ws None) or in a phase workspace (ssdk_ssd_loss_read_box_losses)."""
    import torch
    dev = ws.device if ws is not None else torch.device('cuda', torch.cuda.current_device() if device is None else device)
    cls = torch.empty((B, P), dtype=torch.float32, device=dev)
    negl = torch.empty_like(cls)
    check(lib().ssdk_ssd_loss_read_box_losses(context(dev.index), dptr(ws), int(B), int(P), dptr(cls), dptr(negl), stream_ptr()))
    return cls, negl


class LayerDesc(C.Structure):
    _fields_ = [('op', C.c_int), ('input', C.c_int), ('cout', C.c_int), ('kh', C.c_int), ('kw', C.c_int),
                ('stride', C.c_int), ('dilation', C.c_int), ('pad_t', C.c_int), ('pad_l', C.c_int),
                ('pad_b', C.c_int), ('pad_r', C.c_int), ('act', C.c_int), ('n_boxes', C.c_int),
                ('kernel', c_float_p), ('bias', c_float_p), ('bn_scale', c_float_p), ('bn_shift', c_float_p),
                ('kernel2', c_float_p), ('bias2', c_float_p), ('mean', c_float_p), ('stddev', c_float_p),
                ('swap', c_int_p), ('bn_gamma', c_float_p), ('bn_beta', c_float_p), ('bn_mean', c_float_p), ('bn_var', c_float_p),
                ('bn_eps', C.c_float), ('bn_momentum', C.c_float)]


class ModelDesc(C.Structure):
    _fields_ = [('batch', C.c_int), ('img_height', C.c_int), ('img_width', C.c_int), ('img_channels', C.c_int),
                ('n_classes_total', C.c_int), ('n_layers', C.c_int), ('layers', C.POINTER(LayerDesc)),
                ('precision', C.c_int), ('anchors_f32', c_float_p), ('variances', C.c_float * 4), ('training', C.c_int)]


class LayerPlan(C.Structure):
    _fields_ = [(n, C.c_int) for n in ('kernel', 'bn', 'split', 'stages', 'kblocks', 'n_tiles_m', 'n_tiles_n', 'grid', 'k_split',
                                       'epilogue', 'head_fused', 'im2col_vec8', 'bm')]


class BackwardPlan(C.Structure):
    _fields_ = [(n, C.c_int) for n in ('dgrad', 'dgrad_bn', 'dgrad_mask', 'dgrad_accumulate', 'dgrad_n_tiles_m', 'dgrad_n_tiles_n',
                                       'dgrad_grid', 'wgrad', 'wgrad_bn', 'a_boxes', 'bw', 'bh', 'co_tiles', 'ci_tiles', 'k_split',
                                       'n_gemms', 'stages', 'grid', 'kv', 'direct_fast')]


PLAN_KERNELS = {0: None, 1: 'gemm', 2: 'im2col_gemm', 3: 'first_tc', 4: 'direct', 5: 'gemm_swap'}
PLAN_EPILOGUES = {0: 'split', 1: 'f32', 2: 'atomic', 3: 'head'}
DGRAD_PATHS = {0: None, 1: 'gemm', 2: 'strided'}
WGRAD_PATHS = {0: None, 1: 'native', 2: 'transposed', 3: 'im2col', 4: 'direct'}


def model_layer_plan(handle, layer):
    """The launch plan of one layer of a model plan, as a dict (ssdk_model_layer_plan)."""
    p = LayerPlan()
    check(lib().ssdk_model_layer_plan(handle, int(layer), C.byref(p)))
    out = {n: getattr(p, n) for n, _ in LayerPlan._fields_}
    out['kernel'] = PLAN_KERNELS[p.kernel]
    out['epilogue'] = PLAN_EPILOGUES[p.epilogue]
    return out


def trainer_layer_plan(handle, layer):
    """The backward launches of one layer of a trainer, as a dict (ssdk_trainer_layer_plan)."""
    p = BackwardPlan()
    check(lib().ssdk_trainer_layer_plan(handle, int(layer), C.byref(p)))
    out = {n: getattr(p, n) for n, _ in BackwardPlan._fields_}
    out['dgrad'] = DGRAD_PATHS[p.dgrad]
    out['wgrad'] = WGRAD_PATHS[p.wgrad]
    return out


class CocoMatch(C.Structure):
    _fields_ = [(n, C.c_int) for n in ('n_seg', 'n_gt', 'n_det', 'n_area', 'n_thr')] + \
               [(n, C.c_void_p) for n in ('seg_gt', 'seg_det', 'seg_cat', 'gt_box', 'gt_area', 'gt_flags', 'det_box', 'det_area',
                                          'area_rng', 'iou_thrs', 'gt_matched', 'det_flags', 'det_match', 'seg_npig', 'npig')]


class CocoAccumulate(C.Structure):
    _fields_ = [(n, C.c_int) for n in ('n_thr', 'n_area', 'n_det', 'n_rec', 'n_k', 'n_a', 'n_m', 'out_k', 'out_a', 'out_m')] + \
               [(n, C.c_void_p) for n in ('cat_off', 'ord_det', 'ord_rank', 'ord_score', 'det_flags', 'npig', 'rec_thrs', 'rec_sorted',
                                          'rec_perm', 'sel_cat', 'sel_area', 'sel_max_det', 'precision', 'scores', 'recall')]


OP_INPUT, OP_CONV, OP_MAXPOOL, OP_L2NORM, OP_HEAD, OP_TENSOR = range(6)
ACT_NONE, ACT_RELU, ACT_ELU = range(3)

# Every function of include/ssdk.h, in its order: name -> (restype, argtypes).  tests/test_abi_cpu.py holds it to the header.
_p, _i, _ll, _f, _d = C.c_void_p, C.c_int, C.c_longlong, C.c_float, C.c_double
SIGNATURES = {
    'ssdk_version': (_i, []),
    'ssdk_last_error': (C.c_char_p, []),
    'ssdk_ctx_create': (_i, [_i, C.POINTER(_p)]),
    'ssdk_ctx_destroy': (_i, [_p]),
    'ssdk_ctx_launch_count': (C.c_int64, [_p]),
    'ssdk_anchors_count': (_i, [C.POINTER(AnchorCfg), c_int_p, c_int_p]),
    'ssdk_anchors_generate': (_i, [C.POINTER(AnchorCfg), c_double_p, c_float_p]),
    'ssdk_encoder_create': (_i, [_p, C.POINTER(EncodeCfg), c_double_p, C.POINTER(_p)]),
    'ssdk_encoder_destroy': (_i, [_p]),
    'ssdk_encode': (_i, [_p, _p, _i, c_int_p, _p, _i, _i, _i, _p, _p, _p, _p]),
    'ssdk_iou_matrix': (_i, [_p, _p, _i, _p, _p]),
    'ssdk_iou': (_i, [_p, _p, _i, _p, _i, _i, _i, _i, _p, _p]),
    'ssdk_assemble_batch': (_i, [_p, _p, _i, _p, _i, _i, _p, _i, _p, _p, _p, _p]),
    'ssdk_assemble_images': (_i, [_p, _p, _p, _p, _i, _p, _i, _i, _i, _p, _p]),
    'ssdk_eval_match': (_i, [_p, _i, _p, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p, _d, _i, _p, _p, _p]),
    'ssdk_eval_cumsum': (_i, [_p, _p, _p, _p, _i, _p, _p, _p]),
    'ssdk_eval_collect': (_i, [_p, _p, _i, _i, _p, _p, c_int_p, _i, _i, _i, _i, _i, _p, _p, _p, _p, _p, _p]),
    'ssdk_cocoeval_match': (_i, [_p, C.POINTER(CocoMatch), _p]),
    'ssdk_cocoeval_accumulate': (_i, [_p, C.POINTER(CocoAccumulate), _p]),
    'ssdk_decode': (_i, [_p, C.POINTER(DecodeCfg), _p, _i, _p, _p, _p, _p]),
    'ssdk_nms': (_i, [_p, _p, _p, _i, _i, _d, _d, _i, _i, _p, _p, _p, _p]),
    'ssdk_ssd_loss': (_i, [_p, _p, _p, _i, _i, _i, _i, _i, _f, _p, _p, _p, _p, _p]),
    'ssdk_ssd_loss_ws_layout': (_i, [_i, _i, C.POINTER(LossWsLayout)]),
    'ssdk_ssd_loss_phase': (_i, [_p, _i, _p, _p, _i, _i, _i, _i, _i, _f, _p, _i, _p, _i, _p, _p, _p, _p, _p]),
    'ssdk_focal_loss': (_i, [_p, _p, _p, _i, _i, _i, _f, _f, _f, _p, _p, _p, _p]),
    'ssdk_focal_loss_phase': (_i, [_p, _i, _p, _p, _i, _i, _i, _f, _f, _f, _p, _i, _p, _p, _p, _p]),
    'ssdk_ssd_loss_plan': (_i, [_p, _p, _p, _i, _i, _i, _i, _i, C.POINTER(LossPlan)]),
    'ssdk_ssd_loss_read_box_losses': (_i, [_p, _p, _i, _i, _p, _p, _p]),
    'ssdk_l2_normalize': (_i, [_p, _p, _ll, _i, _p, _p, _p]),
    'ssdk_conv2d_fwd': (_i, [_p, _p] + [_i] * 4 + [_p, _p] + [_i] * 11 + [_p, _p]),
    'ssdk_maxpool': (_i, [_p, _p] + [_i] * 11 + [_p, _p]),
    'ssdk_schedule_preview': (_i, [_i, c_int_p, c_int_p, c_int_p, _i, _i, C.POINTER(C.c_ubyte), c_int_p, c_int_p]),
    'ssdk_model_create': (_i, [_p, C.POINTER(ModelDesc), C.POINTER(_p)]),
    'ssdk_model_destroy': (_i, [_p]),
    'ssdk_model_num_priors': (_i, [_p, c_int_p]),
    'ssdk_model_layer_shape': (_i, [_p, _i, c_int_p, c_int_p, c_int_p]),
    'ssdk_model_forward': (_i, [_p, _p, _p, _p]),
    'ssdk_model_read_layer': (_i, [_p, _i, _p, _p]),
    'ssdk_model_layer_planes_shape': (_i, [_p, _i, c_int_p, c_int_p, c_int_p, c_int_p]),
    'ssdk_model_read_layer_planes': (_i, [_p, _i, _p, _p, _p]),
    'ssdk_model_flops': (_i, [_p, c_double_p, c_double_p]),
    'ssdk_model_set_timing': (_i, [_p, _i]),
    'ssdk_model_last_conv_ms': (_i, [_p, c_float_p]),
    'ssdk_model_layer_ms': (_i, [_p, _i, c_float_p]),
    'ssdk_model_layer_plan': (_i, [_p, _i, C.POINTER(LayerPlan)]),
    'ssdk_trainer_create': (_i, [_p, _p, C.POINTER(_p)]),
    'ssdk_trainer_destroy': (_i, [_p]),
    'ssdk_trainer_num_params': (_i, [_p, C.POINTER(_ll)]),
    'ssdk_trainer_param_span': (_i, [_p, _i, _i, C.POINTER(_ll), C.POINTER(_ll)]),
    'ssdk_trainer_grad_shape': (_i, [_p, _i, c_int_p, c_int_p, c_int_p, c_int_p]),
    'ssdk_trainer_read_grad': (_i, [_p, _i, _p, _p]),
    'ssdk_trainer_read_grad_planes': (_i, [_p, _i, _p, _p, _p]),
    'ssdk_train_backward_layers': (_i, [_p, _p, _i, _i, _p]),
    'ssdk_train_apply': (_i, [_p, _f, _f, _f, _f, _p]),
    'ssdk_train_apply_adam': (_i, [_p, _f, _f, _f, _f, _f, _f, _i, _p]),
    'ssdk_trainer_read_bn_stats': (_i, [_p, _i, _p, _p, _p]),
    'ssdk_trainer_read_bn_input': (_i, [_p, _i, _p, _p]),
    'ssdk_trainer_read_params': (_i, [_p, _p, _p]),
    'ssdk_trainer_read_opt_state': (_i, [_p, _i, _p, _p]),
    'ssdk_trainer_write_opt_state': (_i, [_p, _i, _p, _p]),
    'ssdk_trainer_layer_plan': (_i, [_p, _i, C.POINTER(BackwardPlan)]),
}

_lib = None
_lock = threading.Lock()


class SSDKError(RuntimeError):
    pass


def lib():
    """Load libssdk.so.  There is no fallback: a missing library is a hard error."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(_LIB_PATH):
            raise SSDKError("libssdk.so is not built (%s). Run `python -m ssd_keras_b200.build` "
                            "(or __graft_entry__.build()); there is no CPU/PyTorch fallback." % _LIB_PATH)
        L = C.CDLL(_LIB_PATH)
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = restype, argtypes
        _lib = L
    return _lib


def check(rc):
    """Translate a status code into the exception the reference would raise."""
    if rc == SSDK_OK:
        return
    msg = lib().ssdk_last_error().decode('utf-8', 'replace')
    if rc == SSDK_ERR_INVALID:
        raise ValueError(msg)
    if rc == SSDK_ERR_UNSUPPORTED:
        raise NotImplementedError(msg)
    if rc == SSDK_ERR_NOMEM:
        raise MemoryError(msg)
    raise SSDKError('libssdk error %d: %s' % (rc, msg))


def np_ptr(a, ctype):
    return a.ctypes.data_as(C.POINTER(ctype))


_ctx = {}


def context(device=None):
    """One ssdk_ctx per (process, device, thread)."""
    import torch
    if not torch.cuda.is_available():
        raise SSDKError('No CUDA device: ssd_keras_b200 has no CPU fallback')
    if device is None:
        device = torch.cuda.current_device()
    key = (device, threading.get_ident())
    if key not in _ctx:
        h = C.c_void_p()
        check(lib().ssdk_ctx_create(int(device), C.byref(h)))
        _ctx[key] = h
    return _ctx[key]


def launch_count(device=None):
    return int(lib().ssdk_ctx_launch_count(context(device)))


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def dptr(t):
    """Device pointer of a contiguous torch CUDA tensor (or None)."""
    if t is None:
        return C.c_void_p(0)
    assert t.is_cuda and t.is_contiguous()
    return C.c_void_p(t.data_ptr())


# ---------------------------------------------------------------------------------------------
# host-only helper: anchors (works without a GPU)
# ---------------------------------------------------------------------------------------------
def _pair_or_nan(v):
    if v is None:
        return float('nan'), float('nan')
    if isinstance(v, (list, tuple, np.ndarray)) and len(v) == 2:
        return float(v[0]), float(v[1])
    return float(v), float(v)


def generate_anchors(img_height, img_width, predictor_sizes, scales, aspect_ratios_per_layer, two_boxes_for_ar1=True,
                     steps=None, offsets=None, clip_boxes=False, coords='centroids', normalize_coords=True):
    """-> (anchors float64 (P,4), anchors float32 (P,4), n_boxes per layer) via ssdk_anchors_generate."""
    if coords not in COORDS:
        raise ValueError("Unexpected value for `coords`. Supported values are 'minmax', 'corners' and 'centroids'.")
    L = lib()
    ps = np.asarray(predictor_sizes, dtype=np.int32).reshape(-1, 2)
    n = ps.shape[0]
    fm_h = np.ascontiguousarray(ps[:, 0]); fm_w = np.ascontiguousarray(ps[:, 1])
    sc = np.ascontiguousarray(np.asarray(scales, dtype=np.float64))
    n_ar = np.array([len(a) for a in aspect_ratios_per_layer], dtype=np.int32)
    ars = np.ascontiguousarray(np.concatenate([np.asarray(a, dtype=np.float64) for a in aspect_ratios_per_layer]))
    st = np.array([_pair_or_nan(s) for s in (steps if steps is not None else [None] * n)], dtype=np.float64)
    of = np.array([_pair_or_nan(o) for o in (offsets if offsets is not None else [None] * n)], dtype=np.float64)
    st_h, st_w = np.ascontiguousarray(st[:, 0]), np.ascontiguousarray(st[:, 1])
    of_h, of_w = np.ascontiguousarray(of[:, 0]), np.ascontiguousarray(of[:, 1])
    cfg = AnchorCfg(int(img_height), int(img_width), int(n), np_ptr(fm_h, C.c_int), np_ptr(fm_w, C.c_int),
                    np_ptr(sc, C.c_double), np_ptr(n_ar, C.c_int), np_ptr(ars, C.c_double), int(bool(two_boxes_for_ar1)),
                    np_ptr(st_h, C.c_double), np_ptr(st_w, C.c_double), np_ptr(of_h, C.c_double), np_ptr(of_w, C.c_double),
                    int(bool(clip_boxes)), COORDS[coords], int(bool(normalize_coords)))
    P = C.c_int(0)
    nb = np.zeros(n, dtype=np.int32)
    check(L.ssdk_anchors_count(C.byref(cfg), C.byref(P), np_ptr(nb, C.c_int)))
    a64 = np.empty((P.value, 4), dtype=np.float64)
    a32 = np.empty((P.value, 4), dtype=np.float32)
    check(L.ssdk_anchors_generate(C.byref(cfg), np_ptr(a64, C.c_double), np_ptr(a32, C.c_float)))
    return a64, a32, nb.tolist()
