"""``ssd_300`` on H100 -- same signature as the reference builder (``models/keras_ssd300.py:31-59``).

Returns an ``SSDModel`` (see ``_graph.py``) instead of a Keras ``Model``: VGG-16 (atrous fc6/fc7) + extra
layers + L2Normalization + six fused conf/loc predictor heads, executed as wgmma implicit-GEMM kernels."""

from .. import _ffi
from ._graph import SSDModel, Spec, records_config, resolve_box_args, same_pad, tf_same_pool_pad

RELU = _ffi.ACT_RELU


def _vgg_base(specs, img_height, img_width):
    """conv1_1 .. fc7 (reference :274-299).  Returns the running spatial size."""
    h, w = img_height, img_width
    prev = 'input'
    cfg = [('conv1_1', 64), ('conv1_2', 64), 'pool1', ('conv2_1', 128), ('conv2_2', 128), 'pool2',
           ('conv3_1', 256), ('conv3_2', 256), ('conv3_3', 256), 'pool3',
           ('conv4_1', 512), ('conv4_2', 512), ('conv4_3', 512), 'pool4',
           ('conv5_1', 512), ('conv5_2', 512), ('conv5_3', 512)]
    for item in cfg:
        if isinstance(item, str):
            pt, pb = tf_same_pool_pad(h, 2, 2)
            pl, pr = tf_same_pool_pad(w, 2, 2)
            specs.append(Spec(item, _ffi.OP_MAXPOOL, prev, k=(2, 2), stride=2, pad=(pt, pl, pb, pr)))
            h, w = -(-h // 2), -(-w // 2)
        else:
            specs.append(Spec(item[0], _ffi.OP_CONV, prev, cout=item[1], k=(3, 3), pad=same_pad(3), act=RELU))
        prev = specs[-1].name
    specs.append(Spec('pool5', _ffi.OP_MAXPOOL, prev, k=(3, 3), stride=1, pad=(1, 1, 1, 1)))
    specs.append(Spec('fc6', _ffi.OP_CONV, 'pool5', cout=1024, k=(3, 3), dilation=6, pad=same_pad(3, 6), act=RELU))
    specs.append(Spec('fc7', _ffi.OP_CONV, 'fc6', cout=1024, k=(1, 1), act=RELU))
    return h, w


def _extra(specs, n1, n2, inp, c1, c2, stride, pad, k=3):
    """1x1 reduce + (ZeroPadding2D +) 3x3 'valid' conv (reference :301-313)."""
    specs.append(Spec(n1, _ffi.OP_CONV, inp, cout=c1, k=(1, 1), act=RELU))
    specs.append(Spec(n2, _ffi.OP_CONV, n1, cout=c2, k=(k, k), stride=stride, pad=(pad, pad, pad, pad), act=RELU))
    return n2


def _input_spec(subtract_mean, divide_by_stddev, swap_channels):
    return Spec('input', _ffi.OP_INPUT, params={'mean': subtract_mean, 'stddev': divide_by_stddev,
                                                'swap': list(swap_channels) if swap_channels else None})


def _finish(specs, sources, n_boxes):
    specs.append(Spec('conv4_3_norm', _ffi.OP_L2NORM, 'conv4_3'))
    for src, nb in zip(sources, n_boxes):
        specs.append(Spec(src + '_mbox', _ffi.OP_HEAD, src, k=(3, 3), pad=same_pad(3), n_boxes=nb,
                          params={'conf_name': src + '_mbox_conf', 'loc_name': src + '_mbox_loc'}))


@records_config('ssd_300')
def ssd_300(image_size, n_classes, mode='training', l2_regularization=0.0005, min_scale=None, max_scale=None, scales=None,
            aspect_ratios_global=None,
            aspect_ratios_per_layer=[[1.0, 2.0, 0.5], [1.0, 2.0, 0.5, 3.0, 1.0 / 3.0], [1.0, 2.0, 0.5, 3.0, 1.0 / 3.0],
                                     [1.0, 2.0, 0.5, 3.0, 1.0 / 3.0], [1.0, 2.0, 0.5], [1.0, 2.0, 0.5]],
            two_boxes_for_ar1=True, steps=[8, 16, 32, 64, 100, 300], offsets=None, clip_boxes=False,
            variances=[0.1, 0.1, 0.2, 0.2], coords='centroids', normalize_coords=True, subtract_mean=[123, 117, 104],
            divide_by_stddev=None, swap_channels=[2, 1, 0], confidence_thresh=0.01, iou_threshold=0.45, top_k=200,
            nms_max_output_size=400, return_predictor_sizes=False, precision='bf16x3', weights_seed=0):
    n_predictor_layers = 6
    n_classes += 1
    img_height, img_width, img_channels = image_size[0], image_size[1], image_size[2]
    scales, aspect_ratios, n_boxes, variances = resolve_box_args(n_predictor_layers, min_scale, max_scale, scales,
                                                                 aspect_ratios_global, aspect_ratios_per_layer,
                                                                 two_boxes_for_ar1, steps, offsets, variances)
    if mode not in ('training', 'inference', 'inference_fast'):
        raise ValueError("`mode` must be one of 'training', 'inference' or 'inference_fast', but received '{}'.".format(mode))
    specs = [_input_spec(subtract_mean, divide_by_stddev, swap_channels)]
    _vgg_base(specs, img_height, img_width)
    _extra(specs, 'conv6_1', 'conv6_2', 'fc7', 256, 512, 2, 1)
    _extra(specs, 'conv7_1', 'conv7_2', 'conv6_2', 128, 256, 2, 1)
    _extra(specs, 'conv8_1', 'conv8_2', 'conv7_2', 128, 256, 1, 0)
    _extra(specs, 'conv9_1', 'conv9_2', 'conv8_2', 128, 256, 1, 0)
    _finish(specs, ['conv4_3_norm', 'fc7', 'conv6_2', 'conv7_2', 'conv8_2', 'conv9_2'], n_boxes)
    anchor_cfg = dict(scales=scales, aspect_ratios_per_layer=aspect_ratios, two_boxes_for_ar1=two_boxes_for_ar1, steps=steps,
                      offsets=offsets, clip_boxes=clip_boxes, coords=coords, normalize_coords=normalize_coords)
    decode_cfg = dict(confidence_thresh=confidence_thresh, iou_threshold=iou_threshold, top_k=top_k,
                      nms_max_output_size=nms_max_output_size, coords=coords, normalize_coords=normalize_coords,
                      img_height=img_height, img_width=img_width)
    model = SSDModel(specs, img_height, img_width, img_channels, n_classes, anchor_cfg, variances, mode, decode_cfg,
                     l2_reg=l2_regularization, precision=precision, seed=weights_seed)
    if return_predictor_sizes:
        return model, model.predictor_sizes
    return model
