"""``build_model`` (SSD7) on H100 -- same signature as the reference builder (``models/keras_ssd7.py:30-53``);
``ssd_7`` is an alias.  Seven conv + BatchNormalization(eps 1e-3, folded) + ELU stages with 'valid' 2x2 pools and
four predictor heads on conv4..conv7 (:277-331)."""
from .. import _ffi
from ._graph import SSDModel, Spec, records_config, resolve_box_args, same_pad


@records_config('build_model')
def build_model(image_size, n_classes, mode='training', l2_regularization=0.0, min_scale=0.1, max_scale=0.9, scales=None,
                aspect_ratios_global=[0.5, 1.0, 2.0], aspect_ratios_per_layer=None, two_boxes_for_ar1=True, steps=None,
                offsets=None, clip_boxes=False, variances=[1.0, 1.0, 1.0, 1.0], coords='centroids', normalize_coords=False,
                subtract_mean=None, divide_by_stddev=None, swap_channels=False, confidence_thresh=0.01, iou_threshold=0.45,
                top_k=200, nms_max_output_size=400, return_predictor_sizes=False, precision='bf16x3', weights_seed=0):
    n_predictor_layers = 4
    n_classes += 1
    img_height, img_width, img_channels = image_size[0], image_size[1], image_size[2]
    scales, aspect_ratios, n_boxes, variances = resolve_box_args(n_predictor_layers, min_scale, max_scale, scales,
                                                                 aspect_ratios_global, aspect_ratios_per_layer,
                                                                 two_boxes_for_ar1, steps, offsets, variances)
    if mode not in ('training', 'inference', 'inference_fast'):
        raise ValueError("`mode` must be one of 'training', 'inference' or 'inference_fast', but received '{}'.".format(mode))
    specs = [Spec('input', _ffi.OP_INPUT, params={'mean': subtract_mean, 'stddev': divide_by_stddev,
                                                  'swap': list(swap_channels) if swap_channels else None})]
    chans = [32, 48, 64, 64, 48, 48, 32]
    prev = 'input'
    for i, c in enumerate(chans, start=1):
        k = 5 if i == 1 else 3
        specs.append(Spec('conv%d' % i, _ffi.OP_CONV, prev, cout=c, k=(k, k), pad=same_pad(k), act=_ffi.ACT_ELU, bn='bn%d' % i))
        prev = 'conv%d' % i
        if i < 7:
            specs.append(Spec('pool%d' % i, _ffi.OP_MAXPOOL, prev, k=(2, 2), stride=2))
            prev = 'pool%d' % i
    for j, i in enumerate((4, 5, 6, 7)):
        specs.append(Spec('head%d' % i, _ffi.OP_HEAD, 'conv%d' % i, k=(3, 3), pad=same_pad(3), n_boxes=n_boxes[j],
                          params={'conf_name': 'classes%d' % i, 'loc_name': 'boxes%d' % i}))
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


ssd_7 = build_model
