"""``ssd_512`` on H100 -- same signature as the reference builder (``models/keras_ssd512.py:31-60``):
the SSD300 graph with seven predictor layers (extra stride-2 stages and the 4x4 'valid' conv10_2, :312-321)."""
from ._graph import SSDModel, records_config, resolve_box_args
from .keras_ssd300 import _extra, _finish, _input_spec, _vgg_base


@records_config('ssd_512')
def ssd_512(image_size, n_classes, mode='training', l2_regularization=0.0005, min_scale=None, max_scale=None, scales=None,
            aspect_ratios_global=None,
            aspect_ratios_per_layer=[[1.0, 2.0, 0.5], [1.0, 2.0, 0.5, 3.0, 1.0 / 3.0], [1.0, 2.0, 0.5, 3.0, 1.0 / 3.0],
                                     [1.0, 2.0, 0.5, 3.0, 1.0 / 3.0], [1.0, 2.0, 0.5, 3.0, 1.0 / 3.0], [1.0, 2.0, 0.5],
                                     [1.0, 2.0, 0.5]],
            two_boxes_for_ar1=True, steps=[8, 16, 32, 64, 128, 256, 512], offsets=None, clip_boxes=False,
            variances=[0.1, 0.1, 0.2, 0.2], coords='centroids', normalize_coords=True, subtract_mean=[123, 117, 104],
            divide_by_stddev=None, swap_channels=[2, 1, 0], confidence_thresh=0.01, iou_threshold=0.45, top_k=200,
            nms_max_output_size=400, return_predictor_sizes=False, precision='bf16x3', weights_seed=0):
    n_predictor_layers = 7
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
    _extra(specs, 'conv8_1', 'conv8_2', 'conv7_2', 128, 256, 2, 1)
    _extra(specs, 'conv9_1', 'conv9_2', 'conv8_2', 128, 256, 2, 1)
    _extra(specs, 'conv10_1', 'conv10_2', 'conv9_2', 128, 256, 1, 1, k=4)
    _finish(specs, ['conv4_3_norm', 'fc7', 'conv6_2', 'conv7_2', 'conv8_2', 'conv9_2', 'conv10_2'], n_boxes)
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
