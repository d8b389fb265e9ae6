"""MS COCO helpers (reference ``eval_utils/coco_utils.py:30-200``): the category maps and a detection results file.

``predict_all_to_json`` predicts through ``dataset_predict`` (the reference's ``ConvertTo3Channels`` / ``RandomPadFixedAR`` /
``Resize`` chain and its inverters on the device) and writes the same JSON text as the reference."""
import json

import numpy as np


def get_coco_category_maps(annotations_file):
    """Reference :30-60: ``(cats_to_classes, classes_to_cats, cats_to_names, classes_to_names)`` from any COCO annotations
    file; the classes are the categories numbered from 1 in file order, ``classes_to_names[0]`` is 'background'."""
    with open(annotations_file, 'r') as f:
        annotations = json.load(f)
    cats_to_classes, classes_to_cats, cats_to_names, classes_to_names = {}, {}, {}, ['background']
    for i, cat in enumerate(annotations['categories']):
        cats_to_classes[cat['id']] = i + 1
        classes_to_cats[i + 1] = cat['id']
        cats_to_names[cat['id']] = cat['name']
        classes_to_names.append(cat['name'])
    return cats_to_classes, classes_to_cats, cats_to_names, classes_to_names


def predict_all_to_json(out_file, model, img_height, img_width, classes_to_cats, data_generator, batch_size,
                        data_generator_mode='resize', model_mode='training', confidence_thresh=0.01, iou_threshold=0.45, top_k=200,
                        pred_coords='centroids', normalize_coords=True):
    """Reference :62-200: predictions over the whole dataset in the COCO detection results format, one dict per box with
    ``image_id``, ``category_id`` (``classes_to_cats`` of the class), ``score`` (``float(round(conf, 3))``) and ``bbox``
    ``[xmin, ymin, width, height]`` (corners rounded to one decimal, then the differences).  'training'-mode models are
    decoded with ``decode_detections`` and its default ``border_pixels='half'``, as there.

    ``data_generator_mode='pad'`` works as in ``Evaluator`` (a seeded ``np.random`` places every image where the reference's
    ``RandomPadFixedAR`` does).  The reference's own 'pad' branch raises ``TypeError`` (it passes ``clip_boxes`` to
    ``RandomPadFixedAR``, which does not take it)."""
    from .dataset_predict import predict_dataset
    if data_generator_mode not in ('resize', 'pad'):
        raise ValueError("Unexpected argument value: `data_generator_mode` can be either of 'resize' or 'pad', but received '{}'."
                         .format(data_generator_mode))
    det = predict_dataset(model, data_generator, img_height, img_width, batch_size, mode=data_generator_mode, model_mode=model_mode,
                          decode_kwargs=dict(confidence_thresh=confidence_thresh, iou_threshold=iou_threshold, top_k=top_k,
                                             input_coords=pred_coords, normalize_coords=normalize_coords))
    print("Number of images in the evaluation dataset: {}".format(len(det.image_ids)))
    img, cls, conf, box = det.host()
    score = np.round(conf, 3)                 # round(numpy scalar, 3): multiply, rint and divide in the scalar's type
    results = []
    for i, c, s, b in zip(img.tolist(), cls.tolist(), score.tolist(), box.tolist()):
        xmin, ymin, xmax, ymax = b
        results.append({'image_id': det.image_ids[i], 'category_id': classes_to_cats[c], 'score': s,
                        'bbox': [xmin, ymin, xmax - xmin, ymax - ymin]})
    with open(out_file, 'w') as f:
        json.dump(results, f)
    print("Prediction results saved in '{}'".format(out_file))
