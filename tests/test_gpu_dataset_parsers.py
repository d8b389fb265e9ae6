"""The notebooks that start from ``parse_xml`` / ``parse_json``, scaled down to the dataset of tests/voc_dataset.py, on the
device: the VOC evaluation notebook (the Evaluator call and its step-by-step cells), the COCO evaluation notebook
(``predict_all_to_json`` and the device ``COCOeval``) and the data cells of the SSD300 training notebook (``fit_generator``
with its callbacks).  A parsed dataset must give exactly what a constructor-built dataset with the golden lists gives (existing
tests pin that path to the reference), and ``generate()`` over a parsed dataset must reproduce the reference's batches
(tests/golden/make_dataset_parsers_golden.py) bit for bit."""
import contextlib
import csv
import io
import json
import os

import numpy as np
import pytest

import voc_dataset as ds

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_dataset_parsers_golden.json')
SCALES_VOC = [0.1, 0.2, 0.37, 0.54, 0.71, 0.88, 1.05]
SCALES_COCO = [0.07, 0.15, 0.33, 0.51, 0.69, 0.87, 1.05]
MEAN = [123, 117, 104]


@pytest.fixture(scope='module')
def golden():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    import __graft_entry__ as entry
    entry.build()
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.fixture(scope='module')
def root(tmp_path_factory, golden):
    path = str(tmp_path_factory.mktemp('voc') / 'data') + os.sep
    ds.write(path)
    assert ds.digest(path) == golden['digest']
    return path


def ssd300(n_classes, mode, scales, seed, input_scale=1.0):
    """The notebooks' SSD300 with seeded he-normal weights; ``input_scale`` multiplies conv1_1's kernel (the pixels are not
    divided by 127.5, so 1/128 keeps the activations of the whole network O(1), as the notebook's pretrained trunk does)."""
    from oracle import synth
    from oracle.model import SSD300_AR, vgg_weight_shapes
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    extra = dict(confidence_thresh=0.01, iou_threshold=0.45, top_k=200, nms_max_output_size=400) if mode == 'inference' else {}
    model = ssd_300(image_size=(300, 300, 3), n_classes=n_classes, mode=mode, l2_regularization=0.0005, scales=scales,
                    aspect_ratios_per_layer=SSD300_AR, two_boxes_for_ar1=True, steps=[8, 16, 32, 64, 100, 300],
                    offsets=[0.5] * 6, clip_boxes=False, variances=[0.1, 0.1, 0.2, 0.2], normalize_coords=True, subtract_mean=MEAN,
                    swap_channels=[2, 1, 0], **extra)
    w = synth.synth_weights(seed, vgg_weight_shapes(300, n_classes), bias_scale=0.02)
    w['conv4_3_norm/gamma'] = np.full((512,), 20.0, np.float32)
    w['conv1_1/kernel'] *= np.float32(input_scale)
    model.set_weights(w)
    return model


def built_dataset(root, record, **kwargs):
    """A constructor-built dataset with the golden's lists."""
    from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator
    return DataGenerator(filenames=[os.path.join(root, f) for f in record['filenames']], labels=record['labels'],
                         image_ids=record['image_ids'], eval_neutral=record['eval_neutral'], **kwargs)


def voc_evaluation_notebook(model, dataset):
    """The evaluation cells of ssd300_evaluation.ipynb."""
    from ssd_keras_b200.eval_utils.average_precision_evaluator import Evaluator
    evaluator = Evaluator(model=model, n_classes=20, data_generator=dataset, model_mode='inference')
    results = evaluator(img_height=300, img_width=300, batch_size=8, data_generator_mode='resize', round_confidences=False,
                        matching_iou_threshold=0.5, border_pixels='include', sorting_algorithm='quicksort', average_precision_mode='sample',
                        num_recall_points=11, ignore_neutral_boxes=True, return_precisions=True, return_recalls=True,
                        return_average_precisions=True, verbose=True)
    evaluator.get_num_gt_per_class(ignore_neutral_boxes=True, verbose=False, ret=False)
    evaluator.match_predictions(ignore_neutral_boxes=True, matching_iou_threshold=0.5, border_pixels='include',
                                sorting_algorithm='quicksort', verbose=True, ret=False)
    precisions, recalls = evaluator.compute_precision_recall(verbose=True, ret=True)
    average_precisions = evaluator.compute_average_precisions(mode='integrate', num_recall_points=11, verbose=True, ret=True)
    mean_average_precision = evaluator.compute_mean_average_precision(ret=True)
    return results, (mean_average_precision, average_precisions, precisions, recalls), evaluator.num_gt_per_class


def assert_identical(a, b, where):
    if isinstance(a, (list, tuple)):
        assert len(a) == len(b), where
        for k, (x, y) in enumerate(zip(a, b)):
            assert_identical(x, y, '%s[%d]' % (where, k))
    else:
        x, y = np.asarray(a), np.asarray(b)
        assert x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y, equal_nan=True), where


def test_voc_evaluation_notebook(root, golden):
    from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator
    im07, an07, sets07 = ds.voc_dirs(root, 'VOC2007')
    model = ssd300(20, 'inference', SCALES_VOC, 3)
    dataset = DataGenerator()
    dataset.parse_xml(images_dirs=[im07], image_set_filenames=[os.path.join(sets07, 'test.txt')], annotations_dirs=[an07],
                      classes=ds.VOC_CLASSES, include_classes='all', exclude_truncated=False, exclude_difficult=False, ret=False)
    reference = built_dataset(root, golden['xml']['test'])
    assert dataset.get_dataset() == reference.get_dataset()
    with contextlib.redirect_stdout(io.StringIO()):
        got = voc_evaluation_notebook(model, dataset)
        want = voc_evaluation_notebook(model, reference)
    assert_identical(got, want, 'results')
    mean_ap, aps, precisions, recalls = got[0]
    assert sum(got[2]) > 0 and sum(len(p) for p in precisions) > 0 and np.isfinite(mean_ap)


def coco_evaluation_notebook(model, dataset, annotations, results_file):
    """The prediction and evaluation cells of ssd300_evaluation_COCO.ipynb, batch size scaled to wrap the 8 images."""
    from ssd_keras_b200.eval_utils.coco_eval import COCO, COCOeval
    from ssd_keras_b200.eval_utils.coco_utils import get_coco_category_maps, predict_all_to_json
    cats_to_classes, classes_to_cats, cats_to_names, classes_to_names = get_coco_category_maps(annotations)
    predict_all_to_json(out_file=results_file, model=model, img_height=300, img_width=300, classes_to_cats=classes_to_cats,
                        data_generator=dataset, batch_size=3, data_generator_mode='resize', model_mode='inference', confidence_thresh=0.01,
                        iou_threshold=0.45, top_k=200, normalize_coords=True)
    coco_gt = COCO(annotations)
    coco_dt = coco_gt.loadRes(results_file)
    image_ids = sorted(coco_gt.getImgIds())
    coco_eval = COCOeval(cocoGt=coco_gt, cocoDt=coco_dt, iouType='bbox')
    coco_eval.params.imgIds = image_ids
    coco_eval.evaluate()
    coco_eval.accumulate()
    coco_eval.summarize()
    with open(results_file) as f:
        return f.read(), np.asarray(coco_eval.stats)


def test_coco_evaluation_notebook(root, golden, tmp_path):
    from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator
    val_dir, val = ds.coco_paths(root, 'val')
    model = ssd300(len(ds.COCO_CATS), 'inference', SCALES_COCO, 4)
    dataset = DataGenerator()
    dataset.parse_json(images_dirs=[val_dir], annotations_filenames=[val], ground_truth_available=False, include_classes='all', ret=False)
    reference = built_dataset(root, golden['json']['no_gt'])
    assert dataset.get_dataset() == reference.get_dataset() and dataset.labels is None
    with contextlib.redirect_stdout(io.StringIO()):
        got = coco_evaluation_notebook(model, dataset, val, str(tmp_path / 'parsed.json'))
        want = coco_evaluation_notebook(model, reference, val, str(tmp_path / 'built.json'))
    assert got[0] == want[0] and len(json.loads(got[0])) > 100
    assert np.array_equal(got[1], want[1]) and got[1].shape == (12,)


def test_generate_over_parsed_xml_equals_the_reference(root, golden):
    from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator
    from ssd_keras_b200.data_generator.object_detection_2d_geometric_ops import Resize
    from ssd_keras_b200.data_generator.object_detection_2d_photometric_ops import ConvertTo3Channels
    g = golden['generate']
    im07, an07, sets07 = ds.voc_dirs(root, 'VOC2007')
    gen = DataGenerator()
    gen.parse_xml(images_dirs=[im07], image_set_filenames=[os.path.join(sets07, 'test.txt')], annotations_dirs=[an07])
    np.random.seed(g['seed'])
    it = gen.generate(batch_size=g['batch_size'], shuffle=True, transformations=[ConvertTo3Channels(), Resize(300, 300)], label_encoder=None,
                      returns={'processed_images', 'processed_labels', 'filenames', 'image_ids', 'evaluation-neutral', 'original_labels'},
                      keep_images_without_gt=False)
    for k, want in enumerate(g['batches']):
        x, y, files, ids, neutral, original = next(it)
        x = x.cpu().numpy()
        assert np.array_equal(x, np.round(x)) and x.min() >= 0 and x.max() <= 255
        assert [ds.image_digest(a) for a in x.astype(np.uint8)] == want['x'] and list(x.shape) == want['x_shape'], k
        assert [a.tolist() for a in y] == want['labels'] and all(a.dtype == np.float64 for a in y), k
        assert ds.rel(root, files) == want['filenames'] and ids == want['image_ids'] and neutral == want['eval_neutral'], k
        assert [np.asarray(a).tolist() for a in original] == want['original_labels'], k
        state = np.random.get_state()
        assert ds.image_digest(state[1]) == want['state_digest'] and state[2] == want['pos'], k


def test_ssd300_training_notebook(root, tmp_path):
    """The data cells of ssd300_training.ipynb (without the optional HDF5 cell), then fit_generator over a few steps and
    epochs with the notebook's callbacks."""
    from oracle.model import SSD300_AR
    from ssd_keras_b200.callbacks import CSVLogger, LearningRateScheduler, TerminateOnNaN
    from ssd_keras_b200.data_generator.data_augmentation_chain_original_ssd import SSDDataAugmentation
    from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator
    from ssd_keras_b200.data_generator.object_detection_2d_geometric_ops import Resize
    from ssd_keras_b200.data_generator.object_detection_2d_photometric_ops import ConvertTo3Channels
    from ssd_keras_b200.keras_loss_function.keras_ssd_loss import SSDLoss
    from ssd_keras_b200.optimizers import SGD
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    model = ssd300(20, 'training', SCALES_VOC, 5, input_scale=1 / 128)
    model.compile(optimizer=SGD(lr=0.001, momentum=0.9, decay=0.0, nesterov=False), loss=SSDLoss(neg_pos_ratio=3, alpha=1.0).compute_loss)
    train_dataset = DataGenerator(load_images_into_memory=False, hdf5_dataset_path=None)
    val_dataset = DataGenerator(load_images_into_memory=False, hdf5_dataset_path=None)
    im07, an07, sets07 = ds.voc_dirs(root, 'VOC2007')
    im12, an12, sets12 = ds.voc_dirs(root, 'VOC2012')
    train_dataset.parse_xml(images_dirs=[im07, im12], image_set_filenames=[os.path.join(sets07, 'trainval.txt'), os.path.join(sets12, 'trainval.txt')],
                            annotations_dirs=[an07, an12], classes=ds.VOC_CLASSES, include_classes='all', exclude_truncated=False,
                            exclude_difficult=False, ret=False)
    val_dataset.parse_xml(images_dirs=[im07], image_set_filenames=[os.path.join(sets07, 'test.txt')], annotations_dirs=[an07],
                          classes=ds.VOC_CLASSES, include_classes='all', exclude_truncated=False, exclude_difficult=True, ret=False)
    batch_size = 4
    ssd_data_augmentation = SSDDataAugmentation(img_height=300, img_width=300, background=MEAN)
    predictor_sizes = [model.get_layer(n).output_shape[1:3] for n in ('conv4_3_norm_mbox_conf', 'fc7_mbox_conf', 'conv6_2_mbox_conf',
                                                                      'conv7_2_mbox_conf', 'conv8_2_mbox_conf', 'conv9_2_mbox_conf')]
    ssd_input_encoder = SSDInputEncoder(img_height=300, img_width=300, n_classes=20, predictor_sizes=predictor_sizes, scales=SCALES_VOC,
                                        aspect_ratios_per_layer=SSD300_AR, two_boxes_for_ar1=True, steps=[8, 16, 32, 64, 100, 300],
                                        offsets=[0.5] * 6, clip_boxes=False, variances=[0.1, 0.1, 0.2, 0.2], matching_type='multi',
                                        pos_iou_threshold=0.5, neg_iou_limit=0.5, normalize_coords=True)
    np.random.seed(7)
    train_generator = train_dataset.generate(batch_size=batch_size, shuffle=True, transformations=[ssd_data_augmentation],
                                             label_encoder=ssd_input_encoder, returns={'processed_images', 'encoded_labels'},
                                             keep_images_without_gt=False)
    val_generator = val_dataset.generate(batch_size=batch_size, shuffle=False, transformations=[ConvertTo3Channels(), Resize(height=300, width=300)],
                                         label_encoder=ssd_input_encoder, returns={'processed_images', 'encoded_labels'},
                                         keep_images_without_gt=False)
    assert train_dataset.get_dataset_size() == 12 and val_dataset.get_dataset_size() == 10

    def lr_schedule(epoch):
        return 0.001 if epoch < 2 else 0.0001

    log = str(tmp_path / 'ssd300_pascal_07+12_training_log.csv')
    callbacks = [LearningRateScheduler(schedule=lr_schedule, verbose=1), TerminateOnNaN(), CSVLogger(filename=log, separator=',', append=True)]
    epochs = 3
    with contextlib.redirect_stdout(io.StringIO()):
        history = model.fit_generator(generator=train_generator, steps_per_epoch=2, epochs=epochs, callbacks=callbacks,
                                      validation_data=val_generator, validation_steps=2, initial_epoch=0)
    loss, val_loss = history.history['loss'], history.history['val_loss']
    assert len(loss) == len(val_loss) == epochs and all(np.isfinite(loss)) and all(np.isfinite(val_loss)), (loss, val_loss)
    assert model.optimizer.lr == 0.0001
    with open(log, newline='') as f:
        rows = list(csv.reader(f))
    assert rows[0][0] == 'epoch' and [r[0] for r in rows[1:]] == [str(e) for e in range(epochs)]
