"""The SSD7, variable-input-size and satellite chains on the device: ``DataGenerator.generate`` against the real reference's
batches (tests/golden/make_augmentation_chains_golden.py), bit for bit in the images and the processed labels, its encoded
labels against the oracle encoder, and the SSD7 notebook scaled down: PNG files and a CSV, ``parse_csv``,
``DataAugmentationConstantInputSize``, an encoder from ``build_model``'s predictor sizes, ``fit_generator`` with ``Adam`` and
``SSDLoss``, and a validation generator without transformations."""
import random

import numpy as np
import pytest

from test_augmentation_chains_cpu import RUNS, assert_states, golden_generator, seed

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()


def _encoder_config(h, w):
    return dict(img_height=h, img_width=w, n_classes=5, predictor_sizes=[(h // 4, w // 4), (h // 8, w // 8), (h // 16, w // 16)],
                scales=[0.1, 0.3, 0.6, 0.9], aspect_ratios_global=[0.5, 1.0, 2.0], two_boxes_for_ar1=True, steps=None, offsets=None,
                clip_boxes=False, variances=[1.0, 1.0, 1.0, 1.0], matching_type='multi', pos_iou_threshold=0.5, neg_iou_limit=0.3,
                normalize_coords=True)


@pytest.mark.parametrize('name', sorted(RUNS))
def test_generate_equals_the_reference(name):
    from oracle.encoder import OracleEncoder
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    g, gen, chain, keep = golden_generator(name)
    h, w = g[name + '_b0_x'].shape[1:3]
    cfg = _encoder_config(h, w)
    seed(g, name)
    it = gen.generate(batch_size=int(g['batch_size']), shuffle=True, transformations=[chain()], label_encoder=SSDInputEncoder(**cfg),
                      returns={'processed_images', 'encoded_labels', 'processed_labels', 'filenames'}, keep_images_without_gt=keep)
    for k in range(int(g[name + '_n_batches'])):
        p = '%s_b%d_' % (name, k)
        x, y_enc, labels, files = next(it)
        assert [int(f) for f in files] == g[p + 'files'].tolist(), p
        assert np.array_equal(x.cpu().numpy(), g[p + 'x'].astype(np.float32)), p
        counts = g[p + 'counts']
        assert [len(a) for a in labels] == counts.tolist(), p
        assert np.array_equal(np.concatenate(labels), g[p + 'labels']), p
        ref = np.split(g[p + 'labels'], np.cumsum(counts)[:-1])
        y_ref = OracleEncoder(**cfg)(ref).astype(np.float32)
        y = y_enc.cpu().numpy()
        np.testing.assert_array_equal(y[:, :, :6] > 0.5, y_ref[:, :, :6] > 0.5)
        np.testing.assert_allclose(y, y_ref, rtol=1e-6, atol=1e-6)
        assert_states(g, p)


def _write_dataset(root, n, h, w, rng):
    """n PNGs with 1-3 bright rectangles of three classes on a dark, noisy background, and their CSV."""
    from PIL import Image
    (root / 'images').mkdir()
    rows = ['frame,xmin,xmax,ymin,ymax,class_id']
    for i in range(n):
        img = rng.integers(0, 40, (h, w, 3)).astype(np.uint8)
        for _ in range(int(rng.integers(1, 4))):
            cls = int(rng.integers(1, 4))
            bh, bw = int(rng.integers(h // 5, h // 2)), int(rng.integers(w // 6, w // 3))
            y0, x0 = int(rng.integers(0, h - bh)), int(rng.integers(0, w - bw))
            img[y0:y0 + bh, x0:x0 + bw] = (200 if cls == 1 else 60, 200 if cls == 2 else 60, 200 if cls == 3 else 60)
            rows.append('%d.png,%d,%d,%d,%d,%d' % (i, x0, x0 + bw, y0, y0 + bh, cls))
        Image.fromarray(img).save(str(root / 'images' / ('%d.png' % i)))
    (root / 'labels.csv').write_text('\n'.join(rows) + '\n')


def test_ssd7_notebook_end_to_end(tmp_path):
    from ssd_keras_b200.data_generator.data_augmentation_chain_constant_input_size import DataAugmentationConstantInputSize
    from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator
    from ssd_keras_b200.keras_loss_function.keras_ssd_loss import SSDLoss
    from ssd_keras_b200.models.keras_ssd7 import build_model
    from ssd_keras_b200.optimizers import Adam
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    h, w, n_classes = 120, 192, 3
    scales, ars = [0.08, 0.16, 0.32, 0.64, 0.96], [0.5, 1.0, 2.0]
    _write_dataset(tmp_path, 16, h, w, np.random.default_rng(5))
    model, predictor_sizes = build_model((h, w, 3), n_classes, mode='training', l2_regularization=0.0005, scales=scales,
                                         aspect_ratios_global=ars, two_boxes_for_ar1=True, variances=[1.0, 1.0, 1.0, 1.0],
                                         normalize_coords=True, subtract_mean=127.5, divide_by_stddev=127.5, return_predictor_sizes=True)
    model.compile(optimizer=Adam(lr=0.001), loss=SSDLoss(neg_pos_ratio=3, alpha=1.0).compute_loss)
    train, val = DataGenerator(load_images_into_memory=False), DataGenerator(load_images_into_memory=True)
    for gen in (train, val):
        gen.parse_csv(images_dir=str(tmp_path / 'images'), labels_filename=str(tmp_path / 'labels.csv'),
                      input_format=['image_name', 'xmin', 'xmax', 'ymin', 'ymax', 'class_id'], include_classes='all')
    assert train.get_dataset_size() == 16 and train.labels[0].dtype == np.int64
    augmentation = DataAugmentationConstantInputSize(random_brightness=(-48, 48, 0.5), random_contrast=(0.5, 1.8, 0.5),
                                                     random_saturation=(0.5, 1.8, 0.5), random_hue=(18, 0.5), random_flip=0.5,
                                                     random_translate=((0.03, 0.5), (0.03, 0.5), 0.5), random_scale=(0.5, 2.0, 0.5),
                                                     n_trials_max=3, clip_boxes=True, overlap_criterion='area', bounds_box_filter=(0.3, 1.0),
                                                     bounds_validator=(0.5, 1.0), n_boxes_min=1, background=(0, 0, 0))
    encoder = SSDInputEncoder(img_height=h, img_width=w, n_classes=n_classes, predictor_sizes=predictor_sizes, scales=scales,
                              aspect_ratios_global=ars, two_boxes_for_ar1=True, steps=None, offsets=None, clip_boxes=False,
                              variances=[1.0, 1.0, 1.0, 1.0], matching_type='multi', pos_iou_threshold=0.5, neg_iou_limit=0.3,
                              normalize_coords=True)
    np.random.seed(0)
    random.seed(0)
    train_gen = train.generate(batch_size=4, shuffle=True, transformations=[augmentation], label_encoder=encoder,
                               returns={'processed_images', 'encoded_labels'}, keep_images_without_gt=False)
    val_gen = val.generate(batch_size=4, shuffle=False, transformations=[], label_encoder=encoder,
                           returns={'processed_images', 'encoded_labels'}, keep_images_without_gt=False)
    history = model.fit_generator(generator=train_gen, steps_per_epoch=8, epochs=5, validation_data=val_gen, validation_steps=4)
    loss, val_loss = history.history['loss'], history.history['val_loss']
    assert len(loss) == 5 and all(np.isfinite(loss)) and all(np.isfinite(val_loss)), (loss, val_loss)
    assert loss[-1] < loss[0] and val_loss[-1] < val_loss[0], (loss, val_loss)
