"""The notebooks' train and predict loops on ``DataGenerator.generate``'s device batches (models/_keras_api.py, models/_graph.py).

- ``fit_generator`` pulls batch i+1 while step i runs: from the same seeds it trains and validates on the batches of a serial
  ``train_on_batch`` loop, bit for bit, with the same learning rates, on SSD7 with Adam fed by the SSD7 notebook's chain (whose
  degenerate-box read-back runs on the generator's side stream) and on a small SSD300-style graph with SGD fed by
  ``SSDDataAugmentation``.  Each run keeps a device copy of every batch as its step was enqueued, so a batch the ahead-pull
  overwrote before its step read it would show up as a different batch.  The losses, weights and optimizer state are held to
  the drift between two serial runs (the training step is not bit-reproducible run to run).
- ``predict`` / ``predict_on_batch`` / ``predict_generator`` take the CUDA batches of ``generate()`` and return what the host
  copies give, in 'training', 'inference' and 'inference_fast' modes; a CUDA batch of another dtype, device or size raises.
- The SSD7 notebook's prediction cells run as written."""
import importlib.util
import os
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
H7, W7, B7, N_CLASSES = 96, 128, 4, 5
SCALES7 = [0.08, 0.16, 0.32, 0.64, 0.96]
CHAIN7 = dict(random_brightness=(-48, 48, 0.5), random_contrast=(0.5, 1.8, 0.5), random_saturation=(0.5, 1.8, 0.5),
              random_hue=(18, 0.5), random_flip=0.5, random_translate=((0.03, 0.5), (0.03, 0.5), 0.5), random_scale=(0.5, 2.0, 0.5),
              n_trials_max=3, clip_boxes=True, overlap_criterion='area', bounds_box_filter=(0.3, 1.0), bounds_validator=(0.5, 1.0),
              n_boxes_min=1, background=(0, 0, 0))


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


def _images(seed, shapes, n_classes):
    """Blocks of random colour with 1-4 boxes of 8-40 px per image, int64 labels as the parsers give them."""
    rng = np.random.default_rng(seed)
    images, labels = [], []
    for h, w in shapes:
        base = rng.integers(0, 256, (h // 8 + 2, w // 8 + 2, 3), dtype=np.uint8)
        images.append(np.ascontiguousarray(np.repeat(np.repeat(base, 8, 0), 8, 1)[:h, :w]))
        k = int(rng.integers(1, 5))
        x0, y0 = rng.integers(0, w - 44, k), rng.integers(0, h - 44, k)
        labels.append(np.stack([rng.integers(1, n_classes + 1, k), x0, y0, x0 + rng.integers(8, 40, k), y0 + rng.integers(8, 40, k)], 1))
    return images, labels


def _dataset(images, labels):
    """A fresh in-memory DataGenerator: generate() shuffles the dataset's lists in place, so every run gets its own."""
    from ssd_keras_b200.data_generator.object_detection_2d_data_generator import DataGenerator
    gen = DataGenerator(filenames=['img_%02d.png' % i for i in range(len(images))], labels=[l.copy() for l in labels])
    gen.images = list(images)
    return gen


# -- SSD7, Adam, the SSD7 notebook's chain ------------------------------------------------------------------------------------
def _ssd7(mode='training'):
    from ssd_keras_b200.models.keras_ssd7 import build_model
    return build_model((H7, W7, 3), N_CLASSES, mode=mode, l2_regularization=0.0005, scales=SCALES7, aspect_ratios_global=[0.5, 1.0, 2.0],
                       two_boxes_for_ar1=True, variances=[1.0, 1.0, 1.0, 1.0], normalize_coords=True, subtract_mean=127.5,
                       divide_by_stddev=127.5, return_predictor_sizes=True)


def _ssd7_encoder(predictor_sizes):
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    return SSDInputEncoder(img_height=H7, img_width=W7, n_classes=N_CLASSES, predictor_sizes=predictor_sizes, scales=SCALES7,
                           aspect_ratios_global=[0.5, 1.0, 2.0], two_boxes_for_ar1=True, clip_boxes=False, variances=[1.0, 1.0, 1.0, 1.0],
                           matching_type='multi', pos_iou_threshold=0.5, neg_iou_limit=0.3, normalize_coords=True)


def _ssd7_setup():
    from ssd_keras_b200.data_generator.data_augmentation_chain_constant_input_size import DataAugmentationConstantInputSize
    from ssd_keras_b200.keras_loss_function.keras_ssd_loss import SSDLoss
    from ssd_keras_b200.optimizers import Adam
    train, val = _images(1, [(H7, W7)] * 16, N_CLASSES), _images(2, [(H7, W7)] * 8, N_CLASSES)

    def make():
        model, sizes = _ssd7()
        model.compile(optimizer=Adam(lr=0.001, beta_1=0.9, beta_2=0.999, epsilon=1e-08, decay=0.0),
                      loss=SSDLoss(neg_pos_ratio=3, alpha=1.0).compute_loss)
        enc = _ssd7_encoder(sizes)
        gens = [_dataset(*d).generate(batch_size=B7, shuffle=True, transformations=[DataAugmentationConstantInputSize(**CHAIN7)],
                                      label_encoder=enc, returns={'processed_images', 'encoded_labels'}, keep_images_without_gt=True)
                for d in (train, val)]
        return model, gens[0], gens[1]
    return make


# -- a small SSD300-style graph, SGD, SSDDataAugmentation -----------------------------------------------------------------------
HW3, B3 = 64, 4
CASE3 = ('vgg_two_heads', HW3, B3, [('conv', 'c1', 64, 3, 1, 1, 1, 1), ('conv', 'c2', 64, 3, 1, 1, 1, 1), ('l2norm', 'n2', 'c2'),
                                     ('head', 'h1', 'n2'), ('pool', 'p1', 2, 2, 0), ('conv', 'c3', 128, 3, 1, 1, 1, 1),
                                     ('head', 'h2', 'c3')])


def _train_check():
    spec = importlib.util.spec_from_file_location('train_check', os.path.join(ROOT, 'tools', 'train_check.py'))
    tc = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tc)
    return tc


def _ssd300_setup():
    from ssd_keras_b200.data_generator.data_augmentation_chain_original_ssd import SSDDataAugmentation
    from ssd_keras_b200.keras_loss_function.keras_ssd_loss import SSDLoss
    from ssd_keras_b200.optimizers import SGD
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    tc = _train_check()
    rng = np.random.default_rng(3)
    shapes = [(int(rng.integers(70, 140)), int(rng.integers(70, 140))) for _ in range(24)]
    data = _images(4, shapes, 4)
    train, val = (data[0][:16], data[1][:16]), (data[0][16:], data[1][16:])

    def make():
        model, _, n_cls = tc.build(CASE3)
        model.compile(optimizer=SGD(lr=1e-3, momentum=0.9, decay=0.0, nesterov=False), loss=SSDLoss(neg_pos_ratio=3, alpha=1.0).compute_loss)
        a = model.anchor_cfg
        enc = SSDInputEncoder(HW3, HW3, n_cls - 1, model.predictor_sizes, scales=a['scales'], aspect_ratios_per_layer=a['aspect_ratios_per_layer'],
                              two_boxes_for_ar1=True, clip_boxes=False, variances=[0.1, 0.1, 0.2, 0.2], matching_type='multi',
                              pos_iou_threshold=0.5, neg_iou_limit=0.5, normalize_coords=True)
        gens = [_dataset(*d).generate(batch_size=B3, shuffle=True, transformations=[SSDDataAugmentation(HW3, HW3)], label_encoder=enc,
                                      returns={'processed_images', 'encoded_labels'}) for d in (train, val)]
        return model, gens[0], gens[1]
    return make


def _keep_batches(model, kept):
    """Wraps the model's step enqueues so that they keep a device copy of each batch (and the learning rate a training step
    used)."""
    enqueue, enqueue_test = model._enqueue_train_step, model._enqueue_test_step

    def keeping(x, y):
        kept.append((x.clone(), y.clone(), model.optimizer.lr))
        return enqueue(x, y)

    def keeping_test(x, y):
        kept.append((x.clone(), y.clone(), None))
        return enqueue_test(x, y)
    model._enqueue_train_step, model._enqueue_test_step = keeping, keeping_test


def _run(make, fit, epochs=2, steps=4, val_steps=2, seed=7):
    """Trains a fresh model over the seeded batches, with fit_generator or with a serial train_on_batch loop; returns the
    per-step losses, the validation losses, the batches (training and validation, in order) with the learning rates, the
    weights and the optimizer state."""
    np.random.seed(seed)
    random.seed(seed)
    model, train, val = make()
    kept, losses = [], []
    _keep_batches(model, kept)
    if fit:
        class Losses:
            def on_batch_end(self, batch, logs):
                losses.append(logs['loss'])

            def on_epoch_begin(self, epoch, logs):
                model.optimizer.lr = model.optimizer.lr * 0.5 if epoch else model.optimizer.lr
        h = model.fit_generator(train, steps_per_epoch=steps, epochs=epochs, callbacks=[Losses()], validation_data=val, validation_steps=val_steps)
        val_losses = h.history['val_loss']
    else:
        val_losses = []
        for epoch in range(epochs):
            if epoch:
                model.optimizer.lr = model.optimizer.lr * 0.5
            for _ in range(steps):
                losses.append(model.train_on_batch(*next(train)[:2]))
            tot, n = 0.0, 0
            for _ in range(val_steps):
                x, y = next(val)[:2]
                tot += model.test_on_batch(x, y) * len(x)
                n += len(x)
            val_losses.append(tot / n)
    return dict(losses=losses, val_losses=val_losses, batches=[(x.cpu().numpy(), y.cpu().numpy(), lr) for x, y, lr in kept],
                weights=model.get_weights(), opt=model._fit_trainer.get_optimizer_state())


def _distance(a, b):
    """Largest relative difference of the losses, largest absolute difference of the weights and of the optimizer state."""
    rel = lambda u, v: float(np.max(np.abs(np.subtract(u, v)) / np.abs(v)))          # noqa: E731
    w = max(float(np.max(np.abs(a['weights'][k] - b['weights'][k]))) for k in a['weights'])
    o = max(float(np.max(np.abs(sa[k] - sb[k]))) for sa, sb in zip(a['opt']['slots'], b['opt']['slots']) for k in sa)
    return {'losses': max(rel(a['losses'], b['losses']), rel(a['val_losses'], b['val_losses'])), 'weights': w, 'opt': o}


@pytest.mark.parametrize('setup', ['ssd7_adam', 'ssd300_sgd'])
def test_fit_generator_equals_the_serial_loop(setup):
    make = {'ssd7_adam': _ssd7_setup, 'ssd300_sgd': _ssd300_setup}[setup]()
    serial = _run(make, fit=False)
    piped = _run(make, fit=True)
    again = _run(make, fit=False)
    # what the loop's order decides, bit for bit: every training and validation batch in its place, with the learning rate of
    # each step, and so the loss of the first step
    assert len(serial['batches']) == len(piped['batches']) == 2 * (4 + 2)
    for (xs, ys, lrs), (xp, yp, lrp) in zip(serial['batches'], piped['batches']):
        assert np.array_equal(xs, xp) and np.array_equal(ys, yp) and lrs == lrp
    assert all(np.isfinite(serial['losses'])) and len(set(serial['losses'])) > 1
    assert piped['losses'][0] == serial['losses'][0]
    assert len(piped['losses']) == 8 and len(piped['val_losses']) == 2
    assert serial['opt']['iterations'] == piped['opt']['iterations'] == 8
    assert sorted(serial['weights']) == sorted(piped['weights']) and len(serial['opt']['slots']) == len(piped['opt']['slots'])
    # From the first update on, two runs of the same serial loop differ: the weight and bias gradients are summed with float
    # atomics, in the order the blocks finish, and how far two runs drift apart varies from run to run (with Adam, whose
    # update has the size of the learning rate whatever the gradient's, by up to ~5e-3 in the weights after 8 steps).  The
    # pipelined run must stay within 16 times that drift or 1e-5, whichever is larger (with SGD it has differed from the
    # serial run by 1.3e-6 in the weights, against a drift of 6e-8); a step trained twice, skipped or on another batch would
    # move weights by about lr x gradient, far more than that.
    spread, gap = _distance(again, serial), _distance(piped, serial)
    print('%s: serial vs serial %s, fit_generator vs serial %s' % (setup, spread, gap))
    for k in gap:
        assert gap[k] <= max(16 * spread[k], 1e-5), (k, gap, spread)


# -- prediction on device batches -------------------------------------------------------------------------------------------
def _predict_batches(returns=('processed_images',), seed=11):
    from ssd_keras_b200.data_generator.data_augmentation_chain_constant_input_size import DataAugmentationConstantInputSize
    np.random.seed(seed)
    random.seed(seed)
    gen = _dataset(*_images(5, [(H7, W7)] * 12, N_CLASSES)).generate(
        batch_size=B7, shuffle=True, transformations=[DataAugmentationConstantInputSize(**CHAIN7)], returns=set(returns),
        keep_images_without_gt=True)
    return gen


@pytest.mark.parametrize('mode', ['training', 'inference', 'inference_fast'])
def test_predict_takes_generate_batches(mode):
    import torch
    model, _ = _ssd7(mode)
    gen = _predict_batches()
    batches = [next(gen)[0] for _ in range(3)]
    assert all(b.is_cuda and b.dtype == torch.float32 for b in batches)
    per_batch = []
    for x in batches:
        y_dev = model.predict(x)
        y_host = model.predict(x.cpu().numpy())
        assert isinstance(y_dev, np.ndarray) and y_dev.dtype == y_host.dtype and np.array_equal(y_dev, y_host)
        assert np.array_equal(model.predict_on_batch(x), y_host)
        assert np.array_equal(model.predict_on_batch(x.cpu().numpy()), y_host)
        per_batch.append(y_host)
    # predict slices a CUDA array on the device: a batch size that does not divide N gives what the host copy gives
    both = torch.cat(batches[:2])
    assert np.array_equal(model.predict(both, batch_size=3), model.predict(both.cpu().numpy(), batch_size=3))
    # predict_generator over generate() itself, from the same seed
    assert np.array_equal(model.predict_generator(_predict_batches(), steps=3), np.concatenate(per_batch))


def test_device_batches_of_another_dtype_device_or_size_are_refused(monkeypatch):
    import torch
    model, _ = _ssd7()
    x = next(_predict_batches())[0]
    for bad in (x.double(), x.half(), x[:, :, :-1]):
        with pytest.raises(ValueError):
            model.predict(bad)
        with pytest.raises(ValueError):
            model.predict_on_batch(bad)
        with pytest.raises(ValueError):
            list(model.predict_stream([bad]))
    calls = [model.predict, model.predict_on_batch]
    if torch.cuda.device_count() > 1:
        other = x.to('cuda:1')
        calls.append(lambda t: model.predict_generator(iter([(t, None)]), steps=1))
    else:                                                   # one GPU: the model's device is made to be another one
        other = x
        monkeypatch.setattr(torch.cuda, 'current_device', lambda: 1)
    for call in calls:
        with pytest.raises(ValueError, match='cuda:'):
            call(other)


def test_ssd7_notebook_prediction_cells():
    """ssd7_training.ipynb's prediction cells: generate() with transformations=[] and the notebook's returns, predict on the
    CUDA batch, decode_detections on the result."""
    from ssd_keras_b200.ssd_encoder_decoder.ssd_output_decoder import decode_detections
    model, _ = _ssd7()
    images, labels = _images(6, [(H7, W7)] * 6, N_CLASSES)
    val_dataset = _dataset(images, labels)
    np.random.seed(0)
    predict_generator = val_dataset.generate(batch_size=1, shuffle=True, transformations=[], label_encoder=None,
                                             returns={'processed_images', 'processed_labels', 'filenames'}, keep_images_without_gt=False)
    for _ in range(3):
        batch_images, batch_labels, batch_filenames = next(predict_generator)
        i = int(batch_filenames[0][4:6])
        assert np.array_equal(batch_images.cpu().numpy()[0], images[i].astype(np.float32))
        assert np.array_equal(batch_labels[0], labels[i].astype(np.float64))
        y_pred = model.predict(batch_images)
        assert np.array_equal(y_pred, model.predict(batch_images.cpu().numpy()))
        y_pred_decoded = decode_detections(y_pred, confidence_thresh=0.5, iou_threshold=0.45, top_k=200, normalize_coords=True,
                                           img_height=H7, img_width=W7)
        assert len(y_pred_decoded) == 1 and y_pred_decoded[0].ndim == 2 and y_pred_decoded[0].shape[1] == 6
