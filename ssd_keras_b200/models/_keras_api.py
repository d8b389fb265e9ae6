"""The training side of the Keras ``Model`` surface the reference's notebooks use (``ssd300_training.ipynb:153-173, 437-448``,
``ssd7_training.ipynb:153-156, 330-340``): ``compile(optimizer, loss)``, ``train_on_batch``, ``test_on_batch``,
``fit_generator(generator, steps_per_epoch, epochs, callbacks, validation_data, validation_steps, initial_epoch)`` and
``evaluate_generator`` -- thin host code over ``SSDTrainer`` (encode-free: the generator yields ``(images, y_encoded)`` exactly as
the reference's ``DataGenerator.generate(..., label_encoder=SSDInputEncoder, returns={'processed_images', 'encoded_labels'})``).

A step is two halves: enqueueing its device work (``_enqueue_train_step`` / ``_enqueue_test_step``, which return the per-image
loss tensor without waiting) and reading the mean loss as a float (``_read_loss``, which waits for the step).
``train_on_batch`` / ``test_on_batch`` run them back to back.  ``fit_generator`` and ``evaluate_generator`` pull the next batch
from the generator between the two, so that the host work of batch i+1 (the shuffle, the augmentation draws, decoding and
packing) runs while the device computes step i, as Keras' generator queue lets it."""
import numpy as np


class History:
    """keras.callbacks.History: ``history`` maps a metric name to its per-epoch values, ``epoch`` lists the epochs run."""

    def __init__(self):
        self.epoch, self.history = [], {}


def _pull(it):
    """The next ``(x, y)`` of a generator, or the exception pulling it raised: a loop that pulls a batch ahead raises it where a
    serial loop would have pulled that batch, after the steps and callbacks before it."""
    try:
        return next(it)[:2]
    except Exception as e:                               # noqa: BLE001 -- re-raised by the step that needs the batch
        return e


def _call(callbacks, name, *args):
    for cb in callbacks:
        fn = getattr(cb, name, None)
        if callable(fn):
            fn(*args)


# the dataset-name prefix of each optimiser slot below /optimizer_weights: Keras' SGD keeps [iterations] + moments, Adam
# [iterations] + ms + vs
SLOT_PREFIXES = {'sgd': ('moments',), 'adam': ('ms', 'vs')}


class KerasTrainingMixin:
    optimizer = None
    _compiled = None
    _fit_trainer = None
    _pending_opt_state = None          # optimiser state loaded by load_model, applied to the next trainer _trainer_for makes
    stop_training = False

    def compile(self, optimizer, loss=None, **kwargs):
        """``optimizer``: ``ssd_keras_b200.optimizers.SGD`` / ``Adam`` (or any object with their attributes, or 'sgd' / 'adam');
        ``loss``: ``SSDLoss(...).compute_loss`` (the bound method, as in the reference) or the ``SSDLoss`` object, or the same of
        an ``SSDFocalLoss``."""
        from .. import optimizers
        from ..keras_loss_function.keras_ssd_loss import KernelLoss
        if kwargs:
            raise TypeError('compile() got unsupported arguments: %s' % sorted(kwargs))
        if isinstance(optimizer, str):
            if optimizer.lower() not in ('sgd', 'adam'):
                raise ValueError("optimizer must be 'sgd' or 'adam' (the two the reference trains with), got %r" % (optimizer,))
            optimizer = optimizers.SGD() if optimizer.lower() == 'sgd' else optimizers.Adam()
        kind = getattr(optimizer, 'kind', type(optimizer).__name__.lower())
        if kind not in ('sgd', 'adam') or not hasattr(optimizer, 'lr'):
            raise ValueError('unsupported optimizer %r: SGD (lr, momentum) and Adam (lr, beta_1, beta_2, epsilon) are implemented' % (optimizer,))
        owner = getattr(loss, '__self__', loss)
        if not isinstance(owner, KernelLoss):
            raise ValueError('loss must be SSDLoss(...).compute_loss (keras_loss_function/keras_ssd_loss.py:98) or '
                             'SSDFocalLoss(...).compute_loss: the training step computes that loss and its gradient on the device')
        self.optimizer, self._compiled = optimizer, (kind, owner)
        self._fit_trainer = None
        self._pending_opt_state = None

    # -- the training half of a full-model file (Keras' training_config and /optimizer_weights) --------------------------------
    def _training_config(self):
        """Keras' ``training_config`` root attribute of ``model.save``, with the loss's parameters under its ``config_key``
        (``'ssd_loss'`` or ``'ssd_focal_loss'``), which load_model rebuilds the loss from when ``custom_objects`` does not bring
        it."""
        kind, lossobj = self._compiled
        o = self.optimizer
        if kind == 'sgd':
            opt = {'class_name': 'SGD', 'config': {'lr': float(o.lr), 'momentum': float(getattr(o, 'momentum', 0.0)), 'decay': 0.0,
                                                   'nesterov': False}}
        else:
            opt = {'class_name': 'Adam', 'config': {'lr': float(o.lr), 'beta_1': float(getattr(o, 'beta_1', 0.9)),
                                                    'beta_2': float(getattr(o, 'beta_2', 0.999)), 'decay': 0.0,
                                                    'epsilon': float(getattr(o, 'epsilon', 1e-8)), 'amsgrad': False}}
        out = {'optimizer_config': opt, 'loss': 'compute_loss', 'metrics': [], 'sample_weight_mode': None, 'loss_weights': None}
        out[lossobj.config_key] = lossobj.config()
        return out

    def _optimizer_weights(self):
        """``[(name, array), ...]`` for ``/optimizer_weights`` in Keras' order -- ``iterations:0``, then each slot in the trainer's
        parameter order -- from the trainer that has been training, or the loaded state still waiting for one; ``[]`` when the
        model has not trained."""
        t = self._fit_trainer
        state = t.get_optimizer_state() if t is not None and t.iterations > 0 else self._pending_opt_state
        if state is None:
            return []
        out = [('iterations:0', np.array(state['iterations'], np.int64))]
        for prefix, named in zip(SLOT_PREFIXES[self._compiled[0]], state['slots']):
            out += [('%s/%s:0' % (prefix, k), v) for k, v in named.items()]
        return out

    def _restore_training(self, config, opt_weights, custom_objects):
        """``load_model``'s ``compile=True``: compile with the stored optimizer and learning rate, and keep the stored optimizer
        state (checked against this model) for the trainer of the next step."""
        from .. import optimizers
        from ..keras_loss_function.keras_ssd_focal_loss import SSDFocalLoss
        from ..keras_loss_function.keras_ssd_loss import KernelLoss, SSDLoss
        from ..training import check_optimizer_state
        oc = config['optimizer_config']
        c = oc['config']
        if oc['class_name'] == 'SGD':
            opt = optimizers.SGD(lr=c['lr'], momentum=c.get('momentum', 0.0))
        elif oc['class_name'] == 'Adam':
            opt = optimizers.Adam(lr=c['lr'], beta_1=c.get('beta_1', 0.9), beta_2=c.get('beta_2', 0.999), epsilon=c.get('epsilon', 1e-8))
        else:
            raise ValueError('training_config names the optimizer %r: SGD and Adam are implemented' % (oc['class_name'],))
        loss = (custom_objects or {}).get('compute_loss')
        if not isinstance(getattr(loss, '__self__', None), KernelLoss):
            cls = next((c for c in (SSDFocalLoss, SSDLoss) if c.config_key in config), SSDLoss)
            loss = cls(**config[cls.config_key]).compute_loss
        self.compile(optimizer=opt, loss=loss)
        if not opt_weights:
            return
        if opt_weights[0][0] != 'iterations:0':
            raise ValueError('optimizer weights must start with iterations:0, got %s' % opt_weights[0][0])
        prefixes = SLOT_PREFIXES[opt.kind]
        slots = {}
        for name, arr in opt_weights[1:]:
            prefix, _, key = name.partition('/')
            if prefix not in prefixes or not key.endswith(':0'):
                raise ValueError('optimizer weight %s does not belong to %s' % (name, oc['class_name']))
            slots.setdefault(prefixes.index(prefix), {})[key[:-2]] = arr
        if sorted(slots) != list(range(len(slots))):
            raise ValueError('optimizer weights: %s has no %s slot' % (oc['class_name'], prefixes[0]))
        state = {'iterations': int(opt_weights[0][1]), 'slots': [slots[i] for i in range(len(slots))]}
        check_optimizer_state(self, opt.kind, state)
        self._pending_opt_state = state

    def _trainer_for(self, batch):
        from ..training import SSDTrainer
        if self._compiled is None:
            raise RuntimeError('You must compile a model before training/testing. Use `model.compile(optimizer, loss)`.')
        kind, lossobj = self._compiled
        t = self._fit_trainer
        if t is None or t.batch != batch:
            if t is not None:
                raise ValueError('this model has been training on batches of %d images; a batch of %d would need its own optimizer '
                                 'state (the reference generator yields constant-size batches)' % (t.batch, batch))
            o = self.optimizer
            t = SSDTrainer(self, batch, lr=o.lr, momentum=getattr(o, 'momentum', 0.0), optimizer=kind, beta_1=getattr(o, 'beta_1', 0.9),
                           beta_2=getattr(o, 'beta_2', 0.999), epsilon=getattr(o, 'epsilon', 1e-8), loss=lossobj)
            if self._pending_opt_state is not None:
                t.set_optimizer_state(self._pending_opt_state)
                self._pending_opt_state = None
            self._fit_trainer = t
        t.lr = float(self.optimizer.lr)                  # a callback (or the caller) may have changed the learning rate
        return t

    @staticmethod
    def _to_cuda(a):
        import torch
        if torch.is_tensor(a):
            return a.to(device='cuda', dtype=torch.float32).contiguous()
        return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()

    def _enqueue_train_step(self, x, y):
        """Enqueues forward, loss, backward and update of one optimizer step on ``(x, y)`` on the current stream; returns the
        per-image loss, a CUDA tensor (B,), without waiting for the device."""
        if self._compiled is None:
            raise RuntimeError('You must compile a model before training/testing. Use `model.compile(optimizer, loss)`.')
        xd, yd = self._to_cuda(x), self._to_cuda(y)
        return self._trainer_for(int(xd.shape[0])).train_on_batch(xd, yd)

    def _enqueue_test_step(self, x, y):
        """Enqueues the inference-phase forward and loss of ``(x, y)``; returns the per-image loss tensor (B,) without waiting."""
        if self._compiled is None:
            raise RuntimeError('You must compile a model before training/testing. Use `model.compile(optimizer, loss)`.')
        xd, yd = self._to_cuda(x), self._to_cuda(y)
        if self.decoder is not None:
            raise ValueError("test_on_batch needs the raw predictions: build the model with mode='training'")
        return self._compiled[1].compute_loss(yd, self.forward_device(xd))

    @staticmethod
    def _read_loss(loss):
        """The scalar Keras reports for a step: the mean over the batch of its per-image loss, as a float (waits for the step)."""
        return float(loss.mean().item())

    def train_on_batch(self, x, y):
        """One optimizer step on ``(x, y)``; returns the scalar Keras reports: the mean over the batch of ``compute_loss``."""
        return self._read_loss(self._enqueue_train_step(x, y))

    def test_on_batch(self, x, y):
        """The same scalar without an update, in the inference phase (moving BatchNormalization statistics), like Keras."""
        return self._read_loss(self._enqueue_test_step(x, y))

    def _split_step(self, public, enqueue):
        """``(enqueue, read)`` for the steps of the generator loops.  A ``train_on_batch`` / ``test_on_batch`` that a subclass or
        the caller has replaced is what Keras' loops call, so it is called whole in the enqueue's place and its float read as
        it is."""
        fn = getattr(self, public)
        if getattr(fn, '__func__', None) is getattr(KerasTrainingMixin, public):
            return enqueue, self._read_loss
        return fn, float

    def evaluate_generator(self, generator, steps):
        """Keras' ``evaluate_generator``: the mean over the images of ``steps`` batches of ``test_on_batch``'s loss.  The next
        batch is pulled from ``generator`` while the device computes the loss of the current one."""
        enqueue, read = self._split_step('test_on_batch', self._enqueue_test_step)
        it = iter(generator)
        steps = int(steps)
        tot, n = 0.0, 0
        batch = next(it)[:2] if steps > 0 else None
        for step in range(steps):
            if isinstance(batch, Exception):
                raise batch
            x, y = batch
            pending = enqueue(x, y)
            if step + 1 < steps:
                batch = _pull(it)
            tot += read(pending) * len(x)
            n += len(x)
        return tot / max(n, 1)

    def fit_generator(self, generator, steps_per_epoch, epochs=1, verbose=0, callbacks=None, validation_data=None,
                      validation_steps=None, initial_epoch=0):
        """Keras' loop: ``epochs - initial_epoch`` epochs of ``steps_per_epoch`` batches from ``generator`` (an endless iterator of
        ``(images, y_encoded)``), the epoch's mean loss in ``history['loss']``, the validation loss in ``history['val_loss']``.
        Callbacks are duck-typed: ``set_model``, ``on_train_begin/end(logs)``, ``on_epoch_begin/end(epoch, logs)``,
        ``on_batch_end(batch, logs)`` are called where present; a callback may set ``model.optimizer.lr`` or ``model.stop_training``.

        Each step but the last of an epoch runs as: enqueue step i on the device, pull batch i+1 from ``generator``, read the
        loss of step i, call ``on_batch_end(i)``.  The host therefore plans and assembles batch i+1 while the device trains on
        batch i; the learning rate a callback sets in ``on_batch_end(i)`` is the one step i+1 uses, as in a serial loop.  The
        last step of an epoch pulls nothing ahead, so validation and the next epoch find ``generator`` where a serial loop
        leaves it (the training and validation generators may be one object).  Every step trains on the batch, with the
        learning rate, that a serial ``train_on_batch`` loop gives it, and the callbacks and history see what they see
        there, with one difference: when a callback stops training in the middle of an epoch, the batch after the last one
        trained has already been pulled and is not trained on (Keras' queue does the same)."""
        callbacks = list(callbacks or [])
        hist = History()
        _call(callbacks, 'set_model', self)
        self.stop_training = False
        _call(callbacks, 'on_train_begin', {})
        enqueue, read = self._split_step('train_on_batch', self._enqueue_train_step)
        it = iter(generator)
        steps = int(steps_per_epoch)
        for epoch in range(int(initial_epoch), int(epochs)):
            _call(callbacks, 'on_epoch_begin', epoch, {})
            tot, n = 0.0, 0
            batch = next(it)[:2] if steps > 0 else None
            for step in range(steps):
                if isinstance(batch, Exception):
                    raise batch
                x, y = batch
                pending = enqueue(x, y)
                if step + 1 < steps:
                    batch = _pull(it)
                l = read(pending)
                tot += l * len(x)
                n += len(x)
                _call(callbacks, 'on_batch_end', step, {'loss': l, 'size': len(x)})
                if not np.isfinite(l):
                    self.stop_training = any(type(cb).__name__ == 'TerminateOnNaN' for cb in callbacks) or self.stop_training
                if self.stop_training:
                    break
            logs = {'loss': tot / max(n, 1)}
            if validation_data is not None:
                if validation_steps is None:
                    raise ValueError('`validation_steps` must be given when `validation_data` is a generator')
                logs['val_loss'] = self.evaluate_generator(validation_data, validation_steps)
            hist.epoch.append(epoch)
            for k, v in logs.items():
                hist.history.setdefault(k, []).append(v)
            if verbose:
                print('Epoch %d/%d - ' % (epoch + 1, epochs) + ' - '.join('%s: %.4f' % kv for kv in logs.items()), flush=True)
            _call(callbacks, 'on_epoch_end', epoch, logs)
            if self.stop_training:
                break
        _call(callbacks, 'on_train_end', {})
        self.history = hist
        return hist
