"""The order of ``fit_generator`` / ``evaluate_generator`` (models/_keras_api.py) with the device step stubbed out: each step but
the last of an epoch is enqueued, then the next batch is pulled, then the loss is read and ``on_batch_end`` called.  The
history, the callback arguments and the learning rates each step sees are those of a serial ``train_on_batch`` loop, written
out below; a mid-epoch stop pulls exactly one batch more than that loop."""
import itertools

import numpy as np
import pytest

from ssd_keras_b200 import optimizers
from ssd_keras_b200.keras_loss_function.keras_ssd_loss import SSDLoss
from ssd_keras_b200.models.keras_ssd7 import build_model


def _model(log):
    """An SSD7 whose device halves only record: the enqueue returns the batch number, the read turns it into a loss."""
    m = build_model((96, 96, 3), 5, mode='training', scales=[0.08, 0.16, 0.32, 0.64, 0.96])
    m.compile(optimizer=optimizers.SGD(lr=1e-3, momentum=0.9), loss=SSDLoss().compute_loss)

    def enqueue(x, y):
        log.append(('enqueue', int(x[0, 0]), m.optimizer.lr))
        return int(x[0, 0])

    def enqueue_test(x, y):
        log.append(('enqueue_test', int(x[0, 0])))
        return -1 - int(x[0, 0])

    def read(token):
        log.append(('read', token))
        return 0.5 + 0.125 * (-1 - token) if token < 0 else 10.0 - 0.75 * token + (token % 3) * 0.3

    m._enqueue_train_step, m._enqueue_test_step, m._read_loss = enqueue, enqueue_test, read
    return m


NAN = float('nan')


def _generator(log):
    """Endless ``(x, y)`` batches of 1-3 images; ``x`` carries the batch number."""
    for j in itertools.count():
        log.append(('next', j))
        yield np.full((j % 3 + 1, 1), j, np.float32), np.zeros((j % 3 + 1, 1), np.float32)


class _Recorder:
    def __init__(self, log, stop_at=None, batch_decay=None):
        self.log, self.stop_at, self.batch_decay = log, stop_at, batch_decay

    def set_model(self, model):
        self.model = model
        self.log.append(('set_model',))

    def on_train_begin(self, logs):
        self.log.append(('train_begin', dict(logs)))

    def on_epoch_begin(self, epoch, logs):
        self.model.optimizer.lr = 1e-3 * 0.5 ** epoch               # a LearningRateScheduler
        self.log.append(('epoch_begin', epoch, dict(logs)))

    def on_batch_end(self, batch, logs):
        self.log.append(('batch_end', batch, dict(logs)))
        if self.batch_decay:
            self.model.optimizer.lr *= self.batch_decay
        if self.stop_at is not None and len([e for e in self.log if e[0] == 'batch_end']) == self.stop_at:
            self.model.stop_training = True

    def on_epoch_end(self, epoch, logs):
        self.log.append(('epoch_end', epoch, dict(logs)))

    def on_train_end(self, logs):
        self.log.append(('train_end', dict(logs)))


def _serial_fit(model, generator, steps_per_epoch, epochs=1, callbacks=None, validation_data=None, validation_steps=None,
                initial_epoch=0):
    """The serial loop: pull a batch, train on it, read its loss, call back; then the next batch."""
    from ssd_keras_b200.models._keras_api import History, _call
    callbacks = list(callbacks or [])
    hist = History()
    _call(callbacks, 'set_model', model)
    model.stop_training = False
    _call(callbacks, 'on_train_begin', {})
    it = iter(generator)
    for epoch in range(initial_epoch, epochs):
        _call(callbacks, 'on_epoch_begin', epoch, {})
        tot, n = 0.0, 0
        for step in range(steps_per_epoch):
            x, y = next(it)[:2]
            l = model.train_on_batch(x, y)
            tot += l * len(x)
            n += len(x)
            _call(callbacks, 'on_batch_end', step, {'loss': l, 'size': len(x)})
            if not np.isfinite(l):
                model.stop_training = any(type(cb).__name__ == 'TerminateOnNaN' for cb in callbacks) or model.stop_training
            if model.stop_training:
                break
        logs = {'loss': tot / max(n, 1)}
        if validation_data is not None:
            vit = iter(validation_data)
            vt, vn = 0.0, 0
            for _ in range(validation_steps):
                x, y = next(vit)[:2]
                vt += model.test_on_batch(x, y) * len(x)
                vn += len(x)
            logs['val_loss'] = vt / max(vn, 1)
        hist.epoch.append(epoch)
        for k, v in logs.items():
            hist.history.setdefault(k, []).append(v)
        _call(callbacks, 'on_epoch_end', epoch, logs)
        if model.stop_training:
            break
    _call(callbacks, 'on_train_end', {})
    return hist


def _without_pulls(log):
    return [e for e in log if e[0] != 'next']


def test_each_step_pulls_the_next_batch_before_its_loss_is_read():
    log = []
    m = _model(log)
    m.fit_generator(_generator(log), steps_per_epoch=3, epochs=2, callbacks=[_Recorder(log)])
    order = [e[:2] if e[0] in ('next', 'enqueue', 'read', 'batch_end') else e[:1] for e in log]
    epoch = [('epoch_begin',), ('next', 0), ('enqueue', 0), ('next', 1), ('read', 0), ('batch_end', 0),
             ('enqueue', 1), ('next', 2), ('read', 1), ('batch_end', 1), ('enqueue', 2), ('read', 2), ('batch_end', 2), ('epoch_end',)]
    second = [(e[0], e[1] + 3) if e[0] in ('next', 'enqueue', 'read') else e for e in epoch]
    assert order == [('set_model',), ('train_begin',)] + epoch + second + [('train_end',)]


def test_evaluate_generator_pulls_ahead_within_its_steps():
    log = []
    m = _model(log)
    v = m.evaluate_generator(_generator(log), 3)
    assert log == [('next', 0), ('enqueue_test', 0), ('next', 1), ('read', -1), ('enqueue_test', 1), ('next', 2), ('read', -2),
                   ('enqueue_test', 2), ('read', -3)]
    assert v == (0.5 * 1 + 0.625 * 2 + 0.75 * 3) / 6
    assert m.evaluate_generator(_generator([]), 0) == 0.0


@pytest.mark.parametrize('initial_epoch', [0, 1])
def test_shared_training_and_validation_generator_sees_the_serial_batches(initial_epoch):
    """No pull past the last step of an epoch: validation and the next epoch take the batches a serial loop gives them."""
    logs = {}
    for name, fit in (('pipelined', None), ('serial', _serial_fit)):
        log = logs[name] = []
        m = _model(log)
        g = _generator(log)
        kw = dict(steps_per_epoch=3, epochs=3, callbacks=[_Recorder(log)], validation_data=g, validation_steps=2,
                  initial_epoch=initial_epoch)
        h = m.fit_generator(g, **kw) if fit is None else fit(m, g, **kw)
        logs[name + '_history'] = (h.epoch, h.history)
    n_epochs = 3 - initial_epoch
    assert [e for e in logs['pipelined'] if e[0] == 'next'] == [('next', j) for j in range(5 * n_epochs)]
    assert [e for e in logs['pipelined'] if e[0] == 'enqueue_test'] == [('enqueue_test', 5 * k + j) for k in range(n_epochs) for j in (3, 4)]
    assert _without_pulls(logs['pipelined']) == _without_pulls(logs['serial'])
    assert logs['pipelined_history'] == logs['serial_history']


@pytest.mark.parametrize('batch_decay', [None, 0.9])
def test_history_callbacks_and_learning_rates_equal_the_serial_loop(batch_decay):
    """Everything but the pulls, in order: callback arguments, the learning rate each enqueued step saw (set per epoch, and
    per batch in on_batch_end), the losses read and the history."""
    runs = {}
    for name, fit in (('pipelined', None), ('serial', _serial_fit)):
        log = []
        m = _model(log)
        kw = dict(steps_per_epoch=4, epochs=3, callbacks=[_Recorder(log, batch_decay=batch_decay)],
                  validation_data=_generator([]), validation_steps=3)
        h = m.fit_generator(_generator(log), **kw) if fit is None else fit(m, _generator(log), **kw)
        runs[name] = (_without_pulls(log), h.epoch, h.history, m.optimizer.lr)
    assert runs['pipelined'] == runs['serial']
    lrs = [e[2] for e in runs['pipelined'][0] if e[0] == 'enqueue']
    assert len(lrs) == 12 and len(set(lrs)) == (3 if batch_decay is None else 12)


@pytest.mark.parametrize('stop_at', [2, 4, 7])
def test_a_mid_epoch_stop_consumes_exactly_one_extra_batch(stop_at):
    """A callback stops training after the stop_at-th step (4 steps per epoch): in the middle of an epoch one batch has been
    pulled and is never trained on; at the end of an epoch (step 4) none."""
    runs = {}
    for name, fit in (('pipelined', None), ('serial', _serial_fit)):
        log = []
        m = _model(log)
        kw = dict(steps_per_epoch=4, epochs=3, callbacks=[_Recorder(log, stop_at=stop_at)])
        h = m.fit_generator(_generator(log), **kw) if fit is None else fit(m, _generator(log), **kw)
        runs[name] = (log, h.epoch, h.history)
    pulled = {k: len([e for e in v[0] if e[0] == 'next']) for k, v in runs.items()}
    assert pulled['serial'] == stop_at
    assert pulled['pipelined'] == stop_at + (0 if stop_at % 4 == 0 else 1)
    assert _without_pulls(runs['pipelined'][0]) == _without_pulls(runs['serial'][0])
    assert runs['pipelined'][1:] == runs['serial'][1:]


def test_terminate_on_nan_stops_as_the_serial_loop_does():
    from ssd_keras_b200 import callbacks as cb
    runs = {}
    for name, fit in (('pipelined', None), ('serial', _serial_fit)):
        log = []
        m = _model(log)
        read = m._read_loss
        m._read_loss = lambda t: NAN if t == 5 else read(t)
        kw = dict(steps_per_epoch=4, epochs=3, callbacks=[_Recorder(log), cb.TerminateOnNaN()])
        h = m.fit_generator(_generator(log), **kw) if fit is None else fit(m, _generator(log), **kw)
        steps = [e for e in log if e[0] in ('enqueue', 'read', 'batch_end', 'epoch_begin')]    # the epoch means hold a NaN
        runs[name] = (steps, h.epoch, len([e for e in log if e[0] == 'next']))
    assert runs['pipelined'][:2] == runs['serial'][:2]
    assert runs['serial'][1] == [0, 1] and (runs['serial'][2], runs['pipelined'][2]) == (6, 7)


def test_a_failing_pull_surfaces_where_the_serial_loop_meets_it():
    """The generator raises when asked for batch 2: step 1 is still read and reported before the error propagates."""
    log = []
    m = _model(log)

    def gen():
        for j in range(2):
            log.append(('next', j))
            yield np.full((1, 1), j, np.float32), np.zeros((1, 1), np.float32)
        raise RuntimeError('no batch 2')
    with pytest.raises(RuntimeError, match='no batch 2'):
        m.fit_generator(gen(), steps_per_epoch=4, callbacks=[_Recorder(log)])
    assert [e[:2] for e in log if e[0] in ('read', 'batch_end')] == [('read', 0), ('batch_end', 0), ('read', 1), ('batch_end', 1)]
