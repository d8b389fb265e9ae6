"""Resuming a run from a full-model checkpoint, host side: ``model.save`` writes Keras' ``training_config`` and
``/optimizer_weights``, ``load_model`` compiles the model again and keeps the optimizer state for the first training step
(ssd300_training.ipynb / ssd7_training.ipynb: ``ModelCheckpoint(save_weights_only=False)``, then ``load_model(path,
custom_objects={'compute_loss': ...})`` and ``fit_generator(..., initial_epoch=...)``).  The optimizer state is set by hand or
comes from a stub trainer: no device needed (tests/test_gpu_resume_training.py covers the device)."""
import json

import numpy as np
import pytest

from ssd_keras_b200 import optimizers
from ssd_keras_b200.keras_loss_function.keras_ssd_loss import SSDLoss
from ssd_keras_b200.misc_utils.hdf5_lite import read_attributes, read_datasets, read_keras_weights, read_optimizer_weights
from ssd_keras_b200.models import load_model
from ssd_keras_b200.models.keras_ssd7 import build_model


def _model():
    return build_model((96, 96, 3), 5, mode='training', scales=[0.08, 0.16, 0.32, 0.64, 0.96], weights_seed=3)


def _trainable(m):
    return {k: s for k, s in m.weight_shapes().items() if not k.endswith(('/moving_mean', '/moving_variance'))}


def _state(m, n_slots, iterations, seed=0):
    rng = np.random.default_rng(seed)
    return {'iterations': iterations,
            'slots': [{k: rng.standard_normal(s).astype(np.float32) for k, s in _trainable(m).items()} for _ in range(n_slots)]}


class _StubTrainer:
    """What KerasTrainingMixin reads of the trainer it has been training with."""

    def __init__(self, state):
        self.state, self.iterations = state, state['iterations']

    def get_optimizer_state(self):
        return self.state


def _trained(opt, loss, n_slots, iterations=7, seed=0):
    m = _model()
    m.compile(optimizer=opt, loss=loss.compute_loss)
    st = _state(m, n_slots, iterations, seed)
    m._fit_trainer = _StubTrainer(st)
    return m, st


def _same_state(a, b):
    return a['iterations'] == b['iterations'] and len(a['slots']) == len(b['slots']) and all(
        sorted(x) == sorted(y) and all(np.array_equal(x[k], y[k]) for k in x) for x, y in zip(a['slots'], b['slots']))


@pytest.mark.parametrize('kind', ['sgd', 'adam'])
def test_file_layout_weight_names_and_training_config(kind, tmp_path):
    loss = SSDLoss(neg_pos_ratio=2, n_neg_min=5, alpha=0.5)
    if kind == 'sgd':
        opt, prefixes = optimizers.SGD(lr=1e-3, momentum=0.9), ('moments',)
    else:
        opt, prefixes = optimizers.Adam(lr=1e-3, beta_1=0.8, beta_2=0.99, epsilon=1e-7), ('ms', 'vs')
    m, st = _trained(opt, loss, len(prefixes))
    m.optimizer.lr = 2.5e-4                                  # a LearningRateScheduler's value: the file keeps the current lr
    p = str(tmp_path / 'ckpt.h5')
    m.save(p)
    tc = json.loads(bytes(read_attributes(p)['training_config']).rstrip(b'\x00').decode())
    oc = tc['optimizer_config']
    if kind == 'sgd':
        assert oc == {'class_name': 'SGD', 'config': {'lr': 2.5e-4, 'momentum': 0.9, 'decay': 0.0, 'nesterov': False}}
    else:
        assert oc == {'class_name': 'Adam', 'config': {'lr': 2.5e-4, 'beta_1': 0.8, 'beta_2': 0.99, 'decay': 0.0, 'epsilon': 1e-7,
                                                       'amsgrad': False}}
    assert tc['loss'] == 'compute_loss' and tc['ssd_loss'] == {'neg_pos_ratio': 2, 'n_neg_min': 5, 'alpha': 0.5}
    ow = read_optimizer_weights(p)
    order = list(_trainable(m))                              # the trainer's parameter order
    want = ['iterations:0'] + ['%s/%s:0' % (pre, k) for pre in prefixes for k in st['slots'][0] if k in order]
    assert [n for n, _ in ow] == want
    assert ow[0][1].dtype == np.int64 and ow[0][1].shape == () and int(ow[0][1]) == 7
    for (n, a) in ow[1:]:
        pre, key = n.split('/', 1)
        assert np.array_equal(a, st['slots'][prefixes.index(pre)][key[:-2]]), n
    ds = read_datasets(p)
    assert '/optimizer_weights/iterations:0' in ds and '/optimizer_weights/%s/conv1/kernel:0' % prefixes[-1] in ds
    assert '/model_weights/conv1/conv1/kernel:0' in ds
    assert sorted(read_keras_weights(p)) == sorted(m.weights)   # the optimizer group is not read as weights
    assert sorted(load_model(p, compile=False).get_weights()) == sorted(m.weights)


def test_uncompiled_or_untrained_models_write_no_optimizer_weights(tmp_path):
    m = _model()
    m.save(str(tmp_path / 'plain.h5'))
    assert 'training_config' not in read_attributes(str(tmp_path / 'plain.h5'))
    assert read_optimizer_weights(str(tmp_path / 'plain.h5')) == []
    m.compile(optimizer=optimizers.SGD(lr=1e-3, momentum=0.9), loss=SSDLoss().compute_loss)
    m.save(str(tmp_path / 'compiled.h5'))
    assert 'training_config' in read_attributes(str(tmp_path / 'compiled.h5'))
    assert read_optimizer_weights(str(tmp_path / 'compiled.h5')) == []
    m2, _ = _trained(optimizers.SGD(lr=1e-3, momentum=0.9), SSDLoss(), 1)
    m2.save(str(tmp_path / 'no_opt.h5'), include_optimizer=False)
    assert 'training_config' not in read_attributes(str(tmp_path / 'no_opt.h5'))
    assert read_optimizer_weights(str(tmp_path / 'no_opt.h5')) == []
    m3 = load_model(str(tmp_path / 'compiled.h5'))             # compiled, no state to resume
    assert m3._compiled[0] == 'sgd' and m3._pending_opt_state is None


def test_load_model_with_and_without_custom_objects(tmp_path):
    loss = SSDLoss(neg_pos_ratio=4, n_neg_min=2, alpha=2.0)
    m, st = _trained(optimizers.Adam(lr=3e-4), loss, 2)
    p = str(tmp_path / 'ckpt.h5')
    m.save(p)
    mine = SSDLoss(neg_pos_ratio=4, n_neg_min=2, alpha=2.0)
    a = load_model(p, custom_objects={'AnchorBoxes': None, 'compute_loss': mine.compute_loss})
    assert a._compiled[0] == 'adam' and a._compiled[1] is mine
    assert isinstance(a.optimizer, optimizers.Adam) and a.optimizer.lr == 3e-4
    assert _same_state(a._pending_opt_state, st)
    b = load_model(p)
    lo = b._compiled[1]
    assert isinstance(lo, SSDLoss) and (lo.neg_pos_ratio, lo.n_neg_min, lo.alpha) == (4, 2, 2.0)
    assert _same_state(b._pending_opt_state, st)
    c = load_model(p, custom_objects={'compute_loss': None})   # not an SSDLoss method: rebuilt from the file
    assert isinstance(c._compiled[1], SSDLoss) and c._compiled[1].alpha == 2.0
    d = load_model(p, compile=False)
    assert d._compiled is None and d._pending_opt_state is None
    for k in m.weights:
        assert np.array_equal(d.weights[k], m.weights[k])


def test_pending_state_is_dropped_by_compile_set_weights_load_weights(tmp_path):
    m, st = _trained(optimizers.SGD(lr=1e-3, momentum=0.9), SSDLoss(), 1)
    p = str(tmp_path / 'ckpt.h5')
    m.save(p)
    m.save_weights(str(tmp_path / 'w.h5'))
    a = load_model(p)
    assert a._pending_opt_state is not None
    a.compile(optimizer=optimizers.SGD(lr=1e-3, momentum=0.9), loss=SSDLoss().compute_loss)
    assert a._pending_opt_state is None
    b = load_model(p)
    b.set_weights(b.get_weights())
    assert b._pending_opt_state is None
    c = load_model(p)
    c.load_weights(str(tmp_path / 'w.h5'))
    assert c._pending_opt_state is None
    for x in (a, b, c):                                      # nothing left to save but the training config
        x.save(str(tmp_path / 'again.h5'))
        assert read_optimizer_weights(str(tmp_path / 'again.h5')) == []


@pytest.mark.parametrize('kind', ['sgd', 'adam'])
def test_saving_a_loaded_untrained_model_rewrites_the_state_bit_for_bit(kind, tmp_path):
    opt = optimizers.SGD(lr=1e-3, momentum=0.9) if kind == 'sgd' else optimizers.Adam(lr=1e-3)
    m, _ = _trained(opt, SSDLoss(), 1 if kind == 'sgd' else 2, iterations=12345)
    p1, p2 = str(tmp_path / 'a.h5'), str(tmp_path / 'b.h5')
    m.save(p1)
    load_model(p1).save(p2)
    w1, w2 = read_optimizer_weights(p1), read_optimizer_weights(p2)
    assert [n for n, _ in w1] == [n for n, _ in w2]
    assert all(a.dtype == b.dtype and a.tobytes() == b.tobytes() for (_, a), (_, b) in zip(w1, w2))
    assert read_attributes(p1)['training_config'].tobytes() == read_attributes(p2)['training_config'].tobytes()


def test_a_state_that_does_not_fit_the_model_is_refused_at_load(tmp_path):
    p = str(tmp_path / 'bad.h5')
    # a wrong shape
    m, st = _trained(optimizers.SGD(lr=1e-3, momentum=0.9), SSDLoss(), 1)
    st['slots'][0]['conv4/bias'] = st['slots'][0]['conv4/bias'][:-1]
    m.save(p)
    with pytest.raises(ValueError, match='conv4/bias'):
        load_model(p)
    load_model(p, compile=False)                             # the weights alone still load
    # a missing weight
    m, st = _trained(optimizers.SGD(lr=1e-3, momentum=0.9), SSDLoss(), 1)
    del st['slots'][0]['bn3/beta']
    m.save(p)
    with pytest.raises(ValueError, match='bn3/beta'):
        load_model(p)
    # one slot for Adam after it has taken steps
    m, st = _trained(optimizers.Adam(lr=1e-3), SSDLoss(), 1)
    m.save(p)
    with pytest.raises(ValueError, match='slot'):
        load_model(p)
    # a state written for another model
    other = build_model((96, 96, 3), 3, mode='training', scales=[0.08, 0.16, 0.32, 0.64, 0.96])
    other.compile(optimizer=optimizers.SGD(lr=1e-3, momentum=0.9), loss=SSDLoss().compute_loss)
    other._fit_trainer = _StubTrainer(_state(other, 1, 3))
    other.save(p)
    mine = _model()
    mine.compile(optimizer=optimizers.SGD(lr=1e-3, momentum=0.9), loss=SSDLoss().compute_loss)
    from ssd_keras_b200.training import check_optimizer_state
    with pytest.raises(ValueError, match='classes4/kernel'):
        check_optimizer_state(mine, 'sgd', load_model(p)._pending_opt_state)
