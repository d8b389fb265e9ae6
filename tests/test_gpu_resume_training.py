"""GPU tests of resuming a run from a full-model checkpoint, as the training notebooks do it (ssd300_training.ipynb,
ssd7_training.ipynb: ``ModelCheckpoint(save_weights_only=False)`` during ``fit_generator``, later ``load_model(path,
custom_objects={'compute_loss': ssd_loss.compute_loss})`` and ``fit_generator(..., initial_epoch=...)``):
- ssdk_trainer_write_opt_state is the bit-exact inverse of ssdk_trainer_read_opt_state on every span kind (conv / head kernel,
  bias, L2Normalization gamma, BatchNormalization gamma / beta), Adam's v included before its first update;
- the loaded model's trainer starts from the saved parameters, moving statistics, optimizer slots, step count and learning rate,
  bit for bit, at the saved batch size or another one;
- its first update is the one the restored state implies (oracle/opexact.py's optimizer references and bound), and not the one a
  fresh state would give.  The ratios go to SSDK_KERNEL_ERRORS_LOG (conv_cases.log_ratio)."""
import itertools

import numpy as np
import pytest

import conv_cases as cc
from oracle import opexact, synth

pytestmark = pytest.mark.gpu

SC7 = [0.08, 0.16, 0.32, 0.64, 0.96]
SC300 = [0.1, 0.2, 0.37, 0.54, 0.71, 0.88, 1.05]
TAGS = ('kernel', 'bias', 'gamma', 'bn_gamma', 'bn_beta')


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


def _ssd7():
    from ssd_keras_b200.models.keras_ssd7 import build_model
    return build_model((96, 96, 3), 5, mode='training', l2_regularization=5e-4, scales=SC7, normalize_coords=True, weights_seed=2,
                       subtract_mean=[127.5] * 3, divide_by_stddev=[127.5] * 3)


def _ssd300():
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    return ssd_300((300, 300, 3), 20, mode='training', scales=SC300, divide_by_stddev=[64.0] * 3, weights_seed=2)


def _vgg_heads_l2norm():
    """tools/train_check.py's VGG-style case: 3x3 convs, an L2Normalization, two fused heads, a pool."""
    import importlib.util
    import os
    root = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
    spec = importlib.util.spec_from_file_location('train_check', os.path.join(root, 'tools', 'train_check.py'))
    tc = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tc)
    return tc.build(tc.CASES[2])[0]


def _batches(m, B, n, seed):
    """(images, y_encoded) pairs for model m."""
    from oracle.encoder import OracleEncoder
    H, W, ncls = m.img_height, m.img_width, m.n_classes - 1
    if H == 300:
        enc = OracleEncoder(H, W, ncls, m.predictor_sizes, scales=SC300, aspect_ratios_per_layer=m.anchor_cfg['aspect_ratios_per_layer'],
                            steps=[8, 16, 32, 64, 100, 300], variances=[0.1, 0.1, 0.2, 0.2])
    else:
        enc = OracleEncoder(H, W, ncls, m.predictor_sizes, scales=SC7, aspect_ratios_global=[0.5, 1.0, 2.0], variances=[1.0] * 4,
                            pos_iou_threshold=0.4, neg_iou_limit=0.3, normalize_coords=True)
    assert np.array_equal(enc.anchors, m.anchors)
    return [(synth.synth_images(seed + i, B, H, W), enc(synth.synth_gt(seed + 50 + i, B, 4, W, H, ncls)).astype(np.float32))
            for i in range(n)]


def _flat(tr, fn, *args):
    """A flat float32 view of the trainer in the gradient's layout (ssdk_trainer_read_params / _read_opt_state)."""
    import torch
    from ssd_keras_b200 import _ffi
    out = torch.empty_like(tr.grad)
    _ffi.check(fn(tr.handle, *args, _ffi.dptr(out), _ffi.stream_ptr()))
    return out.cpu().numpy()


def _kernel_shapes(tr):
    """{(layer name, tag): (cout, kh, kw, cin) for kernel spans, None otherwise} of every parameter span."""
    from ssd_keras_b200 import _ffi
    m = tr.model
    out = {}
    for (name, tag) in tr.spans():
        ks = None
        if tag == 'kernel':
            s = m.specs[m.index[name]]
            cin = m._shapes[m.index[s.inp]][2]
            cout = s.cout if s.op == _ffi.OP_CONV else s.n_boxes * (m.n_classes + 4)
            ks = (cout, s.kh, s.kw, cin)
        out[(name, tag)] = ks
    return out


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same_state(a, b):
    return a['iterations'] == b['iterations'] and len(a['slots']) == len(b['slots']) and all(
        sorted(x) == sorted(y) and all(np.array_equal(_bits(x[k]), _bits(y[k])) for k in x) for x, y in zip(a['slots'], b['slots']))


# ------------------------------------------------------------------------------------------------------------------------------
# the entry point: write is the inverse of read, bit for bit
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('graph', ['ssd7', 'vgg_heads_l2norm'])
def test_write_then_read_every_slot_is_bit_exact(graph):
    import torch
    from ssd_keras_b200 import _ffi
    from ssd_keras_b200.training import SSDTrainer
    m = _ssd7() if graph == 'ssd7' else _vgg_heads_l2norm()
    tr = SSDTrainer(m, 2, lr=1e-3, optimizer='adam')
    want_tags = {'kernel', 'bias', 'bn_gamma', 'bn_beta'} if graph == 'ssd7' else {'kernel', 'bias', 'gamma'}
    assert {tag for _, tag in tr.spans()} == want_tags
    assert sum(c for _, c in tr.spans().values()) == tr.n_params
    rng = np.random.default_rng(5)
    lib = _ffi.lib()
    with pytest.raises(ValueError, match='slot'):           # v does not exist before the first Adam update or write
        _flat(tr, lib.ssdk_trainer_read_opt_state, 1)
    for slot in (1, 0, 1):                                  # slot 1 first: made by its write, before any update
        bits = rng.integers(0, 2 ** 32, tr.n_params, dtype=np.uint64).astype(np.uint32)
        bits[:8] = [0, 0x80000000, 1, 0x807fffff, 0x7f800000, 0xff800000, 0x7fc00001, 0x3f800000]   # +-0, denormals, inf, NaN
        src = torch.from_numpy(bits.view(np.float32).copy()).cuda()
        _ffi.check(lib.ssdk_trainer_write_opt_state(tr.handle, slot, _ffi.dptr(src), _ffi.stream_ptr()))
        got = _flat(tr, lib.ssdk_trainer_read_opt_state, slot)
        assert np.array_equal(got.view(np.uint32), bits), (graph, slot)
    src = torch.zeros_like(tr.grad)
    for bad in (2, -1):
        with pytest.raises(ValueError, match='slot'):
            _ffi.check(lib.ssdk_trainer_write_opt_state(tr.handle, bad, _ffi.dptr(src), _ffi.stream_ptr()))
    with pytest.raises(ValueError, match='NULL'):
        _ffi.check(lib.ssdk_trainer_write_opt_state(tr.handle, 0, None, _ffi.stream_ptr()))
    with pytest.raises(ValueError, match='NULL'):
        _ffi.check(lib.ssdk_trainer_write_opt_state(None, 0, _ffi.dptr(src), _ffi.stream_ptr()))
    # the same through the Keras-named state: HWIO kernels, heads split into conf / loc
    st = {'iterations': 9, 'slots': [{k: rng.standard_normal(np.shape(v)).astype(np.float32) for k, v in tr.gradients().items()}
                                     for _ in range(2)]}
    tr.set_optimizer_state(st)
    assert tr.iterations == 9 and _same_state(tr.get_optimizer_state(), st)
    with pytest.raises(ValueError, match='slot'):
        tr.set_optimizer_state({'iterations': 9, 'slots': st['slots'][:1]})


# ------------------------------------------------------------------------------------------------------------------------------
# resume through the notebooks' calls
# ------------------------------------------------------------------------------------------------------------------------------
CASES = [dict(name='sgd_ssd300', kind='sgd', B=2, B2=3), dict(name='adam_ssd7', kind='adam', B=4, B2=2)]


@pytest.mark.parametrize('case', CASES, ids=[c['name'] for c in CASES])
def test_resume_from_a_checkpoint_through_the_notebook_calls(case, tmp_path):
    import torch
    from ssd_keras_b200 import _ffi
    from ssd_keras_b200.callbacks import LearningRateScheduler, ModelCheckpoint
    from ssd_keras_b200.keras_loss_function.keras_ssd_loss import SSDLoss
    from ssd_keras_b200.models import load_model
    from ssd_keras_b200.optimizers import SGD, Adam
    sgd = case['kind'] == 'sgd'
    build = _ssd300 if sgd else _ssd7
    B, B2 = case['B'], case['B2']
    lr0 = 1e-3

    def schedule(epoch):
        return lr0 * 0.5 ** epoch
    m = build()
    data = _batches(m, B, 2, seed=3)
    ssd_loss = SSDLoss(neg_pos_ratio=3, alpha=1.0)
    m.compile(optimizer=SGD(lr=lr0, momentum=0.9, decay=0.0, nesterov=False) if sgd else Adam(lr=lr0, beta_1=0.9, beta_2=0.999,
                                                                                            epsilon=1e-08, decay=0.0),
              loss=ssd_loss.compute_loss)
    ckpt = ModelCheckpoint(str(tmp_path / 'epoch-{epoch:02d}.h5'), monitor='loss', save_best_only=False, save_weights_only=False)
    m.fit_generator(itertools.cycle(data), steps_per_epoch=2, epochs=2, callbacks=[ckpt, LearningRateScheduler(schedule)])
    path = str(tmp_path / 'epoch-02.h5')
    t0 = m._fit_trainer
    lib = _ffi.lib()
    # the state at save time: nothing has trained since the last checkpoint
    st0, w0, p0 = t0.get_optimizer_state(), t0.get_weights(), _flat(t0, lib.ssdk_trainer_read_params)
    assert st0['iterations'] == 4 and len(st0['slots']) == (1 if sgd else 2)

    def restored(model, batch):
        t = model._trainer_for(batch)
        assert model.optimizer.lr == m.optimizer.lr == schedule(1)
        assert t.iterations == 4 and _same_state(t.get_optimizer_state(), st0)
        assert np.array_equal(_bits(_flat(t, lib.ssdk_trainer_read_params)), _bits(p0))
        w = t.get_weights()                                  # the masters and the BatchNormalization moving statistics
        assert sorted(w) == sorted(w0) and all(np.array_equal(_bits(w[k]), _bits(w0[k])) for k in w0)
        return t

    # the first update after resume is the one the restored state implies
    m2 = load_model(path, custom_objects={'compute_loss': ssd_loss.compute_loss})
    assert m2._compiled[1] is ssd_loss
    t2 = restored(m2, B)
    x, y = data[0]
    t2.forward_backward(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda())
    g = t2.grad.cpu().numpy()
    w_b, s0 = _flat(t2, lib.ssdk_trainer_read_params), _flat(t2, lib.ssdk_trainer_read_opt_state, 0)
    s1 = None if sgd else _flat(t2, lib.ssdk_trainer_read_opt_state, 1)
    t2.apply(1.0)
    assert t2.iterations == 5
    w_a, m_a = _flat(t2, lib.ssdk_trainer_read_params), _flat(t2, lib.ssdk_trainer_read_opt_state, 0)
    v_a = None if sgd else _flat(t2, lib.ssdk_trainer_read_opt_state, 1)
    ratio, fresh = 0.0, 0.0
    for key, ks in _kernel_shapes(t2).items():
        o, c = t2.spans()[key]
        e = o + c
        common = dict(l2=t2.l2, scale=1.0, kernel_shape=ks)
        if sgd:
            got = {'w': w_a[o:e], 'v': m_a[o:e]}
            ref, bnd, _ = opexact.sgd_ref(w_b[o:e], s0[o:e], g[o:e], t2.lr, t2.momentum, **common)
            ref0, _, _ = opexact.sgd_ref(w_b[o:e], np.zeros(c, np.float32), g[o:e], t2.lr, t2.momentum, **common)
        else:
            got = {'w': w_a[o:e], 'm': m_a[o:e], 'v': v_a[o:e]}
            hyper = (t2.lr, t2.beta_1, t2.beta_2, t2.epsilon)
            ref, bnd, _ = opexact.adam_ref(w_b[o:e], s0[o:e], s1[o:e], g[o:e], *hyper, 5, **common)
            z = np.zeros(c, np.float32)
            ref0, _, _ = opexact.adam_ref(w_b[o:e], z, z, g[o:e], *hyper, 1, **common)
        r = opexact.state_ratio(got, ref, bnd)
        assert r <= 1.0, (case['name'], key, r)
        ratio, fresh = max(ratio, r), max(fresh, opexact.state_ratio(got, ref0, bnd))
    cc.log_ratio(dict(test='resume_first_update', case=case['name'], ratio=ratio, fresh_state_ratio=fresh))
    print('%s: first update after resume, |err| / bound = %.3g; against a fresh optimizer state = %.3g' % (case['name'], ratio, fresh))
    assert fresh > 1.0, ('a fresh optimizer state passes the bound', fresh)
    # resume at another batch size, then train on through the notebook's loop
    m3 = load_model(path, custom_objects={'compute_loss': ssd_loss.compute_loss})
    t3 = restored(m3, B2)
    assert t3.batch == B2
    h = m3.fit_generator(itertools.cycle(_batches(m3, B2, 2, seed=9)), steps_per_epoch=2, epochs=3, callbacks=[LearningRateScheduler(schedule)],
                         initial_epoch=2)
    assert h.epoch == [2] and np.isfinite(h.history['loss'][0])
    assert m3._fit_trainer is t3 and t3.iterations == 6 and t3.lr == schedule(2)
