"""GPU parity tests for the training step (SURVEY.md A16 / BASELINE config 3): loss, every gradient and the SGD-momentum
update of ``SSDLoss.loss_and_grad`` / ``ssdk_train_backward_layers`` / ``ssdk_train_apply`` against float64 torch autograd
over the same layer specs (oracle/graph.py) on identical weights, images and encoded ground truth.

Tolerance: the backward GEMMs run in the same bf16x3 mode as the forward pass (~16 significant bits per product, fp32
accumulation); gradients are compared at 2e-3 of the tensor's max magnitude (measured 5e-6 .. 2e-4; 1e-3 where one ReLU
mask element differs from the float64 run), updated weights at 2e-5 relative (what the gradient bar implies for these graphs;
measured 1e-6 .. 1.1e-5).  Losses: 1e-4 relative, also at the end of the full 23-layer SSD300 forward (measured 3.9e-5 against float64
with the cross-term accumulator of DESIGN.md section 3.1, 1.2e-4 without it; the loss kernel itself is checked at 1e-6 on
identical y_pred in test_gpu_codec.py); 5e-4 for SSD512."""
import importlib.util
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))


def _train_check():
    spec = importlib.util.spec_from_file_location('train_check', os.path.join(ROOT, 'tools', 'train_check.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


@pytest.mark.parametrize('case', [0, 1, 2, 3])
def test_small_graph_gradients(case):
    """conv / pool / 1x1 / l2norm / two heads / stride-2 / dilated / 'valid' graphs: all gradients + one SGD step."""
    assert _train_check().run_case(case) == 0


def _ssd300(B, seed=2):
    from oracle import synth
    from oracle.encoder import OracleEncoder
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    sc = [0.1, 0.2, 0.37, 0.54, 0.71, 0.88, 1.05]
    m = ssd_300((300, 300, 3), 20, mode='training', scales=sc, divide_by_stddev=[64.0] * 3, weights_seed=seed)
    w = m.get_weights()
    rng = np.random.default_rng(seed)
    for k in w:
        if k.endswith('/bias'):
            w[k] = (rng.standard_normal(w[k].shape) * 0.05).astype(np.float32)
    m.set_weights(w)
    enc = OracleEncoder(300, 300, 20, m.predictor_sizes, scales=sc, aspect_ratios_per_layer=m.anchor_cfg['aspect_ratios_per_layer'],
                        steps=[8, 16, 32, 64, 100, 300], variances=[0.1, 0.1, 0.2, 0.2])
    assert np.array_equal(enc.anchors, m.anchors)
    x = synth.synth_images(seed, B, 300, 300)
    y_true = enc(synth.synth_gt(seed + 1, B, 4, 300, 300, 20)).astype(np.float32)
    return m, w, x, y_true


def test_ssd300_step_matches_autograd():
    """SSD300, batch 2: loss, all 72 gradient tensors and the updated weights against float64 autograd."""
    import torch
    from oracle import graph as og
    from ssd_keras_b200.training import SSDTrainer
    B = 2
    m, w, x, y_true = _ssd300(B)
    lr, mom, l2 = 1e-3, 0.9, 5e-4
    tr = SSDTrainer(m, B, lr=lr, momentum=mom, l2_regularization=l2)
    xd, ytd = torch.from_numpy(x).cuda(), torch.from_numpy(y_true).cuda()
    loss, _ = tr.forward_backward(xd, ytd)
    torch.cuda.synchronize()
    grads = tr.gradients()
    params = og.make_params(m.specs, w, dtype=torch.float64)
    yp, _ = og.forward(m.specs, params, x, 21, m.anchors, [0.1, 0.1, 0.2, 0.2], dtype=torch.float64)
    lvec = og.ssd_loss_torch(y_true, yp)
    lvec.mean().backward()
    ref_l = lvec.detach().numpy()
    assert np.abs(loss.cpu().numpy() - ref_l).max() <= 1e-4 * np.abs(ref_l).max()
    assert set(grads) == set(w)
    # Deep in the backbone the comparison is ill-conditioned: a forward value within rounding distance of 0 flips its ReLU'
    # mask and moves one gradient entry by O(1e-3) of the tensor's max (tools/train_diag.py: conv6_1/bias has exactly one
    # channel off by 2.2e-3, all others <= 2e-5), and every layer below inherits that perturbation.  float32 torch autograd
    # deviates from float64 by 1e-3 .. 6e-3 (max-norm) on this very input.  So per tensor: median error <= 2e-3 of the
    # tensor's max, max-norm error <= 2e-2 as a guard against structural mistakes (the small graphs above are tight).
    worst_med, worst_max = 0.0, 0.0
    for k in sorted(grads):
        ref = params[k].grad.numpy()
        e = np.abs(grads[k] - ref).ravel() / (np.abs(ref).max() + 1e-30)
        worst_med, worst_max = max(worst_med, float(np.median(e))), max(worst_max, float(e.max()))
        assert np.median(e) < 2e-3 and e.max() < 2e-2, 'gradient %s: median err %.3e, max err %.3e' % (k, np.median(e), e.max())
    print('ssd300 B=2: worst gradient median err %.2e, max-norm %.2e' % (worst_med, worst_max))
    tr.apply(1.0)
    new_w = tr.get_weights()
    # the optimiser arithmetic, on the gradients the device produced (their own error is bounded above)
    ref_w, _ = og.sgd_step(w, grads, {}, lr, mom, l2)
    for k in w:
        assert np.abs(new_w[k] - ref_w[k]).max() <= 2e-6 * np.abs(ref_w[k]).max() + 1e-9, k


def test_ssd300_loss_decreases():
    """Ten SGD steps on one fixed batch: the mean loss falls, stays finite, and the forward plan picks up the new weights."""
    import torch
    from ssd_keras_b200.training import SSDTrainer
    B = 4
    m, w, x, y_true = _ssd300(B, seed=5)
    tr = SSDTrainer(m, B, lr=1e-3, momentum=0.9)
    xd, ytd = torch.from_numpy(x).cuda(), torch.from_numpy(y_true).cuda()
    losses = [float(tr.train_on_batch(xd, ytd).mean().item()) for _ in range(10)]
    assert all(np.isfinite(losses)), losses
    assert losses[-1] < 0.8 * losses[0], losses


def test_ssd512_step_matches_autograd():
    """SSD512, batch 1: exercises the geometries SSD300 does not have (64x64 ... 1x1 maps, the 4x4 'valid' conv10_2 whose
    weight gradient takes the transposed-operand fallback, seven heads).  Same bars as the SSD300 check."""
    import torch
    from oracle import graph as og
    from oracle import synth
    from oracle.encoder import OracleEncoder
    from ssd_keras_b200.models.keras_ssd512 import ssd_512
    from ssd_keras_b200.training import SSDTrainer
    sc = [0.04, 0.1, 0.26, 0.42, 0.58, 0.74, 0.9, 1.06]
    m = ssd_512((512, 512, 3), 20, mode='training', scales=sc, divide_by_stddev=[64.0] * 3, weights_seed=3)
    w = m.get_weights()
    rng = np.random.default_rng(3)
    for k in w:
        if k.endswith('/bias'):
            w[k] = (rng.standard_normal(w[k].shape) * 0.05).astype(np.float32)
    m.set_weights(w)
    enc = OracleEncoder(512, 512, 20, m.predictor_sizes, scales=sc, aspect_ratios_per_layer=m.anchor_cfg['aspect_ratios_per_layer'],
                        steps=[8, 16, 32, 64, 128, 256, 512], variances=[0.1, 0.1, 0.2, 0.2])
    assert np.array_equal(enc.anchors, m.anchors)
    x = synth.synth_images(9, 1, 512, 512)
    y_true = enc(synth.synth_gt(10, 1, 6, 512, 512, 20)).astype(np.float32)
    tr = SSDTrainer(m, 1, lr=1e-3, momentum=0.9, l2_regularization=5e-4)
    loss, _ = tr.forward_backward(torch.from_numpy(x).cuda(), torch.from_numpy(y_true).cuda())
    torch.cuda.synchronize()
    grads = tr.gradients()
    params = og.make_params(m.specs, w, dtype=torch.float64)
    yp, _ = og.forward(m.specs, params, x, 21, m.anchors, [0.1, 0.1, 0.2, 0.2], dtype=torch.float64)
    lvec = og.ssd_loss_torch(y_true, yp)
    lvec.mean().backward()
    ref_l = lvec.detach().numpy()
    assert np.abs(loss.cpu().numpy() - ref_l).max() <= 5e-4 * np.abs(ref_l).max()
    assert set(grads) == set(w)
    for k in sorted(grads):
        ref = params[k].grad.numpy()
        e = np.abs(grads[k] - ref).ravel() / (np.abs(ref).max() + 1e-30)
        assert np.median(e) < 2e-3 and e.max() < 2e-2, 'gradient %s: median err %.3e, max err %.3e' % (k, np.median(e), e.max())


def test_trained_weights_belong_to_the_model(tmp_path):
    """Keras' train_on_batch mutates the model: after SSDTrainer steps, predict() with another batch size, get_weights() and
    save_weights() must see the trained weights; set_weights() after building a trainer must not leave it pointing at a freed
    plan; a batch of the wrong size is refused instead of read out of bounds."""
    import torch
    from ssd_keras_b200.models.keras_ssd300 import ssd_300
    from ssd_keras_b200.training import SSDTrainer
    B = 2
    m, w, x, y_true = _ssd300(B)
    xd, ytd = torch.from_numpy(x).cuda(), torch.from_numpy(y_true).cuda()
    tr = SSDTrainer(m, B, lr=1e-3, momentum=0.9, l2_regularization=5e-4)
    y0 = m.predict(x[:1])                                   # an inference-side plan (batch 1) built from the initial weights
    l_first = tr.train_on_batch(xd, ytd).cpu().numpy()
    tr.train_on_batch(xd, ytd)
    w_tr, w_m = tr.get_weights(), m.get_weights()
    assert set(w_tr) <= set(w_m)
    for k in w_tr:
        np.testing.assert_array_equal(w_tr[k], w_m[k])
    assert any(not np.array_equal(w_m[k], w[k]) for k in w_tr if k.endswith('/kernel'))
    y1 = m.predict(x[:1])
    assert not np.allclose(y0[:, :, :25], y1[:, :, :25])    # the stale batch-1 plan was rebuilt
    sc = [0.1, 0.2, 0.37, 0.54, 0.71, 0.88, 1.05]
    m2 = ssd_300((300, 300, 3), 20, mode='training', scales=sc, divide_by_stddev=[64.0] * 3)
    m2.set_weights(w_m)
    np.testing.assert_array_equal(m2.predict(x[:1]), y1)    # same weights, same kernels -> same bits
    p = str(tmp_path / 'trained.npz')
    m.save_weights(p)
    with np.load(p) as f:
        for k in w_tr:
            np.testing.assert_array_equal(f[k], w_tr[k])
    # the sync kept the training plan (and its momentum): training goes on
    assert np.isfinite(tr.train_on_batch(xd, ytd).cpu().numpy()).all()
    # new weights under a live trainer: it re-attaches to a fresh plan; the first step equals the very first step above
    m.set_weights(w)
    np.testing.assert_allclose(tr.train_on_batch(xd, ytd).cpu().numpy(), l_first, rtol=1e-6)
    with pytest.raises(ValueError):
        tr.forward_backward(xd[:1], ytd[:1])
    with pytest.raises(ValueError):
        tr.forward_backward(xd, ytd[:, :100])


def test_ssd7_training_step_batchnorm_elu_adam():
    """SSD7 (conv + BatchNormalization + ELU stages, models/keras_ssd7.py:277-309) trained like ssd7_training.ipynb:153 does:
    BatchNormalization in its training phase (batch statistics), Adam.  Loss, every gradient incl. the BatchNormalization
    gamma / beta, the Adam update and the moving statistics against float64 autograd of the same graph."""
    import torch
    from oracle import graph as og
    from oracle import synth
    from oracle.encoder import OracleEncoder
    from ssd_keras_b200.models.keras_ssd7 import build_model
    from ssd_keras_b200.training import SSDTrainer
    B, H, W, ncls = 4, 96, 128, 5
    sc = [0.08, 0.16, 0.32, 0.64, 0.96]
    pre = dict(subtract_mean=127.5, divide_by_stddev=127.5)
    m = build_model((H, W, 3), ncls, mode='training', l2_regularization=5e-4, scales=sc, normalize_coords=True, weights_seed=4, **pre)
    w = m.get_weights()
    rng = np.random.default_rng(3)
    for k in w:
        if k.endswith('/bias'):
            w[k] = (rng.standard_normal(w[k].shape) * 0.05).astype(np.float32)
        elif k.endswith('/gamma'):
            w[k] = rng.uniform(0.8, 1.2, w[k].shape).astype(np.float32)
        elif k.endswith('/beta'):
            w[k] = (rng.standard_normal(w[k].shape) * 0.1).astype(np.float32)
    m.set_weights(w)
    enc = OracleEncoder(H, W, ncls, m.predictor_sizes, scales=sc, aspect_ratios_global=[0.5, 1.0, 2.0], variances=[1.0] * 4,
                        pos_iou_threshold=0.4, neg_iou_limit=0.3, normalize_coords=True)
    assert np.array_equal(enc.anchors, m.anchors)
    x = synth.synth_images(7, B, H, W)
    y_true = enc(synth.synth_gt(8, B, 3, W, H, ncls)).astype(np.float32)
    lr = 1e-3
    tr = SSDTrainer(m, B, lr=lr, l2_regularization=5e-4, optimizer='adam')
    xd, ytd = torch.from_numpy(x).cuda(), torch.from_numpy(y_true).cuda()
    loss, _ = tr.forward_backward(xd, ytd)
    torch.cuda.synchronize()
    grads = tr.gradients()
    params = og.make_params(m.specs, w, dtype=torch.float64)
    yp, outs = og.forward(m.specs, params, x, ncls + 1, m.anchors, [1.0] * 4, dtype=torch.float64, bn_training=True)
    lvec = og.ssd_loss_torch(y_true, yp)
    lvec.mean().backward()
    ref_l = lvec.detach().numpy()
    assert np.abs(loss.cpu().numpy() - ref_l).max() <= 1e-4 * np.abs(ref_l).max()
    trainable = [k for k in w if not k.endswith(('/moving_mean', '/moving_variance'))]
    assert set(grads) == set(trainable)
    errs = {}
    bn_convs = {s.name for s in m.specs if getattr(s, 'bn', None)}
    for k in trainable:
        ref = params[k].grad.numpy()
        if k.endswith('/bias') and k.split('/')[0] in bn_convs:
            # a bias in front of a BatchNormalization has an exactly zero gradient (the batch mean removes it): the float64
            # reference is rounding noise, ours must be small against the layer's beta gradient (same sum, not cancelled)
            scale = np.abs(params[[s.bn for s in m.specs if s.name == k.split('/')[0]][0] + '/beta'].grad.numpy()).max()
            errs[k] = float(np.abs(grads[k]).max() / scale) / 10.0 if scale > 0 else float(np.abs(grads[k]).max())
            continue
        errs[k] = float(np.abs(grads[k] - ref).max() / (np.abs(ref).max() + 1e-30))
    bad = {k: v for k, v in errs.items() if v > 2e-3}
    assert not bad, bad
    # one Adam step; moving statistics after one training-phase forward
    tr.apply(1.0)
    torch.cuda.synchronize()
    new_w = tr.get_weights()
    ref_w, _, _ = og.adam_step({k: w[k] for k in trainable}, {k: params[k].grad.numpy() for k in trainable}, {}, {}, 1, lr=lr, l2_reg=5e-4)
    for k in trainable:
        # the very first Adam step moves every weight by lr * sign(g) (m / sqrt(v) = +-1): compare the step, not just the weight
        step, ref_step = new_w[k] - w[k], ref_w[k] - w[k]
        if k.endswith('/bias') and k.split('/')[0] in bn_convs:
            continue                                            # zero gradient: the step is lr * sign(noise)
        g_ref = params[k].grad.numpy().astype(np.float64)
        if k.endswith('/kernel'):
            g_ref = g_ref + 2.0 * 5e-4 * w[k]                  # what Adam sees: loss gradient + l2 term (they can cancel)
        g_ref = np.abs(g_ref)
        # where the step is well conditioned: m / (sqrt(v) + 1e-8) amplifies the relative error of g by 1e-8 / |g|
        big = g_ref > max(1e-3 * g_ref.max(), 1e-5)
        np.testing.assert_allclose(step[big], ref_step[big], rtol=2e-3, atol=2e-6)
    for s in m.specs:
        if getattr(s, 'bn', None):
            mu, var = outs[s.bn + '/batch_mean'].numpy(), outs[s.bn + '/batch_var'].numpy()
            n = float(B * m._shapes[m.index[s.name]][0] * m._shapes[m.index[s.name]][1])
            exp_mean = 0.99 * w[s.bn + '/moving_mean'] + 0.01 * mu
            exp_var = 0.99 * w[s.bn + '/moving_variance'] + 0.01 * var * n / (n - 1.0)
            np.testing.assert_allclose(new_w[s.bn + '/moving_mean'], exp_mean, rtol=1e-4, atol=1e-5)
            np.testing.assert_allclose(new_w[s.bn + '/moving_variance'], exp_var, rtol=1e-4, atol=1e-5)
    # the model owns the result: an inference-phase predict uses the updated moving statistics and weights
    y_after = m.predict(x[:1])
    assert np.isfinite(y_after).all()
    # a few more steps: the loss goes down
    l0 = float(loss.mean().item())
    for _ in range(8):
        l = tr.train_on_batch(xd, ytd)
    assert float(l.mean().item()) < l0
