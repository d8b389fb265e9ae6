"""GPU tests of the focal loss kernels (focal_count_kernel, focal_loss_kernel in csrc/focal_loss.cu) against the float64 reference
and bound of tests/focal_reference.py, call by call:
- every case runs ssdk_focal_loss with the loss (fwd), the gradient (bwd) and both (fwd_bwd); the loss of fwd and fwd_bwd, and
  the gradient of bwd and fwd_bwd, are the same bits; both are held to the bound, and every listed perturbation of the reference
  (gamma dropped, the two weights swapped, N per image, one box left out, the clamp's gradient ignored) must exceed it;
- the cases cover the benchmark shapes, a large class count, P around the 128-row tile, odd widths and 4-byte offsets (the plain
  loads, which give the float4 path's bits), upstream with zero and negative entries, the clamp's edges and q = 1, no positives;
- two calls are bit-identical, and 1, 2 and 4 emulated ranks through ssdk_focal_loss_phase give the single launch's bits;
- refused parameters raise ValueError before any launch;
- training: the dy the trainer hands to the backward pass is the loss kernel's gradient, for SSDLoss and the focal loss in both
  loss modes, an SSD7 fit_generator run lowers the loss, and save -> load_model -> fit_generator(initial_epoch=...) resumes.
Ratios go to SSDK_KERNEL_ERRORS_LOG (conv_cases.log_ratio).
"""
import itertools

import numpy as np
import pytest

import conv_cases as cc
import focal_reference as fr
from test_focal_loss_cpu import make_batch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


ALL = ('fwd', 'bwd', 'fwd_bwd')
BASE_PERTURB = ('no_gamma', 'swap_alpha', 'per_image_n', 'drop_box')


def case(name, B, P, C, seed, gamma=2.0, focal_alpha=0.25, alpha=1.0, upstream=None, offset=False, grad_offset=False,
         perturb=BASE_PERTURB, **gen):
    return dict(name=name, B=B, P=P, C=C, seed=seed, gamma=gamma, focal_alpha=focal_alpha, alpha=alpha, upstream=upstream,
                offset=offset, grad_offset=grad_offset, perturb=perturb, gen=gen)


CASES = [
    case('ssd300_b32_c21', 32, 8732, 21, 1, pos=0.02, neutral=0.05, edge=False),
    case('ssd512_b16_c81', 16, 24564, 81, 2, pos=0.01, neutral=0.05, edge=False, perturb=('no_gamma', 'swap_alpha', 'drop_box')),
    case('large_c_1001', 2, 300, 1001, 3, pos=0.1, gamma=1.0, focal_alpha=0.6, alpha=0.5),
    case('p1', 1, 1, 4, 4, pos=1.0, neutral=0.0, perturb=('no_gamma', 'swap_alpha', 'drop_box')),
    case('p127', 3, 127, 4, 5),
    case('p128', 3, 128, 4, 6),
    case('p129', 3, 129, 4, 7),
    case('odd_width_c5', 3, 301, 5, 8),
    case('offset4_inputs', 2, 256, 20, 9, offset=True),
    case('offset4_grad', 2, 384, 20, 10, grad_offset=True),
    case('upstream_zero_negative', 4, 300, 6, 11, upstream=(0.5, 0.0, -1.25, 2.0), alpha=0.25),
    case('edges_gamma0.5', 3, 400, 6, 12, gamma=0.5, pos=0.3, perturb=BASE_PERTURB + ('no_clamp_grad',)),
    case('edges_gamma0', 3, 400, 6, 13, gamma=0.0, focal_alpha=0.4, pos=0.3,
         perturb=('swap_alpha', 'per_image_n', 'drop_box', 'no_clamp_grad')),
    case('edges_gamma2.5', 3, 400, 7, 14, gamma=2.5, pos=0.3, perturb=BASE_PERTURB + ('no_clamp_grad',)),
    case('no_positives', 2, 300, 6, 15, pos=0.0, perturb=('no_gamma', 'swap_alpha', 'drop_box')),
]


def make_case(c):
    g = dict(c['gen'])
    yt, yp = make_batch(c['seed'], c['B'], c['P'], c['C'], pos=g.get('pos', 0.2), neutral=g.get('neutral', 0.1),
                        edge=g.get('edge', True))
    up = None if c['upstream'] is None else np.asarray(c['upstream'], np.float32)
    return yt, yp, up


def _dev(a, offset=False):
    """A device copy of a, at a 4-byte offset from a 16-byte aligned allocation if asked."""
    import torch
    a = np.ascontiguousarray(a, np.float32)
    buf = torch.zeros(a.size + 4, dtype=torch.float32, device='cuda')
    v = buf[int(offset): int(offset) + a.size]
    v.copy_(torch.from_numpy(a.reshape(-1)))
    return v.view(a.shape)


def _cfg(c):
    return float(c['gamma']), float(c['focal_alpha']), float(c['alpha'])


def run_focal(mode, yt_d, yp_d, cfg, up_d=None, grad_offset=False):
    """One ssdk_focal_loss call -> (loss, grad) as NumPy (None where the mode writes nothing)."""
    import torch
    from ssd_keras_b200 import _ffi
    B, P, W = yp_d.shape
    loss = torch.full((B,), np.nan, dtype=torch.float32, device='cuda') if mode != 'bwd' else None
    grad = _dev(np.full(yp_d.shape, np.nan, np.float32), grad_offset) if mode != 'fwd' else None
    up = up_d if mode != 'fwd' else None
    d = _ffi.dptr
    _ffi.check(_ffi.lib().ssdk_focal_loss(_ffi.context(), d(yt_d), d(yp_d), B, P, W - 12, *cfg, d(up), d(loss), d(grad),
                                          _ffi.stream_ptr()))
    torch.cuda.synchronize()
    return (None if loss is None else loss.cpu().numpy()), (None if grad is None else grad.cpu().numpy())


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def judge(name, yt, yp, cfg, up, outs, perturb, global_B=None, log=True):
    """outs: {mode: (loss, grad)}.  Holds them to the reference and requires every perturbation to fail -> the ratios."""
    loss = outs.get('fwd_bwd', outs.get('fwd', (None, None)))[0]
    grad = outs.get('fwd_bwd', outs.get('bwd', (None, None)))[1]
    if 'fwd' in outs and 'fwd_bwd' in outs:
        assert np.array_equal(_bits(outs['fwd'][0]), _bits(outs['fwd_bwd'][0])), name
    if 'bwd' in outs and 'fwd_bwd' in outs:
        assert np.array_equal(_bits(outs['bwd'][1]), _bits(outs['fwd_bwd'][1])), name
    kw = dict(upstream=up, global_B=global_B)
    ref = fr.focal_parts(yt, yp, *cfg, **kw)
    bnd = fr.focal_bound(yt, yp, *cfg, **kw)
    r = {'loss': fr.ratio(loss, ref['loss'], bnd['loss']) if loss is not None else 0.0,
         'grad': fr.ratio(grad, ref['grad'], bnd['grad']) if grad is not None else 0.0}
    assert max(r.values()) <= 1.0, (name, r)
    pert = {}
    for p in perturb:
        rp = fr.focal_parts(yt, yp, *cfg, perturb=p, **kw)
        pert[p] = max(fr.ratio(loss, rp['loss'], bnd['loss']) if loss is not None else 0.0,
                      fr.ratio(grad, rp['grad'], bnd['grad']) if grad is not None else 0.0)
        assert pert[p] > 1.0, (name, p, pert[p])
    if log:
        cc.log_ratio({'kernel': 'focal_loss', 'case': name, **r, 'perturbed': {p: min(v, 1e300) for p, v in pert.items()}})
    print('%s: loss %.3g, grad %.3g of the bound; perturbed %s' % (name, r['loss'], r['grad'],
                                                                   {p: float('%.3g' % min(v, 1e300)) for p, v in pert.items()}))
    return r


@pytest.mark.parametrize('c', CASES, ids=[c['name'] for c in CASES])
def test_focal_loss_case(c):
    yt, yp, up = make_case(c)
    yt_d, yp_d = _dev(yt, c['offset']), _dev(yp, c['offset'])
    up_d = None if up is None else _dev(up)
    cfg = _cfg(c)
    outs = {m: run_focal(m, yt_d, yp_d, cfg, up_d, c['grad_offset']) for m in ALL}
    judge(c['name'], yt, yp, cfg, up, outs, c['perturb'])
    again = run_focal('fwd_bwd', yt_d, yp_d, cfg, up_d, c['grad_offset'])
    assert np.array_equal(_bits(again[0]), _bits(outs['fwd_bwd'][0])) and np.array_equal(_bits(again[1]), _bits(outs['fwd_bwd'][1]))
    if c['offset'] or c['grad_offset']:                  # the plain loads and stores give the float4 path's bits
        aligned = run_focal('fwd_bwd', _dev(yt), _dev(yp), cfg, up_d)
        assert np.array_equal(_bits(aligned[0]), _bits(outs['fwd_bwd'][0])) and np.array_equal(_bits(aligned[1]), _bits(outs['fwd_bwd'][1]))


def _phase_run(yt, yp, cfg, shards):
    """The phase-wise loss of `shards` emulated ranks on one GPU (the count's all-reduce replaced by a sum) -> (loss, grad)."""
    import torch
    from ssd_keras_b200 import _ffi
    B, P, W = yt.shape
    per = B // shards
    d, lib, ctx = _ffi.dptr, _ffi.lib(), _ffi.context()
    shard = [(torch.from_numpy(yt[r * per:(r + 1) * per]).cuda(), torch.from_numpy(yp[r * per:(r + 1) * per]).cuda())
             for r in range(shards)]
    counts = [torch.zeros((1,), dtype=torch.int64, device='cuda') for _ in range(shards)]
    for (t, p), cnt in zip(shard, counts):
        _ffi.check(lib.ssdk_focal_loss_phase(ctx, 0, d(t), d(p), per, P, W - 12, *cfg, d(cnt), B, None, None, None, _ffi.stream_ptr()))
    total = sum(c.clone() for c in counts)
    fixed = np.rint(yt[..., 1:W - 12].max(-1).astype(np.float64) * 2.0 ** 32).astype(np.int64).sum()
    assert int(total.item()) == int(fixed)
    losses, grads = [], []
    for (t, p), cnt in zip(shard, counts):
        cnt.copy_(total)
        loss = torch.empty((per,), dtype=torch.float32, device='cuda')
        grad = torch.empty_like(p)
        _ffi.check(lib.ssdk_focal_loss_phase(ctx, 1, d(t), d(p), per, P, W - 12, *cfg, d(cnt), B, None, d(loss), d(grad),
                                             _ffi.stream_ptr()))
        losses.append(loss.cpu().numpy()); grads.append(grad.cpu().numpy())
    return np.concatenate(losses), np.concatenate(grads)


PHASE_CASES = [case('phase_ssd300_c21', 8, 2000, 21, 20, pos=0.05), case('phase_soft_edges', 4, 500, 6, 21, gamma=0.5, pos=0.3)]


@pytest.mark.parametrize('shards', [1, 2, 4])
@pytest.mark.parametrize('c', PHASE_CASES, ids=[c['name'] for c in PHASE_CASES])
def test_phases_match_the_single_launch_bit_for_bit(c, shards):
    yt, yp, _ = make_case(c)
    cfg = _cfg(c)
    fused = run_focal('fwd_bwd', _dev(yt), _dev(yp), cfg)
    judge(c['name'], yt, yp, cfg, None, {'fwd_bwd': fused}, BASE_PERTURB, log=shards == 1)
    loss, grad = _phase_run(yt, yp, cfg, shards)
    assert np.array_equal(_bits(loss), _bits(fused[0])) and np.array_equal(_bits(grad), _bits(fused[1])), (c['name'], shards)
    if shards > 1:                                         # a rank's own count in the normalisation must fail
        per = c['B'] // shards
        bnd = fr.focal_bound(yt, yp, *cfg)
        local = np.concatenate([fr.focal_parts(yt[r * per:(r + 1) * per], yp[r * per:(r + 1) * per], *cfg, global_B=c['B'])['loss']
                                for r in range(shards)])
        assert fr.ratio(loss, local, bnd['loss']) > 1.0


def test_refused_calls_launch_nothing():
    import torch
    from ssd_keras_b200 import _ffi
    yt, yp = _dev(np.zeros((2, 10, 18), np.float32)), _dev(np.full((2, 10, 18), 0.5, np.float32))
    out = torch.empty((2,), dtype=torch.float32, device='cuda')
    cnt = torch.zeros((1,), dtype=torch.int64, device='cuda')
    d, lib, ctx, st = _ffi.dptr, _ffi.lib(), _ffi.context(), _ffi.stream_ptr()
    bad = [dict(gamma=-0.5), dict(gamma=float('nan')), dict(focal_alpha=-0.1), dict(focal_alpha=1.5), dict(focal_alpha=float('nan'))]
    for kw in bad:
        a = dict(gamma=2.0, focal_alpha=0.25)
        a.update(kw)
        n0 = _ffi.launch_count()
        with pytest.raises(ValueError):
            _ffi.check(lib.ssdk_focal_loss(ctx, d(yt), d(yp), 2, 10, 6, a['gamma'], a['focal_alpha'], 1.0, None, d(out), None, st))
        with pytest.raises(ValueError):
            _ffi.check(lib.ssdk_focal_loss_phase(ctx, 0, d(yt), d(yp), 2, 10, 6, a['gamma'], a['focal_alpha'], 1.0, d(cnt), 2, None,
                                                 None, None, st))
        assert _ffi.launch_count() == n0, kw
    n0 = _ffi.launch_count()
    with pytest.raises(ValueError, match='both NULL'):
        _ffi.check(lib.ssdk_focal_loss(ctx, d(yt), d(yp), 2, 10, 6, 2.0, 0.25, 1.0, None, None, None, st))
    with pytest.raises(ValueError, match='phase'):
        _ffi.check(lib.ssdk_focal_loss_phase(ctx, 2, d(yt), d(yp), 2, 10, 6, 2.0, 0.25, 1.0, d(cnt), 2, None, d(out), None, st))
    with pytest.raises(ValueError, match='global_B'):
        _ffi.check(lib.ssdk_focal_loss_phase(ctx, 1, d(yt), d(yp), 2, 10, 6, 2.0, 0.25, 1.0, d(cnt), 1, None, d(out), None, st))
    with pytest.raises(ValueError, match='shape'):
        _ffi.check(lib.ssdk_focal_loss(ctx, d(yt), d(yp), 2, 10, 1, 2.0, 0.25, 1.0, None, d(out), None, st))
    assert _ffi.launch_count() == n0
    torch.cuda.synchronize()


def test_compute_loss_autograd_is_the_kernel():
    """SSDFocalLoss.compute_loss: the forward is ssdk_focal_loss's loss, backward(upstream) its gradient for that upstream."""
    import torch
    from ssd_keras_b200.keras_loss_function.keras_ssd_focal_loss import SSDFocalLoss
    yt, yp, _ = make_case(case('autograd', 3, 500, 9, 30, pos=0.1))
    f = SSDFocalLoss(gamma=1.5, focal_alpha=0.4, alpha=0.8)
    cfg = (f.gamma, f.focal_alpha, f.alpha)
    ytd, ypd = _dev(yt), _dev(yp).clone().requires_grad_(True)
    loss = f.compute_loss(ytd, ypd)
    up = torch.tensor([0.25, -1.0, 0.0], device='cuda')
    (loss * up).sum().backward()
    want_loss, want_grad = run_focal('fwd_bwd', _dev(yt), _dev(yp), cfg, _dev(up.cpu().numpy()))
    assert np.array_equal(_bits(loss.detach().cpu().numpy()), _bits(want_loss))
    assert np.array_equal(_bits(ypd.grad.cpu().numpy()), _bits(want_grad))


# ------------------------------------------------------------------------------------------------------------------------------
# training
# ------------------------------------------------------------------------------------------------------------------------------
SC7 = [0.08, 0.16, 0.32, 0.64, 0.96]


def _ssd7():
    from ssd_keras_b200.models.keras_ssd7 import build_model
    return build_model((96, 96, 3), 5, mode='training', l2_regularization=5e-4, scales=SC7, normalize_coords=True, weights_seed=2,
                       subtract_mean=[127.5] * 3, divide_by_stddev=[127.5] * 3)


def _batches(m, B, n, seed):
    from oracle import synth
    from oracle.encoder import OracleEncoder
    H, W, ncls = m.img_height, m.img_width, m.n_classes - 1
    enc = OracleEncoder(H, W, ncls, m.predictor_sizes, scales=SC7, aspect_ratios_global=[0.5, 1.0, 2.0], variances=[1.0] * 4,
                        pos_iou_threshold=0.4, neg_iou_limit=0.3, normalize_coords=True)
    return [(synth.synth_images(seed + i, B, H, W), enc(synth.synth_gt(seed + 50 + i, B, 4, W, H, ncls)).astype(np.float32))
            for i in range(n)]


def _single_launch(lossobj, yt_d, yp_d):
    """The loss's own ssdk_ssd_loss / ssdk_focal_loss call with the loss, a gradient output and no upstream -> (loss, grad)."""
    import torch
    from ssd_keras_b200 import _ffi
    from ssd_keras_b200.keras_loss_function.keras_ssd_focal_loss import SSDFocalLoss
    if isinstance(lossobj, SSDFocalLoss):
        return run_focal('fwd_bwd', yt_d, yp_d, (lossobj.gamma, lossobj.focal_alpha, lossobj.alpha))
    B, P, W = yp_d.shape
    loss = torch.full((B,), np.nan, dtype=torch.float32, device='cuda')
    grad = torch.full_like(yp_d, np.nan)
    d = _ffi.dptr
    _ffi.check(_ffi.lib().ssdk_ssd_loss(_ffi.context(), d(yt_d), d(yp_d), B, P, W - 12, lossobj.neg_pos_ratio, lossobj.n_neg_min,
                                        lossobj.alpha, None, d(loss), None, d(grad), _ffi.stream_ptr()))
    torch.cuda.synchronize()
    return loss.cpu().numpy(), grad.cpu().numpy()


@pytest.mark.parametrize('loss_mode', ['replica', 'global'])
@pytest.mark.parametrize('loss_name', ['ssd', 'focal'])
def test_trainer_hands_the_kernel_gradient_to_the_backward_pass(loss_name, loss_mode):
    """Either loss writes d loss / d y_pred into the trainer's buffer: the bits of its own single launch, which the backward pass
    then reads.  A NULL d loss / d y_pred is refused before the gradient buffer is touched."""
    import torch
    from ssd_keras_b200 import _ffi
    from ssd_keras_b200.keras_loss_function.keras_ssd_focal_loss import SSDFocalLoss
    from ssd_keras_b200.keras_loss_function.keras_ssd_loss import SSDLoss
    from ssd_keras_b200.training import SSDTrainer
    m = _ssd7()
    lossobj = SSDLoss(neg_pos_ratio=3, n_neg_min=0, alpha=1.0) if loss_name == 'ssd' else SSDFocalLoss(gamma=2.0, focal_alpha=0.25)
    tr = SSDTrainer(m, 2, lr=1e-3, loss=lossobj, loss_mode=loss_mode, optimizer='adam')
    x, y = _batches(m, 2, 1, seed=4)[0]
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    loss, y_pred, dy = tr._loss_and_dy(xd, yd)
    assert dy is tr._dy
    y_pred = y_pred.clone()
    want_loss, want_grad = _single_launch(lossobj, yd, y_pred)
    assert np.array_equal(_bits(loss.cpu().numpy()), _bits(want_loss)) and np.array_equal(_bits(dy.cpu().numpy()), _bits(want_grad))
    tr._backward_layers(dy, len(m.specs) - 1, 0)
    g = tr.grad.cpu().numpy()
    assert np.all(np.isfinite(g)) and np.any(g != 0)
    with pytest.raises(ValueError, match='NULL'):
        _ffi.check(_ffi.lib().ssdk_train_backward_layers(tr.handle, None, len(m.specs) - 1, 0, _ffi.stream_ptr()))
    assert np.array_equal(_bits(tr.grad.cpu().numpy()), _bits(g))


def test_fit_generator_with_focal_loss_trains_and_resumes(tmp_path):
    from ssd_keras_b200.callbacks import ModelCheckpoint
    from ssd_keras_b200.keras_loss_function.keras_ssd_focal_loss import SSDFocalLoss
    from ssd_keras_b200.models import load_model
    from ssd_keras_b200.optimizers import Adam
    m = _ssd7()
    data = _batches(m, 4, 2, seed=3)
    focal = SSDFocalLoss(gamma=2.0, focal_alpha=0.25, alpha=1.0)
    m.compile(optimizer=Adam(lr=1e-3, beta_1=0.9, beta_2=0.999, epsilon=1e-08, decay=0.0), loss=focal.compute_loss)
    assert np.isfinite(m.test_on_batch(*data[0])) and np.isfinite(m.evaluate_generator(itertools.cycle(data), 2))
    ckpt = ModelCheckpoint(str(tmp_path / 'epoch-{epoch:02d}.h5'), monitor='loss', save_best_only=False, save_weights_only=False)
    h = m.fit_generator(itertools.cycle(data), steps_per_epoch=2, epochs=6, callbacks=[ckpt])
    print('focal fit_generator: loss per epoch %s' % ['%.5g' % v for v in h.history['loss']])
    assert all(np.isfinite(h.history['loss'])) and h.history['loss'][-1] < h.history['loss'][0]
    t0 = m._fit_trainer
    st0 = t0.get_optimizer_state()
    m2 = load_model(str(tmp_path / 'epoch-06.h5'))
    lossobj = m2._compiled[1]
    assert isinstance(lossobj, SSDFocalLoss) and lossobj.config() == focal.config()
    t2 = m2._trainer_for(4)
    assert t2.loss is lossobj and t2.iterations == st0['iterations'] == 12
    h2 = m2.fit_generator(itertools.cycle(data), steps_per_epoch=2, epochs=7, initial_epoch=6)
    assert h2.epoch == [6] and np.isfinite(h2.history['loss'][0]) and t2.iterations == 14
