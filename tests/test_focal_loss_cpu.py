"""The focal loss without a device: the float64 reference of tests/focal_reference.py against an independent torch float64
autograd of the loss expression (and the analytic limit where autograd has none), its gamma = 0 cross-check against SSDLoss's
per-box log-loss, the parameter refusals, and the ``compile`` / ``training_config`` / ``load_model`` round trip of
``SSDFocalLoss`` next to files written with ``SSDLoss``."""
import json

import numpy as np
import pytest

import focal_reference as fr
from ssd_keras_b200 import optimizers
from ssd_keras_b200.keras_loss_function.keras_ssd_focal_loss import SSDFocalLoss
from ssd_keras_b200.keras_loss_function.keras_ssd_loss import SSDLoss
from ssd_keras_b200.misc_utils.hdf5_lite import read_attributes
from ssd_keras_b200.models import load_model
from ssd_keras_b200.models.keras_ssd7 import build_model

EDGE_Q = (0.0, 1e-16, float(np.float32(1e-15)), 1.0)


def make_batch(seed, B, P, C, pos=0.2, neutral=0.1, soft=0.3, edge=True):
    """(y_true, y_pred) float32: background rows, one-hot and soft positives (fractional class values, a second non-zero class
    entry on some), neutral all-zero rows; y_pred rows are softmax outputs and offsets around y_true, and with ``edge`` the
    class entries of some non-zero y_true values are set to 0, 1e-16, 1e-15 and 1."""
    rng = np.random.default_rng(seed)
    W = C + 12
    kind = rng.choice(3, size=(B, P), p=[1 - pos - neutral, pos, neutral])
    yt = np.zeros((B, P, W), np.float32)
    yt[..., 0] = kind == 0
    bi, pi = np.nonzero(kind == 1)
    ci = rng.integers(1, C, bi.size)
    s = rng.random(bi.size) < soft
    yt[bi, pi, ci] = np.where(s, rng.uniform(0.3, 0.95, bi.size), 1.0)
    yt[bi[s], pi[s], 0] = rng.uniform(0.0, 0.3, int(s.sum()))
    yt[..., C:C + 4] = rng.normal(0, 1, (B, P, 4))
    yt[..., C + 4:] = rng.uniform(0.05, 1, (B, P, 8))
    z = rng.normal(0, 2, (B, P, C))
    e = np.exp(z - z.max(-1, keepdims=True))
    yp = np.zeros_like(yt)
    yp[..., :C] = e / e.sum(-1, keepdims=True)
    yp[..., C:C + 4] = yt[..., C:C + 4] + rng.normal(0, 1.0, (B, P, 4))
    yp[..., C + 4:] = rng.uniform(0.05, 1, (B, P, 8))
    if edge:
        nb, npp, nc = np.nonzero(yt[..., :C])
        pick = rng.random(nb.size) < 0.2
        yp[nb[pick], npp[pick], nc[pick]] = rng.choice(EDGE_Q, int(pick.sum()))
    return yt, yp.astype(np.float32)


def torch_autograd(yt, yp, gamma, focal_alpha, alpha, upstream):
    """The loss written directly in torch float64 and differentiated by autograd -> (loss (B,), grad)."""
    import torch
    t = torch.from_numpy(yt.astype(np.float64))
    q = torch.from_numpy(yp.astype(np.float64)).requires_grad_(True)
    B, P, W = t.shape
    C = W - 12
    fa = float(np.float32(focal_alpha))
    w = torch.full((C,), fa, dtype=torch.float64)
    w[0] = 1 - fa
    qc = q[..., :C]
    cls = (t[..., :C] * w * (1 - qc) ** float(np.float32(gamma)) * -torch.log(torch.clamp(qc, min=fr.EPS))).sum(-1)
    pos = t[..., 1:C].max(-1).values
    d = t[..., C:C + 4] - q[..., C:C + 4]
    loc = torch.where(d.abs() < 1, 0.5 * d * d, d.abs() - 0.5).sum(-1)
    N = float(pos.sum())
    loss = B * (cls.sum(-1) + float(np.float32(alpha)) * (loc * pos).sum(-1)) / max(1.0, N)
    (loss * torch.from_numpy(upstream.astype(np.float64))).sum().backward()
    return loss.detach().numpy(), q.grad.numpy()


@pytest.mark.parametrize('gamma', [0.0, 0.5, 2.0, 2.5])
@pytest.mark.parametrize('positives', ['some', 'none'])
def test_reference_matches_torch_autograd(gamma, positives):
    B, P, C = 3, 50, 6
    yt, yp = make_batch(int(gamma * 10) + 3, B, P, C, pos=0.3 if positives == 'some' else 0.0)
    fa, alpha = 0.3, 0.75
    up = np.array([0.5, 0.0, -1.25], np.float32)
    ref = fr.focal_parts(yt, yp, gamma, fa, alpha, upstream=up)
    assert (ref['n_pos'] == 0) == (positives == 'none')
    loss, grad = torch_autograd(yt, yp, gamma, fa, alpha, up)
    np.testing.assert_allclose(ref['loss'], loss, rtol=1e-12, atol=0)
    q = yp.astype(np.float64)
    t = yt[..., :C]
    at_one = np.zeros(yp.shape, bool)
    at_one[..., :C] = (q[..., :C] == 1.0) & (t != 0)
    assert at_one.any() and (q[..., :C][t != 0] == 0).any() and (q[..., :C][t != 0] == np.float32(1e-16)).any()
    assert (q[..., :C][t != 0] == fr.EPS).any()
    ok = ~at_one
    np.testing.assert_allclose(ref['grad'][ok], grad[ok], rtol=1e-12, atol=1e-300)
    # q = 1: autograd meets 0 * inf for gamma < 1; the reference takes the limit, -s w t [gamma == 0] (no log term, and the
    # (1 - q)^gamma / q term is 0 for gamma > 0)
    if gamma < 1 and gamma > 0:
        assert np.isnan(grad[at_one]).all()
    b, p, c = np.nonzero(at_one)
    s = up[b].astype(np.float64) * B / max(1.0, ref['n_pos'])
    w = np.where(c == 0, 1 - float(np.float32(fa)), float(np.float32(fa)))
    limit = -s * w * t[b, p, c] * (1.0 if gamma == 0 else 0.0)
    assert np.array_equal(ref['grad'][at_one], limit)
    assert np.all(ref['grad'][..., C + 4:] == 0)


def test_gamma0_is_half_the_log_loss_of_ssd_loss():
    from oracle.loss import _per_box_losses
    yt, yp = make_batch(11, 4, 200, 21, edge=False)
    cls = fr.focal_parts(yt, yp, gamma=0.0, focal_alpha=0.5)['cls']
    _, _, ssd_cls, _ = _per_box_losses(yt, yp)
    np.testing.assert_allclose(cls, 0.5 * ssd_cls.astype(np.float64), rtol=2e-6, atol=1e-12)


def test_neutral_rows_carry_nothing_and_n_is_the_soft_positive_sum():
    yt, yp = make_batch(12, 2, 80, 5, neutral=0.3)
    ref = fr.focal_parts(yt, yp, 2.0, 0.25, 1.0)
    neutral = ~yt[..., :5].any(-1)
    assert neutral.any() and np.all(ref['cls'][neutral] == 0) and np.all(ref['grad'][neutral][:, :5] == 0)
    assert ref['n_pos'] == float(yt[..., 1:5].max(-1).astype(np.float64).sum()) and ref['n_pos'] != int(ref['n_pos'])


@pytest.mark.parametrize('kw', [dict(gamma=-0.5), dict(gamma=float('nan')), dict(gamma=float('inf')), dict(focal_alpha=-0.01),
                                dict(focal_alpha=1.01), dict(focal_alpha=float('nan'))])
def test_refused_parameters(kw):
    with pytest.raises(ValueError):
        SSDFocalLoss(**kw)


def test_accepted_parameter_edges():
    for kw in (dict(gamma=0), dict(focal_alpha=0.0), dict(focal_alpha=1.0), dict(gamma=np.float32(2.0), focal_alpha=np.float64(0.5))):
        f = SSDFocalLoss(**kw)
        assert all(isinstance(v, float) for v in f.config().values())


def _model():
    return build_model((96, 96, 3), 5, mode='training', scales=[0.08, 0.16, 0.32, 0.64, 0.96], weights_seed=3)


def _training_config(path):
    return json.loads(bytes(read_attributes(path)['training_config']).rstrip(b'\x00').decode())


def test_compile_save_and_load_model_round_trip(tmp_path):
    focal = SSDFocalLoss(gamma=1.5, focal_alpha=0.3, alpha=0.5)
    m = _model()
    with pytest.raises(ValueError):
        m.compile(optimizer=optimizers.Adam(lr=1e-3), loss=lambda yt, yp: yp)
    m.compile(optimizer=optimizers.Adam(lr=1e-3), loss=focal)                 # the object itself
    assert m._compiled[1] is focal
    m.compile(optimizer=optimizers.Adam(lr=1e-3), loss=focal.compute_loss)    # or its bound compute_loss, as the notebooks do
    assert m._compiled == ('adam', focal)
    p = str(tmp_path / 'focal.h5')
    m.save(p)
    tc = _training_config(p)
    assert tc['ssd_focal_loss'] == {'gamma': 1.5, 'focal_alpha': 0.3, 'alpha': 0.5} and 'ssd_loss' not in tc
    assert tc['loss'] == 'compute_loss'
    m2 = load_model(p)
    lossobj = m2._compiled[1]
    assert isinstance(lossobj, SSDFocalLoss) and lossobj.config() == focal.config() and m2._compiled[0] == 'adam'
    mine = SSDFocalLoss(gamma=3.0)                                              # the owner of custom_objects' compute_loss wins
    assert load_model(p, custom_objects={'compute_loss': mine.compute_loss})._compiled[1] is mine
    ssd = SSDLoss(neg_pos_ratio=2)
    assert load_model(p, custom_objects={'compute_loss': ssd.compute_loss})._compiled[1] is ssd
    assert isinstance(load_model(p, custom_objects={'compute_loss': None})._compiled[1], SSDFocalLoss)
    assert load_model(p, compile=False)._compiled is None


def test_files_written_with_ssd_loss_load_as_before(tmp_path):
    m = _model()
    m.compile(optimizer=optimizers.SGD(lr=1e-3, momentum=0.9), loss=SSDLoss(neg_pos_ratio=2, n_neg_min=5, alpha=0.5).compute_loss)
    p = str(tmp_path / 'ssd.h5')
    m.save(p)
    tc = _training_config(p)
    assert 'ssd_focal_loss' not in tc and tc['ssd_loss'] == {'neg_pos_ratio': 2, 'n_neg_min': 5, 'alpha': 0.5}
    assert list(tc) == ['optimizer_config', 'loss', 'metrics', 'sample_weight_mode', 'loss_weights', 'ssd_loss']
    lossobj = load_model(p)._compiled[1]
    assert type(lossobj) is SSDLoss and (lossobj.neg_pos_ratio, lossobj.n_neg_min, lossobj.alpha) == (2, 5, 0.5)
    focal = SSDFocalLoss()
    assert load_model(p, custom_objects={'compute_loss': focal.compute_loss})._compiled[1] is focal
