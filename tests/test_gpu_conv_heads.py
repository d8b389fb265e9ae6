"""GPU tests of the predictor heads: the conf + loc convolution of one source layer and the rows of y_pred it produces
(models/keras_ssd300.py:363-419: Reshape, softmax, Concat with the anchors and variances).

Each case is a graph of a tensor input and one head.  The plan must be the variant the case declares: the fused epilogue for
Pascal VOC's 25-column boxes (epi_head_fixed<25>) at 4, 6 and 8 boxes, the generic fused epilogue for other class counts, or
the unfused GEMM + head_finalize_kernel.  Logits and box offsets are bounded as in tests/test_gpu_ops.py (oracle/opexact.py);
probabilities through the bound on their row's logits.  Anchors and variances must match bit for bit.  The comparison is
repeated against perturbed references, which must fail."""
import numpy as np
import pytest

import conv_cases as cc
from oracle import opexact

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


HEAD_CASES = cc.HEAD_CASES


def _head_refs(x_st, kc, bc, kl, bl, mode, perturb):
    """Class logits and box offsets with their magnitudes and perturbed versions (a dropped bias is one of the class logits')."""
    geo = dict(pads=(1, 1, 1, 1), mode=mode)
    zc, Ac, pc = opexact.conv_ref(x_st, kc, bc, perturb=perturb, **geo)
    zl, Al, pl = opexact.conv_ref(x_st, kl, bl, perturb=[p for p in perturb if p[0] != 'bias'], **geo)
    return zc, Ac, zl, Al, {p: (pc[p], pl.get(p, zl)) for p in perturb}


@pytest.mark.parametrize('case', HEAD_CASES, ids=[c['name'] for c in HEAD_CASES])
def test_head_variant_within_operand_exact_bound(case, monkeypatch):
    from ssd_keras_b200 import _ffi
    for k, v in case['env'].items():
        monkeypatch.setenv(k, v)
    B, Hh, Ww, cin, nb, C = case['B'], case['H'], case['W'], case['cin'], case['nb'], case['C']
    rng = np.random.default_rng(sum(map(ord, case['name'])))
    x = rng.standard_normal((B, Hh, Ww, cin)).astype(np.float32)
    sd = np.sqrt(2.0 / (9 * cin))
    kc = (rng.standard_normal((3, 3, cin, nb * C)) * sd).astype(np.float32)
    kl = (rng.standard_normal((3, 3, cin, nb * 4)) * sd).astype(np.float32)
    bc = (rng.standard_normal(nb * C) * 0.5).astype(np.float32)
    bl = (rng.standard_normal(nb * 4) * 0.1).astype(np.float32)
    P = Hh * Ww * nb
    anchors = rng.uniform(-1, 2, (P, 4)).astype(np.float32)
    variances = (0.1, 0.1, 0.2, 0.2)
    layer = dict(op=_ffi.OP_HEAD, k=3, pads=(1, 1, 1, 1), n_boxes=nb, kernel=kc, bias=bc, kernel2=kl, bias2=bl)
    g = cc.Graph(B, Hh, Ww, cin, [layer], prec=case['prec'], n_classes=C, anchors=anchors, variances=variances)
    try:
        assert g.P == P
        plan = g.plan(1)
        cc.assert_plan(plan, case['expect'], case['name'])
        y = g.forward(x, width=C + 12)
        x_st = x                                        # the kernel reads split(x)
    finally:
        g.close()
    assert np.array_equal(y[:, :, C + 4:C + 8], np.broadcast_to(anchors, (B, P, 4)))
    assert np.array_equal(y[:, :, C + 8:], np.broadcast_to(np.float32(variances), (B, P, 4)))
    n_steps = cc.n_steps_of(plan, 9, cin)
    zc, Ac, zl, Al, pert = _head_refs(x_st, kc, bc, kl, bl, case['prec'], cc.perturbations(plan, 9, cin, case['prec'] == 'bf16x3', bc))
    zc, Ac = zc.reshape(B, P, C), Ac.reshape(B, P, C)
    zl, Al = zl.reshape(B, P, 4), Al.reshape(B, P, 4)
    p_ref, p_bnd = opexact.softmax_ref(zc, Ac, n_steps, C)
    l_bnd = opexact.bound(zl, Al, n_steps, 'f32')

    def ratio(p, l):
        return max(opexact.err_ratio(y[:, :, :C], p, p_bnd), opexact.err_ratio(y[:, :, C:C + 4], l, l_bnd))

    r = ratio(p_ref, zl)
    perturbed = {}
    for d, (pc, pl) in pert.items():
        pp, _ = opexact.softmax_ref(pc.reshape(B, P, C), np.zeros((B, P, C)), n_steps, C)
        perturbed[d[0]] = ratio(pp, pl.reshape(B, P, 4))
    cc.log_ratio(dict(test='head', case=case['name'], kernel=plan['kernel'], bn=plan['bn'], split=plan['split'],
                      epilogue=plan['epilogue'], ratio=r, perturbed=perturbed))
    assert r <= 1.0, (case['name'], r)
    for k, v in perturbed.items():
        assert v > 1.0, '%s: the bound does not see a dropped %s (ratio %.3g)' % (case['name'], k, v)
