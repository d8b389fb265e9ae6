"""GPU tests of conv_swap_kernel (tests/swap_cases.py): every case is a one-layer graph whose plan must be the swapped-operand
variant, and whose output is held to the operand-exact float64 bound of oracle/opexact.py, as tests/test_gpu_ops.py holds the
other convolution kernels.  The perturbed references -- a dropped cross term, the middle tap, the middle tap's last 64-channel
k-block, the largest bias -- must each fail.  The zero border and padding channels of the output planes must stay zero."""
import numpy as np
import pytest

import conv_cases as cc
import swap_cases as sc
from oracle import opexact

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


@pytest.mark.parametrize('case', sc.SWAP_CASES, ids=[c['name'] for c in sc.SWAP_CASES])
def test_swapped_conv_within_operand_exact_bound(case, monkeypatch):
    for k, v in case['env'].items():
        monkeypatch.setenv(k, v)
    x, w, b, scale, shift = cc.case_data(case, seed=sum(map(ord, case['name'])))
    layer = dict(cout=case['cout'], k=case['k'], stride=case['stride'], dil=case['dil'], pads=case['pads'], act=case['act'],
                 kernel=w, bias=b, bn_scale=scale, bn_shift=shift)
    g = cc.Graph(case['B'], case['H'], case['W'], case['cin'], [layer], prec=case['prec'])
    try:
        plan = g.plan(1)
        cc.assert_plan(plan, case['expect'], case['name'])
        g.forward(x)
        y = g.read(1)
        planes = g.planes(1)
    finally:
        g.close()
    for p in cc.outside(planes, case['H'], case['W'], case['cout']):
        assert not p.any(), '%s: the output border or padding channels were written' % case['name']
    geo = dict(stride=case['stride'], dil=case['dil'], pads=case['pads'], mode=case['prec'], act=case['act'], bn_scale=scale,
               bn_shift=shift)
    taps = case['k'] * case['k']
    y_ref, A, pert = opexact.conv_ref(x, w, b, perturb=cc.perturbations(plan, taps, case['cin'], case['prec'] == 'bf16x3', b), **geo)
    bnd = opexact.bound(y_ref, A, opexact.n_steps_gemm(taps, plan['kblocks']), 'bf16' if case['prec'] == 'bf16' else 'split')
    ratio = opexact.err_ratio(y, y_ref, bnd)
    perturbed = {p[0]: opexact.err_ratio(y, yp, bnd) for p, yp in pert.items()}
    cc.log_ratio(dict(test='forward', case=case['name'], kernel=plan['kernel'], bn=plan['bn'], split=plan['split'],
                      ratio=ratio, perturbed=perturbed))
    assert ratio <= 1.0, (case['name'], ratio)
    assert {p[0] for p in pert} >= ({'cross'} if case['prec'] == 'bf16x3' else set()) | {'tap', 'kblock'}
    for k, r in perturbed.items():
        assert r > 1.0, '%s: the bound does not see a dropped %s (ratio %.3g)' % (case['name'], k, r)
