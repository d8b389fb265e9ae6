"""GPU tests of the launch regimes only full-size layers reach (tests/regime_cases.py), against the operand-exact float64
references of oracle/opexact.py, on one- and two-layer training graphs sized just past each threshold:
- the regimes are asserted from the device's own SM count, the forward kernels from the training plan and the weight-gradient
  kernel from the backward plan;
- the forward pass of the training plan, layer by layer: a conv's stored planes against conv_ref (a BatchNormalization
  conv's z against conv_ref without activation, its output against bn_fwd_ref on that z); the perturbed references -- a
  dropped cross term, the middle tap, its last 64-channel k-block, the largest bias -- must each fail; borders and padding
  channels stay zero;
- BatchNormalization over three passes with its moving statistics (biased variance, no eps, an uncleared accumulator must
  fail), the moving variance starting at 0 so that the biased-variance perturbation stays visible at 288 000 pixels;
- the backward pass, one layer at a time, through the harness of tests/test_gpu_backward_kernels.py (BatchNormalization
  backward, data gradients masked by swap-written planes, native and direct weight gradients, the head), the direct weight
  gradient with the step count of its own summation order (opexact.n_steps_wgrad_direct).
Two perturbations of the per-launch suite are logged but not asserted here: a dropped pixel row of the bias gradient and
the cross term (X_hi * dZ_lo) of a GEMM weight gradient (native, transposed).  Each drops a random-signed sum of
O(sqrt(pixels)) terms, while the bound of these sums grows with the pixels (oracle/opexact.py, sections 3 and 4): at
50 000 - 290 000 pixels they stay below it (measured ratios about 0.001 and 0.17 - 0.65).  Ratios go to SSDK_KERNEL_ERRORS_LOG
(conv_cases.log_ratio)."""
import numpy as np
import pytest

import conv_cases as cc
import regime_cases as rc
import test_gpu_backward_kernels as tb
import test_gpu_train_step_kernels as ts
from oracle import opexact

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _judge_forward(case, g, info, before):
    """Every conv layer of the forward pass just run, against the float64 reference of the planes it read.  before: {layer:
    (moving mean, moving variance)} of the BatchNormalization layers, read before the pass."""
    n = len(case['layers']) + 1
    store = 'split' if case['prec'] == 'bf16x3' else 'bf16'
    shape0 = dict(H=case['H'], W=case['W'], C=case['cin'])
    for i in range(1, n):
        inf = info[i]
        if inf['op'] != 'conv':
            continue
        pi = inf['input']
        pinf = info[pi] if pi else shape0
        plan = g.plan(i)
        taps = inf['k'] ** 2
        xin = cc.interior(g.planes(pi), pinf['H'], pinf['W'], pinf['C'])
        if plan['kernel'] == 'direct':
            mode, steps = 'fp32', opexact.n_steps_direct(taps, pinf['C'])
        else:
            mode, steps = case['prec'], opexact.n_steps_gemm(taps, plan['kblocks'])
        bn = inf['bn_gamma'] is not None
        perts = cc.perturbations(plan, taps, pinf['C'], mode == 'bf16x3', inf['b'])
        ref, A, pv = opexact.conv_ref(xin, inf['w'], inf['b'], stride=inf['stride'], dil=inf['dil'], pads=inf['pads'], mode=mode,
                                      act=None if bn else inf['act'], perturb=perts)
        bnd = opexact.bound(ref, A, steps, store)
        planes = g.planes(i)
        got = g.read_bn_input(i) if bn else tb._fval(planes, inf)
        ratio = opexact.err_ratio(got, ref, bnd)
        perturbed = {p[0]: opexact.err_ratio(got, v, bnd) for p, v in pv.items()}
        cc.log_ratio(dict(test='full_size_forward', case=case['name'], layer=i, what='z' if bn else 'y', kernel=plan['kernel'],
                          prec=case['prec'], ratio=ratio, perturbed=perturbed))
        assert ratio <= 1.0, (case['name'], i, ratio)
        assert {p[0] for p in perts} >= ({'cross'} if mode == 'bf16x3' else set()) | {'tap', 'kblock', 'bias'}
        for k, r in perturbed.items():
            assert r > 1.0, '%s layer %d: the bound does not see a dropped %s (ratio %.3g)' % (case['name'], i, k, r)
        if bn:
            r, _ = ts.bn_pass_ratios(case['name'], 0, g, info, [i], before, {}, store)
            cc.log_ratio(dict(test='full_size_forward', case=case['name'], layer=i, what='bn', prec=case['prec'], ratio=r, perturbed={}))
        for o in cc.outside(planes, inf['H'], inf['W'], inf['C']):
            assert not np.any(o), (case['name'], i, 'border / padding channels of the forward planes not zero')


def _bn_three_passes(case, g, info):
    """Three forward passes of small-spread inputs (a variance near eps, so that dropping eps shows in bf16), from moving
    statistics (0, 0)."""
    n = len(case['layers']) + 1
    bn_layers = [i for i in range(1, n) if info[i].get('bn_gamma') is not None]
    store = 'split' if case['prec'] == 'bf16x3' else 'bf16'
    rng = np.random.default_rng(21)
    z_prev = {}
    shape = (case['B'], case['H'], case['W'], case['cin'])
    for p in range(3):
        x = rng.standard_normal(shape) * (0.1, 0.06, 0.15)[p] + 0.05 * p
        if case['input_layer'] is not None:                           # the same values after (x - 127.5) / 127.5
            x = 127.5 + 127.5 * x
        before = {i: g.bn_stats(i, info[i]['C']) for i in bn_layers}
        if p == 0:
            assert all(not np.any(m) and not np.any(v) for m, v in before.values())
        g.forward(x.astype(np.float32), width=case['C'] + 12)
        ratio, pr = ts.bn_pass_ratios(case['name'], p, g, info, bn_layers, before, z_prev, store)
        ts._judge(dict(test='full_size_bn_forward', case=case['name'], pass_=p), ratio, pr)
        assert {k[0] for k in pr} == {'biased', 'no_eps'} | ({'acc'} if p else set()), pr


# logged, not asserted: see the module docstring
UNASSERTED = {'bias': ('row',), 'wgrad_native': ('cross',), 'wgrad_transposed': ('cross',)}


@pytest.mark.parametrize('case', rc.REGIME_CASES, ids=[c['name'] for c in rc.REGIME_CASES])
def test_full_size_regime_within_operand_exact_bounds(case):
    sm = _sm_count()
    reached = rc.regimes(case, sm)
    assert case['regimes'] <= reached, ('%s: with %d SMs the size rules give %s' % (case['name'], sm, sorted(reached)))
    g, info, x, P = tb._build(case, moving_var=0.0)
    try:
        for i, kernel in case['fwd'].items():
            plan = g.plan(i)
            assert plan['kernel'] == kernel, (case['name'], i, plan)
            if kernel == 'gemm_swap':
                assert plan['bm'] == 192, (case['name'], i, plan)
        plans = tb.check_backward_plans(case, g, info)
        for i, r in rc.reach(case, sm).items():
            if r['wgrad'] is not None:
                assert plans[i]['wgrad'] == 'direct' and plans[i]['direct_fast'] == int(r['wgrad'][3]), (case['name'], i, plans[i])
        bn_layers = [i for i in info if info[i].get('bn_gamma') is not None]
        if bn_layers:
            _bn_three_passes(case, g, info)
        before = {i: g.bn_stats(i, info[i]['C']) for i in bn_layers}
        tb.check_backward(case, g, info, x, P, plans, sm_count=sm, unasserted=UNASSERTED,
                          on_forward=lambda g_: _judge_forward(case, g_, info, before))
    finally:
        g.close()
