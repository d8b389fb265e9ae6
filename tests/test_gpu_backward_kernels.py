"""GPU tests of every backward launch, one layer at a time, against the operand-exact float64 references of oracle/opexact.py.

Each case of BACKWARD_CASES is a small graph with a tensor input.  After one forward pass the backward pass runs one layer per
call (ssdk_train_backward_layers(t, dy, i, i)), top down, from a random d loss / d y_pred that is non-zero on every column.
Around each call every gradient buffer and the flat parameter gradient are snapshotted, so each launch is judged on the
operands it actually read:
- what the layer writes (its head gradient, its weight / bias / gamma spans, its producer's gradient) is held to the bound
  of its reference, and every listed perturbation of that reference must fail the bound;
- every other gradient buffer and parameter span is bit-identical to its snapshot;
- the zero border and padding channels of every gradient plane stay zero (the next implicit GEMM reads them as padding).
Each case also asserts ssdk_trainer_layer_plan for the variants it claims.  Ratios go to SSDK_KERNEL_ERRORS_LOG (conv_cases).
"""
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


# ------------------------------------------------------------------------------------------------------------------------------
# the case table (plain data: tests/test_opexact_cpu.py checks that it reaches every backward variant)
# ------------------------------------------------------------------------------------------------------------------------------
def conv(cout, k, input=None, stride=1, dil=1, pads='same', act='relu', ints=False, bn=False):
    """bn: followed by BatchNormalization in Keras' training phase (raw gamma / beta / moving statistics, bn_train)."""
    return dict(op='conv', cout=cout, k=k, input=input, stride=stride, dil=dil, pads=pads, act=act, ints=ints, bn=bn)


def head(nb, input=None):
    return dict(op='head', nb=nb, input=input)


def pool(k, stride, pads=(0, 0, 0, 0), input=None):
    return dict(op='pool', k=k, stride=stride, pads=pads, input=input)


def l2(input=None):
    return dict(op='l2', input=input)


def bcase(name, B, H, W, cin, layers, expect, C=6, prec='bf16x3', env=None, x='normal'):
    """expect: {layer: {plan field: value}} of ssdk_trainer_layer_plan ('min_<field>': at least that value).  x: 'normal', 'int' (values in {-2..2}), or 'zero_pixel'
    (normal with pixel (0, 1, 1) all zero)."""
    return dict(name=name, B=B, H=H, W=W, cin=cin, layers=layers, expect=expect, C=C, prec=prec, env=env or {}, x=x)


def D(bn, mask, acc):
    return dict(dgrad='gemm', dgrad_bn=bn, dgrad_mask=mask, dgrad_accumulate=acc)


def S(mask, acc):
    return dict(dgrad='strided', dgrad_mask=mask, dgrad_accumulate=acc)


BACKWARD_CASES = [
    # --- data-gradient GEMM (bf16x3: BN 64 / 128 / 160), native weight gradient (BNc 64 / 128, split) ---
    bcase('dgrad_bn64_mask_acc_native', 2, 12, 12, 64, [conv(64, 3), conv(64, 3), head(2), head(3, input=1)],
          {2: dict(D(64, 1, 1), wgrad='native', wgrad_bn=64, a_boxes=1), 1: dict(wgrad='native'), 3: D(64, 1, 0)}),
    bcase('dgrad_bn128_linear_native128', 1, 10, 11, 128, [conv(128, 3, act=None), conv(136, 3), head(2)],
          {2: dict(D(128, 0, 0), wgrad='native', wgrad_bn=128, a_boxes=2, co_tiles=2), 1: dict(wgrad='native', ci_tiles=1)}),
    bcase('dgrad_bn160_head_c21', 1, 9, 10, 64, [conv(144, 3), head(4, input=1)], {2: D(160, 1, 0)}, C=21),
    bcase('dgrad_1x1_valid4x4_dil6', 1, 20, 20, 64, [conv(64, 1, pads='valid'), conv(64, 4, pads='valid'), conv(64, 3, dil=6), head(2)],
          {2: dict(D(64, 1, 0), wgrad='transposed'), 3: dict(D(64, 1, 0), wgrad='native'), 1: dict(wgrad='native')}),
    bcase('dgrad_linear_acc', 1, 10, 10, 64, [conv(64, 3, act=None), conv(64, 3), head(2), head(1, input=1)], {2: D(64, 0, 1)}),
    bcase('dgrad_asym_pads_valid3x3', 2, 11, 10, 64, [conv(64, 3, pads=(0, 0, 2, 2)), conv(64, 3, pads='valid'), head(2)],
          {2: dict(D(64, 1, 0), wgrad='native'), 1: dict(wgrad='native')}),
    bcase('native_bw64_ksplit', 2, 8, 64, 64, [conv(64, 3), conv(64, 3), head(1)],
          {2: dict(wgrad='native', bw=64, min_k_split=2), 1: dict(bw=64)}),
    bcase('native_bw32', 2, 24, 30, 64, [conv(64, 3), conv(64, 3), head(1)], {2: dict(wgrad='native', bw=32)}),
    bcase('native_bw16_ci_tiles', 1, 16, 14, 64, [conv(256, 3), conv(64, 3), head(1)],
          {2: dict(wgrad='native', bw=16, wgrad_bn=128, ci_tiles=2)}),
    # a native weight gradient whose dW span starts at an odd float offset: behind a head of 3 x (21 + 4) biases
    bcase('native_unaligned_dw_span', 1, 10, 10, 64, [head(3), conv(64, 3, input=0), head(2)], {2: dict(wgrad='native', k_split=1)},
          C=21),
    # --- transposed / im2col weight gradients ---
    bcase('transposed_cin8_cin24', 2, 12, 12, 8, [conv(24, 3), conv(72, 3), conv(64, 3, dil=2), head(2)],
          {1: dict(wgrad='transposed', n_gemms=9), 2: dict(wgrad='transposed'), 3: dict(wgrad='transposed')}),
    bcase('transposed_env_cin16', 2, 19, 19, 16, [conv(64, 3), conv(128, 3), head(4)],
          {2: dict(wgrad='transposed', n_gemms=9, dgrad='gemm', min_k_split=2), 1: dict(wgrad='transposed')},
          env={'SSDK_WGRAD_TRANSPOSED': '1'}),
    bcase('transposed_ksplit1_tiny', 1, 3, 3, 8, [conv(16, 3), head(1)], {1: dict(wgrad='transposed', k_split=1)}),
    bcase('transposed_4x4_valid', 1, 12, 12, 64, [conv(64, 4, pads='valid'), head(2)], {1: dict(wgrad='transposed', n_gemms=16)}),
    # --- strided: GEMM to fp32 columns + col2im_kernel; im2col weight gradient ---
    bcase('strided_s2_pad1_mask_acc', 2, 13, 13, 32, [conv(32, 3), conv(64, 3, stride=2, pads=(1, 1, 1, 1)), head(2), head(2, input=1)],
          {2: dict(S(1, 1), wgrad='im2col', n_gemms=1)}),
    bcase('strided_valid_linear', 1, 12, 12, 16, [conv(16, 3, act=None), conv(32, 3, stride=2, pads='valid'), head(2)],
          {2: dict(S(0, 0), wgrad='im2col')}),
    bcase('strided_mask_noacc', 1, 11, 11, 16, [conv(16, 3), conv(32, 3, stride=2, pads=(1, 1, 1, 1)), head(2)], {2: S(1, 0)}),
    bcase('strided_linear_acc', 1, 12, 12, 16, [conv(16, 3, act=None), conv(32, 3, stride=2, pads='valid'), head(2), head(1, input=1)],
          {2: S(0, 1)}),
    bcase('im2col_cin3_cout40', 2, 14, 13, 3, [conv(40, 3), head(2)], {1: dict(wgrad='im2col')}),
    # --- image-facing direct weight gradient: 3x3 fast path, generic kernel, and > 48 KB of shared accumulators ---
    bcase('direct3x3_cin3', 2, 13, 15, 3, [conv(64, 3), head(2)], {1: dict(wgrad='direct', direct_fast=1)}),
    bcase('direct5x5_cin3', 2, 12, 12, 3, [conv(32, 5), head(2)], {1: dict(wgrad='direct', direct_fast=0)}),
    bcase('direct3x3_dil2_cin4', 1, 14, 14, 4, [conv(48, 3, dil=2), head(2)], {1: dict(wgrad='direct', direct_fast=0)}),
    bcase('direct_cin1', 1, 12, 12, 1, [conv(16, 3), head(2)], {1: dict(wgrad='direct', direct_fast=0)}),
    bcase('direct3x3_cin3_cout480_51840B', 1, 10, 10, 3, [conv(480, 3), head(2)], {1: dict(wgrad='direct', direct_fast=1)}),
    bcase('direct5x5_cin3_cout176_52800B', 1, 10, 10, 3, [conv(176, 5), head(2)], {1: dict(wgrad='direct', direct_fast=0)}),
    # --- max-pool backward: ties from exact small integers ---
    bcase('pool2x2_even_mask', 2, 12, 12, 8, [conv(16, 1, pads='valid', ints=True), pool(2, 2), head(2)], {}, x='int'),
    bcase('pool2x2_odd_endpad_linear_acc', 2, 11, 13, 8,
          [conv(16, 1, pads='valid', act=None, ints=True), pool(2, 2, pads=(0, 0, 1, 1)), head(2), head(1, input=1)], {}, x='int'),
    bcase('pool3x3_s1_p1_mask_acc', 1, 10, 9, 8, [conv(16, 1, pads='valid', ints=True), pool(3, 1, pads=(1, 1, 1, 1)), head(2),
                                                  head(1, input=1)], {}, x='int'),
    # --- L2Normalization backward: clamped branch (all-zero pixel), gamma gradient ---
    bcase('l2norm_linear_zero_pixel', 2, 8, 9, 16, [conv(32, 1, pads='valid', act=None), l2(), head(2)], {}, x='zero_pixel'),
    bcase('l2norm_mask_acc', 1, 9, 8, 16, [conv(24, 3), l2(), head(2), head(1, input=1)], {}),
    # --- BatchNormalization backward (bn_bwd_reduce_kernel + bn_bwd_apply_kernel): ELU, ReLU, none; C = 24 and 136 ---
    bcase('bn_elu24_relu136_none64', 2, 9, 10, 16, [conv(24, 3, act='elu', bn=True), conv(136, 3, bn=True), conv(64, 1, pads='valid',
                                                    act=None, bn=True), head(2)],
          {2: D(64, 0, 0), 3: D(160, 1, 0)}),
    bcase('bf16_bn_elu24_relu136', 1, 10, 9, 8, [conv(24, 3, act='elu', bn=True), conv(136, 3, bn=True), head(2)], {}, prec='bf16'),
    # --- heads: VOC width (25 columns per box) and generic; two heads with distinct prior offsets ---
    bcase('heads_voc25_two', 2, 8, 8, 64, [conv(64, 3), head(4), head(6, input=1)], {}, C=21),
    # --- single-pass bf16 (BN 64 / 128 / 256, native wgrad without the split, strided, direct, pool, l2norm) ---
    bcase('bf16_dgrad_native64', 2, 12, 12, 64, [conv(64, 3), conv(64, 3), head(2), head(3, input=1)],
          {2: dict(D(64, 1, 1), wgrad='native', wgrad_bn=64)}, prec='bf16'),
    bcase('bf16_dgrad128_native128', 1, 10, 10, 128, [conv(128, 3), conv(128, 3), head(2)],
          {2: dict(D(128, 1, 0), wgrad='native', wgrad_bn=128)}, prec='bf16'),
    bcase('bf16_dgrad256_head', 1, 8, 8, 64, [conv(264, 3), head(8, input=1)], {2: D(256, 1, 0)}, C=21, prec='bf16'),
    bcase('bf16_transposed_strided', 2, 13, 13, 8, [conv(16, 3), conv(64, 3, stride=2, pads=(1, 1, 1, 1)), head(2), head(2, input=1)],
          {1: dict(wgrad='transposed'), 2: dict(S(1, 1), wgrad='im2col')}, prec='bf16'),
    bcase('bf16_direct_pool_l2', 1, 12, 12, 3, [conv(16, 3), pool(2, 2), l2(), head(2), head(1, input=1)], {1: dict(wgrad='direct')},
          prec='bf16'),
]


# ------------------------------------------------------------------------------------------------------------------------------
# building a case
# ------------------------------------------------------------------------------------------------------------------------------
def _pads(spec, k):
    p = spec['pads']
    if p == 'same':
        q = spec['dil'] * (k - 1) // 2
        return (q, q, q, q)
    return (0, 0, 0, 0) if p == 'valid' else tuple(p)


def _build(case, seed=0):
    from ssd_keras_b200 import _ffi
    rng = np.random.default_rng(seed)
    C = case['C']
    chans, shapes, layers, info = {0: case['cin']}, {0: (case['H'], case['W'])}, [], {}
    P = 0
    for i, spec in enumerate(case['layers'], start=1):
        inp = i - 1 if spec['input'] is None else spec['input']
        cin, (H, W) = chans[inp], shapes[inp]
        op = spec['op']
        if op in ('conv', 'head'):
            k = spec.get('k', 3)
            pads = _pads(spec, k) if op == 'conv' else (1, 1, 1, 1)
            stride, dil = spec.get('stride', 1), spec.get('dil', 1)
            if op == 'conv':
                cout = spec['cout']
                if spec['ints']:
                    w = rng.integers(-1, 2, (k, k, cin, cout)).astype(np.float32)
                    b = np.zeros(cout, np.float32)
                else:
                    w = (rng.standard_normal((k, k, cin, cout)) * np.sqrt(2.0 / (k * k * cin))).astype(np.float32)
                    b = (rng.standard_normal(cout) * 0.1).astype(np.float32) if case['x'] != 'zero_pixel' else np.zeros(cout, np.float32)
                layers.append(dict(cout=cout, k=k, input=inp, stride=stride, dil=dil, pads=pads, act=spec['act'], kernel=w, bias=b))
                if spec['bn']:
                    layers[-1].update(bn_gamma=rng.uniform(0.5, 1.5, cout).astype(np.float32), bn_beta=(rng.standard_normal(cout) * 0.2).astype(np.float32),
                                      bn_mean=np.zeros(cout, np.float32), bn_var=np.ones(cout, np.float32))
                master = w
            else:
                nb = spec['nb']
                kc = (rng.standard_normal((3, 3, cin, nb * C)) * np.sqrt(2.0 / (9 * cin))).astype(np.float32)
                kl = (rng.standard_normal((3, 3, cin, nb * 4)) * np.sqrt(2.0 / (9 * cin))).astype(np.float32)
                bc, bl = (rng.standard_normal(nb * C) * 0.1).astype(np.float32), (rng.standard_normal(nb * 4) * 0.1).astype(np.float32)
                layers.append(dict(op=_ffi.OP_HEAD, input=inp, k=3, pads=pads, n_boxes=nb, kernel=kc, bias=bc, kernel2=kl, bias2=bl))
                cout = nb * (C + 4)
                master = np.concatenate([np.concatenate([kc[..., b * C:(b + 1) * C], kl[..., b * 4:(b + 1) * 4]], -1) for b in range(nb)], -1)
            Ho = (H + pads[0] + pads[2] - dil * (k - 1) - 1) // stride + 1
            Wo = (W + pads[1] + pads[3] - dil * (k - 1) - 1) // stride + 1
            info[i] = dict(op=op, input=inp, k=k, pads=pads, stride=stride, dil=dil, w=master, act=spec.get('act'),
                           bn_gamma=layers[-1].get('bn_gamma'), bn_beta=layers[-1].get('bn_beta'))
            if op == 'head':
                info[i].update(nb=spec['nb'], prior_off=P)
                P += Ho * Wo * spec['nb']
        elif op == 'pool':
            k, s_ = spec['k'], spec['stride']
            pads = tuple(spec['pads'])
            layers.append(dict(op=_ffi.OP_MAXPOOL, input=inp, k=k, stride=s_, pads=pads))
            cout = cin
            Ho, Wo = (H + pads[0] + pads[2] - k) // s_ + 1, (W + pads[1] + pads[3] - k) // s_ + 1
            info[i] = dict(op=op, input=inp, k=k, stride=s_, pads=pads)
        else:
            gamma = rng.uniform(0.5, 20.0, cin).astype(np.float32)
            layers.append(dict(op=_ffi.OP_L2NORM, input=inp, kernel=gamma))
            cout, (Ho, Wo) = cin, (H, W)
            info[i] = dict(op=op, input=inp, gamma=gamma)
        chans[i], shapes[i] = cout, (Ho, Wo)
        info[i].update(C=cout, H=Ho, W=Wo)
    g = cc.Graph(case['B'], case['H'], case['W'], case['cin'], layers, prec=case['prec'], n_classes=C,
                 anchors=np.zeros((P, 4), np.float32), training=True)
    if case['x'] == 'int':
        x = rng.integers(-2, 3, (case['B'], case['H'], case['W'], case['cin'])).astype(np.float32)
    else:
        x = rng.standard_normal((case['B'], case['H'], case['W'], case['cin'])).astype(np.float32)
        if case['x'] == 'zero_pixel':
            x[0, 1, 1] = 0.0
    return g, info, x, P


# ------------------------------------------------------------------------------------------------------------------------------
# the checks
# ------------------------------------------------------------------------------------------------------------------------------
def _judge(case, layer, what, got, ref, A, kappa_or_steps, store, perts, exact=False, use_kappa=False):
    """|got - ref| / bound <= 1, every perturbed reference > 1; logged."""
    if use_kappa:
        bnd = kappa_or_steps * A + opexact.UNIT[store] * np.abs(ref)
    else:
        bnd = opexact.bound(ref, A, kappa_or_steps, store)
    bnd = np.maximum(bnd, np.finfo(np.float64).tiny)
    got = np.asarray(got, np.float64)
    r = opexact.err_ratio(got, ref, bnd)
    rp = {str(k): opexact.err_ratio(got, v, bnd) for k, v in perts.items()}
    cc.log_ratio(dict(test='backward', case=case['name'], layer=layer, what=what, prec=case['prec'], ratio=r, perturbed=rp))
    assert r <= 1.0, (case['name'], layer, what, r)
    for k, v in rp.items():
        assert v > 1.0, (case['name'], layer, what, 'perturbation %s passes the bound' % k, v)
    if exact:
        assert np.array_equal(got, ref), (case['name'], layer, what, 'not bit-exact', float(np.abs(got - ref).max()))


def _vals(planes, inf):
    hi, lo = cc.interior(planes, inf['H'], inf['W'], inf['C'])
    return hi, lo


def _fval(planes, inf):
    hi, lo = _vals(planes, inf)
    return hi.astype(np.float64) + (0.0 if lo is None else lo)


def _span(g, layer, which):
    import ctypes
    from ssd_keras_b200 import _ffi
    off, cnt = ctypes.c_longlong(), ctypes.c_longlong()
    _ffi.check(_ffi.lib().ssdk_trainer_param_span(g.t, layer, which, ctypes.byref(off), ctypes.byref(cnt)))
    return (off.value, off.value + cnt.value) if cnt.value else None


def _relu_producer(info, pi):
    return pi in info and info[pi]['op'] == 'conv' and info[pi]['act'] == 'relu'


@pytest.mark.parametrize('case', BACKWARD_CASES, ids=[c['name'] for c in BACKWARD_CASES])
def test_backward_kernels_one_layer_at_a_time(case, monkeypatch):
    import torch
    for k, v in case['env'].items():
        monkeypatch.setenv(k, v)
    g, info, x, P = _build(case)
    try:
        n = len(case['layers']) + 1
        plans = {i: g.backward_plan(i) for i in range(n)}
        for i, exp in case['expect'].items():
            mins = {k[4:]: v for k, v in exp.items() if k.startswith('min_')}
            cc.assert_plan(plans[i], {k: v for k, v in exp.items() if not k.startswith('min_')}, '%s layer %d' % (case['name'], i))
            for k, v in mins.items():
                assert plans[i][k] >= v, (case['name'], i, k, plans[i])
        # the tensor input has no backward launches; a layer reading it has no data gradient; a native patch is 64 pixels
        assert plans[0]['wgrad'] is None and plans[0]['dgrad'] is None, plans[0]
        for i in range(1, n):
            if info[i]['input'] == 0:
                assert plans[i]['dgrad'] is None, (case['name'], i, plans[i])
            if plans[i]['wgrad'] == 'native':
                assert plans[i]['bw'] * plans[i]['bh'] == 64, (case['name'], i, plans[i])
        C = case['C']
        g.forward(x, width=C + 12)
        fwd = {i: g.read(i) for i in range(n)}
        # the stored planes each weight gradient multiplies (heads have none: their outputs are only an input of nothing)
        xplanes = {i: cc.interior(g.planes(i), *(fwd[i].shape[1:])) for i in range(n) if i == 0 or info[i]['op'] != 'head'}
        bn_z = {i: g.read_bn_input(i) for i in range(1, n) if info[i].get('bn_gamma') is not None}
        rng = np.random.default_rng(7)
        dy = rng.standard_normal((case['B'], P, C + 12)).astype(np.float32)
        dyt = torch.from_numpy(dy).cuda()
        mode, store = case['prec'], ('split' if case['prec'] == 'bf16x3' else 'bf16')
        written = set()
        for i in range(n - 1, 0, -1):
            inf = info[i]
            pi = inf['input']
            (pb, fb), (pa, fa) = g.step(i, dyt)
            touched_planes, touched_flat = set(), np.zeros(fa.shape, bool)
            if inf['op'] == 'head':
                touched_planes.add(i)
                rows = dy[:, inf['prior_off']:inf['prior_off'] + inf['H'] * inf['W'] * inf['nb']].reshape(
                    case['B'], inf['H'], inf['W'], inf['nb'], C + 12)
                ref, A, kap, perts = opexact.head_bwd_ref(fwd[i], rows, inf['nb'], C, perturb=[('dot',)])
                _judge(case, i, 'head_bwd', _fval(pa[i], inf), ref, A, kap, store, perts, use_kappa=True)
            if i in bn_z:
                # BatchNormalization backward, in place on the layer's gradient planes, before the conv's own launches read them
                touched_planes.add(i)
                pert = [('m1',), ('m2',)] + ([('elu1',)] if inf['act'] == 'elu' else [])
                ref, A, kap, dgam, dbet, Ag, Ab, kp, perts = opexact.bn_bwd_ref(bn_z[i], fwd[i], _fval(pb[i], inf), inf['bn_gamma'],
                                                                               act=inf['act'], perturb=pert)
                _judge(case, i, 'bn_bwd', _fval(pa[i], inf), ref, A, kap, store, perts, use_kappa=True)
                for which, r_, a_, what in ((3, dgam, Ag, 'bn_dgamma'), (4, dbet, Ab, 'bn_dbeta')):
                    sp = _span(g, i, which)
                    touched_flat[sp[0]:sp[1]] = True
                    _judge(case, i, what, fa[sp[0]:sp[1]], r_, a_, kp, 'f32', {}, use_kappa=True)
            if inf['op'] in ('conv', 'head'):
                plan = plans[i]
                dz = _vals(pa[i], inf)
                taps = inf['k'] * inf['k']
                geo = dict(stride=inf['stride'], dil=inf['dil'], pads=inf['pads'])
                # weight gradient
                sw, sb = _span(g, i, 0), _span(g, i, 1)
                touched_flat[sw[0]:sw[1]] = True
                touched_flat[sb[0]:sb[1]] = True
                got_w = fa[sw[0]:sw[1]].reshape(-1, inf['k'], inf['k'], info[pi]['C'] if pi in info else case['cin'])
                if plan['wgrad'] == 'direct':
                    ref, A, perts = opexact.wgrad_ref(xplanes[pi], dz, inf['k'], inf['k'], mode='fp32', perturb=[('tap', taps // 2)], **geo)
                    steps = inf['H'] * inf['W'] * case['B'] + 1
                else:
                    # one K block: a bw x bh patch of the native kernel; the first 64 output pixels of image 0 on the GEMM paths
                    blk = ('pixels', 0, 0, 0, plan['bh'], plan['bw']) if plan['wgrad'] == 'native' else ('first', 0, 64)
                    pert = [('tap', taps // 2), ('kblock', 0), blk] + ([('cross',)] if mode == 'bf16x3' else [])
                    ref, A, perts = opexact.wgrad_ref(xplanes[pi], dz, inf['k'], inf['k'], mode=mode, perturb=pert, **geo)
                    steps = opexact.n_steps_wgrad(plan, 3 if mode == 'bf16x3' else 1)
                _judge(case, i, 'wgrad_' + plan['wgrad'], got_w, ref, A, steps, 'f32', perts)
                rows_abs = np.abs(dz[0]).sum(axis=(2, 3))                 # drop the pixel row that carries the most gradient
                n_, y_ = np.unravel_index(int(np.argmax(rows_abs)), rows_abs.shape)
                ref, A, nb_, perts = opexact.bias_grad_ref(dz, perturb=[('row', int(n_), int(y_))])
                _judge(case, i, 'bias', fa[sb[0]:sb[1]], ref, A, nb_ + 1, 'f32', perts)
                # data gradient
                if plan['dgrad'] is not None:
                    pinf = info[pi]
                    touched_planes.add(pi)
                    assert plan['dgrad_accumulate'] == (pi in written) and plan['dgrad_mask'] == _relu_producer(info, pi), (plan, i)
                    mask = fwd[pi] if plan['dgrad_mask'] else None
                    old = _fval(pb[pi], pinf) if pi in written else None
                    kb = -(-pa[i][0].shape[-1] // 64)
                    pert = [('tap', taps // 2), ('kblock', taps // 2, (inf['C'] - 1) // 64)] + ([('cross',)] if mode == 'bf16x3' else [])
                    pert += ([('mask',)] if mask is not None else []) + ([('old',)] if old is not None else [])
                    ref, A, perts = opexact.dgrad_ref(dz, inf['w'], (pinf['H'], pinf['W']), mode=mode, mask=mask, old=old, perturb=pert, **geo)
                    _judge(case, i, 'dgrad_' + plan['dgrad'], _fval(pa[pi], pinf), ref, A, opexact.n_steps_dgrad(plan, taps, kb), store, perts)
                    written.add(pi)
            elif inf['op'] == 'pool':
                pinf = info[pi]
                touched_planes.add(pi)
                relu = _relu_producer(info, pi)
                old = _fval(pb[pi], pinf) if pi in written else None
                pert = [('last',)] + ([('mask',)] if relu else []) + ([('old',)] if old is not None else [])
                ref, A, steps, perts = opexact.pool_bwd_ref(fwd[pi], _fval(pa[i], inf), inf['k'], inf['k'], inf['stride'], inf['pads'][0],
                                                            inf['pads'][1], relu_mask=relu, old=old, perturb=pert)
                exact = inf['k'] == inf['stride'] and old is None and case['x'] == 'int'
                _judge(case, i, 'pool_bwd', _fval(pa[pi], pinf), ref, A, steps, store, perts, exact=exact)
                written.add(pi)
            elif inf['op'] == 'l2':
                pinf = info[pi]
                touched_planes.add(pi)
                relu = _relu_producer(info, pi)
                old = _fval(pb[pi], pinf) if pi in written else None
                pert = [('proj',)] + ([('mask',)] if relu else []) + ([('old',)] if old is not None else [])
                ref, A, kap, gref, gA, gsteps, perts = opexact.l2norm_bwd_ref(fwd[pi], _fval(pa[i], inf), inf['gamma'], relu_mask=relu,
                                                                            old=old, perturb=pert)
                if case['x'] == 'zero_pixel':
                    assert not np.any(fwd[pi][0, 1, 1]), 'the clamped branch needs an all-zero pixel'
                _judge(case, i, 'l2norm_bwd', _fval(pa[pi], pinf), ref, A, kap, store, perts, use_kappa=True)
                sg = _span(g, i, 2)
                touched_flat[sg[0]:sg[1]] = True
                _judge(case, i, 'l2norm_dgamma', fa[sg[0]:sg[1]], gref, gA, gsteps, 'f32', {})
                written.add(pi)
            # nothing else moved; borders and padding channels of every plane are zero
            for j in g.grad_layers:
                if j not in touched_planes:
                    for a, b in zip(pb[j][:2], pa[j][:2]):
                        assert (a is None and b is None) or np.array_equal(a, b), (case['name'], i, 'gradient of layer %d changed' % j)
                for o in cc.outside(pa[j], info[j]['H'], info[j]['W'], info[j]['C']):
                    assert not np.any(o), (case['name'], i, 'border / padding channels of layer %d gradient not zero' % j)
            assert np.array_equal(fb[~touched_flat], fa[~touched_flat]), (case['name'], i, 'parameter gradients outside the layer changed')
        # ssdk_trainer_read_grad unpacks the same planes
        for j in g.grad_layers:
            assert np.array_equal(g.read_grad(j), _fval(g.grad_planes(j), info[j]).astype(np.float32)), (case['name'], j)
    finally:
        g.close()
