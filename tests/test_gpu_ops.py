"""GPU tests of the convolution kernels and of the stand-alone layer calls (SURVEY 8b).

Convolutions: every case of tests/conv_cases.py FORWARD_CASES is a one-layer graph whose plan must be the variant the case
declares (ssdk_model_layer_plan).  Its output is compared element by element with the operand-exact float64 reference of
oracle/opexact.py: the same bf16 hi / lo split products the kernel issues, with the bound kappa * A + unit * |y_ref| derived
there (fp32 accumulation plus the output store).  The same comparison is repeated against perturbed references -- a dropped
cross term, tap, 64-channel k-block or bias -- and each of these must fail, so the bound is tight enough to see a stale ring
stage or a lost K range.  Set SSDK_KERNEL_ERRORS_LOG to a file name to record every measured ratio (tests/conv_cases.py).

``CASES`` below is kept as a check of the ``ops.conv2d`` API (argument handling, padding modes, the one-layer plan it builds
and destroys) against plain float64 convolutions at 1e-4 of the tensor's max; the kernels themselves are held to the
operand-exact bound above.  Max-pooling of bf16-exact inputs is exact."""
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


def _ref_conv(x, k, b, stride, dil, pads, act):
    import torch
    import torch.nn.functional as F
    pt, pl, pb, pr = pads
    xt = torch.from_numpy(x.astype(np.float64)).permute(0, 3, 1, 2)
    xt = F.pad(xt, (pl, pr, pt, pb))
    w = torch.from_numpy(k.astype(np.float64)).permute(3, 2, 0, 1)
    y = F.conv2d(xt, w, None if b is None else torch.from_numpy(b.astype(np.float64)), stride=stride, dilation=dil)
    if act == 'relu':
        y = F.relu(y)
    elif act == 'elu':
        y = F.elu(y)
    return y.permute(0, 2, 3, 1).numpy()


@pytest.mark.parametrize('case', cc.FORWARD_CASES, ids=[c['name'] for c in cc.FORWARD_CASES])
def test_conv_kernel_variant_within_operand_exact_bound(case, monkeypatch):
    import torch
    for k, v in case['env'].items():
        monkeypatch.setenv(k, v)
    x, w, b, scale, shift = cc.case_data(case, seed=sum(map(ord, case['name'])))
    layer = dict(cout=case['cout'], k=case['k'], stride=case['stride'], dil=case['dil'], pads=case['pads'], act=case['act'],
                 kernel=w, bias=b, bn_scale=scale, bn_shift=shift)
    g = cc.Graph(case['B'], case['H'], case['W'], case['cin'], [layer], prec=case['prec'])
    try:
        plan = g.plan(1)
        cc.assert_plan(plan, case['expect'], case['name'])
        if case['persistent']:
            units = plan['n_tiles_m'] * plan['n_tiles_n'] * plan['k_split']
            sms = torch.cuda.get_device_properties(0).multi_processor_count
            assert plan['grid'] == sms and units >= 3 * sms, (plan, sms)
            nk = case['k'] * case['k'] * plan['kblocks']
            assert (nk < plan['stages']) if case['persistent'] == 'nk<stages' else (nk % plan['stages'] != 0), (nk, plan)
        g.forward(x)
        x_st = g.read(0)                                # the input as conv_direct_kernel reads it (hi + lo, or hi)
        y = g.read(1)
    finally:
        g.close()
    mode = 'fp32' if plan['kernel'] == 'direct' else case['prec']
    if mode != 'fp32':
        x_st = x                                        # the tensor-core kernels read split(x): split the input itself
    geo = dict(stride=case['stride'], dil=case['dil'], pads=case['pads'], mode=mode, act=case['act'], bn_scale=scale, bn_shift=shift)
    taps = case['k'] * case['k']
    y_ref, A, pert = opexact.conv_ref(x_st, w, b, perturb=cc.perturbations(plan, taps, case['cin'], mode == 'bf16x3', b), **geo)
    n_steps = cc.n_steps_of(plan, taps, case['cin'])
    store = 'bf16' if case['prec'] == 'bf16' else 'split'
    bnd = opexact.bound(y_ref, A, n_steps, store)
    ratio = opexact.err_ratio(y, y_ref, bnd)
    perturbed = {p[0]: opexact.err_ratio(y, yp, bnd) for p, yp in pert.items()}
    cc.log_ratio(dict(test='forward', case=case['name'], kernel=plan['kernel'], bn=plan['bn'], split=plan['split'],
                      ratio=ratio, perturbed=perturbed))
    assert ratio <= 1.0, (case['name'], ratio)
    for k, r in perturbed.items():
        assert r > 1.0, '%s: the bound does not see a dropped %s (ratio %.3g)' % (case['name'], k, r)


CASES = [
    # B, H, W, Cin, Cout, k, stride, dil, padding, act, bias
    (2, 19, 23, 64, 128, 3, 1, 1, 'same', 'relu', True),        # the VGG layers' shape class
    (2, 20, 20, 3, 64, 3, 1, 1, 'same', 'relu', True),          # image-facing layer (gathered A tile)
    (1, 10, 12, 16, 32, 1, 1, 1, 'valid', None, False),         # 1x1, no bias, linear
    (2, 19, 19, 32, 64, 3, 2, 1, (1, 1, 1, 1), 'relu', True),   # ZeroPadding2D(1) + 'valid' stride 2 (conv6_2 ... conv7_2)
    (1, 19, 19, 64, 256, 3, 1, 6, 'same', 'relu', True),        # fc6: dilation 6
    (1, 7, 7, 128, 256, 3, 1, 1, 'valid', 'elu', True),         # 'valid' 3x3 (conv8_2 / conv9_2), ELU
    (1, 9, 9, 24, 40, 3, 1, 1, 'same', None, True),             # channel counts that are not multiples of 64 / 16
]


@pytest.mark.parametrize('idx', range(len(CASES)))
def test_conv2d_matches_float64_reference(idx):
    case = CASES[idx]
    from ssd_keras_b200 import ops
    B, H, W, Cin, Cout, k, stride, dil, padding, act, has_bias = case
    rng = np.random.default_rng(100 + idx)
    x = rng.standard_normal((B, H, W, Cin)).astype(np.float32)
    ker = (rng.standard_normal((k, k, Cin, Cout)) * np.sqrt(2.0 / (k * k * Cin))).astype(np.float32)
    b = (rng.standard_normal(Cout) * 0.1).astype(np.float32) if has_bias else None
    y = ops.conv2d(x, ker, b, strides=stride, padding=padding, dilation_rate=dil, activation=act).cpu().numpy()
    if padding == 'same':
        p = dil * (k - 1) // 2
        pads = (p, p, p, p)
    elif padding == 'valid':
        pads = (0, 0, 0, 0)
    else:
        pads = padding
    ref = _ref_conv(x, ker, b, stride, dil, pads, act)
    assert y.shape == ref.shape
    err = np.abs(y - ref).max() / np.abs(ref).max()
    assert err < 1e-4, err


def test_conv2d_single_pass_mode_and_errors():
    from ssd_keras_b200 import ops
    rng = np.random.default_rng(3)
    x = rng.standard_normal((1, 8, 8, 16)).astype(np.float32)
    ker = (rng.standard_normal((3, 3, 16, 32)) * 0.1).astype(np.float32)
    y3 = ops.conv2d(x, ker, None).cpu().numpy()
    y1 = ops.conv2d(x, ker, None, precision='bf16').cpu().numpy()
    ref = _ref_conv(x, ker, None, 1, 1, (1, 1, 1, 1), None)
    assert np.abs(y3 - ref).max() / np.abs(ref).max() < 1e-4
    assert np.abs(y1 - ref).max() / np.abs(ref).max() > 1e-4                  # one bf16 pass is really a different path
    with pytest.raises(ValueError):
        ops.conv2d(x, ker[:, :, :8], None)
    with pytest.raises(ValueError):
        ops.conv2d(x, ker, None, strides=2, padding='same')
    with pytest.raises(Exception):
        ops.conv2d(x, ker[..., :12], None)                                    # 12 output channels: not a multiple of 8
    # a NaN weight of the image-facing layer whose payload lies in the low 16 bits stays NaN in its bf16 weight image (not Inf);
    # no activation: ReLU would turn the NaN into 0
    x3 = rng.standard_normal((1, 9, 10, 3)).astype(np.float32)
    k3 = (rng.standard_normal((3, 3, 3, 16)) * 0.1).astype(np.float32)
    k3.view(np.uint32)[1, 1, 2, 5] = 0x7f800001                             # centre tap: reaches every output pixel
    g = cc.Graph(1, 9, 10, 3, [dict(cout=16, k=3, pads=(1, 1, 1, 1), act=None, kernel=k3)], prec='bf16')
    try:
        cc.assert_plan(g.plan(1), dict(kernel='first_tc', split=0), 'nan_weight')
        g.forward(x3)
        y3 = g.read(1)
    finally:
        g.close()
    assert np.isnan(y3[..., 5]).all() and not np.isinf(y3).any()
    assert np.isfinite(np.delete(y3, 5, axis=-1)).all()


@pytest.mark.parametrize('shape,pool,stride,padding', [
    ((2, 75, 75, 64), 2, 2, 'same'),          # pool3 of SSD300: odd extent, TensorFlow 'same' (75 -> 38)
    ((2, 20, 20, 128), 2, 2, 'valid'),
    ((1, 19, 19, 512), 3, 1, 'same'),         # pool5
    ((1, 13, 11, 24), 3, 2, 'valid'),
])
def test_max_pool2d_is_exact_on_bf16_exact_inputs(shape, pool, stride, padding):
    import torch
    import torch.nn.functional as F
    from ssd_keras_b200 import ops
    from ssd_keras_b200.models._graph import tf_same_pool_pad
    rng = np.random.default_rng(sum(shape))
    x = rng.integers(-120, 120, size=shape).astype(np.float32)
    y = ops.max_pool2d(x, pool, stride, padding).cpu().numpy()
    xt = torch.from_numpy(x).permute(0, 3, 1, 2)
    if padding == 'same':
        (pt, pb), (pl, pr) = tf_same_pool_pad(shape[1], pool, stride), tf_same_pool_pad(shape[2], pool, stride)
        xt = F.pad(xt, (pl, pr, pt, pb), value=float('-inf'))
    ref = F.max_pool2d(xt, pool, stride).permute(0, 2, 3, 1).numpy()
    assert y.shape == ref.shape and np.array_equal(y, ref)
