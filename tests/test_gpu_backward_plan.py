"""GPU tests of the backward plan of a graph with a tensor input: tensor -> c1 -> c2 -> head, and a second head on c1.

ssdk_trainer_layer_plan must report the paths the plan builder documents -- the native weight-gradient kernel for stride-1
layers, the per-tap transposed GEMMs under SSDK_WGRAD_TRANSPOSED=1, the im2col GEMM and the strided data gradient (GEMM +
col2im) for stride 2, the ReLU mask of a ReLU producer and accumulation into a gradient that a second consumer already wrote.

The backward pass then runs from a caller's dL/dy_pred (ssdk_train_backward_dy) that is zero on the class columns and random on
the box offsets.  The softmax backward then passes dy through exactly, so the weight gradient of the head on c2 is a single
GEMM of known operands: c2's stored output and split(dy).  It is compared with the operand-exact float64 reference and bound of
oracle/opexact.py (native and transposed weight-gradient kernels), and a reference without one 8x8 pixel patch of one image
must fail that bound."""
import ctypes

import numpy as np
import pytest

import conv_cases as cc
from oracle import opexact
from ssd_keras_b200._ffi import OP_HEAD

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


B, H, W, CIN, C, NB = 2, 19, 19, 16, 21, 4


def _graph(stride, env, monkeypatch):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(0)
    cin, nb = CIN, NB

    def ker(k, ci, co):
        return (rng.standard_normal((k, k, ci, co)) * np.sqrt(2.0 / (k * k * ci))).astype(np.float32)

    def head(inp, ci):
        return dict(op=OP_HEAD, input=inp, k=3, pads=(1, 1, 1, 1), n_boxes=nb, kernel=ker(3, ci, nb * C), bias=np.zeros(nb * C, np.float32),
                    kernel2=ker(3, ci, nb * 4), bias2=np.zeros(nb * 4, np.float32))
    layers = [
        dict(cout=64, k=3, pads=(1, 1, 1, 1), act='relu', kernel=ker(3, cin, 64), bias=np.zeros(64, np.float32)),     # 1
        dict(cout=128, k=3, stride=stride, pads=(1, 1, 1, 1), act='relu', kernel=ker(3, 64, 128),                     # 2
             bias=np.zeros(128, np.float32)),
        head(2, 128),                                                                                                 # 3
        head(1, 64),                                                                                                  # 4
    ]
    Ho = (H + 2 - 3) // stride + 1
    P = (Ho * Ho + H * W) * nb
    return cc.Graph(B, H, W, cin, layers, n_classes=C, anchors=np.zeros((P, 4), np.float32), training=True)


@pytest.mark.parametrize('name,stride,env,wgrad', [
    ('native', 1, {}, 'native'),
    ('transposed', 1, {'SSDK_WGRAD_TRANSPOSED': '1'}, 'transposed'),
    ('strided', 2, {}, 'im2col'),
])
def test_trainer_layer_plan_reports_backward_paths(name, stride, env, wgrad, monkeypatch):
    g = _graph(stride, env, monkeypatch)
    try:
        c1, c2, h2 = g.backward_plan(1), g.backward_plan(2), g.backward_plan(3)
        assert g.backward_plan(0)['wgrad'] is None and g.backward_plan(0)['dgrad'] is None
        _check_head_weight_gradient(g, h2, name)
    finally:
        g.close()
    assert c2['wgrad'] == wgrad, c2
    if wgrad == 'native':
        assert c2['bw'] * c2['bh'] == 64 and c2['wgrad_bn'] in (64, 128) and c2['a_boxes'] >= 1, c2
    elif wgrad == 'transposed':
        assert c2['n_gemms'] == 9, c2
    else:
        assert c2['n_gemms'] == 1, c2
    # c2's data gradient lands in c1's gradient, which the head on c1 (layer 4, differentiated first) already holds
    assert c2['dgrad'] == ('strided' if stride == 2 else 'gemm') and c2['dgrad_mask'] == 1, c2
    if stride == 1:
        assert c2['dgrad_bn'] == 64 and c2['dgrad_accumulate'] == 1, c2
    # the head on c2: 128 input channels, the only consumer of c2
    assert h2['dgrad'] == 'gemm' and h2['dgrad_bn'] == 128 and h2['dgrad_mask'] == 1 and h2['dgrad_accumulate'] == 0, h2
    # c1 reads the graph's tensor input, which has no gradient; with 16 input channels (the native kernel takes multiples of 64)
    # its weight gradient runs on transposed operands
    assert c1['dgrad'] is None and c1['wgrad'] == 'transposed' and c1['n_gemms'] == 9, c1


def _check_head_weight_gradient(g, plan, name):
    import torch
    from ssd_keras_b200 import _ffi
    L = _ffi.lib()
    rng = np.random.default_rng(1)
    x = rng.standard_normal((B, H, W, CIN)).astype(np.float32)
    g.forward(x, width=C + 12)
    dy = np.zeros((B, g.P, C + 12), np.float32)
    dy[:, :, C:C + 4] = rng.standard_normal((B, g.P, 4))
    dyt = torch.from_numpy(dy).cuda()
    _ffi.check(L.ssdk_train_backward_dy(g.t, _ffi.dptr(dyt), _ffi.stream_ptr()))
    torch.cuda.synchronize()
    off, cnt = ctypes.c_longlong(), ctypes.c_longlong()
    _ffi.check(L.ssdk_trainer_param_span(g.t, 3, 0, ctypes.byref(off), ctypes.byref(cnt)))
    dw = g.grad[off.value:off.value + cnt.value].cpu().numpy().reshape(NB * (C + 4), 3, 3, 128)     # (cout, kh, kw, cin)
    # c2's stored output is the kernel's X operand.  Splitting hi + lo again can trade half an ulp between the planes where lo
    # is a tie (same value); that moves the omitted lo*lo product by 2**-16 of one product in ~0.1 % of them, far below kappa.
    X = g.read(2)
    Ho, Wo = X.shape[1], X.shape[2]
    dz = dy[:, :Ho * Wo * NB, C:C + 4].reshape(B, Ho, Wo, NB * 4)  # the head on c2 owns the first priors
    loc = np.array([b * (C + 4) + C + j for b in range(NB) for j in range(4)])
    conf = np.setdiff1d(np.arange(NB * (C + 4)), loc)
    assert not np.any(dw[conf]), 'class columns with a zero gradient must have a zero weight gradient'
    xh, xl = opexact.split(X)
    dh, dl = opexact.split(dz)

    def wgrad(terms, mask=1.0):
        """sum over pixels of pad(x)[tap window] * dz -> (cout, kh, kw, cin), float64"""
        out = np.zeros((NB * 4, 3, 3, 128))
        for xo, d in terms:
            xp = np.pad(xo.astype(np.float64), ((0, 0), (1, 1), (1, 1), (0, 0)))
            d = d.astype(np.float64) * mask
            for kh in range(3):
                for kw in range(3):
                    out[:, kh, kw] += np.einsum('bhwc,bhwo->oc', xp[:, kh:kh + Ho, kw:kw + Wo], d)
        return out
    terms = [(xh, dh), (xh, dl), (xl, dh)]
    ref = wgrad(terms)
    A = wgrad([(np.abs(a), np.abs(d)) for a, d in terms])
    patch = np.ones((B, Ho, Wo, 1))
    patch[0, :8, :8] = 0                                           # one 64-pixel patch of image 0
    pert = wgrad(terms, patch)
    # every 16 pixels of the padded grid (row pitch rounded up to 8) are one k-step, three products each with split operands;
    # the k_split partial sums meet in fp32 atomics
    n_steps = 3 * -(-B * (Ho + 2) * (Wo + 9) // 16) + plan['k_split'] + 1
    bnd = opexact.bound(ref, A, n_steps, 'f32')
    got = dw[loc]
    r, rp = opexact.err_ratio(got, ref, bnd), opexact.err_ratio(got, pert, bnd)
    cc.log_ratio(dict(test='wgrad', case=name, wgrad=plan['wgrad'], bn=plan['wgrad_bn'], ratio=r, perturbed={'patch': rp}))
    assert r <= 1.0, (name, r)
    assert rp > 1.0, (name, rp)
