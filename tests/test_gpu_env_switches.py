"""The library's environment switches (the table above ssdk::env_int in csrc/common.cuh) take whole decimal integers: anything
else is refused under the variable's name, and a switch that turns a path off or on does so by its value, not by being set."""
import numpy as np
import pytest

import conv_cases as cc
import decode_cases as dc
import encode_cases as ec

pytestmark = pytest.mark.gpu

SWITCHES = ('SSDK_ENC_TPC', 'SSDK_NMS_TWO_STAGE', 'SSDK_OVERLAP', 'SSDK_NO_HEAD_FUSION')


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


@pytest.fixture
def env(monkeypatch):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    return monkeypatch


def encode():
    import torch
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    cfg = ec.golden_configs()['ssd300']
    gts = ec.gen_random(80, 2, 5, cfg)
    offs = np.cumsum([0] + [g.shape[0] for g in gts]).astype(np.int32)
    y = SSDInputEncoder(**cfg).encode_device(torch.from_numpy(np.concatenate(gts)).cuda(), offs)
    torch.cuda.synchronize()
    return y


def decode():
    import torch
    from ssd_keras_b200.ssd_encoder_decoder.ssd_output_decoder import FAST, PER_CLASS, decode_device
    c = dc.CASES[0]
    y = torch.from_numpy(np.ascontiguousarray(dc.inputs(c['name']))).cuda()
    out = decode_device(y, FAST if c['fast'] else PER_CLASS, c['api'] == 'layer', c['conf'], c['iou'], c['top_k'], c['cap'],
                        c['coords'], c['norm'], c['H'], c['W'], c['border'])
    torch.cuda.synchronize()
    return out


def head_graph():
    """An inference plan of a tensor input and one predictor head that the default plan fuses (Pascal VOC's 25-column boxes)."""
    from ssd_keras_b200 import _ffi
    B, H, W, cin, nb, C = 2, 10, 9, 64, 4, 21
    rng = np.random.default_rng(81)
    layer = dict(op=_ffi.OP_HEAD, k=3, pads=(1, 1, 1, 1), n_boxes=nb,
                 kernel=rng.standard_normal((3, 3, cin, nb * C)).astype(np.float32), bias=np.zeros(nb * C, np.float32),
                 kernel2=rng.standard_normal((3, 3, cin, nb * 4)).astype(np.float32), bias2=np.zeros(nb * 4, np.float32))
    return cc.Graph(B, H, W, cin, [layer], n_classes=C, anchors=rng.uniform(0, 1, (H * W * nb, 4)).astype(np.float32))


def create_model():
    head_graph().close()


@pytest.mark.parametrize('name, value, call', [('SSDK_ENC_TPC', 'abc', encode), ('SSDK_NMS_TWO_STAGE', 'yes', decode),
                                               ('SSDK_OVERLAP', 'on', create_model)])
def test_malformed_switch_is_refused(env, name, value, call):
    env.setenv(name, value)
    with pytest.raises(ValueError, match=name):
        call()
    env.delenv(name)
    call()


@pytest.mark.parametrize('value, fused', [('0', 1), ('1', 0)])
def test_no_head_fusion_by_value(env, value, fused):
    env.setenv('SSDK_NO_HEAD_FUSION', value)
    g = head_graph()
    try:
        assert g.plan(1)['head_fused'] == fused
    finally:
        g.close()
