"""GPU tests for the stand-alone layer calls ``ssdk_conv2d_fwd`` / ``ssdk_maxpool`` (SURVEY 8b) through ``ssd_keras_b200.ops``:
the same wgmma plan the model graphs use, run as a one-layer graph, against float64 torch-CPU references of the Keras layers
(``Conv2D`` / ``MaxPooling2D`` as used in models/keras_ssd300.py:274-335).  Tolerance of the bf16x3 convolution: 1e-4 of the
tensor's max magnitude (the bar of tests/test_gpu_model.py); max-pooling of bf16-exact inputs is exact."""
import numpy as np
import pytest

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
    assert 1e-4 < np.abs(y1 - ref).max() / np.abs(ref).max() < 5e-2          # one bf16 pass: ~3e-3, and really a different path
    with pytest.raises(ValueError):
        ops.conv2d(x, ker[:, :, :8], None)
    with pytest.raises(ValueError):
        ops.conv2d(x, ker, None, strides=2, padding='same')
    with pytest.raises(Exception):
        ops.conv2d(x, ker[..., :12], None)                                    # 12 output channels: not a multiple of 8


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
