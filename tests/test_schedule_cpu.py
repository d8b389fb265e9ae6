"""Host logic of the two-stream schedule of inference plans (csrc/model.cu: overlap_assign, exported as ssdk_schedule_preview), on the
launch grids of an SSD300 batch-32 plan on a 148-SM device and on edge cases.  No device needed."""
import ctypes as C

import numpy as np
import pytest

from ssd_keras_b200 import _ffi

# (name, kind, grid, input): kind 0 = pool / L2Norm / input, 1 = trunk convolution, 2 = predictor head
SSD300_B32 = [
    ('input', 0, 0, None), ('conv1_1', 1, 1 << 30, 'input'), ('conv1_2', 1, 148, 'conv1_1'), ('pool1', 0, 0, 'conv1_2'),
    ('conv2_1', 1, 148, 'pool1'), ('conv2_2', 1, 148, 'conv2_1'), ('pool2', 0, 0, 'conv2_2'),
    ('conv3_1', 1, 148, 'pool2'), ('conv3_2', 1, 148, 'conv3_1'), ('conv3_3', 1, 148, 'conv3_2'), ('pool3', 0, 0, 'conv3_3'),
    ('conv4_1', 1, 148, 'pool3'), ('conv4_2', 1, 148, 'conv4_1'), ('conv4_3', 1, 148, 'conv4_2'), ('pool4', 0, 0, 'conv4_3'),
    ('conv5_1', 1, 148, 'pool4'), ('conv5_2', 1, 148, 'conv5_1'), ('conv5_3', 1, 148, 'conv5_2'), ('pool5', 0, 0, 'conv5_3'),
    ('fc6', 1, 148, 'pool5'), ('fc7', 1, 148, 'fc6'),
    ('conv6_1', 1, 110, 'fc7'), ('conv6_2', 1, 50, 'conv6_1'), ('conv7_1', 1, 36, 'conv6_2'), ('conv7_2', 1, 7, 'conv7_1'),
    ('conv8_1', 1, 13, 'conv7_2'), ('conv8_2', 1, 7, 'conv8_1'), ('conv9_1', 1, 7, 'conv8_2'), ('conv9_2', 1, 3, 'conv9_1'),
    ('conv4_3_norm', 0, 0, 'conv4_3'),
    ('conv4_3_norm_mbox', 2, 148, 'conv4_3_norm'), ('fc7_mbox', 2, 110, 'fc7'), ('conv6_2_mbox', 2, 36, 'conv6_2'),
    ('conv7_2_mbox', 2, 13, 'conv7_2'), ('conv8_2_mbox', 2, 7, 'conv8_2'), ('conv9_2_mbox', 2, 3, 'conv9_2'),
]


def preview(layers, R, sms=148):
    names = [l[0] for l in layers]
    n = len(layers)
    kind = (C.c_int * n)(*[l[1] for l in layers])
    grid = (C.c_int * n)(*[l[2] for l in layers])
    inp = (C.c_int * n)(*[-1 if l[3] is None else names.index(l[3]) for l in layers])
    side = (C.c_ubyte * n)()
    frm, cap = C.c_int(), C.c_int()
    lib = _ffi.lib()
    lib.ssdk_schedule_preview.argtypes = [C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int, C.c_int,
                                          C.POINTER(C.c_ubyte), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.ssdk_schedule_preview.restype = C.c_int
    _ffi.check(lib.ssdk_schedule_preview(n, kind, grid, inp, R, sms, side, C.byref(frm), C.byref(cap)))
    return {names[i] for i in range(n) if side[i]}, (names[frm.value] if frm.value >= 0 else None), cap.value


def test_ssd300_batch32_default_split():
    side, frm, cap = preview(SSD300_B32, 0)                  # default R = 148 / 3 + 1 = 50
    assert frm == 'conv6_2' and cap == 148 - 50
    assert side == {'conv6_2', 'conv7_1', 'conv7_2', 'conv8_1', 'conv8_2', 'conv9_1', 'conv9_2',
                    'conv6_2_mbox', 'conv7_2_mbox', 'conv8_2_mbox', 'conv9_2_mbox'}
    # the wide heads (and the L2Normalization in front of one) stay on the caller's stream
    assert not side & {'conv4_3_norm', 'conv4_3_norm_mbox', 'fc7_mbox', 'conv6_1'}


def test_ssd300_batch32_other_reserves():
    side, frm, cap = preview(SSD300_B32, 37)
    assert frm == 'conv7_1' and cap == 148 - 36 and 'conv6_2' not in side and 'conv6_2_mbox' in side
    side, frm, cap = preview(SSD300_B32, 14)
    assert frm == 'conv7_2' and cap == 148 - 13 and 'conv6_2_mbox' not in side and 'conv7_2_mbox' in side
    side, frm, cap = preview(SSD300_B32, 120)               # the fc7 head turns narrow too, the conv4_3 head keeps 38 SMs
    assert frm == 'conv6_1' and cap == 148 - 110 and 'fc7_mbox' in side and 'conv4_3_norm_mbox' not in side


def test_no_split_when_nothing_can_overlap():
    # every GEMM wide: single stream
    wide = [(n, k, 148 if k else 0, i) for n, k, g, i in SSD300_B32]
    assert preview(wide, 0) == (set(), None, 0)
    # every GEMM narrow (tiny batch): nothing wide is left to run next to the narrow launches
    small = [(n, k, (min(g, 40) if 0 < g < (1 << 30) else g), i) for n, k, g, i in SSD300_B32]
    assert preview(small, 0) == (set(), None, 0)
    # a trunk that ends wide
    assert preview(SSD300_B32[:21], 0) == (set(), None, 0)


def test_elementwise_consumer_follows_a_narrow_producer():
    layers = [('input', 0, 0, None), ('c1', 1, 148, 'input'), ('c2', 1, 20, 'c1'), ('p2', 0, 0, 'c2'), ('n2', 0, 0, 'p2'),
              ('h1', 2, 148, 'c1'), ('h2', 2, 20, 'n2')]
    side, frm, cap = preview(layers, 50)
    assert frm == 'c2' and side == {'c2', 'p2', 'n2', 'h2'} and cap == 128


def test_bad_arguments():
    lib = _ffi.lib()
    assert hasattr(lib, 'ssdk_schedule_preview')
    with pytest.raises(Exception):
        preview([('a', 0, 0, None), ('b', 3, 1, 'a')], 0)
